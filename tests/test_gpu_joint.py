"""Refining one calibration from two recordings on the H100 (joint.refine_replays): two simulated 60 s Livox recordings of the same rig,
the extrinsic and the lag given to calib_sim explicitly, with different trajectory seeds. With one recording the joint search is
Replay.refine bit for bit; the joint trace at 1 and 4 replay jobs is the same, and with two GPUs visible, with the recordings on
different devices too; the report parses; the refined total lag is within 3 ms of the simulated one; the refined joint MME is at or
below every start candidate's. The extrinsic errors against the truth, beside each recording's own Replay.refine at the same budget, the
axis lines and the wall time per candidate are printed, not asserted."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import _build, assess, host, joint, refine  # noqa: E402

SECONDS = 60.0
SEEDS = (0, 1)
T_OFF = 0.013
T_TRUE = np.array([-0.02, 0.03, 0.15])
BUDGET = 30      # joint candidates
JOBS = 4


def _r_true():
    import calib_sim
    return calib_sim._rot(2, 1.5) @ calib_sim._rot(1, -0.03) @ calib_sim._rot(0, 0.02)


def _events(seed, seconds=SECONDS):
    """test_bag_node.livox_events' scenario for one trajectory seed, with the extrinsic and the lag passed to calib_sim explicitly"""
    import calib_sim
    import lio_case
    import test_bag_node as tb
    from lidar_imu_init_b200 import scenes
    S = calib_sim.make_streams(seed=seed, duration=seconds, t_off=T_OFF, R_LI=_r_true(), T_LI=T_TRUE)
    path = lio_case.TruePath(seed, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    ev, k_imu = [], 0
    for k in range(int(seconds * 10) - 1):
        stamp = path.t0 + 0.1 * k
        m = scenes.livox_message(scene, path.lidar, stamp, 20_000, seed=1000 + k, dup_frac=0.01, tie_frac=0.05, noise_frac=0.01,
                                 bad_line_frac=0.01)
        while k_imu < len(ti) and ti[k_imu] <= stamp + 0.13:
            ev.append(("imu", *tb.split_time(ti[k_imu]), (wi[k_imu], ai[k_imu])))
            k_imu += 1
        ev.append(("lidar", *tb.split_time(stamp), m))
    return ev


def _play(tmp, b, device=0):
    import test_bag_node as tb
    from lidar_imu_init_b200 import run
    from lidar_imu_init_b200.node import Log
    bag = str(tmp / f"rec{b}.bag")
    if not os.path.exists(bag):
        tb.write_event_bag(bag, _events(SEEDS[b]), chunk_msgs=300)
    args = run.parse_args(["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", str(tmp / f"rec{b}_dev{device}"), "--device",
                           str(device), "--max-map-points", "3000000", "--refine"])
    nd, wall = run.play(args, Log(quiet=True))
    assert nd.replay.base is not None and nd.replay.info()["skipped"] == 0, f"recording {b} did not hand over"
    return nd


def _err(R, T):
    c = np.clip((np.trace(np.asarray(R) @ _r_true().T) - 1.0) / 2.0, -1.0, 1.0)
    return float(np.degrees(np.arccos(c))), float(np.linalg.norm(np.asarray(T) - T_TRUE)) * 1000.0


def _close(nd):
    nd.replay.close()
    nd.odom.g.close()


@pytest.fixture(scope="module")
def recs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("joint")
    tb.sim_config(tmp, online_refine_time=10.0)
    nodes = []
    seen = {"tmp": tmp, "nodes": nodes}
    try:
        for b in range(len(SEEDS)):
            nodes.append(_play(tmp, b))
        seen["finals"] = [host.state_pose(nd.odom.state)[2:] for nd in nodes]
        yield seen
    finally:
        for nd in nodes:
            _close(nd)


def _same_trace(a, b):
    assert [(r["stage"], r["R"].tobytes(), r["T"].tobytes(), r["shift_ms"]) for r in a["trace"]] == \
           [(r["stage"], r["R"].tobytes(), r["T"].tobytes(), r["shift_ms"]) for r in b["trace"]]
    assert [np.array(r["mmes"]).tobytes() for r in a["trace"]] == [np.array(r["mmes"]).tobytes() for r in b["trace"]]
    assert (a["status"], a["best"], a["start"], a["steps"], a["time_lag"]) == (b["status"], b["best"], b["start"], b["steps"], b["time_lag"])
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a["states"], b["states"]))
    assert str(a["axes"]) == str(b["axes"]) and str(a["axes_rec"]) == str(b["axes_rec"])


@pytest.mark.gpu
def test_one_recording_is_replay_refine(recs):
    rp, (R_fin, T_fin) = recs["nodes"][0].replay, recs["finals"][0]
    s = rp.refine(R_fin, T_fin, max_replays=8, jobs=JOBS)
    j = joint.refine_replays([rp], [(R_fin, T_fin)], 8, JOBS)
    lab = {"final:0": "final", "li-init:0": "li-init"}
    assert [(lab.get(r["stage"], r["stage"]), r["R"].tobytes(), r["T"].tobytes(), r["shift_ms"], np.float64(r["mme"]).tobytes())
            for r in j["trace"]] == [(r["stage"], r["R"].tobytes(), r["T"].tobytes(), r["shift_ms"], np.float64(r["mme"]).tobytes())
                                     for r in s["trace"]]
    assert (j["status"], j["best"], lab[j["start"]], j["steps"], j["time_lag"]) == (s["status"], s["best"], s["start"], s["steps"], s["time_lag"])
    assert j["states"][0].tobytes() == s["state"].tobytes() and str(j["axes"]) == str(s["axes"])


@pytest.mark.gpu
def test_joint_refinement(recs):
    nodes, finals = recs["nodes"], recs["finals"]
    rps = [nd.replay for nd in nodes]
    t0 = time.perf_counter()
    seq = joint.refine_replays(rps, finals, BUDGET, 1)
    t_seq = time.perf_counter() - t0
    t0 = time.perf_counter()
    par = joint.refine_replays(rps, finals, BUDGET, JOBS)
    t_par = time.perf_counter() - t0
    _same_trace(seq, par)
    recs["par"] = par
    n = len(par["trace"])
    print(f"joint refinement of {len(rps)} recordings, {n} candidates ({n * len(rps)} replays, {par['status']}): 1 job {t_seq:.1f} s "
          f"({t_seq / n:.2f} s per candidate), {JOBS} jobs {t_par:.1f} s ({t_par / n:.2f} s per candidate)", flush=True)
    recs_txt = [dict(bag=f"rec{b}", subframes=rp.info()["frames"], skipped=rp.info()["skipped"], lag=rp.lag, R_init=rp.res["R_LI"],
                     T_init=rp.res["T_LI"], R_final=R, T_final=T) for b, (rp, (R, T)) in enumerate(zip(rps, finals))]
    text = assess.joint_report_text(recs_txt, par, nodes[0].assess.radius, nodes[0].assess.min_neighbors)
    print(text, flush=True)
    rep = assess.parse_joint_report(text)
    assert rep["header"]["candidates"] == n <= BUDGET and len(rep["rows"]) == n and len(rep["result"]) == len(rps)
    assert list(rep["axes"]) == ["joint", 0, 1]
    print(f"lags at the hand-over {[round(x * 1000, 3) for x in par['lags']]} ms, L0 {par['lag0'] * 1000:.3f} ms, refined "
          f"{par['time_lag'] * 1000:.3f} ms, simulated {T_OFF * 1000:.3f} ms", flush=True)
    assert abs(par["time_lag"] - T_OFF) < 0.003
    starts = [r for r in par["trace"] if r["stage"].startswith(("final:", "li-init:"))]
    assert len(starts) == 2 * len(rps) and all(par["mme"] <= r["mme"] for r in starts)
    e = _err(par["R"], par["T"])
    print(f"joint: {e[0]:.4f} deg, {e[1]:.2f} mm from the truth", flush=True)
    for b, (rp, (R, T)) in enumerate(zip(rps, finals)):
        t0 = time.perf_counter()
        own = rp.refine(R, T, max_replays=BUDGET, jobs=JOBS)
        e, ef = _err(own["R"], own["T"]), _err(R, T)
        print(f"recording {b}: own Replay.refine at {BUDGET} replays ({own['status']}, {time.perf_counter() - t0:.1f} s): {e[0]:.4f} deg, "
              f"{e[1]:.2f} mm, lag {own['time_lag'] * 1000:.3f} ms; final {ef[0]:.4f} deg, {ef[1]:.2f} mm; axes "
              f"{ {k: refine.axis_verdict(dp, dm) for k, (_, dp, dm) in own['axes'].items()} }", flush=True)


@pytest.mark.gpu
def test_recordings_on_two_devices(recs):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    if "par" not in recs:
        pytest.skip("the joint refinement on one device did not run")
    nd1 = _play(recs["tmp"], 1, device=1)
    try:
        assert nd1.odom.g.device_id == 1
        two = joint.refine_replays([recs["nodes"][0].replay, nd1.replay], [recs["finals"][0], host.state_pose(nd1.odom.state)[2:]],
                                   BUDGET, JOBS)
        assert all(w.device_id == 1 for w in nd1.replay.workers)
        _same_trace(two, recs["par"])
    finally:
        _close(nd1)
