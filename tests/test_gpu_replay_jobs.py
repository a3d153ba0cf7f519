"""Concurrent replays on the H100, on the 60 s Livox scenario of tests/test_gpu_refine.py, with the contexts driven from real threads: the
native loop replaying the run's own hand-over reproduces every posterior state and the as-run MME bit for bit; Replay.sweep at jobs=4
is bit-equal to the sequential Python sweep, report lines included; Replay.refine(max_replays=30) at jobs=8 has the trace and the
refined result of the sequential search. The timings are printed, not asserted."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import _build, assess, host  # noqa: E402


def _same(a: dict, b: dict) -> bool:
    return a.keys() == b.keys() and all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)


@pytest.fixture(scope="module")
def run60(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("jobs")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {}

    def on_node(nd):
        seen["node"] = nd
        nd.odom.g.close = lambda: None              # kept open for the tests below; closed at teardown
        nd.replay = nd.odom.replay = assess.Replay(nd.odom.g, nd.assess)
    argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", str(tmp / "out"), "--max-map-points", "3000000", "--quiet", "--assess"]
    assert run.main(argv, on_node=on_node) == 0
    nd = seen["node"]
    a = nd.assess
    seen["as_run"] = nd.odom.g.assess_evaluate(radius=a.radius, min_neighbors=a.min_neighbors, as_run=True)
    yield seen
    nd.replay.close()
    capi.LiInitGpu.close(nd.odom.g)


@pytest.mark.gpu
def test_native_replay_of_the_run_is_bit_identical(run60):
    rp = run60["node"].replay
    assert rp.info()["skipped"] == 0 and len(rp.run_states) > 1000
    t0 = time.perf_counter()
    py = rp.run(frozen=False)
    t_py = time.perf_counter() - t0
    t0 = time.perf_counter()
    nat = rp.run_native(frozen=False)
    t_nat = time.perf_counter() - t0
    assert [j for j, _ in nat["states"]] == [j for j, _ in rp.run_states]
    assert all(a.tobytes() == b.tobytes() for (_, a), (_, b) in zip(nat["states"], rp.run_states))
    assert _same(nat["result"], run60["as_run"]) and _same(nat["result"], py["result"]) and nat["rms_m"] == 0.0
    print(f"one replay of the run's hand-over: Python loop {t_py:.2f} s, native loop {t_nat:.2f} s ({len(nat['states'])} updates)", flush=True)


@pytest.mark.gpu
def test_sweep_at_four_jobs_equals_the_sequential_sweep(run60):
    nd = run60["node"]
    rp = nd.replay
    _, _, R_fin, T_fin = host.state_pose(nd.odom.state)
    t0 = time.perf_counter()
    seq = rp.sweep(R_fin, T_fin)
    t_seq = time.perf_counter() - t0
    t0 = time.perf_counter()
    par = rp.sweep(R_fin, T_fin, jobs=4)
    t_par = time.perf_counter() - t0
    assert [r[0] for r in seq] == [r[0] for r in par]
    for (name, _, _, _, a), (_, _, _, _, b) in zip(seq, par):
        assert _same(a["result"], b["result"]), name
        assert a["R_LI"].tobytes() == b["R_LI"].tobytes() and a["T_LI"].tobytes() == b["T_LI"].tobytes(), name
        assert np.float64(a["rms_m"]).tobytes() == np.float64(b["rms_m"]).tobytes(), name
    info, a = rp.info(), rp.assessment
    text = [assess.replay_report_text(info, rp.snapshot_bytes, 0.0, a.radius, a.min_neighbors, rows) for rows in (seq, par)]
    assert text[0] == text[1]
    print(f"17-replay sweep: sequential Python {t_seq:.1f} s, 4 jobs {t_par:.1f} s", flush=True)


@pytest.mark.gpu
def test_refine_at_eight_jobs_equals_the_sequential_search(run60):
    nd = run60["node"]
    rp = nd.replay
    _, _, R_fin, T_fin = host.state_pose(nd.odom.state)
    t0 = time.perf_counter()
    a = rp.refine(R_fin, T_fin, max_replays=30)
    t_seq = time.perf_counter() - t0
    t0 = time.perf_counter()
    b = rp.refine(R_fin, T_fin, max_replays=30, jobs=8)
    t_par = time.perf_counter() - t0
    assert len(a["trace"]) == len(b["trace"]) == 30
    for x, y in zip(a["trace"], b["trace"]):
        assert (x["stage"], x["R"].tobytes(), x["T"].tobytes(), x["shift_ms"]) == (y["stage"], y["R"].tobytes(), y["T"].tobytes(), y["shift_ms"])
        assert _same(x["result"], y["result"])
    assert (a["status"], a["best"], a["start"], a["steps"]) == (b["status"], b["best"], b["start"], b["steps"])
    assert a["state"].tobytes() == b["state"].tobytes() and a["time_lag"] == b["time_lag"]
    assert str(a["axes"]) == str(b["axes"])
    print(f"refine at 30 replays: sequential Python {t_seq:.1f} s, 8 jobs {t_par:.1f} s ({len(rp.workers)} workers)", flush=True)
