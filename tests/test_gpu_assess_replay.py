"""The LIO-phase replay on the H100, on the 60 s Livox scenario of tests/test_gpu_bag.py (simulated lag 13 ms, tests/calib_sim.py):
`run --assess --assess-replay` writes a report that parses; replaying the run's own hand-over reproduces every LIO posterior state, the
final map and the as-run score bit for bit; a frozen replay keeps the candidate extrinsic bit for bit after every update; a gross error
scores a higher MME than the simulated truth. The findings (the truth against the final extrinsic, the lag around the run's) are printed,
not asserted."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import _build, assess, host  # noqa: E402


def _same(a: dict, b: dict) -> bool:
    return a.keys() == b.keys() and all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)


def _rows(xyz):
    """the points in lexicographic order of their bits"""
    b = np.ascontiguousarray(xyz, np.float32).view(np.uint32)
    return b[np.lexsort(b.T[::-1])]


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("assess_replay")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, path = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"S": path.S}

    def on_node(nd):
        g = nd.odom.g
        seen.update(g=g, node=nd)
        g.close = lambda: None                      # kept open for the tests below; closed at teardown
        real_write = nd.replay.write

        def write(p, R_final=None, T_final=None):   # the run's own map and score, before any replay changes them
            seen["map"] = g.map_download()
            seen["as_run"] = g.assess_evaluate(radius=nd.assess.radius, min_neighbors=nd.assess.min_neighbors, as_run=True)
            real_write(p, R_final, T_final)
        nd.replay.write = write
    out = str(tmp / "out")
    argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet", "--assess", "--assess-replay"]
    assert run.main(argv, on_node=on_node) == 0
    seen["out"] = out
    yield seen
    capi.LiInitGpu.close(seen["g"])


@pytest.mark.gpu
def test_report_parses(runs):
    text = open(os.path.join(runs["out"], "result", "assessment_replay.txt")).read()
    print(text, flush=True)
    rep = assess.parse_replay_report(text)
    rp = runs["node"].replay
    info = rp.info()
    assert rep["header"]["subframes"] == info["frames"] > 1000 and rep["header"]["skipped"] == 0
    assert len(rep["rows"]) == 17 and len(rep["axes"]) == 6
    assert rep["rows"]["run"]["rms_m"] == 0.0
    assert rep["rows"]["run"]["mme"] == pytest.approx(runs["as_run"]["mme"], abs=1e-9)
    for name, r in rep["rows"].items():
        if name != "run":   # frozen: the replay ends with its candidate
            assert (r["end_t_x"], r["end_t_y"], r["end_t_z"]) == (r["t_x"], r["t_y"], r["t_z"]), name


@pytest.mark.gpu
def test_replay_of_the_run_is_bit_identical(runs):
    """Every LIO posterior state, the final map's points and the as-run score of the run's own hand-over replayed, bit for bit."""
    rp, g = runs["node"].replay, runs["g"]
    r = rp.run(frozen=False)
    print(f"replay of the run: {len(r['states'])} updates in {r['seconds']:.2f} s", flush=True)
    assert len(r["states"]) == len(rp.run_states) > 1000
    bad = [j for (j, a), (k, b) in zip(r["states"], rp.run_states) if j != k or a.tobytes() != b.tobytes()]
    assert not bad, f"{len(bad)} updates differ, first at sub-frame {bad[0]}"
    # (the download lists the bricks in creation order, which the device's atomics do not fix from run to run: compared as point sets)
    got, want = g.map_download(), runs["map"]
    assert _rows(got).tobytes() == _rows(want).tobytes()
    assert _same(r["result"], runs["as_run"]), (r["result"], runs["as_run"])


@pytest.mark.gpu
def test_frozen_replay_keeps_the_candidate_and_tells_a_gross_error(runs):
    S = runs["S"]
    rp = runs["node"].replay
    R_true, T_true = np.asarray(S["R_LI"], float), np.asarray(S["T_LI"], float)
    true = rp.run(R_true, T_true, frozen=True)
    for _, s in true["states"]:
        assert s[12:21].tobytes() == R_true.reshape(9).tobytes() and s[21:24].tobytes() == T_true.tobytes()
    R_bad = assess.rot_exp([0.0, 0.0, np.radians(3.0)]) @ R_true
    T_bad = T_true + [0.10, 0.0, 0.0]
    bad = rp.run(R_bad, T_bad, frozen=True)
    for _, s in bad["states"]:
        assert s[12:21].tobytes() == R_bad.reshape(9).tobytes() and s[21:24].tobytes() == T_bad.tobytes()
    # the finding: the simulated truth against the run's final extrinsic and against LI-Init's, under replay
    rep = assess.parse_replay_report(open(os.path.join(runs["out"], "result", "assessment_replay.txt")).read())
    rows = rep["rows"]
    print(f"replay MME: truth {true['result']['mme']:.6f} (rms {true['rms_m']:.4f} m), final {rows['final']['mme']:.6f}, li-init "
          f"{rows['li-init']['mme']:.6f}, run {rows['run']['mme']:.6f}, gross {bad['result']['mme']:.6f}; lag -5 ms "
          f"{rows['lag-5']['mme']:.6f}, +5 ms {rows['lag+5']['mme']:.6f}; lag line {rep['lag']}", flush=True)
    assert bad["result"]["mme"] > true["result"]["mme"]
    # where the lag minimum sits: final and the truth at shifts from LI-Init's lag up to past the simulated one
    lag_run = float(rp.res["time_lag_1"]) + float(rp.res["time_lag_2"])
    shift_true = float(S["t_off"]) - lag_run
    _, _, R_fin, T_fin = host.state_pose(runs["node"].odom.state)
    for name, (R, T) in (("final", (R_fin, T_fin)), ("truth", (R_true, T_true))):
        prof = {ms: rp.run(R, T, ms / 1000.0)["result"]["mme"] for ms in (0.0, 5.0, 10.0, 15.0, 20.0, 25.0)}
        prof["true lag"] = rp.run(R, T, shift_true)["result"]["mme"]
        print(f"lag profile of {name} (LI-Init lag {lag_run * 1000:.3f} ms, simulated {S['t_off'] * 1000:.3f} ms, true shift "
              f"{shift_true * 1000:.3f} ms): " + ", ".join(f"{k}: {v:.6f}" for k, v in prof.items()), flush=True)
