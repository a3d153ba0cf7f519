"""The refinement by LIO replay on the H100, on the 60 s Livox scenario of tests/test_gpu_assess_replay.py (simulated lag +13 ms,
tests/calib_sim.py): `run --refine` writes a report that parses; the refined total lag is within 3 ms of the simulated one; the refined
MME is at or below that of the final extrinsic replayed at the simulated lag; the refined candidate replayed once more scores its trace
row bit for bit. The extrinsic errors of the refined, LI-Init's and the final extrinsic against the simulated truth are printed, not
asserted."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import _build, assess, host  # noqa: E402


def _err(R, T, S):
    """(rotation error [deg], translation error [m]) of an extrinsic against the simulated truth"""
    R_true, T_true = np.asarray(S["R_LI"], float), np.asarray(S["T_LI"], float)
    c = np.clip((np.trace(np.asarray(R) @ R_true.T) - 1.0) / 2.0, -1.0, 1.0)
    return float(np.degrees(np.arccos(c))), float(np.linalg.norm(np.asarray(T) - T_true))


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("refine")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, path = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"S": path.S}

    def on_node(nd):
        g = nd.odom.g
        seen.update(g=g, node=nd)
        g.close = lambda: None                      # kept open for the tests below; closed at teardown
        real = nd.replay.write_refinement

        def write_refinement(p, R_final=None, T_final=None, max_replays=None):
            t0 = time.perf_counter()
            seen["ref"] = real(p, R_final, T_final, max_replays)
            seen["wall_s"] = time.perf_counter() - t0
            return seen["ref"]
        nd.replay.write_refinement = write_refinement
    out = str(tmp / "out")
    argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet", "--refine"]
    assert run.main(argv, on_node=on_node) == 0
    seen["out"] = out
    yield seen
    capi.LiInitGpu.close(seen["g"])


@pytest.mark.gpu
def test_report_parses_and_lag_is_found(runs):
    text = open(os.path.join(runs["out"], "result", "refinement.txt")).read()
    print(text, flush=True)
    rep = assess.parse_refine_report(text)
    ref, S = runs["ref"], runs["S"]
    assert rep["header"]["skipped"] == 0 and rep["header"]["subframes"] > 1000
    assert rep["header"]["replays"] == len(rep["rows"]) == len(ref["trace"]) <= 120
    assert len(rep["axes"]) == 6 and rep["result"].startswith("Rotation LiDAR to IMU (degree)     = ")
    times = sorted(r["seconds"] for r in ref["trace"])
    print(f"refinement: {len(ref['trace'])} replays in {runs['wall_s']:.1f} s ({ref['status']}, start {ref['start']}), median replay "
          f"{times[len(times) // 2]:.2f} s; lag at the hand-over {ref['lag0'] * 1000:.3f} ms, refined {ref['time_lag'] * 1000:.3f} ms, "
          f"simulated {S['t_off'] * 1000:.3f} ms: error {(ref['time_lag'] - S['t_off']) * 1000:+.3f} ms", flush=True)
    assert abs(ref["time_lag"] - S["t_off"]) < 0.003


@pytest.mark.gpu
def test_refined_is_sharper_than_final_at_the_true_lag_and_reproducible(runs):
    rp, ref, S = runs["node"].replay, runs["ref"], runs["S"]
    _, _, R_fin, T_fin = host.state_pose(runs["node"].odom.state)
    shift_true = float(S["t_off"]) - rp.lag
    final_true = rp.run(R_fin, T_fin, shift_true)["result"]["mme"]
    again = rp.run(ref["R"], ref["T"], ref["shift_s"])["result"]["mme"]
    R_init, T_init = np.asarray(rp.res["R_LI"], float), np.asarray(rp.res["T_LI"], float)
    e_ref, e_init, e_fin = _err(ref["R"], ref["T"], S), _err(R_init, T_init, S), _err(R_fin, T_fin, S)
    print(f"MME: refined {ref['mme']:.6f}, final at the simulated lag shift ({shift_true * 1000:.3f} ms) {final_true:.6f}; extrinsic error "
          f"against the simulated truth (deg, mm): refined {e_ref[0]:.4f}, {e_ref[1] * 1000:.2f}; li-init {e_init[0]:.4f}, "
          f"{e_init[1] * 1000:.2f}; final {e_fin[0]:.4f}, {e_fin[1] * 1000:.2f}", flush=True)
    assert ref["mme"] <= final_true
    assert np.float64(again).tobytes() == np.float64(ref["mme"]).tobytes()
