"""Profiles of the refined calibration on the H100, on the 60 s Livox scenario of tests/test_gpu_refine.py (simulated lag +13 ms,
tests/calib_sim.py): `run --refine --profile` at a small refinement budget and several replay jobs replays 84 profile candidates and
writes a profile.txt that parses; the lag, whose replayed MME moves by about 0.15 per 5 ms, is `pinned`; three profile candidates
replayed again on the lead context score their rows bit for bit. Each parameter's interval, and where the simulated truth lies against
it, are printed, not asserted: whether the interval covers the truth is a finding about the measure."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import _build, assess, profiles  # noqa: E402

BUDGET = 20     # refinement replays: the starts and stage 1's lag search (13 replays on this scenario), not the compass search
JOBS = 8


def truth(S, centre) -> dict:
    """{param: the simulated truth in the profile's units}: the rotation from the centre to the truth about each IMU axis [deg]
    (rotation vector of R_true R_centre^T), T_true [m], the simulated total lag [ms]"""
    from scipy.spatial.transform import Rotation
    w = np.degrees(Rotation.from_matrix(np.asarray(S["R_LI"], float) @ np.asarray(centre["R"]).T).as_rotvec())
    T = np.asarray(S["T_LI"], float)
    return dict(rot_x=w[0], rot_y=w[1], rot_z=w[2], trans_x=T[0], trans_y=T[1], trans_z=T[2], lag=float(S["t_off"]) * 1000.0)


def interval_lines(prof, S) -> list:
    """one line per parameter: verdict, the fitted minimum and its interval, the truth and where it lies against the interval"""
    tr, out = truth(S, prof["centre"]), []
    for p, f in prof["fits"].items():
        t, lo, hi = tr[p], f["lo_phys"], f["hi_phys"]
        where = "inside" if lo <= t <= hi else "below" if t < lo else "above" if t > hi else "no interval"
        unit = profiles.UNITS[p.split("_")[0]]
        lower = "" if f["lower_k"] == 0 else f"; lowest point k {f['lower_k']:+d} ({f['lower_dmme']:+.6f})"
        lower += "; the fit's minimum is a step or more from the lowest point" if profiles.off_lowest(f) else ""
        out.append(f"{p:7s} {f['verdict']:10s} min {f['u_phys']:+.4f} [{lo:+.4f}, {hi:+.4f}] {unit}, s {f['s']:.2e}, truth {t:+.4f}: "
                   f"{where}{lower}")
    return out


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("profile")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, path = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"S": path.S}

    def on_node(nd):
        g = nd.odom.g
        seen.update(g=g, node=nd)
        g.close = lambda: None                      # kept open for the tests below; closed at teardown
        real_ref, real_prof = nd.replay.write_refinement, nd.replay.write_profile

        def write_refinement(*a, **k):
            seen["ref"] = real_ref(*a, **k)
            return seen["ref"]

        def write_profile(*a, **k):
            t0 = time.perf_counter()
            seen["prof"] = real_prof(*a, **k)
            seen["wall_s"] = time.perf_counter() - t0
            return seen["prof"]
        nd.replay.write_refinement, nd.replay.write_profile = write_refinement, write_profile
    out = str(tmp / "out")
    argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet", "--refine",
            "--refine-max-replays", str(BUDGET), "--replay-jobs", str(JOBS), "--profile"]
    assert run.main(argv, on_node=on_node) == 0
    seen["out"] = out
    yield seen
    seen["node"].replay.close()
    capi.LiInitGpu.close(seen["g"])


@pytest.mark.gpu
def test_profile_report_and_lag_pinned(runs):
    text = open(os.path.join(runs["out"], "result", "profile.txt")).read()
    print(text, flush=True)
    rep = assess.parse_profile_report(text)
    prof, ref, S = runs["prof"], runs["ref"], runs["S"]
    assert rep["header"]["replays"] == len(rep["rows"]) == len(prof["rows"]) == 84 and rep["header"]["jobs"] == JOBS
    assert list(rep["fits"]) == list(profiles.PARAMS) and all(r["valid"] > 0 for r in rep["rows"])
    times = sorted(r["seconds"] for r in prof["rows"])
    print(f"refinement: {len(ref['trace'])} replays ({ref['status']}), lag {ref['time_lag'] * 1000:.3f} ms, MME {ref['mme']:.6f}; profile: "
          f"84 replays in {runs['wall_s']:.1f} s at {JOBS} jobs, median replay {times[len(times) // 2]:.2f} s", flush=True)
    for line in interval_lines(prof, S):
        print(line, flush=True)
    assert prof["fits"]["lag"]["verdict"] == "pinned"


@pytest.mark.gpu
def test_profile_rows_replay_bit_for_bit(runs):
    rp, prof = runs["node"].replay, runs["prof"]
    for p, k in (("rot_z", -3), ("trans_y", 2), ("lag", 6)):
        row = next(r for r in prof["rows"] if (r["param"], r["k"]) == (p, k))
        again = rp.run(row["R"], row["T"], row["shift_s"])["result"]["mme"]
        assert np.float64(again).tobytes() == np.float64(row["mme"]).tobytes(), (p, k)
