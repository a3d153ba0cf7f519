"""The timed map assessment on the H100, on the 60 s Livox scenario of tests/test_gpu_bag.py (simulated lag 13 ms, tests/calib_sim.py):
`run --assess-time` leaves every other result file byte-identical; at shift 0 as-run the timed evaluation is bit-equal to the plain one
and to the published REGISTERED records of sampled updates; sampled scans placed at +-6 ms and at a perturbed extrinsic are within 2
float32 ulps of the numpy restatement and repeat bit for bit; the synthetic known-lag case is recovered; and the findings on the
scenario (lag profile, LI-Init's lag error, what re-undistortion changes in the candidates' MME) are pinned as measured."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import assess_time_oracle as ato  # noqa: E402
from lidar_imu_init_b200 import _build, assess  # noqa: E402

SAMPLE_EVERY = 40   # stored updates kept for the placement checks
SIM_LAG = 0.013


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, host, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("assess_time")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"samples": []}

    def on_node(nd):
        g, o = nd.odom.g, nd.odom
        seen.update(g=g, assessment=nd.assess, node=nd)
        g.close = lambda: None                      # kept open for the tests below; closed at teardown
        real_undistort, real_append = o._undistort_imu, nd.assess.append_timed

        def undistort(raw, poses, state):
            seen["raw"] = g.frame_download(raw.handle)[:, [0, 1, 2, 9]].copy()
            real_undistort(raw, poses, state)

        def append_timed(R, p, RLI, TLI, poses, prior_state):
            info = g.assess_info()
            if info["scans"] % SAMPLE_EVERY == 0:
                Rq, pq, rli, tli = host.state_pose(prior_state)
                seen["samples"].append(dict(off=info["points"], raw=seen["raw"], poses=np.array(poses), stored=g.raw_points(),
                                            prior=(Rq, pq, rli, tli, np.array(prior_state[24:27])), post=(R, p, RLI, TLI),
                                            registered=g.cloud(capi.CLOUD_REGISTERED, R, p, RLI, TLI)[:, :3].copy()))
            real_append(R, p, RLI, TLI, poses, prior_state)
        o._undistort_imu = undistort
        nd.assess.append_timed = append_timed
    outs = []
    for i, extra in enumerate((["--assess"], ["--assess", "--assess-time"])):
        out = str(tmp / f"out{i}")
        argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet"] + extra
        assert run.main(argv, on_node=on_node if "--assess-time" in extra else None) == 0
        outs.append(out)
    seen["outs"] = outs
    yield seen
    capi.LiInitGpu.close(seen["g"])


@pytest.mark.gpu
def test_runner_files_identical_and_time_report_parses(runs):
    a, b = runs["outs"]
    files = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    assert "result/assessment.txt" in files and "result/assessment_time.txt" not in files
    for f in files:
        assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read(), f
    text = open(os.path.join(b, "result", "assessment_time.txt")).read()
    print(text, flush=True)
    rep = assess.parse_time_report(text)
    t = runs["g"].assess_timing_info()
    assert rep["header"]["timed_scans"] == t["timed_scans"] > 500 and rep["header"]["untimed_scans"] == t["untimed_scans"]
    assert len(rep["assessment"]["rows"]) == 14 and len(rep["profile"]) == 2 * assess.LAG_STEPS + 1


@pytest.mark.gpu
def test_shift_zero_as_run_is_bit_equal_to_plain(runs):
    g = runs["g"]
    a = g.assess_evaluate(radius=0.3, min_neighbors=10, as_run=True)
    ha, va, na = g.assess_download()
    wa = g.assess_placed()
    b = g.assess_evaluate_timed(None, None, 0.0, radius=0.3, min_neighbors=10, as_run=True)
    hb, vb, nb = g.assess_download()
    wb = g.assess_placed()
    assert a == b and a["points"] > 5_000_000
    assert wa.tobytes() == wb.tobytes()
    assert ha.tobytes() == hb.tobytes() and va.tobytes() == vb.tobytes() and na.tobytes() == nb.tobytes()
    assert len(runs["samples"]) > 10
    for s in runs["samples"]:
        np.testing.assert_array_equal(wb[s["off"]:s["off"] + len(s["registered"])], s["registered"])


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.gpu
def test_shifted_and_perturbed_placement_matches_restatement(runs):
    g = runs["g"]
    R0, T0 = runs["assessment"].final
    R1, T1 = assess.rot_exp([0.0, 0.0, np.radians(0.5)]) @ R0, T0 + [0.02, 0.0, 0.0]
    worst = 0
    for d, R, T in ((0.006, None, None), (-0.006, None, None), (0.0, R1, T1), (-0.006, R1, T1)):
        g.assess_evaluate_timed(R, T, d, radius=0.3, min_neighbors=10, as_run=R is None)
        w = g.assess_placed()
        g.assess_evaluate_timed(R, T, d, radius=0.3, min_neighbors=10, as_run=R is None)
        assert g.assess_placed().tobytes() == w.tobytes()
        for s in runs["samples"]:
            ref = ato.place_timed([s], d, R, T)
            u = _ulps(w[s["off"]:s["off"] + len(ref)], ref)
            worst = max(worst, int(u.max()))
    print(f"worst difference to the restatement: {worst} float32 ulps", flush=True)
    assert worst <= 2


@pytest.mark.gpu
def test_known_lag_is_recovered(gpu_lib):
    from assess_time_case import R_LI_TRUE, T_LI_TRUE, make_scan, state_of
    from lidar_imu_init_b200 import capi
    rng = np.random.default_rng(7)
    scans = [make_scan(rng, 0.35 + 0.1 * k, n=1500, e=0.010) for k in range(8)]
    g = capi.LiInitGpu(0.5, max_map_points=100_000, max_scan_points=5_000)
    a = assess.Assessment(g, max_points=20_000, radius=0.3, max_scans=16, timed=True, max_pose_rows=1000)
    for s in scans:
        g.raw_upload(s["raw"], 3)
        g.assess_hold()
        R, p, rli, tli, _ = s["prior"]
        g.raw_undistort_imu(s["poses"], R, p, rli, tli)
        a.append_timed(*s["post"], s["poses"], state_of(s["prior"]))
    mme = {k * 5.0: g.assess_evaluate_timed(R_LI_TRUE, T_LI_TRUE, k * 0.005, radius=0.3, query_stride=3)["mme"] for k in range(-4, 3)}
    g.close()
    assert min(mme, key=mme.get) == -10.0, mme


@pytest.mark.gpu
def test_findings(runs):
    """The lag profile of the scenario, LI-Init's lag error, and how far re-undistortion moves the candidates' MME (the measured answer
    to "a second-order effect"), printed and pinned as measured (H100 80GB HBM3, 700 W; DESIGN §4d).

    LI-Init's total lag on this scenario is -2.97 ms against the simulated +13 ms: 16.0 ms short. The profile of the final extrinsic
    falls monotonically from -20 ms (+0.065 MME) through 0 to +20 ms (-0.0056), towards the true lag at a shift of about +16 ms, but
    its slope on that side is small: the lag is reported `flat` with the best shift at the profile's +20 ms edge. Re-undistorting for
    a candidate moves its MME by at most 0.00065 (as-run: exactly 0), against 0.0012-0.068 between the candidates, and leaves every
    axis verdict as the plain sweep has it."""
    A, nd = runs["assessment"], runs["node"]
    rows, prof = A.sweep_time()
    plain = {name: r for name, _, _, r in A.sweep()}
    lag_err_ms = (nd.time_lag - SIM_LAG) * 1e3
    verdict, best = assess.lag_verdict(prof)
    m0 = dict(prof)[0.0]["mme"]
    print(f"LI-Init lag {nd.time_lag * 1e3:.3f} ms, error {lag_err_ms:+.3f} ms; profile " +
          ", ".join(f"{s:+.0f} {r['mme'] - m0:+.6f}" for s, r in prof) + f"; lag {verdict}, best {best:+.1f} ms", flush=True)
    diff = {name: r["mme"] - plain[name]["mme"] for name, _, _, r in rows}
    print("re-undistorted - plain MME: " + ", ".join(f"{k} {v:+.6f}" for k, v in diff.items()), flush=True)
    assert -16.5 < lag_err_ms < -15.5, lag_err_ms
    mme = [r["mme"] for _, r in prof]
    assert all(a > b for a, b in zip(mme, mme[1:])), mme
    assert (verdict, best) == ("flat", 20.0)
    assert 0.06 < mme[0] - m0 < 0.07 and -0.006 < mme[-1] - m0 < -0.005
    assert diff["as-run"] == 0.0
    assert max(abs(v) for v in diff.values()) < 0.001, diff
    timed_v = assess.verdicts({name: r for name, _, _, r in rows})
    plain_v = assess.verdicts(plain)
    assert {k: v[0] for k, v in timed_v.items()} == {k: v[0] for k, v in plain_v.items()}
