"""The timed map assessment (liinit_assess_*_timed, assess_time_kernels.cuh) on the emulated library: timed placement at several lag
shifts and a candidate extrinsic bit-equal to the numpy restatement (tests/assess_time_oracle.py); the as-run evaluation at shift 0
bit-equal to the plain one, for a store that mixes timed and untimed scans; a known lag recovered by the lag profile; refusals and
capacity; the time report; the runner's --assess-time on small ROS1 and ROS 2 bags. Plus (nvcc only) ptxas reports no spills for the
new kernels. Also passes with LIINIT_EMUL_SHUFFLE and LIINIT_EMUL_POISON=1."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import assess_oracle as ao  # noqa: E402
from assess_time_case import R_LI_TRUE, T_LI_TRUE, make_scan, state_of  # noqa: E402
import assess_time_oracle as ato  # noqa: E402
from lidar_imu_init_b200 import _build, assess, capi, config, node  # noqa: E402

emul = pytest.importorskip("liinit_emul")
INVALID = -1


class _Methods:
    assess_reserve = capi.LiInitGpu.assess_reserve
    assess_reserve_timed = capi.LiInitGpu.assess_reserve_timed
    assess_hold = capi.LiInitGpu.assess_hold
    assess_append = capi.LiInitGpu.assess_append
    assess_append_timed = capi.LiInitGpu.assess_append_timed
    assess_info = capi.LiInitGpu.assess_info
    assess_timing_info = capi.LiInitGpu.assess_timing_info
    assess_evaluate = capi.LiInitGpu.assess_evaluate
    assess_evaluate_timed = capi.LiInitGpu.assess_evaluate_timed
    assess_download = capi.LiInitGpu.assess_download
    assess_placed = capi.LiInitGpu.assess_placed


def _emul_lib():
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    L = emul.load()
    capi.set_assess_argtypes(L)
    return L


def gpu(**kw):
    _emul_lib()

    class G(_Methods, emul.EmulGpu):
        pass
    return G(**kw)


def store(g, scans, timed_mask=None):
    """The node's order for each scan: stage, hold, undistort, append_timed (or, untimed: stage, undistort, append). Fills stored."""
    for k, s in enumerate(scans):
        timed = timed_mask is None or timed_mask[k]
        g.raw_upload(s["raw"], 3)
        if timed:
            g.assess_hold()
        R, p, rli, tli, _ = s["prior"]
        g.raw_undistort_imu(s["poses"], R, p, rli, tli)
        s["stored"] = g.raw_points()
        if timed:
            assert g.assess_append_timed(*s["post"], s["poses"], s["prior"])
        else:
            assert g.assess_append(*s["post"])
            s = dict(s, raw=None)
            scans[k] = s


@pytest.fixture(scope="module")
def mixed():
    rng = np.random.default_rng(5)
    scans = [make_scan(rng, 0.3 + 0.1 * k, n=700) for k in range(5)]
    g = gpu()
    g.assess_reserve_timed(10_000, 16, 1000)
    store(g, scans, [True, True, False, True, True])
    return g, scans


def test_timed_placement_matches_restatement(mixed):
    """Placement at shifts 0, +-6 ms and -20 ms (points before row 0), as-run and with a candidate extrinsic, bit-equal to the
    restatement; a repeated call is bit-identical."""
    g, scans = mixed
    assert g.assess_timing_info() == dict(timed_scans=4, untimed_scans=1, pose_rows=4 * 21)
    R = ao.rot_exp([0.01, -0.02, 0.03]) @ R_LI_TRUE
    T = T_LI_TRUE + [0.02, -0.01, 0.03]
    for d in (0.0, 0.006, -0.006, -0.02):
        for cand in ((None, None), (R, T)):
            g.assess_evaluate_timed(*cand, d, radius=0.3, query_stride=50, as_run=cand[0] is None)
            w = g.assess_placed()
            np.testing.assert_array_equal(w, ato.place_timed(scans, d, *cand), err_msg=f"shift {d}")
    g.assess_evaluate_timed(R, T, -0.006, radius=0.3, query_stride=50)
    assert g.assess_placed().tobytes() == ato.place_timed(scans, -0.006, R, T).tobytes()
    # a shift does move the timed points, and leaves the untimed scan's
    w0 = ato.place_timed(scans, 0.0)
    w1 = ato.place_timed(scans, 0.006)
    n0 = len(scans[0]["raw"]) + len(scans[1]["raw"])
    assert (w0[n0:n0 + 700] == w1[n0:n0 + 700]).all() and not (w0[:n0] == w1[:n0]).all()


def test_shift_zero_as_run_equals_plain_evaluation(mixed):
    g, scans = mixed
    for stride in (1, 4):
        a = g.assess_evaluate(radius=0.3, min_neighbors=10, query_stride=stride, as_run=True)
        ha, va, na = g.assess_download()
        wa = g.assess_placed()
        b = g.assess_evaluate_timed(None, None, 0.0, radius=0.3, min_neighbors=10, query_stride=stride, as_run=True)
        hb, vb, nb = g.assess_download()
        assert a == b and a["valid"] > 0
        assert ha.tobytes() == hb.tobytes() and va.tobytes() == vb.tobytes() and na.tobytes() == nb.tobytes()
        assert wa.tobytes() == g.assess_placed().tobytes()
        np.testing.assert_array_equal(wa, ao.place([(s["stored"], *s["post"]) for s in scans]))


def test_known_lag_is_recovered():
    """Tables from the trajectory shifted by e = +10 ms and exact posteriors: the profile's lowest MME is at shift -e, and the lag is
    constrained there."""
    rng = np.random.default_rng(7)
    e = 0.010
    scans = [make_scan(rng, 0.35 + 0.1 * k, n=1500, e=e) for k in range(8)]
    g = gpu()
    a = assess.Assessment(g, max_points=20_000, radius=0.3, max_scans=16, timed=True, max_pose_rows=1000)
    for s in scans:
        g.raw_upload(s["raw"], 3)
        g.assess_hold()
        R, p, rli, tli, _ = s["prior"]
        g.raw_undistort_imu(s["poses"], R, p, rli, tli)
        a.append_timed(*s["post"], s["poses"], state_of(s["prior"]))
    prof = [(k * 5.0, g.assess_evaluate_timed(R_LI_TRUE, T_LI_TRUE, k * 0.005, radius=0.3, query_stride=3)) for k in range(-4, 3)]
    mme = {s: r["mme"] for s, r in prof}
    print("profile " + ", ".join(f"{s:+.0f} ms {m:.5f}" for s, m in mme.items()), flush=True)
    assert min(mme, key=mme.get) == -10.0, mme
    shifted = [(s - (-10.0), r) for s, r in prof]   # centred on -e: both one-step neighbours are worse
    assert assess.lag_verdict(shifted) == ("constrained", 0.0)


def test_refusals_and_capacity_change_nothing():
    rng = np.random.default_rng(11)
    scans = [make_scan(rng, 0.3 + 0.1 * k, n=300) for k in range(3)]
    I, z = np.eye(3), np.zeros(3)
    g = gpu()
    g.assess_reserve(5000, 8)                       # a plain store
    g.raw_upload(scans[0]["raw"], 3)
    for call in (lambda: g.assess_hold(), lambda: g.assess_timing_info(), lambda: g.assess_append_timed(I, z, I, z, scans[0]["poses"], scans[0]["prior"]),
                 lambda: g.assess_evaluate_timed(lag_shift=0.0, as_run=True)):
        with pytest.raises(emul.EmulError) as ex:
            call()
        assert ex.value.code == INVALID
    with pytest.raises(emul.EmulError):
        g.assess_reserve_timed(5000, 8, 1)          # too few pose rows
    assert g.assess_info() == dict(points=0, scans=0, skipped=0)
    g = gpu()
    with pytest.raises(emul.EmulError) as ex:
        g.assess_reserve_timed(5000, 8, 100)
        g.assess_hold()                             # nothing staged
    assert ex.value.code == INVALID
    s0 = scans[0]
    store(g, [s0])
    before = (g.assess_info(), g.assess_timing_info(), g.assess_evaluate_timed(None, None, 0.003, radius=0.3, as_run=True), g.assess_download())
    g2 = scans[1]
    g.raw_upload(g2["raw"], 3)
    with pytest.raises(emul.EmulError) as ex:
        g.assess_append_timed(*g2["post"], g2["poses"], g2["prior"])   # no hold
    assert ex.value.code == INVALID
    g.assess_hold()
    g.raw_upload(g2["raw"], 3)                       # a re-stage ends the hold
    with pytest.raises(emul.EmulError) as ex:
        g.assess_append_timed(*g2["post"], g2["poses"], g2["prior"])
    assert ex.value.code == INVALID
    g.assess_hold()
    for poses in (g2["poses"][:1], np.zeros((4097, 22))):   # npose outside [2, LIINIT_MAX_IMU_POSES]
        with pytest.raises(emul.EmulError) as ex:
            g.assess_append_timed(*g2["post"], poses, g2["prior"])
        assert ex.value.code == INVALID
    for d in (float("nan"), float("inf")):
        with pytest.raises(emul.EmulError) as ex:
            g.assess_evaluate_timed(None, None, d, radius=0.3, as_run=True)
        assert ex.value.code == INVALID
    assert (g.assess_info(), g.assess_timing_info()) == before[:2]
    h, v, n = g.assess_download()
    assert h.tobytes() == before[3][0].tobytes() and n.tobytes() == before[3][2].tobytes()
    # the hold is still valid: the append goes through
    assert g.assess_append_timed(*g2["post"], g2["poses"], g2["prior"])
    assert g.assess_timing_info() == dict(timed_scans=2, untimed_scans=0, pose_rows=42)
    # a full pose pool: stored untimed and counted
    g.assess_reserve_timed(5000, 8, 30)
    store(g, [dict(scans[0]), dict(scans[1])], [True, True])
    assert g.assess_timing_info() == dict(timed_scans=1, untimed_scans=1, pose_rows=21)
    assert g.assess_info() == dict(points=600, scans=2, skipped=0)
    # a full point store: skipped
    g.assess_reserve_timed(500, 8, 100)
    g.raw_upload(scans[0]["raw"], 3)
    g.assess_hold()
    assert g.assess_append_timed(*scans[0]["post"], scans[0]["poses"], scans[0]["prior"])
    g.raw_upload(scans[1]["raw"], 3)
    g.assess_hold()
    assert not g.assess_append_timed(*scans[1]["post"], scans[1]["poses"], scans[1]["prior"])
    assert g.assess_info() == dict(points=300, scans=1, skipped=1)
    assert g.assess_timing_info() == dict(timed_scans=1, untimed_scans=0, pose_rows=21)


def test_time_report_parses(mixed):
    g, scans = mixed
    a = assess.Assessment.__new__(assess.Assessment)
    a.g, a.radius, a.min_neighbors, a.timed = g, 0.3, 10, True
    a.final = (R_LI_TRUE, T_LI_TRUE)
    rows, prof = a.sweep_time(steps=2)
    text = assess.time_report_text(g.assess_info(), g.assess_timing_info(), 0.3, 10, rows, prof, 0.013)
    rep = assess.parse_time_report(text)
    assert rep["header"]["timed_scans"] == 4 and rep["header"]["untimed_scans"] == 1 and rep["header"]["lag_ms"] == 13.0
    assert list(rep["assessment"]["rows"]) == [c[0] for c in assess.candidates(np.eye(3), np.zeros(3))]
    assert len(rep["assessment"]["axes"]) == 6
    assert [p["shift_ms"] for p in rep["profile"]] == [-4.0, -2.0, 0.0, 2.0, 4.0]
    assert rep["profile"][2]["lag_ms"] == 13.0
    assert rep["profile"][2]["mme"] == pytest.approx(rep["assessment"]["rows"]["final"]["mme"], abs=1e-8)
    assert rep["lag"] == assess.lag_verdict(prof)
    plain = g.assess_evaluate(None, None, radius=0.3, as_run=True)
    assert rep["assessment"]["rows"]["as-run"]["mme"] == pytest.approx(plain["mme"], abs=1e-8)
    assert assess.parse_time_report(assess.NOTHING) == {"nothing": True}


def test_node_appends_timed_scans_when_the_assessment_is_timed(tmp_path):
    s = np.zeros(36 + 576)
    s[0:9] = s[12:21] = np.eye(3).reshape(9)

    class Odom:
        state, imu_en, switch_scan, frame_num = s, True, None, 3
        lidar_end_time, published, timing = 0.0, {}, None
        data_accum_finished = data_accum_start = False
        orig_odom_freq, cut_frame_num = 10, 1

        def close(self):
            pass
    o = Odom()
    nd = node.Node(config.Config(), o, str(tmp_path), node.Log(quiet=True))
    calls = []

    class Rec:
        timed = True

        def append(self, *a):
            calls.append("append")

        def append_timed(self, *a):
            calls.append("timed")
    nd.assess = Rec()
    nd.online_calib_finish = True
    nd._after_update()                                # no propagation: untimed
    o.timing = (np.zeros((1, 22)), s)
    nd._after_update()                                # one pose: untimed
    o.timing = (np.zeros((3, 22)), s)
    nd._after_update()
    nd.assess.timed = False
    nd._after_update()
    nd.close(report=False)
    assert calls == ["append", "append", "timed", "append"]


# ---- the runner ----
@pytest.mark.parametrize("fmt", ["ros1", "ros2"])
def test_runner_assess_time_changes_no_other_file(tmp_path, monkeypatch, fmt):
    """run --assess --assess-time on a short recording: every file but assessment_time.txt is byte-identical to a run with --assess
    only, and assessment_time.txt parses (nothing to assess this early)."""
    import test_bag_node as tb
    import test_bag2_node as tb2
    from lidar_imu_init_b200 import run
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    cfg = tb.sim_config(tmp_path)
    _emul_lib()

    class Emul(_Methods, tb._emul_cls()):
        pass

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return tb.emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

    def make():
        o = EmulOdometry(Emul(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        o.preprocess = config.preprocess(cfg)
        return o
    monkeypatch.setattr(run, "make_node", lambda args, cfg, log: node.Node(cfg, make(), args.out, log))
    ev, _ = tb.livox_events(0.6, 300)
    bag = str(tmp_path / ("rec.bag" if fmt == "ros1" else "rec2"))
    if fmt == "ros1":
        tb.write_event_bag(bag, ev)
    else:
        tb2.write_event_bag2(bag, ev, files=1)
    cfgp = str(tmp_path / "sim.yaml")
    outs = []
    for i, extra in enumerate((["--assess"], ["--assess", "--assess-time"])):
        out = str(tmp_path / f"out{i}")
        assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet", "--assess-max-points", "100000"] + extra) == 0
        outs.append(out)
    files = sorted(os.path.relpath(os.path.join(d, f), outs[0]) for d, _, fs in os.walk(outs[0]) for f in fs)
    assert "result/assessment.txt" in files and "result/assessment_time.txt" not in files
    for f in files:
        assert open(os.path.join(outs[0], f), "rb").read() == open(os.path.join(outs[1], f), "rb").read(), f
    text = open(os.path.join(outs[1], "result", "assessment_time.txt")).read()
    assert assess.parse_time_report(text) == {"nothing": True}


# ---- registers (nvcc cross-compiles sm_90a; no GPU needed) ----
def test_timed_assessment_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    flags = [f for f in _build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-shared")]
    r = subprocess.run([nvcc] + flags + ["-cubin", "-Xptxas", "-v", "-o", str(tmp_path / "l.cubin"), os.path.join(_build.CSRC, "liinit_gpu.cu")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    report, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and (k := re.match(r"_Z\d+(k_at_\w+?|k_as_place|k_undistort_imu)P", name)):
            report[k.group(1)] = tuple(int(x) for x in m.groups())
    assert set(report) == {"k_at_scan_end", "k_at_place", "k_as_place", "k_undistort_imu"}, sorted(report)
    assert not {k: v for k, v in report.items() if any(v)}, report
