"""The LIO-phase replay (liinit_map_snapshot / _restore, liinit_replay_*, liinit_*_update_frozen, assess.Replay) without a GPU: the map
snapshot restores every map entry point bit for bit; a restaged sub-frame is the original staging; the frozen IESKF against a numpy
restatement of the reduced update; a replay of the run's own hand-over on the emulated library reproduces the run bit for bit, and a
frozen one keeps the candidate extrinsic; the replay report round-trips; the runner's --assess-replay."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lidar_imu_init_b200 import _build, assess, capi, config, host, node  # noqa: E402

emul = pytest.importorskip("liinit_emul")
INVALID = -1


class _Methods:
    assess_reserve = capi.LiInitGpu.assess_reserve
    assess_append = capi.LiInitGpu.assess_append
    assess_info = capi.LiInitGpu.assess_info
    assess_evaluate = capi.LiInitGpu.assess_evaluate
    assess_download = capi.LiInitGpu.assess_download
    assess_clear = capi.LiInitGpu.assess_clear
    map_snapshot = capi.LiInitGpu.map_snapshot
    map_restore = capi.LiInitGpu.map_restore
    replay_reserve = capi.LiInitGpu.replay_reserve
    replay_append = capi.LiInitGpu.replay_append
    replay_info = capi.LiInitGpu.replay_info
    replay_frame = capi.LiInitGpu.replay_frame
    replay_stage = capi.LiInitGpu.replay_stage


def _frames_cls():
    import test_bag_node as tb
    cls = tb._emul_cls()
    capi.set_assess_argtypes(emul.load())

    class G(_Methods, cls):
        pass
    return G


def _frozen_host():
    H = emul.host_lib()
    H.liinit_scan_update_frozen.restype = C.c_int
    H.liinit_scan_update_frozen.argtypes = [emul.vp, emul._f64, C.c_int, C.c_int, C.POINTER(emul.ScanStats)]
    return H


def scan_update(g, state, max_iteration, imu_en, frozen):
    """liinit_scan_update / _frozen of liinit_host.cpp linked against the emulated library"""
    H = _frozen_host()
    s = np.ascontiguousarray(state, np.float64).copy()
    st = emul.ScanStats()
    rc = (H.liinit_scan_update_frozen if frozen else H.liinit_scan_update)(g.h, s, int(max_iteration), int(imu_en), C.byref(st))
    if rc != 0:
        raise emul.EmulError(rc, (g.L.liinit_last_error(g.h) or b"").decode())
    return s, {k: getattr(st, k) for k, _ in emul.ScanStats._fields_}


def _cloud(rng, n, c=(0.0, 0.0, 0.0)):
    """points on three planes around c"""
    u = rng.uniform(-2, 2, size=(n, 2))
    k = rng.integers(0, 3, n)
    p = np.zeros((n, 3))
    for a in range(3):
        m = k == a
        p[m, a] = 0.01 * rng.normal(size=m.sum())
        p[m, (a + 1) % 3], p[m, (a + 2) % 3] = u[m, 0], u[m, 1]
    return (p + c).astype(np.float32)


def _same(a: dict, b: dict) -> bool:
    """two evaluation results bit for bit (NaN equal to NaN)"""
    return a.keys() == b.keys() and all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)


def _view(g, q):
    xyz, d2, cnt = g.nearest_search(q)
    return (g.map_download().tobytes(), tuple(g.map_stats().values()), g.map_validnum(), xyz.tobytes(), d2.tobytes(), cnt.tobytes(),
            g.raw_points().tobytes())


# ---- map snapshot ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knn_index", [1, 2])   # LIINIT_KNN_BRICKS, LIINIT_KNN_CELLS (the cell directory is snapshot too)
def test_snapshot_restores_every_map_entry_point(knn_index):
    """After snapshot -> add (downsampled and plain) / delete boxes / map_incremental / compaction / a new staged cloud -> restore, the
    map download, map stats, live count, stand-alone 5-NN results and the staged raw cloud are bit-equal to those taken at the snapshot;
    the same update applied after the snapshot and after a restore gives the same map."""
    rng = np.random.default_rng(3)
    G = _frames_cls()
    g = G(0.15, max_map_points=60_000, max_scan_points=5_000, knn_index=knn_index)
    g.map_build(_cloud(rng, 8000))
    g.map_add_points(_cloud(rng, 3000, (0.5, 0.2, 0.0)), True)
    g.raw_upload(np.hstack([_cloud(rng, 900), rng.uniform(0, 100, (900, 1)).astype(np.float32)]), 3)
    q = _cloud(rng, 400, (0.1, 0.1, 0.0))
    before = _view(g, q)
    assert g.map_snapshot() > 0
    changes = [lambda: g.map_add_points(_cloud(np.random.default_rng(9), 4000, (1.0, -0.5, 0.3)), True),
               lambda: g.map_add_points(_cloud(np.random.default_rng(10), 2000, (-1.0, 0.5, 0.0)), False),
               lambda: g.map_delete_boxes([[-0.5, -0.5, -0.5, 0.5, 0.5, 0.5]]),
               lambda: g.map_compact()]
    for ch in changes:
        ch()
    g.scan_upload(_cloud(rng, 500, (0.2, 0.0, 0.1)))
    g.map_incremental(np.eye(3), np.array([0.3, 0.0, 0.0]), np.eye(3), np.zeros(3), 0.15)
    g.raw_upload(np.hstack([_cloud(rng, 300), np.zeros((300, 1), np.float32)]), 3)
    assert _view(g, q) != before
    g.map_restore()
    assert _view(g, q) == before
    # the same update after the snapshot and after a restore: the same map
    changes[0]()
    after1 = _view(g, q)
    g.map_restore()
    changes[0]()
    assert _view(g, q) == after1


def test_restore_without_snapshot_is_refused():
    g = _frames_cls()(0.15, max_map_points=10_000, max_scan_points=1_000)
    with pytest.raises(emul.EmulError) as ex:
        g.map_restore()
    assert ex.value.code == INVALID


# ---- replay store ----------------------------------------------------------------------------------------------------------------------
def _subframes(g, rng, msgs=3):
    import test_bag_node as tb  # noqa: F401
    from lidar_imu_init_b200 import scenes
    scene = scenes.box_scene(20.0, 15.0, 5.0, n_slabs_x=1, n_slabs_y=1)
    out = []
    for k in range(msgs):
        m = scenes.livox_message(scene, lambda t: (np.repeat(np.eye(3)[None], len(t), 0), np.tile([8.0, 6.0, 2.0], (len(t), 1))), 50.0 + 0.1 * k,
                                 600, seed=k, dup_frac=0.01, tie_frac=0.05, noise_frac=0.01, bad_line_frac=0.0)
        out += g.frame_cut_livox(m, lidar_type=1, N_SCANS=6, blind=0.5, point_filter_num=1, required_frame_num=3, scan_count=k + 10, stamp=50.0 + 0.1 * k)
    return [e for e in out if e["n"] > 1]


def _staged(g):
    """the staged raw cloud: xyz, and xyz after a constant-velocity undistortion (which reads every point's time)"""
    a = g.raw_points().copy()
    g.raw_undistort_cv(np.array([0.3, -0.2, 0.5]), np.eye(3).reshape(9), np.array([1.0, 0.5, -0.2]))
    return a.tobytes() + g.raw_points().tobytes()


def test_replay_stage_equals_frame_stage():
    """Each stored sub-frame restages bit-equal to liinit_frame_stage of the original, times included, with its t_beg and end_ms; a full
    store skips and counts; an unknown index or handle is refused."""
    rng = np.random.default_rng(4)
    g = _frames_cls()(0.15, max_map_points=10_000, max_scan_points=5_000)
    subs = _subframes(g, rng)
    assert len(subs) >= 6
    total = sum(e["n"] for e in subs)
    g.replay_reserve(total - subs[-1]["n"], 64)     # room for all but the last
    ref = []
    for e in subs:
        g.frame_stage(e["handle"])
        ref.append(_staged(g))
        g.replay_append(e["handle"], e["t_beg"], e["end_ms"])
    info = g.replay_info()
    assert info == dict(frames=len(subs) - 1, skipped=1, points=total - subs[-1]["n"])
    for j in reversed(range(info["frames"])):
        g.replay_stage(j)
        assert _staged(g) == ref[j], j
        f = g.replay_frame(j)
        assert (f["t_beg"], f["end_ms"], f["n"]) == (subs[j]["t_beg"], np.float32(subs[j]["end_ms"]), subs[j]["n"])
    for call in (lambda: g.replay_stage(info["frames"]), lambda: g.replay_stage(-1), lambda: g.replay_append(1 << 40, 0.0, 1.0)):
        with pytest.raises(emul.EmulError) as ex:
            call()
        assert ex.value.code == INVALID
    g.replay_reserve(10, 1)                           # a reserve clears
    assert g.replay_info() == dict(frames=0, skipped=0, points=0)
    assert not g.replay_append(subs[0]["handle"], 0.0, 1.0) and g.replay_info()["skipped"] == 1


def test_replay_calls_before_reserve_are_refused():
    g = _frames_cls()(0.15, max_map_points=10_000, max_scan_points=1_000)
    for call in (lambda: g.replay_info(), lambda: g.replay_append(0, 0.0, 1.0), lambda: g.replay_stage(0), lambda: g.replay_reserve(0, 4)):
        with pytest.raises(emul.EmulError) as ex:
            call()
        assert ex.value.code == INVALID


# ---- frozen IESKF ----------------------------------------------------------------------------------------------------------------------
FREE = np.r_[0:6, 12:24]


def _random_case(rng):
    _build.build_host()
    s = host.state_init()
    s[0:9] = assess.rot_exp(rng.normal(size=3)).reshape(9)
    s[9:12] = rng.normal(size=3)
    s[12:21] = assess.rot_exp(rng.normal(size=3) * 0.1).reshape(9)
    s[21:24] = rng.normal(size=3) * 0.1
    s[24:36] = rng.normal(size=12) * 0.1
    A = rng.normal(size=(24, 24))
    s[36:] = (A @ A.T * 1e-3 + np.eye(24) * 1e-4).reshape(-1)
    prop = host.boxplus(s, rng.normal(size=24) * 1e-3)
    J = rng.normal(size=(40, 12))
    return s, prop, J.T @ J, rng.normal(size=12)


def _restated(s, prop, HtH, Htr):
    """the reduced update in numpy: the extrinsic's rows / columns dropped from cov, the pose block of HtH / Htr"""
    P = s[36:].reshape(24, 24)[np.ix_(FREE, FREE)]
    S = np.linalg.inv(P)
    S[:6, :6] += 1000.0 * HtH[:6, :6]
    K1 = np.linalg.inv(S)
    vec = host.boxminus(prop, s)[FREE]
    G = K1[:, :6] @ (1000.0 * HtH[:6, :6])
    sol = np.zeros(24)
    sol[FREE] = K1[:, :6] @ (1000.0 * Htr[:6]) + vec - G @ vec[:6]
    return sol, G


def test_frozen_update_matches_restatement():
    rng = np.random.default_rng(8)
    for _ in range(20):
        s, prop, HtH, Htr = _random_case(rng)
        out, sol, KH = host.ieskf_update(s, prop, HtH, Htr, frozen=True)
        want, G = _restated(s, prop, HtH, Htr)
        np.testing.assert_allclose(sol, want, rtol=1e-9, atol=1e-12)
        assert (sol[6:12] == 0).all()
        assert out[12:24].tobytes() == s[12:24].tobytes()           # the extrinsic keeps its bits
        ref = host.boxplus(s, want)
        free = np.r_[0:12, 24:36]
        np.testing.assert_allclose(out[free], ref[free], rtol=0, atol=1e-12)
        cov = out[36:].reshape(24, 24)
        assert (cov[6:12] == 0).all() and (cov[:, 6:12] == 0).all()
        np.testing.assert_allclose(KH[FREE][:, :6], G, rtol=1e-9, atol=1e-12)
        assert (KH[6:12] == 0).all() and (KH[:, 6:12] == 0).all()
        # the flag off is the unfrozen update, which moves the extrinsic
        out_full, _, _ = host.ieskf_update(s, prop, HtH, Htr)
        assert out_full[12:24].tobytes() != s[12:24].tobytes()


def test_frozen_propagation_and_update_keep_the_extrinsic():
    """IMU propagation with zero extrinsic noise, then frozen updates: the extrinsic is bit-equal to its input and its covariance rows and
    columns stay zero throughout."""
    rng = np.random.default_rng(9)
    s, _, HtH, Htr = _random_case(rng)
    cov = s[36:].reshape(24, 24)
    cov[6:12] = 0.0
    cov[:, 6:12] = 0.0
    ext = s[12:24].tobytes()
    imu = host.ImuProcess()
    imu.set_cov("R_LI_cov", 0.0)
    imu.set_cov("T_LI_cov", 0.0)
    t = 10.0
    imu.switch(np.array([[t, 0.0, 0.0, 0.0, 0.0, 0.0, 9.81]]))
    for k in range(5):
        smp = np.array([[t + 0.005 * (i + 1), *(rng.normal(size=3) * 0.2), *(np.array([0, 0, 9.81]) + rng.normal(size=3) * 0.3)] for i in range(20)])
        s, poses = imu.propagate(s, smp, t, 100.0)
        t = smp[-1, 0]
        c = s[36:].reshape(24, 24)
        assert (c[6:12] == 0).all() and (c[:, 6:12] == 0).all() and s[12:24].tobytes() == ext
        prop = s.copy()
        for _ in range(3):
            s, sol, _ = host.ieskf_update(s, prop, HtH * (k + 1), Htr, frozen=True)
            assert s[12:24].tobytes() == ext and (sol[6:12] == 0).all()


# ---- the replay on the emulated library ------------------------------------------------------------------------------------------------
def _emul_run(tmp_path, trigger_at=10, seconds=2.0, max_points=2_000_000):
    """Node over a written bag on the emulated library, with LI-Init's result forced to the simulated truth at update `trigger_at`, and a
    Replay attached. Returns (node, replay, run's final map, run's as-run evaluation)."""
    import lio_case
    import test_bag_node as tb
    from lidar_imu_init_b200 import rosbag
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    G = _frames_cls()
    cfg = tb.sim_config(tmp_path)
    ev, path = tb.livox_events(seconds, 400)
    bag = str(tmp_path / "rec.bag")
    tb.write_event_bag(bag, ev)
    res = lio_case.true_result(path.S)

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return scan_update(self.g, state, self.max_iteration, self.imu_en, self.frozen)

        def initialize(self, timediff_imu_wrt_lidar=0.0):
            return dict(res)

    o = EmulOdometry(G(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
    nd = node.Node(cfg, o, str(tmp_path / "out"), node.Log(quiet=True))

    def on_update(n):
        if n.updates == trigger_at:
            n.odom.data_accum_finished = True
    nd.on_update = on_update
    nd.assess = assess.Assessment(o.g, max_points=500_000, radius=0.3, max_scans=4096)
    nd.replay = o.replay = assess.Replay(o.g, nd.assess, max_points=max_points, max_frames=4096)
    with rosbag.Bag(bag) as b:
        nd.run(b)
    nd.close(report=False)
    return nd, nd.replay, o.g.map_download(), nd.assess.g.assess_evaluate(radius=0.3, as_run=True)


def test_replay_of_the_run_is_bit_identical_and_a_frozen_one_keeps_the_candidate(tmp_path):
    nd, rp, map_run, as_run = _emul_run(tmp_path)
    info = rp.info()
    assert nd.init_scan is not None and info["frames"] >= 8 and info["skipped"] == 0
    assert len(rp.run_states) >= 6
    r = rp.run(frozen=False)
    assert [j for j, _ in r["states"]] == [j for j, _ in rp.run_states]
    for (_, a), (_, b) in zip(r["states"], rp.run_states):
        assert a.tobytes() == b.tobytes()
    assert nd.odom.g.map_download().tobytes() == map_run.tobytes()
    assert _same(r["result"], as_run) and r["rms_m"] == 0.0
    # frozen, a candidate 1 deg / 3 cm away: the extrinsic is the candidate's after every update
    R = assess.rot_exp([0.0, 0.0, np.radians(1.0)]) @ np.asarray(rp.res["R_LI"])
    T = np.asarray(rp.res["T_LI"]) + [0.03, 0.0, 0.0]
    f = rp.run(R, T, 0.002, frozen=True)
    assert len(f["states"]) >= 6
    for _, s in f["states"]:
        assert s[12:21].tobytes() == R.reshape(9).tobytes() and s[21:24].tobytes() == T.tobytes()
        c = s[36:].reshape(24, 24)
        assert (c[6:12] == 0).all() and (c[:, 6:12] == 0).all()
    assert f["rms_m"] > 0


def test_truncated_store_is_refused():
    """A replay store that skipped a sub-frame is not replayed."""
    rng = np.random.default_rng(6)
    g = _frames_cls()(0.15, max_map_points=10_000, max_scan_points=5_000)
    subs = _subframes(g, rng, msgs=1)
    g.assess_reserve(1000, 8)
    rp = assess.Replay(g, assess.Assessment.__new__(assess.Assessment), max_points=subs[0]["n"], max_frames=8)
    rp.base, rp.res = object(), {}
    for e in subs[:2]:
        rp.record_frame(e)
    assert rp.info()["skipped"] == 1 and rp.frames == 1
    with pytest.raises(assess.ReplayError, match="truncated"):
        rp.run(frozen=False)


def test_replay_report_round_trip():
    rng = np.random.default_rng(1)

    def res():
        return dict(valid=int(rng.integers(1, 10**6)), sparse=int(rng.integers(0, 1000)), degenerate=int(rng.integers(0, 100)),
                    mme=float(rng.normal()), mpv=float(rng.uniform(1e-6, 1e-3)))
    R0, T0 = assess.rot_exp([0.01, 0.02, 1.5]), np.array([0.1, -0.02, 0.03])
    names = ["run", "li-init"] + [c[0] for c in assess.candidates(R0, T0)[1:]] + ["lag-5", "lag+5"]
    rows = []
    for name in names:
        shift = {"lag-5": -5.0, "lag+5": 5.0}.get(name, 0.0)
        rows.append((name, R0, T0, shift, dict(result=res(), R_LI=R0, T_LI=T0, rms_m=float(rng.uniform(0, 0.1)))))
    info = dict(frames=1234, skipped=0, points=5_600_000)
    text = assess.replay_report_text(info, 123_456_789, 42.5, 0.3, 10, rows)
    rep = assess.parse_replay_report(text)
    assert rep["header"] == dict(subframes=1234, skipped=0, points=5_600_000, snapshot_mb=123.456789, replay_s=42.5, radius=0.3, n_min=10,
                                 dtheta_deg=0.5, dt_m=0.02)
    assert list(rep["rows"]) == names
    for name, _, _, shift, r in rows:
        got = rep["rows"][name]
        assert got["shift_ms"] == shift and got["rms_m"] == pytest.approx(r["rms_m"], rel=1e-6)
        assert (got["valid"], got["sparse"], got["degenerate"]) == (r["result"]["valid"], r["result"]["sparse"], r["result"]["degenerate"])
        assert got["mme"] == pytest.approx(r["result"]["mme"], abs=1e-9)
    assert rep["axes"] == {k: (v, pytest.approx(dp, abs=1e-9), pytest.approx(dm, abs=1e-9))
                           for k, (v, dp, dm) in assess.verdicts({n: r["result"] for n, _, _, _, r in rows}).items()}
    prof = [(-5.0, rows[-2][4]["result"]), (0.0, rows[2][4]["result"]), (5.0, rows[-1][4]["result"])]
    assert rep["lag"][:2] == assess.lag_verdict(prof)
    assert assess.parse_replay_report(assess.NOTHING) == {"nothing": True}


# ---- the runner ------------------------------------------------------------------------------------------------------------------------
def test_runner_assess_replay(tmp_path, monkeypatch):
    """run --assess --assess-replay on a short recording: every other file is byte-identical to a run with --assess only, and
    assessment_replay.txt is the NOTHING text (no hand-over this early); a non-positive --assess-replay-max-points exits 1."""
    import test_bag_node as tb
    from lidar_imu_init_b200 import run
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    cfg = tb.sim_config(tmp_path)
    G = _frames_cls()

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return scan_update(self.g, state, self.max_iteration, self.imu_en, self.frozen)

    def make():
        o = EmulOdometry(G(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        o.preprocess = config.preprocess(cfg)
        return o
    monkeypatch.setattr(run, "make_node", lambda args, cfg, log: node.Node(cfg, make(), args.out, log))
    ev, _ = tb.livox_events(0.6, 300)
    bag = str(tmp_path / "rec.bag")
    tb.write_event_bag(bag, ev)
    cfgp = str(tmp_path / "sim.yaml")
    outs = []
    for i, extra in enumerate((["--assess"], ["--assess", "--assess-replay", "--assess-replay-max-points", "100000"])):
        out = str(tmp_path / f"out{i}")
        assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet", "--assess-max-points", "100000"] + extra) == 0
        outs.append(out)
    files = sorted(os.path.relpath(os.path.join(d, f), outs[0]) for d, _, fs in os.walk(outs[0]) for f in fs)
    assert "result/assessment.txt" in files and "result/assessment_replay.txt" not in files
    for f in files:
        assert open(os.path.join(outs[0], f), "rb").read() == open(os.path.join(outs[1], f), "rb").read(), f
    assert assess.parse_replay_report(open(os.path.join(outs[1], "result", "assessment_replay.txt")).read()) == {"nothing": True}
    # --assess-replay alone implies the store
    out = str(tmp_path / "out2")
    assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet", "--assess-max-points", "100000", "--assess-replay",
                     "--assess-replay-max-points", "100000"]) == 0
    assert os.path.exists(os.path.join(out, "result", "assessment_replay.txt"))
    assert not os.path.exists(os.path.join(out, "result", "assessment.txt"))
    assert run.main(["--config", cfgp, "--bag", bag, "--out", str(tmp_path / "out3"), "--quiet", "--assess-replay",
                     "--assess-replay-max-points", "0"]) == 1


def test_runner_refuses_a_truncated_store(tmp_path, monkeypatch, capsys):
    """A replay store that overflowed: the runner exits 1 and says so."""
    from lidar_imu_init_b200 import run

    class Truncated:
        def record_imu(self, *a):
            pass

        def record_frame(self, e):
            pass

        def record_update(self, state):
            pass

        def write(self, path, R_final=None, T_final=None):
            raise assess.ReplayError("the replay store is truncated (3 sub-frames skipped): raise its max_points")
    monkeypatch.setattr(assess, "Replay", lambda *a, **k: Truncated())
    import test_bag_node as tb
    cfg = tb.sim_config(tmp_path)
    from lidar_imu_init_b200.odometry import LidarOdometry
    G = _frames_cls()

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return scan_update(self.g, state, self.max_iteration, self.imu_en, self.frozen)

    def make(args, c, log):
        o = EmulOdometry(G(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        return node.Node(c, o, args.out, log)
    monkeypatch.setattr(run, "make_node", make)
    ev, _ = tb.livox_events(0.3, 100)
    bag = str(tmp_path / "rec.bag")
    tb.write_event_bag(bag, ev)
    assert run.main(["--config", str(tmp_path / "sim.yaml"), "--bag", bag, "--out", str(tmp_path / "o"), "--quiet", "--assess-max-points",
                     "100000", "--assess-replay"]) == 1
    assert "truncated" in capsys.readouterr().err
