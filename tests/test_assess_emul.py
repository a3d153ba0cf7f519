"""The map assessment (liinit_assess_*, assess_kernels.cuh) on the emulated library (the kernels compiled for the CPU): per-query
neighbour counts, entropies and plane variances against the numpy restatement (tests/assess_oracle.py) and scipy's kd-tree, placement
against the published REGISTERED clouds, determinism, capacity and refusals; the report of assess.py; and the runner's --assess on small
ROS1 and ROS 2 bags. Also passes with LIINIT_EMUL_SHUFFLE and LIINIT_EMUL_POISON=1."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import assess_oracle as ao  # noqa: E402
from lidar_imu_init_b200 import assess, capi, config, node  # noqa: E402

emul = pytest.importorskip("liinit_emul")
INVALID, CAPACITY = -1, -3


def _emul_lib():
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    L = emul.load()
    capi.set_assess_argtypes(L)
    vp = emul.vp
    L.liinit_cloud_download.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    return L


class _AssessMethods:
    assess_reserve = capi.LiInitGpu.assess_reserve
    assess_append = capi.LiInitGpu.assess_append
    assess_info = capi.LiInitGpu.assess_info
    assess_evaluate = capi.LiInitGpu.assess_evaluate
    assess_download = capi.LiInitGpu.assess_download
    assess_placed = capi.LiInitGpu.assess_placed
    cloud = capi.LiInitGpu.cloud


def gpu(**kw):
    _emul_lib()

    class G(_AssessMethods, emul.EmulGpu):
        pass
    return G(**kw)


def _code(e):
    return e.value.code


# ---- scenes: scans of world points seen from different poses with different extrinsics ----
def _pose(rng, rot_deg, trans):
    return ao.rot_exp(np.radians(rot_deg) * rng.normal(size=3)), rng.normal(size=3) * trans


def _scans_of(world_parts, seed, rot_deg=20.0, trans=1.0):
    """Each part of world points becomes one scan: a random IMU pose and extrinsic, body = the inverse placement in float32."""
    rng = np.random.default_rng(seed)
    scans = []
    for w in world_parts:
        R, p = _pose(rng, rot_deg, trans)
        RLI, TLI = _pose(rng, 5.0, 0.2)
        body = ((np.asarray(w, float) - p) @ R - TLI) @ RLI
        scans.append((body.astype(np.float32), R, p, RLI, TLI))
    return scans


def scene_planes(seed=1, n=2400):
    rng = np.random.default_rng(seed)
    floor = np.c_[rng.uniform(-1.5, 1.5, (n, 2)), rng.normal(0, 0.01, n)]
    wall = np.c_[1.5 + rng.normal(0, 0.01, n // 2), rng.uniform(-1.5, 1.5, n // 2), rng.uniform(0, 1.0, n // 2)]
    pts = rng.permutation(np.r_[floor, wall])
    return _scans_of(np.array_split(pts, 3), seed)


def scene_sphere(seed=2, n=2500):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    pts = d / np.linalg.norm(d, axis=1)[:, None] * (1.0 + rng.normal(0, 0.005, n))[:, None]
    return _scans_of(np.array_split(pts, 2), seed)


def scene_random(seed=3, n=2000):
    rng = np.random.default_rng(seed)
    pts = np.r_[rng.uniform(-0.6, 0.6, (n, 3)), rng.uniform(-4, 4, (200, 3))]   # a dense block and sparse outliers
    return _scans_of(np.array_split(pts, 4), seed)


def scene_lattice():
    """Points on a 0.25 m lattice placed by the identity: neighbours at exactly d = r = 0.5 m (d2 = r2 in binary)."""
    g = np.arange(-4, 5) * 0.25
    pts = np.stack(np.meshgrid(g, g, g[:5], indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    I = np.eye(3)
    return [(pts, I, np.zeros(3), I, np.zeros(3))]


def scene_line():
    """Collinear points along x, y = z = 0, placed by the identity: every neighbourhood has det Sigma = 0."""
    x = (np.arange(200) * 0.01).astype(np.float32)
    pts = np.c_[x, np.zeros(200, np.float32), np.zeros(200, np.float32)].astype(np.float32)
    I = np.eye(3)
    return [(pts, I, np.zeros(3), I, np.zeros(3))]


def load_scans(g, scans, max_points=None, max_scans=64, check_registered=True):
    g.assess_reserve(max_points or sum(len(s[0]) for s in scans), max_scans)
    for body, R, p, RLI, TLI in scans:
        g.raw_upload(body, -1)
        if check_registered:
            reg = g.cloud(capi.CLOUD_REGISTERED, R, p, RLI, TLI)[:, :3]
            np.testing.assert_array_equal(reg, ao.body_to_world(body, R, p, RLI, TLI))
        assert g.assess_append(R, p, RLI, TLI)


def check_against_oracle(g, w_expect, radius, min_nb, stride, res):
    w = g.assess_placed()
    np.testing.assert_array_equal(w, w_expect)
    h, v, n = g.assess_download()
    on, oh, ov, tot = ao.evaluate(w_expect, radius, min_nb, stride)
    np.testing.assert_array_equal(n, on)
    np.testing.assert_array_equal(np.isnan(h), np.isnan(oh))
    ok = ~np.isnan(oh)
    np.testing.assert_allclose(h[ok], oh[ok], rtol=0, atol=1e-9)
    np.testing.assert_allclose(v[ok], ov[ok], rtol=1e-9, atol=0)
    for k in ("queries", "stride", "valid", "sparse", "degenerate"):
        assert res[k] == tot[k], (k, res[k], tot[k])
    if tot["valid"]:
        assert res["mme"] == pytest.approx(tot["mme"], abs=1e-9)
        assert res["mpv"] == pytest.approx(tot["mpv"], rel=1e-9)
    return w, h, v, n


SCENES = {"planes": (scene_planes, 0.3, 10, 3), "sphere": (scene_sphere, 0.25, 10, 2), "random": (scene_random, 0.3, 10, 1)}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_against_restatement(name):
    """As-run and a candidate extrinsic: placement bit-equal to the restatement (and to the REGISTERED cloud at every append), neighbour
    counts exact, h within 1e-9 absolute, v within 1e-9 relative, totals exact; a second evaluation is bit-identical; scipy's kd-tree
    gives the same counts wherever no point lies within 1e-9 m of the radius."""
    from scipy.spatial import cKDTree
    make, r, nmin, s = SCENES[name]
    scans = make()
    g = gpu()
    load_scans(g, scans)
    res = g.assess_evaluate(radius=r, min_neighbors=nmin, query_stride=s, as_run=True)
    assert res["points"] == sum(len(b[0]) for b in scans) and res["scans"] == len(scans)
    w, h, v, n = check_against_oracle(g, ao.place(scans), r, nmin, s, res)
    assert res["valid"] > 0
    res2 = g.assess_evaluate(radius=r, min_neighbors=nmin, query_stride=s, as_run=True)
    assert res2 == res or (math.isnan(res["mme"]) and math.isnan(res2["mme"]))
    h2, v2, n2 = g.assess_download()
    assert h2.tobytes() == h.tobytes() and v2.tobytes() == v.tobytes() and n2.tobytes() == n.tobytes()
    far = ~ao.near_boundary(w, r, s)
    assert far.sum() > 0.9 * len(far)
    kd = cKDTree(w.astype(np.float64)).query_ball_point(w[::s].astype(np.float64), r, return_length=True)
    np.testing.assert_array_equal(n[far], kd[far])
    # a candidate extrinsic replaces every scan's own
    R = ao.rot_exp([0.01, -0.02, 0.03]) @ scans[0][3]
    T = scans[0][4] + [0.02, -0.01, 0.03]
    res3 = g.assess_evaluate(R, T, radius=r, min_neighbors=nmin, query_stride=s)
    check_against_oracle(g, ao.place(scans, R, T), r, nmin, s, res3)


def test_lattice_boundary_and_auto_stride():
    """Neighbours at exactly d2 = r2 count; the automatic stride of a small store is 1."""
    scans = scene_lattice()
    g = gpu()
    load_scans(g, scans)
    res = g.assess_evaluate(radius=0.5, min_neighbors=10, as_run=True)
    assert res["stride"] == 1 and res["queries"] == len(scans[0][0])
    w = ao.place(scans)
    _, _, _, n = check_against_oracle(g, w, 0.5, 10, 1, res)
    # an interior lattice point: 33 lattice points within two steps (the 6 at exactly two steps included)
    k = int(np.flatnonzero((w == [0, 0, -0.5]).all(1))[0])
    assert n[k] == 33
    d2, *_ = ao.neighbour_d2(w, [k])
    assert (d2[0] == 0.25).sum() == 6


def test_collinear_is_degenerate():
    g = gpu()
    load_scans(g, scene_line())
    res = g.assess_evaluate(radius=0.3, min_neighbors=10, as_run=True)
    assert res["degenerate"] == res["queries"] == 200 and res["valid"] == 0 and res["sparse"] == 0
    assert math.isnan(res["mme"]) and math.isnan(res["mpv"])
    h, v, n = g.assess_download()
    assert np.isnan(h).all() and np.isnan(v).all() and (n >= 30).all()


def test_sparse_queries():
    g = gpu()
    load_scans(g, scene_random())
    res = g.assess_evaluate(radius=0.3, min_neighbors=10, query_stride=1, as_run=True)
    assert res["sparse"] > 100 and res["valid"] > 1000
    check_against_oracle(g, ao.place(scene_random()), 0.3, 10, 1, res)


def test_capacity_and_skipped_scans():
    scans = scene_planes()
    sizes = [len(s[0]) for s in scans]
    g = gpu()
    # scan limit: the third scan is skipped
    g.assess_reserve(sum(sizes), 2)
    for body, R, p, RLI, TLI in scans:
        g.raw_upload(body, -1)
        g.assess_append(R, p, RLI, TLI)
    assert g.assess_info() == dict(points=sizes[0] + sizes[1], scans=2, skipped=1)
    # point limit: the second scan (made larger) does not fit, the third does
    scans[1] = (np.r_[scans[1][0], scans[1][0][:100]],) + scans[1][1:]
    g.assess_reserve(sizes[0] + sizes[2], 10)
    assert g.assess_info() == dict(points=0, scans=0, skipped=0)
    got = []
    for body, R, p, RLI, TLI in scans:
        g.raw_upload(body, -1)
        got.append(g.assess_append(R, p, RLI, TLI))
    assert got == [True, False, True]
    assert g.assess_info() == dict(points=sizes[0] + sizes[2], scans=2, skipped=1)
    res = g.assess_evaluate(radius=0.3, min_neighbors=10, query_stride=3, as_run=True)
    check_against_oracle(g, ao.place([scans[0], scans[2]]), 0.3, 10, 3, res)


def test_refusals_change_nothing():
    g = gpu()
    I, z = np.eye(3), np.zeros(3)
    for call in (lambda: g.assess_info(), lambda: g.assess_evaluate(as_run=True), lambda: g.assess_download(), lambda: g.assess_placed()):
        with pytest.raises(emul.EmulError) as e:
            call()
        assert _code(e) == INVALID
    g.raw_upload(scene_lattice()[0][0], -1)
    with pytest.raises(emul.EmulError) as e:
        g.assess_append(I, z, I, z)
    assert _code(e) == INVALID
    for mp, ms in ((0, 4), (-5, 4), (100, 0), (1 << 31, 4)):
        with pytest.raises(emul.EmulError) as e:
            g.assess_reserve(mp, ms)
        assert _code(e) == INVALID
    g.assess_reserve(5000, 8)
    with pytest.raises(emul.EmulError) as e:
        g.assess_evaluate(as_run=True)             # empty store
    assert _code(e) == INVALID
    assert g.assess_append(I, z, I, z)
    res = g.assess_evaluate(radius=0.5, min_neighbors=10, as_run=True)
    before = (g.assess_info(), g.assess_download(), g.raw_points(), g.launch_count() if hasattr(g, "launch_count") else None)
    bad = [dict(radius=0.0), dict(radius=-0.3), dict(radius=float("nan")), dict(radius=float("inf")), dict(min_neighbors=3),
           dict(query_stride=-1)]
    for kw in bad:
        args = dict(radius=0.5, min_neighbors=10, as_run=True)
        args.update(kw)
        with pytest.raises(emul.EmulError) as e:
            g.assess_evaluate(**args)
        assert _code(e) == INVALID, kw
    with pytest.raises(emul.EmulError) as e:
        g.assess_evaluate(radius=0.5)               # a candidate needs R_LI and T_LI
    assert _code(e) == INVALID
    with pytest.raises(emul.EmulError) as e:
        g.assess_evaluate(np.full((3, 3), np.nan), z, radius=0.5)
    assert _code(e) == INVALID
    after = (g.assess_info(), g.assess_download(), g.raw_points(), None)
    assert before[0] == after[0]
    for a, b in zip(before[1], after[1]):
        assert a.tobytes() == b.tobytes()
    np.testing.assert_array_equal(before[2], after[2])
    assert g.assess_evaluate(radius=0.5, min_neighbors=10, as_run=True) == res
    # a placed point beyond the cell range
    g.raw_upload(np.array([[1e9, 0, 0]], np.float32), -1)
    assert g.assess_append(I, z, I, z)
    with pytest.raises(emul.EmulError) as e:
        g.assess_evaluate(radius=0.3, as_run=True)
    assert _code(e) == CAPACITY


def test_evaluation_leaves_the_staged_cloud():
    scans = scene_sphere()
    g = gpu()
    load_scans(g, scans)
    staged = g.raw_points()
    body = g.cloud(capi.CLOUD_BODY)
    g.assess_evaluate(radius=0.25, min_neighbors=10, query_stride=5, as_run=True)
    np.testing.assert_array_equal(g.raw_points(), staged)
    np.testing.assert_array_equal(g.cloud(capi.CLOUD_BODY), body)


# ---- assess.py: candidates, sweep, report ----
def test_candidates_and_verdicts():
    R0, T0 = ao.rot_exp([0.1, 0.2, -0.3]), np.array([0.1, -0.05, 0.2])
    cs = assess.candidates(R0, T0)
    assert [c[0] for c in cs] == ["as-run", "final"] + [f"rot_{a}{s}" for a in "xyz" for s in "+-"] + [f"trans_{a}{s}" for a in "xyz" for s in "+-"]
    d = dict((c[0], c[1:]) for c in cs)
    np.testing.assert_allclose(d["rot_y-"][0] @ R0.T, ao.rot_exp([0, -math.radians(assess.DTHETA_DEG), 0]), atol=1e-15)
    np.testing.assert_array_equal(d["trans_z+"][1], T0 + [0, 0, assess.DT_M])
    rows = {c[0]: dict(mme=0.0) for c in cs}
    rows["rot_x+"]["mme"] = rows["rot_x-"]["mme"] = 0.1
    rows["trans_y+"]["mme"] = 0.1
    v = assess.verdicts(rows)
    assert v["rot_x"][0] == "constrained" and v["trans_y"][0] == "flat" and v["rot_z"][0] == "flat"


def test_sweep_report_parses():
    scans = scene_planes()
    g = gpu()
    a = assess.Assessment(g, max_points=10_000, radius=0.3, max_scans=8)
    for body, R, p, RLI, TLI in scans:
        g.raw_upload(body, -1)
        a.append(R, p, RLI, TLI)
    text = a.report()
    rep = assess.parse_report(text)
    assert rep["header"]["scans"] == 3 and rep["header"]["points"] == sum(len(s[0]) for s in scans) and rep["header"]["n_min"] == 10
    assert list(rep["rows"]) == [c[0] for c in assess.candidates(np.eye(3), np.zeros(3))]
    final = g.assess_evaluate(scans[-1][3], scans[-1][4], radius=0.3, min_neighbors=10)
    assert rep["rows"]["final"]["valid"] == final["valid"]
    assert rep["rows"]["final"]["mme"] == pytest.approx(final["mme"], abs=1e-8)
    assert set(rep["axes"]) == {f"{k}_{a}" for k in ("rot", "trans") for a in "xyz"}
    for axis, (verdict, dp, dm) in rep["axes"].items():
        assert verdict == ("constrained" if dp > 0 and dm > 0 else "flat")
    np.testing.assert_allclose([rep["rows"]["final"][k] for k in ("t_x", "t_y", "t_z")], scans[-1][4], atol=1e-6)
    assert assess.parse_report(assess.Assessment(gpu(), max_points=10).report()) == {"nothing": True}


# ---- the node's hook ----
class _FakeOdom:
    def __init__(self):
        s = np.zeros(36 + 576)
        s[0:9] = s[12:21] = np.eye(3).reshape(9)
        self.state, self.imu_en, self.switch_scan, self.frame_num = s, False, None, 0
        self.lidar_end_time, self.published = 0.0, {}
        self.data_accum_finished = self.data_accum_start = False
        self.orig_odom_freq, self.cut_frame_num = 10, 1

    def close(self):
        pass


def test_node_stores_lio_updates_but_the_switch_scan(tmp_path):
    o = _FakeOdom()
    nd = node.Node(config.Config(), o, str(tmp_path), node.Log(quiet=True))
    calls = []

    class Rec:
        def append(self, R, p, RLI, TLI):
            calls.append(o.frame_num)
    nd.assess = Rec()
    nd.online_calib_finish = True
    o.frame_num = 1
    nd._after_update()                  # LiDAR-only update
    o.imu_en, o.switch_scan, o.frame_num = True, 1, 2
    nd._after_update()                  # the switch scan
    o.frame_num = 3
    nd._after_update()                  # LIO
    o.frame_num = 4
    nd._after_update()
    nd.close(report=False)
    assert calls == [3, 4]


# ---- the runner ----
def _runner_make(cfg):
    import test_bag_node as tb
    from lidar_imu_init_b200.odometry import LidarOdometry
    from lidar_imu_init_b200 import _build
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    _emul_lib()

    class Emul(_AssessMethods, tb._emul_cls()):
        pass

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return tb.emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

    def make():
        o = EmulOdometry(Emul(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        o.preprocess = config.preprocess(cfg)
        return o
    return make


@pytest.mark.parametrize("fmt", ["ros1", "ros2"])
def test_runner_assess_changes_no_other_file(tmp_path, monkeypatch, fmt):
    """run --assess on a short recording (LI-Init does not trigger this early): every other result file is byte-identical to a run
    without the flag, and assessment.txt says there is nothing to assess."""
    import test_bag_node as tb
    import test_bag2_node as tb2
    from lidar_imu_init_b200 import run
    cfg = tb.sim_config(tmp_path)
    make = _runner_make(cfg)
    monkeypatch.setattr(run, "make_node", lambda args, cfg, log: node.Node(cfg, make(), args.out, log))
    ev, _ = tb.livox_events(0.6, 300)
    bag = str(tmp_path / ("rec.bag" if fmt == "ros1" else "rec2"))
    if fmt == "ros1":
        tb.write_event_bag(bag, ev)
    else:
        tb2.write_event_bag2(bag, ev, files=1)
    cfgp = str(tmp_path / "sim.yaml")
    outs = []
    for i, extra in enumerate(([], ["--assess", "--assess-max-points", "100000"])):
        out = str(tmp_path / f"out{i}")
        assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet"] + extra) == 0
        outs.append(out)
    files = sorted(os.path.relpath(os.path.join(d, f), outs[0]) for d, _, fs in os.walk(outs[0]) for f in fs)
    assert ("result/trajectory.txt" in files) and ("Log/mat_out.txt" in files)
    for f in files:
        assert open(os.path.join(outs[0], f), "rb").read() == open(os.path.join(outs[1], f), "rb").read(), f
    text = open(os.path.join(outs[1], "result", "assessment.txt")).read()
    assert text == assess.NOTHING and assess.parse_report(text) == {"nothing": True}
    assert not os.path.exists(os.path.join(outs[0], "result", "assessment.txt"))
    assert run.main(["--config", cfgp, "--bag", bag, "--out", str(tmp_path / "bad"), "--quiet", "--assess", "--assess-radius", "0"]) == 1
