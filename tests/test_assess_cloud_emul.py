"""The assessment cloud (liinit_assess_cloud) on the emulated library (the kernels compiled for the CPU): every stored point scored against
the numpy restatement (tests/assess_oracle.py) and bit-equal to the strided evaluations, batches that do not change a bit, leaf records
against a numpy restatement from the per-point records, refusals that change nothing, the PCD writer, and `run --assess-cloud`."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import assess_cloud_oracle as aco  # noqa: E402
import assess_oracle as ao  # noqa: E402
import test_assess_emul as tae  # noqa: E402
from lidar_imu_init_b200 import assess, capi, node, pcd  # noqa: E402

emul = pytest.importorskip("liinit_emul")
INVALID, CAPACITY = -1, -3
SMALL_BATCH = 700   # LI_AS_CLOUD_BATCH of the variant library: a 2,400-point store runs in four batches


class _Methods(tae._AssessMethods):
    assess_cloud = capi.LiInitGpu.assess_cloud
    launch_count = capi.LiInitGpu.launch_count


def gpu(**kw):
    tae._emul_lib()

    class G(_Methods, emul.EmulGpu):
        pass
    return G(**kw)


@pytest.fixture(scope="module")
def small_batch_gpu(tmp_path_factory):
    """A factory of contexts on a variant of the emulated library built with -DLI_AS_CLOUD_BATCH=SMALL_BATCH (in a temporary directory;
    the default library is left as it is)."""
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    mk = emul._mk
    tmp = tmp_path_factory.mktemp("emul_small_batch")
    saved, saved_defs = (mk.LIB, mk.GEN, mk.build, emul._L), os.environ.get("LIINIT_EMUL_DEFS")
    try:
        mk.LIB, mk.GEN = str(tmp / "libliinit_emul_batch.so"), str(tmp / "gen")
        os.environ["LIINIT_EMUL_DEFS"] = f"-DLI_AS_CLOUD_BATCH={SMALL_BATCH}"
        path = mk.build()
        mk.build = lambda force=False: path
        emul._L = None
        lib = emul.load()
    finally:
        mk.LIB, mk.GEN, mk.build, emul._L = saved
        if saved_defs is None:
            os.environ.pop("LIINIT_EMUL_DEFS", None)
        else:
            os.environ["LIINIT_EMUL_DEFS"] = saved_defs

    def make(**kw):
        keep = emul._L
        emul._L = lib
        try:
            return gpu(**kw)
        finally:
            emul._L = keep
    return make


def _code(e):
    return e.value.code


def _f32_close(dev, ref):
    """float32 records against fp64 restatement values: the same NaNs, and each value the float32 rounding of a number within 1e-9
    (absolute) or 1e-9 (relative) of the restatement, i.e. at most one float32 step from float32(ref)."""
    ref = np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(dev), np.isnan(ref))
    ok = ~np.isnan(ref)
    r32 = ref[ok].astype(np.float32)
    d = np.abs(dev[ok].astype(np.float64) - r32.astype(np.float64))
    assert (d <= np.spacing(np.abs(r32)).astype(np.float64)).all(), d.max()
    assert not ok.any() or (dev[ok] == r32).mean() > 0.99


# scene: (make, radius, n_min)
SCENES = {"planes": (tae.scene_planes, 0.3, 10), "sphere": (tae.scene_sphere, 0.25, 10), "random": (tae.scene_random, 0.3, 10),
          "lattice": (tae.scene_lattice, 0.5, 10), "line": (tae.scene_line, 0.3, 10)}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_every_point_against_restatement(name):
    """leaf 0: one record per stored point in stored order; the placed point, n exact, h and v at float32 of the restatement's values,
    points 1, valid where h is finite; totals over every point with the restatement's counts. Every record is bit-equal to the
    float32 of an evaluation at stride 1 and the totals equal that evaluation's, the fp64 means included."""
    make, r, nmin = SCENES[name]
    scans = make()
    g = gpu()
    tae.load_scans(g, scans, check_registered=False)
    w = ao.place(scans)
    rec, tot = g.assess_cloud(radius=r, min_neighbors=nmin, leaf=0.0, as_run=True)
    assert rec.shape == (len(w), 8) and rec.dtype == np.float32
    np.testing.assert_array_equal(rec[:, :3], w)
    on, oh, ov, otot = ao.evaluate(w, r, nmin, 1)
    np.testing.assert_array_equal(rec[:, 5], on.astype(np.float32))
    _f32_close(rec[:, 3], oh)
    _f32_close(rec[:, 4], ov)
    assert (rec[:, 6] == 1).all()
    np.testing.assert_array_equal(rec[:, 7], (~np.isnan(oh)).astype(np.float32))
    assert tot["points"] == tot["queries"] == len(w) and tot["stride"] == 1 and tot["scans"] == len(scans)
    for k in ("queries", "valid", "sparse", "degenerate"):
        assert tot[k] == otot[k], (k, tot[k], otot[k])
    if otot["valid"]:
        assert tot["mme"] == pytest.approx(otot["mme"], abs=1e-9)
        assert tot["mpv"] == pytest.approx(otot["mpv"], rel=1e-9)
    else:
        assert math.isnan(tot["mme"]) and math.isnan(tot["mpv"])
    res = g.assess_evaluate(radius=r, min_neighbors=nmin, query_stride=1, as_run=True)
    h, v, n = g.assess_download()
    np.testing.assert_array_equal(rec[:, 3], h.astype(np.float32))
    np.testing.assert_array_equal(rec[:, 4], v.astype(np.float32))
    np.testing.assert_array_equal(rec[:, 5], n.astype(np.float32))
    assert res == tot or (math.isnan(res["mme"]) and {k: x for k, x in res.items() if k not in ("mme", "mpv")} ==
                          {k: x for k, x in tot.items() if k not in ("mme", "mpv")})
    # a candidate extrinsic replaces every scan's own, as in an evaluation
    R = ao.rot_exp([0.01, -0.02, 0.03]) @ scans[0][3]
    T = scans[0][4] + [0.02, -0.01, 0.03]
    rec2, tot2 = g.assess_cloud(R, T, radius=r, min_neighbors=nmin, leaf=0.0)
    np.testing.assert_array_equal(rec2[:, :3], ao.place(scans, R, T))
    res2 = g.assess_evaluate(R, T, radius=r, min_neighbors=nmin, query_stride=1)
    h2, _, n2 = g.assess_download()
    np.testing.assert_array_equal(rec2[:, 3], h2.astype(np.float32))
    np.testing.assert_array_equal(rec2[:, 5], n2.astype(np.float32))
    assert res2["valid"] == tot2["valid"] and res2["sparse"] == tot2["sparse"]


def test_batches_do_not_change_a_bit(small_batch_gpu):
    """A 2,400-point store in batches of 700 stored points: records and totals bit-identical to one batch, at leaf 0 and at a leaf; point
    j*s bit-equal to query j of an evaluation at stride s (s = 2, 3, 7) on the same context."""
    scans = tae.scene_planes(n=1600)
    assert sum(len(s[0]) for s in scans) == 2400
    one, many = gpu(), small_batch_gpu()
    for g in (one, many):
        tae.load_scans(g, scans, check_registered=False)
    R = ao.rot_exp([0.004, 0.0, -0.006]) @ scans[0][3]
    T = scans[0][4] + [0.01, 0.0, -0.01]
    for args in (dict(as_run=True), dict(R_LI=R, T_LI=T)):
        for leaf in (0.0, 0.1):
            a, ta = one.assess_cloud(radius=0.3, min_neighbors=10, leaf=leaf, **args)
            b, tb = many.assess_cloud(radius=0.3, min_neighbors=10, leaf=leaf, **args)
            assert a.tobytes() == b.tobytes() and ta == tb
        rec, _ = many.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.0, **args)
        for s in (2, 3, 7):
            res = many.assess_evaluate(radius=0.3, min_neighbors=10, query_stride=s, **args)
            assert res["queries"] == len(rec[::s])
            h, v, n = many.assess_download()
            assert rec[::s, 3].tobytes() == h.astype(np.float32).tobytes()
            assert rec[::s, 4].tobytes() == v.astype(np.float32).tobytes()
            assert rec[::s, 5].tobytes() == n.astype(np.float32).tobytes()
    # a call is bit-identical to the one before it
    c1, t1 = many.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.0, as_run=True)
    c2, t2 = many.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.0, as_run=True)
    assert c1.tobytes() == c2.tobytes() and t1 == t2


@pytest.mark.parametrize("name,leaf", [("planes", 0.1), ("planes", 0.37), ("random", 0.2), ("sphere", 0.05), ("lattice", 0.25),
                                       ("lattice", 0.5), ("line", 0.03)])
def test_leaf_records_against_restatement(name, leaf):
    """Leaf records equal the restatement from the per-point records (fp64 sums in stored order, float32 store, ascending key), NaN
    fields included; the lattice's points sit exactly on leaf boundaries; a size query computes the same number of leaves."""
    make, r, nmin = SCENES[name]
    g = gpu()
    tae.load_scans(g, make(), check_registered=False)
    rec0, t0 = g.assess_cloud(radius=r, min_neighbors=nmin, leaf=0.0, as_run=True)
    recL, tL = g.assess_cloud(radius=r, min_neighbors=nmin, leaf=leaf, as_run=True)
    assert t0 == tL or math.isnan(t0["mme"])
    ref = aco.leaf_records(rec0, leaf)
    np.testing.assert_array_equal(recL, ref)
    assert recL[:, 6].sum() == len(rec0) and recL[:, 7].sum() == rec0[:, 7].sum()
    if name == "random":
        assert (recL[:, 7] == 0).any()              # the sparse outliers: leaves without a valid point
        assert np.isnan(recL[recL[:, 7] == 0, 3:5]).all()
    if name == "lattice":
        q = rec0[:, :3].astype(np.float64) / leaf
        assert (q == np.floor(q)).all(axis=1).sum() > 50
    n = C.c_longlong(-1)
    P = capi.AssessParams(r, nmin, 0, 1, 0)
    assert g.L.liinit_assess_cloud(g.h, C.byref(P), None, None, leaf, None, 0, C.byref(n), None) == 0
    assert n.value == len(recL)


def test_refusals_change_nothing():
    """Refusals leave the last evaluation's download, the store, the staged cloud and the launch count as they were and write no record;
    a successful cloud call leaves the last evaluation's values too."""
    fresh = gpu()
    with pytest.raises(emul.EmulError) as e:
        fresh.assess_cloud(as_run=True)              # before liinit_assess_reserve
    assert _code(e) == INVALID
    scans = tae.scene_planes()
    g = gpu()
    tae.load_scans(g, scans, check_registered=False)
    g.assess_evaluate(radius=0.3, min_neighbors=10, query_stride=3, as_run=True)
    N = g.assess_info()["points"]

    def state():
        return g.assess_info(), [a.tobytes() for a in g.assess_download()], g.raw_points().tobytes()
    before, launches = state(), g.launch_count()

    def call(leaf=0.0, stride=0, cap=N, radius=0.3, nmin=10):
        rec = np.full((max(cap, 1), 8), 7.0, np.float32)
        tot = capi.AssessResult()
        tot.points = -7
        n = C.c_longlong(0)
        P = capi.AssessParams(radius, nmin, stride, 1, 0)
        rc = g.L.liinit_assess_cloud(g.h, C.byref(P), None, None, leaf, rec.ctypes.data_as(C.c_void_p), cap, C.byref(n), C.byref(tot))
        assert (rec == 7.0).all() and tot.points == -7
        return rc, n.value
    assert call(cap=N - 1) == (CAPACITY, N)
    for leaf in (-0.1, float("nan"), float("inf"), float("-inf")):
        assert call(leaf=leaf)[0] == INVALID, leaf
    for stride in (2, 3, -1):
        assert call(stride=stride)[0] == INVALID, stride
    assert call(radius=0.0)[0] == INVALID and call(nmin=3)[0] == INVALID
    assert g.launch_count() == launches
    assert state() == before
    # refusals after the placement: a leaf too small for the cloud, and cap below the number of leaves
    assert call(leaf=1e-12)[0] == CAPACITY
    rc, leaves = call(leaf=0.1, cap=10)
    assert rc == CAPACITY and leaves > 10
    assert state() == before
    # a cloud call leaves the last evaluation's per-query values and the staged cloud
    g.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.1, as_run=True)
    g.assess_cloud(radius=0.25, min_neighbors=12, leaf=0.0, as_run=True)
    assert state() == before
    # the placement hook then returns the cloud's placement
    np.testing.assert_array_equal(g.assess_placed(), ao.place(scans))


def test_pcd_header_and_body(tmp_path):
    rng = np.random.default_rng(5)
    rec = rng.normal(size=(37, 8)).astype(np.float32)
    rec[3, 3:5] = np.nan
    path = str(tmp_path / "a.pcd")
    assert pcd.write_assess(path, rec) == 37
    header, body = aco.read_assess_pcd(path)
    assert header["VERSION"] == "0.7" and header["FIELDS"].split() == list(pcd.ASSESS_FIELDS)
    assert header["SIZE"].split() == ["4"] * 8 and header["TYPE"].split() == ["F"] * 8 and header["COUNT"].split() == ["1"] * 8
    assert header["WIDTH"] == header["POINTS"] == "37" and header["HEIGHT"] == "1" and header["DATA"] == "binary"
    assert body.tobytes() == rec.tobytes()
    # the 48-byte writer is unchanged
    assert pcd.HEADER.splitlines()[2] == "FIELDS x y z _ normal_x normal_y normal_z _ intensity curvature _"


def test_write_cloud_scores_as_run(tmp_path):
    scans = tae.scene_planes()
    g = gpu()
    a = assess.Assessment(g, max_points=10_000, radius=0.3, max_scans=8)
    assert a.write_cloud(str(tmp_path / "none.pcd")) is None and not os.path.exists(tmp_path / "none.pcd")
    for body, R, p, RLI, TLI in scans:
        g.raw_upload(body, -1)
        a.append(R, p, RLI, TLI)
    n, tot = a.write_cloud(str(tmp_path / "c.pcd"), 0.2)
    _, body = aco.read_assess_pcd(str(tmp_path / "c.pcd"))
    rec0, _ = g.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.0, as_run=True)
    np.testing.assert_array_equal(rec0[:, :3], ao.place(scans))
    np.testing.assert_array_equal(body, aco.leaf_records(rec0, 0.2))
    assert n == len(body) and tot["points"] == len(rec0)


@pytest.mark.parametrize("fmt", ["ros1", "ros2"])
def test_runner_assess_cloud_changes_no_other_file(tmp_path, monkeypatch, fmt):
    """run --assess-cloud, with and without --assess, on a short recording (LI-Init does not trigger this early): every other file is
    byte-identical to the run without it, assessment.txt included, and no cloud is written; a bad leaf is refused."""
    import test_bag_node as tb
    import test_bag2_node as tb2
    from lidar_imu_init_b200 import run
    cfg = tb.sim_config(tmp_path)
    make = tae._runner_make(cfg)
    monkeypatch.setattr(run, "make_node", lambda args, cfg, log: node.Node(cfg, make(), args.out, log))
    ev, _ = tb.livox_events(0.6, 300)
    bag = str(tmp_path / ("rec.bag" if fmt == "ros1" else "rec2"))
    if fmt == "ros1":
        tb.write_event_bag(bag, ev)
    else:
        tb2.write_event_bag2(bag, ev, files=1)
    cfgp = str(tmp_path / "sim.yaml")
    pcds = [str(tmp_path / "c1.pcd"), str(tmp_path / "c3.pcd")]
    runs = ([], ["--assess-cloud", pcds[0], "--assess-max-points", "100000"], ["--assess", "--assess-max-points", "100000"],
            ["--assess", "--assess-max-points", "100000", "--assess-cloud", pcds[1], "--assess-cloud-leaf", "0"])
    outs = []
    for i, extra in enumerate(runs):
        out = str(tmp_path / f"out{i}")
        assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet"] + extra) == 0
        outs.append(out)

    def files(d):
        return sorted(os.path.relpath(os.path.join(r, f), d) for r, _, fs in os.walk(d) for f in fs)
    assert files(outs[0]) == files(outs[1]) and files(outs[2]) == files(outs[3]) == sorted(files(outs[0]) + ["result/assessment.txt"])
    for a, b in ((0, 1), (2, 3)):
        for f in files(outs[a]):
            assert open(os.path.join(outs[a], f), "rb").read() == open(os.path.join(outs[b], f), "rb").read(), f
    assert not any(os.path.exists(p) for p in pcds)
    for leaf in ("-0.1", "nan", "inf"):
        assert run.main(["--config", cfgp, "--bag", bag, "--out", str(tmp_path / "bad"), "--quiet", "--assess-cloud", pcds[0],
                         "--assess-cloud-leaf", leaf]) == 1
