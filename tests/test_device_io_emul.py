"""The device-pointer twins of the upload, search and download entry points (liinit_*_device), checked on the CPU build of the library
(tests/emul): each twin against its host twin bit for bit, the stand-alone search's device tie order on constructed ties, every
refusal with nothing changed, and the Python binding's __cuda_array_interface__ dispatch. The CPU build's cudaMalloc memory is what
the library takes for device memory here; any other buffer counts as host memory."""
import ctypes as C

import numpy as np
import pytest

import liinit_emul as le
from lidar_imu_init_b200 import scenes

pytestmark = pytest.mark.skipif(not le.available(), reason="g++ or the CUDA vector-type headers are missing")

vp = C.c_void_p
INVALID, CAPACITY = -1, -3
BRICKS, CELLS = 1, 2
CLOUD_REGISTERED, CLOUD_REGISTERED_DOWN, CLOUD_BODY, CLOUD_EFFECT = 1, 2, 3, 4


def _lib():
    L = le.load()
    L.liinit_emul_device_alloc.restype = vp
    L.liinit_emul_device_alloc.argtypes = [C.c_size_t]
    L.liinit_emul_device_free.argtypes = [vp]
    L.liinit_launch_count.argtypes = [vp, C.POINTER(C.c_longlong)]
    L.liinit_map_size.argtypes = [vp, C.POINTER(C.c_int)]
    L.liinit_cloud_download.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_map_build_device.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_map_add_points_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.liinit_scan_upload_device.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_raw_upload_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
    L.liinit_map_nearest_search_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_double, vp, vp, vp]
    L.liinit_cloud_download_device.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int), vp]
    L.liinit_map_download_device.argtypes = [vp, vp, C.c_int, vp]
    return L


class Dev:
    """Emulated device memory holding a copy of a numpy array, `offset` bytes past a 16-byte aligned allocation."""

    def __init__(self, a, offset=0, nbytes=None):
        self.L = _lib()
        a = None if a is None else np.ascontiguousarray(a)
        self.nbytes = a.nbytes if nbytes is None else nbytes
        self.base = self.L.liinit_emul_device_alloc(self.nbytes + offset + 16)
        assert self.base
        self.ptr = self.base + offset
        if a is not None:
            C.memmove(self.ptr, a.ctypes.data, a.nbytes)

    def read(self, shape, dtype):
        out = np.empty(shape, dtype)
        C.memmove(out.ctypes.data, self.ptr, out.nbytes)
        return out

    def __del__(self):
        self.L.liinit_emul_device_free(self.base)


def _ck(g, rc):
    assert rc == 0, (rc, g.L.liinit_last_error(g.h))


def _rc(g, rc, code, words):
    assert rc == code, (rc, g.L.liinit_last_error(g.h))
    msg = g.L.liinit_last_error(g.h).decode()
    assert words in msg, msg


def _pose(p):
    return [np.ascontiguousarray(x, np.float64).reshape(-1) for x in (p.rot_end, p.pos_end, p.R_LI, p.T_LI)]


def _pptr(pose):
    return [x.ctypes.data_as(vp) for x in pose]


def _strided(xyz, stride):
    """[n, stride] float32 rows with xyz first and junk after"""
    a = np.full((len(xyz), stride), 7.5, np.float32)
    a[:, :3] = xyz
    return a


def _cloud_host(g, which, pose):
    n = C.c_int()
    args = _pptr(pose)
    _ck(g, g.L.liinit_cloud_download(g.h, which, *args, None, 0, C.byref(n)))
    out = np.zeros((n.value, 12), np.float32)
    _ck(g, g.L.liinit_cloud_download(g.h, which, *args, out.ctypes.data_as(vp), n.value, C.byref(n)))
    return out


def _cloud_dev(g, which, pose, cap, host_n):
    """the device twin into a cap-record buffer: (records, count from d_n, count from n or None)"""
    out = Dev(None, nbytes=max(cap, 1) * 48)
    dn = Dev(np.array([-7], np.int32))
    n = C.c_int(-5)
    _ck(g, g.L.liinit_cloud_download_device(g.h, which, *_pptr(pose), out.ptr, cap, C.byref(n) if host_n else None, dn.ptr))
    m = int(dn.read(1, np.int32)[0])
    return out.read((m, 12), np.float32), m, (n.value if host_n else None)


def _state(g):
    """everything a refused call must leave as it was"""
    v, s, lc, rn, sn = C.c_int(), C.c_int(), C.c_longlong(), C.c_int(), C.c_int()
    _ck(g, g.L.liinit_map_validnum(g.h, C.byref(v)))
    _ck(g, g.L.liinit_map_size(g.h, C.byref(s)))
    _ck(g, g.L.liinit_launch_count(g.h, C.byref(lc)))
    _ck(g, g.L.liinit_raw_download(g.h, None, 0, C.byref(rn)))
    _ck(g, g.L.liinit_scan_download_body(g.h, None, 0, C.byref(sn)))
    return v.value, s.value, lc.value, rn.value, sn.value


def _world(body, p):
    return (p.rot_end @ (p.R_LI @ body.T.astype(np.float64) + p.T_LI[:, None]) + p.pos_end[:, None]).T.astype(np.float32)


def _same_set(a, b):
    return sorted(map(bytes, np.ascontiguousarray(a, np.float32))) == sorted(map(bytes, np.ascontiguousarray(b, np.float32)))


@pytest.fixture(scope="module")
def case():
    return scenes.make_config("C2", N=3000, M=60000, open_air_frac=0.02)


def _ctx(c, index=BRICKS):
    return le.EmulGpu(c["ds"], max_map_points=150000, max_scan_points=5000, knn_index=index)


@pytest.mark.parametrize("stride,offset", [(3, 0), (4, 0), (12, 0), (4, 4)], ids=["s3", "s4", "s12", "s4-misaligned"])
def test_map_scan_and_search_twins_bit_identical(case, stride, offset):
    """map_build, scan_upload and nearest_search through device memory (read in place at stride 4, repacked otherwise, a misaligned
    stride-4 buffer through the generic repack): map, pass state, accumulators and neighbours equal to the host twins'."""
    c, p = case, case["pose_init"]
    host, dev = _ctx(c), _ctx(c)
    m_xyz, body = _strided(c["map_xyz"], stride), _strided(c["body_xyz"], stride)
    host.map_build(m_xyz)
    dm, db = Dev(m_xyz, offset), Dev(body, offset)
    _ck(dev, dev.L.liinit_map_build_device(dev.h, dm.ptr, stride, len(m_xyz)))
    assert dev.map_validnum() == host.map_validnum() == len(m_xyz)
    assert dev.map_stats() == host.map_stats()
    assert _same_set(dev.map_download(), host.map_download())
    host.close()
    # the passes and the queries compare the two twins on ONE map: which of several points at exactly the same distance a search
    # returns depends on the map's pool order, and two maps built by different launches (LIINIT_EMUL_SHUFFLE) may differ in it
    poses = ((True, p), (False, scenes.perturb_pose(p, 77, dtheta_deg=0.05, dpos=0.01)), (True, c["pose_gt"]))
    dev.scan_upload(body)
    ref = [(dev.icp_iterate(q.rot_end, q.pos_end, q.R_LI, q.T_LI, False, search), dev.scan_state()) for search, q in poses]
    _ck(dev, dev.L.liinit_scan_upload_device(dev.h, db.ptr, stride, len(body)))
    for (search, q), (rh, sh) in zip(poses, ref):
        rd = dev.icp_iterate(q.rot_end, q.pos_end, q.R_LI, q.T_LI, False, search)
        for a, b in zip(rh, rd):
            assert np.array_equal(np.asarray(a), np.asarray(b))
        sd = dev.scan_state()
        for k in ("world", "near_xyz", "near_cnt", "selected"):
            assert np.array_equal(sh[k], sd[k]), k
        sel = sh["selected"].astype(bool)            # (a normal is only written where its point is selected)
        assert np.array_equal(sh["normvec"][sel], sd["normvec"][sel])
    assert np.array_equal(dev.scan_body(), c["body_xyz"])
    # stand-alone queries: xyz [n, 5, 3], d2 [n, 5], cnt [n] in device memory
    qs = _strided(np.concatenate([_world(c["body_xyz"][:700], c["pose_gt"]), c["map_xyz"][:300]]), stride)
    n = len(qs)
    dq = Dev(qs, offset)
    ox, od, oc = Dev(None, nbytes=n * 60), Dev(None, nbytes=n * 20), Dev(None, nbytes=n * 4)
    _ck(dev, dev.L.liinit_map_nearest_search_device(dev.h, dq.ptr, stride, n, 5.0, ox.ptr, od.ptr, oc.ptr))
    hx, hd, hc = dev.nearest_search(qs)
    assert np.array_equal(ox.read((n, 5, 3), np.float32), hx)
    assert np.array_equal(od.read((n, 5), np.float32), hd)
    assert np.array_equal(oc.read(n, np.int32), hc)
    dev.close()


@pytest.mark.parametrize("index", [BRICKS, CELLS])
def test_raw_upload_clouds_and_effect_twins(case, index):
    """PointType attributes through raw_upload_device -> voxel grid -> REGISTERED / BODY / REGISTERED_DOWN records built in device
    memory, and EFFECT after a search pass with its count on the device, all equal to the host twins'."""
    c, p = case, case["pose_init"]
    rng = np.random.default_rng(5)
    n = 4000
    raw = np.zeros((n, 12), np.float32)
    raw[:, :3] = c["body_xyz"][rng.integers(0, len(c["body_xyz"]), n)] + rng.normal(0, 0.02, (n, 3)).astype(np.float32)
    raw[:, 3] = 1.0
    raw[:, 4:7] = rng.normal(size=(n, 3)).astype(np.float32)
    raw[:, 8] = rng.uniform(0, 255, n).astype(np.float32)
    raw[:, 9] = np.sort(rng.uniform(0, 100, n)).astype(np.float32)
    pose = _pose(p)
    g = _ctx(c, index)            # one map for both twins (the search settles exact-distance ties by its pool order)
    g.map_build(c["map_xyz"])
    draw = Dev(raw)
    want = {}
    for dev in (False, True):
        if dev:
            _ck(g, g.L.liinit_raw_upload_device(g.h, draw.ptr, 12, 9, n))
        else:
            g.raw_upload(raw, 9)
        g.raw_n = n
        pts = g.raw_points()
        clouds = {}
        for which in (CLOUD_REGISTERED, CLOUD_BODY):
            if dev:
                got, m, hn = _cloud_dev(g, which, pose, n + 5, True)
                assert m == hn == n, which
                clouds[which] = got
            else:
                clouds[which] = _cloud_host(g, which, pose)
        nd = g.raw_downsample(0.5)
        if dev:
            got, m, _ = _cloud_dev(g, CLOUD_REGISTERED_DOWN, pose, g.scan_n, False)
            assert m == nd
            clouds[CLOUD_REGISTERED_DOWN] = got
        else:
            clouds[CLOUD_REGISTERED_DOWN] = _cloud_host(g, CLOUD_REGISTERED_DOWN, pose)
        g.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
        if dev:
            got, m, _ = _cloud_dev(g, CLOUD_EFFECT, pose, g.scan_n, False)     # cap covers the scan: the count stays on the device
            got2, m2, hn = _cloud_dev(g, CLOUD_EFFECT, pose, len(want[CLOUD_EFFECT]), True)   # exact cap, host count as well
            assert m == m2 == hn and np.array_equal(got, got2)
            clouds[CLOUD_EFFECT] = got
        else:
            clouds[CLOUD_EFFECT] = _cloud_host(g, CLOUD_EFFECT, pose)
        if not dev:
            want = dict(clouds, pts=pts, nd=nd)
            continue
        assert np.array_equal(pts, want["pts"]) and nd == want["nd"]
        for which, rec in clouds.items():
            assert len(rec) == len(want[which]) and np.array_equal(rec, want[which]), which
    assert len(want[CLOUD_EFFECT]) > 0
    assert np.any(want[CLOUD_REGISTERED_DOWN][:, 4:7] != 0) and np.any(want[CLOUD_REGISTERED_DOWN][:, 8] != 0)   # attributes came along
    # the live map after map_incremental, downloaded into device memory
    g.map_incremental(p.rot_end, p.pos_end, p.R_LI, p.T_LI, c["ds"])
    live = g.map_download()
    out, dn = Dev(None, nbytes=len(live) * 12), Dev(np.array([0], np.int32))
    _ck(g, g.L.liinit_map_download_device(g.h, out.ptr, len(live), dn.ptr))
    assert int(dn.read(1, np.int32)[0]) == len(live)
    assert _same_set(out.read((len(live), 3), np.float32), live)
    g.close()


@pytest.mark.parametrize("stride", [3, 4, 12])
def test_map_add_points_twin_with_downsampling(case, stride):
    c = case
    gt = c["pose_gt"]
    new = ((gt.rot_end @ (gt.R_LI @ c["body_xyz"].T.astype(np.float64) + gt.T_LI[:, None]) + gt.pos_end[:, None]).T + 0.013).astype(np.float32)
    host, dev = _ctx(c), _ctx(c)
    for g in (host, dev):
        g.map_build(c["map_xyz"])
    for lo, hi, down in ((0, 1500, True), (1500, 2500, False), (1000, 3000, True)):
        a = _strided(new[lo:hi], stride)
        want = host.map_add_points(a, down)
        d = Dev(a)
        added = C.c_int(-1)
        _ck(dev, dev.L.liinit_map_add_points_device(dev.h, d.ptr, stride, len(a), int(down), C.byref(added)))
        assert added.value == want
        assert dev.map_validnum() == host.map_validnum()
        assert _same_set(dev.map_download(), host.map_download())
    host.close()
    dev.close()


def _tie_scene(ds):
    """map points in mirror pairs and rings around lattice queries: every query has several neighbours at bit-identical squared
    distances (x, y, z multiples of 1/64, so the distances are exact), in an order the tie rule has to settle by x"""
    rng = np.random.default_rng(11)
    centres = (rng.integers(-300, 300, (400, 3)) * 0.25).astype(np.float32)
    offs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 1, 0], [-1, -1, 0]], np.float32) * np.float32(0.0625)
    pts = (centres[:, None, :] + offs[None]).reshape(-1, 3)
    pts = pts[rng.permutation(len(pts))]
    return np.ascontiguousarray(pts, np.float32), centres


@pytest.mark.parametrize("index", [BRICKS, CELLS])
def test_nearest_search_device_tie_order(oracle_mod, index):
    ds = 0.05
    pts, q = _tie_scene(ds)
    dev = le.EmulGpu(ds, max_map_points=20000, max_scan_points=2000, knn_index=index)   # one map for both twins, as above
    dev.map_build(pts)
    n = len(q)
    dq = Dev(q)
    ox, od, oc = Dev(None, nbytes=n * 60), Dev(None, nbytes=n * 20), Dev(None, nbytes=n * 4)
    _ck(dev, dev.L.liinit_map_nearest_search_device(dev.h, dq.ptr, 3, n, 5.0, ox.ptr, od.ptr, oc.ptr))
    gx, gd, gc = ox.read((n, 5, 3), np.float32), od.read((n, 5), np.float32), oc.read(n, np.int32)
    hx, hd, hc = dev.nearest_search(q)
    assert np.array_equal(gx, hx) and np.array_equal(gd, hd) and np.array_equal(gc, hc)
    ties = np.sum(np.diff(gd, axis=1) == 0, axis=1)
    assert (ties >= 3).mean() > 0.9                     # the scene does tie
    # ikd-Tree under the same_knn rule (tools/emul_fuzz.py): counts and distances always, points where no two candidates tie
    om = oracle_mod.OracleMap(ds, 1 if oracle_mod.has_ikd() else 0)
    om.build(pts)
    ox6, od6, oc6, _ = om.knn(q, k=6)
    assert np.array_equal(gc, np.minimum(oc6, 5))
    valid = np.arange(5)[None, :] < gc[:, None]
    assert np.array_equal(gd, np.where(valid, od6[:, :5], -1))
    d = q[:, None, :] - gx
    dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert np.array_equal(dd[valid], gd[valid])
    # within each run of equal distances the device order is ascending x (PointType_CMP)
    for i in range(n):
        for k in range(gc[i] - 1):
            if gd[i, k] == gd[i, k + 1]:
                assert gx[i, k, 0] <= gx[i, k + 1, 0], (i, k)
    dev.close()


def test_refusals_change_nothing(case):
    """host pointer, null pointer, too small a cap, capacity overrun: LIINIT_ERR_INVALID / _CAPACITY, and map, staged cloud, resident
    scan and launch count as before"""
    c, p = case, case["pose_init"]
    g = _ctx(c)
    g.map_build(c["map_xyz"])
    g.raw_upload(_strided(c["body_xyz"], 12), 9)
    g.raw_downsample(0.5)
    g.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    g.raw_upload(_strided(c["body_xyz"][:1234], 12), 9)
    L, h = g.L, g.h
    hostpts = np.ascontiguousarray(_strided(c["body_xyz"], 4))
    hp = hostpts.ctypes.data_as(vp)
    d4 = Dev(hostpts)
    big = Dev(None, nbytes=6000 * 16)
    out = Dev(None, nbytes=4000 * 60)
    dn = Dev(np.array([0], np.int32))
    pose = _pptr(_pose(p))
    n = C.c_int(-3)
    before = _state(g)
    cases = [
        ("map_build host", lambda: L.liinit_map_build_device(h, hp, 4, 100), INVALID, "not device memory"),
        ("map_build null", lambda: L.liinit_map_build_device(h, None, 4, 100), INVALID, "xyz is null"),
        ("map_build stride", lambda: L.liinit_map_build_device(h, d4.ptr, 5, 100), INVALID, "stride"),
        ("map_build overrun", lambda: L.liinit_map_build_device(h, big.ptr, 4, 150001), CAPACITY, "max_map_points"),
        ("add_points host", lambda: L.liinit_map_add_points_device(h, hp, 4, 100, 1, C.byref(n)), INVALID, "not device memory"),
        ("scan_upload host", lambda: L.liinit_scan_upload_device(h, hp, 4, 100), INVALID, "not device memory"),
        ("scan_upload null", lambda: L.liinit_scan_upload_device(h, None, 4, 100), INVALID, "null"),
        ("scan_upload overrun", lambda: L.liinit_scan_upload_device(h, big.ptr, 4, 5001), CAPACITY, "max_scan_points"),
        ("raw_upload host", lambda: L.liinit_raw_upload_device(h, hp, 4, -1, 100), INVALID, "not device memory"),
        ("raw_upload time index", lambda: L.liinit_raw_upload_device(h, d4.ptr, 4, 4, 100), INVALID, "time_index"),
        ("raw_upload overrun", lambda: L.liinit_raw_upload_device(h, big.ptr, 12, 9, (1 << 20) + 1), CAPACITY, "staging"),
        ("search host queries", lambda: L.liinit_map_nearest_search_device(h, hp, 4, 100, 5.0, out.ptr, None, None), INVALID, "q_xyz"),
        ("search host output", lambda: L.liinit_map_nearest_search_device(h, d4.ptr, 4, 100, 5.0, hp, None, None), INVALID, "out_xyz"),
        ("search null queries", lambda: L.liinit_map_nearest_search_device(h, None, 4, 100, 5.0, out.ptr, None, None), INVALID, "null"),
        ("cloud host records", lambda: L.liinit_cloud_download_device(h, CLOUD_REGISTERED, *pose, hp, 1234, C.byref(n), None), INVALID, "rec12"),
        ("cloud host count", lambda: L.liinit_cloud_download_device(h, CLOUD_REGISTERED, *pose, out.ptr, 1234, None, hp), INVALID, "d_n"),
        ("cloud misaligned", lambda: L.liinit_cloud_download_device(h, CLOUD_BODY, None, None, None, None, out.ptr + 4, 1234, C.byref(n), None),
         INVALID, "aligned"),
        ("cloud small cap", lambda: L.liinit_cloud_download_device(h, CLOUD_REGISTERED, *pose, out.ptr, 1233, C.byref(n), dn.ptr), CAPACITY,
         "cap_points"),
        ("map_download host", lambda: L.liinit_map_download_device(h, hp, 10, dn.ptr), INVALID, "xyz"),
        ("map_download null count", lambda: L.liinit_map_download_device(h, out.ptr, 10, None), INVALID, "d_n"),
    ]
    for name, call, code, words in cases:
        _rc(g, call(), code, words)
        assert _state(g) == before, (name, before, _state(g))
    assert n.value == 1234 and int(dn.read(1, np.int32)[0]) == 0      # too small a cap: the host count as the twin reports it
    # the resident scan and staged cloud still work and are the ones from before
    assert len(g.raw_points()) == 1234
    g.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    g.close()


def test_scan_attach_host_still_refuses_device_memory(case):
    c = case
    g = _ctx(c)
    d = Dev(_strided(c["body_xyz"], 4))
    rc = g.L.liinit_scan_attach_host(g.h, d.ptr, 4, len(c["body_xyz"]))
    _rc(g, rc, INVALID, "page-locked")
    g.scan_attach(c["body_xyz"])                 # a host buffer attaches as before
    g.close()


# ---- the Python binding over the CPU build of the library ------------------------------------------------------------------------
class FakeDevArray:
    """An object exposing __cuda_array_interface__ (version 3) over emulated device memory, as CuPy or torch would."""

    def __init__(self, a, typestr=None, strides=None, ptr=None):
        a = np.ascontiguousarray(a)
        self.mem = Dev(a) if ptr is None else None
        self.__cuda_array_interface__ = dict(shape=a.shape, typestr=typestr or a.dtype.str, data=(ptr or self.mem.ptr, False),
                                             strides=strides, version=3)


@pytest.fixture
def capi_on_emul(monkeypatch):
    from lidar_imu_init_b200 import capi
    monkeypatch.setattr(capi, "_LIB", None)
    monkeypatch.setenv("LIINIT_GPU_LIB", le._mk.build())
    yield capi


def test_binding_dispatches_device_arrays(capi_on_emul, case):
    capi, c = capi_on_emul, case
    p = c["pose_init"]
    mk = lambda: capi.LiInitGpu(c["ds"], max_map_points=150000, max_scan_points=5000)   # noqa: E731
    host, dev = mk(), mk()
    host.map_build(c["map_xyz"])                                     # numpy: the host path, as before
    dev.map_build(FakeDevArray(c["map_xyz"]))
    assert dev.map_validnum() == host.map_validnum() == len(c["map_xyz"])
    assert _same_set(dev.map_download(), host.map_download())
    dev.scan_upload(c["body_xyz"])                                   # both uploads on one map (exact-distance ties, see above)
    a = dev.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    dev.scan_upload(FakeDevArray(_strided(c["body_xyz"], 4)))
    assert dev.scan_n == len(c["body_xyz"])
    b = dev.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))
    new = c["map_xyz"][:500] + np.float32(0.011)
    assert dev.map_add_points(FakeDevArray(new), True) == host.map_add_points(new, True)
    raw = _strided(c["body_xyz"], 12)
    host.raw_upload(raw, 9)
    dev.raw_upload(FakeDevArray(raw), 9)
    assert np.array_equal(dev.raw_points(), host.raw_points())
    # validation: dtype, row layout, and the device (here: host memory behind the interface) with the library's message
    bad = [(FakeDevArray(c["map_xyz"].astype(np.float64)), "float32"),
           (FakeDevArray(np.zeros((10, 5), np.float32)), "[n, 3]"),
           (FakeDevArray(np.zeros((10, 3), np.float32), strides=(16, 4)), "contiguous"),
           (FakeDevArray(np.zeros(30, np.float32)), "[n, 3]")]
    hostmem = np.zeros((10, 3), np.float32)
    bad.append((FakeDevArray(hostmem, ptr=hostmem.ctypes.data), "not device memory"))
    before = _state(dev)
    for arr, words in bad:
        calls = [dev.map_build, dev.scan_upload, lambda a: dev.map_add_points(a, True)]
        if arr.__cuda_array_interface__["shape"] != (10, 5):                 # (a raw cloud may have 5 floats per point)
            calls.append(lambda a: dev.raw_upload(a, -1))
        for call in calls:
            with pytest.raises(capi.LiInitError) as e:
                call(arr)
            assert words in str(e.value) or (words == "[n, 3]" and "raw clouds" in str(e.value)), (words, str(e.value))
    assert _state(dev) == before
    host.close()
    dev.close()
