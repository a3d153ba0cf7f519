"""CPU tests of the node's published clouds (liinit_cloud_download: /cloud_registered, /cloud_registered_body, /cloud_effected and the
pcd_save records) on the CPU build of the device library (tests/emul), bit for bit against the literal checker
(tests/cpp/output_oracle.cpp); the error contract; the publish stage of LidarOdometry (which scans publish, the switch scan, the
pcd_save file sequence) and the PCD files it writes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import frame_oracle as fo  # noqa: E402
import output_oracle as oo  # noqa: E402
from lidar_imu_init_b200 import capi, pcd, scenes  # noqa: E402

emul = pytest.importorskip("liinit_emul")


def _bind():
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    L = emul.load()
    vp = emul.vp
    L.liinit_cloud_download.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_raw_download_world.argtypes = [vp, emul._f64, emul._f64, emul._f64, emul._f64, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_frame_cut_livox.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int, C.POINTER(C.c_int)]
    L.liinit_frame_cut_pcl2.argtypes = [vp, vp, C.POINTER(capi.Pcl2Layout), C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int,
                                        C.POINTER(C.c_int)]
    L.liinit_frame_stage.argtypes = [vp, C.c_longlong]
    L.liinit_frame_download.argtypes = [vp, C.c_longlong, vp, C.c_int, C.POINTER(C.c_int)]

    class EmulOut(emul.EmulGpu):   # the product's binding methods over the emulated library
        cloud = capi.LiInitGpu.cloud
        raw_world = capi.LiInitGpu.raw_world
        frame_cut_livox = capi.LiInitGpu.frame_cut_livox
        frame_cut_pcl2 = capi.LiInitGpu.frame_cut_pcl2
        frame_stage = capi.LiInitGpu.frame_stage
        frame_download = capi.LiInitGpu.frame_download
        frame_size = capi.LiInitGpu.frame_size
    return EmulOut


@pytest.fixture(scope="module")
def Emul():
    return _bind()


@pytest.fixture(scope="module")
def built():
    """LidarOdometry loads the host and calibration libraries (the host library links the device library)"""
    from lidar_imu_init_b200 import _build
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()


def _pose(rng, big=False):
    R = scenes.so3_exp(rng.normal(size=3))
    p = rng.normal(size=3) * (100.0 if big else 5.0)
    RLI = scenes.so3_exp(rng.normal(size=3) * 0.05)
    TLI = rng.normal(size=3) * 0.1
    return R, p, RLI, TLI


def _timed_raw(n, seed, normals=True):
    raw = scenes.timed_scan_points(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 10.0, 0.1, n, seed=seed, det_range=60.0, sigma=0.01)
    if normals:
        rng = np.random.default_rng(seed)
        nv = rng.normal(size=(n, 3))
        raw[:, 4:7] = nv / np.linalg.norm(nv, axis=1, keepdims=True)
        raw[:, 7] = rng.normal(size=n)      # padding of the input: never read
        raw[:, 10:12] = rng.normal(size=(n, 2))
    return raw


def _effect_pass(g, down, pose):
    """a map of the scan itself at the pose, one search pass: most points find a plane"""
    g.map_build(oo.to_world(down, *pose)[:, 0:3])
    g.icp_iterate(*pose, False, True)


@pytest.mark.parametrize("undistort", ["cv", "imu"])
def test_pointtype_upload_all_clouds(Emul, undistort):
    rng = np.random.default_rng(1 if undistort == "cv" else 2)
    g = Emul(0.3, max_map_points=50_000, max_scan_points=4000)
    raw = _timed_raw(3000, seed=11)
    poses = np.zeros((6, 22))
    poses[:, 0] = np.linspace(0, 0.1, 6)
    poses[:, 1:13] = rng.normal(size=(6, 12)) * 0.2
    for k in range(6):
        poses[k, 13:22] = scenes.so3_exp(rng.normal(size=3) * 0.05).reshape(9)
    upose = _pose(rng)
    pose = _pose(rng, big=True)

    def stage():
        g.raw_upload(raw, 9)
        if undistort == "cv":
            g.raw_undistort_cv(np.array([0.02, -0.01, 0.3]), scenes.so3_exp([0.1, 0.2, 0.3]), np.array([0.4, 0.1, 0.0]))
        else:
            g.raw_undistort_imu(poses, *upose)
    # the map: the scan itself at the pose (most points then find a plane); it takes the staging buffer, so it comes first
    stage()
    g.map_build(oo.to_world(oo.voxel_grid(oo.staged_records(g, raw), 0.3), *pose)[:, 0:3])
    stage()
    staged = oo.staged_records(g, raw)
    assert np.abs(staged[:, 8]).max() > 0 and np.abs(staged[:, 4:7]).max() > 0
    oo.check_staged(g, staged, pose)
    down = oo.check_down(g, staged, 0.3, pose)
    assert len(down) < len(staged) and np.abs(down[:, 4:7]).max() > 0
    g.icp_iterate(*pose, False, True)
    assert oo.check_effect(g, down, pose) > len(down) // 4
    g.icp_iterate(*pose, False, False)         # a reuse pass: the effect cloud follows the last pass
    oo.check_effect(g, down, pose)
    g.map_incremental(*pose, 0.3)
    # the switch scan filters the staged cloud again: its attributes survive the voxel grid, the passes and the map update
    pose2 = _pose(rng)
    g.raw_downsample(0.3)
    oo.assert_bits(g.cloud(2, *pose2), oo.to_world(down, *pose2), "REGISTERED_DOWN of the re-filtered cloud")
    g.close()


def test_xyz_only_uploads_have_zero_attributes(Emul):
    rng = np.random.default_rng(3)
    g = Emul(0.3, max_map_points=50_000, max_scan_points=4000)
    raw = _timed_raw(2000, seed=12)
    pose = _pose(rng)
    # a PointType array whose time is not announced at index 9, a 4-float cloud with time in w, packed xyz
    for pts, ti, curv in ((raw, -1, None), (np.ascontiguousarray(raw[:, [0, 1, 2, 9]]), 3, raw[:, 9]), (np.ascontiguousarray(raw[:, 0:3]), -1, None)):
        g.raw_upload(pts, ti)
        staged = oo.records(g.raw_points(), curvature=curv)
        oo.check_staged(g, staged, pose)
        down = oo.check_down(g, staged, 0.3, pose)
        assert not down[:, 4:12].any()
    # the uploaded resident scans: scan_upload, scan_upload_raw, scan_attach_host
    body = np.ascontiguousarray(raw[:1500, 0:3])
    for up in (lambda: g.scan_upload(body), lambda: g.scan_upload_raw(raw[:1500], 0.3), lambda: g.scan_attach(raw[:1500])):
        g.raw_upload(raw, 9)          # a staged cloud with attributes before: they must not leak into the uploaded scan
        g.raw_downsample(0.3)
        up()
        d = g.cloud(2, *pose)
        assert len(d) == g.scan_n and not d[:, 4:8].any() and not d[:, 9:].any() and not d[:, 8].any()
        oo.assert_bits(d[:, 0:3], oo.to_world(oo.records(g.scan_body()), *pose)[:, 0:3])
    g.close()


def test_livox_subframes(Emul):
    """frame_stage of Livox sub-frames: intensity from the message, normals 0."""
    rng = np.random.default_rng(4)
    g = Emul(0.3, max_map_points=50_000, max_scan_points=8000)
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 10.0, 6000, seed=4, dup_frac=0.02, tie_frac=0.1)
    got = g.frame_cut_livox(m, N_SCANS=6, blind=0.5, point_filter_num=1, required_frame_num=3, scan_count=9, stamp=10.0)
    assert len(got) == 3
    for s in got:
        p12 = g.frame_download(s["handle"])
        g.frame_stage(s["handle"])
        pose = _pose(rng)
        g.raw_undistort_cv(np.array([0.01, 0.02, -0.2]), np.eye(3), np.array([0.3, 0.0, 0.1]))
        staged = oo.staged_records(g, p12)
        assert staged[:, 8].any() and not staged[:, 4:7].any()
        oo.check_staged(g, staged, pose)
        down = oo.check_down(g, staged, 0.3, pose)
        _effect_pass(g, down, pose)
        assert oo.check_effect(g, down, pose) > 0
    g.close()


@pytest.mark.parametrize("lidar_type", [2, 3])
def test_pcl2_subframes(Emul, lidar_type):
    rng = np.random.default_rng(5)
    g = Emul(0.5, max_map_points=50_000, max_scan_points=8000)
    data, lay, n = scenes.spinning_pcl2(lidar_type, 16, 300, stamp=50.0, seed=lidar_type, with_time=True, nan_frac=0.02, zero_frac=0.02)
    got = g.frame_cut_pcl2(data, lay, n, lidar_type, N_SCANS=16, blind=0.5, point_filter_num=1, required_frame_num=2, scan_count=25, stamp=50.0)
    assert len(got) == 2
    for s in got:
        p12 = g.frame_download(s["handle"])
        g.frame_stage(s["handle"])
        staged = oo.staged_records(g, p12)
        pose = _pose(rng)
        oo.check_staged(g, staged, pose)
        oo.check_down(g, staged, 0.5, pose)
    g.close()


def test_interleaved_downloads_change_nothing(Emul):
    """The same scan twice, once with every cloud downloaded between the steps: the resident scan, the passes and the map are
    identical."""
    rng = np.random.default_rng(6)
    raw = _timed_raw(2500, seed=13)
    pose = _pose(rng)
    res = []
    for interleave in (False, True):
        g = Emul(0.3, max_map_points=50_000, max_scan_points=4000)

        def dl():
            if interleave:
                for w in (1, 2, 3, 4):
                    try:
                        g.cloud(w, *pose)
                    except emul.EmulError as e:
                        assert e.code == -1
        g.raw_upload(raw, 9)
        dl()
        g.raw_undistort_cv(np.array([0.02, -0.01, 0.3]), np.eye(3), np.array([0.4, 0.1, 0.0]))
        dl()
        g.raw_downsample(0.3)
        dl()
        body = g.scan_body()
        g.map_build(oo.to_world(oo.records(body), *pose)[:, 0:3] + np.float32(0.02))
        dl()
        passes = []
        for it in range(3):
            passes.append(g.icp_iterate(*pose, False, it != 1))
            dl()
        na = g.map_incremental(*pose, 0.3)
        dl()
        res.append((body, passes, na, g.map_download(), g.scan_state()))
        g.close()
    a, b = res
    np.testing.assert_array_equal(a[0], b[0])
    for x, y in zip(a[1], b[1]):
        for u, v in zip(x, y):
            np.testing.assert_array_equal(u, v)
    assert a[2] == b[2]
    np.testing.assert_array_equal(np.sort(a[3].view(np.uint32), axis=0), np.sort(b[3].view(np.uint32), axis=0))
    sel = a[4]["selected"].astype(bool)
    for k in a[4]:   # (the normal of a point the pass did not select is not defined)
        np.testing.assert_array_equal(a[4][k][sel] if k == "normvec" else a[4][k], b[4][k][sel] if k == "normvec" else b[4][k])


def test_error_contract(Emul):
    rng = np.random.default_rng(7)
    g = Emul(0.3, max_map_points=50_000, max_scan_points=4000)
    pose = [np.ascontiguousarray(x, np.float64).reshape(-1) for x in _pose(rng)]
    ptrs = [x.ctypes.data_as(emul.vp) for x in pose]
    n = C.c_int(-5)

    def call(which, out=None, cap=0, p=ptrs):
        return g.L.liinit_cloud_download(g.h, which, *p, None if out is None else out.ctypes.data_as(emul.vp), cap, C.byref(n))

    for w in (1, 2, 3, 4):                     # nothing staged, no scan
        assert call(w) == -1
    for w in (0, 5, -1):
        assert call(w) == -1
    raw = _timed_raw(1200, seed=14)
    g.raw_upload(raw, 9)
    assert call(1) == 0 and n.value == 1200 and call(3, p=[None] * 4) == 0 and n.value == 1200
    assert call(1, p=[None] * 4) == -1         # a world cloud needs the pose
    assert call(2) == -1 and call(4) == -1     # no resident scan yet
    out = np.full((1199, 12), 7.0, np.float32)
    assert call(1, out, 1199) == -3 and (out == 7.0).all()
    assert call(3, out, 1199) == -3 and (out == 7.0).all()
    nd = g.raw_downsample(0.3)
    assert call(2) == 0 and n.value == nd
    assert call(4) == -1                       # no ICP pass on the resident scan yet
    small = np.full((nd - 1, 12), 7.0, np.float32)
    assert call(2, small, nd - 1) == -3 and (small == 7.0).all()
    down = oo.voxel_grid(oo.staged_records(g, raw), 0.3)
    _effect_pass(g, down, pose)
    assert call(4) == 0 and n.value > 1
    m = n.value
    e = np.full((m - 1, 12), 7.0, np.float32)
    assert call(4, e, m - 1) == -3 and (e == 7.0).all()
    e = np.zeros((m, 12), np.float32)
    assert call(4, e, m) == 0 and n.value == m
    g.map_build(np.zeros((1, 3), np.float32))   # the staging buffer is taken by the map build: no staged cloud any more
    assert call(1) == -1 and call(3) == -1 and call(2) == 0
    g.close()


# ---- the publish stage of the loop ---------------------------------------------------------------------------------------------------
def test_pcd_header_and_offsets(tmp_path):
    rng = np.random.default_rng(8)
    rec = rng.normal(size=(37, 12)).astype(np.float32)
    rec[:, [3]] = 1.0
    rec[:, [7, 10, 11]] = 0.0
    path = str(tmp_path / "a.pcd")
    assert pcd.write_binary(path, rec) == 37
    hdr, arr, raw = oo.read_pcd(path)
    assert hdr["VERSION"] == ["0.7"] and hdr["WIDTH"] == ["37"] and hdr["HEIGHT"] == ["1"] and hdr["VIEWPOINT"] == "0 0 0 1 0 0 0".split()
    assert hdr["FIELDS"] == "x y z _ normal_x normal_y normal_z _ intensity curvature _".split()
    assert raw.shape == (37, capi.POINTCLOUD2_POINT_STEP)
    for name, off, dtype, count in capi.POINTCLOUD2_FIELDS:
        assert dtype == 7 and count == 1
        np.testing.assert_array_equal(arr[name], rec[:, off // 4])
        assert arr.dtype.fields[name][1] == off   # the PCD layout puts every field at its PointCloud2 offset
    np.testing.assert_array_equal(raw.view(np.float32), rec)
    assert open(path, "rb").read().startswith(b"# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\n")


def _lio_publish_legs(oracle_mod, publish):
    import lio_case
    from lidar_imu_init_b200.odometry import LidarOdometry
    Emul = _bind()
    kw = dict(max_iteration=4, orig_odom_freq=10, cut_frame_num=5)

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

        def _stage(self, raw):
            self.staged_raw = raw
            super()._stage(raw)

        def _map_build(self, world):
            super()._map_build(world)
            self.map_builds = getattr(self, "map_builds", 0) + 1
    legs = {"oracle": lio_case.make_oracle_odometry(oracle_mod, 0.15, lio_case.default_threads(), **kw),
            "product": EmulOdometry(Emul(0.15, max_map_points=400_000, max_scan_points=316), 0.15, publish=publish, **kw)}
    return lio_case, legs


def test_lio_lockstep_publishes(built, oracle_mod, tmp_path):
    """The 30-scan LIO lockstep of test_lio_host with publishing and pcd_save (interval 3): at every scan the three clouds equal the
    checker on the device's staged cloud and flags with the posterior; the effect count equals effect_feat_num; the switch scan
    republishes the previous cloud with the new pose; every PCD<k>.pcd holds the REGISTERED records of its three scans."""
    from lidar_imu_init_b200 import host
    from lidar_imu_init_b200.odometry import Publish
    lio_case, legs = _lio_publish_legs(oracle_mod, Publish(pcd_save_en=True, interval=3, pcd_dir=str(tmp_path / "PCD")))
    pr = legs["product"]
    seen = dict(scans=0, eff=0, regs=[], switch=None, prev_raw=None)

    def on_scan(j, legs, truth):
        g = pr.g
        pose = host.state_pose(pr.state)
        pub = pr.published
        seen["scans"] += 1
        assert set(pub) == {"registered", "body", "effect"}
        staged = oo.staged_records(g, pr.staged_raw)
        oo.assert_bits(pub["registered"], oo.to_world(staged, *pose), "REGISTERED")
        oo.assert_bits(pub["body"], oo.frame_body(staged), "BODY")
        down = oo.voxel_grid(staged, pr.filter_size_surf)
        sel = g.scan_state()["selected"]
        oo.assert_bits(pub["effect"], oo.effect(down, sel, *pose), "EFFECT")
        assert len(pub["effect"]) == pr.stats["effect_feat_num"] == len(g.scan_effect()[0])
        np.testing.assert_array_equal(pub["effect"][:, 8], np.float32(np.sqrt(1000.0)))
        if pr.switch_scan is not None and seen["switch"] is None:
            seen["switch"] = j
            assert pr.staged_raw is seen["prev_raw"]   # the cloud of the previous scan, with the new pose
        seen["prev_raw"] = pr.staged_raw
        seen["regs"].append(pub["registered"])
        seen["eff"] += len(pub["effect"])

    out = lio_case.run(legs, oracle_mod, seconds=0.7, points=300, t_start=8.0, scans=30, map_from_scene=True, on_scan=on_scan)
    assert out["switch_scan"] == out["init_scan"] + 1 and seen["switch"] is not None and seen["scans"] == 30 and seen["eff"] > 1000
    pr.close()
    files = sorted(os.listdir(tmp_path / "PCD"), key=lambda f: int(f[3:-4]))
    assert files == [f"PCD{k}.pcd" for k in range(1, 11)]
    for k, f in enumerate(files):
        _, _, raw = oo.read_pcd(str(tmp_path / "PCD" / f))
        np.testing.assert_array_equal(raw.view(np.float32), np.concatenate(seen["regs"][3 * k:3 * k + 3]))


class _FakeGpu:
    """Clouds whose content names the scan and the call: enough to check the node logic of the publish stage."""

    def __init__(self):
        self.scan = 0
        self.calls = []

    def cloud(self, which, *pose):
        self.calls.append((self.scan, which))
        r = np.zeros((self.scan % 3 + 1, 12), np.float32)
        r[:, 0] = self.scan
        r[:, 1] = which
        return r


@pytest.mark.parametrize("interval", [1, 3, -1])
def test_pcd_save_sequence(built, tmp_path, interval):
    from lidar_imu_init_b200.odometry import LidarOdometry
    d = tmp_path / "PCD"
    o = LidarOdometry(_FakeGpu(), 0.5, publish=dict(pcd_save_en=True, interval=interval, pcd_dir=str(d)))
    regs = []
    for k in range(8):
        o.g.scan = k
        o._publish(np.eye(3), np.zeros(3), np.eye(3), np.zeros(3))
        regs.append(o.published["registered"])
    files = sorted(os.listdir(d), key=lambda f: f) if d.exists() else []
    if interval > 0:
        want = {f"PCD{k + 1}.pcd": np.concatenate(regs[interval * k:interval * (k + 1)]) for k in range(8 // interval)}
    else:
        assert files == []
        o.close()
        want = {"PCD_all.pcd": np.concatenate(regs)}
    o.close()
    assert sorted(os.listdir(d)) == sorted(want)
    for f, w in want.items():
        np.testing.assert_array_equal(oo.read_pcd(str(d / f))[2].view(np.float32), w)


def test_publish_conditions(built):
    """:1152-1156: REGISTERED with dense_pub_en else REGISTERED_DOWN; pcd_save takes REGISTERED even when the topic does not; BODY only
    with scan_pub_en and scan_body_pub_en; EFFECT always. Off by default."""
    from lidar_imu_init_b200.odometry import LidarOdometry
    assert LidarOdometry(_FakeGpu(), 0.5).publish is None
    pose = (np.eye(3), np.zeros(3), np.eye(3), np.zeros(3))
    cases = [(dict(), [1, 3, 4]), (dict(dense_pub_en=False), [2, 3, 4]), (dict(scan_body_pub_en=False), [1, 4]),
             (dict(scan_pub_en=False), [4]), (dict(scan_pub_en=False, pcd_save_en=True), [1, 4]),
             (dict(dense_pub_en=False, pcd_save_en=True), [2, 1, 3, 4]), (dict(pcd_save_en=True), [1, 3, 4])]
    for prm, calls in cases:
        o = LidarOdometry(_FakeGpu(), 0.5, publish=dict(prm, interval=10 ** 6))
        o._publish(*pose)
        assert [w for _, w in o.g.calls] == calls, prm
        assert ("registered" in o.published) == prm.get("scan_pub_en", True)
        assert ("body" in o.published) == (prm.get("scan_pub_en", True) and prm.get("scan_body_pub_en", True))


def test_no_clouds_on_the_map_build_scan(Emul, built):
    from lidar_imu_init_b200.odometry import LidarOdometry, Publish

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

    o = EmulOdometry(Emul(0.3, max_map_points=50_000, max_scan_points=4000), 0.3, publish=Publish())
    raw = _timed_raw(1500, seed=15)
    o.process_raw(raw, 10.0)
    assert o.map_ready and o.published == {}
    o.process_raw(raw, 10.1)
    assert set(o.published) == {"registered", "body", "effect"} and len(o.published["registered"]) == 1500
