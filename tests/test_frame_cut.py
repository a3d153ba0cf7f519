"""CPU tests of the cut-frame preprocess (Preprocess::process_cut_frame_livox / _pcl2): the literal checker (tests/cpp/frame_oracle.cpp)
against hand-worked messages, one per rule of the reference that is easy to get wrong, and the product's kernels and entry points on
the CPU build of the device library (tests/emul) against the checker, bit for bit."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import frame_oracle as fo  # noqa: E402
from lidar_imu_init_b200 import capi, scenes  # noqa: E402


def lvx(rows):
    """rows of (offset_time ns, x, y, z[, tag, line]) -> Livox records, reflectivity = row index"""
    m = np.zeros(len(rows), capi.LIVOX_POINT)
    for i, r in enumerate(rows):
        m[i]["offset_time"], m[i]["x"], m[i]["y"], m[i]["z"] = r[0], r[1], r[2], r[3]
        m[i]["tag"] = r[4] if len(r) > 4 else 0x10
        m[i]["line"] = r[5] if len(r) > 5 else 0
        m[i]["reflectivity"] = i
    return m


def kept(subs):
    """reflectivities (= record indices) of all output points, in output order"""
    return [int(v) for s in subs for v in s["pts"][:, 3]]


# ---- the checker against hand-worked messages --------------------------------------------------------------------------------------
def test_raw_zero_and_sorted_zero_are_dropped():
    # record 0 is never looked at; of the rest, the earliest point after the sort is dropped
    m = lvx([(0, 5, 0, 0), (4000, 6, 0, 0), (1000, 7, 0, 0), (3000, 8, 0, 0), (2000, 9, 0, 0)])
    subs = fo.cut_livox(m)
    assert kept(subs) == [4, 3, 1]


def test_no_subframe_below_twice_the_cut():
    rows = [(1000 * i, 5 + i, 0, 0) for i in range(8)]
    for V, want in ((5, 0), (6, 3), (3, 0), (7, 3)):
        subs = fo.cut_livox(lvx(rows[:V + 1]), required_frame_num=3, scan_count=5)
        assert len(subs) == want, V
    # before the scan_count threshold there is one cut per message, at any V >= 2
    assert len(fo.cut_livox(lvx(rows[:6]), required_frame_num=3, scan_count=4)) == 1
    assert len(fo.cut_livox(lvx(rows[:2]), required_frame_num=3, scan_count=4)) == 0


def test_scan_count_threshold():
    rows = [(1000 * i, 5 + i, 0, 0) for i in range(13)]
    assert len(fo.cut_livox(lvx(rows), required_frame_num=4, scan_count=4)) == 1
    assert len(fo.cut_livox(lvx(rows), required_frame_num=4, scan_count=5)) == 4
    data, lay, n = scenes.spinning_pcl2(3, 8, 40)
    assert len(fo.cut_pcl2(data, lay, n, 3, required_frame_num=4, scan_count=19)) == 1
    assert len(fo.cut_pcl2(data, lay, n, 3, required_frame_num=4, scan_count=20)) == 4


def test_filter_counter_advances_on_blind_points():
    # point_filter_num 2: records 1..6 valid, record 2 inside the blind zone. The counter counts it: records 2, 4, 6 are taken and 2
    # is then dropped -> {4, 6}, sorted index 0 (record 4) dropped -> [6]. A counter that skipped blind points would take 3 and 5.
    m = lvx([(0, 5, 0, 0), (1000, 5, 1, 0), (2000, 0.1, 0, 0), (3000, 5, 2, 0), (4000, 5, 3, 0), (5000, 5, 4, 0), (6000, 5, 5, 0)])
    assert kept(fo.cut_livox(m, point_filter_num=2, blind=1.0)) == [6]


def test_duplicate_against_zero_slot():
    # blind 0: a point at the origin is kept by the blind test. Record 2 is invalid (noise tag): pl_full[2] stays (0,0,0), so record 3
    # at the origin is a duplicate of that slot and dropped, although record 2's own coordinates differ. Record 5 repeats record 4
    # (taken): dropped. Record 7 repeats record 6, which was not taken (bad line): kept.
    m = lvx([(0, 1, 1, 1), (1000, 3, 0, 0), (2000, 2, 2, 2, 0x20), (3000, 0, 0, 0), (4000, 4, 4, 4), (5000, 4, 4, 4), (6000, 6, 6, 6, 0x10, 9),
             (7000, 6, 6, 6), (8000, 8, 0, 0)])
    assert kept(fo.cut_livox(m, blind=0.0)) == [4, 7, 8]


def test_sub_metre_differences_are_not_duplicates():
    # abs() is the float overload: consecutive points 0.5 m apart are distinct (an int abs would truncate the difference to 0);
    # points 1e-8 apart are duplicates
    m = lvx([(0, 1, 1, 1), (1000, 5, 0, 0), (2000, 5.5, 0, 0), (3000, 5.5, 0.25, 0), (4000, 5.5, 0.25, 1e-8 + 0.0), (5000, 5.5, 0.25, 0.75)])
    assert kept(fo.cut_livox(m)) == [2, 3, 5]


def test_time_chain():
    # t_beg_k = lfet_k / 1000, curvature' = float(curvature + (stamp*1000 - lfet_k)), lfet_{k+1} = lfet_k + curvature'(boundary)
    stamp = 1234.5678
    offs = [0, 7_000_001, 13_000_003, 29_999_999, 41_000_000, 55_555_555, 71_000_017, 88_000_001, 99_999_999]
    m = lvx([(o, 5 + i, i, 0) for i, o in enumerate(offs)])
    subs = fo.cut_livox(m, required_frame_num=2, scan_count=9, stamp=stamp)
    assert len(subs) == 2
    c = [np.float32(o) / np.float32(1e6) for o in offs[2:]]     # sorted points 1.. (record 1 is sorted index 0)
    S = stamp * 1000
    V = len(offs) - 1
    t0 = int(1 * V / 2) - 1
    lfet = S
    want, ends, begs = [], [], []
    for k, (lo, hi) in enumerate(((0, t0), (t0, V - 1))):
        begs.append(lfet / 1000.0)
        seg = [np.float32(np.float64(x) + (S - lfet)) for x in c[lo:hi]]
        want += seg
        ends.append(seg[-1])
        lfet += np.float64(seg[-1])
    got = np.concatenate([s["pts"][:, 4] for s in subs])
    np.testing.assert_array_equal(got.view(np.uint32), np.array(want, np.float32).view(np.uint32))
    assert [s["t_beg"] for s in subs] == begs
    assert [s["end_ms"] for s in subs] == ends
    assert subs[1]["pts"][0, 4] < subs[0]["pts"][-1, 4]   # the second sub-frame starts again near 0


def _velodyne(rows, with_time=False):
    """rows of (x, y, ring) -> Velodyne PointCloud2 bytes without a time field"""
    lay = dict(scenes.PCL2_FIELDS[2])
    if not with_time:
        lay["off_time"] = -1
    buf = np.zeros((len(rows), lay["point_step"]), np.uint8)
    for i, (x, y, r) in enumerate(rows):
        buf[i, 0:4] = np.frombuffer(np.float32(x).tobytes(), np.uint8)
        buf[i, 4:8] = np.frombuffer(np.float32(y).tobytes(), np.uint8)
        buf[i, 16:20] = np.frombuffer(np.float32(i).tobytes(), np.uint8)   # intensity = index
        buf[i, 24:26] = np.frombuffer(np.uint16(r).tobytes(), np.uint8)
    return buf.reshape(-1), lay, len(rows)


def test_rotation_model_wrap_and_first_point():
    # ring 0 at yaw 10, 5, 0, 7, -10, -20 deg; ring 1 at 3, 2. The first point of each ring sets yaw_fp and is dropped. Ring 0 descends
    # at yaw 7 (base 3/3.61 < 10/3.61): it and every later point of the ring get +360/3.61.
    d = np.deg2rad
    rows = [(10 * np.cos(d(a)), 10 * np.sin(d(a)), r) for a, r in ((10, 0), (3, 1), (5, 0), (0, 0), (2, 1), (7, 0), (-10, 0), (-20, 0))]
    data, lay, n = _velodyne(rows)
    subs = fo.cut_pcl2(data, lay, n, 2, N_SCANS=4)
    # bases (yaw_fp - yaw) / 3.61: record 4 (ring 1) 0.28, 2: 1.39, 3: 2.77, then 5: 0.83 < 2.77 -> wrapped, and 6, 7 after it
    assert kept(subs) == [2, 3, 5, 6, 7]   # sorted index 0 (record 4) dropped
    t = dict(zip(kept(subs), subs[0]["pts"][:, 4]))
    wrap = 360.0 / 3.61
    assert t[2] < t[3] < wrap
    assert abs(t[5] - (3 / 3.61 + wrap)) < 1e-4 and abs(t[6] - (20 / 3.61 + wrap)) < 1e-4 and abs(t[7] - (30 / 3.61 + wrap)) < 1e-4
    # with a time field whose last value is positive the rotation model is off: no point is dropped as a ring's first
    data2, lay2, _ = _velodyne(rows, with_time=True)
    b = data2.reshape(n, -1)
    for i in range(n):
        b[i, 20:24] = np.frombuffer(np.float32(0.001 * (i + 1)).tobytes(), np.uint8)
    assert kept(fo.cut_pcl2(b.reshape(-1), lay2, n, 2, N_SCANS=4)) == [1, 2, 3, 4, 5, 6, 7]


def test_rotation_model_rejects_ring_128():
    data, lay, n = _velodyne([(5, 0, 0), (5, 1, 128), (5, 2, 0)])
    assert fo.cut_pcl2(data, lay, n, 2, N_SCANS=4) is None


# ---- the product on the CPU build of the device library -----------------------------------------------------------------------------
emul = pytest.importorskip("liinit_emul")


@pytest.fixture(scope="module")
def eg():
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    L = emul.load()
    vp = emul.vp
    import ctypes as C
    L.liinit_frame_cut_livox.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int, C.POINTER(C.c_int)]
    L.liinit_frame_cut_pcl2.argtypes = [vp, vp, C.POINTER(capi.Pcl2Layout), C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int,
                                        C.POINTER(C.c_int)]
    L.liinit_frame_stage.argtypes = [vp, C.c_longlong]
    L.liinit_frame_download.argtypes = [vp, C.c_longlong, vp, C.c_int, C.POINTER(C.c_int)]

    class EmulFrame(emul.EmulGpu):   # the product's binding methods over the emulated library
        frame_cut_livox = capi.LiInitGpu.frame_cut_livox
        frame_cut_pcl2 = capi.LiInitGpu.frame_cut_pcl2
        frame_stage = capi.LiInitGpu.frame_stage
        frame_download = capi.LiInitGpu.frame_download
        frame_size = capi.LiInitGpu.frame_size

    return EmulFrame(0.5, max_map_points=1000, max_scan_points=4000)


def test_emul_livox_matches_checker(eg):
    # the first of the GPU test's random messages
    rng = np.random.Generator(np.random.PCG64(fo.LIVOX_SEED))
    for _ in range(16):
        m, prm = fo.random_livox(rng)
        want = fo.cut_livox(m, **prm)
        got = eg.frame_cut_livox(m, **prm)
        fo.compare(got, [eg.frame_download(s["handle"]) for s in got], want)


@pytest.mark.parametrize("lidar_type,with_time", [(2, True), (2, False), (3, True), (5, True), (6, True), (6, False)])
def test_emul_pcl2_matches_checker(eg, lidar_type, with_time):
    data, lay, n = scenes.spinning_pcl2(lidar_type, 12, 60, stamp=100.0, seed=lidar_type, with_time=with_time, turns=1.05, nan_frac=0.03,
                                        zero_frac=0.03, extra_pad=4)
    prm = dict(N_SCANS=10, blind=0.5, point_filter_num=2, required_frame_num=3, scan_count=25, stamp=100.0)
    want = fo.cut_pcl2(data, lay, n, lidar_type, **prm)
    got = eg.frame_cut_pcl2(data, lay, n, lidar_type, **prm)
    nb, moved = fo.compare(got, [eg.frame_download(s["handle"]) for s in got], want, curv_tol_ms=0.0 if with_time else fo.YAW_TOL_MS)
    print(f"type {lidar_type} time field {with_time}: {nb} curvatures not bit-equal, {moved} points in another order")
    if with_time or lidar_type in (3, 5):
        assert nb == 0 and moved == 0


def test_emul_stage_equals_raw_upload(eg):
    rng = np.random.Generator(np.random.PCG64(5))
    m, prm = fo.random_livox(rng)
    while len(fo.cut_livox(m, **prm)) == 0:
        m, prm = fo.random_livox(rng)
    got = eg.frame_cut_livox(m, **prm)
    h = got[len(got) // 2]["handle"]
    p12 = eg.frame_download(h)
    eg.frame_stage(h)
    a = eg.raw_points()
    eg.raw_upload(p12, 9)
    b = eg.raw_points()
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def test_emul_errors_leave_state(eg):
    rng = np.random.Generator(np.random.PCG64(8))
    m, prm = fo.random_livox(rng)
    while len(fo.cut_livox(m, **prm)) == 0:
        m, prm = fo.random_livox(rng)
    got = eg.frame_cut_livox(m, **prm)
    before = eg.frame_download(got[0]["handle"])
    with pytest.raises(emul.EmulError) as e:   # more points than the staging capacity (2^20)
        eg.frame_cut_livox(np.zeros((1 << 20) + 1, capi.LIVOX_POINT), **prm)
    assert e.value.code == -3
    with pytest.raises(emul.EmulError) as e:
        eg.frame_cut_livox(m, **dict(prm, point_filter_num=0))
    assert e.value.code == -1
    data, lay, n = _velodyne([(5, 0, 0), (5, 1, 128), (5, 2, 0), (5, 3, 0)])
    with pytest.raises(emul.EmulError) as e:
        eg.frame_cut_pcl2(data, lay, n, 2, N_SCANS=4)
    assert e.value.code == -1
    assert eg.frame_cut_livox(m[:0], **prm) == []
    np.testing.assert_array_equal(eg.frame_download(got[0]["handle"]), before)
    # a handle outlives LIINIT_FRAME_SLOTS later messages at most
    for _ in range(4):
        eg.frame_cut_livox(m, **prm)
    with pytest.raises(emul.EmulError) as e:
        eg.frame_stage(got[0]["handle"])
    assert e.value.code == -1


def _rotation_boundary_rows():
    # ring 0: yaw 0 (first, dropped), -10 deg (base 2.77), 0 (base 0 < 2.77: the first descent, wrapped to float(360/3.61)), then a yaw
    # 5.7e-6 deg above the first whose base rounds to float(360/3.61) itself: not below time_last, so the reference does NOT wrap it;
    # then -20 deg (base 5.54 < time_last: wrapped)
    d = np.deg2rad
    return [(10.0, 0.0, 0), (10 * np.cos(d(-10)), 10 * np.sin(d(-10)), 0), (10.0, 0.0, 0), (10.0, 1e-6, 0),
            (10 * np.cos(d(-20)), 10 * np.sin(d(-20)), 0)]


def test_rotation_model_base_at_the_wrap_value():
    data, lay, n = _velodyne(_rotation_boundary_rows())
    t = dict(zip(kept(fo.cut_pcl2(data, lay, n, 2, N_SCANS=4)), fo.cut_pcl2(data, lay, n, 2, N_SCANS=4)[0]["pts"][:, 4]))
    W = np.float32(360.0 / 3.61)
    assert t[2] == W and t[3] == W and abs(t[4] - (20 / 3.61 + 360 / 3.61)) < 1e-4


def test_emul_rotation_model_base_at_the_wrap_value(eg):
    data, lay, n = _velodyne(_rotation_boundary_rows())
    want = fo.cut_pcl2(data, lay, n, 2, N_SCANS=4)
    got = eg.frame_cut_pcl2(data, lay, n, 2, N_SCANS=4)
    assert fo.compare(got, [eg.frame_download(s["handle"]) for s in got], want) == (0, 0)


def test_emul_callbacks(eg):
    """The LiDAR callbacks of LidarOdometry over the emulated library: the scan_count threshold of PointCloud2 (one sub-frame before
    the 20th message), the loop-back clear, the one-time self sync of the IMU clock, sub-frames whose slot was reused skipped before
    anything changes, and cut_frame_num = 2 for spinning sensors after the hand-over (Livox keeps its own)."""
    from lidar_imu_init_b200 import _build
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    o = LidarOdometry(eg, 0.5, cut_frame_num=3)
    o.preprocess = dict(lidar_type=3, N_SCANS=8, blind=0.5, point_filter_num=1)
    data, lay, n = scenes.spinning_pcl2(3, 8, 60, stamp=10.0)
    o.imu_buffer.push(1000.0, [0, 0, 0], [0, 0, 9.81])   # IMU clock 990 s ahead of the LiDAR's
    for k in range(19):
        o.lidar_cbk_pcl2(data, lay, n, 10.0 + 0.1 * k)
        if k == 0:
            assert o.timediff_set and o.imu_buffer.timediff == 1000.0 - 10.0
    assert o.imu_buffer.timediff == 990.0 and o.scan_count == 19 and len(o.lidar_buffer) == 19
    o.lidar_cbk_pcl2(data, lay, n, 12.0)
    assert len(o.lidar_buffer) == 22                    # the 20th message: cut_frame_num sub-frames
    # only the last LIINIT_FRAME_SLOTS messages are on the device: process_next skips the older entries before any state changes
    o.imu_buffer.rows.clear()
    state = o.state.copy()
    assert o.process_next() is None
    assert o.dropped_subframes == 16 and len(o.lidar_buffer) == 6 and (o.state == state).all()
    o.lidar_cbk_pcl2(data, lay, n, 11.0)                # loop back: the buffer is cleared first
    assert len(o.lidar_buffer) == 3
    res = dict(R_LI=np.eye(3), T_LI=np.zeros(3), grav_L0=np.array([0, 0, -9.81]), gyro_bias=np.zeros(3), acc_bias=np.zeros(3),
               time_lag_1=0.0, time_lag_2=0.0)
    o.hand_over(res)
    assert o.cut_frame_num == 2
    o.lidar_cbk_pcl2(data, lay, n, 12.5)
    assert len(o.lidar_buffer) == 5
    lv = LidarOdometry(eg, 0.5, cut_frame_num=3)
    lv.hand_over(res)
    assert lv.cut_frame_num == 3
