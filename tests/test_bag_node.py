"""The bag runner on the CPU: the ROS1 bag reader against a bag writer built from the format (round trips, delivery order, bags cut
off mid-recording, the errors), the three message decoders, the node's output formats pinned on the reference's own logs
(tests/golden/reference_*), the config loader, the refinement clock, and a short Node run on the emulated device library that must
equal the same messages pushed straight into LidarOdometry."""
import bz2
import ctypes as C
import os
import struct
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lidar_imu_init_b200 import capi, config, node, rosbag, rosmsg, scenes  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


# ---- a ROS1 bag v2.0 writer (test infrastructure) ----------------------------------------------------------------------------------
def _record(fields, data=b""):
    h = b""
    for k, v in fields.items():
        f = k.encode() + b"=" + v
        h += struct.pack("<I", len(f)) + f
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def _conn_record(cid, topic, type_):
    body = b"".join(struct.pack("<I", len(f)) + f for f in (b"topic=" + topic.encode(), b"type=" + type_.encode(),
                                                           b"md5sum=" + b"0" * 32, b"message_definition=" + b"# test\n"))
    return _record({"op": b"\x07", "conn": struct.pack("<I", cid), "topic": topic.encode()}, body)


def write_bag(path, conns, chunks, index=True, cut=None):
    """conns {id: (topic, type)}; chunks [(compression, [(conn, sec, nsec, data bytes)])], written in this order. index=False: no
    index data, connections or chunk infos after the chunks and index_pos 0 (a recording that was never closed). cut: keep only
    the first `cut` bytes. Returns [(conn, sec, nsec, data)] in file order."""
    body, infos, seen, order = b"", [], set(), []
    pos0 = len(rosbag.MAGIC) + 4096
    for comp, msgs in chunks:
        inner, offs = b"", {}
        for cid, sec, nsec, data in msgs:
            if cid not in seen:
                seen.add(cid)
                inner += _conn_record(cid, *conns[cid])
            offs.setdefault(cid, []).append((sec, nsec, len(inner)))
            inner += _record({"op": b"\x02", "conn": struct.pack("<I", cid), "time": struct.pack("<II", sec, nsec)}, data)
            order.append((cid, sec, nsec, data))
        payload = {"none": lambda b: b, "bz2": bz2.compress, "lz4": lambda b: b"\x04\x22\x4d\x18" + b}[comp](inner)
        chunk_pos = pos0 + len(body)
        body += _record({"op": b"\x05", "compression": comp.encode(), "size": struct.pack("<I", len(inner))}, payload)
        if index:
            for cid, entries in offs.items():
                body += _record({"op": b"\x04", "ver": struct.pack("<I", 1), "conn": struct.pack("<I", cid), "count": struct.pack("<I", len(entries))},
                                b"".join(struct.pack("<III", *e) for e in entries))
        times = [s * 10**9 + n for _, s, n, _ in msgs]
        infos.append((chunk_pos, min(times), max(times), {c: len(e) for c, e in offs.items()}))
    index_pos = pos0 + len(body) if index else 0
    if index:
        for cid, (topic, type_) in conns.items():
            body += _conn_record(cid, topic, type_)
        for cpos, t0, t1, counts in infos:
            body += _record({"op": b"\x06", "ver": struct.pack("<I", 1), "chunk_pos": struct.pack("<Q", cpos),
                             "start_time": struct.pack("<II", t0 // 10**9, t0 % 10**9), "end_time": struct.pack("<II", t1 // 10**9, t1 % 10**9),
                             "count": struct.pack("<I", len(counts))}, b"".join(struct.pack("<II", c, n) for c, n in counts.items()))
    hdr = _record({"op": b"\x03", "index_pos": struct.pack("<Q", index_pos), "conn_count": struct.pack("<I", len(conns)),
                   "chunk_count": struct.pack("<I", len(chunks))})
    hdr = _record({"op": b"\x03", "index_pos": struct.pack("<Q", index_pos), "conn_count": struct.pack("<I", len(conns)),
                   "chunk_count": struct.pack("<I", len(chunks))}, b" " * (4096 - len(hdr)))
    out = rosbag.MAGIC + hdr + body
    with open(path, "wb") as f:
        f.write(out if cut is None else out[:cut])
    return order


# ---- message serializers (test infrastructure) ----
def _header(stamp_sec, stamp_nsec, frame="f"):
    return struct.pack("<III", 7, stamp_sec, stamp_nsec) + struct.pack("<I", len(frame)) + frame.encode()


def ser_imu(sec, nsec, gyr, acc):
    return (_header(sec, nsec) + struct.pack("<4d", 0, 0, 0, 1) + struct.pack("<9d", *range(9)) + struct.pack("<3d", *gyr) + struct.pack("<9d", *range(9))
            + struct.pack("<3d", *acc) + struct.pack("<9d", *range(9)))


def ser_livox(sec, nsec, pts):
    a = np.ascontiguousarray(pts.astype(capi.LIVOX_POINT))
    return _header(sec, nsec) + struct.pack("<QIB", 123, len(a), 1) + b"\0\0\0" + struct.pack("<I", len(a)) + a.tobytes()


def ser_pcl2(sec, nsec, fields, point_step, data, n, big=False):
    f = b"".join(struct.pack("<I", len(nm)) + nm.encode() + struct.pack("<IBI", off, dt, cnt) for nm, off, dt, cnt in fields)
    data = bytes(data)
    return (_header(sec, nsec) + struct.pack("<II", 1, n) + struct.pack("<I", len(fields)) + f + struct.pack("<B", int(big))
            + struct.pack("<II", point_step, point_step * n) + struct.pack("<I", len(data)) + data + b"\x01")


def split_time(t):
    """A stamp [s] as ROS time (sec, nsec), rounded to the nanosecond."""
    ns = int(round(t * 1e9))
    return ns // 10**9, ns % 10**9


# ---- reader ----
CONNS = {0: ("/imu", rosmsg.IMU_TYPE), 3: ("/lidar", rosmsg.LIVOX_TYPE)}


def _msgs(conn, times, tag):
    return [(conn, int(t) // 10**9, int(t) % 10**9, f"{tag}{i}".encode() * (i % 5 + 1)) for i, t in enumerate(times)]


def test_reader_none_and_bz2_round_trip(tmp_path):
    for comp in ("none", "bz2"):
        a = _msgs(0, np.arange(10) * 5_000_000 + 10**10, "i")
        b = _msgs(3, np.arange(3) * 33_000_000 + 10**10, "l")
        p = str(tmp_path / f"{comp}.bag")
        write_bag(p, CONNS, [(comp, sorted(a + b, key=lambda m: (m[1], m[2])))])
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            with rosbag.Bag(p) as bag:
                assert bag.topics() == {"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE}
                got = [(m.topic, m.sec, m.nsec, bytes(m.data)) for m in bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE})]
                only = [bytes(m.data) for m in bag.messages({"/lidar": rosmsg.LIVOX_TYPE})]
        want = sorted(a + b, key=lambda m: (m[1] * 10**9 + m[2]))
        assert [(CONNS[c][0], s, n, d) for c, s, n, d in want] == got
        assert only == [d for _, _, _, d in b]


def _interleaved(tmp_path, **kw):
    """Four chunks (none / bz2 mixed) whose IMU and LiDAR records are out of order across chunks, with time ties across connections
    and chunks."""
    rng = np.random.default_rng(5)
    t_imu = np.sort(rng.integers(0, 2_000_000_000, 80)) + 5 * 10**9
    t_lid = np.sort(rng.integers(0, 2_000_000_000, 12)) + 5 * 10**9
    t_lid[3] = t_imu[20]                         # ties across connections
    t_imu[41] = t_imu[40]                        # tie within a connection
    imu, lid = _msgs(0, t_imu, "i"), _msgs(3, t_lid, "l")
    chunks = [("none", imu[0:25] + lid[0:5]), ("bz2", lid[5:8] + imu[25:30] + imu[60:70]), ("none", imu[30:60] + lid[8:10]),
              ("bz2", imu[70:] + lid[10:])]
    p = str(tmp_path / "inter.bag")
    order = write_bag(p, CONNS, chunks, **kw)
    return p, order


def test_reader_order_across_chunks(tmp_path):
    p, order = _interleaved(tmp_path)
    want = [m for _, m in sorted(enumerate(order), key=lambda im: (im[1][1] * 10**9 + im[1][2], im[0]))]
    with rosbag.Bag(p) as bag:
        got = [(m.sec, m.nsec, bytes(m.data)) for m in bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE})]
    assert got == [(s, n, d) for _, s, n, d in want]
    assert [t for t in got] != [(s, n, d) for _, s, n, d in order]     # the file order is not the delivery order


def test_reader_without_index_and_truncated(tmp_path):
    p, order = _interleaved(tmp_path, index=False)
    full = open(p, "rb").read()
    key = lambda im: (im[1][1] * 10**9 + im[1][2], im[0])   # noqa: E731
    want = [m for _, m in sorted(enumerate(order), key=key)]
    with pytest.warns(rosbag.BagWarning, match="no index"):
        with rosbag.Bag(p) as bag:
            got = [(m.sec, m.nsec, bytes(m.data)) for m in bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE})]
    assert got == [(s, n, d) for _, s, n, d in want]
    # an indexed bag cut off inside its third chunk (uncompressed): the messages of the first two chunks and the complete records of
    # the third are delivered
    p2, order2 = _interleaved(tmp_path)
    data = open(p2, "rb").read()
    third = data.find(b"op=\x05", data.find(b"op=\x05", data.find(b"op=\x05") + 1) + 1)
    msg_starts = [i for i in range(third, len(data)) if data.startswith(b"op=\x02", i)]
    cut = msg_starts[10] + 30                    # inside the 11th record of the third chunk
    p3 = str(tmp_path / "cut.bag")
    open(p3, "wb").write(data[:cut])
    n_kept = 25 + 5 + 3 + 5 + 10 + 10
    kept = order2[:n_kept]
    want = [m for _, m in sorted(enumerate(kept), key=key)]
    with pytest.warns(rosbag.BagWarning, match="ends inside a record"):
        with rosbag.Bag(p3) as bag:
            got = [(m.sec, m.nsec, bytes(m.data)) for m in bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE})]
    assert got == [(s, n, d) for _, s, n, d in want]
    # cut inside a bz2 chunk: the records before the cut that the decompressor can give back
    p4 = str(tmp_path / "cut2.bag")
    second = data.find(b"op=\x05", data.find(b"op=\x05") + 1)
    open(p4, "wb").write(data[:second + 200])
    with pytest.warns(rosbag.BagWarning):
        with rosbag.Bag(p4) as bag:
            got = [bytes(m.data) for m in bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE})]
    assert sorted(got) == sorted(d for _, _, _, d in order2[:30])
    assert len(full) > 0


def test_reader_errors(tmp_path):
    p = str(tmp_path / "lz4.bag")
    write_bag(p, CONNS, [("none", _msgs(0, [10**9], "i")), ("lz4", _msgs(3, [2 * 10**9], "l"))])
    with rosbag.Bag(p) as bag:
        with pytest.raises(rosbag.BagError, match=r"chunk at byte \d+ is lz4.*rosbag decompress"):
            list(bag.messages({"/imu": rosmsg.IMU_TYPE, "/lidar": rosmsg.LIVOX_TYPE}))
        with pytest.raises(rosbag.BagError, match=r"no topic '/points'.*/imu \[sensor_msgs/Imu\]; /lidar \[livox_ros_driver/CustomMsg\]"):
            bag.check_topics({"/points": rosmsg.PCL2_TYPE})
        with pytest.raises(rosbag.BagError, match=r"topic '/lidar' carries livox_ros_driver/CustomMsg, expected sensor_msgs/PointCloud2"):
            bag.check_topics({"/lidar": rosmsg.PCL2_TYPE})
    q = str(tmp_path / "not.bag")
    open(q, "wb").write(b"#ROSBAG V1.2\n" + b"\0" * 100)
    with pytest.raises(rosbag.BagError, match="not a ROS1 bag v2.0"):
        rosbag.Bag(q)


# ---- decoders ----
def test_imu_and_livox_round_trip():
    st, g, a = rosmsg.decode_imu(ser_imu(1716257158, 901789000, [0.1, -0.2, 0.3], [9.7, 0.01, -0.5]))
    assert st == 1716257158 + 1e-9 * 901789000
    np.testing.assert_array_equal(g, [0.1, -0.2, 0.3])
    np.testing.assert_array_equal(a, [9.7, 0.01, -0.5])
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), lambda t: (np.broadcast_to(np.eye(3), (len(t), 3, 3)), np.zeros((len(t), 3))),
                             10.0, 500, seed=3, tie_frac=0.1)
    buf = ser_livox(10, 5, m)
    st, pts = rosmsg.decode_livox(buf)
    assert st == 10 + 5e-9 and pts.dtype == capi.LIVOX_POINT and pts.dtype.itemsize == 19
    assert pts.tobytes() == m.tobytes()
    assert np.shares_memory(pts, np.frombuffer(buf, np.uint8))   # a view of the message, no copy
    with pytest.raises(rosmsg.MsgError, match="bytes short"):
        rosmsg.decode_livox(buf[:-1])


# the drivers' PointCloud2 fields (the point structs of the drivers, every field they publish)
DRIVER_FIELDS = {
    2: (32, [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1), ("time", 20, 7, 1), ("ring", 24, 4, 1)]),
    3: (48, [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1), ("t", 20, 6, 1), ("reflectivity", 24, 4, 1), ("ring", 26, 2, 1),
             ("ambient", 28, 4, 1), ("range", 32, 6, 1)]),
    5: (48, [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1), ("timestamp", 24, 8, 1), ("ring", 32, 4, 1)]),
    6: (32, [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 2, 1), ("ring", 18, 4, 1), ("timestamp", 24, 8, 1)]),
}
TIME_NAME = {2: "time", 3: "t", 5: "timestamp", 6: "timestamp"}


@pytest.mark.parametrize("lidar_type", [2, 3, 5, 6])
@pytest.mark.parametrize("with_time", [True, False])
def test_pcl2_layouts(lidar_type, with_time):
    data, lay, n = scenes.spinning_pcl2(lidar_type, 16, 100, stamp=5.0, with_time=with_time)
    step, fields = DRIVER_FIELDS[lidar_type]
    if not with_time:
        fields = [f for f in fields if f[0] != TIME_NAME[lidar_type]]
    buf = ser_pcl2(5, 0, fields, step, data, n)
    st, d, got, m = rosmsg.decode_pcl2(buf, lidar_type)
    assert st == 5.0 and m == n and got == lay == dict(scenes.PCL2_FIELDS[lidar_type], **({} if with_time else {"off_time": -1}))
    assert d.tobytes() == data.tobytes() and np.shares_memory(d, np.frombuffer(buf, np.uint8))


def test_pcl2_rejections():
    data, lay, n = scenes.spinning_pcl2(2, 4, 10)
    step, fields = DRIVER_FIELDS[2]
    bad = [(f[0], f[1], 8 if f[0] == "time" else f[2], 1) for f in fields]
    with pytest.raises(rosmsg.MsgError, match="field 'time' is FLOAT64 x 1; lidar_type 2 expects FLOAT32"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, bad, step, data, n), 2)
    bad = [(f[0], f[1], 2 if f[0] == "ring" else f[2], 1) for f in fields]
    with pytest.raises(rosmsg.MsgError, match="field 'ring' is UINT8"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, bad, step, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="is_bigendian"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, fields, step, data, n, big=True), 2)
    with pytest.raises(rosmsg.MsgError, match="point_step 36"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, fields, 36, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="field 'ring' of lidar_type 2 is missing"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, [f for f in fields if f[0] != "ring"], step, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="field 'ring' is UINT16 x 1; lidar_type 3"):
        rosmsg.decode_pcl2(ser_pcl2(1, 0, fields, step, data, n), 3)


# ---- output formats on the reference's own logs ----
def _vals(line):
    return [float(x) for x in line.split("=")[1].split()]


def test_initialization_result_golden():
    text = open(os.path.join(GOLDEN, "reference_Initialization_result.txt")).read()
    out = ""
    for title, block in (("Initialization result:\n", text.split("Refinement result:\n")[0].split("Initialization result:\n")[1]),
                         ("Refinement result:\n", text.split("Refinement result:\n")[1])):
        L = block.splitlines()
        R = np.array([[float(x) for x in L[i].split()] for i in range(8, 11)])[:, :3]
        out += title + node.calib_result_text(_vals(L[0]), _vals(L[1]), float(L[2].split("=")[1]), _vals(L[3]), _vals(L[4]), _vals(L[5]), R)
    assert out == text
    assert "-0.019749  0.021451  0.170247" in out and "= 0.002907 0.001678 0.005512\n" in out


def test_mat_out_golden():
    rows = open(os.path.join(GOLDEN, "reference_mat_out_rows.txt")).read().splitlines(True)
    assert len(rows) >= 9 and sum(" 0 -0  0 " in r for r in rows) >= 3
    for r in rows:
        t = [float(x) for x in r.split()]
        assert len(t) == 25
        assert node.mat_out_row(t[0:3], t[3:6], t[6:9], t[9:12], t[12:15], t[15:18], t[18:21], t[21:24], t[24]) == r


def test_state_formats():
    """The state-side wrappers: RotMtoEuler's -0 on an identity extrinsic, the scaled accelerometer bias, tf's RPY quaternion."""
    from lidar_imu_init_b200 import host
    s = np.zeros(host.STATE_DOUBLES)
    s[0:9] = s[12:21] = np.eye(3).reshape(9)
    s[30:33] = [9.81, 0, 0]
    row = node.state_mat_out_row(s, node.rot_to_euler(np.eye(3)), 0.0)
    assert row == " 0 -0  0 0 0 0  0 -0  0 0 0 0 0 0 0  0 0 0 0.9822      0      0 0 0 0 0\n"
    R = scenes.rot_from_rpy(0.1, -0.2, 0.3)
    e = node.rot_to_euler(R)
    np.testing.assert_allclose(e, [0.1, -0.2, 0.3], atol=1e-12)
    q = node.quat_from_rpy(*e)
    x, y, z, w = q
    Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    np.testing.assert_allclose(Rq, R, atol=1e-12)


# ---- config ----
AVIA = """common:
    lid_topic:  "/livox/lidar"
#    imu_topic:  "/livox/imu/async"
    imu_topic:  "/wit/imu"

preprocess:
    lidar_type: 1               # Livox series LiDAR
    feature_extract_en: false
    scan_line: 6
    blind: 2

initialization:
    cut_frame_num: 5             # must be positive integer, 1 means do not cut frame
    orig_odom_freq: 10           # original Lidar frequency
    mean_acc_norm: 9.805             # 1 for livox built-in IMU
    online_refine_time: 20.0     # seconds
    data_accum_length: 400
    Rot_LI_cov: [ 0.00005, 0.00005, 0.00005 ]
    Trans_LI_cov: [ 0.00001, 0.00001, 0.00001 ]

mapping:
    filter_size_surf: 0.05
    filter_size_map: 0.15
    gyr_cov: 50

pcd_save:
    pcd_save_en: false
    interval: -1                 # how many LiDAR frames saved in each pcd file;
"""


def test_config_defaults_and_overrides(tmp_path):
    d = config.Config()
    assert (d.max_iteration, d.point_filter_num, d.cube_side_length, d.lid_topic, d.imu_topic) == (4, 2, 200.0, "/livox/lidar", "/livox/imu")
    assert (d.filter_size_surf, d.filter_size_map, d.det_range, d.gyr_cov, d.acc_cov, d.b_gyr_cov, d.b_acc_cov) == (0.5, 0.5, 300.0, 0.1, 0.1, 1e-4, 1e-4)
    assert (d.blind, d.lidar_type, d.scan_line, d.feature_extract_en, d.cut_frame, d.cut_frame_num, d.orig_odom_freq) == (1.0, 1, 16, False, True, 1, 10)
    assert (d.online_refine_time, d.mean_acc_norm, d.data_accum_length) == (20.0, 9.81, 300.0)
    assert (d.scan_publish_en, d.dense_publish_en, d.scan_bodyframe_pub_en, d.pcd_save_en, d.interval) == (True, True, True, False, -1)
    p = tmp_path / "avia.yaml"
    p.write_text(AVIA)
    c = config.load(str(p), ["max_iteration=5", "point_filter_num=3", "cube_side_length=2000", "mapping/acc_cov=2.5"])
    assert (c.lid_topic, c.imu_topic, c.lidar_type, c.scan_line, c.blind, c.cut_frame_num, c.mean_acc_norm) == ("/livox/lidar", "/wit/imu", 1, 6, 2.0, 5, 9.805)
    assert (c.data_accum_length, c.Rot_LI_cov, c.Trans_LI_cov, c.filter_size_surf, c.gyr_cov) == (400.0, [5e-5] * 3, [1e-5] * 3, 0.05, 50.0)
    assert (c.max_iteration, c.point_filter_num, c.cube_side_length, c.acc_cov, c.det_range) == (5, 3, 2000.0, 2.5, 300.0)
    kw = config.odometry_kwargs(c)
    assert kw["publish"] is None and kw["filter_size_map"] == 0.15 and kw["rot_LI_cov"] == [5e-5] * 3 and kw["cut_frame_num"] == 5
    assert config.preprocess(c) == dict(lidar_type=1, N_SCANS=6, blind=2.0, point_filter_num=3)
    for bad, msg in (("max_iteration", "expected name=value"), ("nope=1", "unknown parameter 'nope'"), ("max_iteration=2.5", "is not an int"),
                     ("preprocess/feature_extract_en=maybe", "is not a bool")):
        with pytest.raises(config.ConfigError, match=msg):
            config.load(str(p), [bad])
    with pytest.raises(config.ConfigError, match="No such file"):
        config.load(str(tmp_path / "missing.yaml"))


@pytest.mark.parametrize("override,msg", [("initialization/cut_frame=false", "cut_frame: false is not supported"),
                                          ("preprocess/feature_extract_en=true", "feature_extract_en: true is not supported"),
                                          ("preprocess/lidar_type=4", "L515"), ("preprocess/lidar_type=7", "not a LiDAR type"),
                                          ("initialization/Rot_LI_cov=[1, 2]", "Rot_LI_cov must list three values")])
def test_config_refusals(tmp_path, override, msg):
    p = tmp_path / "avia.yaml"
    p.write_text(AVIA)
    with pytest.raises(config.ConfigError, match=msg):
        config.load(str(p), [override])


# ---- refinement clock ----
def test_refine_clock_precedence():
    # (frame_num % orig_odom_freq) * cut_frame_num == 0, not frame_num % (orig_odom_freq * cut_frame_num) == 0
    ticks = [f for f in range(1, 61) if node.refine_tick(f, 10, 2)]
    assert ticks == [10, 20, 30, 40, 50, 60]
    assert [f for f in range(1, 61) if f % (10 * 2) == 0] == [20, 40, 60]
    assert [f for f in range(1, 31) if node.refine_tick(f, 10, 5)] == [10, 20, 30]
    # the hand-over switches spinning sensors to cut_frame_num 2 and keeps Livox at its value
    from lidar_imu_init_b200.odometry import LidarOdometry
    for lidar_type, want in ((3, 2), (1, 4)):
        o = LidarOdometry.__new__(LidarOdometry)
        o.preprocess, o.cut_frame_num, o.state = dict(lidar_type=lidar_type), 4, np.zeros(612)
        o.state[0:9] = o.state[12:21] = np.eye(3).reshape(9)

        class _B:
            def shift(self, lag):
                self.lag = lag

        class _P:
            def set_mean_acc_norm(self, v):
                pass

            def set_cov(self, w, v):
                pass
        o.imu_buffer, o.imu_proc, o.mean_acc_norm = _B(), _P(), 9.81
        o.hand_over(dict(R_LI=np.eye(3), T_LI=np.zeros(3), grav_L0=[0, 0, -9.81], gyro_bias=np.zeros(3), acc_bias=np.zeros(3), time_lag_1=0.0,
                         time_lag_2=0.0))
        assert o.cut_frame_num == want


# ---- a short Node run on the emulated device library ----
emul = pytest.importorskip("liinit_emul")


def _emul_cls():
    if not emul.available():
        pytest.skip("g++ / CUDA headers missing")
    L = emul.load()
    vp = emul.vp
    L.liinit_frame_cut_livox.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int, C.POINTER(C.c_int)]
    L.liinit_frame_cut_pcl2.argtypes = [vp, vp, C.POINTER(capi.Pcl2Layout), C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame), C.c_int,
                                        C.POINTER(C.c_int)]
    L.liinit_frame_stage.argtypes = [vp, C.c_longlong]
    L.liinit_frame_download.argtypes = [vp, C.c_longlong, vp, C.c_int, C.POINTER(C.c_int)]

    class EmulFrames(emul.EmulGpu):
        frame_cut_livox = capi.LiInitGpu.frame_cut_livox
        frame_cut_pcl2 = capi.LiInitGpu.frame_cut_pcl2
        frame_stage = capi.LiInitGpu.frame_stage
        frame_download = capi.LiInitGpu.frame_download
        frame_size = capi.LiInitGpu.frame_size
    return EmulFrames


def livox_events(seconds, per_msg, seed=0, t_off=0.013, ahead=0.13):
    """The scenario of test_gpu_frame's 60 s run as messages in delivery order: the 200 Hz calib_sim IMU stream runs up to `ahead`
    seconds before each 10 Hz Livox message's stamp. Stamps are ROS times (sec, nsec). Returns [(kind, sec, nsec, payload)] with
    payload (gyr, acc) for "imu" and the CustomMsg records for "lidar", and the simulated path."""
    import calib_sim
    import lio_case
    S = calib_sim.make_streams(seed=seed, duration=seconds, t_off=t_off)
    path = lio_case.TruePath(seed, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    ev, k_imu = [], 0
    for k in range(int(seconds * 10) - 1):
        stamp = path.t0 + 0.1 * k
        m = scenes.livox_message(scene, path.lidar, stamp, per_msg, seed=1000 + k, dup_frac=0.01, tie_frac=0.05, noise_frac=0.01, bad_line_frac=0.01)
        while k_imu < len(ti) and ti[k_imu] <= stamp + ahead:
            ev.append(("imu", *split_time(ti[k_imu]), (wi[k_imu], ai[k_imu])))
            k_imu += 1
        ev.append(("lidar", *split_time(stamp), m))
    return ev, path


def write_event_bag(path, ev, ahead=0.13, chunk_msgs=200, comps=("bz2", "none")):
    """The events as a bag on /imu and /livox/lidar with record times that keep their order: an IMU record at its stamp, a LiDAR
    record at its stamp + ahead (after the IMU samples up to that time; ties go by file position)."""
    conns = {0: ("/imu", rosmsg.IMU_TYPE), 1: ("/livox/lidar", rosmsg.LIVOX_TYPE)}
    recs = []
    for kind, sec, nsec, pl in ev:
        if kind == "imu":
            recs.append((0, sec, nsec, ser_imu(sec, nsec, *pl)))
        else:
            rs, rn = split_time(sec + 1e-9 * nsec + ahead)
            recs.append((1, rs, rn, ser_livox(sec, nsec, pl)))
    for i in range(1, len(recs)):     # record times never decrease in file order
        if recs[i][1] * 10**9 + recs[i][2] < recs[i - 1][1] * 10**9 + recs[i - 1][2]:
            recs[i] = (recs[i][0], recs[i - 1][1], recs[i - 1][2], recs[i][3])
    chunks = [(comps[j % len(comps)], recs[i:i + chunk_msgs]) for j, i in enumerate(range(0, len(recs), chunk_msgs))]
    write_bag(path, conns, chunks)
    return "/imu", "/livox/lidar"


def drive_direct(odom, ev, mean_acc_norm, on_state):
    """The events pushed straight into LidarOdometry, as test_gpu_frame's leg 1 does; on_state(odom) after every update."""
    for kind, sec, nsec, pl in ev:
        t = sec + 1e-9 * nsec
        if kind == "imu":
            odom.imu_buffer.push(t, *pl)
            odom.push_imu(pl[0], pl[1], t, mean_acc_norm)
            continue
        odom.lidar_cbk_livox(pl, t)
        while True:
            f = odom.frame_num
            if odom.process_next() is None:
                break
            if odom.frame_num != f:
                on_state(odom)
                if not odom.imu_en and odom.data_accum_finished:
                    odom.hand_over(odom.initialize(0.0))


def sim_config(tmp_path, **kw):
    """A config file (tmp_path/sim.yaml) for the simulated rig of the scenario (Livox, 6 lines, blind 0.5, cut_frame_num 5, leaf 0.15,
    LidarOdometry's covariances; the launch parameters max_iteration 4 and point_filter_num 1 as top-level keys) and its Config."""
    text = ("max_iteration: 4\npoint_filter_num: 1\ncommon:\n  lid_topic: /livox/lidar\n  imu_topic: /imu\npreprocess:\n  lidar_type: 1\n  scan_line: 6\n  blind: 0.5\n"
            "initialization:\n  cut_frame_num: 5\n  orig_odom_freq: 10\n  mean_acc_norm: 9.81\n  online_refine_time: %g\n  data_accum_length: %g\n"
            "  Rot_LI_cov: [0.00005, 0.00005, 0.00005]\n  Trans_LI_cov: [0.0005, 0.0005, 0.0005]\n"
            "mapping:\n  filter_size_surf: 0.15\n  filter_size_map: 0.15\n  gyr_cov: 0.1\n  acc_cov: 0.1\n"
            % (kw.get("online_refine_time", 20.0), kw.get("data_accum_length", 300)))
    p = tmp_path / "sim.yaml"
    p.write_text(text)
    c = config.load(str(p))
    assert (c.max_iteration, c.point_filter_num) == (4, 1)
    return c


def test_node_run_on_emulated_library(tmp_path):
    """A second and a half of Livox messages and IMU from a written bag through Node: every update's state is bit-identical to the same
    messages pushed straight into LidarOdometry; one mat_out row and one trajectory line per update; no sub-frame is dropped."""
    from lidar_imu_init_b200 import _build
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    Emul = _emul_cls()

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

    cfg = sim_config(tmp_path)
    ev, _ = livox_events(1.5, 500)
    bag = str(tmp_path / "rec.bag")
    write_event_bag(bag, ev, chunk_msgs=47)

    def make():
        o = EmulOdometry(Emul(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        o.preprocess = config.preprocess(cfg)
        return o
    direct = []
    drive_direct(make(), ev, cfg.mean_acc_norm, lambda o: direct.append(o.state.copy()))
    out = str(tmp_path / "out")
    nd = node.Node(cfg, make(), out, node.Log(quiet=True))
    got = []
    nd.on_update = lambda n: got.append(n.odom.state.copy())
    with rosbag.Bag(bag) as b:
        nd.run(b)
    nd.close(report=False)
    assert len(got) == len(direct) > 30
    for a, b_ in zip(got, direct):
        np.testing.assert_array_equal(a, b_)
    assert nd.odom.dropped_subframes == 0
    rows = open(os.path.join(out, "Log", "mat_out.txt")).read().splitlines()
    traj = np.loadtxt(os.path.join(out, "result", "trajectory.txt"))
    assert len(rows) == len(traj) == len(got)
    np.testing.assert_allclose(traj[:, 1:4], np.array([s[9:12] for s in got]), rtol=0, atol=1e-8)
    np.testing.assert_allclose(np.linalg.norm(traj[:, 4:8], axis=1), 1.0, atol=1e-8)
    assert float(rows[-1].split()[-1]) == pytest.approx(nd.total_distance, rel=1e-5)


def test_cli_errors(tmp_path, capsys):
    """The command line exits 1 with a message naming the file and what was wrong."""
    from lidar_imu_init_b200 import run
    cfgp = tmp_path / "avia.yaml"
    cfgp.write_text(AVIA)
    assert run.main(["--config", str(cfgp), "--bag", str(tmp_path / "none.bag"), "--quiet"]) == 1
    assert "none.bag" in capsys.readouterr().err
    p = str(tmp_path / "b.bag")
    write_bag(p, CONNS, [("none", _msgs(0, [10**9], "i"))])
    assert run.main(["--config", str(cfgp), "--bag", p, "--quiet"]) == 1
    err = capsys.readouterr().err
    assert "no topic '/livox/lidar'" in err and "/imu [sensor_msgs/Imu]" in err
    assert run.main(["--config", str(cfgp), "--bag", p, "--param", "initialization/cut_frame=false"]) == 1
    assert "cut_frame: false is not supported" in capsys.readouterr().err
