"""Recording what the node publishes and LI-Init's logs, on the CPU: the output serializers on layouts pinned by hand-computed byte
offsets, the ROS1 md5sums against constants every ROS1 user has seen, the two bag writers read back by the package's own readers (and a
ROS1 recording cut short), the six logs re-emitting the reference's own rows, and the command line on the emulated device library
with and without --record / --debug-logs."""
import os
import struct
import sys
import types
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_bag2_node as t2  # noqa: E402  (the rosbag2 writer of the inputs)
import test_bag_node as tb  # noqa: E402  (the ROS1 writer of the inputs, the scenario)
from lidar_imu_init_b200 import bagwrite, config, node, pubmsg, rosbag, rosbag2  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
F, C = "camera_init", "aft_mapped"


# ---- ROS1 type descriptions ----
IMU_DEFINITION = ("Header header\n\ngeometry_msgs/Quaternion orientation\nfloat64[9] orientation_covariance # Row major about x, y, z axes\n\n"
                  "geometry_msgs/Vector3 angular_velocity\nfloat64[9] angular_velocity_covariance # Row major about x, y, z axes\n\n"
                  "geometry_msgs/Vector3 linear_acceleration\nfloat64[9] linear_acceleration_covariance # Row major x, y z \n")


def test_md5_constants():
    assert pubmsg.md5sum(pubmsg.POINTCLOUD2) == "1158d486dd51d683ce2f1be655c3c181"
    assert pubmsg.md5sum("sensor_msgs/Imu", dict(pubmsg.DEFINITIONS, **{"sensor_msgs/Imu": IMU_DEFINITION})) == "6a62c6daae103f4ff57a132d6f95cec2"
    assert pubmsg.md5sum(pubmsg.ODOMETRY) == "cd5e73d190d741a2f92e81eda573aca7"
    # the constants of PointField enter the text as "type name=value"; a dependency as its md5
    assert pubmsg.md5_text("sensor_msgs/PointField").startswith("uint8 INT8=1\nuint8 UINT8=2\n")
    assert pubmsg.md5_text(pubmsg.PATH) == f"{pubmsg.md5sum('std_msgs/Header')} header\n{pubmsg.md5sum('geometry_msgs/PoseStamped')} poses"
    d = pubmsg.message_definition(pubmsg.ODOMETRY)
    blocks = [b.split("\n", 1)[0] for b in d.split("=" * 80 + "\nMSG: ")[1:]]
    assert blocks == ["std_msgs/Header", "geometry_msgs/PoseWithCovariance", "geometry_msgs/Pose", "geometry_msgs/Point", "geometry_msgs/Quaternion",
                      "geometry_msgs/TwistWithCovariance", "geometry_msgs/Twist", "geometry_msgs/Vector3"]
    assert d.startswith(pubmsg.DEFINITIONS[pubmsg.ODOMETRY] + "\n" + "=" * 80 + "\nMSG: std_msgs/Header\nuint32 seq\n") and not d.endswith("\n\n")
    assert pubmsg.message_definition(pubmsg.TF_MESSAGE).count("MSG: ") == 5          # TransformStamped Header Transform Vector3 Quaternion


def test_ros_time():
    assert pubmsg.ros_time(0.0) == (0, 0)
    assert pubmsg.ros_time(3106.49818432969) == (3106, 498184330)
    assert pubmsg.ros_time(1.9999999999) == (2, 0)                                 # the carry into sec
    assert pubmsg.ros_time(0.0000000015) == (0, 2)                                 # halves away from zero
    assert pubmsg.ros_time(1716257158.9017891) == (1716257158, 901789188)


# ---- layouts by hand ----
def _records(n, seed=0):
    r = np.random.default_rng(seed).normal(size=(n, 12)).astype(np.float32)
    r[:, 3], r[:, [7, 10, 11]] = 1.0, 0.0
    return r


def test_pointcloud2_layout_by_hand():
    rec = _records(2)
    stamp = (1716257158, 901789000)
    b = pubmsg.pointcloud2(stamp, F, rec, "ros1")
    # header seq, sec, nsec 12 + frame 4 + 11 = 27; height, width 8 -> 35; field count 4 -> 39; a field is name (4 + len) + offset 4 +
    # datatype 1 + count 4: x, y, z 3 x 14 = 42, intensity 22, normal_x/y/z 3 x 21 = 63, curvature 22 -> 149 -> 188; is_bigendian
    # 1 -> 189; point_step, row_step 8 -> 197; data length 4 -> 201; data 96 -> 297; is_dense 1 -> 298
    assert len(b) == 298
    assert struct.unpack_from("<IIII", b, 0) == (0, *stamp, 11) and b[16:27] == b"camera_init"
    assert struct.unpack_from("<III", b, 27) == (1, 2, 8)
    assert struct.unpack_from("<I", b, 39) == (1,) and b[43:44] == b"x" and struct.unpack_from("<IBI", b, 44) == (0, 7, 1)
    assert struct.unpack_from("<I", b, 81) == (9,) and b[85:94] == b"intensity" and struct.unpack_from("<IBI", b, 94) == (32, 7, 1)
    assert b[107:115] == b"normal_x" and struct.unpack_from("<IBI", b, 115) == (16, 7, 1)
    assert b[170:179] == b"curvature" and struct.unpack_from("<IBI", b, 179) == (36, 7, 1)
    assert b[188] == 0 and struct.unpack_from("<III", b, 189) == (48, 96, 96) and b[201:297] == rec.tobytes() and b[297] == 1
    c = pubmsg.pointcloud2(stamp, F, rec, "cdr")
    # after the 4-byte encapsulation header: sec, nanosec 8, frame 4 + 12 (with its NUL) -> 24; height, width -> 32; count -> 36;
    # a one-letter field: 4 + 2, padded to 8, offset 4, datatype 1 + 3 pad, count 4 = 20: x, y, z 36..96; intensity 4 + 10 -> 14
    # padded to 16, + 12 = 28: 96..124; normal_x/y/z 4 + 9 -> 16 + 12 = 28 each: 124..208; curvature 208..236; is_bigendian 236;
    # point_step 240, row_step 244, data length 248, data 252..348, is_dense 348 -> 349, 353 in all
    assert len(c) == 353 and c[:4] == b"\0\x01\0\0"
    assert struct.unpack_from("<iII", c, 4) == (*stamp, 12) and c[16:28] == b"camera_init\0"
    assert struct.unpack_from("<III", c, 4 + 24) == (1, 2, 8)
    assert c[4 + 40:4 + 44] == b"x\0\0\0" and struct.unpack_from("<IB", c, 4 + 44) == (0, 7) and struct.unpack_from("<I", c, 4 + 52) == (1,)
    assert struct.unpack_from("<I", c, 4 + 96) == (10,) and c[4 + 100:4 + 110] == b"intensity\0" and struct.unpack_from("<I", c, 4 + 112) == (32,)
    assert c[4 + 128:4 + 137] == b"normal_x\0" and struct.unpack_from("<I", c, 4 + 140) == (16,)
    assert c[4 + 212:4 + 222] == b"curvature\0" and struct.unpack_from("<IB", c, 4 + 224) == (36, 7) and struct.unpack_from("<I", c, 4 + 232) == (1,)
    assert c[4 + 236] == 0 and struct.unpack_from("<III", c, 4 + 240) == (48, 96, 96) and c[4 + 252:4 + 348] == rec.tobytes() and c[4 + 348] == 1
    # the data are the device's records as they are: every field reads back at its offset
    for name, off, dt, count in pubmsg.PCL_XYZINORMAL_FIELDS:
        np.testing.assert_array_equal(np.frombuffer(c, "<f4", 2 * 12, 4 + 252).reshape(2, 12)[:, off // 4], rec[:, off // 4])
    assert sorted(f[1] for f in pubmsg.PCL_XYZINORMAL_FIELDS) == [0, 4, 8, 16, 20, 24, 32, 36]


def test_odometry_and_tf_layouts_by_hand():
    stamp, pos, q = (7, 5), (1.5, -2.0, 3.25), (0.1, 0.2, 0.3, 0.9)
    b = pubmsg.odometry(stamp, F, C, pos, q, "ros1")
    # header 12 + 4 + 11 = 27; child 4 + 10 -> 41; pose 7 x 8 -> 97; covariance 288 -> 385; twist 48 -> 433; covariance 288 -> 721
    assert len(b) == 721
    assert struct.unpack_from("<I", b, 27) == (10,) and b[31:41] == b"aft_mapped" and struct.unpack_from("<7d", b, 41) == pos + q
    assert not any(b[97:])
    c = pubmsg.odometry(stamp, F, C, pos, q, "cdr")
    # header 8 + 4 + 12 = 24; child 4 + 11 -> 39, aligned to 40 for the float64s; pose -> 96; covariance -> 384; twist -> 432;
    # covariance -> 720; 724 with the encapsulation header
    assert len(c) == 724 and struct.unpack_from("<I", c, 4 + 24) == (11,) and c[4 + 28:4 + 39] == b"aft_mapped\0" and c[4 + 39] == 0
    assert struct.unpack_from("<7d", c, 4 + 40) == pos + q and not any(c[4 + 96:])
    t = pubmsg.tf_message(stamp, F, C, pos, q, "ros1")
    # count 4; header 27 -> 31; child 14 -> 45; translation + rotation 56 -> 101
    assert len(t) == 101 and struct.unpack_from("<IIII", t, 0) == (1, 0, 7, 5) and struct.unpack_from("<7d", t, 45) == pos + q
    u = pubmsg.tf_message(stamp, F, C, pos, q, "cdr")
    # count 4; sec 4..8, nanosec ..12, frame 12..28; child 28..43, aligned to 48; 56 -> 104; 108 in all
    assert len(u) == 108 and struct.unpack_from("<IiI", u, 4) == (1, 7, 5) and u[4 + 32:4 + 43] == b"aft_mapped\0"
    assert struct.unpack_from("<7d", u, 4 + 48) == pos + q
    p = pubmsg.path((0, 0), F, [((7, 5), F, pos, q), ((8, 6), F, pos, q)], "cdr")
    # header 24; count 24..28; PoseStamped 1 at 28: header to 52, pose at 56..112; PoseStamped 2 at 112: header to 136, pose 136..192
    assert len(p) == 4 + 192 and struct.unpack_from("<I", p, 4 + 24) == (2,) and struct.unpack_from("<7d", p, 4 + 56) == pos + q
    assert struct.unpack_from("<iI", p, 4 + 112) == (8, 6) and struct.unpack_from("<7d", p, 4 + 136) == pos + q
    assert len(pubmsg.path((0, 0), F, [((7, 5), F, pos, q)] * 3, "ros1")) == 27 + 4 + 3 * (27 + 56)


# ---- writers read back ----
def _messages(n, enc="ros1"):
    """n updates' worth of messages of three topics with growing stamps: [(topic, type, (sec, nsec), data)]"""
    out = []
    for k in range(n):
        st = pubmsg.ros_time(100.0 + 0.02 * k)
        out.append(("/aft_mapped_to_init", pubmsg.ODOMETRY, st, pubmsg.odometry(st, F, C, (k, 0, 0), (0, 0, 0, 1), enc)))
        out.append(("/cloud_effected", pubmsg.POINTCLOUD2, st, pubmsg.pointcloud2(st, F, _records(k % 7 + 1, k), enc)))
        out.append(("/tf", pubmsg.TF_MESSAGE, st, pubmsg.tf_message(st, F, C, (k, 0, 0), (0, 0, 0, 1), enc)))
    return out


@pytest.mark.parametrize("compression", ["none", "bz2"])
def test_ros1_writer_round_trip(tmp_path, compression):
    msgs = _messages(300)
    p = str(tmp_path / "out.bag")
    w = bagwrite.Ros1Writer(p, compression)
    w.CHUNK_BYTES = 20_000
    for m in msgs:
        w.write(*m)
    w.close()
    with warnings.catch_warnings():
        warnings.simplefilter("error")          # an indexed bag: no sequential fallback
        with rosbag.Bag(p) as bag:
            assert bag.topics() == {"/aft_mapped_to_init": pubmsg.ODOMETRY, "/cloud_effected": pubmsg.POINTCLOUD2, "/tf": pubmsg.TF_MESSAGE}
            for c in bag.connections.values():
                assert (c["md5sum"], c["message_definition"]) == pubmsg.connection(c["type"])
            assert len(bag.chunks) > 5 and {c.compression for c in bag.chunks} == {compression}
            wanted = {t: ty for t, ty in bag.topics().items()}
            got = [(m.topic, m.type, (m.sec, m.nsec), bytes(m.data)) for m in bag.messages(wanted)]
    assert got == msgs                          # emission order: the stamps tie within an update, file position decides
    data = open(p, "rb").read()
    hdr = rosbag.parse_header(data, len(rosbag.MAGIC) + 4, len(rosbag.MAGIC) + 4 + struct.unpack_from("<I", data, len(rosbag.MAGIC))[0])
    assert struct.unpack("<Q", hdr["index_pos"])[0] > 0 and struct.unpack("<I", hdr["chunk_count"])[0] == len(bag.chunks)
    assert struct.unpack("<I", hdr["conn_count"])[0] == 3
    with pytest.raises(rosbag.BagError, match="exists"):
        bagwrite.Ros1Writer(p)


def test_ros1_writer_cut_short(tmp_path):
    """A run that ends without closing its recording: the chunks written so far are read back, with the reader's warning."""
    msgs = _messages(200)
    p = str(tmp_path / "cut.bag")
    w = bagwrite.Ros1Writer(p)
    w.CHUNK_BYTES = 30_000
    for m in msgs:
        w.write(*m)
    n_chunks = len(w.infos)
    assert n_chunks > 3 and len(w.chunk) > 0    # the open chunk is never written
    with pytest.warns(rosbag.BagWarning, match="has no index"):
        with rosbag.Bag(p) as bag:
            got = [(m.topic, m.type, (m.sec, m.nsec), bytes(m.data)) for m in bag.messages(bag.topics())]
            assert len(bag.chunks) == n_chunks
    kept = len(got)
    assert 0 < kept < len(msgs) and got == msgs[:kept]
    w.f.close()


def test_ros2_writer_round_trip(tmp_path):
    msgs = _messages(150, "cdr")
    d = str(tmp_path / "rec")
    w = bagwrite.Ros2Writer(d)
    for topic, type_, st, data in msgs:
        w.write(topic, type_, st, data)
    w.close()
    assert sorted(os.listdir(d)) == ["metadata.yaml", "rec_0.db3"]
    meta = open(os.path.join(d, "metadata.yaml")).read()
    assert "  message_count: 450\n" in meta and "        name: /cloud_effected\n        type: sensor_msgs/msg/PointCloud2\n" in meta
    assert "    - rec_0.db3\n" in meta and f"nanoseconds_since_epoch: {100 * 10**9}\n" in meta
    with rosbag2.open_bag(d) as bag:
        assert bag.topics() == {"/aft_mapped_to_init": "nav_msgs/msg/Odometry", "/cloud_effected": "sensor_msgs/msg/PointCloud2",
                                "/tf": "tf2_msgs/msg/TFMessage"}
        got = [(m.topic, (m.sec, m.nsec), bytes(m.data)) for m in bag.messages(bag.topics())]
    assert got == [(t, st, data) for t, _, st, data in msgs]
    with pytest.raises(rosbag.BagError, match="exists"):
        bagwrite.open_writer(d, "ros2")
    with pytest.raises(rosbag.BagError, match="applies to ROS1 bags"):
        bagwrite.open_writer(str(tmp_path / "x"), "ros2", "bz2")


# ---- LI-Init's logs ----
@pytest.mark.parametrize("name", list(node.DEBUG_LOGS))
def test_log_rows_re_emit_reference(name):
    """Rows of the reference's own Log/ files re-emit byte for byte from their printed values."""
    table, precision, groups = node.DEBUG_LOGS[name]
    rows = open(os.path.join(GOLDEN, f"reference_{name[:-4]}_rows.txt")).read().splitlines(True)
    assert len(rows) >= 12
    for r in rows:
        v = [float(x) for x in r.split()]
        assert len(v) == sum(groups)
        assert node.log_row(v, precision, groups) == r
    assert any("  " in r for r in rows)         # an object's coefficients padded to its widest one


def _replayed_calib():
    from lidar_imu_init_b200 import _build, calib
    _build.build_calib()
    g = np.load(os.path.join(GOLDEN, "li_init_log.npz"))
    c = calib.LiCalib()
    eye = np.eye(3)
    imu, lid = g["imu_before"], g["lidar_before"]
    for r in imu:
        c.push_imu(r[0:3], r[4:7], r[7])
    for r in lid:
        c.push_lidar(eye, r[0:3], np.zeros(3), r[4])
    c.push_imu(imu[-1, 0:3], imu[-1, 4:7], imu[-1, 7] + 0.02)      # the element fout_before_filter does not log (test_calib._replay)
    c.push_lidar(eye, lid[-1, 0:3], np.zeros(3), lid[-1, 4] + 0.02)
    c.initialize(10, 5, 0.0, 0.0, from_groups=True)
    return g, c


def test_replay_writes_the_six_logs(tmp_path):
    """li_init_log.npz replayed through li_calib and written by Node: the reference's row count in every file; the before-filter
    files re-emit the reference's printed digits (they are the replay's input), except |ang_vel|, which is computed again from the
    printed, rounded components."""
    g, c = _replayed_calib()
    odom = types.SimpleNamespace(calib=c, close=lambda: None)
    nd = node.Node(config.Config(Rot_LI_cov=[1e-5] * 3, Trans_LI_cov=[1e-5] * 3), odom, str(tmp_path), node.Log(quiet=True))
    nd.open_debug_logs()
    assert sorted(os.listdir(tmp_path / "Log")) == sorted(["mat_out.txt", *node.DEBUG_LOGS])
    assert all(os.path.getsize(tmp_path / "Log" / n) == 0 for n in node.DEBUG_LOGS)
    nd._write_debug_logs()
    nd.close(report=False)
    counts = {"LiDAR_meas.txt": 1331, "IMU_meas.txt": 1331, "IMU_before_filter.txt": 1369, "Lidar_before_filter.txt": 1369, "acc_cost.txt": 1333,
              "Lidar_omg_after_rot.txt": 1333}
    text = {n: open(tmp_path / "Log" / n).read() for n in node.DEBUG_LOGS}
    assert {n: t.count("\n") for n, t in text.items()} == counts
    for n in ("IMU_before_filter.txt", "Lidar_before_filter.txt"):
        mine = text[n].splitlines(True)
        ref = open(os.path.join(GOLDEN, f"reference_{n[:-4]}_rows.txt")).read().splitlines(True)
        for a, b in zip(mine[:6] + mine[-2:], ref[:6] + ref[-2:]):
            ta, tb_ = a.split(), b.split()
            assert ta[:3] + ta[4:] == tb_[:3] + tb_[4:]
            assert float(ta[3]) == pytest.approx(float(tb_[3]), rel=1e-14)
    # the other four agree with the reference to the precision test_calib pins (the first 1000 rows to the printed digits)
    im = np.loadtxt(tmp_path / "Log" / "IMU_meas.txt")
    assert np.abs(im[:1000, 0:4] - g["imu_meas"][:1000, 0:4]).max() < 2e-11
    ar = np.loadtxt(tmp_path / "Log" / "Lidar_omg_after_rot.txt")
    assert np.abs(ar[:1000] - g["after_rot"][:1000]).max() < 1e-8


# ---- the publish stage and the helper ----
class _FakeGpu:
    def __init__(self):
        self.calls = []

    def cloud(self, which, *pose):
        self.calls.append(which)
        return np.zeros((1, 12), np.float32)


def test_record_publish_downloads_only_recorded_clouds():
    from lidar_imu_init_b200.odometry import LidarOdometry
    pose = (np.eye(3), np.zeros(3), np.eye(3), np.zeros(3))
    cfg = config.Config()
    assert config.odometry_kwargs(cfg)["publish"] is None                       # the default stays: no clouds without a recording
    for kw, topics, calls in (({}, config.RECORD_TOPICS, [1, 3, 4]), (dict(dense_publish_en=False), config.RECORD_TOPICS, [2, 3, 4]),
                              (dict(scan_bodyframe_pub_en=False), config.RECORD_TOPICS, [1, 4]), (dict(scan_publish_en=False), config.RECORD_TOPICS, [4]),
                              ({}, ("/cloud_registered_body", "/path"), [3]), ({}, ("/aft_mapped_to_init",), []),
                              (dict(pcd_save_en=True), ("/cloud_effected",), [1, 4])):
        c = config.Config(**kw)
        pub = config.odometry_kwargs(c, pcd_dir="/nonexistent", record_topics=topics)["publish"]
        assert pub == config.record_publish(c, topics, "/nonexistent")
        o = LidarOdometry(_FakeGpu(), 0.5, publish=dict(pub, interval=10 ** 6))
        o._publish(*pose)
        assert o.g.calls == calls, (kw, topics)


# ---- the command line on the emulated device library ----
@pytest.fixture(scope="module")
def emul_run(tmp_path_factory):
    """run.main with the emulated device library in place of the H100 one (the product's make_node, LidarOdometry and Node)."""
    import test_outputs as to
    from lidar_imu_init_b200 import _build, capi, odometry, run
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    Emul = to._bind()
    tmp = tmp_path_factory.mktemp("rec")
    tb.sim_config(tmp)
    ev, _ = tb.livox_events(1.0, 300)
    bags = {"ros1": str(tmp / "in.bag"), "ros2": str(tmp / "in_ros2")}
    tb.write_event_bag(bags["ros1"], ev, chunk_msgs=47)
    t2.write_event_bag2(bags["ros2"], ev, files=1)
    mp = pytest.MonkeyPatch()
    mp.setattr(capi, "LiInitGpu", lambda fsm, max_map_points, max_scan_points, device_id: Emul(fsm, max_map_points=max_map_points,
                                                                                                 max_scan_points=max_scan_points))
    mp.setattr(odometry.LidarOdometry, "_scan_update_resident",
               lambda self, state: to.emul.scan_update(self.g, state, self.max_iteration, self.imu_en))

    def go(inp, out, *extra):
        seen = dict(pub=[])

        def on_node(nd):
            seen["node"] = nd
            nd.on_update = lambda n: seen["pub"].append({k: v.copy() for k, v in n.odom.published.items()})
        argv = ["--config", str(tmp / "sim.yaml"), "--bag", bags[inp], "--out", str(tmp / out), "--quiet", "--max-map-points", "400000",
                "--max-scan-points", "1000", *extra]
        rc = run.main(argv, on_node=on_node)
        return rc, seen
    yield tmp, go
    mp.undo()


def _files(d):
    return sorted(os.path.relpath(os.path.join(r, f), d) for r, _, fs in os.walk(d) for f in fs)


RESULT_FILES = ["Log/mat_out.txt", "result/Initialization_result.txt", "result/trajectory.txt"]


def test_cli_with_and_without_recording(emul_run):
    tmp, go = emul_run
    runs = {}
    for inp in ("ros1", "ros2"):
        runs[inp, False] = go(inp, f"plain_{inp}")
        runs[inp, True] = go(inp, f"rec_{inp}", "--record", str(tmp / f"bag_{inp}" / ("rec.bag" if inp == "ros1" else "rec")),
                             "--debug-logs")
    for k, (rc, _) in runs.items():
        assert rc == 0, k
    # the result files are byte-identical across the four runs; without the flags the output holds exactly them
    want = {f: open(tmp / "plain_ros1" / f, "rb").read() for f in RESULT_FILES}
    for d in ("plain_ros2", "rec_ros1", "rec_ros2"):
        for f in RESULT_FILES:
            assert open(tmp / d / f, "rb").read() == want[f], (d, f)
    assert _files(tmp / "plain_ros1") == _files(tmp / "plain_ros2") == RESULT_FILES
    # --debug-logs: the six logs, empty because LI-Init did not trigger in one second
    assert _files(tmp / "rec_ros1") == sorted(RESULT_FILES + ["Log/" + n for n in node.DEBUG_LOGS])
    assert all(os.path.getsize(tmp / "rec_ros1" / "Log" / n) == 0 for n in node.DEBUG_LOGS)
    traj = open(tmp / "plain_ros1" / "result" / "trajectory.txt").read().splitlines()
    for inp, path in (("ros1", tmp / "bag_ros1" / "rec.bag"), ("ros2", tmp / "bag_ros2" / "rec")):
        seen = runs[inp, True][1]
        nd, pub = seen["node"], seen["pub"]
        n = nd.updates
        assert n == len(traj) == len(pub) > 10 and nd.init_result is None
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            with rosbag2.open_bag(str(path)) as bag:
                fmt = bag.format
                got = {}
                for m in bag.messages(bag.topics()):
                    got.setdefault(m.topic, []).append(m)
        assert fmt == ("ros1" if inp == "ros1" else "cdr")
        assert {t: len(v) for t, v in got.items()} == {"/aft_mapped_to_init": n, "/tf": n, "/cloud_registered": n, "/cloud_registered_body": n,
                                                       "/cloud_effected": n, "/path": n // 5}
        enc = "ros1" if inp == "ros1" else "cdr"
        hdr = 27 if enc == "ros1" else 4 + 24          # the header with frame camera_init
        for k in range(n):
            line = traj[k].split()
            od = got["/aft_mapped_to_init"][k]
            assert abs(od.sec + 1e-9 * od.nsec - float(line[0])) <= 1e-9
            off = hdr + 14 if enc == "ros1" else hdr + 12 + 4      # child_frame_id aft_mapped (CDR: 15 bytes, aligned to 8)
            pose = struct.unpack_from("<7d", bytes(od.data), off)
            assert " ".join("%.9g" % v for v in pose) == " ".join(line[1:8])
            assert bytes(got["/tf"][k].data) == pubmsg.tf_message((od.sec, od.nsec), F, C, pose[:3], pose[3:], enc)
            for key, topic in config.CLOUD_TOPICS.items():
                m = got[topic][k]
                assert (m.sec, m.nsec) == (od.sec, od.nsec)
                assert bytes(m.data) == pubmsg.pointcloud2((m.sec, m.nsec), F, pub[k][key], enc)
        assert sum(len(p["effect"]) for p in pub) > 0 and sum(len(p["registered"]) for p in pub) > 0
        # /path: every 5th update, the poses so far, the start-up stamp 0
        last = bytes(got["/path"][-1].data)
        if enc == "ros1":
            assert struct.unpack_from("<III", last, 0) == (0, 0, 0) and struct.unpack_from("<I", last, 27) == (n // 5,)
        else:
            assert struct.unpack_from("<iI", last, 4) == (0, 0) and struct.unpack_from("<I", last, 4 + 24) == (n // 5,)
        assert [(m.sec, m.nsec) for m in got["/path"]] == [(m.sec, m.nsec) for m in got["/aft_mapped_to_init"][4::5]]


def test_cli_record_topics_and_refusals(emul_run, capsys):
    tmp, go = emul_run
    rc, seen = go("ros1", "some", "--record", str(tmp / "some.bag"), "--record-topics", "/cloud_effected,/path", "--record-format", "ros2",
                  "--record-compression", "none")
    assert rc == 0
    assert all(set(p) == {"effect"} for p in seen["pub"])           # the clouds that are not recorded are not downloaded
    with rosbag2.open_bag(str(tmp / "some.bag")) as bag:
        assert bag.format == "cdr" and bag.topics() == {"/cloud_effected": "sensor_msgs/msg/PointCloud2", "/path": "nav_msgs/msg/Path"}
    rc, _ = go("ros2", "bz", "--record", str(tmp / "bz.bag"), "--record-format", "ros1", "--record-compression", "bz2",
               "--record-topics", "/tf")
    assert rc == 0
    with rosbag.Bag(str(tmp / "bz.bag")) as bag:
        assert {c.compression for c in bag.chunks} == {"bz2"} and bag.count({"/tf": pubmsg.TF_MESSAGE}) == seen["node"].updates
    capsys.readouterr()
    for extra, msg in ((["--record-topics", "/tf,/Laser_map"], "--record-topics '/tf,/Laser_map': unknown topic '/Laser_map'; the node "
                                                                "publishes /cloud_registered"),
                       (["--record-format", "ros2", "--record-compression", "bz2"], "applies to ROS1 bags"),
                       ([], "exists; the recording is not written over")):
        target = str(tmp / "bz.bag") if not extra else str(tmp / "never")
        rc, _ = go("ros1", "refused", "--record", target, *extra)
        assert rc == 1
        assert msg in capsys.readouterr().err
    assert not os.path.exists(tmp / "never") and not os.path.exists(tmp / "refused")
