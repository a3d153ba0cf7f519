"""ROS 2 bags and livox_ros_driver2 recordings on the CPU: the rosbag2 sqlite3 reader against a writer built from the storage's schema
(delivery order across split files, a .db3 read on its own, every refusal), the CDR decoders on layouts pinned by hand-computed byte
offsets, the livox_ros_driver2 definition check of ROS1 bags, and a Node run on the emulated device library that must give the same
states and the same result files from a ROS1 bag and from a ROS 2 bag of the same messages."""
import bz2
import os
import shutil
import sqlite3
import struct
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_bag_node as tb  # noqa: E402  (the ROS1 bag writer, the ROS1 serializers and the scenario)
from lidar_imu_init_b200 import capi, config, node, rosbag, rosbag2, rosmsg, scenes  # noqa: E402


# ---- CDR serializers (test infrastructure) -------------------------------------------------------------------------------------------
class Cdr:
    """CDR little endian: the encapsulation header 00 01 00 00, then every primitive aligned to its size from the byte after it."""

    def __init__(self):
        self.b = bytearray(b"\0\x01\0\0")

    def align(self, n):
        self.b += b"\0" * (-(len(self.b) - 4) % n)

    def put(self, fmt, *v):
        self.align(struct.calcsize("<" + fmt[-1]))
        self.b += struct.pack("<" + fmt, *v)

    def string(self, s):
        e = s.encode() + b"\0"
        self.put("I", len(e))
        self.b += e

    def header(self, sec, nsec, frame):
        self.put("i", sec)
        self.put("I", nsec)
        self.string(frame)


def cdr_imu(sec, nsec, gyr, acc, frame="imu_link"):
    w = Cdr()
    w.header(sec, nsec, frame)
    w.put("4d", 0, 0, 0, 1)
    w.put("9d", *range(9))
    w.put("3d", *gyr)
    w.put("9d", *range(9))
    w.put("3d", *acc)
    w.put("9d", *range(9))
    return bytes(w.b)


def cdr_livox(sec, nsec, pts, pad=False, frame="livox_frame"):
    """livox_ros_driver2/msg/CustomMsg; pad: whether the message carries the last record's pad byte."""
    a = np.zeros(len(pts), capi.LIVOX_POINT_ALIGNED)
    for f in capi.LIVOX_POINT.names:
        a[f] = pts[f]
    w = Cdr()
    w.header(sec, nsec, frame)
    w.put("Q", 123)
    w.put("I", len(a))
    w.put("B", 1)
    w.b += b"\0\0\0"
    w.put("I", len(a))
    w.align(4)
    body = a.tobytes()
    w.b += body if pad or not len(a) else body[:-1]
    return bytes(w.b)


def cdr_pcl2(sec, nsec, fields, point_step, data, n, big=False, frame="velodyne"):
    w = Cdr()
    w.header(sec, nsec, frame)
    w.put("II", 1, n)
    w.put("I", len(fields))
    for nm, off, dt, cnt in fields:
        w.string(nm)
        w.put("I", off)
        w.put("B", dt)
        w.put("I", cnt)
    w.put("B", int(big))
    w.put("II", point_step, point_step * n)
    data = bytes(data)
    w.put("I", len(data))
    w.b += data
    w.put("B", 1)
    return bytes(w.b)


# ---- a rosbag2 sqlite3 writer (test infrastructure) ----
# the schema of rosbag2's sqlite3 storage, with the columns and tables newer distributions add (the reader ignores them)
SCHEMA = """
CREATE TABLE schema(schema_version INTEGER PRIMARY KEY, ros_distro TEXT NOT NULL);
CREATE TABLE metadata(id INTEGER PRIMARY KEY, metadata_version INTEGER NOT NULL, metadata TEXT NOT NULL);
CREATE TABLE topics(id INTEGER PRIMARY KEY, name TEXT NOT NULL, type TEXT NOT NULL, serialization_format TEXT NOT NULL,
                    offered_qos_profiles TEXT NOT NULL, type_description_hash TEXT NOT NULL);
CREATE TABLE messages(id INTEGER PRIMARY KEY, topic_id INTEGER NOT NULL, timestamp INTEGER NOT NULL, data BLOB NOT NULL);
CREATE INDEX timestamp_idx ON messages (timestamp ASC);
INSERT INTO schema VALUES (4, 'jazzy');
"""


def write_db3(path, topics, msgs):
    """topics {id: (name, type)} or {id: (name, type, serialization_format)}; msgs [(topic id, timestamp [ns], data)] in id order."""
    con = sqlite3.connect(path)
    con.executescript(SCHEMA)
    con.executemany("INSERT INTO topics VALUES (?, ?, ?, ?, '', '')", [(k, *v, "cdr")[:4] for k, v in topics.items()])
    con.executemany("INSERT INTO messages(topic_id, timestamp, data) VALUES (?, ?, ?)", msgs)
    con.commit()
    con.close()


def write_bag2(d, topics, files, base="rec"):
    """A rosbag2 directory d: metadata.yaml and one <base>_<i>.db3 per entry of files ([msgs] as write_db3 takes them; an entry may
    also be (i, msgs) to choose the suffix). Returns the .db3 paths."""
    os.makedirs(d, exist_ok=True)
    paths = []
    for j, f in enumerate(files):
        i, msgs = f if isinstance(f, tuple) else (j, f)
        p = os.path.join(d, f"{base}_{i}.db3")
        write_db3(p, topics, msgs)
        paths.append(p)
    with open(os.path.join(d, "metadata.yaml"), "w") as f:
        f.write("rosbag2_bagfile_information:\n  version: 5\n  storage_identifier: sqlite3\n  relative_file_paths:\n"
                + "".join(f"    - {os.path.basename(p)}\n" for p in paths) + "  compression_format: \"\"\n  compression_mode: \"\"\n")
    return paths


def event_records(ev, ahead=0.13):
    """The record times tb.write_event_bag gives the events: an IMU message at its stamp, a LiDAR message at its stamp + ahead, never
    before the previous record. [(kind, sec, nsec, payload, record time [ns])]"""
    out, last = [], -1
    for kind, sec, nsec, pl in ev:
        rs, rn = (sec, nsec) if kind == "imu" else tb.split_time(sec + 1e-9 * nsec + ahead)
        last = max(last, rs * 10**9 + rn)
        out.append((kind, sec, nsec, pl, last))
    return out


def write_event_bag2(d, ev, files=2, pad_every=2):
    """The events of tb.livox_events as a rosbag2 directory on /imu (sensor_msgs/msg/Imu) and /livox/lidar
    (livox_ros_driver2/msg/CustomMsg), with the record times of tb.write_event_bag, split into `files` files; every pad_every-th
    CustomMsg carries its last pad byte."""
    topics = {1: ("/imu", rosmsg.IMU_TYPE_ROS2), 2: ("/livox/lidar", rosmsg.LIVOX_TYPE_ROS2)}
    msgs, k = [], 0
    for kind, sec, nsec, pl, t in event_records(ev):
        if kind == "imu":
            msgs.append((1, t, cdr_imu(sec, nsec, *pl)))
        else:
            msgs.append((2, t, cdr_livox(sec, nsec, pl, pad=k % pad_every == 0)))
            k += 1
    step = -(-len(msgs) // files)
    return write_bag2(d, topics, [msgs[i:i + step] for i in range(0, len(msgs), step)])


# ---- ROS1 connections of livox_ros_driver2 ----
def livox_definition(pkg="livox_ros_driver2", point_fields=None):
    """The message_definition a ROS1 recorder writes for <pkg>/CustomMsg: the message, then its dependencies after separator lines."""
    pf = point_fields or ["uint32 offset_time      # offset time relative to the base time", "float32 x               # X axis, unit:m",
                          "float32 y               # Y axis, unit:m", "float32 z               # Z axis, unit:m",
                          "uint8 reflectivity      # reflectivity, 0~255", "uint8 tag               # livox tag",
                          "uint8 line              # laser number in lidar"]
    sep = "=" * 80
    return ("# Livox publish pointcloud msg format.\n\nstd_msgs/Header header    # ROS standard message header\n"
            "uint64 timebase           # The time of first point\nuint32 point_num          # Total number of pointclouds\n"
            "uint8  lidar_id           # Lidar device id number\nuint8[3]  rsvd            # Reserved use\n"
            "CustomPoint[] points      # Pointcloud data\n\n\n"
            f"{sep}\nMSG: std_msgs/Header\n# Standard metadata for higher-level stamped data types.\nuint32 seq\ntime stamp\nstring frame_id\n\n"
            f"{sep}\nMSG: {pkg}/CustomPoint\n# Livox costom pointcloud format.\n\n" + "\n".join(pf) + "\n")


def _conn_record(cid, topic, type_, definition):
    body = b"".join(struct.pack("<I", len(f)) + f for f in (b"topic=" + topic.encode(), b"type=" + type_.encode(), b"md5sum=" + b"0" * 32,
                                                           b"message_definition=" + definition.encode()))
    return tb._record({"op": b"\x07", "conn": struct.pack("<I", cid), "topic": topic.encode()}, body)


def write_bag_with_definition(path, conns, chunks, definition):
    """An indexed ROS1 bag v2.0 laid out as tb.write_bag lays it out (conns {id: (topic, type)}; chunks [(compression "none" / "bz2",
    [(conn, sec, nsec, data)])]), with `definition` as the message_definition of every connection."""
    u32 = lambda v: struct.pack("<I", v)                                     # noqa: E731
    stamp = lambda t: struct.pack("<II", t // 10**9, t % 10**9)              # noqa: E731
    pos0 = len(rosbag.MAGIC) + 4096                                          # the bag header record is padded to 4096 bytes
    body, infos, seen = b"", [], set()
    for comp, msgs in chunks:
        inner, offs = b"", {}
        for cid, sec, nsec, data in msgs:
            if cid not in seen:
                seen.add(cid)
                inner += _conn_record(cid, *conns[cid], definition)
            offs.setdefault(cid, []).append(struct.pack("<III", sec, nsec, len(inner)))
            inner += tb._record({"op": b"\x02", "conn": u32(cid), "time": struct.pack("<II", sec, nsec)}, data)
        chunk_pos = pos0 + len(body)
        body += tb._record({"op": b"\x05", "compression": comp.encode(), "size": u32(len(inner))},
                           bz2.compress(inner) if comp == "bz2" else inner)
        for cid, entries in offs.items():
            body += tb._record({"op": b"\x04", "ver": u32(1), "conn": u32(cid), "count": u32(len(entries))}, b"".join(entries))
        times = [sec * 10**9 + nsec for _, sec, nsec, _ in msgs]
        infos.append(tb._record({"op": b"\x06", "ver": u32(1), "chunk_pos": struct.pack("<Q", chunk_pos), "start_time": stamp(min(times)),
                                 "end_time": stamp(max(times)), "count": u32(len(offs))},
                                b"".join(struct.pack("<II", c, len(e)) for c, e in offs.items())))
    index_pos = pos0 + len(body)
    body += b"".join(_conn_record(cid, *c, definition) for cid, c in conns.items()) + b"".join(infos)
    hdr = {"op": b"\x03", "index_pos": struct.pack("<Q", index_pos), "conn_count": u32(len(conns)), "chunk_count": u32(len(chunks))}
    with open(path, "wb") as f:
        f.write(rosbag.MAGIC + tb._record(hdr, b" " * (4096 - len(tb._record(hdr)))) + body)


def write_event_bag_livox2(path, ev):
    """tb.write_event_bag's bag with the LiDAR connection typed livox_ros_driver2/CustomMsg (and its recorder's definition)."""
    conns = {0: ("/imu", rosmsg.IMU_TYPE), 1: ("/livox/lidar", rosmsg.LIVOX2_TYPE)}
    recs = [(0 if kind == "imu" else 1, t // 10**9, t % 10**9, tb.ser_imu(sec, nsec, *pl) if kind == "imu" else tb.ser_livox(sec, nsec, pl))
            for kind, sec, nsec, pl, t in event_records(ev)]
    write_bag_with_definition(path, conns, [(("bz2", "none")[j % 2], recs[i:i + 300]) for j, i in enumerate(range(0, len(recs), 300))],
                              livox_definition())


# ---- layouts pinned by hand-computed byte counts ----
def test_imu_layout_by_hand():
    gyr, acc = [0.1, -0.2, 0.3], [9.7, 0.01, -0.5]
    b = cdr_imu(1716257158, 901789000, gyr, acc, frame="imu_link")
    # header: sec, nanosec (8) + string length (4) + "imu_link\0" (9) = 21; padded to 24; 37 float64 = 296 -> 320 after the 4-byte
    # encapsulation header, 324 in all
    assert len(b) == 324
    assert b[:4] == b"\0\x01\0\0" and struct.unpack_from("<iII", b, 4) == (1716257158, 901789000, 9) and b[16:25] == b"imu_link\0"
    assert b[25:28] == b"\0\0\0"
    assert struct.unpack_from("<4d", b, 28) == (0, 0, 0, 1)
    assert struct.unpack_from("<3d", b, 4 + 24 + 13 * 8) == tuple(gyr)               # orientation + its covariance = 13 float64
    assert struct.unpack_from("<3d", b, 4 + 24 + 25 * 8) == tuple(acc)               # + angular_velocity + its covariance
    st, g, a = rosmsg.decode_imu_cdr(b)
    st1, g1, a1 = rosmsg.decode_imu(tb.ser_imu(1716257158, 901789000, gyr, acc))
    assert st == st1 == 1716257158 + 1e-9 * 901789000
    np.testing.assert_array_equal(g, g1)
    np.testing.assert_array_equal(a, a1)
    with pytest.raises(rosmsg.MsgError, match="sensor_msgs/msg/Imu: message ends at byte 323, 1 bytes short"):
        rosmsg.decode_imu_cdr(b[:-1])


def test_pcl2_layout_by_hand():
    data, lay, n = scenes.spinning_pcl2(2, 4, 10)
    step, fields = tb.DRIVER_FIELDS[2]                 # x y z intensity time ring
    b = cdr_pcl2(5, 7, fields, step, data, n, frame="velodyne")
    # after the encapsulation header: header 8 + 4 + "velodyne\0" 9 = 21 -> height, width at 24..32 -> field count 32..36;
    # a PointField is its name (4 + len + NUL, padded to 4) + offset 4 + datatype 1 + 3 pad + count 4:
    # x, y, z 3 x (8 + 12) = 60; intensity (16 + 12) = 28; time (12 + 12) = 24; ring 24 -> 36 + 136 = 172; is_bigendian 172;
    # point_step 176, row_step 180, data length 184, data at 188
    data_off = 4 + 188
    assert struct.unpack_from("<I", b, data_off - 4)[0] == len(data) == n * step
    assert b[data_off:data_off + len(data)] == bytes(data)
    assert len(b) == data_off + len(data) + 1                                   # is_dense
    assert struct.unpack_from("<II", b, 4 + 176) == (step, step * n)
    assert struct.unpack_from("<I", b, 4 + 36) == (2,) and b[4 + 40:4 + 42] == b"x\0" and b[4 + 42:4 + 44] == b"\0\0"
    st, d, got, m = rosmsg.decode_pcl2_cdr(b, 2)
    assert (st, m, got) == (5 + 7e-9, n, lay)
    assert np.shares_memory(d, np.frombuffer(b, np.uint8)) and d.tobytes() == bytes(data)


def test_livox_layout_by_hand_short_and_padded():
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), lambda t: (np.broadcast_to(np.eye(3), (len(t), 3, 3)), np.zeros((len(t), 3))),
                             10.0, 3, seed=3)
    assert len(m) == 3
    short, padded = cdr_livox(10, 5, m, pad=False, frame="livox_frame"), cdr_livox(10, 5, m, pad=True, frame="livox_frame")
    # header 8 + 4 + "livox_frame\0" 12 = 24; timebase 24..32 (8-aligned); point_num 32..36; lidar_id 36; rsvd 37..40; count 40..44;
    # the records from 44: 3 x 20 - 1 = 59 bytes (no pad after the last one) or 60
    assert len(short) == 4 + 44 + 59 == 107 and len(padded) == 108
    assert struct.unpack_from("<QIB", short, 4 + 24) == (123, 3, 1) and struct.unpack_from("<I", short, 4 + 40) == (3,)
    assert short[4 + 44:4 + 44 + 19] == m[:1].tobytes() and short[4 + 63] == 0 and short[4 + 64:4 + 83] == m[1:2].tobytes()
    ros1 = rosmsg.decode_livox(tb.ser_livox(10, 5, m))[1]
    for b, view in ((short, False), (padded, True)):
        st, pts = rosmsg.decode_livox_cdr(b)
        assert st == 10 + 5e-9 and pts.dtype == capi.LIVOX_POINT_ALIGNED and pts.dtype.itemsize == 20 and len(pts) == 3
        assert pts.astype(capi.LIVOX_POINT).tobytes() == m.tobytes() == ros1.tobytes()
        assert np.shares_memory(pts, np.frombuffer(b, np.uint8)) == view
    # a view of the message never ends past it: the short message's records are a copy of 3 x 20 bytes
    pts = rosmsg.decode_livox_cdr(short)[1]
    assert pts.nbytes == 60 and pts.flags.owndata and pts.view(np.uint8)[-1] == 0
    pts = rosmsg.decode_livox_cdr(padded)[1]
    buf = np.frombuffer(padded, np.uint8)
    assert pts.ctypes.data + pts.nbytes == buf.ctypes.data + len(padded)
    with pytest.raises(rosmsg.MsgError, match="bytes short"):
        rosmsg.decode_livox_cdr(short[:-1])
    bad = bytearray(padded)
    struct.pack_into("<I", bad, 4 + 32, 4)
    with pytest.raises(rosmsg.MsgError, match="point_num 4 but 3 points"):
        rosmsg.decode_livox_cdr(bytes(bad))
    st, pts = rosmsg.decode_livox_cdr(cdr_livox(1, 0, m[:0]))
    assert len(pts) == 0
    # a header that does not end on a multiple of 8: 8 + 4 + "a\0" 2 = 14; timebase 16..24 after 2 pad bytes; point_num 24..28;
    # lidar_id 28; rsvd 29..32; count 32..36; the records from 36: 36 + 59 = 95 after the encapsulation header, 99 in all
    short = cdr_livox(10, 5, m, pad=False, frame="a")
    assert len(short) == 4 + 95 == 99 and short[4 + 12:4 + 16] == b"a\0\0\0"
    assert struct.unpack_from("<QIB", short, 4 + 16) == (123, 3, 1) and struct.unpack_from("<I", short, 4 + 32) == (3,)
    assert short[4 + 36:4 + 55] == m[:1].tobytes()
    st, pts = rosmsg.decode_livox_cdr(short)
    assert st == 10 + 5e-9 and pts.astype(capi.LIVOX_POINT).tobytes() == m.tobytes()


@pytest.mark.parametrize("n", [1, 2, 7, 500])
def test_livox_cdr_matches_ros1(n):
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), lambda t: (np.broadcast_to(np.eye(3), (len(t), 3, 3)), np.zeros((len(t), 3))),
                             10.0, n, seed=n, tie_frac=0.1)
    m = m[:n]
    want = rosmsg.decode_livox(tb.ser_livox(3, 9, m))
    for pad in (False, True):
        st, pts = rosmsg.decode_livox_cdr(cdr_livox(3, 9, m, pad=pad))
        assert st == want[0] and len(pts) == len(m)
        assert pts.astype(capi.LIVOX_POINT).tobytes() == want[1].tobytes()


@pytest.mark.parametrize("lidar_type", [2, 3, 5, 6])
@pytest.mark.parametrize("with_time", [True, False])
def test_pcl2_cdr_matches_ros1(lidar_type, with_time):
    data, lay, n = scenes.spinning_pcl2(lidar_type, 16, 100, stamp=5.0, with_time=with_time)
    step, fields = tb.DRIVER_FIELDS[lidar_type]
    if not with_time:
        fields = [f for f in fields if f[0] != tb.TIME_NAME[lidar_type]]
    st, d, got, m = rosmsg.decode_pcl2_cdr(cdr_pcl2(5, 0, fields, step, data, n), lidar_type)
    st1, d1, got1, m1 = rosmsg.decode_pcl2(tb.ser_pcl2(5, 0, fields, step, data, n), lidar_type)
    assert (st, got, m) == (st1, got1, m1) and d.tobytes() == d1.tobytes()


def test_pcl2_cdr_rejections():
    """The shared field check, under the ROS 2 type name; Ouster's UINT16 ring of ROS 2 drivers keeps its refusal."""
    data, lay, n = scenes.spinning_pcl2(2, 4, 10)
    step, fields = tb.DRIVER_FIELDS[2]
    bad = [(f[0], f[1], 8 if f[0] == "time" else f[2], 1) for f in fields]
    with pytest.raises(rosmsg.MsgError, match="sensor_msgs/msg/PointCloud2: field 'time' is FLOAT64 x 1; lidar_type 2 expects FLOAT32"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, bad, step, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="sensor_msgs/msg/PointCloud2: is_bigendian"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, fields, step, data, n, big=True), 2)
    with pytest.raises(rosmsg.MsgError, match="point_step 36"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, fields, 36, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="field 'ring' of lidar_type 2 is missing"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, [f for f in fields if f[0] != "ring"], step, data, n), 2)
    with pytest.raises(rosmsg.MsgError, match="field 'ring' is UINT16 x 1; lidar_type 3 expects UINT8"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, fields, step, data, n), 3)
    with pytest.raises(rosmsg.MsgError, match="lidar_type 1 reads no PointCloud2"):
        rosmsg.decode_pcl2_cdr(cdr_pcl2(1, 0, fields, step, data, n), 1)
    b = cdr_pcl2(1, 0, fields, step, data, n)
    with pytest.raises(rosmsg.MsgError, match="big-endian CDR"):
        rosmsg.decode_pcl2_cdr(b"\0\0\0\0" + b[4:], 2)
    with pytest.raises(rosmsg.MsgError, match="encapsulation header 00 03 00 00 is not CDR little endian"):
        rosmsg.decode_pcl2_cdr(b"\0\x03\0\0" + b[4:], 2)


def test_decoders_table():
    for fmt, types in (("ros1", (rosmsg.LIVOX_TYPE, rosmsg.LIVOX2_TYPE)), ("cdr", (rosmsg.LIVOX_TYPE_ROS2,))):
        assert rosmsg.decoders(fmt, 1).lidar_types == types
    assert rosmsg.decoders("ros1", 3).lidar_types == (rosmsg.PCL2_TYPE,) and rosmsg.decoders("cdr", 3).imu_types == (rosmsg.IMU_TYPE_ROS2,)
    c = config.Config(lid_topic="/l", imu_topic="/i", lidar_type=2)
    assert config.wanted_topics(c, "cdr") == {"/l": (rosmsg.PCL2_TYPE_ROS2,), "/i": (rosmsg.IMU_TYPE_ROS2,)}
    with pytest.raises(ValueError, match="unknown bag format"):
        rosmsg.decoders("mcap", 1)


# ---- the rosbag2 reader ----
TOPICS = {1: ("/imu", rosmsg.IMU_TYPE_ROS2), 2: ("/lidar", rosmsg.LIVOX_TYPE_ROS2)}
WANTED = {"/imu": rosmsg.IMU_TYPE_ROS2, "/lidar": rosmsg.LIVOX_TYPE_ROS2}


def _payload(tag, i):
    return b"\0\x01\0\0" + f"{tag}{i}".encode()


def test_reader_order_across_split_files(tmp_path):
    """Timestamps tie across the two files and inside each; the files are rec_9 and rec_10, whose numeric order is not their name
    order; messages are inserted out of timestamp order."""
    rng = np.random.default_rng(2)
    ts = [int(x) for x in rng.integers(0, 20, 60) * 1_000_000 + 7 * 10**9]
    f9 = [(1 + (i % 3 == 0), ts[i], _payload("a", i)) for i in range(30)]
    f10 = [(1 + (i % 4 == 0), ts[i], _payload("b", i)) for i in range(30, 60)]
    d = str(tmp_path / "rec")
    p9, p10 = write_bag2(d, TOPICS, [(9, f9), (10, f10)])
    want = sorted([(t, 0, i, tid, data) for i, (tid, t, data) in enumerate(f9)] + [(t, 1, i, tid, data) for i, (tid, t, data) in enumerate(f10)])
    assert len({w[0] for w in want}) < len(want)
    assert any(a[0] == b[0] and a[1] != b[1] for a, b in zip(want, want[1:]))     # a tie across the files
    with rosbag2.Bag2(d) as bag:
        assert bag.topics() == {"/imu": rosmsg.IMU_TYPE_ROS2, "/lidar": rosmsg.LIVOX_TYPE_ROS2}
        assert [os.path.basename(f[0]) for f in bag.files] == ["rec_9.db3", "rec_10.db3"]
        got = [(m.topic, m.type, m.sec, m.nsec, bytes(m.data)) for m in bag.messages(WANTED)]
        assert bag.count(WANTED) == 60 and bag.count({"/imu": rosmsg.IMU_TYPE_ROS2}) == sum(1 for w in want if w[3] == 1)
        only = [bytes(m.data) for m in bag.messages({"/lidar": rosmsg.LIVOX_TYPE_ROS2})]
        assert bag.time_bounds() == (min(ts), max(ts))
    assert got == [(TOPICS[tid][0], TOPICS[tid][1], t // 10**9, t % 10**9, data) for t, _, _, tid, data in want]
    assert only == [w[4] for w in want if w[3] == 2]
    with rosbag2.Bag2(p10) as bag:                        # a .db3 on its own
        got = [bytes(m.data) for m in bag.messages(WANTED)]
    assert got == [data for _, _, _, _, data in sorted((t, 0, i, tid, data) for i, (tid, t, data) in enumerate(f10))]
    for p in (d, p10):
        with rosbag2.open_bag(p) as bag:
            assert isinstance(bag, rosbag2.Bag2) and bag.format == "cdr"


def test_open_bag_by_content(tmp_path):
    p = str(tmp_path / "a.bag")
    tb.write_bag(p, tb.CONNS, [("none", tb._msgs(0, [10**9], "i"))])
    q = str(tmp_path / "rec.bag")                        # a .db3 under another name
    write_db3(q, TOPICS, [(1, 5, _payload("x", 0))])
    with rosbag2.open_bag(p) as a, rosbag2.open_bag(q) as b:
        assert isinstance(a, rosbag.Bag) and a.format == "ros1" and isinstance(b, rosbag2.Bag2)
    r = str(tmp_path / "x.db3")
    open(r, "wb").write(b"PK\3\4 not a bag")
    with pytest.raises(rosbag.BagError, match=r"neither a ROS1 bag, a rosbag2 directory nor a rosbag2 \.db3 file"):
        rosbag2.open_bag(r)


def test_reader_refusals(tmp_path):
    d = str(tmp_path / "ok")
    write_bag2(d, {**TOPICS, 3: ("/json", "std_msgs/msg/String", "json")}, [[(1, 5, _payload("i", 0)), (3, 6, b"{}")]])
    with rosbag2.Bag2(d) as bag:
        with pytest.raises(rosbag.BagError, match=r"no topic '/points' in the bag; it has: /imu \[sensor_msgs/msg/Imu\]; /json "
                                                  r"\[std_msgs/msg/String\]; /lidar \[livox_ros_driver2/msg/CustomMsg\]"):
            bag.check_topics({"/points": rosmsg.PCL2_TYPE_ROS2})
        with pytest.raises(rosbag.BagError, match=r"topic '/lidar' carries livox_ros_driver2/msg/CustomMsg, expected "
                                                  r"sensor_msgs/msg/PointCloud2; the bag has: /imu"):
            bag.check_topics({"/lidar": rosmsg.PCL2_TYPE_ROS2})
        with pytest.raises(rosbag.BagError, match=r"rec_0\.db3: topic '/json' is serialized as 'json'; only cdr is read"):
            bag.check_topics({"/json": "std_msgs/msg/String"})
        assert [bytes(m.data) for m in bag.messages({"/imu": rosmsg.IMU_TYPE_ROS2})] == [_payload("i", 0)]
    # per-message compression, big-endian CDR
    for data, msg in ((b"\x28\xb5\x2f\xfd" + b"\0" * 20, r"message 2 on /lidar starts with a zstd frame"),
                      (b"\0\0\0\0" + b"\0" * 20, r"message 2 on /lidar is big-endian CDR \(encapsulation 00 00 00 00\)")):
        e = str(tmp_path / f"m{len(msg)}")
        write_bag2(e, TOPICS, [[(1, 5, _payload("i", 0)), (2, 6, data)]])
        with rosbag2.Bag2(e) as bag:
            it = bag.messages(WANTED)
            assert bytes(next(it).data) == _payload("i", 0)
            with pytest.raises(rosbag.BagError, match=r"rec_0\.db3: " + msg):
                next(it)
    # per-file compression, MCAP, no .db3
    z = tmp_path / "z"
    z.mkdir()
    (z / "metadata.yaml").write_text("rosbag2_bagfile_information:\n  compression_mode: FILE\n")
    (z / "rec_0.db3.zstd").write_bytes(b"\x28\xb5\x2f\xfd" + b"\0" * 30)
    with pytest.raises(rosbag.BagError, match=r"rec_0\.db3\.zstd: a rosbag2 file compressed with zstd"):
        rosbag2.Bag2(str(z))
    with pytest.raises(rosbag.BagError, match=r"rec_0\.db3\.zstd: a rosbag2 file compressed with zstd"):
        rosbag2.open_bag(str(z / "rec_0.db3.zstd"))
    mc = tmp_path / "mc"
    mc.mkdir()
    (mc / "rec_0.mcap").write_bytes(b"\x89MCAP0\r\n" + b"\0" * 30)
    with pytest.raises(rosbag.BagError, match=r"rec_0\.mcap: an MCAP file; only the sqlite3 storage"):
        rosbag2.Bag2(str(mc))
    with pytest.raises(rosbag.BagError, match=r"rec_0\.mcap: an MCAP file"):
        rosbag2.open_bag(str(mc / "rec_0.mcap"))
    empty = tmp_path / "empty"
    empty.mkdir()
    (empty / "metadata.yaml").write_text("x: 1\n")
    with pytest.raises(rosbag.BagError, match=r"empty: a directory without a \.db3 file; it holds: metadata\.yaml"):
        rosbag2.Bag2(str(empty))
    nodb = tmp_path / "nodb.db3"
    sqlite3.connect(str(nodb)).executescript("CREATE TABLE t(x INTEGER); INSERT INTO t VALUES (1);")
    with pytest.raises(rosbag.BagError, match=r"nodb\.db3: not a rosbag2 database"):
        rosbag2.Bag2(str(nodb))


def _wal_recording(d, n, checkpointed):
    """A WAL-mode recording copied into directory d while its recorder still had it open (a recorder that died): n messages, of which
    the first `checkpointed` are in the .db3 and the rest only in its .db3-wal (with none checkpointed, the tables are there too).
    Returns the messages [(topic id, timestamp, data)]."""
    src = os.path.join(d + "_live", "rec_0.db3")
    os.makedirs(os.path.dirname(src))
    os.makedirs(d)
    msgs = [(1 + i % 2, 1000 + i, _payload("w", i)) for i in range(n)]
    con = sqlite3.connect(src)
    con.execute("PRAGMA journal_mode=WAL")
    con.execute("PRAGMA wal_autocheckpoint=0")
    con.executescript(SCHEMA)
    con.executemany("INSERT INTO topics VALUES (?, ?, ?, 'cdr', '', '')", [(k, *v) for k, v in TOPICS.items()])
    con.executemany("INSERT INTO messages(topic_id, timestamp, data) VALUES (?, ?, ?)", msgs[:checkpointed])
    con.commit()
    if checkpointed:
        con.execute("PRAGMA wal_checkpoint(TRUNCATE)")
    con.executemany("INSERT INTO messages(topic_id, timestamp, data) VALUES (?, ?, ?)", msgs[checkpointed:])
    con.commit()
    for f in ("rec_0.db3", "rec_0.db3-wal"):
        shutil.copy(os.path.join(os.path.dirname(src), f), d)
    con.close()
    assert os.path.getsize(os.path.join(d, "rec_0.db3-wal")) > 0
    return msgs


@pytest.mark.parametrize("checkpointed", [100, 0])
def test_reader_wal_tail(tmp_path, checkpointed):
    """The messages still in a write-ahead log are read too, with a warning; an empty log is a finished recording."""
    d = str(tmp_path / "rec")
    msgs = _wal_recording(d, 150, checkpointed)
    with pytest.warns(rosbag.BagWarning, match=r"rec_0\.db3-wal: the recording's newest messages are still in its write-ahead log"):
        bag = rosbag2.Bag2(d)
    with bag:
        assert bag.count(WANTED) == 150 and bag.time_bounds() == (1000, 1149)
        got = [(m.topic, m.sec * 10**9 + m.nsec, bytes(m.data)) for m in bag.messages(WANTED)]
    assert got == [(TOPICS[tid][0], t, data) for tid, t, data in msgs]
    e = str(tmp_path / "done")
    write_bag2(e, TOPICS, [msgs[:10]])
    open(os.path.join(e, "rec_0.db3-wal"), "wb").close()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        with rosbag2.Bag2(e) as bag:
            assert bag.count(WANTED) == 10


@pytest.mark.skipif(os.geteuid() == 0, reason="file permissions do not bind root")
def test_reader_wal_in_read_only_directory(tmp_path):
    """Where SQLite cannot replay the log (a read-only directory without the recording's .db3-shm), the file is refused and the log
    named, rather than read without its newest messages."""
    d = str(tmp_path / "rec")
    _wal_recording(d, 50, 20)
    for f in os.listdir(d):
        os.chmod(os.path.join(d, f), 0o444)
    os.chmod(d, 0o555)
    try:
        with pytest.warns(rosbag.BagWarning):
            with pytest.raises(rosbag.BagError, match=r"rec_0\.db3: its write-ahead log .*rec_0\.db3-wal holds messages that were never "
                                                      r"checkpointed, and SQLite cannot replay it here"):
                rosbag2.Bag2(d)
    finally:
        os.chmod(d, 0o755)


def _damaged_db3(path, topics=TOPICS):
    """A .db3 whose topics (ids 1 and 2) are intact but one page in the middle of its messages is overwritten (a damaged file)."""
    write_db3(path, topics, [(1 + i % 2, i, b"\0\x01\0\0" + bytes(3000)) for i in range(300)])
    b = bytearray(open(path, "rb").read())
    page = struct.unpack_from(">H", b, 16)[0]
    mid = len(b) // page // 2
    b[mid * page:(mid + 1) * page] = b"\xff" * page
    open(path, "wb").write(b)


def test_reader_damaged_database(tmp_path):
    p = str(tmp_path / "rec_0.db3")
    _damaged_db3(p)
    msg = r"rec_0\.db3: reading the database failed \(database disk image is malformed\); the file is damaged"
    with rosbag2.Bag2(p) as bag:
        assert set(bag.topics()) == {"/imu", "/lidar"}
        with pytest.raises(rosbag.BagError, match=msg):
            bag.count(WANTED)
        n = 0
        with pytest.raises(rosbag.BagError, match=msg):
            for _ in bag.messages(WANTED):
                n += 1
        assert 0 < n < 300


# ---- ROS1 bags of livox_ros_driver2 ----
def test_livox2_ros1_definition_check(tmp_path):
    assert rosmsg.definition_mismatch(rosmsg.LIVOX2_TYPE, livox_definition()) is None
    assert rosmsg.definition_mismatch(rosmsg.LIVOX2_TYPE, livox_definition().replace("# ", "#").replace("\n\n", "\n\n\n  \n")) is None
    assert rosmsg.definition_mismatch(rosmsg.LIVOX_TYPE, "") is None                  # only livox_ros_driver2 is checked
    pf = ["uint32 offset_time", "float32 x", "float32 y", "float32 z", "uint8 reflectivity", "uint8 tag", "uint8 line"]
    assert "CustomPoint field 'x' is 'float64 x'" in rosmsg.definition_mismatch(
        rosmsg.LIVOX2_TYPE, livox_definition(point_fields=[p.replace("float32 x", "float64 x") for p in pf]))
    assert "CustomPoint field 'curvature' is not in" in rosmsg.definition_mismatch(rosmsg.LIVOX2_TYPE,
                                                                                    livox_definition(point_fields=pf + ["float32 curvature"]))
    assert "CustomPoint lacks field 'line'" in rosmsg.definition_mismatch(rosmsg.LIVOX2_TYPE, livox_definition(point_fields=pf[:-1]))
    assert "CustomMsg field 'point_num' is 'uint64 point_num'" in rosmsg.definition_mismatch(
        rosmsg.LIVOX2_TYPE, livox_definition().replace("uint32 point_num", "uint64 point_num"))
    assert "no CustomPoint" in rosmsg.definition_mismatch(rosmsg.LIVOX2_TYPE, livox_definition().split("=" * 80)[0])

    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), lambda t: (np.broadcast_to(np.eye(3), (len(t), 3, 3)), np.zeros((len(t), 3))),
                             10.0, 50, seed=1)
    conns = {0: ("/imu", rosmsg.IMU_TYPE), 1: ("/livox/lidar", rosmsg.LIVOX2_TYPE)}
    chunks = [("none", [(0, 1, 0, tb.ser_imu(1, 0, [0, 0, 0], [0, 0, 9.8])), (1, 1, 5, tb.ser_livox(1, 5, m))])]
    wanted = config.wanted_topics(config.Config(lid_topic="/livox/lidar", imu_topic="/imu"), "ros1")
    p = str(tmp_path / "ok.bag")
    write_bag_with_definition(p, conns, chunks, livox_definition())
    with rosbag.Bag(p) as bag:
        got = [m_ for m_ in bag.messages(wanted)]
        assert got[1].type == rosmsg.LIVOX2_TYPE
        assert rosmsg.decoders("ros1", 1).lidar(got[1].data)[1].tobytes() == m.tobytes()
    q = str(tmp_path / "bad.bag")
    write_bag_with_definition(q, conns, chunks, livox_definition(point_fields=[p_.replace("float32 z", "float64 z") for p_ in pf]))
    with rosbag.Bag(q) as bag:
        with pytest.raises(rosbag.BagError, match=r"topic '/livox/lidar' carries livox_ros_driver2/CustomMsg, whose message_definition "
                                                  r"differs from livox_ros_driver/CustomMsg: CustomPoint field 'z' is 'float64 z'"):
            bag.check_topics(wanted)
    # a PointCloud2 config does not take a CustomMsg of either driver
    with rosbag.Bag(p) as bag:
        with pytest.raises(rosbag.BagError, match="carries livox_ros_driver2/CustomMsg, expected sensor_msgs/PointCloud2"):
            bag.check_topics(config.wanted_topics(config.Config(lid_topic="/livox/lidar", imu_topic="/imu", lidar_type=2), "ros1"))


# ---- Node on the emulated device library: a ROS1 bag and a ROS 2 bag of the same messages ----
def _emul_odometry(cfg):
    from lidar_imu_init_b200 import _build
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    Emul = tb._emul_cls()

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return tb.emul.scan_update(self.g, state, self.max_iteration, self.imu_en)

    def make():
        o = EmulOdometry(Emul(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        o.preprocess = config.preprocess(cfg)
        return o
    return make


OUT_FILES = (("result", "Initialization_result.txt"), ("Log", "mat_out.txt"), ("result", "trajectory.txt"))


def _node_run(cfg, make, bag_path, out):
    nd = node.Node(cfg, make(), out, node.Log(quiet=True))
    states = []
    nd.on_update = lambda n: states.append(n.odom.state.copy())
    with rosbag2.open_bag(bag_path) as b:
        nd.run(b)
    nd.close(report=False)
    return nd, states


def test_node_ros1_and_ros2_bags_agree(tmp_path):
    """A second and a half of the Livox scenario: the ROS 2 bag (split into two files, short and padded CustomMsgs) and the ROS1 bags
    (livox_ros_driver and livox_ros_driver2) give identical states at every update and byte-identical result files. (LI-Init does not
    trigger this early; tests/test_gpu_bag2.py runs the whole scenario.)"""
    cfg = tb.sim_config(tmp_path)
    make = _emul_odometry(cfg)
    ev, _ = tb.livox_events(1.5, 500)
    b1, b2, b3 = str(tmp_path / "rec.bag"), str(tmp_path / "rec2"), str(tmp_path / "rec_livox2.bag")
    tb.write_event_bag(b1, ev, chunk_msgs=47)
    write_event_bag2(b2, ev, files=2)
    write_event_bag_livox2(b3, ev)
    runs = [_node_run(cfg, make, b, str(tmp_path / f"out{i}")) for i, b in enumerate((b1, b2, b3))]
    (n1, s1), (n2, s2), (n3, s3) = runs
    assert len(s1) == len(s2) == len(s3) > 30
    for j, (a, b, c) in enumerate(zip(s1, s2, s3)):
        np.testing.assert_array_equal(a, b, err_msg=f"update {j}")
        np.testing.assert_array_equal(a, c, err_msg=f"update {j}")
    assert n1.odom.dropped_subframes == n2.odom.dropped_subframes == n3.odom.dropped_subframes == 0
    for d, f in OUT_FILES:
        want = open(os.path.join(tmp_path, "out0", d, f), "rb").read()
        for i in (1, 2):
            assert open(os.path.join(tmp_path, f"out{i}", d, f), "rb").read() == want, (i, f)
    assert open(os.path.join(tmp_path, "out1", "Log", "mat_out.txt")).read().count("\n") == len(s1)


def test_cli_on_rosbag2(tmp_path, capsys, monkeypatch):
    """run.main on a rosbag2 directory and on one of its .db3 files (with the emulated library in place of the device), and its exit
    code and message for an MCAP file and a compressed recording."""
    from lidar_imu_init_b200 import run
    cfg = tb.sim_config(tmp_path)
    make = _emul_odometry(cfg)
    monkeypatch.setattr(run, "make_node", lambda args, cfg, log: node.Node(cfg, make(), args.out, log))
    ev, _ = tb.livox_events(0.6, 300)
    d = str(tmp_path / "rec2")
    paths = write_event_bag2(d, ev, files=1)
    cfgp = str(tmp_path / "sim.yaml")
    seen = []
    for i, bag in enumerate((d, paths[0])):
        out = str(tmp_path / f"cli{i}")
        assert run.main(["--config", cfgp, "--bag", bag, "--out", out, "--quiet"], on_node=seen.append) == 0
        rows = open(os.path.join(out, "Log", "mat_out.txt")).read().splitlines()
        assert len(rows) == seen[-1].updates > 5
    assert open(os.path.join(tmp_path, "cli0", "Log", "mat_out.txt")).read() == open(os.path.join(tmp_path, "cli1", "Log", "mat_out.txt")).read()
    capsys.readouterr()
    mc = str(tmp_path / "rec.mcap")
    open(mc, "wb").write(b"\x89MCAP0\r\n" + b"\0" * 64)
    assert run.main(["--config", cfgp, "--bag", mc, "--quiet"]) == 1
    assert capsys.readouterr().err == f"error: {mc}: an MCAP file; only the sqlite3 storage of rosbag2 (.db3) is read\n"
    assert run.main(["--config", cfgp, "--bag", str(tmp_path / "rec2" / "rec_0.db3"), "--param", "preprocess/lidar_type=3", "--quiet"]) == 1
    assert "topic '/livox/lidar' carries livox_ros_driver2/msg/CustomMsg, expected sensor_msgs/msg/PointCloud2" in capsys.readouterr().err
    bad = tmp_path / "damaged"
    bad.mkdir()
    _damaged_db3(str(bad / "rec_0.db3"), {1: ("/imu", rosmsg.IMU_TYPE_ROS2), 2: ("/livox/lidar", rosmsg.LIVOX_TYPE_ROS2)})
    assert run.main(["--config", cfgp, "--bag", str(bad), "--out", str(tmp_path / "cli_bad"), "--quiet"]) == 1
    err = capsys.readouterr().err
    assert err.startswith("error: ") and "rec_0.db3: reading the database failed (database disk image is malformed)" in err
