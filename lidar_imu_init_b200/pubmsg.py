"""The messages the node publishes (laserMapping.cpp:561-706), serialized as a ROS1 bag stores them and as a rosbag2 recording stores
them (CDR), with the ROS1 type descriptions a bag's connection records carry (md5sum, message_definition).

Types: sensor_msgs/PointCloud2 (/cloud_registered, /cloud_registered_body, /cloud_effected), nav_msgs/Odometry (/aft_mapped_to_init),
tf2_msgs/TFMessage (/tf) and nav_msgs/Path (/path). ROS 2 names put `msg/` after the package (ros2_type). The ROS1 encoding is
little endian with u32 counts before strings and variable arrays, and a std_msgs/Header of {u32 seq, time stamp, string frame_id}; the
node never sets seq, so it is 0. CDR follows rosmsg's rules (rosmsg.cdr_pad): the encapsulation header 00 01 00 00, every primitive
aligned to its size, strings with their NUL counted, and a Header of {int32 sec, uint32 nanosec, string frame_id}.

PointCloud2 is what pcl::toROSMsg leaves for a pcl::PointCloud<pcl::PointXYZINormal> built as the node builds its clouds: height 1,
width n, the 8 fields in the order of PCL's POINT_CLOUD_REGISTER_POINT_STRUCT for the type (x y z intensity normal_x normal_y normal_z
curvature) at their offsets in the 48-byte struct, FLOAT32 x 1 each, is_bigendian false, point_step 48, row_step 48 n, is_dense true
(a cloud made by PointCloud(width, height)). The data are the 48-byte records of liinit_cloud_download as they are, with no repacking.
PCL is not available here: the field order and is_dense are our reading of PCL's sources, not checked against PCL itself.

DEFINITIONS holds the fields and constants of the .msg files of ROS's common_msgs (sensor_msgs, nav_msgs), geometry_msgs, std_msgs
and tf2_msgs, without their comments. md5sum computes a type's md5 with genmsg's algorithm (compute_md5_text): constants as
"type name=value", then one line per field, "type name" for a built-in type and "<md5 of the type> name" for a message type, joined
by newlines; message_definition is genmsg's full text: the type's text, then every dependency (depth first, in field order, each once)
after a line of 80 '=' and "MSG: <type>".
"""
from __future__ import annotations

import functools
import hashlib
import math
import struct

import numpy as np

from .rosmsg import cdr_pad

POINTCLOUD2 = "sensor_msgs/PointCloud2"
ODOMETRY = "nav_msgs/Odometry"
PATH = "nav_msgs/Path"
TF_MESSAGE = "tf2_msgs/TFMessage"

# pcl::PointXYZINormal as a PointCloud2: (name, offset, datatype, count) in PCL's registration order; datatype 7 = FLOAT32
PCL_XYZINORMAL_FIELDS = (("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 32, 7, 1), ("normal_x", 16, 7, 1),
                         ("normal_y", 20, 7, 1), ("normal_z", 24, 7, 1), ("curvature", 36, 7, 1))
POINT_STEP = 48

DEFINITIONS = {
    "std_msgs/Header": "uint32 seq\ntime stamp\nstring frame_id\n",
    "geometry_msgs/Point": "float64 x\nfloat64 y\nfloat64 z\n",
    "geometry_msgs/Quaternion": "float64 x\nfloat64 y\nfloat64 z\nfloat64 w\n",
    "geometry_msgs/Vector3": "float64 x\nfloat64 y\nfloat64 z\n",
    "geometry_msgs/Pose": "Point position\nQuaternion orientation\n",
    "geometry_msgs/PoseWithCovariance": "Pose pose\nfloat64[36] covariance\n",
    "geometry_msgs/Twist": "Vector3  linear\nVector3  angular\n",
    "geometry_msgs/TwistWithCovariance": "Twist twist\nfloat64[36] covariance\n",
    "geometry_msgs/PoseStamped": "Header header\nPose pose\n",
    "geometry_msgs/Transform": "Vector3 translation\nQuaternion rotation\n",
    "geometry_msgs/TransformStamped": "Header header\nstring child_frame_id\nTransform transform\n",
    "sensor_msgs/PointField": ("uint8 INT8    = 1\nuint8 UINT8   = 2\nuint8 INT16   = 3\nuint8 UINT16  = 4\nuint8 INT32   = 5\n"
                               "uint8 UINT32  = 6\nuint8 FLOAT32 = 7\nuint8 FLOAT64 = 8\n\nstring name\nuint32 offset\nuint8  datatype\n"
                               "uint32 count\n"),
    "sensor_msgs/PointCloud2": ("Header header\n\nuint32 height\nuint32 width\n\nPointField[] fields\n\nbool    is_bigendian\n"
                                "uint32  point_step\nuint32  row_step\nuint8[] data\n\nbool is_dense\n"),
    "nav_msgs/Odometry": ("Header header\nstring child_frame_id\ngeometry_msgs/PoseWithCovariance pose\n"
                          "geometry_msgs/TwistWithCovariance twist\n"),
    "nav_msgs/Path": "Header header\ngeometry_msgs/PoseStamped[] poses\n",
    "tf2_msgs/TFMessage": "geometry_msgs/TransformStamped[] transforms\n",
}
BUILTINS = {"bool", "int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float32", "float64", "string", "time",
            "duration", "byte", "char"}


def ros2_type(t: str) -> str:
    """sensor_msgs/PointCloud2 -> sensor_msgs/msg/PointCloud2"""
    pkg, name = t.split("/")
    return f"{pkg}/msg/{name}"


def _spec(full: str, text: str):
    """The constants [(type, name, value)] and fields [(type as written, name, resolved message type or None)] of a .msg text."""
    pkg = full.split("/")[0]
    consts, fields = [], []
    for line in text.splitlines():
        line = line.split("#", 1)[0].strip()
        if not line:
            continue
        t, rest = line.split(None, 1)
        if "=" in rest and t in BUILTINS:
            name, val = rest.split("=", 1)
            consts.append((t, name.strip(), val.strip()))
            continue
        base = t.split("[", 1)[0]
        if base in BUILTINS:
            msg = None
        elif base == "Header":
            msg = "std_msgs/Header"
        else:
            msg = base if "/" in base else f"{pkg}/{base}"
        fields.append((t, rest.strip(), msg))
    return consts, fields


def _text(t: str, defs) -> str:
    if t not in defs:
        raise KeyError(f"no message definition of {t}")
    return defs[t]


def md5_text(t: str, defs=None) -> str:
    """genmsg's compute_md5_text of type t."""
    defs = DEFINITIONS if defs is None else defs
    consts, fields = _spec(t, _text(t, defs))
    lines = [f"{ct} {cn}={cv}" for ct, cn, cv in consts]
    lines += [f"{ft} {fn}" if msg is None else f"{md5sum(msg, defs)} {fn}" for ft, fn, msg in fields]
    return "\n".join(lines)


def md5sum(t: str, defs=None) -> str:
    """The md5sum of a ROS1 message type, as genmsg computes it."""
    return hashlib.md5(md5_text(t, defs).encode()).hexdigest()


def _depends(t: str, defs) -> list:
    out = []
    for _, _, msg in _spec(t, _text(t, defs))[1]:
        if msg is not None:
            out.append(msg)
            out += _depends(msg, defs)
    return list(dict.fromkeys(out))


def message_definition(t: str, defs=None) -> str:
    """genmsg's compute_full_text of type t: the message_definition of a ROS1 connection."""
    defs = DEFINITIONS if defs is None else defs
    s = _text(t, defs) + "\n"
    for d in _depends(t, defs):
        s += "=" * 80 + "\n" + f"MSG: {d}\n" + _text(d, defs) + "\n"
    return s[:-1]


@functools.lru_cache(maxsize=None)
def connection(t: str):
    """(md5sum, message_definition) of one of the published types."""
    return md5sum(t), message_definition(t)


def ros_time(t: float):
    """ros::Time().fromSec(t) (roscpp_core time.h): sec = floor(t), nsec = boost::math::round((t - sec) * 1e9) (halves away from
    zero), a carry of nsec into sec."""
    sec = math.floor(t)
    v = (t - sec) * 1e9
    nsec = math.ceil(v)
    if nsec - v > 0.5:
        nsec -= 1
    return sec + nsec // 1_000_000_000, nsec % 1_000_000_000


# ---- the two encodings ----
class _Ros1:
    def __init__(self):
        self.b = bytearray()

    def put(self, fmt, *v):
        """fmt: items of one size"""
        self.b += struct.pack("<" + fmt, *v)

    def string(self, s):
        e = s.encode()
        self.put("I", len(e))
        self.b += e

    def header(self, stamp, frame):
        self.put("III", 0, *stamp)
        self.string(frame)


class _Cdr(_Ros1):
    def __init__(self):
        self.b = bytearray(b"\0\x01\0\0")

    def put(self, fmt, *v):
        self.b += b"\0" * cdr_pad(len(self.b), struct.calcsize("<" + fmt[-1]))
        super().put(fmt, *v)

    def string(self, s):
        e = s.encode() + b"\0"
        self.put("I", len(e))
        self.b += e

    def header(self, stamp, frame):
        self.put("iI", *stamp)
        self.string(frame)


ENCODINGS = {"ros1": _Ros1, "cdr": _Cdr}


def _pose(w, pos, quat):
    w.put("7d", *pos, *quat)


def pointcloud2(stamp, frame: str, rec12, enc: str) -> bytes:
    """sensor_msgs/PointCloud2 of [n, 12] float32 pcl::PointXYZINormal records (see the module's docstring); stamp = (sec, nsec)."""
    a = np.ascontiguousarray(rec12, "<f4").reshape(-1, 12)
    w = ENCODINGS[enc]()
    w.header(stamp, frame)
    w.put("II", 1, len(a))
    w.put("I", len(PCL_XYZINORMAL_FIELDS))
    for name, off, dt, count in PCL_XYZINORMAL_FIELDS:
        w.string(name)
        w.put("I", off)
        w.put("B", dt)
        w.put("I", count)
    w.put("B", 0)                                # is_bigendian
    w.put("II", POINT_STEP, POINT_STEP * len(a))
    w.put("I", a.nbytes)
    w.b += a.tobytes()
    w.put("B", 1)                                # is_dense
    return bytes(w.b)


def odometry(stamp, frame: str, child: str, pos, quat, enc: str) -> bytes:
    """nav_msgs/Odometry as publish_odometry (:665-684) fills it: the header, child_frame_id and pose.pose; the pose covariance, the
    twist and its covariance stay 0. quat = [x, y, z, w]."""
    w = ENCODINGS[enc]()
    w.header(stamp, frame)
    w.string(child)
    _pose(w, pos, quat)
    w.put("36d", *([0.0] * 36))
    w.put("6d", *([0.0] * 6))
    w.put("36d", *([0.0] * 36))
    return bytes(w.b)


def tf_message(stamp, frame: str, child: str, pos, quat, enc: str) -> bytes:
    """tf2_msgs/TFMessage of one geometry_msgs/TransformStamped (the TransformBroadcaster of publish_odometry)."""
    w = ENCODINGS[enc]()
    w.put("I", 1)
    w.header(stamp, frame)
    w.string(child)
    _pose(w, pos, quat)
    return bytes(w.b)


def path(stamp, frame: str, poses, enc: str) -> bytes:
    """nav_msgs/Path; poses [(stamp, frame, pos, quat)] as geometry_msgs/PoseStamped."""
    w = ENCODINGS[enc]()
    w.header(stamp, frame)
    w.put("I", len(poses))
    for st, fr, pos, quat in poses:
        w.header(st, fr)
        _pose(w, pos, quat)
    return bytes(w.b)
