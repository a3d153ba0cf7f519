"""Decoders of the message types LI-Init reads, from their serialized form in a ROS1 bag and in a ROS 2 bag (CDR).

ROS1 (little endian; strings and variable arrays carry a u32 count first; a time is u32 sec + u32 nsec and reads as sec + 1e-9 * nsec,
as ros::Time::toSec does):
- sensor_msgs/Imu: the stamp, angular_velocity and linear_acceleration.
- livox_ros_driver/CustomMsg: the stamp and a zero-copy view of its 19-byte CustomPoint records (capi.LIVOX_POINT), which
  liinit_frame_cut_livox takes as they are. livox_ros_driver2/CustomMsg has the same fields (definition_mismatch checks that) and
  decodes the same way.
- sensor_msgs/PointCloud2: the stamp, the data buffer as it is and the liinit_pcl2_layout of the configured driver, built from the
  message's fields and checked against the driver's point type.

ROS 2 (CDR, as rosbag2 stores it): a 4-byte encapsulation header 00 01 xx xx (CDR, little endian) comes first; every primitive is then
aligned to its own size (8 for 64-bit values), counted from the byte after that header. A string is a u32 length that counts its NUL,
then the bytes; a sequence is a u32 count, then the elements; a fixed array has no count. std_msgs/msg/Header is {int32 sec,
uint32 nanosec, string frame_id}, with no seq. The stamp reads as sec + 1e-9 * nanosec, the formula of the ROS1 decoders (decision):
the same data recorded in either format then drives a bit-identical run. Each CDR decoder returns exactly what the ROS1 decoder of the
same message returns:
- sensor_msgs/msg/Imu and sensor_msgs/msg/PointCloud2: as their ROS1 twins (the PointCloud2 layout check is shared).
- livox_ros_driver2/msg/CustomMsg: CDR pads every CustomPoint to 4 bytes, so the records have a stride of 20 (capi.LIVOX_POINT_ALIGNED),
  except that the last one has no pad byte. The points are a zero-copy view when the message holds 20 * n bytes from the first
  record on, and a padded copy when it ends one byte short: liinit_frame_cut_livox reads n * stride bytes.
"""
from __future__ import annotations

import functools
import struct
from typing import NamedTuple

import numpy as np

from .capi import LIVOX_POINT, LIVOX_POINT_ALIGNED

IMU_TYPE = "sensor_msgs/Imu"
LIVOX_TYPE = "livox_ros_driver/CustomMsg"
LIVOX2_TYPE = "livox_ros_driver2/CustomMsg"      # ROS1 bags of livox_ros_driver2 (the MID-360's driver)
PCL2_TYPE = "sensor_msgs/PointCloud2"
# ROS 2 type names
IMU_TYPE_ROS2 = "sensor_msgs/msg/Imu"
LIVOX_TYPE_ROS2 = "livox_ros_driver2/msg/CustomMsg"
PCL2_TYPE_ROS2 = "sensor_msgs/msg/PointCloud2"

# sensor_msgs/PointField datatypes
INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
_DT_NAME = {INT8: "INT8", UINT8: "UINT8", INT16: "INT16", UINT16: "UINT16", INT32: "INT32", UINT32: "UINT32", FLOAT32: "FLOAT32", FLOAT64: "FLOAT64"}
_DT_SIZE = {INT8: 1, UINT8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, FLOAT64: 8}

# The point types of the drivers (include/liinit_gpu.h, LIINIT_LIDAR_*): layout key -> (field name, datatype). The time field may be
# missing (the cut then reads times 0, or takes the rotation model); every other field must be there.
PCL2_POINT_TYPES = {
    2: dict(off_x=("x", FLOAT32), off_y=("y", FLOAT32), off_z=("z", FLOAT32), off_intensity=("intensity", FLOAT32), off_time=("time", FLOAT32),
            off_ring=("ring", UINT16)),                                                                               # velodyne_ros::Point
    3: dict(off_x=("x", FLOAT32), off_y=("y", FLOAT32), off_z=("z", FLOAT32), off_intensity=("intensity", FLOAT32), off_time=("t", UINT32),
            off_ring=("ring", UINT8)),                                                                                # ouster_ros::Point
    5: dict(off_x=("x", FLOAT32), off_y=("y", FLOAT32), off_z=("z", FLOAT32), off_intensity=("intensity", FLOAT32),
            off_time=("timestamp", FLOAT64), off_ring=("ring", UINT16)),                                              # pandar_ros::Point
    6: dict(off_x=("x", FLOAT32), off_y=("y", FLOAT32), off_z=("z", FLOAT32), off_intensity=("intensity", UINT8),
            off_time=("timestamp", FLOAT64), off_ring=("ring", UINT16)),                                              # robosense_ros::Point
}


class MsgError(ValueError):
    pass


class _Reader:
    def __init__(self, buf, what):
        self.b = memoryview(buf)
        self.p = 0
        self.what = what

    def take(self, n):
        if self.p + n > len(self.b):
            raise MsgError(f"{self.what}: message ends at byte {len(self.b)}, {self.p + n - len(self.b)} bytes short")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def unpack(self, fmt):
        s = struct.calcsize(fmt)
        return struct.unpack(fmt, self.take(s))

    def u32(self):
        return self.unpack("<I")[0]

    def string(self):
        return bytes(self.take(self.u32())).decode("utf-8", "replace")

    def header(self):
        """std_msgs/Header -> stamp [s]"""
        _seq, sec, nsec = self.unpack("<III")
        self.string()
        return sec + 1e-9 * nsec


def decode_imu(buf):
    """sensor_msgs/Imu -> (stamp [s], angular_velocity [3], linear_acceleration [3]); the orientation and the covariances are skipped."""
    r = _Reader(buf, IMU_TYPE)
    stamp = r.header()
    r.take(8 * (4 + 9))
    gyr = np.array(r.unpack("<3d"))
    r.take(8 * 9)
    acc = np.array(r.unpack("<3d"))
    r.take(8 * 9)
    return stamp, gyr, acc


def decode_livox(buf):
    """livox_ros_driver/CustomMsg -> (stamp [s], points): points is a read-only structured view of capi.LIVOX_POINT over the
    message's own bytes (stride 19), no copy."""
    r = _Reader(buf, LIVOX_TYPE)
    stamp = r.header()
    _timebase, point_num, _lidar_id = r.unpack("<QIB")
    r.take(3)                                   # rsvd u8[3]
    n = r.u32()
    if n != point_num:
        raise MsgError(f"{LIVOX_TYPE}: point_num {point_num} but {n} points")
    r.take(n * LIVOX_POINT.itemsize)
    pts = np.frombuffer(r.b, LIVOX_POINT, n, r.p - n * LIVOX_POINT.itemsize)
    return stamp, pts


def _check_lidar_type(what, lidar_type):
    if lidar_type not in PCL2_POINT_TYPES:
        raise MsgError(f"{what}: lidar_type {lidar_type} reads no PointCloud2 (2 Velodyne, 3 Ouster, 5 Pandar, 6 Robosense)")


def _pcl2_layout(what, lidar_type, height, width, fields, big, point_step, row_step, data):
    """The checks and the layout shared by both formats: fields {name: (offset, datatype, count)} -> (data as uint8, layout, n)."""
    if big:
        raise MsgError(f"{what}: is_bigendian is set; only little-endian point data is read")
    n = height * width
    if point_step == 0 or len(data) != n * point_step or row_step != width * point_step:
        raise MsgError(f"{what}: point_step {point_step} / row_step {row_step} disagree with {height} x {width} points in "
                       f"{len(data)} data bytes")
    lay = dict(point_step=point_step)
    for key, (name, dt) in PCL2_POINT_TYPES[lidar_type].items():
        if name not in fields:
            if key == "off_time":
                lay[key] = -1
                continue
            raise MsgError(f"{what}: field {name!r} of lidar_type {lidar_type} is missing; the message has {sorted(fields)}")
        off, got, count = fields[name]
        if got != dt or count != 1:
            raise MsgError(f"{what}: field {name!r} is {_DT_NAME.get(got, got)} x {count}; lidar_type {lidar_type} expects "
                           f"{_DT_NAME[dt]} x 1")
        if off + _DT_SIZE[dt] > point_step:
            raise MsgError(f"{what}: field {name!r} at offset {off} overruns point_step {point_step}")
        lay[key] = off
    return np.frombuffer(data, np.uint8), lay, n


def decode_pcl2(buf, lidar_type: int):
    """sensor_msgs/PointCloud2 -> (stamp [s], data (a view of the message bytes), layout dict for capi.frame_cut_pcl2, n points).
    Rejects a field of the driver's point type with another datatype or count, big-endian data, a point_step too short for a field and
    a point_step that disagrees with the data length, naming what is wrong."""
    _check_lidar_type(PCL2_TYPE, lidar_type)
    r = _Reader(buf, PCL2_TYPE)
    stamp = r.header()
    height, width = r.unpack("<II")
    fields = {}
    for _ in range(r.u32()):
        name = r.string()
        off, dt, count = r.unpack("<IBI")
        fields[name] = (off, dt, count)
    (big,) = r.unpack("<B")
    point_step, row_step = r.unpack("<II")
    data = r.take(r.u32())
    return (stamp, *_pcl2_layout(PCL2_TYPE, lidar_type, height, width, fields, big, point_step, row_step, data))


# ---- ROS 2 (CDR) ----

def cdr_pad(pos: int, size: int) -> int:
    """The padding CDR puts before a primitive of `size` bytes at byte `pos` of a message, counted from the message's first byte (the
    alignment is counted from the byte after the 4-byte encapsulation header). Shared by the decoders and pubmsg's serializers."""
    return -(pos - 4) % size


class _CdrReader(_Reader):
    """CDR little endian after the 4-byte encapsulation header; unpack aligns to the size of the format's last item (every format
    used here has items of one size)."""

    def __init__(self, buf, what):
        super().__init__(buf, what)
        head = bytes(self.b[:4])
        if len(head) == 4 and head[:2] == b"\0\x01":
            self.p = 4
        elif head[:2] == b"\0\0":
            raise MsgError(f"{what}: big-endian CDR (encapsulation {head.hex(' ')}); only little-endian CDR is read")
        else:
            raise MsgError(f"{what}: encapsulation header {head.hex(' ') or '(empty message)'} is not CDR little endian (00 01)")

    def align(self, n):
        self.p += cdr_pad(self.p, n)

    def unpack(self, fmt):
        self.align(struct.calcsize("<" + fmt[-1]))
        return super().unpack(fmt)

    def string(self):
        s = bytes(self.take(self.u32()))
        return (s[:-1] if s.endswith(b"\0") else s).decode("utf-8", "replace")

    def header(self):
        """std_msgs/msg/Header -> stamp [s]"""
        sec, nsec = self.unpack("<iI")
        self.string()
        return sec + 1e-9 * nsec


def decode_imu_cdr(buf):
    """sensor_msgs/msg/Imu (CDR) -> (stamp [s], angular_velocity [3], linear_acceleration [3]), as decode_imu."""
    r = _CdrReader(buf, IMU_TYPE_ROS2)
    stamp = r.header()
    r.unpack("<13d")                            # orientation, its covariance
    gyr = np.array(r.unpack("<3d"))
    r.unpack("<9d")
    acc = np.array(r.unpack("<3d"))
    r.unpack("<9d")
    return stamp, gyr, acc


def decode_livox_cdr(buf):
    """livox_ros_driver2/msg/CustomMsg (CDR) -> (stamp [s], points): points are capi.LIVOX_POINT_ALIGNED records (stride 20), a
    read-only view of the message's bytes, or a padded copy when the message ends at the last record's 19th byte."""
    r = _CdrReader(buf, LIVOX_TYPE_ROS2)
    stamp = r.header()
    _timebase, = r.unpack("<Q")
    point_num = r.u32()
    _lidar_id, = r.unpack("<B")
    r.take(3)                                   # rsvd u8[3]
    n = r.u32()
    if n != point_num:
        raise MsgError(f"{LIVOX_TYPE_ROS2}: point_num {point_num} but {n} points")
    stride = LIVOX_POINT_ALIGNED.itemsize
    start = r.p
    r.take(stride * n - 1 if n else 0)          # the last record has no pad byte
    if len(r.b) - start >= stride * n:
        return stamp, np.frombuffer(r.b, LIVOX_POINT_ALIGNED, n, start)
    pts = np.zeros(n, LIVOX_POINT_ALIGNED)
    pts.view(np.uint8)[:stride * n - 1] = r.b[start:r.p]
    return stamp, pts


def decode_pcl2_cdr(buf, lidar_type: int):
    """sensor_msgs/msg/PointCloud2 (CDR) -> (stamp [s], data, layout, n points), as decode_pcl2 and with its checks."""
    _check_lidar_type(PCL2_TYPE_ROS2, lidar_type)
    r = _CdrReader(buf, PCL2_TYPE_ROS2)
    stamp = r.header()
    height, width = r.unpack("<II")
    fields = {}
    for _ in range(r.u32()):                    # PointField {string name, u32 offset, u8 datatype, u32 count}
        name = r.string()
        (off,) = r.unpack("<I")
        (dt,) = r.unpack("<B")
        (count,) = r.unpack("<I")
        fields[name] = (off, dt, count)
    (big,) = r.unpack("<B")
    point_step, row_step = r.unpack("<II")
    data = r.take(r.u32())                      # is_dense follows; it is not read
    return (stamp, *_pcl2_layout(PCL2_TYPE_ROS2, lidar_type, height, width, fields, big, point_step, row_step, data))


# ---- livox_ros_driver2 in ROS1 bags ----
# the fields of livox_ros_driver/CustomMsg and CustomPoint, as (type, name) with message types without their package
LIVOX_FIELDS = (("Header", "header"), ("uint64", "timebase"), ("uint32", "point_num"), ("uint8", "lidar_id"), ("uint8[3]", "rsvd"),
                ("CustomPoint[]", "points"))
CUSTOM_POINT_FIELDS = (("uint32", "offset_time"), ("float32", "x"), ("float32", "y"), ("float32", "z"), ("uint8", "reflectivity"),
                       ("uint8", "tag"), ("uint8", "line"))


def _definition_sections(text):
    """A ROS1 connection's message_definition -> {message name without package ('' for the top one): [(type, name)]}. Comments and
    blank lines do not count; a type's package is dropped."""
    out, name = {}, ""
    out[name] = []
    for line in text.splitlines():
        line = line.split("#", 1)[0].strip()
        if not line:
            continue
        if set(line) == {"="}:
            name = None
            continue
        if name is None and line.startswith("MSG:"):
            name = line[4:].strip().rsplit("/", 1)[-1]
            out[name] = []
            continue
        parts = line.split(None, 1)
        t, f = parts[0], (parts[1].replace(" ", "") if len(parts) > 1 else "")
        out.setdefault(name, []).append((t.rsplit("/", 1)[-1], f))
    return out


def _first_difference(what, got, want):
    for (gt, gn), (wt, wn) in zip(got, want):
        if (gt, gn) != (wt, wn):
            return f"{what} field {gn!r} is '{gt} {gn}', {LIVOX_TYPE} has '{wt} {wn}'"
    if len(got) > len(want):
        return f"{what} field {got[len(want)][1]!r} is not in {LIVOX_TYPE}"
    if len(got) < len(want):
        return f"{what} lacks field {want[len(got)][1]!r} of {LIVOX_TYPE}"
    return None


def definition_mismatch(type_: str, definition: str):
    """For a ROS1 connection of livox_ros_driver2/CustomMsg: None when its message_definition lists the fields of
    livox_ros_driver/CustomMsg and CustomPoint (same order, same types), else what differs first. None for every other type."""
    if type_ != LIVOX2_TYPE:
        return None
    sec = _definition_sections(definition)
    why = _first_difference("CustomMsg", sec[""], LIVOX_FIELDS)
    if why is None:
        if "CustomPoint" not in sec:
            return "the definition has no CustomPoint"
        why = _first_difference("CustomPoint", sec["CustomPoint"], CUSTOM_POINT_FIELDS)
    return why


# ---- which decoder reads which message ----
class Decoders(NamedTuple):
    """The accepted types of the node's LiDAR and IMU topics in one bag format, and their decoders (each takes the message bytes)."""
    lidar_types: tuple
    lidar: object
    imu_types: tuple
    imu: object


FORMATS = ("ros1", "cdr")


def decoders(fmt: str, lidar_type: int) -> Decoders:
    """fmt: the bag's format ("ros1": a ROS1 bag, "cdr": a rosbag2 recording); lidar_type: preprocess/lidar_type (1 Livox, else
    PointCloud2)."""
    if fmt == "ros1":
        if lidar_type == 1:
            return Decoders((LIVOX_TYPE, LIVOX2_TYPE), decode_livox, (IMU_TYPE,), decode_imu)
        return Decoders((PCL2_TYPE,), functools.partial(decode_pcl2, lidar_type=lidar_type), (IMU_TYPE,), decode_imu)
    if fmt == "cdr":
        if lidar_type == 1:
            return Decoders((LIVOX_TYPE_ROS2,), decode_livox_cdr, (IMU_TYPE_ROS2,), decode_imu_cdr)
        return Decoders((PCL2_TYPE_ROS2,), functools.partial(decode_pcl2_cdr, lidar_type=lidar_type), (IMU_TYPE_ROS2,), decode_imu_cdr)
    raise ValueError(f"unknown bag format {fmt!r}; known: {', '.join(FORMATS)}")
