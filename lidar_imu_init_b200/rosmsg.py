"""Decoders of the three ROS1 message types LI-Init reads, from their serialized form (little endian; strings and variable arrays carry
a u32 count first; a time is u32 sec + u32 nsec and reads as sec + 1e-9 * nsec, as ros::Time::toSec does).

- sensor_msgs/Imu: the stamp, angular_velocity and linear_acceleration.
- livox_ros_driver/CustomMsg: the stamp and a zero-copy view of its 19-byte CustomPoint records (capi.LIVOX_POINT), which
  liinit_frame_cut_livox takes as they are.
- sensor_msgs/PointCloud2: the stamp, the data buffer as it is and the liinit_pcl2_layout of the configured driver, built from the
  message's fields and checked against the driver's point type.
"""
from __future__ import annotations

import struct

import numpy as np

from .capi import LIVOX_POINT

IMU_TYPE = "sensor_msgs/Imu"
LIVOX_TYPE = "livox_ros_driver/CustomMsg"
PCL2_TYPE = "sensor_msgs/PointCloud2"

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


def decode_pcl2(buf, lidar_type: int):
    """sensor_msgs/PointCloud2 -> (stamp [s], data (a view of the message bytes), layout dict for capi.frame_cut_pcl2, n points).
    Rejects a field of the driver's point type with another datatype or count, big-endian data, a point_step too short for a field and
    a point_step that disagrees with the data length, naming what is wrong."""
    if lidar_type not in PCL2_POINT_TYPES:
        raise MsgError(f"{PCL2_TYPE}: lidar_type {lidar_type} reads no PointCloud2 (2 Velodyne, 3 Ouster, 5 Pandar, 6 Robosense)")
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
    if big:
        raise MsgError(f"{PCL2_TYPE}: is_bigendian is set; only little-endian point data is read")
    n = height * width
    if point_step == 0 or len(data) != n * point_step or row_step != width * point_step:
        raise MsgError(f"{PCL2_TYPE}: point_step {point_step} / row_step {row_step} disagree with {height} x {width} points in "
                       f"{len(data)} data bytes")
    lay = dict(point_step=point_step)
    for key, (name, dt) in PCL2_POINT_TYPES[lidar_type].items():
        if name not in fields:
            if key == "off_time":
                lay[key] = -1
                continue
            raise MsgError(f"{PCL2_TYPE}: field {name!r} of lidar_type {lidar_type} is missing; the message has {sorted(fields)}")
        off, got, count = fields[name]
        if got != dt or count != 1:
            raise MsgError(f"{PCL2_TYPE}: field {name!r} is {_DT_NAME.get(got, got)} x {count}; lidar_type {lidar_type} expects "
                           f"{_DT_NAME[dt]} x 1")
        if off + _DT_SIZE[dt] > point_step:
            raise MsgError(f"{PCL2_TYPE}: field {name!r} at offset {off} overruns point_step {point_step}")
        lay[key] = off
    return stamp, np.frombuffer(data, np.uint8), lay, n
