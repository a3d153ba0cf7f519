"""ctypes binding of tests/cpp/lio_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU checker of the LIO mode (IMU propagation restated
literally from IMU_Processing.hpp:269-382, pointBodyToWorld). Compiled on first use into a per-user temporary directory, so that the
tests also run from a read-only tree; the package never loads it."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "lio_oracle.cpp")
_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_L = None


def load():
    global _L
    if _L is not None:
        return _L
    src = open(SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"liinit-lio-oracle-{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, f"liblio_oracle_{hashlib.sha1(src).hexdigest()[:12]}.so")
    if not os.path.exists(lib):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        tmp = lib + f".{os.getpid()}.tmp"
        # the flags of oracle/Makefile: -O3, no FMA contraction
        subprocess.check_call([gxx, "-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC])
        os.replace(tmp, lib)
    L = C.CDLL(lib)
    L.lio_oracle_propagate_imu.restype = C.c_int
    L.lio_oracle_propagate_imu.argtypes = [_f64p, _f64p, _f64p, C.c_int, C.c_double, C.c_double, _f64p]
    L.lio_oracle_body_to_world.restype = None
    L.lio_oracle_body_to_world.argtypes = [_f32p, C.c_int, _f64p, _f64p, _f64p, _f64p, _f32p]
    L.lio_oracle_state_doubles.restype = C.c_int
    assert L.lio_oracle_state_doubles() == 612
    _L = L
    return L


def _c32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class OracleImu:
    """The ImuProcess members of the IMU branch as the flat 33-double block of lio_oracle_propagate_imu (constructor defaults of
    IMU_Processing.hpp:92-108, acc_s_last and last_lidar_end_time_ 0, scales / mean_acc_norm as the node sets them). Same methods as
    lidar_imu_init_b200.host.ImuProcess."""

    def __init__(self, mean_acc_norm=9.81, cov_acc_scale=0.1, cov_gyr_scale=0.1):
        self.m = np.zeros(33)
        self.m[14:20] = 0.1           # cov_acc, cov_gyr
        self.m[20:23] = 0.00001       # cov_R_LI
        self.m[23:26] = 0.0001        # cov_T_LI
        self.m[26:32] = 0.0001        # cov_bias_gyr, cov_bias_acc
        self.m[32] = mean_acc_norm
        self.acc_scale = np.full(3, cov_acc_scale, float)
        self.gyr_scale = np.full(3, cov_gyr_scale, float)
        self.need_init = True

    def set_cov(self, which, v):
        v = np.full(3, v, float) if np.isscalar(v) else np.asarray(v, float)
        if which == "acc_cov":
            self.acc_scale = v
        elif which == "gyr_cov":
            self.gyr_scale = v
        else:
            o = dict(R_LI_cov=20, T_LI_cov=23, gyr_bias_cov=26, acc_bias_cov=29)[which]
            self.m[o:o + 3] = v

    def set_mean_acc_norm(self, v):
        self.m[32] = float(v)

    def switch(self, samples):
        """Process, IMU_Processing.hpp:445-453."""
        a = np.asarray(samples, float).reshape(-1, 7)
        if len(a):
            self.m[0:7] = a[-1]
            self.m[14:17], self.m[17:20] = self.acc_scale, self.gyr_scale
            self.need_init = False

    def propagate(self, state, samples, pcl_beg_time, pcl_end_offset_ms):
        s = _c64(state).copy()
        a = _c64(samples).reshape(-1, 7)
        poses = np.zeros((len(a) + 1, 22))
        n = load().lio_oracle_propagate_imu(self.m, s, a.reshape(-1), len(a), float(pcl_beg_time), float(pcl_end_offset_ms), poses.reshape(-1))
        return s, poses[:n]


def body_to_world(xyz, rot_end, pos_end, R_LI, T_LI):
    xyz = _c32(xyz).reshape(-1, 3)
    out = np.zeros_like(xyz)
    load().lio_oracle_body_to_world(xyz, len(xyz), _c64(rot_end).reshape(9), _c64(pos_end), _c64(R_LI).reshape(9), _c64(T_LI), out)
    return out
