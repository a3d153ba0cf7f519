"""ctypes binding of include/liinit_calib.h -- the LI-Init batch initialisation (host only, SURVEY.md 8f row N4).

Mirrors the reference's LI_Init object (include/LI_init/LI_init.h:208-357): push IMU / LiDAR odometry samples, ask
whether the excitation suffices, run LI_Initialization, read the calibrated extrinsic / time offset / biases / gravity.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build

_LIB = None

SYMBOLS = ["li_calib_create", "li_calib_destroy", "li_calib_set_data_accum_length", "li_calib_set_solver", "li_calib_push_imu_all", "li_calib_push_lidar",
           "li_calib_push_imu", "li_calib_sizes", "li_calib_clear_imu_all", "li_calib_data_sufficiency", "li_calib_initialize",
           "li_calib_log_rows"]
LOG_COLUMNS = {"IMU_meas": (0, 11), "LiDAR_meas": (1, 11), "Lidar_omg_after_rot": (2, 4), "acc_cost": (3, 8), "IMU_before_filter": (4, 8),
               "Lidar_before_filter": (5, 5)}


class CalibResult(C.Structure):
    _fields_ = [("R_LI", C.c_double * 9), ("T_LI", C.c_double * 3), ("gyro_bias", C.c_double * 3), ("acc_bias", C.c_double * 3),
                ("grav_L0", C.c_double * 3), ("time_lag_1", C.c_double), ("time_lag_2", C.c_double), ("time_L_I", C.c_double),
                ("euler_deg", C.c_double * 3), ("lag_frames", C.c_int), ("n_samples", C.c_int), ("iters_rot", C.c_int),
                ("iters_rot_bias", C.c_int), ("iters_trans", C.c_int), ("cost_rot", C.c_double), ("cost_rot_bias", C.c_double),
                ("cost_trans", C.c_double)]


class CalibError(RuntimeError):
    pass


def load():
    global _LIB
    if _LIB is None:
        path = _build.CALIB_LIB
        if not os.path.exists(path):
            _build.build_calib()
        L = C.CDLL(path)
        dp = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
        vp = C.c_void_p
        L.li_calib_create.argtypes = [C.POINTER(vp)]
        L.li_calib_destroy.argtypes = [vp]
        L.li_calib_destroy.restype = None
        L.li_calib_set_data_accum_length.argtypes = [vp, C.c_double]
        L.li_calib_set_data_accum_length.restype = None
        L.li_calib_set_solver.argtypes = [vp, C.c_int]
        L.li_calib_set_solver.restype = None
        L.li_calib_push_imu_all.argtypes = [vp, dp, dp, C.c_double, C.c_double]
        L.li_calib_push_lidar.argtypes = [vp, dp, dp, dp, C.c_double]
        L.li_calib_push_imu.argtypes = [vp, dp, dp, C.c_double]
        L.li_calib_sizes.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.li_calib_clear_imu_all.argtypes = [vp]
        L.li_calib_clear_imu_all.restype = None
        L.li_calib_data_sufficiency.argtypes = [vp, C.c_int, dp, C.c_int, C.c_int, dp, C.POINTER(C.c_int)]
        L.li_calib_initialize.argtypes = [vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(CalibResult)]
        L.li_calib_log_rows.argtypes = [vp, C.c_int, vp, C.c_int, C.POINTER(C.c_int)]
        _LIB = L
    return _LIB


def _v(a):
    return np.ascontiguousarray(a, np.float64).reshape(-1)


class LiCalib:
    def __init__(self, data_accum_length: float | None = None, converge_fully: bool = False):
        self.L = load()
        h = C.c_void_p()
        if self.L.li_calib_create(C.byref(h)) != 0:
            raise CalibError("li_calib_create failed")
        self.h = h
        if data_accum_length is not None:
            self.L.li_calib_set_data_accum_length(self.h, float(data_accum_length))
        self.L.li_calib_set_solver(self.h, int(converge_fully))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.li_calib_destroy(self.h)
            self.h = None

    def _ck(self, r, what):
        if r != 0:
            raise CalibError(f"{what}: error {r}")

    def push_imu_all(self, omg, acc, t, mean_acc_norm=9.81):
        self._ck(self.L.li_calib_push_imu_all(self.h, _v(omg), _v(acc), float(mean_acc_norm), float(t)), "push_imu_all")

    def push_lidar(self, R, omg, vel, t):
        self._ck(self.L.li_calib_push_lidar(self.h, _v(R), _v(omg), _v(vel), float(t)), "push_lidar")

    def push_imu(self, omg, acc, t):
        self._ck(self.L.li_calib_push_imu(self.h, _v(omg), _v(acc), float(t)), "push_imu")

    def clear_imu_all(self):
        """IMU_buffer_clear: drop the IMU samples pushed so far (the node's IMU loop-back)."""
        self.L.li_calib_clear_imu_all(self.h)

    def sizes(self):
        a, i, l = C.c_int(0), C.c_int(0), C.c_int(0)
        self._ck(self.L.li_calib_sizes(self.h, C.byref(a), C.byref(i), C.byref(l)), "sizes")
        return a.value, i.value, l.value

    def data_sufficiency(self, frame_num, lidar_omg, orig_odom_freq, cut_frame_num):
        pr = np.zeros(3)
        ok = C.c_int(0)
        self._ck(self.L.li_calib_data_sufficiency(self.h, int(frame_num), _v(lidar_omg), int(orig_odom_freq), int(cut_frame_num), pr,
                                                  C.byref(ok)), "data_sufficiency")
        return bool(ok.value), pr

    def initialize(self, orig_odom_freq, cut_frame_num, timediff_imu_wrt_lidar=0.0, move_start_time=0.0, from_groups=False):
        res = CalibResult()
        self._ck(self.L.li_calib_initialize(self.h, int(orig_odom_freq), int(cut_frame_num), float(timediff_imu_wrt_lidar),
                                            float(move_start_time), int(from_groups), C.byref(res)), "initialize")
        out = {}
        for name, _ in CalibResult._fields_:
            v = getattr(res, name)
            out[name] = np.array(v[:]) if hasattr(v, "__len__") else v
        out["R_LI"] = out["R_LI"].reshape(3, 3)
        return out

    def log_rows(self, name):
        which, cols = LOG_COLUMNS[name]
        n = C.c_int(0)
        self._ck(self.L.li_calib_log_rows(self.h, which, None, 0, C.byref(n)), "log_rows")
        out = np.zeros((max(n.value, 1), cols))
        self._ck(self.L.li_calib_log_rows(self.h, which, out.ctypes.data_as(C.c_void_p), n.value, C.byref(n)), "log_rows")
        return out[:n.value]
