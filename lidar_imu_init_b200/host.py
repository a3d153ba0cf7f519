"""ctypes binding of the host-side library (csrc/host/liinit_host.h): StatesGroup algebra, the IESKF update in
information form and the per-scan driver loop of laserMapping.cpp:936-1134 over the C-ABI."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build, capi

STATE_DOUBLES = 612  # rot_end9 pos3 R_LI9 T_LI3 vel3 bg3 ba3 grav3 cov576 (struct liinit_state)
_LIB = None
_f64 = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")


class ScanStats(C.Structure):
    _fields_ = [("iterations", C.c_int), ("search_passes", C.c_int), ("effect_feat_num", C.c_int), ("converged", C.c_int),
                ("last_rot_deg", C.c_double), ("last_trans_cm", C.c_double), ("res_sq", C.c_double)]


class Imu(C.Structure):
    """struct liinit_imu: the members of ImuProcess that its IMU branch uses (csrc/host/liinit_host.h)."""
    _fields_ = [("last_imu", C.c_double * 7), ("angvel_last", C.c_double * 3), ("acc_s_last", C.c_double * 3), ("last_lidar_end_time", C.c_double),
                ("cov_acc", C.c_double * 3), ("cov_gyr", C.c_double * 3), ("cov_acc_scale", C.c_double * 3), ("cov_gyr_scale", C.c_double * 3),
                ("cov_R_LI", C.c_double * 3), ("cov_T_LI", C.c_double * 3), ("cov_bias_gyr", C.c_double * 3), ("cov_bias_acc", C.c_double * 3),
                ("mean_acc_norm", C.c_double), ("need_init", C.c_int), ("reserved", C.c_int)]


class ReplayJob(C.Structure):
    """struct liinit_replay_job: where the native LIO loop of a replay starts (csrc/host/liinit_host.h)."""
    _fields_ = [("state", C.c_double * STATE_DOUBLES), ("imu", Imu), ("buf_rows", C.c_void_p), ("samples", C.c_void_p), ("events", C.c_void_p),
                ("last_stamp", C.c_double), ("timediff", C.c_double), ("time_lag", C.c_double), ("filter_size_surf", C.c_double),
                ("filter_size_map", C.c_double), ("n_buf", C.c_int), ("n_samples", C.c_int), ("n_events", C.c_int), ("frame_num", C.c_int),
                ("switch_scan", C.c_int), ("max_iteration", C.c_int), ("frozen", C.c_int), ("reserved", C.c_int)]


REPLAY_IMU = -1          # LIINIT_REPLAY_IMU: an event that is the next recorded IMU sample
IMU_SAMPLE_DOUBLES = 7   # {stamp, gyr xyz, acc xyz}
POSE6D_DOUBLES = 22      # {offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]}
MAX_IMU_POSES = 4096     # LIINIT_MAX_IMU_POSES (include/liinit_gpu.h)


def load():
    global _LIB
    if _LIB is not None:
        return _LIB
    capi.load()  # libliinit_gpu.so first (the host library links against it)
    if not os.path.exists(_build.HOST_LIB):
        raise FileNotFoundError(f"{_build.HOST_LIB} is missing: run __graft_entry__.build()")
    L = C.CDLL(_build.HOST_LIB)
    L.liinit_state_init.argtypes = [_f64]
    L.liinit_state_boxplus.argtypes = [_f64, _f64]
    L.liinit_state_boxminus.argtypes = [_f64, _f64, _f64]
    L.liinit_so3_exp.argtypes = [_f64, _f64]
    L.liinit_so3_log.argtypes = [_f64, _f64]
    L.liinit_ieskf_update.restype = C.c_int
    L.liinit_ieskf_update.argtypes = [_f64, _f64, _f64, _f64, _f64, C.c_void_p]
    L.liinit_scan_update.restype = C.c_int
    L.liinit_scan_update.argtypes = [C.c_void_p, _f64, C.c_int, C.c_int, C.POINTER(ScanStats)]
    L.liinit_ieskf_update_frozen.restype = C.c_int
    L.liinit_ieskf_update_frozen.argtypes = [_f64, _f64, _f64, _f64, _f64, C.c_void_p]
    L.liinit_scan_update_frozen.restype = C.c_int
    L.liinit_scan_update_frozen.argtypes = [C.c_void_p, _f64, C.c_int, C.c_int, C.POINTER(ScanStats)]
    L.liinit_propagate_cv.restype = None
    L.liinit_propagate_cv.argtypes = [_f64, C.c_double, _f64, _f64]
    pimu = C.POINTER(Imu)
    L.liinit_imu_init.restype = None
    L.liinit_imu_init.argtypes = [pimu]
    for f in ("gyr_cov", "acc_cov", "R_LI_cov", "T_LI_cov", "gyr_bias_cov", "acc_bias_cov"):
        getattr(L, "liinit_imu_set_" + f).restype = None
        getattr(L, "liinit_imu_set_" + f).argtypes = [pimu, _f64]
    L.liinit_imu_set_mean_acc_norm.restype = None
    L.liinit_imu_set_mean_acc_norm.argtypes = [pimu, C.c_double]
    L.liinit_imu_switch.restype = C.c_int
    L.liinit_imu_switch.argtypes = [pimu, _f64, C.c_int]
    L.liinit_imu_propagate.restype = C.c_int
    L.liinit_imu_propagate.argtypes = [pimu, _f64, _f64, C.c_int, C.c_double, C.c_double, _f64, C.POINTER(C.c_int)]
    set_replay_run_argtypes(L)
    L.liinit_fov_segment.restype = C.c_int
    L.liinit_fov_segment.argtypes = [_f64, C.c_double, C.c_double, np.ctypeslib.ndpointer(dtype=np.float32, flags='C_CONTIGUOUS'), C.POINTER(C.c_int),
                                     np.ctypeslib.ndpointer(dtype=np.float32, flags='C_CONTIGUOUS')]
    _LIB = L
    return L


def set_replay_run_argtypes(L):
    """argtypes of liinit_replay_run on a loaded host library"""
    L.liinit_replay_run.restype = C.c_int
    L.liinit_replay_run.argtypes = [C.c_void_p, C.POINTER(ReplayJob), _f64, np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS"), C.c_int,
                                    C.POINTER(C.c_int)]


def replay_run(gpu, odom, samples, events, lib=None):
    """liinit_replay_run on gpu's context from a handed-over LidarOdometry `odom` (its state, IMU processor, IMU buffer and loop
    settings): samples [k, 7] the recorded IMU samples {t, gyr, acc} as they arrived, events int32 (a stored sub-frame index or
    REPLAY_IMU). lib: the host library to run it in (default: this package's). Returns [(stored sub-frame index, posterior state)] of
    every update; raises capi.LiInitError with the context's message when a call failed."""
    L = load() if lib is None else lib
    samples = np.ascontiguousarray(samples, np.float64).reshape(-1, IMU_SAMPLE_DOUBLES)
    events = np.ascontiguousarray(events, np.int32)
    ib = odom.imu_buffer
    buf = np.ascontiguousarray(np.array(list(ib.rows), np.float64).reshape(-1, IMU_SAMPLE_DOUBLES))
    job = ReplayJob()
    job.state[:] = [float(x) for x in np.asarray(odom.state, np.float64)]
    job.imu = Imu.from_buffer_copy(odom.imu_proc.m)
    job.buf_rows, job.samples, job.events = buf.ctypes.data, samples.ctypes.data, events.ctypes.data
    job.last_stamp, job.timediff, job.time_lag = float(ib.last_stamp), float(ib.timediff), float(ib.time_lag)
    job.filter_size_surf, job.filter_size_map = float(odom.filter_size_surf), float(odom.ds)
    job.n_buf, job.n_samples, job.n_events = len(buf), len(samples), len(events)
    job.frame_num = int(odom.frame_num)
    job.switch_scan = -1 if odom.switch_scan is None else int(odom.switch_scan)
    job.max_iteration, job.frozen = int(odom.max_iteration), int(bool(odom.frozen))
    cap = int(np.count_nonzero(events >= 0))
    states = np.zeros((max(cap, 1), STATE_DOUBLES))
    frames = np.zeros(max(cap, 1), np.int32)
    n = C.c_int(0)
    rc = L.liinit_replay_run(gpu.h, C.byref(job), states.reshape(-1), frames, cap, C.byref(n))
    if rc != 0:
        raise capi.LiInitError(rc, "liinit_replay_run: " + (gpu.L.liinit_last_error(gpu.h) or b"").decode())
    return [(int(frames[k]), states[k].copy()) for k in range(n.value)]


def state_init():
    s = np.zeros(STATE_DOUBLES)
    load().liinit_state_init(s)
    return s


def state_from_pose(rot_end, pos_end, R_LI, T_LI):
    s = state_init()
    s[0:9] = np.asarray(rot_end, float).reshape(9)
    s[9:12] = pos_end
    s[12:21] = np.asarray(R_LI, float).reshape(9)
    s[21:24] = T_LI
    return s


def state_pose(s):
    return s[0:9].reshape(3, 3).copy(), s[9:12].copy(), s[12:21].reshape(3, 3).copy(), s[21:24].copy()


def boxplus(s, d):
    s = np.ascontiguousarray(s, np.float64).copy()
    load().liinit_state_boxplus(s, np.ascontiguousarray(d, np.float64))
    return s


def boxminus(a, b):
    o = np.zeros(24)
    load().liinit_state_boxminus(np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64), o)
    return o


def ieskf_update(state, state_prop, HtH, Htr, frozen=False):
    """One IESKF update; frozen: the extrinsic held constant (liinit_ieskf_update_frozen)."""
    s = np.ascontiguousarray(state, np.float64).copy()
    sol = np.zeros(24)
    KH = np.zeros((24, 12))
    L = load()
    rc = (L.liinit_ieskf_update_frozen if frozen else L.liinit_ieskf_update)(s, np.ascontiguousarray(state_prop, np.float64), np.ascontiguousarray(HtH, np.float64).reshape(144),
                                    np.ascontiguousarray(Htr, np.float64), sol, KH.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise RuntimeError("liinit_ieskf_update failed (singular covariance?)")
    return s, sol, KH


def propagate_cv(state, dt, cov_gyr_scale=0.1, cov_acc_scale=0.1):
    """Constant-velocity propagation of the LiDAR-only mode (IMU_Processing.hpp:212-243); covariance scales as
    mapping/gyr_cov, mapping/acc_cov (laserMapping.cpp:776-777,833-834)."""
    s = np.ascontiguousarray(state, np.float64).copy()
    load().liinit_propagate_cv(s, float(dt), np.full(3, cov_gyr_scale, np.float64) if np.isscalar(cov_gyr_scale) else np.ascontiguousarray(cov_gyr_scale, np.float64),
                               np.full(3, cov_acc_scale, np.float64) if np.isscalar(cov_acc_scale) else np.ascontiguousarray(cov_acc_scale, np.float64))
    return s


def scan_update(gpu: capi.LiInitGpu, state, max_iteration=5, imu_en=False, frozen=False):
    """Per-scan ICP + IESKF update on the scan already uploaded to `gpu`; frozen: the extrinsic held constant
    (liinit_scan_update_frozen). Returns (posterior state, stats dict)."""
    s = np.ascontiguousarray(state, np.float64).copy()
    st = ScanStats()
    L = load()
    rc = (L.liinit_scan_update_frozen if frozen else L.liinit_scan_update)(gpu.h, s, int(max_iteration), int(imu_en), C.byref(st))
    if rc != 0:
        raise capi.LiInitError(rc, (gpu.L.liinit_last_error(gpu.h) or b"").decode())
    return s, {k: getattr(st, k) for k, _ in ScanStats._fields_}


class ImuProcess:
    """The IMU branch of ImuProcess (IMU_Processing.hpp) over liinit_imu_*: its members live in a struct liinit_imu."""

    def __init__(self):
        self.m = Imu()
        load().liinit_imu_init(C.byref(self.m))

    def set_cov(self, which: str, v):
        """which: gyr_cov, acc_cov (the scales), R_LI_cov, T_LI_cov, gyr_bias_cov or acc_bias_cov."""
        v = np.full(3, v, np.float64) if np.isscalar(v) else np.ascontiguousarray(v, np.float64)
        getattr(load(), "liinit_imu_set_" + which)(C.byref(self.m), v)

    def set_mean_acc_norm(self, v: float):
        load().liinit_imu_set_mean_acc_norm(C.byref(self.m), float(v))

    @property
    def need_init(self) -> bool:
        return bool(self.m.need_init)

    def switch(self, samples):
        """The switch scan (Process :445-453): samples [k, 7] {stamp, gyr, acc}."""
        a = np.ascontiguousarray(samples, np.float64).reshape(-1, IMU_SAMPLE_DOUBLES)
        rc = load().liinit_imu_switch(C.byref(self.m), a.reshape(-1), len(a))
        if rc != 0:
            raise capi.LiInitError(rc, "liinit_imu_switch")

    def propagate(self, state, samples, pcl_beg_time: float, pcl_end_offset_ms: float):
        """propagation_and_undist without its point loop: returns (propagated state, IMUpose table [npose, 22])."""
        s = np.ascontiguousarray(state, np.float64).copy()
        a = np.ascontiguousarray(samples, np.float64).reshape(-1, IMU_SAMPLE_DOUBLES)
        poses = np.zeros((len(a) + 1, POSE6D_DOUBLES))
        n = C.c_int(0)
        rc = load().liinit_imu_propagate(C.byref(self.m), s, a.reshape(-1), len(a), float(pcl_beg_time), float(pcl_end_offset_ms), poses.reshape(-1),
                                         C.byref(n))
        if rc != 0:
            raise capi.LiInitError(rc, "liinit_imu_propagate: " + ("IMU pose table longer than %d poses" % MAX_IMU_POSES if rc == -3 else
                                                                   "called before the switch scan"))
        return s, poses[:n.value]


class FovSegmenter:
    """lasermap_fov_segment (laserMapping.cpp:260-305) with its two globals (LocalMap_Points, Localmap_Initialized)."""

    def __init__(self, cube_len: float, det_range: float):
        self.cube_len, self.det_range = float(cube_len), float(det_range)
        self.box = np.zeros(6, np.float32)
        self.init = C.c_int(0)

    def update(self, pos_lidar):
        out = np.zeros(18, np.float32)
        n = load().liinit_fov_segment(np.ascontiguousarray(pos_lidar, np.float64), self.cube_len, self.det_range, self.box, C.byref(self.init), out)
        return out.reshape(3, 6)[:n].copy()
