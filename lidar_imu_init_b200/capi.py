"""ctypes binding of the C-ABI (include/liinit_gpu.h). Thin: one method per entry point.

The CUDA library is REQUIRED: importing a handle without the built
libliinit_gpu.so, or on a machine without a usable GPU, raises -- there is no
CPU fallback on the product path.

Point arrays may be numpy arrays (the host entry points) or any object with a
__cuda_array_interface__, such as a torch CUDA tensor or a CuPy array (the
liinit_*_device twins: read in place on the GPU). Results of device calls are
torch tensors on the context's device; torch is imported only on those paths.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build

_LIB = None


class LiInitError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"liinit error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("filter_size_map", C.c_float), ("max_map_points", C.c_int), ("max_scan_points", C.c_int), ("device_id", C.c_int),
                ("brick_cells_log2", C.c_int), ("hash_capacity_log2", C.c_int), ("knn_group_lanes", C.c_int), ("knn_seed_radius_cells", C.c_float), ("knn_index", C.c_int), ("reserved", C.c_int * 6)]


class FrameParams(C.Structure):   # liinit_frame_params
    _fields_ = [("lidar_type", C.c_int), ("N_SCANS", C.c_int), ("blind", C.c_double), ("point_filter_num", C.c_int), ("required_frame_num", C.c_int),
                ("scan_count", C.c_int), ("stamp", C.c_double)]


class Pcl2Layout(C.Structure):   # liinit_pcl2_layout
    _fields_ = [("point_step", C.c_int), ("off_x", C.c_int), ("off_y", C.c_int), ("off_z", C.c_int), ("off_intensity", C.c_int), ("off_time", C.c_int),
                ("off_ring", C.c_int)]


class AssessParams(C.Structure):   # liinit_assess_params
    _fields_ = [("radius", C.c_double), ("min_neighbors", C.c_int), ("query_stride", C.c_int), ("as_run", C.c_int), ("reserved", C.c_int)]


class AssessResult(C.Structure):   # liinit_assess_result
    _fields_ = [("points", C.c_longlong), ("queries", C.c_longlong), ("stride", C.c_int), ("scans", C.c_int), ("valid", C.c_longlong),
                ("sparse", C.c_longlong), ("degenerate", C.c_longlong), ("mme", C.c_double), ("mpv", C.c_double)]


class AssessTiming(C.Structure):   # liinit_assess_timing
    _fields_ = [("poses", C.c_void_p), ("npose", C.c_int), ("reserved", C.c_int), ("rot", C.c_double * 9), ("pos", C.c_double * 3),
                ("R_LI", C.c_double * 9), ("T_LI", C.c_double * 3), ("vel", C.c_double * 3)]


ASSESS_MAX_QUERIES = 2_000_000   # LIINIT_ASSESS_MAX_QUERIES


class SubFrame(C.Structure):   # liinit_subframe
    _fields_ = [("handle", C.c_longlong), ("t_beg", C.c_double), ("end_ms", C.c_float), ("n", C.c_int)]


FRAME_MAX_CUT = 256   # LIINIT_FRAME_MAX_CUT
# liinit_cloud_download: the node's published clouds
CLOUD_REGISTERED = 1        # feats_undistort -> world (publish_frame_world with dense_pub_en; pcd_save)
CLOUD_REGISTERED_DOWN = 2   # feats_down_body -> world (publish_frame_world without dense_pub_en)
CLOUD_BODY = 3              # feats_undistort as it is (publish_frame_body)
CLOUD_EFFECT = 4            # laserCloudOri -> world (publish_effect_world)
# the sensor_msgs/PointCloud2 of pcl::toROSMsg(PointCloudXYZI) whose data the [n, 12] float32 records are: (name, offset, datatype,
# count); datatype 7 = FLOAT32
POINTCLOUD2_POINT_STEP = 48
POINTCLOUD2_FIELDS = (("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("normal_x", 16, 7, 1), ("normal_y", 20, 7, 1), ("normal_z", 24, 7, 1),
                      ("intensity", 32, 7, 1), ("curvature", 36, 7, 1))
# Livox CustomPoint: 19 bytes on the wire, 20 as the ROS struct (align=True)
LIVOX_POINT = np.dtype([("offset_time", "<u4"), ("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("reflectivity", "u1"), ("tag", "u1"), ("line", "u1")])
LIVOX_POINT_ALIGNED = np.dtype(LIVOX_POINT.descr, align=True)    # (np.dtype(LIVOX_POINT, align=True) would keep 19 bytes)

_f32 = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64 = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i32 = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")

SYMBOLS = [
    "liinit_create", "liinit_destroy", "liinit_last_error", "liinit_set_stream", "liinit_map_build", "liinit_map_add_points", "liinit_map_delete_boxes",
    "liinit_map_compact", "liinit_map_validnum", "liinit_map_size", "liinit_map_download", "liinit_map_nearest_search", "liinit_scan_upload", "liinit_scan_attach_host", "liinit_scan_upload_raw", "liinit_scan_download_body", "liinit_raw_upload", "liinit_raw_undistort_cv", "liinit_raw_undistort_imu",
    "liinit_raw_download", "liinit_raw_download_world", "liinit_raw_downsample",
    "liinit_frame_cut_livox", "liinit_frame_cut_pcl2", "liinit_frame_stage", "liinit_frame_download",
    "liinit_icp_iterate", "liinit_icp_iterate_device", "liinit_scan_download_effect", "liinit_scan_download_state",
    "liinit_cloud_download", "liinit_map_incremental", "liinit_last_pass_timing", "liinit_last_pass_kernel_times", "liinit_launch_count", "liinit_map_stats", "liinit_knn_index",
    "liinit_comm_unique_id", "liinit_comm_init", "liinit_comm_info", "liinit_comm_last_local", "liinit_comm_mode", "liinit_debug_esti_plane", "liinit_set_reseed",
    "liinit_get_stream", "liinit_map_build_device", "liinit_map_add_points_device", "liinit_scan_upload_device", "liinit_raw_upload_device",
    "liinit_map_nearest_search_device", "liinit_cloud_download_device", "liinit_map_download_device",
    "liinit_assess_reserve", "liinit_assess_append", "liinit_assess_info", "liinit_assess_evaluate", "liinit_assess_download",
    "liinit_assess_download_placed", "liinit_assess_cloud", "liinit_assess_reserve_timed", "liinit_assess_hold", "liinit_assess_append_timed",
    "liinit_assess_timing_info", "liinit_assess_evaluate_timed", "liinit_assess_clear", "liinit_map_snapshot", "liinit_map_restore",
    "liinit_replay_reserve", "liinit_replay_append", "liinit_replay_info", "liinit_replay_frame", "liinit_replay_stage",
    "liinit_replay_share", "liinit_replay_unshare",
]


def lib_path() -> str:
    # LIINIT_GPU_LIB: developer override to A/B alternative builds of the same C-ABI
    return os.environ.get("LIINIT_GPU_LIB") or _build.GPU_LIB


def load():
    """dlopen the in-tree CUDA library (no compute). Raises if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise FileNotFoundError(f"{p} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc) first. "
                                "There is no CPU fallback.")
    L = C.CDLL(p)
    vp = C.c_void_p
    L.liinit_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.liinit_destroy.argtypes = [vp]
    L.liinit_last_error.restype = C.c_char_p
    L.liinit_last_error.argtypes = [vp]
    L.liinit_set_stream.argtypes = [vp, vp]
    L.liinit_map_build.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_map_add_points.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.liinit_map_delete_boxes.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_map_compact.argtypes = [vp]
    L.liinit_map_validnum.argtypes = [vp, C.POINTER(C.c_int)]
    L.liinit_map_size.argtypes = [vp, C.POINTER(C.c_int)]
    L.liinit_map_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_map_nearest_search.argtypes = [vp, vp, C.c_int, C.c_int, C.c_double, vp, vp, vp]
    L.liinit_scan_upload.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_scan_attach_host.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_scan_upload_raw.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int)]
    L.liinit_raw_upload.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
    L.liinit_raw_undistort_cv.argtypes = [vp, _f64, _f64, _f64]
    L.liinit_raw_undistort_imu.argtypes = [vp, _f64, C.c_int, _f64, _f64, _f64, _f64]
    L.liinit_raw_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_raw_download_world.argtypes = [vp, _f64, _f64, _f64, _f64, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_raw_downsample.argtypes = [vp, C.c_float, C.POINTER(C.c_int)]
    L.liinit_frame_cut_livox.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(FrameParams), C.POINTER(SubFrame), C.c_int, C.POINTER(C.c_int)]
    L.liinit_frame_cut_pcl2.argtypes = [vp, vp, C.POINTER(Pcl2Layout), C.c_int, C.POINTER(FrameParams), C.POINTER(SubFrame), C.c_int,
                                        C.POINTER(C.c_int)]
    L.liinit_frame_stage.argtypes = [vp, C.c_longlong]
    L.liinit_frame_download.argtypes = [vp, C.c_longlong, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_scan_download_body.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_icp_iterate.argtypes = [vp, _f64, _f64, _f64, _f64, C.c_int, C.c_int, _f64, _f64, C.POINTER(C.c_int), C.POINTER(C.c_double)]
    L.liinit_icp_iterate_device.argtypes = [vp, _f64, _f64, _f64, _f64, C.c_int, C.c_int, vp]
    L.liinit_scan_download_effect.argtypes = [vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_scan_download_state.argtypes = [vp, vp, vp, vp, vp, vp]
    L.liinit_cloud_download.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
    L.liinit_map_incremental.argtypes = [vp, _f64, _f64, _f64, _f64, C.c_double, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.liinit_last_pass_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    L.liinit_last_pass_kernel_times.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.liinit_launch_count.argtypes = [vp, C.POINTER(C.c_longlong)]
    L.liinit_knn_index.argtypes = [vp, C.POINTER(C.c_int)]
    L.liinit_map_stats.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.liinit_comm_unique_id.argtypes = [vp]
    L.liinit_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_debug_esti_plane.argtypes = [vp, vp, C.c_int, vp, vp]
    L.liinit_comm_last_local.argtypes = [vp, _f64]
    L.liinit_comm_mode.argtypes = [vp, C.POINTER(C.c_int)]
    L.liinit_set_reseed.argtypes = [vp, C.c_int]
    L.liinit_comm_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.liinit_get_stream.argtypes = [vp, C.POINTER(vp)]
    L.liinit_map_build_device.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_map_add_points_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.liinit_scan_upload_device.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liinit_raw_upload_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
    L.liinit_map_nearest_search_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_double, vp, vp, vp]
    L.liinit_cloud_download_device.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int), vp]
    L.liinit_map_download_device.argtypes = [vp, vp, C.c_int, vp]
    set_assess_argtypes(L)
    for s in SYMBOLS:
        getattr(L, s).restype = getattr(L, s).restype if s == "liinit_last_error" else C.c_int
    _LIB = L
    return L


def set_assess_argtypes(L):
    """argtypes of the liinit_assess_* entry points on a loaded library"""
    vp = C.c_void_p
    L.liinit_assess_reserve.argtypes = [vp, C.c_longlong, C.c_int]
    L.liinit_assess_append.argtypes = [vp, _f64, _f64, _f64, _f64, C.POINTER(C.c_int)]
    L.liinit_assess_info.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.liinit_assess_evaluate.argtypes = [vp, C.POINTER(AssessParams), vp, vp, C.POINTER(AssessResult)]
    L.liinit_assess_download.argtypes = [vp, vp, vp, vp, C.c_longlong, C.POINTER(C.c_longlong)]
    L.liinit_assess_download_placed.argtypes = [vp, vp, C.c_longlong, C.POINTER(C.c_longlong)]
    L.liinit_assess_cloud.argtypes = [vp, C.POINTER(AssessParams), vp, vp, C.c_double, vp, C.c_longlong, C.POINTER(C.c_longlong),
                                      C.POINTER(AssessResult)]
    L.liinit_assess_reserve_timed.argtypes = [vp, C.c_longlong, C.c_int, C.c_longlong]
    L.liinit_assess_hold.argtypes = [vp]
    L.liinit_assess_append_timed.argtypes = [vp, _f64, _f64, _f64, _f64, C.POINTER(AssessTiming), C.POINTER(C.c_int)]
    L.liinit_assess_timing_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
    L.liinit_assess_evaluate_timed.argtypes = [vp, C.POINTER(AssessParams), vp, vp, C.c_double, C.POINTER(AssessResult)]
    for s in ("reserve", "append", "info", "evaluate", "download", "download_placed", "cloud", "reserve_timed", "hold", "append_timed",
              "timing_info", "evaluate_timed"):
        getattr(L, "liinit_assess_" + s).restype = C.c_int
    set_replay_argtypes(L)


def set_replay_argtypes(L):
    """argtypes of the LIO-phase replay entry points (liinit_assess_clear, liinit_map_snapshot / _restore, liinit_replay_*)"""
    vp = C.c_void_p
    L.liinit_assess_clear.argtypes = [vp]
    L.liinit_map_snapshot.argtypes = [vp, C.POINTER(C.c_longlong)]
    L.liinit_map_restore.argtypes = [vp]
    L.liinit_replay_reserve.argtypes = [vp, C.c_longlong, C.c_int]
    L.liinit_replay_append.argtypes = [vp, C.c_longlong, C.c_double, C.c_float, C.POINTER(C.c_int)]
    L.liinit_replay_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
    L.liinit_replay_frame.argtypes = [vp, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int)]
    L.liinit_replay_stage.argtypes = [vp, C.c_int]
    L.liinit_replay_share.argtypes = [vp, vp]
    L.liinit_replay_unshare.argtypes = [vp]
    for s in ("liinit_assess_clear", "liinit_map_snapshot", "liinit_map_restore", "liinit_replay_reserve", "liinit_replay_append",
              "liinit_replay_info", "liinit_replay_frame", "liinit_replay_stage", "liinit_replay_share", "liinit_replay_unshare"):
        getattr(L, s).restype = C.c_int


def _pts(a):
    """float32 C-contiguous [n, stride] with stride in (3, 4, 12)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] not in (3, 4, 12):
        raise ValueError("points must be [n,3], [n,4] or [n,12] float32")
    return a


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _cai(a):
    """The __cuda_array_interface__ of a device array, None for anything else (numpy arrays, CPU tensors)."""
    return getattr(a, "__cuda_array_interface__", None)


def _dev_rows(ci, widths):
    """(pointer, row stride in floats, rows) of a device array of float32 rows, C-contiguous, of one of the given widths."""
    if np.dtype(ci["typestr"]) != np.float32:
        raise LiInitError(-1, f"device points must be float32, not {np.dtype(ci['typestr'])}")
    shape = tuple(ci["shape"])
    if len(shape) != 2 or not widths(shape[1]):
        raise LiInitError(-1, f"device points of shape {shape}: the C-ABI takes [n, 3], [n, 4] or [n, 12] rows (raw clouds: [n, >= 3])")
    st = ci.get("strides")
    if st is not None and shape[0] > 0 and (st[1] != 4 or (shape[0] > 1 and st[0] != 4 * shape[1])):
        raise LiInitError(-1, f"device points with byte strides {tuple(st)}: rows must be contiguous float32 (e.g. .contiguous())")
    return C.c_void_p(ci["data"][0]), shape[1], shape[0]


def _xyz_rows(ci):
    return _dev_rows(ci, lambda w: w in (3, 4, 12))


def _torch():
    import torch
    return torch


class LiInitGpu:
    """One context = one GPU + one device-resident map + one resident scan."""

    def __init__(self, filter_size_map=0.15, max_map_points=6_000_000, max_scan_points=300_000, device_id=0, brick_cells_log2=0,
                 hash_capacity_log2=0, knn_group_lanes=0, knn_seed_radius_cells=0.0, knn_index=0):
        self.L = load()
        self.config = dict(filter_size_map=filter_size_map, max_map_points=max_map_points, max_scan_points=max_scan_points, device_id=device_id,
                           brick_cells_log2=brick_cells_log2, hash_capacity_log2=hash_capacity_log2, knn_group_lanes=knn_group_lanes,
                           knn_seed_radius_cells=knn_seed_radius_cells, knn_index=knn_index)
        cfg = Config(filter_size_map, max_map_points, max_scan_points, device_id, brick_cells_log2, hash_capacity_log2, knn_group_lanes, knn_seed_radius_cells,
                     knn_index)
        h = C.c_void_p()
        rc = self.L.liinit_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise LiInitError(rc, (self.L.liinit_last_error(None) or b"").decode())
        self.h = h
        self.scan_n = 0
        self.device_id = device_id
        self._tstream = None   # (stream pointer, torch.cuda.ExternalStream) of the context's stream

    def twin(self):
        """A new context with this one's configuration (an empty map)."""
        return type(self)(**self.config)

    def close(self):
        """Destroy the context. A lead whose replay store workers still share is refused (LiInitError) and stays open."""
        if getattr(self, "h", None):
            self._ck(self.L.liinit_destroy(self.h))
            self.h = None
            self._share_lead = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise LiInitError(rc, (self.L.liinit_last_error(self.h) or b"").decode())

    def set_stream(self, cuda_stream: int):
        self._ck(self.L.liinit_set_stream(self.h, C.c_void_p(cuda_stream)))

    def stream(self) -> int:
        """The cudaStream_t the context runs on (its own, or the one given to set_stream)."""
        s = C.c_void_p()
        self._ck(self.L.liinit_get_stream(self.h, C.byref(s)))
        return s.value or 0

    # ---- device calls: stream handshake with torch ----
    def _enter(self):
        """Before a device call: the context's stream waits for what torch's current stream has queued so far (an event, no device-wide
        synchronise), so a tensor written by torch just before is ready. Without torch or a CUDA device there is nothing to wait for."""
        try:
            torch = _torch()
        except ImportError:
            return None
        if not torch.cuda.is_available():
            return None
        ptr = self.stream()
        if self._tstream is None or self._tstream[0] != ptr:
            self._tstream = (ptr, torch.cuda.ExternalStream(ptr, device=torch.device("cuda", self.device_id)))
        ours, cur = self._tstream[1], torch.cuda.current_stream(self.device_id)
        ours.wait_stream(cur)
        return ours, cur

    @staticmethod
    def _leave(tok):
        """After a device call: torch's current stream waits for the context's stream, so results (and the reuse of the inputs' memory
        by torch's allocator) come after the call's work."""
        if tok is not None:
            tok[1].wait_stream(tok[0])

    def _dev_call(self, fn, *args):
        tok = self._enter()
        try:
            self._ck(fn(self.h, *args))
        finally:
            self._leave(tok)

    def _empty(self, shape, dtype):
        torch = _torch()
        return torch.empty(shape, dtype=getattr(torch, dtype), device=torch.device("cuda", self.device_id))

    @staticmethod
    def _tptr(t):
        return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None

    # ---- map ----
    def map_build(self, xyz):
        ci = _cai(xyz)
        if ci is not None:
            self._dev_call(self.L.liinit_map_build_device, *_xyz_rows(ci))
            return
        a = _pts(xyz)
        self._ck(self.L.liinit_map_build(self.h, _ptr(a), a.shape[1], a.shape[0]))

    def map_add_points(self, xyz, downsample_on: bool) -> int:
        ci = _cai(xyz)
        if ci is not None:
            p, stride, n = _xyz_rows(ci)
            added = C.c_int(0)
            if n == 0:
                return 0
            self._dev_call(self.L.liinit_map_add_points_device, p, stride, n, int(downsample_on), C.byref(added))
            return added.value
        a = _pts(xyz)
        added = C.c_int(0)
        if a.shape[0] == 0:
            return 0
        self._ck(self.L.liinit_map_add_points(self.h, _ptr(a), a.shape[1], a.shape[0], int(downsample_on), C.byref(added)))
        return added.value

    def map_delete_boxes(self, boxes) -> int:
        """boxes: [n, 6] float32 rows {min x,y,z, max x,y,z}; returns the number of deleted points."""
        b = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 6)
        d = C.c_int(0)
        self._ck(self.L.liinit_map_delete_boxes(self.h, _ptr(b), len(b), C.byref(d)))
        return d.value

    def map_compact(self):
        self._ck(self.L.liinit_map_compact(self.h))

    def map_validnum(self) -> int:
        n = C.c_int(0)
        self._ck(self.L.liinit_map_validnum(self.h, C.byref(n)))
        return n.value

    def map_size(self) -> int:
        n = C.c_int(0)
        self._ck(self.L.liinit_map_size(self.h, C.byref(n)))
        return n.value

    def map_download(self, device: bool = False):
        """The live map points as [n, 3] float32: numpy, or with device=True a torch tensor on the context's device."""
        if device:
            n = self.map_validnum()
            out = self._empty((n, 3), "float32")
            dn = self._empty((1,), "int32")
            self._dev_call(self.L.liinit_map_download_device, self._tptr(out), n, self._tptr(dn))
            return out
        n = self.map_validnum()
        out = np.zeros((max(n, 1), 3), np.float32)
        m = C.c_int(0)
        self._ck(self.L.liinit_map_download(self.h, _ptr(out), n, C.byref(m)))
        return out[:min(n, m.value)]

    def map_stats(self):
        b, s, pu, pc = C.c_int(0), C.c_int(0), C.c_longlong(0), C.c_longlong(0)
        self._ck(self.L.liinit_map_stats(self.h, C.byref(b), C.byref(s), C.byref(pu), C.byref(pc)))
        return dict(bricks=b.value, hash_slots=s.value, pool_used=pu.value, pool_cap=pc.value)

    def nearest_search(self, q, max_dist=5.0):
        """(xyz [n, 5, 3], d2 [n, 5], cnt [n]): numpy for host queries, torch tensors on the context's device for device queries."""
        ci = _cai(q)
        if ci is not None:
            p, stride, n = _xyz_rows(ci)
            xyz, d2, cnt = self._empty((n, 5, 3), "float32"), self._empty((n, 5), "float32"), self._empty((n,), "int32")
            self._dev_call(self.L.liinit_map_nearest_search_device, p, stride, n, max_dist, self._tptr(xyz), self._tptr(d2), self._tptr(cnt))
            return xyz, d2, cnt
        a = _pts(q)
        n = a.shape[0]
        xyz = np.zeros((n, 5, 3), np.float32)
        d2 = np.zeros((n, 5), np.float32)
        cnt = np.zeros(n, np.int32)
        self._ck(self.L.liinit_map_nearest_search(self.h, _ptr(a), a.shape[1], n, max_dist, _ptr(xyz), _ptr(d2), _ptr(cnt)))
        return xyz, d2, cnt

    # ---- scan ----
    def scan_upload(self, body):
        ci = _cai(body)
        if ci is not None:
            p, stride, n = _xyz_rows(ci)
            self._dev_call(self.L.liinit_scan_upload_device, p, stride, n)
            self.scan_n = n
            return
        a = _pts(body)
        self._ck(self.L.liinit_scan_upload(self.h, _ptr(a), a.shape[1], a.shape[0]))
        self.scan_n = a.shape[0]

    def scan_upload_raw(self, pts, leaf_size: float) -> int:
        """Voxel-grid downsample on the device (PCL VoxelGrid semantics), result becomes the resident scan."""
        a = _pts(pts)
        nd = C.c_int(0)
        self._ck(self.L.liinit_scan_upload_raw(self.h, _ptr(a), a.shape[1], a.shape[0], float(leaf_size), C.byref(nd)))
        self.scan_n = nd.value
        return nd.value

    # ---- raw-scan front end ----
    def raw_upload(self, pts, time_index: int = -1):
        ci = _cai(pts)
        if ci is not None:
            p, stride, n = _dev_rows(ci, lambda w: w >= 3)
            self._dev_call(self.L.liinit_raw_upload_device, p, stride, int(time_index), n)
            self.raw_n = n
            return
        a = np.ascontiguousarray(pts, dtype=np.float32)
        self._ck(self.L.liinit_raw_upload(self.h, _ptr(a), a.shape[1], int(time_index), a.shape[0]))
        self.raw_n = a.shape[0]

    def raw_undistort_cv(self, omega, rot_end, vel_end):
        self._ck(self.L.liinit_raw_undistort_cv(self.h, np.ascontiguousarray(omega, np.float64), np.ascontiguousarray(rot_end, np.float64).reshape(9),
                                                np.ascontiguousarray(vel_end, np.float64)))

    def raw_undistort_imu(self, poses, rot_end, pos_end, R_LI, T_LI):
        P = np.ascontiguousarray(poses, np.float64).reshape(-1, 22)
        self._ck(self.L.liinit_raw_undistort_imu(self.h, P.reshape(-1), len(P), np.ascontiguousarray(rot_end, np.float64).reshape(9),
                                                 np.ascontiguousarray(pos_end, np.float64), np.ascontiguousarray(R_LI, np.float64).reshape(9),
                                                 np.ascontiguousarray(T_LI, np.float64)))

    def raw_points(self):
        n = C.c_int(0)
        out = np.zeros((max(getattr(self, "raw_n", 0), 1), 3), np.float32)
        self._ck(self.L.liinit_raw_download(self.h, _ptr(out), len(out), C.byref(n)))
        return out[:n.value]

    def raw_world(self, rot_end, pos_end, R_LI, T_LI):
        """The staged (undistorted) raw cloud in the world frame, [n, 3] float32 in upload order (pointBodyToWorld)."""
        n = C.c_int(0)
        args = (np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64),
                np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64))
        self._ck(self.L.liinit_raw_download_world(self.h, *args, None, 0, C.byref(n)))
        out = np.zeros((n.value, 3), np.float32)
        self._ck(self.L.liinit_raw_download_world(self.h, *args, _ptr(out), n.value, C.byref(n)))
        return out

    def raw_downsample(self, leaf_size: float) -> int:
        nd = C.c_int(0)
        self._ck(self.L.liinit_raw_downsample(self.h, float(leaf_size), C.byref(nd)))
        self.scan_n = nd.value
        return nd.value

    # ---- cut-frame preprocess: driver message -> sub-frames on the device ----
    def frame_cut_livox(self, points, lidar_type=1, N_SCANS=6, blind=0.01, point_filter_num=1, required_frame_num=1, scan_count=0,
                        stamp=0.0):
        """Preprocess::process_cut_frame_livox. points: a structured array of LIVOX_POINT (19 bytes) or LIVOX_POINT_ALIGNED (20 bytes)
        records. Returns a list of dicts {handle, t_beg, end_ms, n}, in time order."""
        a = np.ascontiguousarray(points)
        stride, n = a.dtype.itemsize, len(a)
        P = FrameParams(lidar_type, N_SCANS, blind, point_filter_num, required_frame_num, scan_count, stamp)
        out = (SubFrame * max(required_frame_num, 1))()
        k = C.c_int(0)
        self._ck(self.L.liinit_frame_cut_livox(self.h, _ptr(a), stride, n, C.byref(P), out, len(out), C.byref(k)))
        return [dict(handle=out[i].handle, t_beg=out[i].t_beg, end_ms=out[i].end_ms, n=out[i].n) for i in range(k.value)]

    def frame_cut_pcl2(self, data, layout, n, lidar_type, N_SCANS=16, blind=0.01, point_filter_num=1, required_frame_num=1, scan_count=0,
                       stamp=0.0):
        """Preprocess::process_cut_frame_pcl2. data: the PointCloud2 data buffer (bytes or uint8 array); layout: dict of point_step and
        the byte offsets off_x, off_y, off_z, off_intensity, off_time, off_ring (-1 or missing = absent)."""
        a = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else data).view(np.uint8)
        if a.nbytes < int(n) * int(layout["point_step"]):
            raise ValueError(f"data holds {a.nbytes} bytes, fewer than n * point_step = {int(n) * int(layout['point_step'])}")
        Lo = Pcl2Layout(layout["point_step"], *[int(layout.get(f, -1)) for f in ("off_x", "off_y", "off_z", "off_intensity", "off_time", "off_ring")])
        P = FrameParams(lidar_type, N_SCANS, blind, point_filter_num, required_frame_num, scan_count, stamp)
        out = (SubFrame * max(required_frame_num, 1))()
        k = C.c_int(0)
        self._ck(self.L.liinit_frame_cut_pcl2(self.h, _ptr(a), C.byref(Lo), int(n), C.byref(P), out, len(out), C.byref(k)))
        return [dict(handle=out[i].handle, t_beg=out[i].t_beg, end_ms=out[i].end_ms, n=out[i].n) for i in range(k.value)]

    def frame_stage(self, handle: int):
        """The sub-frame becomes the staged raw cloud, as raw_upload(its PointType points, 9) would leave it."""
        self._ck(self.L.liinit_frame_stage(self.h, int(handle)))
        n = C.c_int(0)
        self._ck(self.L.liinit_frame_download(self.h, int(handle), None, 0, C.byref(n)))
        self.raw_n = n.value

    def frame_size(self, handle: int):
        """Points of a sub-frame the device still holds; None when its message slot has been reused by a later cut."""
        n = C.c_int(0)
        rc = self.L.liinit_frame_download(self.h, int(handle), None, 0, C.byref(n))
        if rc == -1:
            return None
        self._ck(rc)
        return n.value

    def frame_download(self, handle: int):
        """The sub-frame as [n, 12] float32 PointType rows (x, y, z, 1, normals 0, intensity, curvature, 0, 0)."""
        n = C.c_int(0)
        self._ck(self.L.liinit_frame_download(self.h, int(handle), None, 0, C.byref(n)))
        out = np.zeros((n.value, 12), np.float32)
        self._ck(self.L.liinit_frame_download(self.h, int(handle), _ptr(out), n.value, C.byref(n)))
        return out

    def scan_body(self):
        n = C.c_int(0)
        out = np.zeros((max(self.scan_n, 1), 3), np.float32)
        self._ck(self.L.liinit_scan_download_body(self.h, _ptr(out), self.scan_n, C.byref(n)))
        return out[:n.value]

    def scan_upload_ptr(self, host_ptr: int, stride: int, n: int):
        """Upload from a raw host pointer (e.g. pinned torch tensor)."""
        self._ck(self.L.liinit_scan_upload(self.h, C.c_void_p(host_ptr), stride, n))
        self.scan_n = n

    def scan_attach_ptr(self, host_ptr: int, stride: int, n: int):
        """Zero-copy variant: `host_ptr` is page-locked memory the first search pass reads over PCIe (see the header)."""
        self._ck(self.L.liinit_scan_attach_host(self.h, C.c_void_p(host_ptr), stride, n))
        self.scan_n = n

    def icp_iterate(self, rot_end, pos_end, R_LI, T_LI, imu_en: bool, search: bool):
        HtH = np.zeros((12, 12))
        Htr = np.zeros(12)
        m = C.c_int(0)
        rs = C.c_double(0)
        self._ck(self.L.liinit_icp_iterate(self.h, np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64),
                                           np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64),
                                           int(imu_en), int(search), HtH.reshape(144), Htr, C.byref(m), C.byref(rs)))
        return HtH, Htr, m.value, rs.value

    def icp_iterate_device(self, rot_end, pos_end, R_LI, T_LI, imu_en: bool, search: bool, d_out_ptr: int):
        self._ck(self.L.liinit_icp_iterate_device(self.h, np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64),
                                                  np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64),
                                                  int(imu_en), int(search), C.c_void_p(d_out_ptr)))

    def scan_state(self):
        n = self.scan_n
        out = dict(world=np.zeros((n, 3), np.float32), near_xyz=np.zeros((n, 5, 3), np.float32), near_cnt=np.zeros(n, np.int32),
                   selected=np.zeros(n, np.uint8), normvec=np.zeros((n, 4), np.float32))
        self._ck(self.L.liinit_scan_download_state(self.h, _ptr(out["world"]), _ptr(out["near_xyz"]), _ptr(out["near_cnt"]),
                                                   _ptr(out["selected"]), _ptr(out["normvec"])))
        return out

    def scan_effect(self):
        n = self.scan_n
        ori = np.zeros((n, 3), np.float32)
        nv = np.zeros((n, 4), np.float32)
        m = C.c_int(0)
        self._ck(self.L.liinit_scan_download_effect(self.h, _ptr(ori), _ptr(nv), n, C.byref(m)))
        return ori[:m.value], nv[:m.value]

    def cloud(self, which: int, rot_end=None, pos_end=None, R_LI=None, T_LI=None, device: bool = False):
        """One of the node's published clouds (CLOUD_*) as [n, 12] float32 pcl::PointXYZINormal records (the PointCloud2 data of
        POINTCLOUD2_FIELDS). The world-frame clouds need the pose (the posterior the node publishes with); CLOUD_BODY ignores it.
        device=True: a torch tensor on the context's device, built there in place."""
        pose = [None] * 4
        if rot_end is not None:
            pose = [np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64).reshape(3),
                    np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64).reshape(3)]
        args = [_ptr(a) for a in pose]
        n = C.c_int(0)
        if device:
            self._dev_call(self.L.liinit_cloud_download_device, int(which), *args, None, 0, C.byref(n), None)
            out = self._empty((n.value, 12), "float32")
            self._dev_call(self.L.liinit_cloud_download_device, int(which), *args, self._tptr(out), n.value, C.byref(n), None)
            return out
        self._ck(self.L.liinit_cloud_download(self.h, int(which), *args, None, 0, C.byref(n)))
        out = np.zeros((n.value, 12), np.float32)
        self._ck(self.L.liinit_cloud_download(self.h, int(which), *args, _ptr(out), n.value, C.byref(n)))
        return out

    def map_incremental(self, rot_end, pos_end, R_LI, T_LI, ds: float, flg_EKF_inited: bool = True):
        na, nn = C.c_int(0), C.c_int(0)
        self._ck(self.L.liinit_map_incremental(self.h, np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64),
                                               np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64),
                                               float(ds), int(flg_EKF_inited), C.byref(na), C.byref(nn)))
        return na.value, nn.value

    def last_pass_timing(self):
        ms, nl = C.c_float(0), C.c_int(0)
        self._ck(self.L.liinit_last_pass_timing(self.h, C.byref(ms), C.byref(nl)))
        return ms.value, nl.value

    def last_pass_kernel_times(self):
        a, b = C.c_float(0), C.c_float(0)
        self._ck(self.L.liinit_last_pass_kernel_times(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def debug_esti_plane(self, nb):
        """esti_plane of the device for neighbour sets nb [n, 5, 3] -> (pabcd [n, 4] f64, valid [n] bool)"""
        a = np.ascontiguousarray(nb, np.float32).reshape(-1, 15)
        out = np.zeros((len(a), 4))
        ok = np.zeros(len(a), np.uint8)
        self._ck(self.L.liinit_debug_esti_plane(self.h, _ptr(a), len(a), _ptr(out), _ptr(ok)))
        return out, ok.astype(bool)

    # ---- multi-GPU: the all-reduce of the accumulators and the gathers of per-point results live behind the C-ABI ----
    @staticmethod
    def comm_unique_id() -> bytes:
        """ncclGetUniqueId through the library (call on one rank, distribute the 128 bytes)."""
        L = load()
        buf = C.create_string_buffer(128)
        rc = L.liinit_comm_unique_id(buf)
        if rc != 0:
            raise LiInitError(rc, (L.liinit_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, unique_id: bytes, nranks: int, rank: int):
        """Collective: attach this context to an nranks-wide communicator. From then on icp_iterate returns the sum over the
        ranks and every rank works on its slot of the uploaded frame."""
        assert len(unique_id) == 128
        buf = C.create_string_buffer(unique_id, 128)
        self._ck(self.L.liinit_comm_init(self.h, buf, int(nranks), int(rank)))

    def set_reseed(self, enabled: bool):
        """later search passes of a scan start from the previous pass's neighbours (default on); off = every search from scratch"""
        self._ck(self.L.liinit_set_reseed(self.h, int(enabled)))

    def comm_mode(self) -> str:
        v = C.c_int(0)
        self._ck(self.L.liinit_comm_mode(self.h, C.byref(v)))
        return "peer memory (fused in the plane kernel)" if v.value else "ncclAllReduce"

    def comm_last_local(self):
        out = np.zeros(160)
        self._ck(self.L.liinit_comm_last_local(self.h, out))
        return out

    def comm_info(self):
        a, b, c, d = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        self._ck(self.L.liinit_comm_info(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(nranks=a.value, rank=b.value, shard_lo=c.value, shard_n=d.value)

    # ---- map assessment (DESIGN §4d) ----
    def assess_reserve(self, max_points: int, max_scans: int):
        """Allocate (or clear) the store of LIO scans and the evaluation buffers."""
        self._ck(self.L.liinit_assess_reserve(self.h, int(max_points), int(max_scans)))

    def assess_append(self, rot_end, pos_end, R_LI, T_LI) -> bool:
        """Store the staged cloud with its update's pose and extrinsic; False when the store had no room (the scan is counted as
        skipped)."""
        ok = C.c_int(0)
        self._ck(self.L.liinit_assess_append(self.h, np.ascontiguousarray(rot_end, np.float64).reshape(9), np.ascontiguousarray(pos_end, np.float64).reshape(3),
                                             np.ascontiguousarray(R_LI, np.float64).reshape(9), np.ascontiguousarray(T_LI, np.float64).reshape(3),
                                             C.byref(ok)))
        return bool(ok.value)

    def assess_info(self) -> dict:
        p, s, k = C.c_longlong(0), C.c_int(0), C.c_int(0)
        self._ck(self.L.liinit_assess_info(self.h, C.byref(p), C.byref(s), C.byref(k)))
        return dict(points=p.value, scans=s.value, skipped=k.value)

    def assess_evaluate(self, R_LI=None, T_LI=None, radius: float = 0.3, min_neighbors: int = 10, query_stride: int = 0,
                        as_run: bool = False) -> dict:
        """One evaluation of the stored scans with the candidate extrinsic (as_run: each scan's own). Returns the liinit_assess_result
        fields as a dict."""
        P = AssessParams(float(radius), int(min_neighbors), int(query_stride), int(bool(as_run)), 0)
        R = None if R_LI is None else np.ascontiguousarray(R_LI, np.float64).reshape(9)
        T = None if T_LI is None else np.ascontiguousarray(T_LI, np.float64).reshape(3)
        out = AssessResult()
        self._ck(self.L.liinit_assess_evaluate(self.h, C.byref(P), _ptr(R), _ptr(T), C.byref(out)))
        return {k: getattr(out, k) for k, _ in AssessResult._fields_}

    def assess_download(self):
        """(h, v, n) of every query of the last evaluation: float64, float64 (NaN when sparse or degenerate), int32."""
        q = C.c_longlong(0)
        self._ck(self.L.liinit_assess_download(self.h, None, None, None, 0, C.byref(q)))
        h, v, n = np.zeros(q.value), np.zeros(q.value), np.zeros(q.value, np.int32)
        self._ck(self.L.liinit_assess_download(self.h, _ptr(h), _ptr(v), _ptr(n), q.value, C.byref(q)))
        return h, v, n

    def assess_placed(self):
        """The stored points as the last evaluation placed them, [n, 3] float32 in stored order."""
        m = C.c_longlong(0)
        self._ck(self.L.liinit_assess_download_placed(self.h, None, 0, C.byref(m)))
        out = np.zeros((m.value, 3), np.float32)
        self._ck(self.L.liinit_assess_download_placed(self.h, _ptr(out), m.value, C.byref(m)))
        return out

    def assess_cloud(self, R_LI=None, T_LI=None, radius: float = 0.3, min_neighbors: int = 10, leaf: float = 0.1, as_run: bool = False):
        """Every stored point scored with the candidate extrinsic (as_run: each scan's own), as [n, 8] float32 records
        x y z entropy plane_variance neighbors points valid: one per stored point (leaf 0) or per occupied leaf of edge `leaf` [m].
        Returns (records, totals), totals the liinit_assess_result fields over every stored point. Leaves the last evaluation's
        per-query values (assess_download) as they are."""
        P = AssessParams(float(radius), int(min_neighbors), 1, int(bool(as_run)), 0)
        R = None if R_LI is None else np.ascontiguousarray(R_LI, np.float64).reshape(9)
        T = None if T_LI is None else np.ascontiguousarray(T_LI, np.float64).reshape(3)
        n = C.c_longlong(0)
        self._ck(self.L.liinit_assess_cloud(self.h, C.byref(P), _ptr(R), _ptr(T), float(leaf), None, 0, C.byref(n), None))
        rec = np.zeros((n.value, 8), np.float32)
        out = AssessResult()
        self._ck(self.L.liinit_assess_cloud(self.h, C.byref(P), _ptr(R), _ptr(T), float(leaf), _ptr(rec), n.value, C.byref(n), C.byref(out)))
        return rec[:n.value], {k: getattr(out, k) for k, _ in AssessResult._fields_}

    def assess_reserve_timed(self, max_points: int, max_scans: int, max_pose_rows: int):
        """Allocate (or clear) a timed store: the plain store plus the raw points and IMU pose tables of the timed scans."""
        self._ck(self.L.liinit_assess_reserve_timed(self.h, int(max_points), int(max_scans), int(max_pose_rows)))

    def assess_hold(self):
        """Hold the staged raw cloud for the next assess_append_timed (call it before the IMU undistortion)."""
        self._ck(self.L.liinit_assess_hold(self.h))

    def assess_append_timed(self, rot_end, pos_end, R_LI, T_LI, poses, prior) -> bool:
        """assess_append, plus the held raw cloud, its pose table (npose x 22, as given to raw_undistort_imu) and the propagated state
        of that call, prior = (rot_end, pos_end, R_LI, T_LI, vel_end). False when the store had no room (the scan is skipped)."""
        P = np.ascontiguousarray(poses, np.float64).reshape(-1, 22)
        t = AssessTiming()
        t.poses = P.ctypes.data
        t.npose = len(P)
        for name, v, k in zip(("rot", "pos", "R_LI", "T_LI", "vel"), prior, (9, 3, 9, 3, 3)):
            getattr(t, name)[:] = [float(x) for x in np.asarray(v, np.float64).reshape(k)]
        ok = C.c_int(0)
        self._ck(self.L.liinit_assess_append_timed(self.h, np.ascontiguousarray(rot_end, np.float64).reshape(9),
                                                   np.ascontiguousarray(pos_end, np.float64).reshape(3), np.ascontiguousarray(R_LI, np.float64).reshape(9),
                                                   np.ascontiguousarray(T_LI, np.float64).reshape(3), C.byref(t), C.byref(ok)))
        return bool(ok.value)

    def assess_timing_info(self) -> dict:
        a, b, r = C.c_int(0), C.c_int(0), C.c_longlong(0)
        self._ck(self.L.liinit_assess_timing_info(self.h, C.byref(a), C.byref(b), C.byref(r)))
        return dict(timed_scans=a.value, untimed_scans=b.value, pose_rows=r.value)

    def assess_evaluate_timed(self, R_LI=None, T_LI=None, lag_shift: float = 0.0, radius: float = 0.3, min_neighbors: int = 10,
                              query_stride: int = 0, as_run: bool = False) -> dict:
        """assess_evaluate with the timed scans re-undistorted for the candidate extrinsic and the lag shift [s]."""
        P = AssessParams(float(radius), int(min_neighbors), int(query_stride), int(bool(as_run)), 0)
        R = None if R_LI is None else np.ascontiguousarray(R_LI, np.float64).reshape(9)
        T = None if T_LI is None else np.ascontiguousarray(T_LI, np.float64).reshape(3)
        out = AssessResult()
        self._ck(self.L.liinit_assess_evaluate_timed(self.h, C.byref(P), _ptr(R), _ptr(T), float(lag_shift), C.byref(out)))
        return {k: getattr(out, k) for k, _ in AssessResult._fields_}

    def assess_clear(self):
        """Empty the assessment store, keeping its reservation."""
        self._ck(self.L.liinit_assess_clear(self.h))

    # ---- LIO-phase replay (DESIGN §4d) ----
    def map_snapshot(self) -> int:
        """Copy the map state and the staged raw cloud on the device; returns the bytes copied."""
        b = C.c_longlong(0)
        self._ck(self.L.liinit_map_snapshot(self.h, C.byref(b)))
        self._snap_raw_n = getattr(self, "raw_n", 0)
        return b.value

    def map_restore(self):
        """Put the map and the staged raw cloud back as map_snapshot found them."""
        self._ck(self.L.liinit_map_restore(self.h))
        self.raw_n = self._snap_raw_n

    def replay_reserve(self, max_points: int, max_frames: int):
        """Allocate (or clear) the store of the LIO phase's sub-frames."""
        self._ck(self.L.liinit_replay_reserve(self.h, int(max_points), int(max_frames)))

    def replay_append(self, handle: int, t_beg: float, end_ms) -> bool:
        """Keep sub-frame `handle` with its lidar_beg_time and end offset [ms]; False when the store had no room (counted as skipped)."""
        ok = C.c_int(0)
        self._ck(self.L.liinit_replay_append(self.h, int(handle), float(t_beg), float(np.float32(end_ms)), C.byref(ok)))
        return bool(ok.value)

    def replay_info(self) -> dict:
        f, k, p = C.c_int(0), C.c_int(0), C.c_longlong(0)
        self._ck(self.L.liinit_replay_info(self.h, C.byref(f), C.byref(k), C.byref(p)))
        return dict(frames=f.value, skipped=k.value, points=p.value)

    def replay_frame(self, j: int) -> dict:
        """{t_beg, end_ms (float32), n} of stored sub-frame j."""
        t, e, n = C.c_double(0), C.c_float(0), C.c_int(0)
        self._ck(self.L.liinit_replay_frame(self.h, int(j), C.byref(t), C.byref(e), C.byref(n)))
        return dict(t_beg=t.value, end_ms=np.float32(e.value), n=n.value)

    def replay_stage(self, j: int):
        """Stored sub-frame j becomes the staged raw cloud, as frame_stage left the original."""
        self._ck(self.L.liinit_replay_stage(self.h, int(j)))
        self.raw_n = self.replay_frame(j)["n"]

    def replay_share(self, lead):
        """Read `lead`'s replay store and map snapshot from now on (liinit_replay_share); this context keeps its own map and
        assessment store. Keeps a reference to the lead, which cannot be destroyed while this context shares it."""
        self._ck(self.L.liinit_replay_share(self.h, lead.h))
        self._share_lead = lead
        self._snap_raw_n = getattr(lead, "_snap_raw_n", 0)

    def replay_unshare(self):
        self._ck(self.L.liinit_replay_unshare(self.h))
        self._share_lead = None

    def knn_index(self) -> int:
        """1 = LIINIT_KNN_BRICKS (lockstep groups over whole bricks), 2 = LIINIT_KNN_CELLS (cell directory, thread per point)."""
        v = C.c_int()
        self._ck(self.L.liinit_knn_index(self.h, C.byref(v)))
        return v.value

    def launch_count(self) -> int:
        n = C.c_longlong(0)
        self._ck(self.L.liinit_launch_count(self.h, C.byref(n)))
        return n.value
