"""Wall time of the published clouds (liinit_cloud_download) at 230k raw points, and what the attribute channel costs the raw chain
(information only). Host clock around each call, ending in a device synchronise, median over --reps after warm-up.

  python tools/output_bench.py [--reps 50] [--old-lib PATH] [--out DIR]

1. Each cloud of a 230k-point, 128-ring Ouster PointCloud2 sub-frame (times given; CV undistortion; voxel grid 0.5 m; one search
   pass against a map of the scan itself) into a pageable numpy array and into page-locked host memory. Beside it, the way it was
   done before the records existed: liinit_raw_download_world (xyz), liinit_frame_download (the sub-frame again, for the
   intensities) and a numpy join into the same records.
2. With --old-lib (a build of libliinit_gpu.so without the attribute channel, e.g. the parent commit's): liinit_frame_stage,
   liinit_raw_upload (PointType, time index 9) and liinit_raw_downsample of the same sub-frame on both libraries, alternating
   old / new every repetition in one process, same calls through plain ctypes.
Prints the card name and power limit of the same run and one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _median(fn, reps, sync):
    for _ in range(3):
        fn()
        sync()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


class _Raw:
    """the raw-chain calls of one library through plain ctypes (the same code for the old and the new build)"""

    def __init__(self, path, data, lay, n):
        from lidar_imu_init_b200 import capi
        L = C.CDLL(path)
        vp = C.c_void_p
        L.liinit_create.argtypes = [C.POINTER(capi.Config), C.POINTER(vp)]
        L.liinit_destroy.argtypes = [vp]
        L.liinit_frame_cut_pcl2.argtypes = [vp, vp, C.POINTER(capi.Pcl2Layout), C.c_int, C.POINTER(capi.FrameParams), C.POINTER(capi.SubFrame),
                                            C.c_int, C.POINTER(C.c_int)]
        L.liinit_frame_stage.argtypes = [vp, C.c_longlong]
        L.liinit_frame_download.argtypes = [vp, C.c_longlong, vp, C.c_int, C.POINTER(C.c_int)]
        L.liinit_raw_upload.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.liinit_raw_downsample.argtypes = [vp, C.c_float, C.POINTER(C.c_int)]
        self.L, self.h = L, vp()
        cfg = capi.Config(0.5, 1_000_000, 300_000, 0, 0, 0, 0, 0.0, 0)
        assert L.liinit_create(C.byref(cfg), C.byref(self.h)) == 0
        Lo = capi.Pcl2Layout(lay["point_step"], *[lay[f] for f in ("off_x", "off_y", "off_z", "off_intensity", "off_time", "off_ring")])
        P = capi.FrameParams(3, 128, 0.5, 1, 1, 30, 100.0)
        out = (capi.SubFrame * 4)()
        k = C.c_int(0)
        assert L.liinit_frame_cut_pcl2(self.h, data.ctypes.data_as(vp), C.byref(Lo), n, C.byref(P), out, 4, C.byref(k)) == 0 and k.value == 1
        self.handle = out[0].handle
        self.p12 = np.zeros((out[0].n, 12), np.float32)
        assert L.liinit_frame_download(self.h, self.handle, self.p12.ctypes.data_as(vp), out[0].n, C.byref(k)) == 0
        self.nd = C.c_int(0)

    def frame_stage(self):
        assert self.L.liinit_frame_stage(self.h, self.handle) == 0

    def raw_upload(self):
        assert self.L.liinit_raw_upload(self.h, self.p12.ctypes.data_as(C.c_void_p), 12, 9, len(self.p12)) == 0

    def raw_downsample(self):
        assert self.L.liinit_raw_downsample(self.h, 0.5, C.byref(self.nd)) == 0

    def close(self):
        self.L.liinit_destroy(self.h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--old-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from lidar_imu_init_b200 import _build, capi, scenes
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    sync = torch.cuda.synchronize
    card = _card()
    print("card, power limit:", card, flush=True)
    res = dict(card=card)
    data, lay, n = scenes.spinning_pcl2(3, 128, 1800, stamp=100.0, seed=2, with_time=True)
    g = capi.LiInitGpu(0.5, max_map_points=2_000_000, max_scan_points=300_000)
    got = g.frame_cut_pcl2(data, lay, n, 3, N_SCANS=128, blind=0.5, point_filter_num=1, required_frame_num=1, scan_count=30, stamp=100.0)
    h = got[0]["handle"]
    R, p = scenes.so3_exp([0.1, -0.2, 0.7]), np.array([12.0, -3.0, 1.5])
    RLI, TLI = scenes.so3_exp([0.01, 0.02, 0.03]), np.array([0.05, -0.02, 0.1])
    pose = (R, p, RLI, TLI)

    def stage():
        g.frame_stage(h)
        g.raw_undistort_cv(np.array([0.01, 0.02, 0.4]), np.eye(3), np.array([1.0, 0.2, 0.0]))
    stage()
    g.raw_downsample(0.5)
    body = g.scan_body()
    g.map_build(((R @ (RLI @ body.T.astype(np.float64) + TLI[:, None])) + p[:, None]).T.astype(np.float32))
    stage()
    nd = g.raw_downsample(0.5)
    g.icp_iterate(R, p, RLI, TLI, False, True)
    res["points"] = dict(raw=int(got[0]["n"]), down=int(nd))
    args = [np.ascontiguousarray(x, np.float64).reshape(-1) for x in pose]
    ptrs = [x.ctypes.data_as(C.c_void_p) for x in args]
    k = C.c_int(0)
    for which, name in ((1, "registered"), (2, "registered_down"), (3, "body"), (4, "effect")):
        g._ck(g.L.liinit_cloud_download(g.h, which, *ptrs, None, 0, C.byref(k)))
        m = k.value
        pageable = np.zeros((m, 12), np.float32)
        pinned = torch.empty((m, 12), dtype=torch.float32, pin_memory=True)
        for dst, dname in ((pageable.ctypes.data, "pageable"), (pinned.data_ptr(), "pinned")):
            def call(dst=dst, which=which, m=m):
                g._ck(g.L.liinit_cloud_download(g.h, which, *ptrs, C.c_void_p(dst), m, C.byref(k)))
            res[f"{name}_{dname}_ms"] = _median(call, a.reps, sync)
        res[f"{name}_points"] = m
    # before: xyz in the world frame, the sub-frame again for its intensities, a join on the host into the same records
    p12 = np.zeros((got[0]["n"], 12), np.float32)

    def before():
        w = g.raw_world(*pose)
        f = g.frame_download(h)
        p12[:, 0:3] = w
        p12[:, 3] = 1.0
        p12[:, 4:8] = f[:, 4:8]
        p12[:, 8] = f[:, 8]
        p12[:, 9:12] = 0.0
    res["registered_before_ms"] = _median(before, a.reps, sync)
    before()
    assert np.array_equal(p12, g.cloud(1, *pose))
    g.close()
    if a.old_lib:
        libs = {"old": _Raw(a.old_lib, data, lay, n), "new": _Raw(_build.GPU_LIB, data, lay, n)}
        for op in ("frame_stage", "raw_upload", "raw_downsample"):
            ts = {v: [] for v in libs}
            for v, r in libs.items():      # warm-up
                for _ in range(3):
                    r.frame_stage()
                    getattr(r, op)()
                    sync()
            for _ in range(a.reps):
                for v, r in libs.items():
                    r.frame_stage()          # (the voxel grid needs a staged cloud)
                    sync()
                    t = time.perf_counter()
                    getattr(r, op)()
                    sync()
                    ts[v].append((time.perf_counter() - t) * 1e3)
            for v in libs:
                res[f"{op}_{v}_ms"] = float(np.median(ts[v]))
        for r in libs.values():
            r.close()
    line = json.dumps(dict(res, unit="ms (median wall time, ending in a device synchronise)"))
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "output_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
