"""Host-memory entry points against their device-pointer twins (liinit_*_device) on the same context, timed alternately in one process.

    python tools/device_io_bench.py [--steps 20] [--warmup 3] [--out FILE.json]

Cases (what a caller whose clouds are already on the GPU pays with each path):
  scan+search   the 240k-point C2 scan: upload, then the first search pass (liinit_icp_iterate, which synchronises)
  raw+voxel     a 230k-point PointType raw cloud: upload, then the voxel grid (liinit_raw_downsample, which synchronises)
  registered    /cloud_registered of that cloud: records into page-locked host memory against records built in device memory
  queries       2^20 stand-alone 5-NN queries: results to host arrays against results left in device tensors
Host inputs are numpy arrays (pageable memory), device inputs CUDA tensors already resident. Every step of both paths is timed with the
host clock between two device synchronisations, and its outputs are compared with the other path's: a mismatch stops the run. The card
and its power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import capi, scenes  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return (time.perf_counter() - t0) * 1e3, out


def run_case(name, host_fn, dev_fn, same, steps, warmup, sync):
    th, td = [], []
    for k in range(warmup + steps):
        a, ra = timed(host_fn, sync)
        b, rb = timed(dev_fn, sync)
        if not same(ra, rb):
            raise SystemExit(f"{name}: host and device paths differ at step {k}")
        if k >= warmup:
            th.append(a)
            td.append(b)
    r = dict(case=name, host_ms_median=float(np.median(th)), device_ms_median=float(np.median(td)), host_ms_min=float(np.min(th)),
             device_ms_min=float(np.min(td)), steps=steps)
    print(f"{name:>12}: host {r['host_ms_median']:8.3f} ms  device {r['device_ms_median']:8.3f} ms  (median of {steps}; min "
          f"{r['host_ms_min']:.3f} / {r['device_ms_min']:.3f})", flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    name, pl = card()
    print(f"device: {name}, power limit {pl}", flush=True)
    sync = torch.cuda.synchronize
    res = []

    # scan upload + first search pass, C2 (240k points)
    c = scenes.make_config("C2")
    p = c["pose_init"]
    N = len(c["body_xyz"])
    g = capi.LiInitGpu(c["ds"], max_map_points=2 * len(c["map_xyz"]), max_scan_points=N + 16)
    g.set_reseed(False)
    g.map_build(c["map_xyz"])
    body_h = np.ascontiguousarray(c["body_xyz"])
    body_d = torch.from_numpy(np.concatenate([body_h, np.zeros((N, 1), np.float32)], 1)).cuda()

    def scan(src):
        g.scan_upload(src)
        return g.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    same_pass = lambda x, y: all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(x, y))  # noqa: E731
    res.append(run_case("scan+search", lambda: scan(body_h), lambda: scan(body_d), same_pass, a.steps, a.warmup, sync))

    # queries: 2^20 stand-alone 5-NN
    nq = 1 << 20
    poses = [p] + [scenes.perturb_pose(c["pose_gt"], 40 + i, 0.3, 0.05) for i in range(nq // N + 1)]
    q_h = np.ascontiguousarray(np.concatenate([(P.rot_end @ (P.R_LI @ body_h.T.astype(np.float64) + P.T_LI[:, None]) + P.pos_end[:, None]).T.astype(np.float32)
                          for P in poses])[:nq])
    q_d = torch.from_numpy(q_h).cuda()
    same_q = lambda x, y: all(np.array_equal(u, v.cpu().numpy()) for u, v in zip(x, y))  # noqa: E731
    res.append(run_case("queries", lambda: g.nearest_search(q_h), lambda: g.nearest_search(q_d), same_q, a.steps, a.warmup, sync))
    g.close()

    # PointType raw cloud (230k points): upload + voxel grid; then /cloud_registered
    def pose_at(t):
        t = np.atleast_1d(np.asarray(t, float))
        cy, sy = np.cos(0.3 * t), np.sin(0.3 * t)
        R = np.zeros((len(t), 3, 3))
        R[:, 0, 0], R[:, 0, 1], R[:, 1, 0], R[:, 1, 1], R[:, 2, 2] = cy, -sy, sy, cy, 1.0
        return R, np.stack([7.0 + 0.5 * np.sin(t), np.full_like(t, 7.5), np.full_like(t, 1.5)], 1)
    n = 230_000
    raw_h = scenes.timed_scan_points(scenes.box_scene(15.0, 15.0, 6.0, 2, 2), pose_at, 10.0, 0.1, n, seed=7, det_range=60.0)
    raw_h = np.ascontiguousarray(raw_h)
    raw_d = torch.from_numpy(raw_h).cuda()
    g = capi.LiInitGpu(0.3, max_map_points=2_000_000, max_scan_points=n + 16)
    res.append(run_case("raw+voxel", lambda: (g.raw_upload(raw_h, 9), g.raw_downsample(0.3))[1],
                        lambda: (g.raw_upload(raw_d, 9), g.raw_downsample(0.3))[1], lambda x, y: x == y, a.steps, a.warmup, sync))
    pose = [np.ascontiguousarray(x, np.float64).reshape(-1) for x in (p.rot_end, p.pos_end, p.R_LI, p.T_LI)]
    pp = [x.ctypes.data_as(capi.C.c_void_p) for x in pose]
    pinned = torch.empty((n, 12), dtype=torch.float32).pin_memory()
    rec_d = torch.empty((n, 12), dtype=torch.float32, device="cuda")
    cnt = capi.C.c_int()

    def reg_host():
        g._ck(g.L.liinit_cloud_download(g.h, capi.CLOUD_REGISTERED, *pp, capi.C.c_void_p(pinned.data_ptr()), n, capi.C.byref(cnt)))
        return pinned

    def reg_dev():
        g._dev_call(g.L.liinit_cloud_download_device, capi.CLOUD_REGISTERED, *pp, capi.C.c_void_p(rec_d.data_ptr()), n, capi.C.byref(cnt), None)
        return rec_d
    res.append(run_case("registered", reg_host, reg_dev, lambda x, y: torch.equal(x, y.cpu()), a.steps, a.warmup, sync))
    g.close()
    out = dict(device=name, power_limit=pl, cases=res)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
