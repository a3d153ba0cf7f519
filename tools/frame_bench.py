"""Wall time of the cut-frame preprocess for one driver message (information only): pinned host buffer -> sub-frame table, a host
clock around liinit_frame_cut_* (which ends in a stream synchronise), after warm-up; the CPU checker's single-thread time beside it.

  python tools/frame_bench.py [--reps 50] [--out DIR]

Messages: a 24k-point Livox CustomMsg (cut_frame_num 5) and a 230k-point, 128-ring spinning LiDAR PointCloud2 (Ouster layout with
times; Velodyne layout without a time field, i.e. the constant-rotation model; cut_frame_num 2). Prints the card name and power limit
of the same run and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _pinned(a):
    import torch
    t = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return t


def _time(fn, reps):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import frame_oracle as fo
    from lidar_imu_init_b200 import capi, scenes
    card = _card()
    print("card, power limit:", card, flush=True)
    g = capi.LiInitGpu(0.5, max_map_points=100_000, max_scan_points=300_000)
    res = dict(card=card)
    livox = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 100.0, 24_000, seed=1, tie_frac=0.05)
    prm = dict(N_SCANS=6, blind=0.5, point_filter_num=1, required_frame_num=5, scan_count=10, stamp=100.0)
    pin = _pinned(livox)
    P = capi.FrameParams(1, 6, 0.5, 1, 5, 10, 100.0)
    out = (capi.SubFrame * 8)()
    k = capi.C.c_int(0)

    def cut_livox():
        g._ck(g.L.liinit_frame_cut_livox(g.h, capi.C.c_void_p(pin.data_ptr()), livox.dtype.itemsize, len(livox), capi.C.byref(P), out, 8,
                                         capi.C.byref(k)))
    res["livox_24k_ms"] = _time(cut_livox, a.reps)
    res["livox_24k_checker_ms"] = _time(lambda: fo.cut_livox(livox, **prm), max(3, a.reps // 10))
    for name, lt, with_time in (("ouster_230k", 3, True), ("velodyne_230k_rotation", 2, False)):
        data, lay, n = scenes.spinning_pcl2(lt, 128, 1800, stamp=100.0, seed=2, with_time=with_time)
        pin2 = _pinned(data)
        Lo = capi.Pcl2Layout(lay["point_step"], *[lay[f] for f in ("off_x", "off_y", "off_z", "off_intensity", "off_time", "off_ring")])
        P2 = capi.FrameParams(lt, 128, 0.5, 1, 2, 30, 100.0)

        def cut_pcl2():
            g._ck(g.L.liinit_frame_cut_pcl2(g.h, capi.C.c_void_p(pin2.data_ptr()), capi.C.byref(Lo), n, capi.C.byref(P2), out, 8, capi.C.byref(k)))
        res[name + "_ms"] = _time(cut_pcl2, a.reps)
        res[name + "_checker_ms"] = _time(lambda: fo.cut_pcl2(data, lay, n, lt, N_SCANS=128, blind=0.5, required_frame_num=2, scan_count=30,
                                                              stamp=100.0), max(3, a.reps // 10))
    g.close()
    line = json.dumps(dict(res, unit="ms (median, min)"))
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "frame_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
