"""One library variant (LIINIT_GPU_LIB), one line: search-kernel ms at both poses of the C2 scene cached in /tmp/c2_probe.npz.
   python tools/probe_variant.py [G]   (G: lanes per point, 0 = group_for's choice)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from lidar_imu_init_b200 import capi
if not os.path.exists('/tmp/c2_probe.npz'):
    from lidar_imu_init_b200 import scenes
    c = scenes.make_config("C2")
    np.savez('/tmp/c2_probe.npz', map=c["map_xyz"], body=c["body_xyz"], init_R=c["pose_init"].rot_end, init_p=c["pose_init"].pos_end,
             gt_R=c["pose_gt"].rot_end, gt_p=c["pose_gt"].pos_end)
z = np.load('/tmp/c2_probe.npz')
G = int(sys.argv[1]) if len(sys.argv) > 1 else 0
g = capi.LiInitGpu(0.15, max_map_points=6_000_000, max_scan_points=250_000, knn_index=1, knn_group_lanes=G)
g.map_build(z["map"]); g.scan_upload(z["body"])
out = [os.path.basename(os.environ.get("LIINIT_GPU_LIB", "default")) + f" G={G}"]
for pose in ("init", "gt"):
    R, p = z[pose + "_R"], z[pose + "_p"]
    I, zero = np.eye(3), np.zeros(3)
    ks = []
    for it in range(12):
        H, b, m, rs = g.icp_iterate(R, p, I, zero, False, True)
        ks.append(g.last_pass_kernel_times())
    ks = np.array(ks)
    out.append(f"{pose}: m={m} knn {np.median(ks[3:, 0]):.4f} (min {ks[:, 0].min():.4f}) plane {np.median(ks[3:, 1]):.4f} trace(HtH)={np.trace(H):.9e}")
print(" | ".join(out), flush=True)
