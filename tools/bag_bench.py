"""Wall time of a bag replay per recorded second, and the real-time factor, for information only.

    python tools/bag_bench.py --config cfg.yaml --bag rec.bag [--param k=v ...] [--device N]
    python tools/bag_bench.py --synthetic SECONDS [--ros2]   # writes the Livox scenario of tests/test_gpu_bag.py (20k points / message);
                                                             # --ros2: as the rosbag2 directory of tests/test_gpu_bag2.py

--bag takes whatever `run --bag` takes: a ROS1 bag, a rosbag2 directory or a .db3 file. --record also replays the bag a second time
with `run --record` (every topic the node publishes, in the format of the input) and reports both runs and the recording's size.

Prints one JSON line: recorded seconds, wall seconds, wall per recorded second and the real-time factor (recorded / wall; > 1 is
faster than real time); with --record also record_wall_s, record_real_time_factor and record_bytes. The bag and the outputs go to a
temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config")
    ap.add_argument("--bag")
    ap.add_argument("--param", action="append", default=[])
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--synthetic", type=float, default=0.0, help="seconds of the synthetic Livox scenario")
    ap.add_argument("--ros2", action="store_true", help="write the synthetic scenario as a ROS 2 bag (livox_ros_driver2/msg/CustomMsg)")
    ap.add_argument("--record", action="store_true", help="replay once more with run --record and report both")
    a = ap.parse_args()
    from lidar_imu_init_b200 import rosbag, rosbag2, run
    with tempfile.TemporaryDirectory() as tmp:
        if a.synthetic:
            import pathlib

            import test_bag_node as tb
            ev, _ = tb.livox_events(a.synthetic, 20_000)
            if a.ros2:
                import test_bag2_node as t2
                a.bag = os.path.join(tmp, "sim_ros2")
                t2.write_event_bag2(a.bag, ev, files=3)
            else:
                a.bag = os.path.join(tmp, "sim.bag")
                tb.write_event_bag(a.bag, ev, chunk_msgs=300)
            tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
            a.config = os.path.join(tmp, "sim.yaml")
        with rosbag2.open_bag(a.bag) as b:
            if isinstance(b, rosbag.Bag):
                times = [e[1] for c in b.chunks for e in c.entries]
                bounds = (min(times), max(times)) if times else None
            else:
                bounds = b.time_bounds()
            fmt = b.format
        if bounds is None:
            sys.exit(f"{a.bag}: the bag holds no messages")
        t0, t1 = bounds
        recorded = (t1 - t0) * 1e-9
        seen = {}
        argv = ["--config", a.config, "--bag", a.bag, "--out", os.path.join(tmp, "out"), "--device", str(a.device), "--quiet"]
        for p in a.param:
            argv += ["--param", p]
        t0 = time.perf_counter()
        rc = run.main(argv, on_node=lambda nd: seen.update(node=nd))
        wall = time.perf_counter() - t0
        if rc != 0:
            sys.exit(rc)
        nd = seen["node"]
        res = dict(format=fmt, recorded_s=round(recorded, 3), wall_s=round(wall, 3), wall_per_recorded_s=round(wall / recorded, 4),
                   real_time_factor=round(recorded / wall, 3), updates=nd.updates, dropped_subframes=nd.odom.dropped_subframes,
                   init_frame=nd.init_scan, refine_frame=nd.refine_scan)
        if a.record:
            rec = os.path.join(tmp, "recording")
            argv[argv.index("--out") + 1] = os.path.join(tmp, "out_record")
            t0 = time.perf_counter()
            rc = run.main(argv + ["--record", rec])
            wall_r = time.perf_counter() - t0
            if rc != 0:
                sys.exit(rc)
            size = os.path.getsize(rec) if os.path.isfile(rec) else sum(os.path.getsize(os.path.join(rec, f)) for f in os.listdir(rec))
            res.update(record_wall_s=round(wall_r, 3), record_real_time_factor=round(recorded / wall_r, 3), record_bytes=size)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
