"""Time a joint refinement over several simulated recordings of one rig (tests/test_gpu_joint.py's scenario).

    python tools/joint_bench.py [--seconds 60] [--seeds 0,1] [--max-candidates 30] [--jobs 4] [--devices 0]

Writes one bag per trajectory seed (same extrinsic and lag) to a temporary directory and plays each as `python -m
lidar_imu_init_b200.joint` does, recording b on devices[b % n] with its --jobs contexts, measuring the device memory each recording takes
(free memory before it is played and after its workers exist). Then times joint.refine_replays with a host clock (every replay ends in a
device synchronise). Prints one JSON line with the card's name and power limit, the candidates and replays, the wall time and time per
candidate, each recording's device memory, the refined lag, and the extrinsic errors against the simulated truth.
"""
from __future__ import annotations

import argparse
import json
import os
import pathlib
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from assess_time_bench import card  # noqa: E402  (tools/)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--seeds", default="0,1")
    ap.add_argument("--max-candidates", type=int, default=30)
    ap.add_argument("--jobs", type=int, default=4)
    ap.add_argument("--devices", default="0")
    a = ap.parse_args()
    import test_bag_node as tb
    import test_gpu_joint as tg
    from lidar_imu_init_b200 import host, joint, run
    from lidar_imu_init_b200.node import Log
    seeds, devs = [int(s) for s in a.seeds.split(",")], joint.devices(a.devices)
    nodes, mem = [], []
    with tempfile.TemporaryDirectory() as tmp:
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        try:
            for b, seed in enumerate(seeds):
                bag = os.path.join(tmp, f"rec{b}.bag")
                tb.write_event_bag(bag, tg._events(seed, a.seconds), chunk_msgs=300)
                dev = devs[b % len(devs)]
                free0 = joint._free_bytes(dev)
                nd, _ = run.play(run.parse_args(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, f"rec{b}"),
                                                 "--device", str(dev), "--max-map-points", "3000000", "--refine"]), Log(quiet=True))
                nodes.append(nd)
                nd.replay.pool(a.jobs)
                mem.append(round((free0 - joint._free_bytes(dev)) / 1e6, 1))
            finals = [host.state_pose(nd.odom.state)[2:] for nd in nodes]
            ref = joint.refine_replays([nd.replay for nd in nodes], finals, a.max_candidates, a.jobs)
        finally:
            for nd in nodes:
                nd.replay.close()
                nd.odom.g.close()
    n = len(ref["trace"])
    e = tg._err(ref["R"], ref["T"])
    out = dict(card=card(), recordings=len(seeds), seconds=a.seconds, devices=devs, jobs=a.jobs, candidates=n, replays=n * len(seeds),
               status=ref["status"], wall_s=round(ref["wall_s"], 2), s_per_candidate=round(ref["wall_s"] / n, 3), device_mb=mem,
               lags_ms=[round(x * 1000, 3) for x in ref["lags"]], lag_ms=round(ref["time_lag"] * 1000, 3), sim_lag_ms=tg.T_OFF * 1000,
               rot_err_deg=round(e[0], 4), trans_err_mm=round(e[1], 2),
               final_err=[[round(x, 4) for x in tg._err(R, T)] for R, T in finals])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
