"""Time the LIO-phase replay on the synthetic Livox scenario (tests/test_gpu_bag.py).

    python tools/assess_replay_bench.py [--seconds 60] [--device N]

Runs the scenario with `run --assess` and a Replay attached (the bag and the outputs go to a temporary directory), then times, with a host
clock around calls that end in a device synchronise: one frozen replay of the final extrinsic (median of 3 after a warm-up) and the whole
17-replay sweep; and with CUDA events the map restore (median of 5), which copies what the snapshot at the hand-over copied. Prints one
JSON line with the card's name and power limit.
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

from assess_time_bench import card  # noqa: E402  (tools/)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import pathlib

    import torch

    import test_bag_node as tb
    from lidar_imu_init_b200 import assess, host, run
    with tempfile.TemporaryDirectory() as tmp:
        ev, _ = tb.livox_events(a.seconds, 20_000)
        bag = os.path.join(tmp, "sim.bag")
        tb.write_event_bag(bag, ev, chunk_msgs=300)
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        seen = {}

        def on_node(nd):
            seen["nd"] = nd
            nd.odom.g.close = lambda: None
            nd.replay = nd.odom.replay = assess.Replay(nd.odom.g, nd.assess)
        rc = run.main(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, "out"), "--device", str(a.device),
                       "--quiet", "--assess"], on_node=on_node)
        if rc != 0:
            sys.exit(rc)
        nd = seen["nd"]
        g, rp = nd.odom.g, nd.replay
        _, _, R, T = host.state_pose(nd.odom.state)
        rp.run(R, T)                                           # warm-up
        one = sorted(rp.run(R, T)["seconds"] for _ in range(3))
        t0 = time.perf_counter()
        rows = rp.sweep(R, T)
        sweep_s = time.perf_counter() - t0
        torch.cuda.set_device(a.device)
        stream = torch.cuda.ExternalStream(g.stream(), device=torch.device("cuda", a.device))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(6):
            e0.record(stream)
            g.map_restore()
            e1.record(stream)
            torch.cuda.synchronize(a.device)
            ts.append(e0.elapsed_time(e1))
        info = rp.info()
        out = dict(card=card(), subframes=info["frames"], points=info["points"], updates=len(rp.run_states),
                   snapshot_mb=round(rp.snapshot_bytes / 1e6, 1), restore_ms=round(sorted(ts[1:])[2], 3),
                   replay_s=round(one[1], 2), replay_s_all=[round(t, 2) for t in one], sweep_s=round(sweep_s, 1), sweep_replays=len(rows),
                   mme={name: round(r["result"]["mme"], 6) for name, _, _, _, r in rows})
        type(g).close(g)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
