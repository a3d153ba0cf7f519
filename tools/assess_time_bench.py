"""Time the timed map assessment on the stored LIO phase of the synthetic Livox scenario (tests/test_gpu_bag.py).

    python tools/assess_time_bench.py [--seconds 60] [--device N]

Replays the scenario with `run --assess-time` (the bag and the outputs go to a temporary directory), then times on the stored scans, with
CUDA events around the calls and a synchronise: one plain evaluation of the final extrinsic, one timed evaluation at a 4 ms lag shift
(medians of 5, after a warm-up of each) and the whole sweep_time (14 candidates and the lag profile). Prints one JSON line with the
card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import pathlib

    import torch

    import test_bag_node as tb
    from lidar_imu_init_b200 import assess, run
    with tempfile.TemporaryDirectory() as tmp:
        ev, _ = tb.livox_events(a.seconds, 20_000)
        bag = os.path.join(tmp, "sim.bag")
        tb.write_event_bag(bag, ev, chunk_msgs=300)
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        seen = {}

        def on_node(nd):
            seen["nd"] = nd
            seen["g"] = nd.odom.g
            nd.odom.g.close = lambda: None
        rc = run.main(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, "out"), "--device", str(a.device),
                       "--quiet", "--assess-time"], on_node=on_node)
        if rc != 0:
            sys.exit(rc)
        g, A = seen["g"], seen["nd"].assess
        R, T = A.final
        torch.cuda.set_device(a.device)
        stream = torch.cuda.ExternalStream(g.stream(), device=torch.device("cuda", a.device))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed(fn):
            e0.record(stream)
            out = fn()
            e1.record(stream)
            torch.cuda.synchronize(a.device)
            return e0.elapsed_time(e1), out

        def median5(fn):
            fn()                                                 # warm-up
            ts = sorted(timed(fn)[0] for _ in range(5))
            return ts[2], ts
        ms_plain, all_plain = median5(lambda: g.assess_evaluate(R, T))
        ms_timed, all_timed = median5(lambda: g.assess_evaluate_timed(R, T, 0.004))
        ms_sweep, (rows, prof) = timed(lambda: A.sweep_time())
        info, ti = g.assess_info(), g.assess_timing_info()
        out = dict(card=card(), points=info["points"], scans=info["scans"], timed_scans=ti["timed_scans"], untimed_scans=ti["untimed_scans"],
                   pose_rows=ti["pose_rows"], evaluate_ms=round(ms_plain, 2), evaluate_ms_all=[round(t, 2) for t in all_plain],
                   evaluate_timed_ms=round(ms_timed, 2), evaluate_timed_ms_all=[round(t, 2) for t in all_timed],
                   sweep_time_ms=round(ms_sweep, 1), sweep_time_evaluations=len(rows) + len(prof), lag=assess.lag_verdict(prof))
        type(g).close(g)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
