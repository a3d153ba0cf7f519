"""Time the map assessment on the stored LIO phase of the synthetic Livox scenario (tools/bag_bench.py --synthetic, tests/test_gpu_bag.py).

    python tools/assess_bench.py [--seconds 60] [--sample 2000] [--device N]

Replays the scenario with `run --assess` (the bag and the outputs go to a temporary directory), then times on the stored scans, with
CUDA events around the calls and a synchronise: one evaluation of the final extrinsic (after a warm-up evaluation) and the 14-candidate
sweep. In the same call it times the numpy restatement (tests/assess_oracle.py, kd-tree candidates) on a query sample and extrapolates
it to all queries, with the number of host cores. Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

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
    ap.add_argument("--sample", type=int, default=2000, help="queries of the numpy restatement")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import numpy as np
    import torch

    import assess_oracle as ao
    import test_bag_node as tb
    from lidar_imu_init_b200 import assess, run
    with tempfile.TemporaryDirectory() as tmp:
        import pathlib
        ev, _ = tb.livox_events(a.seconds, 20_000)
        bag = os.path.join(tmp, "sim.bag")
        tb.write_event_bag(bag, ev, chunk_msgs=300)
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        seen = {}

        def on_node(nd):
            seen["nd"] = nd
            seen["g"] = nd.odom.g
            nd.odom.g.close = lambda: None
        t0 = time.perf_counter()
        rc = run.main(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, "out"), "--device", str(a.device),
                       "--quiet", "--assess"], on_node=on_node)
        replay = time.perf_counter() - t0
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
        g.assess_evaluate(R, T)                                  # warm-up
        evals = [timed(lambda: g.assess_evaluate(R, T)) for _ in range(5)]
        ms_eval = sorted(t for t, _ in evals)[2]
        res = evals[0][1]
        ms_sweep, _ = timed(lambda: A.sweep())
        # the numpy restatement on a query sample, extrapolated
        from scipy.spatial import cKDTree
        w = g.assess_placed()
        t0 = time.perf_counter()
        tree = cKDTree(w.astype(np.float64))
        t_tree = time.perf_counter() - t0
        ks = np.linspace(0, res["queries"] - 1, a.sample).astype(np.int64) * res["stride"]
        t0 = time.perf_counter()
        ao.evaluate_sample(w, tree, ks, 0.3, 10)
        t_q = (time.perf_counter() - t0) / a.sample
        cpu_eval = t_tree + t_q * res["queries"]
        out = dict(card=card(), points=res["points"], scans=res["scans"], queries=res["queries"], stride=res["stride"], valid=res["valid"],
                   evaluate_ms=round(ms_eval, 2), evaluate_ms_all=[round(t, 2) for t, _ in evals], sweep14_ms=round(ms_sweep, 1),
                   numpy_kdtree_s=round(t_tree, 2), numpy_per_query_ms=round(1e3 * t_q, 3), numpy_eval_extrapolated_s=round(cpu_eval, 1),
                   numpy_sweep_extrapolated_s=round(14 * cpu_eval, 1), host_cores=os.cpu_count(), replay_with_assess_s=round(replay, 1),
                   sweep_finds=sorted(k for k, v in assess.verdicts({n: r for n, _, _, r in A.sweep()}).items() if v[0] == "constrained"))
        type(g).close(g)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
