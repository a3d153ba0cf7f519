"""Time concurrent LIO replays on the synthetic Livox scenario (tests/test_gpu_bag.py).

    python tools/replay_jobs_bench.py [--seconds 60] [--jobs 1,2,4,8,12] [--device N]

Runs the scenario with `run --assess` and a Replay attached (the bag and the outputs go to a temporary directory), then, with a host clock
around calls that end in a device synchronise:
  - one frozen replay of the final extrinsic by the Python loop (Replay.run) and by the native loop (Replay.run_native), medians of 3;
  - the 17-replay sweep by the Python loop, then at each K of --jobs by the native loop on K contexts (Replay.sweep(jobs=K)), with the
    device bytes each new worker took (free device memory before and after it was created);
  - Replay.refine at the default budget with the K whose sweep was fastest;
  - Replay.refine with a budget of 600 at that K: its status, and how many replays it used.
Prints one JSON line with the card's name and power limit, read in the same process.
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
    ap.add_argument("--jobs", default="1,2,4,8,12")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import pathlib

    import numpy as np
    import torch

    import test_bag_node as tb
    from lidar_imu_init_b200 import assess, host, run
    ks = [int(k) for k in a.jobs.split(",")]
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
                       "--max-map-points", "3000000", "--quiet", "--assess"], on_node=on_node)
        if rc != 0:
            sys.exit(rc)
        nd = seen["nd"]
        g, rp = nd.odom.g, nd.replay
        _, _, R_fin, T_fin = host.state_pose(nd.odom.state)

        def timed(fn, n=3):
            ts, r = [], None
            for _ in range(n):
                t0 = time.perf_counter()
                r = fn()
                ts.append(time.perf_counter() - t0)
            return float(np.median(ts)), r
        t_py, r_py = timed(lambda: rp.run(R_fin, T_fin, 0.0, True))
        t_nat, r_nat = timed(lambda: rp.run_native(R_fin, T_fin, 0.0, True))
        same = r_py["result"] == r_nat["result"]
        t0 = time.perf_counter()
        rp.sweep(R_fin, T_fin)
        sweep = {"python": round(time.perf_counter() - t0, 2)}
        worker_bytes = []
        for k in ks:
            while len(rp.workers) < k - 1:
                torch.cuda.synchronize(a.device)
                free0 = torch.cuda.mem_get_info(a.device)[0]
                rp.pool(len(rp.workers) + 2)
                torch.cuda.synchronize(a.device)
                worker_bytes.append(free0 - torch.cuda.mem_get_info(a.device)[0])
            cands = [(None if n == "run" else R, None if n == "run" else T, ms / 1000.0, fz) for n, R, T, ms, fz in _plan(rp, R_fin, T_fin)]
            t0 = time.perf_counter()
            rp.run_many(cands, k, native=True)
            sweep[str(k)] = round(time.perf_counter() - t0, 2)
        best = min(ks, key=lambda k: sweep[str(k)])
        t0 = time.perf_counter()
        ref = rp.refine(R_fin, T_fin, None, best)
        ref_wall = time.perf_counter() - t0
        t0 = time.perf_counter()
        ref600 = rp.refine(R_fin, T_fin, 600, best)
        ref600_wall = time.perf_counter() - t0
        out = dict(card=card(), subframes=rp.info()["frames"], points=rp.info()["points"],
                   one_replay_s=dict(python=round(t_py, 3), native=round(t_nat, 3), bit_equal=same),
                   sweep17_s=sweep, worker_device_mb=[round(b / 1e6, 1) for b in worker_bytes], best_jobs=best,
                   refine_default=dict(jobs=best, replays=len(ref["trace"]), status=ref["status"], wall_s=round(ref_wall, 1),
                                       lag_ms=round(ref["time_lag"] * 1000, 3), axes={k: refine_verdict(t) for k, t in ref["axes"].items()}),
                   refine_600=dict(jobs=best, replays=len(ref600["trace"]), status=ref600["status"], wall_s=round(ref600_wall, 1),
                                   lag_ms=round(ref600["time_lag"] * 1000, 3), axes={k: refine_verdict(t) for k, t in ref600["axes"].items()}))
        rp.close()
        type(g).close(g)
    print(json.dumps(out))


def refine_verdict(t):
    from lidar_imu_init_b200.refine import axis_verdict
    return axis_verdict(t[1], t[2])


def _plan(rp, R_fin, T_fin):
    """the sweep's 17 candidates (name, R, T, shift_ms, frozen), as Replay.sweep makes them"""
    import numpy as np

    from lidar_imu_init_b200 import assess
    R_init = np.asarray(rp.res["R_LI"], float).reshape(3, 3)
    T_init = np.asarray(rp.res["T_LI"], float).reshape(3)
    plan = [("run", R_init, T_init, 0.0, False), ("li-init", R_init, T_init, 0.0, True)]
    plan += [(name, R, T, 0.0, True) for name, R, T in assess.candidates(R_fin, T_fin)[1:]]
    plan += [(f"lag{s:+g}", plan[2][1], plan[2][2], s, True) for s in (-assess.REPLAY_LAG_MS, assess.REPLAY_LAG_MS)]
    return plan


if __name__ == "__main__":
    main()
