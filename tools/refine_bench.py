"""Time the refinement by LIO replay on the synthetic Livox scenario (tests/test_gpu_bag.py).

    python tools/refine_bench.py [--seconds 60] [--max-replays 120] [--device N]

Runs the scenario with `run --assess` and a Replay attached (the bag and the outputs go to a temporary directory), then times, with a host
clock around calls that end in a device synchronise, the whole Replay.refine from the run's final extrinsic. Prints one JSON line with
the card's name and power limit, the replays used, the wall time, the median time of one replay, and the refined lag and extrinsic with
their errors against the simulated truth (and those of LI-Init's and the final extrinsic).
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
    ap.add_argument("--max-replays", type=int, default=None)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import pathlib

    import numpy as np

    import test_bag_node as tb
    from lidar_imu_init_b200 import assess, host, run
    with tempfile.TemporaryDirectory() as tmp:
        ev, path = tb.livox_events(a.seconds, 20_000)
        S = path.S
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
        _, _, R_fin, T_fin = host.state_pose(nd.odom.state)
        t0 = time.perf_counter()
        ref = rp.refine(R_fin, T_fin, a.max_replays)
        wall = time.perf_counter() - t0
        name = card()

        def err(R, T):
            c = np.clip((np.trace(np.asarray(R) @ np.asarray(S["R_LI"]).T) - 1.0) / 2.0, -1.0, 1.0)
            return dict(rot_deg=round(float(np.degrees(np.arccos(c))), 4), trans_mm=round(float(np.linalg.norm(np.asarray(T) - S["T_LI"])) * 1000, 2))
        times = sorted(r["seconds"] for r in ref["trace"])
        stages = {}
        for r in ref["trace"]:
            stages[r["stage"]] = stages.get(r["stage"], 0) + 1
        v = ref["calib"]
        out = dict(card=name, subframes=rp.info()["frames"], replays=len(ref["trace"]), stages=stages, status=ref["status"], start=ref["start"],
                   at_edge=ref["at_edge"], wall_s=round(wall, 1), replay_median_s=round(times[len(times) // 2], 3),
                   replay_min_max_s=[round(times[0], 3), round(times[-1], 3)],
                   lag_ms=dict(handover=round(ref["lag0"] * 1000, 3), refined=round(ref["time_lag"] * 1000, 3), simulated=round(S["t_off"] * 1000, 3),
                               error=round((ref["time_lag"] - S["t_off"]) * 1000, 3)),
                   mme=dict(start=round(ref["trace"][[r["stage"] for r in ref["trace"]].index(ref["start"])]["mme"], 6), refined=round(ref["mme"], 6)),
                   refined=dict(euler_deg=[round(float(x), 4) for x in v["euler_deg"]], T_LI=[round(float(x), 5) for x in v["T_LI"]]),
                   error=dict(refined=err(ref["R"], ref["T"]), li_init=err(rp.res["R_LI"], rp.res["T_LI"]), final=err(R_fin, T_fin)),
                   axes={k: [round(x, 9) for x in t] for k, t in ref["axes"].items()})
        type(g).close(g)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
