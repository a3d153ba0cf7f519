"""Time the profiles of a refined calibration on the synthetic Livox scenario (tests/test_gpu_profile.py).

    python tools/profile_bench.py [--seconds 60] [--max-replays 20] [--refine-jobs 8] [--jobs 1,4,8] [--steps 6] [--device N]

Plays the scenario as `run --refine` does (the bag and the outputs go to a temporary directory), refines at the given small budget, then
times Replay.profile around the result at each job count with a host clock (every replay ends in a device synchronise). Prints one
JSON line with the card's name and power limit (read in the same process), the refinement, the profile's wall time and median replay
time per job count, whether every job count gave the same rows bit for bit, and each parameter's verdict, minimum and interval beside
the simulated truth.
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
    ap.add_argument("--max-replays", type=int, default=20)
    ap.add_argument("--refine-jobs", type=int, default=8)
    ap.add_argument("--jobs", default="1,4,8")
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import numpy as np

    import test_bag_node as tb
    import test_gpu_profile as tg
    from lidar_imu_init_b200 import host, profiles, run
    from lidar_imu_init_b200.node import Log
    name = card()
    with tempfile.TemporaryDirectory() as tmp:
        ev, path = tb.livox_events(a.seconds, 20_000)
        bag = os.path.join(tmp, "sim.bag")
        tb.write_event_bag(bag, ev, chunk_msgs=300)
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        nd, _ = run.play(run.parse_args(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, "out"),
                                         "--device", str(a.device), "--max-map-points", "3000000", "--refine"]), Log(quiet=True))
        rp = nd.replay
        try:
            subframes = rp.info()["frames"]
            _, _, R_fin, T_fin = host.state_pose(nd.odom.state)
            ref = rp.refine(R_fin, T_fin, a.max_replays, jobs=a.refine_jobs)
            profs = {}
            for j in (int(x) for x in a.jobs.split(",")):
                profs[j] = rp.profile(ref, j, a.steps)
        finally:
            rp.close()
            nd.odom.g.close()
    first = next(iter(profs.values()))
    rows = {j: [np.float64(r["mme"]).tobytes() for r in p["rows"]] for j, p in profs.items()}
    tr = tg.truth(path.S, first["centre"])
    out = dict(card=name, subframes=subframes,
               refine=dict(replays=len(ref["trace"]), status=ref["status"], jobs=a.refine_jobs, lag_ms=round(ref["time_lag"] * 1000, 3),
                           mme=round(ref["mme"], 6)),
               profile=dict(replays=first["replays"], steps=first["steps"],
                            wall_s={j: round(p["wall_s"], 2) for j, p in profs.items()},
                            replay_median_s={j: round(sorted(r["seconds"] for r in p["rows"])[len(p["rows"]) // 2], 3) for j, p in profs.items()},
                            same_rows=all(r == rows[next(iter(rows))] for r in rows.values())),
               fits={p: dict(verdict=f["verdict"], min=round(f["u_phys"], 5), lo=round(f["lo_phys"], 5), hi=round(f["hi_phys"], 5),
                             s=float("%.3g" % f["s"]), lower_k=f["lower_k"], off_lowest=profiles.off_lowest(f), truth=round(float(tr[p]), 5)) for p, f in first["fits"].items()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
