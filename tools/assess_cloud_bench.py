"""Time the assessment cloud (liinit_assess_cloud) on the stored LIO phase of the synthetic Livox scenario (tools/assess_bench.py).

    python tools/assess_cloud_bench.py [--seconds 60] [--repeat 5] [--device N]

Replays the scenario with `run --assess` (the bag and the outputs go to a temporary directory), then times on the stored scans, with CUDA
events on the context's stream around each call and a synchronise, after a warm-up call of each kind:
  - one evaluation of the as-run extrinsic (the automatic stride), for comparison;
  - the cloud's device work alone (totals only, no records) at leaf 0;
  - the whole binding call at leaf 0 and at leaf 0.1 m: a size query, the device work and the records' download.
Prints one JSON line with the card's name and power limit, read in the same call.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch

    import test_bag_node as tb
    from assess_bench import card
    from lidar_imu_init_b200 import capi, run
    with tempfile.TemporaryDirectory() as tmp:
        import pathlib
        ev, _ = tb.livox_events(a.seconds, 20_000)
        bag = os.path.join(tmp, "sim.bag")
        tb.write_event_bag(bag, ev, chunk_msgs=300)
        tb.sim_config(pathlib.Path(tmp), online_refine_time=10.0)
        seen = {}

        def on_node(nd):
            seen["g"] = nd.odom.g
            nd.odom.g.close = lambda: None
        rc = run.main(["--config", os.path.join(tmp, "sim.yaml"), "--bag", bag, "--out", os.path.join(tmp, "out"), "--device", str(a.device),
                       "--quiet", "--assess"], on_node=on_node)
        if rc != 0:
            sys.exit(rc)
        g = seen["g"]
        torch.cuda.set_device(a.device)
        stream = torch.cuda.ExternalStream(g.stream(), device=torch.device("cuda", a.device))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed(fn):
            fn()                                                  # warm-up
            ts, out = [], None
            for _ in range(a.repeat):
                e0.record(stream)
                out = fn()
                e1.record(stream)
                torch.cuda.synchronize(a.device)
                ts.append(e0.elapsed_time(e1))
            return sorted(ts), out

        def device_only():
            P = capi.AssessParams(0.3, 10, 1, 1, 0)
            n, tot = C.c_longlong(0), capi.AssessResult()
            g._ck(g.L.liinit_assess_cloud(g.h, C.byref(P), None, None, 0.0, None, 0, C.byref(n), C.byref(tot)))
            return tot
        t_eval, res = timed(lambda: g.assess_evaluate(radius=0.3, min_neighbors=10, as_run=True))
        t_dev, tot = timed(device_only)
        t_rec0, (rec0, _) = timed(lambda: g.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.0, as_run=True))
        t_rec1, (rec1, _) = timed(lambda: g.assess_cloud(radius=0.3, min_neighbors=10, leaf=0.1, as_run=True))
        med = lambda ts: round(ts[len(ts) // 2], 2)   # noqa: E731
        out = dict(card=card(), points=tot.points, scans=tot.scans, valid=tot.valid, mme_full=round(tot.mme, 6), evaluate_stride=res["stride"],
                   mme_strided=round(res["mme"], 6), batches=-(-tot.points // capi.ASSESS_MAX_QUERIES), evaluate_ms=med(t_eval),
                   cloud_device_ms=med(t_dev), cloud_leaf0_ms=med(t_rec0), cloud_leaf0_records=len(rec0), cloud_leaf01_ms=med(t_rec1),
                   cloud_leaf01_records=len(rec1), all_ms=dict(evaluate=[round(t, 2) for t in t_eval], device=[round(t, 2) for t in t_dev],
                                                               leaf0=[round(t, 2) for t in t_rec0], leaf01=[round(t, 2) for t in t_rec1]))
        type(g).close(g)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
