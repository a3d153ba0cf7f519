"""Refine one calibration from several recordings of the same rig (DESIGN §4d, "Refining from several recordings"):

    python -m lidar_imu_init_b200.joint --config CFG --bag A --bag B [...] --out DIR [--devices 0,1,...] [--replay-jobs K]
                                        [--max-candidates N] [--param NAME=VALUE ...] [--max-map-points N] [--assess-radius R]
                                        [--assess-max-points N] [--assess-replay-max-points N] [--profile] [--quiet]

Whether an axis of the extrinsic is observable depends on the motion of a recording; several recordings with different excitation
constrain what one leaves flat. Each recording b is played as `run --config CFG --bag <b> --out DIR/rec<b>` plays it, writing the same
files, and its LIO phase is recorded for replay. Then refine.search runs once over every recording's map: a candidate (R_LI, T_LI, L),
L the total lag [s], is shared by all recordings; recording b handed over at its own total lag lambda_b and replays the candidate frozen
with the lag shift L - lambda_b. The search variable is the shift s of refine.search, L = L0 + s with L0 the mean of the lambda_b, and
recording b's shift is computed as s + (L0 - lambda_b), which is s itself for one recording. A candidate's joint score is the mean of the
recordings' as-run MMEs, summed in recording order; it is NaN when any of them is. The search starts from the lowest of every
recording's final extrinsic and LI-Init's result (`final:<b>`, `li-init:<b>`, in recording order) at s = 0.

--max-candidates counts joint candidates (default refine.MAX_REPLAYS); each costs one replay per recording. A batch of candidates is
expanded into its replays, and all of them run at once over every recording's contexts (assess.run_across). Recording b's context and
its --replay-jobs - 1 workers live on device devices[b % len(devices)] (--devices, default 0). Writes DIR/result/refinement_joint.txt
(assess.joint_report_text). Exits 1 with a message on a config, bag or library error, a recording that does not reach the hand-over or
whose replay store is truncated, the same bag given twice, or a bad --devices, --replay-jobs or --max-candidates.

--profile then replays a profile through the refined calibration along each of its seven parameters, on every recording, and fits
where each profile has its minimum, for the joint score and for each recording (profile_replays): DIR/result/profile_joint.txt.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np

from . import assess
from . import config as cfgmod
from . import refine


class JointError(RuntimeError):
    pass


def mean_lag(lags) -> float:
    """L0: the mean of the recordings' total lags [s], summed in recording order in float64 (for one recording its lag exactly)."""
    s = 0.0
    for x in lags:
        s += float(x)
    return s / len(lags)


def _mean(mmes) -> float:
    s = 0.0
    for m in mmes:
        s += float(m)
    return s / len(mmes)


def search(score_many, lags, starts, max_candidates=refine.MAX_REPLAYS) -> dict:
    """refine.search over the joint score. score_many([(b, R, T, shift_b [s])]) -> [MME of recording b's replay]; lags: lambda_b [s];
    starts: [(label, R, T)] at s = 0. Returns refine.search's dict, with on every trace row "mmes" (the recordings' MMEs, in recording
    order) and "lag" (its total lag [s]), plus "lags", "lag0" (L0), "time_lag" (the refined total lag [s]), "mmes" (the recordings'
    MMEs of the best candidate), "offsets" (L0 - lambda_b) and "axes_rec" (per recording, the axes in refine.search's form: the MME
    differences of that recording's replays at the final compass neighbours)."""
    B = len(lags)
    L0 = mean_lag(lags)
    offsets = [L0 - float(x) for x in lags]
    per = {}

    def many(cands):
        got = list(score_many([(b, R, T, s + offsets[b]) for R, T, s in cands for b in range(B)]))
        out = []
        for i, (R, T, s) in enumerate(cands):
            m = [float(x) for x in got[i * B:(i + 1) * B]]
            per[refine.key(R, T, s)] = m
            out.append(_mean(m))
        return out
    out = refine.search(lambda R, T, s: many([(R, T, s)])[0], starts[0][1], starts[0][2], 0.0, max_candidates, score_many=many,
                        starts=starts)
    for row in out["trace"]:
        row["mmes"] = per[refine.key(row["R"], row["T"], row["shift_ms"] / 1000.0)]
        row["lag"] = L0 + row["shift_ms"] / 1000.0
    best = per[refine.key(out["R"], out["T"], out["shift_s"])]
    dth, dt = out["steps"]
    mv = refine.moves(out["R"], out["T"], dth, dt)
    nan = [float("nan")] * B
    nb = {(axis, sgn): per.get(refine.key(Rm, Tm, out["shift_s"]), nan) for axis, sgn, Rm, Tm in mv}
    out["axes_rec"] = [{axis: (dth if axis.startswith("rot") else dt, nb[axis, 1.0][b] - best[b], nb[axis, -1.0][b] - best[b])
                        for axis, _, _, _ in mv[::2]} for b in range(B)]
    out.update(lags=[float(x) for x in lags], lag0=L0, time_lag=L0 + out["shift_s"], mmes=best, offsets=offsets)
    return out


def refine_replays(replays, finals, max_candidates=None, jobs: int = 1) -> dict:
    """The joint search with frozen replays of every recording as its scorer. replays: the recordings' assess.Replay, in order; finals:
    their runs' final extrinsics [(R, T)]; jobs: contexts per recording. Returns search's dict with, on every trace row, "results" (the
    recordings' as-run evaluations) and "seconds" (their replays' wall times); and "wall_s", "states" (each recording's last posterior
    state of its replay of the best candidate) and "calibs" (node.state_calib_values of those states at the refined total lag)."""
    from .node import state_calib_values
    for b, rp in enumerate(replays):
        if rp.base is None or not rp.frames:
            raise JointError(f"recording {b}: nothing to replay: the run did not reach the hand-over")
    kept = {}

    def score_many(items):
        runs = assess.run_across([(replays[b], (R, T, s, True)) for b, R, T, s in items], jobs)
        for (b, R, T, s), r in zip(items, runs):
            kept[b, refine.key(R, T, s)] = (r["result"], r["seconds"], r["states"][-1][1] if r["states"] else None)
        return [r["result"]["mme"] for r in runs]
    starts = []
    for b, (rp, (R, T)) in enumerate(zip(replays, finals)):
        starts += [(f"final:{b}", R, T), (f"li-init:{b}", rp.res["R_LI"], rp.res["T_LI"])]
    t0 = time.perf_counter()
    out = search(score_many, [rp.lag for rp in replays], starts, refine.MAX_REPLAYS if max_candidates is None else max_candidates)
    out["wall_s"] = time.perf_counter() - t0
    for row in out["trace"]:
        got = [kept[b, refine.key(row["R"], row["T"], row["shift_ms"] / 1000.0 + out["offsets"][b])] for b in range(len(replays))]
        row["results"], row["seconds"] = [g[0] for g in got], [g[1] for g in got]
    out["states"] = [kept[b, refine.key(out["R"], out["T"], out["shift_s"] + out["offsets"][b])][2] for b in range(len(replays))]
    for b, s in enumerate(out["states"]):
        if s is None:
            raise JointError(f"recording {b}: the best replay made no LIO update: nothing to take the biases and gravity from")
    out["calibs"] = [state_calib_values(s, out["time_lag"]) for s in out["states"]]
    return out


def profile_replays(replays, ref, jobs: int = 1, steps=None) -> dict:
    """profiles.profile around refine_replays' result `ref` over the joint score: every candidate (R, T, s) replayed frozen by recording
    b at the shift s + offsets[b], all of them at once (assess.run_across); the centre's joint and per-recording MMEs are ref's. Returns
    profile's dict for the joint mean with, on every row, "mmes", "results" and "seconds" (per recording, in recording order); and "recs"
    (per recording, profiles.fit_all of its own MMEs: which recording pins which parameter, at no extra replay), "wall_s", "jobs",
    "replays" (all recordings') and "status" (the refinement's)."""
    from . import profiles as pf
    B = len(replays)
    kept = []

    def score_many(cands):
        runs = assess.run_across([(replays[b], (R, T, s + ref["offsets"][b], True)) for R, T, s in cands for b in range(B)], jobs)
        kept[:] = [runs[i * B:(i + 1) * B] for i in range(len(cands))]
        return [_mean([r["result"]["mme"] for r in rs]) for rs in kept]
    n = pf.STEPS if steps is None else steps
    t0 = time.perf_counter()
    out = pf.profile(score_many, ref["R"], ref["T"], ref["shift_s"], ref["mme"], n, lag0=ref["lag0"])
    out["wall_s"] = time.perf_counter() - t0
    for row, rs in zip(out["rows"], kept):
        row["mmes"] = [float(r["result"]["mme"]) for r in rs]
        row["results"], row["seconds"] = [r["result"] for r in rs], [r["seconds"] for r in rs]
    c = out["centre"]
    c["mmes"] = [float(m) for m in ref["mmes"]]
    out["recs"] = [pf.fit_all([row["mmes"][b] for row in out["rows"]], c["mmes"][b], c["T"], c["lag_s"], n) for b in range(B)]
    out.update(jobs=jobs, replays=len(out["rows"]) * B, status=ref["status"])
    return out


# ---- the command line ------------------------------------------------------------------------------------------------------------------
def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m lidar_imu_init_b200.joint", description=__doc__.split("\n\n")[0],
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config", required=True, help="a reference config YAML, the same for every recording")
    ap.add_argument("--bag", action="append", required=True, help="a recording of the rig (repeatable, at least one)")
    ap.add_argument("--out", default=".", help="output directory: DIR/rec<b>/ per recording, DIR/result/refinement_joint.txt")
    ap.add_argument("--param", action="append", default=[], metavar="NAME=VALUE", help="a node parameter (repeatable), as for run")
    ap.add_argument("--devices", default="0", metavar="LIST", help="CUDA devices, comma-separated; recording b runs on the "
                    "(b mod n)-th (default 0)")
    ap.add_argument("--replay-jobs", metavar="K", help="contexts per recording that replay at once (default 1)")
    ap.add_argument("--max-candidates", metavar="N", help=f"joint candidates the search may score, each one replay per recording "
                    f"(default {refine.MAX_REPLAYS})")
    ap.add_argument("--max-map-points", type=int, default=6_000_000, help="capacity of each device map (default 6000000)")
    ap.add_argument("--assess-radius", type=float, default=assess.RADIUS, metavar="R",
                    help=f"neighbourhood radius of the score [m] (default {assess.RADIUS:g})")
    ap.add_argument("--assess-max-points", type=int, default=assess.MAX_POINTS, metavar="N",
                    help=f"LIO points each recording's assessment store keeps (default {assess.MAX_POINTS})")
    ap.add_argument("--assess-replay-max-points", type=int, default=assess.REPLAY_MAX_POINTS, metavar="N",
                    help=f"raw LIO-phase points each recording's replay store keeps (default {assess.REPLAY_MAX_POINTS})")
    ap.add_argument("--profile", action="store_true", help="after the refinement, replay a profile through the result along each "
                    "parameter and fit where its minimum lies, jointly and per recording: DIR/result/profile_joint.txt")
    ap.add_argument("--quiet", action="store_true", help="no progress on stderr")
    return ap.parse_args(argv)


def _positive(value, name, default) -> int:
    if value is None:
        return default
    try:
        n = int(value)
    except ValueError:
        n = 0
    if n < 1:
        raise cfgmod.ConfigError(f"{name} {value!r}: must be a positive integer")
    return n


def devices(text: str) -> list:
    """--devices as a list of distinct non-negative device indices."""
    try:
        out = [int(x) for x in text.split(",")]
    except ValueError:
        out = []
    if not out or any(d < 0 for d in out) or len(set(out)) != len(out):
        raise cfgmod.ConfigError(f"--devices {text!r}: must be distinct non-negative device indices, comma-separated")
    return out


def _free_bytes(device):
    """Free memory of a CUDA device [bytes] after a synchronise, or None without a CUDA device (a CPU build of the kernels)."""
    try:
        import torch
        if not torch.cuda.is_available():
            return None
        torch.cuda.synchronize(device)
        return torch.cuda.mem_get_info(device)[0]
    except Exception:
        return None


def main(argv=None, on_node=None) -> int:
    """The command line; on_node(node), when given, is called with each recording's Node before its bag is played."""
    from . import capi, host, run
    from .node import Log
    args = parse_args(argv)
    log = Log(quiet=args.quiet)
    nodes = []
    try:
        jobs = _positive(args.replay_jobs, "--replay-jobs", 1)
        max_candidates = _positive(args.max_candidates, "--max-candidates", refine.MAX_REPLAYS)
        devs = devices(args.devices)
        seen = {}
        for b, bag in enumerate(args.bag):
            real = os.path.realpath(bag)
            if real in seen:
                raise cfgmod.ConfigError(f"--bag {bag!r} is given twice (recordings {seen[real]} and {b})")
            seen[real] = b
        for b, bag in enumerate(args.bag):
            dev = devs[b % len(devs)]
            argv_b = ["--config", args.config, "--bag", bag, "--out", os.path.join(args.out, f"rec{b}"), "--device", str(dev),
                      "--max-map-points", str(args.max_map_points), "--assess-radius", repr(args.assess_radius),
                      "--assess-max-points", str(args.assess_max_points), "--assess-replay-max-points", str(args.assess_replay_max_points),
                      "--refine"] + [f"--param={p}" for p in args.param]
            free0 = _free_bytes(dev)
            try:
                nd, wall = run.play(run.parse_args(argv_b), log, on_node)
                nodes.append(nd)
                rp = nd.replay
                if rp.base is None or not rp.frames:
                    raise JointError(f"recording {b} ({bag}): nothing to replay: the run did not reach the hand-over")
                if rp.info()["skipped"]:
                    raise JointError(f"recording {b} ({bag}): the replay store is truncated ({rp.info()['skipped']} sub-frames skipped): "
                                     "raise --assess-replay-max-points")
                rp.pool(jobs)
            except capi.LiInitError as e:
                raise JointError(f"recording {b} ({bag}) does not fit on device {dev} with {jobs} replay job"
                                 f"{'s' if jobs > 1 else ''}: {e}") from None
            free1 = _free_bytes(dev)
            used = "not measured" if free0 is None or free1 is None else f"{(free0 - free1) / 1e6:.1f} MB"
            log.info(f"recording {b} ({bag}): device {dev}, {rp.info()['frames']} sub-frames, lag {rp.lag * 1000.0:.3f} ms, device "
                     f"memory {used} (the context's reserves and {jobs - 1} worker{'s' if jobs != 2 else ''}), {wall:.1f} s")
        finals = [host.state_pose(nd.odom.state)[2:] for nd in nodes]
        ref = refine_replays([nd.replay for nd in nodes], finals, max_candidates, jobs)
        path = os.path.join(args.out, "result", "refinement_joint.txt")
        os.makedirs(os.path.dirname(path), exist_ok=True)
        recs = [dict(bag=bag, subframes=nd.replay.info()["frames"], skipped=nd.replay.info()["skipped"], lag=nd.replay.lag,
                     R_init=nd.replay.res["R_LI"], T_init=nd.replay.res["T_LI"], R_final=R, T_final=T)
                for bag, nd, (R, T) in zip(args.bag, nodes, finals)]
        with open(path, "w") as f:
            f.write(assess.joint_report_text(recs, ref, args.assess_radius, nodes[0].assess.min_neighbors))
        log.info(summary(path, ref, len(nodes), jobs))
        if args.profile:
            prof = profile_replays([nd.replay for nd in nodes], ref, jobs)
            path = os.path.join(args.out, "result", "profile_joint.txt")
            with open(path, "w") as f:
                f.write(assess.profile_report_text(prof))
            log.info(run.profile_summary(path, prof, jobs))
        return 0
    except run.errors() + (JointError,) as e:
        sys.stderr.write(f"error: {e}\n")
        return 1
    finally:
        for nd in nodes:
            nd.replay.close()
            nd.odom.g.close()


def summary(path: str, ref: dict, recordings: int, jobs: int) -> str:
    s = ref["trace"][[r["stage"] for r in ref["trace"]].index(ref["start"])]
    c = np.clip((np.trace(ref["R"] @ s["R"].T) - 1.0) / 2.0, -1.0, 1.0)
    return (f"joint refinement written to {path}: {len(ref['trace'])} candidates, {len(ref['trace']) * recordings} replays of "
            f"{recordings} recordings in {ref['wall_s']:.1f} s ({ref['status']}, {jobs} replay job{'s' if jobs > 1 else ''} each); "
            f"lag {ref['lag0'] * 1000.0:.3f} -> {ref['time_lag'] * 1000.0:.3f} ms; from {ref['start']}: rotation "
            f"{np.degrees(np.arccos(c)):.4f} deg, translation {np.linalg.norm(ref['T'] - s['T']) * 1000.0:.2f} mm; joint MME "
            f"{s['mme']:.6f} -> {ref['mme']:.6f}")


if __name__ == "__main__":
    sys.exit(main())
