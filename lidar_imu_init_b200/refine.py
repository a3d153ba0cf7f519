"""Refining a calibration where the replayed map is sharpest (DESIGN §4d, "Refining by replay").

search() looks for the extrinsic (R_LI, T_LI) and the lag shift whose map has the lowest MME, over a scoring callable score(R, T,
shift_s) -> MME: assess.Replay.run with the candidate held fixed in production (assess.Replay.refine), a synthetic function in the
tests. It starts from the lower-scoring of the run's final extrinsic and LI-Init's, both at shift0, then

1. lag: brackets the minimum with LAG_STEP_MS steps downhill from shift0 (no further than LAG_CAP_MS) and narrows the bracket by
   golden-section search to LAG_TOL_MS;
2. extrinsic: a compass search over the 12 moves of the sweep (R <- Exp(+-dtheta e_a) R, T <- T +- dt e_a), starting at the sweep's
   steps: each round moves to the best strictly lower move, or halves both steps when none is lower, until both steps are at or below
   DTHETA_MIN_DEG / DT_MIN_M;
3. lag: golden-section search again, LAG_LOCAL_MS around the lag of stage 1, at the refined extrinsic; when that moves the lag, one more
   compass search at the final steps, so that the end condition holds at the final lag too.

Every evaluation is cached by the exact bytes of (R, T, shift_s): a revisited candidate is not scored again, and every score is one row
of the trace. The candidate kept at every point is the lowest MME so far, the first of equals, so an axis along which the MME does not
change keeps its value. The search stops early when max_replays scores are spent.

With score_many(candidates) -> [MME], the candidates the search needs together are scored as one batch: the start pair, stage 1's
first pair, each golden-section opening pair and each compass round (at most 12). A batch drops cached candidates and repeated keys and
is cut at the remaining budget; its rows are appended, and the best row updated, in the order the one-at-a-time search scores them.
With a deterministic scorer the trace, the result, the status and the axes are those of the one-at-a-time search at the same budget.

With starts=[(label, R, T), ...] the search starts from the lowest of those, scored as one batch at shift0, instead of the (final,
LI-Init) pair: joint.py starts from every recording's pair.
"""
from __future__ import annotations

import math

import numpy as np

from .assess import AXES, DT_M, DTHETA_DEG, rot_exp

LAG_STEP_MS = 5.0       # stage 1 bracket step [ms]
LAG_CAP_MS = 50.0       # the lag shift stays within +-LAG_CAP_MS of shift0 [ms]
LAG_TOL_MS = 0.5        # golden-section bracket width at which a lag search stops [ms]
LAG_LOCAL_MS = 2.0      # stage 3 searches +-LAG_LOCAL_MS around the lag of stage 1 [ms]
DTHETA_MIN_DEG = 0.05   # the compass search stops when its steps are at or below these
DT_MIN_M = 0.002
MAX_REPLAYS = 120
_GOLD = (math.sqrt(5.0) - 1.0) / 2.0


class _Budget(Exception):
    pass


def key(R, T, shift_s) -> bytes:
    """The cache key of a candidate: the exact bytes of R (3x3), T (3) and the lag shift [s], as float64."""
    return (np.ascontiguousarray(R, np.float64).tobytes() + np.ascontiguousarray(T, np.float64).tobytes()
            + np.float64(shift_s).tobytes())


def _lower(a: float, b: float) -> bool:
    """a strictly lower than b; a NaN MME (no valid query) is never lower, and anything is lower than NaN."""
    return (a == a) and (b != b or a < b)


def moves(R, T, dtheta_deg, dt) -> list:
    """[(axis, sign, R, T)] of the 12 compass moves around (R, T), in the sweep's order: rot_x+, rot_x-, ..., trans_z-."""
    out = []
    for a, ax in enumerate(AXES):
        for sgn in (1.0, -1.0):
            out.append((f"rot_{ax}", sgn, rot_exp(sgn * math.radians(dtheta_deg) * np.eye(3)[a]) @ R, T))
    for a, ax in enumerate(AXES):
        for sgn in (1.0, -1.0):
            out.append((f"trans_{ax}", sgn, R, T + sgn * dt * np.eye(3)[a]))
    return out


def search(score, R0, T0, shift0=0.0, max_replays=MAX_REPLAYS, R_init=None, T_init=None, score_many=None, starts=None) -> dict:
    """The refinement; R0 / T0: the run's final extrinsic, R_init / T_init (optional): LI-Init's; shift0: the lag shift both start at
    [s]; score_many (optional): scores a list of (R, T, shift_s) at once, for the search's batches; starts (optional): [(label, R, T)]
    scored as one batch at shift0 in place of the (final, li-init) pair, R0 / T0 and R_init / T_init then unused. Returns {"R", "T",
    "shift_ms", "shift_s", "mme": the best candidate; "start": "final" or "li-init" (the label of a start); "status": "converged" or
    "budget"; "at_edge": stage 1's minimum lay at the +-LAG_CAP_MS cap; "trace": [{"stage", "R", "T", "shift_ms", "mme"}] in evaluation
    order; "best": the index of the best row; "steps": the compass steps (dtheta [deg], dt [m]) it ended with; "axes": {"rot_x": (step,
    MME(+step) - MME, MME(-step) - MME), ...} around the best candidate, NaN where that neighbour was not scored}."""
    if isinstance(max_replays, bool) or int(max_replays) != max_replays or max_replays < 1:
        raise ValueError(f"max_replays {max_replays!r}: must be a positive integer")
    trace, cache = [], {}
    st = dict(best=None, steps=(DTHETA_DEG, DT_M), at_edge=False, start=None)

    def f(stage, R, T, ms):
        return fmany([(stage, R, T, ms)])[0]

    def fmany(items):
        """[MME] of [(stage, R, T, shift_ms)], scored as f would one after the other: the uncached keys, each once, up to the budget,
        in one call of score_many"""
        items = [(stage, np.array(R, np.float64).reshape(3, 3), np.array(T, np.float64).reshape(3), ms) for stage, R, T, ms in items]
        keys = [key(R, T, ms / 1000.0) for _, R, T, ms in items]
        todo = list(dict.fromkeys(k for k in keys if k not in cache))[:max(max_replays - len(trace), 0)]
        if todo:
            at = {k: i for i, k in reversed(list(enumerate(keys)))}
            cands = [(items[at[k]][1], items[at[k]][2], items[at[k]][3] / 1000.0) for k in todo]
            got = score_many(cands) if score_many is not None and len(cands) > 1 else [score(*c) for c in cands]
            fresh = dict(zip(todo, (float(m) for m in got)))
        else:
            fresh = {}
        out = []
        for (stage, R, T, ms), k in zip(items, keys):
            if k not in cache:
                if k not in fresh:
                    raise _Budget
                m = cache[k] = fresh[k]
                trace.append(dict(stage=stage, R=R, T=T, shift_ms=ms, mme=m))
                if st["best"] is None or _lower(m, trace[st["best"]]["mme"]):
                    st["best"] = len(trace) - 1
            out.append(cache[k])
        return out

    def centre():
        b = trace[st["best"]]
        return b["R"], b["T"], b["shift_ms"]

    lo, hi = shift0 * 1000.0 - LAG_CAP_MS, shift0 * 1000.0 + LAG_CAP_MS

    def golden(stage, a, b):
        """golden-section search of the lag on [a, b] at the best extrinsic"""
        R, T, _ = centre()
        x1, x2 = b - _GOLD * (b - a), a + _GOLD * (b - a)
        f1, f2 = fmany([(stage, R, T, x1), (stage, R, T, x2)])
        while True:
            if not _lower(f2, f1):
                b, x2, f2 = x2, x1, f1
                if b - a <= LAG_TOL_MS:
                    return
                x1 = b - _GOLD * (b - a)
                f1 = f(stage, R, T, x1)
            else:
                a, x1, f1 = x1, x2, f2
                if b - a <= LAG_TOL_MS:
                    return
                x2 = a + _GOLD * (b - a)
                f2 = f(stage, R, T, x2)

    def compass(stage, dth, dt):
        while True:
            st["steps"] = (dth, dt)
            before = st["best"]
            R, T, ms = centre()
            fmany([(stage, Rm, Tm, ms) for _, _, Rm, Tm in moves(R, T, dth, dt)])
            if st["best"] != before:
                continue
            if dth <= DTHETA_MIN_DEG and dt <= DT_MIN_M:
                return
            dth, dt = dth / 2.0, dt / 2.0

    status = "converged"
    try:
        c = shift0 * 1000.0
        if starts is None:
            starts = [("final", R0, T0)] + ([("li-init", R_init, T_init)] if R_init is not None else [])
        st["start"] = starts[0][0]      # (max_replays >= 1: the first start is always scored)
        fmany([(label, R, T, c) for label, R, T in starts])
        st["start"] = trace[st["best"]]["stage"]
        # stage 1: bracket downhill in LAG_STEP_MS steps, then golden-section search
        R, T, _ = centre()
        fc = trace[st["best"]]["mme"]
        fp, fm = fmany([("lag", R, T, c + LAG_STEP_MS), ("lag", R, T, c - LAG_STEP_MS)])
        if not (_lower(fp, fc) or _lower(fm, fc)):
            golden("lag", c - LAG_STEP_MS, c + LAG_STEP_MS)
        else:
            d = 1.0 if not _lower(fm, fp) else -1.0
            k, fk = 1, fp if d > 0 else fm
            while True:
                if k * LAG_STEP_MS >= LAG_CAP_MS:
                    st["at_edge"] = True
                    break
                fn = f("lag", R, T, c + d * (k + 1) * LAG_STEP_MS)
                if not _lower(fn, fk):
                    a, b = sorted((c + d * (k - 1) * LAG_STEP_MS, c + d * (k + 1) * LAG_STEP_MS))
                    golden("lag", a, b)
                    break
                k, fk = k + 1, fn
        lag1 = centre()[2]
        # stage 2: the extrinsic at that lag
        compass("ext", DTHETA_DEG, DT_M)
        # stage 3: the lag again, near stage 1's, at the refined extrinsic; the extrinsic again if that moved the lag
        before = st["best"]
        golden("lag2", max(lo, lag1 - LAG_LOCAL_MS), min(hi, lag1 + LAG_LOCAL_MS))
        if st["best"] != before:
            compass("ext2", *st["steps"])
    except _Budget:
        status = "budget"

    best = trace[st["best"]]
    R, T, ms = centre()
    dth, dt = st["steps"]
    nb = {}
    for axis, sgn, Rm, Tm in moves(R, T, dth, dt):
        nb[axis, sgn] = cache.get(key(Rm, Tm, ms / 1000.0), math.nan) - best["mme"]
    axes = {axis: (dth if axis.startswith("rot") else dt, nb[axis, 1.0], nb[axis, -1.0]) for axis, _, _, _ in moves(R, T, dth, dt)[::2]}
    return dict(R=R, T=T, shift_ms=ms, shift_s=ms / 1000.0, mme=best["mme"], start=st["start"], status=status, at_edge=st["at_edge"],
                trace=trace, best=st["best"], steps=(dth, dt), axes=axes)


def axis_verdict(d_plus: float, d_minus: float) -> str:
    """`constrained` when both neighbours score a higher MME than the centre, `flat` when one does not, `unmeasured` when one was not
    scored (the budget ran out first)."""
    if d_plus != d_plus or d_minus != d_minus:
        return "unmeasured"
    return "constrained" if d_plus > 0 and d_minus > 0 else "flat"
