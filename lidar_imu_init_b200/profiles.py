"""How precisely a recording determines a refined calibration (DESIGN §4d, "Profiles of the result").

profile() replays an MME profile through a centre candidate (R_LI, T_LI, lag shift) along each of its seven parameters, rot_x rot_y
rot_z trans_x trans_y trans_z lag, one at a time, and fits where each profile has its minimum. Every candidate is made from the centre
by one operation, never chained: for k = -n..n, k != 0 (n = steps),

    rotation     R' = Exp(k h_rot e_a) R     (about the IMU axes, as refine.moves turns)
    translation  T' = T + k h_trans e_a
    lag          shift' = shift + k h_lag

All 7 * 2n candidates go to one call of score_many, in parameter order and then ascending k. The centre is not replayed again: replays
are deterministic, so its score is the refinement's best row. Per parameter, y = c0 + c1 u + c2 u^2 is fitted by least squares over the
2n + 1 points, u in steps, centre included, and

    s^2 = RSS / (2n - 2),  C = s^2 (X^T X)^-1,  u* = -c1 / (2 c2),
    se(u*) by the delta method (gradient (0, -1/(2 c2), c1/(2 c2^2))),  interval u* -+ t_{0.975, 2n-2} se.

What the interval means: where this recording's MME profile has its minimum along that parameter, given how rough the profile is at
that scale. It is not a bound on the error against the truth: the measure itself can be biased (DESIGN §4d found the lag 1.46 ms from
the simulated one). It is conditional: the other six parameters stay at the centre. A profile the quadratic does not fit, such as the
V-shaped lag profile, has a larger s and a wider interval, but its vertex can also move away from where the profile is lowest: an
asymmetric V puts u* on the side of the shallower slope, and the interval can then miss the profile's minimum altogether. The points
say where the minimum can be: for a convex profile it lies within one step of the lowest point, lower_k (0: the centre). A fit whose
u* is a step or more from lower_k (off_lowest(); for instance the interval excludes the centre while no point scores below it) has
placed the minimum where the profile's own points say it is not, and its interval is not to be read at face value.

Verdict per parameter, the first that holds: `unmeasured` (a score is NaN), `flat` (c2 <= t sqrt(C[2,2]): no curvature distinguishable
from zero over the range), `edge` (|u*| > n: the minimum lies outside the profile), `pinned`.
"""
from __future__ import annotations

import math

import numpy as np

from .assess import AXES, rot_exp

PARAMS = ("rot_x", "rot_y", "rot_z", "trans_x", "trans_y", "trans_z", "lag")
STEPS = 6               # n: offsets k = -n..n steps
MIN_STEPS, MAX_STEPS = 2, 16
H_ROT_DEG = 0.1         # rotation step [deg]
H_TRANS_M = 0.005       # translation step [m]
H_LAG_MS = 0.5          # lag step [ms]
# t_{0.975, dof}, dof = 2n - 2 for n = MIN_STEPS..MAX_STEPS (tests/test_profiles.py checks it against scipy.stats.t.ppf)
T975 = {2: 4.302652729749462, 4: 2.7764451051977934, 6: 2.4469118511449786, 8: 2.306004135204166, 10: 2.228138851986274,
        12: 2.1788128296672284, 14: 2.144786687917804, 16: 2.1199052992212546, 18: 2.1009220402410382, 20: 2.085963447265864,
        22: 2.0738730679040254, 24: 2.0638985616280245, 26: 2.0555294386428735, 28: 2.0484071417952454, 30: 2.0422724563012378}
UNITS = {"rot": "deg", "trans": "m", "lag": "ms"}


def check_steps(steps) -> int:
    if isinstance(steps, bool) or int(steps) != steps or not MIN_STEPS <= steps <= MAX_STEPS:
        raise ValueError(f"profile steps {steps!r}: must be an integer from {MIN_STEPS} to {MAX_STEPS}")
    return int(steps)


def offsets(steps) -> list:
    """k = -n..n without 0, ascending."""
    return [k for k in range(-steps, steps + 1) if k != 0]


def candidates(R, T, shift_s, steps=STEPS) -> list:
    """[(param, k, R', T', shift')]: the 7 * 2n profile candidates around (R, T, shift_s), in parameter order and then ascending k."""
    R, T = np.asarray(R, np.float64).reshape(3, 3), np.asarray(T, np.float64).reshape(3)
    out = []
    for a, ax in enumerate(AXES):
        out += [(f"rot_{ax}", k, rot_exp(k * math.radians(H_ROT_DEG) * np.eye(3)[a]) @ R, T.copy(), shift_s) for k in offsets(steps)]
    for a, ax in enumerate(AXES):
        out += [(f"trans_{ax}", k, R.copy(), T + k * H_TRANS_M * np.eye(3)[a], shift_s) for k in offsets(steps)]
    out += [("lag", k, R.copy(), T.copy(), shift_s + k * (H_LAG_MS / 1000.0)) for k in offsets(steps)]
    return out


def physical(param: str, u, T, lag_s):
    """u [steps] of a parameter in its unit: a rotation offset about the IMU axis from the centre [deg]; an absolute T[a] [m]; the
    absolute total lag [ms]. T: the centre's translation; lag_s: the centre's total lag [s]."""
    if param.startswith("rot"):
        return u * H_ROT_DEG
    if param.startswith("trans"):
        return float(T[AXES.index(param[-1])]) + u * H_TRANS_M
    return lag_s * 1000.0 + u * H_LAG_MS


def fit(ys, centre_mme, steps=STEPS) -> dict:
    """The quadratic fit of one parameter's profile: ys, the 2n scores at ascending k != 0; centre_mme, the score at k = 0. Returns
    {"verdict", "c": (c0, c1, c2), "s", "u", "se", "lo", "hi" (u* and its interval [steps]), "centre_inside", "lower_k", "lower_dmme"
    (the lowest point of the profile and its MME minus the centre's; 0 and 0.0 when no point scores strictly lower than the centre)}.
    The scores are fitted as differences to the centre's, which gives the same fit and keeps a constant profile exactly flat."""
    n = check_steps(steps)
    ys = [float(y) for y in ys]
    if len(ys) != 2 * n:
        raise ValueError(f"{len(ys)} profile scores for {n} steps: want {2 * n}")
    u = np.arange(-n, n + 1, dtype=np.float64)
    y = np.array(ys[:n] + [float(centre_mme)] + ys[n:], np.float64)
    lower_k, lower_d = 0, 0.0
    for k, v in zip(offsets(n), ys):
        if v - centre_mme < lower_d:
            lower_k, lower_d = k, v - centre_mme
    out = dict(lower_k=lower_k, lower_dmme=lower_d)
    nan = math.nan
    if np.isnan(y).any():
        return dict(out, verdict="unmeasured", c=(nan, nan, nan), s=nan, u=nan, se=nan, lo=nan, hi=nan, centre_inside=False)
    X = np.stack([np.ones_like(u), u, u * u], axis=1)
    XtX_inv = np.linalg.inv(X.T @ X)
    d = y - float(centre_mme)
    c = XtX_inv @ (X.T @ d)
    dof = 2 * n - 2
    rss = float(np.sum((d - X @ c) ** 2))
    s2 = rss / dof
    C = s2 * XtX_inv
    c0, c1, c2 = float(c[0]) + float(centre_mme), float(c[1]), float(c[2])
    t = T975[dof]
    with np.errstate(divide="ignore", invalid="ignore"):
        us = np.float64(-c1) / np.float64(2.0 * c2)
        g = np.array([0.0, np.float64(-1.0) / np.float64(2.0 * c2), np.float64(c1) / np.float64(2.0 * c2 * c2)])
        se = float(np.sqrt(g @ C @ g))
    us = float(us)
    lo, hi = us - t * se, us + t * se
    if c2 <= t * math.sqrt(C[2, 2]):
        verdict = "flat"
    elif abs(us) > n:
        verdict = "edge"
    else:
        verdict = "pinned"
    return dict(out, verdict=verdict, c=(c0, c1, c2), s=math.sqrt(s2), u=us, se=se, lo=lo, hi=hi, centre_inside=bool(lo <= 0.0 <= hi))


def off_lowest(f: dict) -> bool:
    """A fit whose minimum u* lies a step or more from the lowest profile point (lower_k; 0: the centre). The points bracket a convex
    profile's minimum within one step of its lowest point, so such a u* is the parabola's misfit, not where the profile is lowest."""
    return bool(abs(f["u"] - f["lower_k"]) >= 1.0)


def fit_all(mmes, centre_mme, T, lag_s, steps=STEPS) -> dict:
    """{param: fit(...) with "u_phys", "lo_phys", "hi_phys" (physical())} from the 7 * 2n scores in candidates' order."""
    n = check_steps(steps)
    out = {}
    for i, p in enumerate(PARAMS):
        f = fit(mmes[i * 2 * n:(i + 1) * 2 * n], centre_mme, n)
        f.update(u_phys=physical(p, f["u"], T, lag_s), lo_phys=physical(p, f["lo"], T, lag_s), hi_phys=physical(p, f["hi"], T, lag_s))
        out[p] = f
    return out


def profile(score_many, R, T, shift_s, centre_mme, steps=STEPS, lag0=0.0) -> dict:
    """The profiles around the centre (R, T, shift_s [s]) whose score is centre_mme. score_many([(R, T, shift_s)]) -> [MME] is called
    once, with every candidate; lag0: the total lag at shift 0 [s] (the lag is reported as lag0 + shift). Returns {"steps", "centre":
    {"R", "T", "shift_s", "lag_s", "mme"}, "rows": [{"param", "k", "offset" (physical()), "R", "T", "shift_s", "mme"}] in
    candidates' order, "fits": {param: fit_all's dict}}."""
    n = check_steps(steps)
    R, T = np.asarray(R, np.float64).reshape(3, 3), np.asarray(T, np.float64).reshape(3)
    cands = candidates(R, T, shift_s, n)
    got = [float(m) for m in score_many([(Rc, Tc, s) for _, _, Rc, Tc, s in cands])]
    if len(got) != len(cands):
        raise ValueError(f"score_many returned {len(got)} scores for {len(cands)} candidates")
    lag_s = float(lag0) + float(shift_s)
    rows = [dict(param=p, k=k, offset=physical(p, float(k), T, lag_s), R=Rc, T=Tc, shift_s=s, mme=m)
            for (p, k, Rc, Tc, s), m in zip(cands, got)]
    return dict(steps=n, centre=dict(R=R, T=T, shift_s=shift_s, lag_s=lag_s, mme=float(centre_mme)), rows=rows,
                fits=fit_all(got, centre_mme, T, lag_s, n))
