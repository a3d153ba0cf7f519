"""How sharp a map a calibration builds (DESIGN §4d): the LIO scans of a run are stored on the device (LiInitGpu.assess_append after
every LIO update but the switch scan), and each candidate extrinsic is scored by the mean map entropy (MME) and mean plane variance
(MPV) of the map it builds (LiInitGpu.assess_evaluate).

The sweep scores 14 candidates: the run as it went (each scan with its own extrinsic), the final extrinsic, and the final extrinsic
rotated by +-DTHETA_DEG about each IMU axis (R = Exp(+-dtheta e_a) R_final) and shifted by +-DT_M along it. An axis whose two
perturbations both score a higher MME than the final extrinsic is reported `constrained`, any other `flat`: the recording did not pin
that axis down as far as this measure can tell. This is a report, not a verdict on the calibration.

write_cloud shows where the as-run map is blurred: every stored point scored (LiInitGpu.assess_cloud), thinned to leaves on the device,
as a PCD that a viewer colours by entropy.

A timed assessment (Assessment(timed=True)) also keeps each LIO scan's raw cloud, IMU pose table and propagated state, so that every
evaluation re-undistorts the scans for its candidate (LiInitGpu.assess_evaluate_timed). sweep_time scores the 14 candidates that way
and a lag profile: the final extrinsic at lag shifts of k * LAG_STEP_MS, |k| <= LAG_STEPS. The lag is `constrained` when both one-step
shifts score a higher MME than the run's lag, `flat` otherwise.
"""
from __future__ import annotations

import math

import numpy as np

DTHETA_DEG = 0.5        # rotation perturbation of the sweep [deg]
DT_M = 0.02             # translation perturbation of the sweep [m]
RADIUS = 0.3            # neighbourhood radius [m]
MIN_NEIGHBORS = 10
MAX_POINTS = 30_000_000
MAX_SCANS = 1 << 16
CLOUD_LEAF = 0.1        # leaf edge of the assessment cloud [m]; 0: one record per stored point
MAX_POSE_ROWS = 1 << 20  # IMU pose rows a timed store keeps (about 87 min of a 200 Hz IMU)
LAG_STEP_MS = 2.0       # lag profile step [ms]
LAG_STEPS = 10          # lag profile: shifts -LAG_STEPS .. LAG_STEPS steps
AXES = ("x", "y", "z")
NOTHING = "nothing to assess: no LIO scan was stored (LI-Init did not trigger, or the run ended at the hand-over)\n"


def rot_exp(v) -> np.ndarray:
    """Exp of so(3) (Rodrigues)."""
    v = np.asarray(v, float)
    th = float(np.linalg.norm(v))
    if th == 0.0:
        return np.eye(3)
    k = v / th
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    return np.eye(3) + math.sin(th) * K + (1.0 - math.cos(th)) * (K @ K)


def candidates(R_final, T_final, dtheta_deg=DTHETA_DEG, dt=DT_M) -> list:
    """[(name, R_LI, T_LI)]: as-run (None, None), final, rot_<a><+|->, trans_<a><+|->."""
    R0, T0 = np.asarray(R_final, float).reshape(3, 3), np.asarray(T_final, float).reshape(3)
    out = [("as-run", None, None), ("final", R0, T0)]
    for a, ax in enumerate(AXES):
        for sgn, tag in ((1.0, "+"), (-1.0, "-")):
            out.append((f"rot_{ax}{tag}", rot_exp(sgn * math.radians(dtheta_deg) * np.eye(3)[a]) @ R0, T0))
    for a, ax in enumerate(AXES):
        for sgn, tag in ((1.0, "+"), (-1.0, "-")):
            out.append((f"trans_{ax}{tag}", R0, T0 + sgn * dt * np.eye(3)[a]))
    return out


def verdicts(rows) -> dict:
    """{"rot_x": (verdict, MME(+) - MME(final), MME(-) - MME(final)), ...} from the sweep's rows {name: result}."""
    f = rows["final"]["mme"]
    out = {}
    for kind in ("rot", "trans"):
        for ax in AXES:
            dp, dm = rows[f"{kind}_{ax}+"]["mme"] - f, rows[f"{kind}_{ax}-"]["mme"] - f
            out[f"{kind}_{ax}"] = ("constrained" if dp > 0 and dm > 0 else "flat", dp, dm)
    return out


class Assessment:
    """The store of one run's LIO scans on a context and the sweep over it."""

    def __init__(self, gpu, max_points=MAX_POINTS, radius=RADIUS, min_neighbors=MIN_NEIGHBORS, max_scans=MAX_SCANS, timed=False,
                 max_pose_rows=MAX_POSE_ROWS):
        if not (radius > 0 and math.isfinite(radius)):
            raise ValueError(f"assessment radius {radius!r}: must be positive")
        self.g, self.radius, self.min_neighbors = gpu, float(radius), int(min_neighbors)
        self.timed = bool(timed)
        if self.timed:
            self.g.assess_reserve_timed(int(max_points), int(max_scans), int(max_pose_rows))
        else:
            self.g.assess_reserve(int(max_points), int(max_scans))
        self.final = None   # (R_LI, T_LI) of the last stored scan

    def append(self, rot_end, pos_end, R_LI, T_LI):
        if self.g.assess_append(rot_end, pos_end, R_LI, T_LI):
            self.final = (np.array(R_LI, float).reshape(3, 3), np.array(T_LI, float).reshape(3))

    def append_timed(self, rot_end, pos_end, R_LI, T_LI, poses, prior_state):
        """append for a scan undistorted from the IMU pose table `poses` with the propagated state prior_state (liinit_state layout;
        its raw cloud was held by LiInitGpu.assess_hold)."""
        from . import host
        R, p, rli, tli = host.state_pose(prior_state)
        prior = (R, p, rli, tli, np.asarray(prior_state, float)[24:27])
        if self.g.assess_append_timed(rot_end, pos_end, R_LI, T_LI, poses, prior):
            self.final = (np.array(R_LI, float).reshape(3, 3), np.array(T_LI, float).reshape(3))

    def sweep(self, dtheta_deg=DTHETA_DEG, dt=DT_M) -> list:
        """[(name, R_LI, T_LI, result)] of the 14 candidates; R_LI / T_LI of as-run are the final extrinsic's, for the report."""
        out = []
        for name, R, T in candidates(*self.final, dtheta_deg=dtheta_deg, dt=dt):
            res = self.g.assess_evaluate(R, T, radius=self.radius, min_neighbors=self.min_neighbors, as_run=R is None)
            out.append((name, self.final[0] if R is None else R, self.final[1] if T is None else T, res))
        return out

    def sweep_time(self, dtheta_deg=DTHETA_DEG, dt=DT_M, step_ms=LAG_STEP_MS, steps=LAG_STEPS):
        """Timed store: ([(name, R_LI, T_LI, result)] of the 14 candidates re-undistorted at the run's lag, [(shift_ms, result)] of the
        final extrinsic at lag shifts k * step_ms, k = -steps .. steps)."""
        ev = lambda R, T, d: self.g.assess_evaluate_timed(R, T, d, radius=self.radius, min_neighbors=self.min_neighbors,  # noqa: E731
                                                          as_run=R is None)
        rows = []
        for name, R, T in candidates(*self.final, dtheta_deg=dtheta_deg, dt=dt):
            rows.append((name, self.final[0] if R is None else R, self.final[1] if T is None else T, ev(R, T, 0.0)))
        prof = [(k * step_ms, ev(self.final[0], self.final[1], k * step_ms / 1000.0)) for k in range(-steps, steps + 1)]
        return rows, prof

    def report(self) -> str:
        if self.final is None:
            return NOTHING
        return report_text(self.g.assess_info(), self.radius, self.min_neighbors, self.sweep())

    def report_time(self, lag: float) -> str:
        """result/assessment_time.txt of a timed store; lag: the run's total IMU-to-LiDAR time lag [s]."""
        if self.final is None:
            return NOTHING
        rows, prof = self.sweep_time()
        return time_report_text(self.g.assess_info(), self.g.assess_timing_info(), self.radius, self.min_neighbors, rows, prof, lag)

    def write_time(self, path: str, lag: float):
        with open(path, "w") as f:
            f.write(self.report_time(lag))

    def write(self, path: str):
        with open(path, "w") as f:
            f.write(self.report())

    def write_cloud(self, path: str, leaf: float = CLOUD_LEAF):
        """The per-point (leaf 0) or per-leaf entropy and plane variance of the as-run map, the map the run built, as a binary PCD
        (pcd.write_assess). Returns (number of records, totals over every stored point), or None, writing nothing, when no scan was
        stored."""
        from . import pcd
        if self.final is None:
            return None
        rec, tot = self.g.assess_cloud(radius=self.radius, min_neighbors=self.min_neighbors, leaf=leaf, as_run=True)
        pcd.write_assess(path, rec)
        return len(rec), tot


def report_text(info: dict, radius: float, min_neighbors: int, sweep: list, dtheta_deg=DTHETA_DEG, dt=DT_M) -> str:
    """result/assessment.txt: a header line of key value pairs, a column line, one fixed-column row per candidate, one line per axis."""
    from .node import rot_to_euler
    r0 = sweep[0][3]
    lines = [f"radius {radius:.6f} n_min {min_neighbors} stride {r0['stride']} scans {info['scans']} skipped {info['skipped']} "
             f"points {info['points']} queries {r0['queries']} dtheta_deg {dtheta_deg:.6f} dt_m {dt:.6f}",
             "%-9s %11s %11s %11s %10s %10s %10s %10s %10s %10s %15s %15s" % ("candidate", "roll_deg", "pitch_deg", "yaw_deg", "t_x", "t_y",
                                                                            "t_z", "valid", "sparse", "degenerate", "mme", "mpv")]
    for name, R, T, res in sweep:
        e = np.degrees(rot_to_euler(R))
        lines.append("%-9s %11.6f %11.6f %11.6f %10.6f %10.6f %10.6f %10d %10d %10d %15.9f %15.9e" % (
            name, e[0], e[1], e[2], T[0], T[1], T[2], res["valid"], res["sparse"], res["degenerate"], res["mme"], res["mpv"]))
    for axis, (v, dp, dm) in verdicts({name: res for name, _, _, res in sweep}).items():
        lines.append("%-7s %-11s %15.9f %15.9f" % (axis, v, dp, dm))
    return "\n".join(lines) + "\n"


def parse_report(text: str) -> dict:
    """The inverse of report_text: {"header": {...}, "rows": {name: {...}}, "axes": {axis: (verdict, d_plus, d_minus)}}, or
    {"nothing": True}."""
    if text == NOTHING:
        return {"nothing": True}
    ls = text.splitlines()
    h = ls[0].split()
    header = {h[i]: float(h[i + 1]) if "." in h[i + 1] else int(h[i + 1]) for i in range(0, len(h), 2)}
    cols = ls[1].split()
    rows = {}
    for line in ls[2:16]:
        f = line.split()
        rows[f[0]] = {c: (int(x) if c in ("valid", "sparse", "degenerate") else float(x)) for c, x in zip(cols[1:], f[1:])}
    axes = {}
    for line in ls[16:]:
        f = line.split()
        axes[f[0]] = (f[1], float(f[2]), float(f[3]))
    return {"header": header, "rows": rows, "axes": axes}


def lag_verdict(profile) -> tuple:
    """(verdict, best shift [ms]) of a lag profile [(shift_ms, result)] with shift 0 in the middle: `constrained` when both one-step
    shifts score a higher MME than shift 0; the best shift has the lowest MME (the first of equals)."""
    m = {s: r["mme"] for s, r in profile}
    k = [s for s, _ in profile]
    i0 = k.index(0.0)
    v = "constrained" if m[k[i0 - 1]] > m[0.0] and m[k[i0 + 1]] > m[0.0] else "flat"
    best = min((s for s in k if m[s] == m[s]), key=lambda s: m[s], default=0.0)   # (NaN: no valid query)
    return v, best


def time_report_text(info: dict, timing: dict, radius: float, min_neighbors: int, rows: list, profile: list, lag: float,
                     dtheta_deg=DTHETA_DEG, dt=DT_M) -> str:
    """result/assessment_time.txt: a header line (timed / untimed scans, pose rows, the run's lag), the 14 re-undistorted candidates in
    assessment.txt's format, a column line and one row per lag shift, and the lag line."""
    lines = [f"timed_scans {timing['timed_scans']} untimed_scans {timing['untimed_scans']} pose_rows {timing['pose_rows']} "
             f"lag_ms {lag * 1000.0:.6f} lag_step_ms {profile[1][0] - profile[0][0]:.6f}",
             report_text(info, radius, min_neighbors, rows, dtheta_deg, dt).rstrip("\n"),
             "%10s %11s %10s %10s %10s %15s %15s" % ("shift_ms", "lag_ms", "valid", "sparse", "degenerate", "mme", "mpv")]
    for s, r in profile:
        lines.append("%10.3f %11.6f %10d %10d %10d %15.9f %15.9e" % (s, lag * 1000.0 + s, r["valid"], r["sparse"], r["degenerate"], r["mme"],
                                                                   r["mpv"]))
    v, best = lag_verdict(profile)
    lines.append(f"lag {v} best_shift_ms {best:.3f}")
    return "\n".join(lines) + "\n"


def parse_time_report(text: str) -> dict:
    """The inverse of time_report_text: {"header": {...}, "assessment": parse_report's dict of the 14 candidates, "profile":
    [{shift_ms, lag_ms, valid, sparse, degenerate, mme, mpv}], "lag": (verdict, best shift [ms])}, or {"nothing": True}."""
    if text == NOTHING:
        return {"nothing": True}
    ls = text.splitlines()
    h = ls[0].split()
    header = {h[i]: float(h[i + 1]) if "." in h[i + 1] else int(h[i + 1]) for i in range(0, len(h), 2)}
    rep = parse_report("\n".join(ls[1:23]) + "\n")
    cols = ls[23].split()
    prof = []
    for line in ls[24:-1]:
        prof.append({c: (int(x) if c in ("valid", "sparse", "degenerate") else float(x)) for c, x in zip(cols, line.split())})
    f = ls[-1].split()
    assert f[0] == "lag" and f[2] == "best_shift_ms", ls[-1]
    return {"header": header, "assessment": rep, "profile": prof, "lag": (f[1], float(f[3]))}
