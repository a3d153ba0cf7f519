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
from collections import deque

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


# ---- LIO-phase replay -----------------------------------------------------------------------------------------------------------------
REPLAY_MAX_POINTS = 30_000_000   # raw LIO-phase points the replay store keeps on the device (20 bytes each)
REPLAY_LAG_MS = 5.0              # lag shifts of the replay sweep [ms]


class ReplayError(RuntimeError):
    pass


def _clone_odometry(odom):
    """A copy of a LidarOdometry whose loop state can change without touching the original: the state, the IMU processor, the IMU buffer
    and the per-scan bookkeeping are copied; the device context and the configuration are shared. It publishes nothing and feeds no
    timed store."""
    import copy
    from collections import deque

    from . import host
    from .odometry import ImuBuffer
    o = copy.copy(odom)
    o.state = np.array(odom.state, float, copy=True)
    o.imu_proc = copy.copy(odom.imu_proc)
    o.imu_proc.m = host.Imu.from_buffer_copy(odom.imu_proc.m)
    ib = ImuBuffer(odom.imu_buffer.timediff)
    ib.time_lag, ib.last_stamp = odom.imu_buffer.time_lag, odom.imu_buffer.last_stamp
    ib.rows = deque(np.array(r, float, copy=True) for r in odom.imu_buffer.rows)
    o.imu_buffer = ib
    o.preprocess = dict(odom.preprocess)
    o.lidar_buffer = deque()
    o.publish, o.published = None, {}
    o.assess_hold, o.timing, o.replay = False, None, None
    return o


class Replay:
    """Runs the LIO phase of a run again from the hand-over with a candidate calibration, and scores the map that run builds (DESIGN §4d).

    During the run (Node.replay, LidarOdometry.replay): capture() takes the LiDAR-only odometry and the device map as LI-Init found them,
    before the hand-over; after it, every sub-frame the loop processes goes to the device replay store (record_frame), every IMU sample
    is kept in arrival order (record_imu) and every posterior state too (record_update). run() restores the map, hands over with the
    candidate extrinsic and the candidate lag (LidarOdometry.hand_over on a copy of the captured odometry), and drives the same loop body
    (process_raw, staging from the store) over the recorded input; the updates but the switch scan fill the plain assessment store, which
    is then scored as run."""

    def __init__(self, gpu, assessment: Assessment, max_points=REPLAY_MAX_POINTS, max_frames=MAX_SCANS):
        self.g, self.assessment = gpu, assessment
        self.g.replay_reserve(int(max_points), int(max_frames))
        self.base = None          # the LidarOdometry before the hand-over (a copy)
        self.res = None           # LI-Init's result
        self.snapshot_bytes = 0
        self.staged_points = 0    # points of the raw cloud staged at the snapshot (the first updates may store it again)
        self.events = []          # after the hand-over, in arrival order: stored sub-frame index (int) or IMU sample (stamp, gyr, acc)
        self.frames = 0
        self.run_states = []      # (stored sub-frame index, posterior state) of the run's updates after the hand-over
        # concurrent replays (run_many): worker contexts that share this context's replay store and map snapshot, created once
        self.workers = []
        self.jobs = 1             # replays at once of write() and write_refinement()
        self.threads = None       # threads of a batch; None: one per context (a CPU build of the kernels needs 1)
        self.host_lib = None      # the host library that runs the native loop (None: the package's)
        self._recorded = None     # (IMU samples [k, 7], int32 event codes) of self.events for the native loop

    # ---- recording ----
    def capture(self, odom, res):
        if self.base is not None:
            raise ReplayError("the hand-over has been captured already")
        self.snapshot_bytes = self.g.map_snapshot()
        self.staged_points = int(getattr(self.g, "raw_n", 0))
        self.base = _clone_odometry(odom)
        self.res = dict(res)

    def record_imu(self, stamp, gyr, acc):
        if self.base is not None:
            self.events.append((float(stamp), np.array(gyr, float), np.array(acc, float)))

    def record_frame(self, entry):
        if self.base is not None and self.g.replay_append(entry["handle"], entry["t_beg"], entry["end_ms"]):
            self.events.append(self.frames)
            self.frames += 1

    def record_update(self, state):
        if self.base is not None and self.frames:
            self.run_states.append((self.frames - 1, np.array(state, float, copy=True)))

    def info(self) -> dict:
        return self.g.replay_info()

    # ---- replay ----
    def run(self, R_LI=None, T_LI=None, lag_shift: float = 0.0, frozen: bool = True) -> dict:
        """One replay. R_LI / T_LI: the candidate extrinsic (None: LI-Init's); lag_shift [s]: added to LI-Init's total lag; frozen: the
        extrinsic is held constant by every update. Returns {"result": the as-run evaluation, "states": [(sub-frame index, posterior
        state)], "R_LI", "T_LI": the extrinsic the replay ended with, "rms_m": RMS LiDAR position difference to the run's updates at the
        same sub-frames, "seconds"}."""
        import time

        from .odometry import ReplayFrame
        if self.base is None:
            raise ReplayError("nothing to replay: the run did not reach the hand-over")
        info = self.info()
        if info["skipped"]:
            raise ReplayError(f"the replay store is truncated ({info['skipped']} sub-frames skipped): raise its max_points")
        t0 = time.perf_counter()
        frames = [self.g.replay_frame(j) for j in range(info["frames"])]
        o = self._hand_over(self.g, R_LI, T_LI, lag_shift, frozen)
        states = []
        pending = deque()
        for ev in self.events:
            if isinstance(ev, int):
                pending.append(ev)
            else:
                o.imu_buffer.push(*ev)
            # sync_packages: a sub-frame waits for an IMU stamp at or after its end
            while pending:
                f = frames[pending[0]]
                t_end = f["t_beg"] + float(f["end_ms"]) / 1000.0
                if not o.imu_buffer.rows or not o.imu_buffer.ready(t_end):
                    break
                j = pending.popleft()
                frame_num = o.frame_num
                o.process_raw(ReplayFrame(j, f["end_ms"], f["n"]), f["t_beg"], o.imu_buffer.pop(t_end))
                if o.frame_num != frame_num:
                    states.append((j, o.state.copy()))
                    if o.switch_scan != o.frame_num - 1:
                        R, p, rli, tli = host_pose(o.state)
                        self.g.assess_append(R, p, rli, tli)
        a = self.assessment
        result = self.g.assess_evaluate(radius=a.radius, min_neighbors=a.min_neighbors, as_run=True)
        _, _, rli, tli = host_pose(o.state)
        return dict(result=result, states=states, R_LI=rli, T_LI=tli, rms_m=trajectory_rms(self.run_states, states),
                    seconds=time.perf_counter() - t0)

    def _hand_over(self, g, R_LI, T_LI, lag_shift, frozen):
        """The start of a replay on context g: the map restored, a copy of the captured odometry handed over with the candidate extrinsic
        (None: LI-Init's) and lag shift [s], for a frozen replay the extrinsic's covariance and propagation noise zeroed, the assessment
        store emptied. Returns the odometry."""
        res = dict(self.res)
        if R_LI is not None:
            res["R_LI"], res["T_LI"] = np.asarray(R_LI, float).reshape(3, 3), np.asarray(T_LI, float).reshape(3)
        res["time_lag_2"] = float(res["time_lag_2"]) + float(lag_shift)
        o = _clone_odometry(self.base)
        o.g = g
        g.map_restore()
        o.hand_over(res)
        if frozen:
            o.frozen = True
            cov = o.state[36:].reshape(24, 24)
            cov[6:12, :] = 0.0
            cov[:, 6:12] = 0.0
            o.imu_proc.set_cov("R_LI_cov", 0.0)
            o.imu_proc.set_cov("T_LI_cov", 0.0)
        g.assess_clear()
        return o

    def run_native(self, R_LI=None, T_LI=None, lag_shift: float = 0.0, frozen: bool = True, g=None) -> dict:
        """run() with the loop after the hand-over in native code (host.replay_run), on context g: this one (None) or a worker of
        run_many. Returns run()'s dict, bit for bit."""
        import time

        from . import host
        if self.base is None:
            raise ReplayError("nothing to replay: the run did not reach the hand-over")
        g = self.g if g is None else g
        info = self.info()
        if info["skipped"]:
            raise ReplayError(f"the replay store is truncated ({info['skipped']} sub-frames skipped): raise its max_points")
        if not self.base.map_ready:
            raise ReplayError("nothing to replay: the map was not built at the hand-over")
        t0 = time.perf_counter()
        if self._recorded is None or self._recorded[2] != len(self.events):
            imu = [e for e in self.events if not isinstance(e, int)]
            samples = np.array([np.concatenate([[t], gyr, acc]) for t, gyr, acc in imu], np.float64).reshape(-1, 7)
            codes = np.array([e if isinstance(e, int) else host.REPLAY_IMU for e in self.events], np.int32)
            self._recorded = (samples, codes, len(self.events))
        o = self._hand_over(g, R_LI, T_LI, lag_shift, frozen)
        states = host.replay_run(g, o, self._recorded[0], self._recorded[1], lib=self.host_lib)
        if g is not self.g and g.assess_info()["skipped"]:
            raise ReplayError("a replay worker's assessment store overflowed: replay with one job")
        a = self.assessment
        result = g.assess_evaluate(radius=a.radius, min_neighbors=a.min_neighbors, as_run=True)
        _, _, rli, tli = host_pose(states[-1][1] if states else o.state)
        return dict(result=result, states=states, R_LI=rli, T_LI=tli, rms_m=trajectory_rms(self.run_states, states),
                    seconds=time.perf_counter() - t0)

    def pool(self, jobs: int) -> list:
        """The contexts of a batch of `jobs` concurrent replays: this one and jobs - 1 workers. A worker is a context of this one's
        configuration that shares its replay store and map snapshot (liinit_replay_share), with an assessment store sized to the replay
        store's points and frames; workers are created on first need and kept until close()."""
        if isinstance(jobs, bool) or int(jobs) != jobs or jobs < 1:
            raise ValueError(f"replay jobs {jobs!r}: must be a positive integer")
        if self.base is None:
            raise ReplayError("nothing to replay: the run did not reach the hand-over")
        info = self.info()
        while len(self.workers) < jobs - 1:
            w = self.g.twin()
            try:
                w.replay_share(self.g)
                w.assess_reserve(info["points"] + self.staged_points, info["frames"] + 1)
            except BaseException:
                w.close()
                raise
            self.workers.append(w)
        return [self.g] + self.workers[:jobs - 1]

    def run_many(self, cands, jobs: int = 1, threads=None, native=None) -> list:
        """Every candidate (R_LI, T_LI, lag_shift [s], frozen) replayed on the contexts of pool(jobs), one thread per context taking
        the candidates in list order. Returns run()'s dicts in list order; "seconds" is each replay's own wall time. native (default:
        jobs > 1): the native loop (run_native), else run() on this context. threads (default self.threads, else one per context): 1
        drives the contexts in turn from the calling thread."""
        return run_across([(self, c) for c in cands], jobs, threads, native)

    def close(self):
        """Destroy the workers (the context they share can then be destroyed)."""
        while self.workers:
            self.workers.pop().close()

    def sweep(self, R_final, T_final, dtheta_deg=DTHETA_DEG, dt=DT_M, lag_ms=REPLAY_LAG_MS, jobs: int = 1) -> list:
        """[(name, R_LI, T_LI, shift_ms, replay)] of the 17 replays: the run itself (not frozen), LI-Init's result, the final extrinsic,
        its 12 perturbations, and the final extrinsic at lag shifts of -+lag_ms; all frozen but the first. jobs: replays at once
        (run_many)."""
        R_init = np.asarray(self.res["R_LI"], float).reshape(3, 3)
        T_init = np.asarray(self.res["T_LI"], float).reshape(3)
        plan = [("run", R_init, T_init, 0.0, False), ("li-init", R_init, T_init, 0.0, True)]
        plan += [(name, R, T, 0.0, True) for name, R, T in candidates(R_final, T_final, dtheta_deg, dt)[1:]]
        plan += [(f"lag{s:+g}", plan[2][1], plan[2][2], s, True) for s in (-lag_ms, lag_ms)]
        runs = self.run_many([(None if name == "run" else R, None if name == "run" else T, shift_ms / 1000.0, frozen)
                              for name, R, T, shift_ms, frozen in plan], jobs)
        return [(name, R, T, shift_ms, r) for (name, R, T, shift_ms, _), r in zip(plan, runs)]

    def report(self, R_final, T_final, jobs: int = 1) -> str:
        import time
        t0 = time.perf_counter()
        rows = self.sweep(R_final, T_final, jobs=jobs)
        wall = time.perf_counter() - t0
        return replay_report_text(self.info(), self.snapshot_bytes, wall, self.assessment.radius, self.assessment.min_neighbors, rows)

    def write(self, path: str, R_final=None, T_final=None):
        """result/assessment_replay.txt, self.jobs replays at once; R_final / T_final: the run's final extrinsic. NOTHING when the run
        did not hand over."""
        with open(path, "w") as f:
            f.write(NOTHING if self.base is None or not self.frames else self.report(R_final, T_final, self.jobs))

    @property
    def lag(self) -> float:
        """The node's total lag at the hand-over, time_lag_IMU_wtr_lidar + timediff_imu_wrt_lidar [s]; a replay's lag shift adds to it."""
        return float(self.base.imu_buffer.timediff) + float(self.res["time_lag_1"]) + float(self.res["time_lag_2"])

    def refine(self, R_final, T_final, max_replays=None, jobs: int = 1) -> dict:
        """refine.search with frozen replays as the scorer, from the run's final extrinsic and LI-Init's at shift 0. Returns search's
        dict with, on every trace row, the replay's "result" (the as-run evaluation) and "seconds"; and "wall_s", "lag0" (the lag at the
        hand-over [s]), "time_lag" (the refined total lag [s]), "state" (the best replay's last posterior state, whose extrinsic is the
        refined one) and "calib" (node.state_calib_values of that state and lag, the arguments of node.calib_result_text). jobs: replays
        at once; the search scores its batches with run_many."""
        import time

        from . import refine as rf
        from .node import state_calib_values
        kept = {}

        def score_many(cands):
            runs = self.run_many([(R, T, shift_s, True) for R, T, shift_s in cands], jobs)
            for (R, T, shift_s), r in zip(cands, runs):
                kept[rf.key(R, T, shift_s)] = (r["result"], r["seconds"], r["states"][-1][1] if r["states"] else None)
            return [r["result"]["mme"] for r in runs]
        t0 = time.perf_counter()
        out = rf.search(lambda R, T, shift_s: score_many([(R, T, shift_s)])[0], R_final, T_final, 0.0,
                        rf.MAX_REPLAYS if max_replays is None else max_replays, R_init=self.res["R_LI"], T_init=self.res["T_LI"],
                        score_many=score_many)
        out["wall_s"] = time.perf_counter() - t0
        for row in out["trace"]:
            row["result"], row["seconds"], _ = kept[rf.key(row["R"], row["T"], row["shift_ms"] / 1000.0)]
        state = kept[rf.key(out["R"], out["T"], out["shift_s"])][2]
        if state is None:
            raise ReplayError("the best replay made no LIO update: nothing to take the biases and gravity from")
        out["lag0"] = self.lag
        out["time_lag"] = self.lag + out["shift_s"]
        out["state"] = state
        out["calib"] = state_calib_values(state, out["time_lag"])
        return out

    def write_refinement(self, path: str, R_final=None, T_final=None, max_replays=None):
        """result/refinement.txt (refine_report_text), self.jobs replays at once; R_final / T_final: the run's final extrinsic. Returns
        refine's dict, or None, writing NOTHING, when the run did not hand over."""
        if self.base is None or not self.frames:
            with open(path, "w") as f:
                f.write(NOTHING)
            return None
        ref = self.refine(R_final, T_final, max_replays, self.jobs)
        with open(path, "w") as f:
            f.write(refine_report_text(self.info(), ref, self.assessment.radius, self.assessment.min_neighbors))
        return ref

    def profile(self, ref, jobs: int = 1, steps=None) -> dict:
        """profiles.profile around refine's result `ref` (its R, T and shift; its MME is the centre's, not replayed again), with frozen
        replays as the scorer, all at once on the contexts of pool(jobs). Returns profile's dict with, on every row, the replay's
        "result" and "seconds"; and "wall_s", "jobs", "replays" and "status" (the refinement's)."""
        import time

        from . import profiles as pf
        kept = []

        def score_many(cands):
            kept[:] = self.run_many([(R, T, s, True) for R, T, s in cands], jobs)
            return [r["result"]["mme"] for r in kept]
        t0 = time.perf_counter()
        out = pf.profile(score_many, ref["R"], ref["T"], ref["shift_s"], ref["mme"], pf.STEPS if steps is None else steps, lag0=self.lag)
        out["wall_s"] = time.perf_counter() - t0
        for row, r in zip(out["rows"], kept):
            row["result"], row["seconds"] = r["result"], r["seconds"]
        out.update(jobs=jobs, replays=len(out["rows"]), status=ref["status"])
        return out

    def write_profile(self, path: str, ref, steps=None):
        """result/profile.txt (profile_report_text) around refine's result `ref`, self.jobs replays at once. Returns profile's dict, or
        None, writing NOTHING, when there is no refinement (ref None: the run did not hand over)."""
        if ref is None:
            with open(path, "w") as f:
                f.write(NOTHING)
            return None
        prof = self.profile(ref, self.jobs, steps)
        with open(path, "w") as f:
            f.write(profile_report_text(prof))
        return prof


def run_across(tasks, jobs: int = 1, threads=None, native=None) -> list:
    """Replays of one or more recordings at once: tasks [(replay, (R_LI, T_LI, lag_shift [s], frozen))]. Every replay named runs its
    own tasks on the contexts of its pool(jobs), one thread per context, the threads of every replay at once, each taking its replay's
    tasks in list order. Returns Replay.run's dicts in task order; an error of a task stops the batch and the first such error by task
    order is raised. native (default: more than one context in all): the native loop (run_native), else Replay.run. threads (default
    the smallest Replay.threads set, else one per context): 1 drives the contexts in turn from the calling thread, each replay's tasks on
    its contexts round robin."""
    import threading
    tasks = list(tasks)
    replays = list(dict.fromkeys(rp for rp, _ in tasks))
    pools = {rp: rp.pool(jobs) for rp in replays}
    nctx = sum(len(p) for p in pools.values())
    if not (nctx > 1 if native is None else native):
        return [rp.run(*c) for rp, c in tasks]
    if threads is None:
        threads = min((rp.threads for rp in replays if rp.threads is not None), default=None)
    out = [None] * len(tasks)
    if (threads is not None and int(threads) <= 1) or len(tasks) <= 1:
        seen = dict.fromkeys(replays, 0)
        for i, (rp, c) in enumerate(tasks):
            out[i] = rp.run_native(*c, g=pools[rp][seen[rp] % len(pools[rp])])
            seen[rp] += 1
        return out
    # contexts round robin across the replays, so that a thread limit below the contexts still serves every replay
    ctxs = [(rp, p[k]) for k in range(max(len(p) for p in pools.values())) for rp, p in pools.items() if k < len(p)]
    if threads is not None:
        ctxs = ctxs[:max(int(threads), len(replays))]
    lock, errors = threading.Lock(), []
    nxt = {rp: iter([i for i, (r, _) in enumerate(tasks) if r is rp]) for rp in replays}

    def work(rp, g):
        while True:
            with lock:
                i = None if errors else next(nxt[rp], None)
            if i is None:
                return
            try:
                out[i] = rp.run_native(*tasks[i][1], g=g)
            except BaseException as e:
                with lock:
                    errors.append((i, e))
                return
    ts = [threading.Thread(target=work, args=c) for c in ctxs]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise min(errors, key=lambda x: x[0])[1]
    return out


def host_pose(state):
    from . import host
    return host.state_pose(state)


def trajectory_rms(run_states, states) -> float:
    """RMS difference [m] of the LiDAR positions (R T_LI + p) of two lists of (sub-frame index, state), over the indices both have."""
    def lidar(s):
        R, p, _, tli = host_pose(s)
        return R @ tli + p
    a = dict(run_states)
    d = [lidar(s) - lidar(a[j]) for j, s in states if j in a]
    return float(np.sqrt(np.mean(np.sum(np.square(d), axis=1)))) if d else float("nan")


def replay_report_text(info: dict, snapshot_bytes: int, wall_s: float, radius: float, min_neighbors: int, rows: list, dtheta_deg=DTHETA_DEG,
                       dt=DT_M) -> str:
    """result/assessment_replay.txt: a header line of key value pairs, a column line, one fixed-column row per replay (the candidate, its
    lag shift, the as-run score of the map the replay built, the extrinsic it ended with and the RMS LiDAR position difference to the run),
    one line per axis and the lag line."""
    from .node import rot_to_euler
    lines = [f"subframes {info['frames']} skipped {info['skipped']} points {info['points']} snapshot_mb {snapshot_bytes / 1e6:.6f} "
             f"replay_s {wall_s:.6f} radius {radius:.6f} n_min {min_neighbors} dtheta_deg {dtheta_deg:.6f} dt_m {dt:.6f}",
             "%-9s %11s %11s %11s %10s %10s %10s %9s %10s %10s %10s %15s %15s %11s %11s %11s %10s %10s %10s %12s" % (
                 "candidate", "roll_deg", "pitch_deg", "yaw_deg", "t_x", "t_y", "t_z", "shift_ms", "valid", "sparse", "degenerate", "mme",
                 "mpv", "end_roll", "end_pitch", "end_yaw", "end_t_x", "end_t_y", "end_t_z", "rms_m")]
    for name, R, T, shift_ms, r in rows:
        e, ee, res, te = np.degrees(rot_to_euler(R)), np.degrees(rot_to_euler(r["R_LI"])), r["result"], r["T_LI"]
        lines.append("%-9s %11.6f %11.6f %11.6f %10.6f %10.6f %10.6f %9.3f %10d %10d %10d %15.9f %15.9e %11.6f %11.6f %11.6f %10.6f %10.6f %10.6f "
                     "%12.6e" % (name, e[0], e[1], e[2], T[0], T[1], T[2], shift_ms, res["valid"], res["sparse"], res["degenerate"], res["mme"],
                                 res["mpv"], ee[0], ee[1], ee[2], te[0], te[1], te[2], r["rms_m"]))
    by_name = {name: r["result"] for name, _, _, _, r in rows}
    for axis, (v, dp, dm) in verdicts(by_name).items():
        lines.append("%-7s %-11s %15.9f %15.9f" % (axis, v, dp, dm))
    prof = [(s, r["result"]) for name, _, _, s, r in rows if name.startswith("lag")]
    prof = sorted(prof + [(0.0, by_name["final"])], key=lambda x: x[0])
    v, best = lag_verdict(prof)
    m = {s: r["mme"] for s, r in prof}
    lines.append(f"lag {v} best_shift_ms {best:.3f} d_minus {m[prof[0][0]] - m[0.0]:.9f} d_plus {m[prof[-1][0]] - m[0.0]:.9f}")
    return "\n".join(lines) + "\n"


def parse_replay_report(text: str) -> dict:
    """The inverse of replay_report_text: {"header": {...}, "rows": {name: {...}}, "axes": {axis: (verdict, d_plus, d_minus)},
    "lag": (verdict, best shift [ms], d_minus, d_plus)}, or {"nothing": True}."""
    if text == NOTHING:
        return {"nothing": True}
    ls = text.splitlines()
    h = ls[0].split()
    header = {h[i]: float(h[i + 1]) if "." in h[i + 1] else int(h[i + 1]) for i in range(0, len(h), 2)}
    cols = ls[1].split()
    rows, axes = {}, {}
    i = 2
    while i < len(ls) and len(ls[i].split()) == len(cols):
        f = ls[i].split()
        rows[f[0]] = {c: (int(x) if c in ("valid", "sparse", "degenerate") else float(x)) for c, x in zip(cols[1:], f[1:])}
        i += 1
    for line in ls[i:-1]:
        f = line.split()
        axes[f[0]] = (f[1], float(f[2]), float(f[3]))
    f = ls[-1].split()
    assert f[0] == "lag" and f[2] == "best_shift_ms" and f[4] == "d_minus" and f[6] == "d_plus", ls[-1]
    return {"header": header, "rows": rows, "axes": axes, "lag": (f[1], float(f[3]), float(f[5]), float(f[7]))}


REFINED = "Refined result:"
_REFINE_INT = ("subframes", "skipped", "replays", "at_edge", "n_min", "valid", "sparse", "degenerate")


def refine_report_text(info: dict, ref: dict, radius: float, min_neighbors: int) -> str:
    """result/refinement.txt of Replay.refine's dict: a header line of key value pairs (the replay store's sub-frames and skipped ones,
    the start candidate, the replays, the wall time, converged or budget, whether stage 1's lag minimum lay at the cap, the lag at the
    hand-over, the refined lag shift and total lag, the score's radius and n_min), a column line, one fixed-column row per replay in
    evaluation order (its stage, the candidate, its lag shift, the as-run score of the map it built and its time), one line per axis (its
    verdict, the final step [deg or m] and the MME differences of its + and - neighbours at that step to the refined candidate), then
    `Refined result:` and node.calib_result_text."""
    from .node import calib_result_text, rot_to_euler
    from .refine import axis_verdict
    lines = [f"subframes {info['frames']} skipped {info['skipped']} start {ref['start']} replays {len(ref['trace'])} "
             f"wall_s {ref['wall_s']:.6f} status {ref['status']} at_edge {int(ref['at_edge'])} lag0_ms {ref['lag0'] * 1000.0:.6f} "
             f"shift_ms {ref['shift_ms']:.6f} lag_ms {ref['time_lag'] * 1000.0:.6f} radius {radius:.6f} n_min {min_neighbors}",
             "%-7s %11s %11s %11s %10s %10s %10s %11s %10s %10s %10s %15s %15s %9s" % (
                 "stage", "roll_deg", "pitch_deg", "yaw_deg", "t_x", "t_y", "t_z", "shift_ms", "valid", "sparse", "degenerate", "mme", "mpv",
                 "seconds")]
    for r in ref["trace"]:
        e, T, res = np.degrees(rot_to_euler(r["R"])), r["T"], r["result"]
        lines.append("%-7s %11.6f %11.6f %11.6f %10.6f %10.6f %10.6f %11.6f %10d %10d %10d %15.9f %15.9e %9.3f" % (
            r["stage"], e[0], e[1], e[2], T[0], T[1], T[2], r["shift_ms"], res["valid"], res["sparse"], res["degenerate"], res["mme"],
            res["mpv"], r["seconds"]))
    for axis, (step, dp, dm) in ref["axes"].items():
        lines.append("%-7s %-11s %12.6f %15.9f %15.9f" % (axis, axis_verdict(dp, dm), step, dp, dm))
    return "\n".join(lines) + "\n" + REFINED + "\n" + calib_result_text(**ref["calib"])


def parse_refine_report(text: str) -> dict:
    """The inverse of refine_report_text: {"header": {...}, "rows": [{"stage", ...}] in evaluation order, "axes": {axis: (verdict, step,
    d_plus, d_minus)}, "result": the calib_result_text block}, or {"nothing": True}."""
    if text == NOTHING:
        return {"nothing": True}
    head, result = text.split("\n" + REFINED + "\n", 1)
    ls = head.splitlines()

    def val(x):
        for t in (int, float):
            try:
                return t(x)
            except ValueError:
                pass
        return x
    h = ls[0].split()
    header = {h[i]: val(h[i + 1]) for i in range(0, len(h), 2)}
    cols = ls[1].split()
    n = header["replays"]
    rows = [{c: (x if c == "stage" else int(x) if c in _REFINE_INT else float(x)) for c, x in zip(cols, line.split())}
            for line in ls[2:2 + n]]
    axes = {}
    for line in ls[2 + n:]:
        f = line.split()
        axes[f[0]] = (f[1], float(f[2]), float(f[3]), float(f[4]))
    return {"header": header, "rows": rows, "axes": axes, "result": result}


_JOINT_INT = ("recordings", "candidates", "replays", "jobs", "at_edge", "n_min", "subframes", "skipped")


def _euler_t(R, T) -> str:
    from .node import rot_to_euler
    e = np.degrees(rot_to_euler(np.asarray(R, float).reshape(3, 3)))
    T = np.asarray(T, float).reshape(3)
    return "%.6f,%.6f,%.6f %.6f,%.6f,%.6f" % (e[0], e[1], e[2], T[0], T[1], T[2])


def joint_report_text(recs: list, ref: dict, radius: float, min_neighbors: int) -> str:
    """result/refinement_joint.txt of joint.refine_replays' dict. recs: per recording {"bag", "subframes", "skipped", "lag" (its total lag
    at the hand-over [s]), "R_init", "T_init" (LI-Init's result), "R_final", "T_final" (the run's final extrinsic)}. A header line of key
    value pairs (the recordings, candidates and replays, the start, the wall time, converged or budget, at_edge, L0, the refined shift and
    total lag, the score's radius and n_min); one `rec` line per recording (sub-frames, skipped, its lag, LI-Init's and the final
    extrinsic as roll,pitch,yaw [deg] and x,y,z [m], then the bag to the end of the line); a column line and one fixed-column row per
    candidate in evaluation order (its stage, the candidate, its total lag, the joint MME and the recordings' MMEs); one line per axis for
    the joint score (`joint`) and per recording (`rec<b>`): verdict, final step, the + and - neighbour differences; then `Refined
    result:` and, per recording, `Recording <b>:` and node.calib_result_text of its replay of the refined candidate."""
    from .node import calib_result_text, rot_to_euler
    from .refine import axis_verdict
    B = len(recs)
    lines = [f"recordings {B} candidates {len(ref['trace'])} replays {len(ref['trace']) * B} start {ref['start']} "
             f"wall_s {ref['wall_s']:.6f} status {ref['status']} at_edge {int(ref['at_edge'])} lag0_ms {ref['lag0'] * 1000.0:.6f} "
             f"shift_ms {ref['shift_ms']:.6f} lag_ms {ref['time_lag'] * 1000.0:.6f} radius {radius:.6f} n_min {min_neighbors}"]
    for b, r in enumerate(recs):
        lines.append(f"rec {b} subframes {r['subframes']} skipped {r['skipped']} lag_ms {r['lag'] * 1000.0:.6f} "
                     f"li_init {_euler_t(r['R_init'], r['T_init'])} final {_euler_t(r['R_final'], r['T_final'])} bag {r['bag']}")
    lines.append("%-10s %11s %11s %11s %10s %10s %10s %11s %15s" % ("stage", "roll_deg", "pitch_deg", "yaw_deg", "t_x", "t_y", "t_z", "lag_ms",
                                                                 "mme") + "".join(" %15s" % f"mme_{b}" for b in range(B)))
    for r in ref["trace"]:
        e, T = np.degrees(rot_to_euler(r["R"])), r["T"]
        lines.append("%-10s %11.6f %11.6f %11.6f %10.6f %10.6f %10.6f %11.6f %15.9f" % (r["stage"], e[0], e[1], e[2], T[0], T[1], T[2],
                                                                                   r["lag"] * 1000.0, r["mme"])
                     + "".join(" %15.9f" % m for m in r["mmes"]))
    for who, axes in [("joint", ref["axes"])] + [(f"rec{b}", a) for b, a in enumerate(ref["axes_rec"])]:
        for axis, (step, dp, dm) in axes.items():
            lines.append("%-6s %-7s %-11s %12.6f %15.9f %15.9f" % (who, axis, axis_verdict(dp, dm), step, dp, dm))
    blocks = "".join(f"Recording {b}:\n" + calib_result_text(**c) for b, c in enumerate(ref["calibs"]))
    return "\n".join(lines) + "\n" + REFINED + "\n" + blocks


def parse_joint_report(text: str) -> dict:
    """The inverse of joint_report_text: {"header": {...}, "recs": [{"subframes", "skipped", "lag_ms", "li_init", "final" (each
    (roll, pitch, yaw, x, y, z)), "bag"}], "rows": [{"stage", ..., "mme", "mmes": [...]}] in evaluation order, "axes": {"joint" or b:
    {axis: (verdict, step, d_plus, d_minus)}}, "result": [the calib_result_text block of each recording]}."""
    import re
    head, result = text.split("\n" + REFINED + "\n", 1)
    ls = head.splitlines()

    def val(x):
        for t in (int, float):
            try:
                return t(x)
            except ValueError:
                pass
        return x
    h = ls[0].split()
    header = {h[i]: val(h[i + 1]) for i in range(0, len(h), 2)}
    B, n = header["recordings"], header["candidates"]
    recs = []
    for line in ls[1:1 + B]:
        kv, bag = line.split(" bag ", 1)
        f = kv.split()
        assert f[0] == "rec" and int(f[1]) == len(recs), line
        r = {f[i]: val(f[i + 1]) for i in (2, 4, 6)}
        r["li_init"] = tuple(float(x) for x in (f[9] + "," + f[10]).split(","))
        r["final"] = tuple(float(x) for x in (f[12] + "," + f[13]).split(","))
        r["bag"] = bag
        recs.append(r)
    cols = ls[1 + B].split()
    rows = []
    for line in ls[2 + B:2 + B + n]:
        f = line.split()
        row = {c: (x if c == "stage" else float(x)) for c, x in zip(cols[:9], f[:9])}
        row["mmes"] = [float(x) for x in f[9:]]
        rows.append(row)
    axes = {}
    for line in ls[2 + B + n:]:
        f = line.split()
        who = "joint" if f[0] == "joint" else int(f[0][3:])
        axes.setdefault(who, {})[f[1]] = (f[2], float(f[3]), float(f[4]), float(f[5]))
    blocks = re.split(r"^Recording \d+:\n", result, flags=re.M)[1:]
    return {"header": header, "recs": recs, "rows": rows, "axes": axes, "result": blocks}


_FIT_COLS = ("c0", "c1", "c2", "s", "u_star", "se", "min", "lo", "hi")


def profile_report_text(prof: dict) -> str:
    """result/profile.txt of Replay.profile's dict, or result/profile_joint.txt of joint.profile_replays' (which has "recs"). A header
    line of key value pairs (for a joint profile the recordings and candidates; the replays, the jobs, the wall time, the refinement's
    status, the steps n and each parameter's step); the centre line (its roll,pitch,yaw [deg] and x,y,z [m], its total lag and shift
    [ms], its MME and, joint, the recordings' MMEs); a column line and one fixed-column row per profile point in evaluation order (the
    parameter, k, its offset in the parameter's unit, then the as-run valid queries, MME and replay time, per recording for a joint
    profile after the joint MME); a column line and one fit line per parameter: `fit`, or `joint` and `rec<b>` for a joint profile, the
    parameter, its verdict and unit, c0 c1 c2, s, u* and se [steps], the minimum and the interval lo hi in the unit, whether the centre
    lies inside it, and the lowest profile point's k and MME difference to the centre."""
    from .profiles import H_LAG_MS, H_ROT_DEG, H_TRANS_M, UNITS
    c = prof["centre"]
    joint = "recs" in prof
    B = len(prof["recs"]) if joint else 1
    head = (f"recordings {B} candidates {len(prof['rows'])} " if joint else "") + (
        f"replays {len(prof['rows']) * B} jobs {prof['jobs']} wall_s {prof['wall_s']:.6f} status {prof['status']} steps {prof['steps']} "
        f"h_rot_deg {H_ROT_DEG:.6f} h_trans_m {H_TRANS_M:.6f} h_lag_ms {H_LAG_MS:.6f}")
    centre = f"centre {_euler_t(c['R'], c['T'])} lag_ms {c['lag_s'] * 1000.0:.6f} shift_ms {c['shift_s'] * 1000.0:.6f} mme {c['mme']:.9f}"
    if joint:
        centre += " mmes " + ",".join("%.9f" % m for m in c["mmes"])
    cols = ["param", "k", "offset"] + (["mme"] + [f"{x}_{b}" for b in range(B) for x in ("valid", "mme", "seconds")] if joint else
                                       ["valid", "mme", "seconds"])
    lines = ["profile " + head, centre, "%-7s %3s %16s" % tuple(cols[:3]) + "".join(" %15s" % x for x in cols[3:])]
    for r in prof["rows"]:
        line = "%-7s %3d %16.9f" % (r["param"], r["k"], r["offset"])
        if joint:
            line += " %15.9f" % r["mme"]
        results, secs = (r["results"], r["seconds"]) if joint else ([r["result"]], [r["seconds"]])
        for res, sec in zip(results, secs):
            line += " %15d %15.9f %15.3f" % (res["valid"], res["mme"], sec)
        lines.append(line)
    lines.append("%-6s %-7s %-10s %-4s" % ("who", "param", "verdict", "unit") + "".join(" %16s" % x for x in _FIT_COLS)
                 + " %13s %7s %16s" % ("centre_inside", "lower_k", "lower_dmme"))
    whos = [("joint", prof["fits"])] + [(f"rec{b}", f) for b, f in enumerate(prof["recs"])] if joint else [("fit", prof["fits"])]
    for who, fits in whos:
        for p, f in fits.items():
            vals = (*f["c"], f["s"], f["u"], f["se"], f["u_phys"], f["lo_phys"], f["hi_phys"])
            lines.append("%-6s %-7s %-10s %-4s" % (who, p, f["verdict"], UNITS[p.split("_")[0]]) + "".join(" %16.9e" % v for v in vals)
                         + " %13d %7d %16.9e" % (int(f["centre_inside"]), f["lower_k"], f["lower_dmme"]))
    return "\n".join(lines) + "\n"


def parse_profile_report(text: str) -> dict:
    """The inverse of profile_report_text: {"header": {...}, "centre": {"euler_deg", "t_m" (tuples), "lag_ms", "shift_ms", "mme" and,
    joint, "mmes"}, "rows": [{"param", "k", "offset", "valid", "mme", "seconds"}, or for a joint profile {"param", "k", "offset", "mme",
    "valid", "mmes", "seconds" (lists per recording)}] in evaluation order, "fits": {param: {"verdict", "unit", "c0", ..., "hi",
    "centre_inside", "lower_k", "lower_dmme"}} or, joint, {"joint" or b: {param: ...}}}, or {"nothing": True}."""
    if text == NOTHING:
        return {"nothing": True}
    ls = text.splitlines()
    h = ls[0].split()
    assert h[0] == "profile", ls[0]
    header = {h[i]: (h[i + 1] if h[i] == "status" else float(h[i + 1]) if "." in h[i + 1] else int(h[i + 1])) for i in range(1, len(h), 2)}
    joint = "recordings" in header
    B = header["recordings"] if joint else 1
    f = ls[1].split()
    assert f[0] == "centre", ls[1]
    e, t = (tuple(float(x) for x in v.split(",")) for v in f[1:3])
    centre = dict(euler_deg=e, t_m=t, **{f[i]: float(f[i + 1]) for i in range(3, 9, 2)})
    if joint:
        centre["mmes"] = [float(x) for x in f[10].split(",")]
    n = header["candidates"] if joint else header["replays"]
    rows = []
    for line in ls[3:3 + n]:
        f = line.split()
        row = dict(param=f[0], k=int(f[1]), offset=float(f[2]))
        if joint:
            row.update(mme=float(f[3]), valid=[int(x) for x in f[4::3]], mmes=[float(x) for x in f[5::3]],
                       seconds=[float(x) for x in f[6::3]])
        else:
            row.update(valid=int(f[3]), mme=float(f[4]), seconds=float(f[5]))
        rows.append(row)
    fits = {}
    for line in ls[4 + n:]:
        f = line.split()
        fit = dict(verdict=f[2], unit=f[3], **{k: float(x) for k, x in zip(_FIT_COLS, f[4:13])})
        fit.update(centre_inside=bool(int(f[13])), lower_k=int(f[14]), lower_dmme=float(f[15]))
        who = "fit" if f[0] == "fit" else "joint" if f[0] == "joint" else int(f[0][3:])
        fits.setdefault(who, {})[f[1]] = fit
    return {"header": header, "centre": centre, "rows": rows, "fits": fits["fit"] if not joint else fits}
