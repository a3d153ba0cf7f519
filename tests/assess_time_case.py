"""A synthetic timed-assessment case: a trajectory with time-varying yaw rate and acceleration, a room, and scans with IMU pose tables
built from the trajectory (optionally shifted by a known lag). Test infrastructure for the timed assessment tests."""
import math

import numpy as np

from assess_oracle import rot_exp

R_LI_TRUE = rot_exp([0.02, -0.03, 0.05])
T_LI_TRUE = np.array([0.1, -0.05, 0.08])


def yaw(t):
    return 3.0 / math.pi * (1.0 - math.cos(math.pi * t))   # yaw rate 3 sin(pi t) rad/s


def truth(t):
    """(R, p, v, a, omega) of the IMU at time t."""
    c, s = math.cos(yaw(t)), math.sin(yaw(t))
    R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    p = np.array([0.8 * t + 0.3 * math.sin(2 * t), 0.4 * t, 0.05 * math.sin(3 * t)])
    v = np.array([0.8 + 0.6 * math.cos(2 * t), 0.4, 0.15 * math.cos(3 * t)])
    a = np.array([-1.2 * math.sin(2 * t), 0.0, -0.45 * math.sin(3 * t)])
    return R, p, v, a, np.array([0.0, 0.0, 3.0 * math.sin(math.pi * t)])


def room(rng, n):
    """n points on the floor and four walls of a 6 m x 6 m x 2 m room, noise-free."""
    k = rng.integers(0, 5, n)
    u, v = rng.uniform(-3, 3, n), rng.uniform(0, 2, n)
    pts = np.c_[rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), np.zeros(n)]
    for f, (ax, val) in enumerate(((0, -3.0), (0, 3.0), (1, -3.0), (1, 3.0))):
        m = k == f + 1
        pts[m, ax] = val
        pts[m, 1 - ax] = u[m]
        pts[m, 2] = v[m]
    return pts


def make_scan(rng, tb, n=1500, e=0.0, dur=0.1, imu_dt=0.005):
    """One scan over [tb, tb + dur]: raw [n, 4] float32 (LiDAR-frame xyz at each point's time, time [ms]), the pose table built from the
    trajectory shifted by e (a row at offset o holds the truth at tb + o + e), the prior (propagated) state at the scan end + e, and
    the exact posterior at the scan end."""
    tau = np.sort(rng.uniform(0.0, dur * 1000.0, n)).astype(np.float32)
    tau[:5] = 0.0                                   # points at the first row's time: no head row at shift 0
    w = room(rng, n)
    raw = np.zeros((n, 4), np.float32)
    for i in range(n):
        R, p, *_ = truth(tb + float(tau[i]) / 1000.0)
        raw[i, :3] = R_LI_TRUE.T @ (R.T @ (w[i] - p) - T_LI_TRUE)
    raw[:, 3] = tau
    offs = [0.0] + [o for o in np.arange(imu_dt, dur + 1e-12, imu_dt)]
    rows = []
    for o in offs:
        R, p, v, a, om = truth(tb + o + e)
        _, _, _, am, omm = truth(tb + o + e + imu_dt / 2)   # the rates over the next sample interval
        rows.append(np.r_[o, am, omm, v, p, R.reshape(9)])
    R, p, v, _, _ = truth(tb + dur + e)
    prior = (R, p, R_LI_TRUE, T_LI_TRUE, v)
    Rq, pq, *_ = truth(tb + dur)
    return dict(raw=raw, poses=np.array(rows), prior=prior, post=(Rq, pq, R_LI_TRUE, T_LI_TRUE))


def state_of(prior):
    s = np.zeros(36 + 576)
    s[0:9], s[9:12], s[12:21], s[21:24], s[24:27] = np.asarray(prior[0]).reshape(9), prior[1], np.asarray(prior[2]).reshape(9), prior[3], prior[4]
    return s
