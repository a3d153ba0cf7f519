"""numpy restatement of the timed assessment's placement (DESIGN §4d, include/liinit_gpu.h liinit_assess_evaluate_timed): the IMU
undistortion of k_undistort_imu redone at a lag shift towards the carried scan-end state, then li_body_to_world. fp64 without
contraction, the C source's association, float32 stores; sin and cos from Python's math (the libm the emulated kernels call).
Test infrastructure: the device's placed points are checked against it."""
from __future__ import annotations

import math

import numpy as np

from assess_oracle import body_to_world

D = 22   # Pose6D doubles: offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]


def so3_exp_dt(w, dt):
    """li_so3_exp_dt for per-point angular velocities w [m, 3] and times dt [m]: [m, 9]."""
    w = np.asarray(w, float).reshape(-1, 3)
    dt = np.broadcast_to(np.asarray(dt, float), (len(w),))
    n = np.sqrt(w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1] + w[:, 2] * w[:, 2])
    R = np.zeros((len(w), 9))
    R[:, 0] = R[:, 4] = R[:, 8] = 1.0
    on = n > 0.0000001
    if not on.any():
        return R
    nn = np.where(on, n, 1.0)
    r0, r1, r2 = w[:, 0] / nn, w[:, 1] / nn, w[:, 2] / nn
    a = n * dt
    s = np.array([math.sin(x) for x in a])
    c = 1.0 - np.array([math.cos(x) for x in a])
    z = np.zeros(len(w))
    K = [z, -r2, r1, r2, z, -r0, -r1, r0, z]
    KK = [None] * 9
    for i in range(3):
        for j in range(3):
            KK[3 * i + j] = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j]
    out = R.copy()
    for i in range(9):
        out[:, i] = R[:, i] + s * K[i] + c * KK[i]
    return np.where(on[:, None], out, R)


def _mat(A, B):
    """row-major 3x3 products, per point: (A[3a] B[b] + A[3a+1] B[3+b]) + A[3a+2] B[6+b]"""
    return np.stack([A[:, 3 * a] * B[:, b] + A[:, 3 * a + 1] * B[:, 3 + b] + A[:, 3 * a + 2] * B[:, 6 + b] for a in range(3) for b in range(3)], 1)


def scan_end(prior, poses, delta):
    """k_at_scan_end: (R_e [9], p_e [3]) of a scan for lag shift delta; prior = (rot, pos, R_LI, T_LI, vel)."""
    R, p = np.asarray(prior[0], float).reshape(9), np.asarray(prior[1], float).reshape(3)
    if delta == 0.0:
        return R, p
    last = np.asarray(poses, float).reshape(-1, D)[-1]
    X = so3_exp_dt(last[4:7][None], delta)
    Re = _mat(R[None], X)[0]
    v = np.asarray(prior[4], float).reshape(3)
    pe = np.array([p[a] + v[a] * delta + 0.5 * last[1 + a] * delta * delta for a in range(3)])
    return Re, pe


def undistort(raw, poses, Re, pe, RLI, TLI, delta):
    """k_at_place's undistortion of raw [n, 4] float32 (xyz, time ms) of one scan: [n, 3] float32."""
    P = np.asarray(poses, float).reshape(-1, D)
    raw = np.asarray(raw, np.float32)
    t0 = raw[:, 3].astype(np.float64) / 1000.0
    t = t0 + delta if delta != 0.0 else t0
    head = np.full(len(raw), -1)
    for k in range(len(P) - 1):
        head = np.where(t > P[k, 0], k, head)
    if delta != 0.0:
        head = np.where(head < 0, 0, head)
    out = raw[:, :3].copy()
    m = head >= 0
    if not m.any():
        return out
    h = P[head[m]]
    tm = t[m]
    dt = tm - h[:, 0]
    E = so3_exp_dt(h[:, 4:7], dt)
    Ri = _mat(h[:, 13:22], E)
    Pi = [h[:, 10 + a] + h[:, 7 + a] * dt + 0.5 * h[:, 1 + a] * dt * dt for a in range(3)]
    x, y, z = (raw[m, a].astype(np.float64) for a in range(3))
    RLI, TLI = np.asarray(RLI, float).reshape(9), np.asarray(TLI, float).reshape(3)
    Rs, ps = np.asarray(Re, float).reshape(9), np.asarray(pe, float).reshape(3)
    q = [RLI[3 * a] * x + RLI[3 * a + 1] * y + RLI[3 * a + 2] * z + TLI[a] for a in range(3)]
    u = [Ri[:, 3 * a] * q[0] + Ri[:, 3 * a + 1] * q[1] + Ri[:, 3 * a + 2] * q[2] + Pi[a] - ps[a] for a in range(3)]
    v = [Rs[a] * u[0] + Rs[3 + a] * u[1] + Rs[6 + a] * u[2] - TLI[a] for a in range(3)]
    w = [RLI[a] * v[0] + RLI[3 + a] * v[1] + RLI[6 + a] * v[2] for a in range(3)]
    out[m] = np.stack(w, 1).astype(np.float32)
    return out


def place_timed(scans, delta=0.0, R_LI=None, T_LI=None):
    """scans: [dict(stored=[n, 3] float32 as appended, post=(rot, pos, R_LI, T_LI), and for a timed scan raw=[n, 4] float32,
    poses=[npose, 22], prior=(rot, pos, R_LI, T_LI, vel))] in stored order. R_LI / T_LI None: as-run (the prior extrinsic for the
    undistortion, the posterior one for the placement). Returns the placed [N, 3] float32 cloud."""
    out = []
    for s in scans:
        R, p, rli, tli = s["post"]
        body = s["stored"]
        if s.get("raw") is not None:
            Re, pe = scan_end(s["prior"], s["poses"], delta)
            u_rli = s["prior"][2] if R_LI is None else R_LI
            u_tli = s["prior"][3] if T_LI is None else T_LI
            body = undistort(s["raw"], s["poses"], Re, pe, u_rli, u_tli, delta)
        out.append(body_to_world(body, R, p, rli if R_LI is None else R_LI, tli if T_LI is None else T_LI))
    return np.concatenate(out)
