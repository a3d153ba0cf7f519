"""numpy restatement of the map assessment (DESIGN §4d, include/liinit_gpu.h liinit_assess_*): placement, fixed-radius neighbourhoods by
brute force, moments, entropy and plane variance, and the totals. Test infrastructure: the device's values are checked against it."""
from __future__ import annotations

import math

import numpy as np

H0 = 3.0 * math.log(2.0 * math.pi * math.e)


def body_to_world(body, R, p, RLI, TLI):
    """li_body_to_world (csrc/common.cuh) for [n, 3] float32 points: fp64 without contraction, left-to-right sums, float32 store."""
    b = np.asarray(body, np.float32).astype(np.float64)
    R, RLI = np.asarray(R, float).reshape(3, 3), np.asarray(RLI, float).reshape(3, 3)
    p, TLI = np.asarray(p, float).reshape(3), np.asarray(TLI, float).reshape(3)
    t = [((RLI[a, 0] * b[:, 0] + RLI[a, 1] * b[:, 1]) + RLI[a, 2] * b[:, 2]) + TLI[a] for a in range(3)]
    g = [((R[a, 0] * t[0] + R[a, 1] * t[1]) + R[a, 2] * t[2]) + p[a] for a in range(3)]
    return np.stack(g, axis=1).astype(np.float32)


def place(scans, R_LI=None, T_LI=None):
    """scans: [(body [n, 3] float32, rot_end, pos_end, R_LI, T_LI)] in stored order. With R_LI / T_LI None every scan uses its own
    extrinsic (as-run). Returns the placed [N, 3] float32 cloud in stored order."""
    out = []
    for body, R, p, rli, tli in scans:
        out.append(body_to_world(body, R, p, rli if R_LI is None else R_LI, tli if T_LI is None else T_LI))
    return np.concatenate(out) if out else np.zeros((0, 3), np.float32)


def auto_stride(n, max_queries=2_000_000):
    return max(1, -(-n // max_queries))


def neighbour_d2(w, k_idx):
    """d2 of every stored point to each query, [len(k_idx), N] float64, in the definition's association."""
    W = np.asarray(w, np.float32).astype(np.float64)
    Q = W[k_idx]
    dx = W[None, :, 0] - Q[:, None, 0]
    dy = W[None, :, 1] - Q[:, None, 1]
    dz = W[None, :, 2] - Q[:, None, 2]
    return (dx * dx + dy * dy) + dz * dz, dx, dy, dz


def evaluate(w, radius=0.3, min_neighbors=10, stride=0, chunk=256):
    """Per-query (n, h, v) and the totals of one evaluation of the placed cloud w [N, 3] float32."""
    N = len(w)
    s = stride or auto_stride(N)
    k_all = np.arange(0, N, s)
    r2 = radius * radius
    n_out = np.zeros(len(k_all), np.int64)
    h_out = np.full(len(k_all), np.nan)
    v_out = np.full(len(k_all), np.nan)
    for c0 in range(0, len(k_all), chunk):
        ks = k_all[c0:c0 + chunk]
        d2, dx, dy, dz = neighbour_d2(w, ks)
        m = d2 <= r2
        for j in range(len(ks)):
            sel = m[j]
            n = int(sel.sum())
            n_out[c0 + j] = n
            if n < min_neighbors:
                continue
            x, y, z = dx[j, sel], dy[j, sel], dz[j, sel]
            mx, my, mz = x.sum() / n, y.sum() / n, z.sum() / n
            cxx, cxy, cxz = (x * x).sum() / n - mx * mx, (x * y).sum() / n - mx * my, (x * z).sum() / n - mx * mz
            cyy, cyz, czz = (y * y).sum() / n - my * my, (y * z).sum() / n - my * mz, (z * z).sum() / n - mz * mz
            det = cxx * (cyy * czz - cyz * cyz) - cxy * (cxy * czz - cyz * cxz) + cxz * (cxy * cyz - cyy * cxz)
            if det > 0:
                h_out[c0 + j] = 0.5 * (H0 + math.log(det))
                v_out[c0 + j] = np.linalg.eigvalsh(np.array([[cxx, cxy, cxz], [cxy, cyy, cyz], [cxz, cyz, czz]]))[0]
    valid = ~np.isnan(h_out)
    sparse = n_out < min_neighbors
    tot = dict(queries=len(k_all), stride=s, valid=int(valid.sum()), sparse=int(sparse.sum()), degenerate=int((~valid & ~sparse).sum()),
               mme=float(h_out[valid].mean()) if valid.any() else math.nan, mpv=float(v_out[valid].mean()) if valid.any() else math.nan)
    return n_out, h_out, v_out, tot


def evaluate_sample(w, tree, k_idx, radius=0.3, min_neighbors=10):
    """(n, h, v) of the queries k_idx of a large placed cloud: the candidates come from a kd-tree over w (float64) at radius + 1 mm,
    the definitions are then applied to them exactly as in evaluate()."""
    W = np.asarray(w, np.float32).astype(np.float64)
    r2 = radius * radius
    n_out = np.zeros(len(k_idx), np.int64)
    h_out = np.full(len(k_idx), np.nan)
    v_out = np.full(len(k_idx), np.nan)
    for j, (k, cand) in enumerate(zip(k_idx, tree.query_ball_point(W[k_idx], radius + 1e-3))):
        C = W[np.sort(np.asarray(cand, np.int64))]
        dx, dy, dz = C[:, 0] - W[k, 0], C[:, 1] - W[k, 1], C[:, 2] - W[k, 2]
        sel = ((dx * dx + dy * dy) + dz * dz) <= r2
        n = int(sel.sum())
        n_out[j] = n
        if n < min_neighbors:
            continue
        x, y, z = dx[sel], dy[sel], dz[sel]
        mx, my, mz = x.sum() / n, y.sum() / n, z.sum() / n
        cxx, cxy, cxz = (x * x).sum() / n - mx * mx, (x * y).sum() / n - mx * my, (x * z).sum() / n - mx * mz
        cyy, cyz, czz = (y * y).sum() / n - my * my, (y * z).sum() / n - my * mz, (z * z).sum() / n - mz * mz
        det = cxx * (cyy * czz - cyz * cyz) - cxy * (cxy * czz - cyz * cxz) + cxz * (cxy * cyz - cyy * cxz)
        if det > 0:
            h_out[j] = 0.5 * (H0 + math.log(det))
            v_out[j] = np.linalg.eigvalsh(np.array([[cxx, cxy, cxz], [cxy, cyy, cyz], [cxz, cyz, czz]]))[0]
    return n_out, h_out, v_out


def near_boundary(w, radius, stride, tol=1e-9):
    """Queries with some stored point whose distance is within tol of the radius (excluded from the kd-tree comparison)."""
    k_all = np.arange(0, len(w), stride)
    out = np.zeros(len(k_all), bool)
    for c0 in range(0, len(k_all), 256):
        d2, *_ = neighbour_d2(w, k_all[c0:c0 + 256])
        out[c0:c0 + 256] = (np.abs(np.sqrt(d2) - radius) <= tol).any(axis=1)
    return out


def rot_exp(axis_angle):
    """Exp of so(3) (Rodrigues)."""
    v = np.asarray(axis_angle, float)
    th = np.linalg.norm(v)
    if th == 0:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K
