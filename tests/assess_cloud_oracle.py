"""numpy restatement of the leaf records of liinit_assess_cloud (include/liinit_gpu.h, DESIGN §4d) from its per-point records, and a
reader of the assessment PCD (lidar_imu_init_b200/pcd.py write_assess). Test infrastructure."""
from __future__ import annotations

import numpy as np


def leaf_keys(w, leaf):
    """Leaf key of every placed point [N, 3] float32: floor(w / leaf) per axis (fp64 division), ((z - z0) ny + (y - y0)) nx + (x - x0)
    over the bounding box of the leaves."""
    c = np.floor(np.asarray(w, np.float32).astype(np.float64) / leaf).astype(np.int64)
    lo = c.min(axis=0)
    ext = c.max(axis=0) - lo + 1
    return ((c[:, 2] - lo[2]) * ext[1] + (c[:, 1] - lo[1])) * ext[0] + (c[:, 0] - lo[0])


def leaf_records(rec0, leaf):
    """[leaves, 8] float32 in ascending leaf key from the per-point records [N, 8] (stored order): fp64 sums over each leaf's points in
    stored order -- the centroid and the mean neighbour count over all of them, mean h and v over the valid ones (NaN when none is),
    the point count and the valid count -- divided in fp64 and stored as float32."""
    rec0 = np.asarray(rec0, np.float32)
    key = leaf_keys(rec0[:, :3], leaf)
    order = np.argsort(key, kind="stable")          # stable: stored order inside a leaf
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    counts = np.diff(np.r_[starts, len(ks)])
    nl = len(starts)
    leaf_of = np.repeat(np.arange(nl), counts)
    rank = np.arange(len(ks)) - starts[leaf_of]
    R = rec0[order].astype(np.float64)
    valid = R[:, 7] != 0
    S = np.zeros((nl, 6))
    nv = np.zeros(nl, np.int64)
    # one step per rank: every leaf adds its rank-th point, so each leaf's sums run left to right in stored order
    by_rank = np.argsort(rank, kind="stable")
    bounds = np.searchsorted(rank[by_rank], np.arange(int(rank.max()) + 2))
    for k in range(int(rank.max()) + 1):
        idx = by_rank[bounds[k]:bounds[k + 1]]
        L = leaf_of[idx]
        S[L, 0:3] += R[idx, 0:3]
        S[L, 5] += R[idx, 5]
        iv = idx[valid[idx]]
        Lv = leaf_of[iv]
        S[Lv, 3] += R[iv, 3]
        S[Lv, 4] += R[iv, 4]
        nv[Lv] += 1
    cnt = counts.astype(np.float64)
    out = np.zeros((nl, 8), np.float32)
    out[:, 0:3] = (S[:, 0:3] / cnt[:, None]).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        out[:, 3] = np.where(nv > 0, S[:, 3] / np.maximum(nv, 1), np.nan).astype(np.float32)
        out[:, 4] = np.where(nv > 0, S[:, 4] / np.maximum(nv, 1), np.nan).astype(np.float32)
    out[:, 5] = (S[:, 5] / cnt).astype(np.float32)
    out[:, 6] = counts.astype(np.float32)
    out[:, 7] = nv.astype(np.float32)
    return out


def read_assess_pcd(path):
    """(header {key: value string}, [n, 8] float32 records) of a binary assessment PCD."""
    data = open(path, "rb").read()
    end = data.index(b"DATA binary\n") + len(b"DATA binary\n")
    header = {}
    for line in data[:end].decode("ascii").splitlines():
        if line and not line.startswith("#"):
            k, _, v = line.partition(" ")
            header[k] = v
    n = int(header["POINTS"])
    body = np.frombuffer(data[end:], "<f4")
    assert body.size == 8 * n, (body.size, n)
    return header, body.reshape(n, 8)
