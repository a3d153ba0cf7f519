"""ctypes binding of tests/cpp/frame_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU checker of the cut-frame preprocess
(Preprocess::process_cut_frame_livox / _pcl2 restated literally). Compiled on first use into a per-user temporary directory, so that the
tests also run from a read-only tree; the package never loads it. Also the random messages the CPU and GPU tests share, and the
comparison of a product cut with the checker's."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

from lidar_imu_init_b200 import scenes
from lidar_imu_init_b200.capi import LIVOX_POINT

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_oracle.cpp")
_L = None
_vp = C.c_void_p


def load():
    global _L
    if _L is not None:
        return _L
    src = open(SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"liinit-frame-oracle-{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, f"libframe_oracle_{hashlib.sha1(src).hexdigest()[:12]}.so")
    if not os.path.exists(lib):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        tmp = lib + f".{os.getpid()}.tmp"
        subprocess.check_call([gxx, "-O2", "-std=c++14", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC])
        os.replace(tmp, lib)
    L = C.CDLL(lib)
    tail = [_vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp]
    L.frame_oracle_livox.restype = C.c_int
    L.frame_oracle_livox.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, C.c_double] + tail
    L.frame_oracle_pcl2.restype = C.c_int
    L.frame_oracle_pcl2.argtypes = [_vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, C.c_double] + tail
    _L = L
    return L


def _p(a):
    return a.ctypes.data_as(_vp)


def _run(fn, args, n):
    cap_sub = 260
    pts = np.zeros((max(n, 1), 5), np.float32)
    sn = np.zeros(cap_sub, np.int32)
    tb = np.zeros(cap_sub, np.float64)
    en = np.zeros(cap_sub, np.float32)
    k, m = C.c_int(0), C.c_int(0)
    rc = fn(*args, _p(pts), len(pts), _p(sn), _p(tb), _p(en), cap_sub, C.byref(k), C.byref(m))
    if rc != 0:
        return None
    subs, o = [], 0
    for i in range(k.value):
        subs.append(dict(pts=pts[o:o + sn[i]].copy(), n=int(sn[i]), t_beg=float(tb[i]), end_ms=np.float32(en[i])))
        o += sn[i]
    return subs


def cut_livox(records, N_SCANS=6, blind=0.01, point_filter_num=1, required_frame_num=1, scan_count=0, stamp=0.0):
    """process_cut_frame_livox on a structured array of Livox records: list of sub-frames {pts [n, 5] (x, y, z, intensity, curvature),
    n, t_beg [s], end_ms}."""
    a = np.ascontiguousarray(records)
    return _run(load().frame_oracle_livox, (_p(a), a.dtype.itemsize, len(a), N_SCANS, blind, point_filter_num, required_frame_num, scan_count,
                                             stamp), len(a))


def cut_pcl2(data, layout, n, lidar_type, N_SCANS=16, blind=0.01, point_filter_num=1, required_frame_num=1, scan_count=0, stamp=0.0):
    """process_cut_frame_pcl2; None when the rotation model meets a ring >= 128."""
    a = np.ascontiguousarray(data, np.uint8)
    offs = np.array([layout.get(f, -1) for f in ("off_x", "off_y", "off_z", "off_intensity", "off_time", "off_ring")], np.int32)
    return _run(load().frame_oracle_pcl2, (_p(a), layout["point_step"], _p(offs), lidar_type, n, N_SCANS, blind, point_filter_num,
                                            required_frame_num, scan_count, stamp), n)


# ---- random messages ---------------------------------------------------------------------------------------------------------
def _pose_at(t):
    """a LiDAR yawing at 0.3 rad/s and swaying along x inside the 15 m box"""
    t = np.atleast_1d(np.asarray(t, float))
    c, s = np.cos(0.3 * t), np.sin(0.3 * t)
    R = np.zeros((len(t), 3, 3))
    R[:, 0, 0], R[:, 0, 1], R[:, 1, 0], R[:, 1, 1], R[:, 2, 2] = c, -s, s, c, 1.0
    p = np.stack([7.0 + 0.5 * np.sin(t), np.full_like(t, 7.5), np.full_like(t, 1.5)], 1)
    return R, p


_SCENE = None


LIVOX_SEED = 2024   # the random messages of the GPU test; the CPU test on the emulated library takes the first of them


def random_livox(rng: np.random.Generator):
    """(records, params) over the space the tests cover: point_filter_num 1-5, N_SCANS 4 / 6, required_frame_num 1-6 on both sides of
    the scan_count rule, degenerate valid sizes V in {0, 1, 2, R..2R-1, 2R}, ties, offsets above 2^24 ns, noise tags, bad lines,
    zero points and duplicates."""
    global _SCENE
    if _SCENE is None:
        _SCENE = scenes.box_scene(15.0, 15.0, 6.0)
    prm = dict(N_SCANS=int(rng.choice([4, 6])), blind=float(rng.choice([0.0, 0.01, 0.5, 2.0])), point_filter_num=int(rng.integers(1, 6)),
               required_frame_num=int(rng.integers(1, 7)), scan_count=int(rng.integers(0, 10)), stamp=float(rng.uniform(0.0, 2000.0)))
    R = prm["required_frame_num"] if prm["scan_count"] >= 5 else 1
    kind = rng.uniform()
    if kind < 0.3:
        # degenerate sizes: every record valid and taken, distinct, outside the blind zone -> V = n - 1
        prm.update(point_filter_num=1, blind=float(rng.choice([0.0, 0.01])))
        V = int(rng.choice([0, 1, 2, R, 2 * R - 1, 2 * R, int(rng.integers(R, 2 * R + 1))]))
        n = V + 1
        m = np.zeros(n, LIVOX_POINT)
        m["x"] = rng.uniform(1.0, 20.0, n)
        m["y"] = rng.uniform(-5.0, 5.0, n)
        m["z"] = rng.uniform(-1.0, 1.0, n)
        m["offset_time"] = rng.integers(0, 100_000_000, n)
        m["reflectivity"] = rng.integers(0, 256, n)
        m["line"] = rng.integers(0, prm["N_SCANS"], n)
        return m, prm
    n = int(rng.integers(50, 3000))
    m = scenes.livox_message(_SCENE, _pose_at, prm["stamp"], n, seed=int(rng.integers(1 << 30)), n_scans=prm["N_SCANS"],
                             noise_frac=float(rng.choice([0.0, 0.05])), bad_line_frac=float(rng.choice([0.0, 0.05])),
                             zero_frac=float(rng.choice([0.0, 0.05])), dup_frac=float(rng.choice([0.0, 0.1])),
                             tie_frac=float(rng.choice([0.0, 0.2])), aligned=bool(rng.integers(2)))
    return m, prm


def f32_ulps(a, b):
    """distance in float32 units in the last place, elementwise"""
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def _rows(p4):
    r = np.ascontiguousarray(p4).view(np.uint32)
    return r[np.lexsort(r.T[::-1])]


def compare(got, got_pts, want, curv_tol_ms=0.0):
    """got: the product's sub-frame dicts, got_pts: their downloads [n, 12]; want: the checker's sub-frames. With curv_tol_ms == 0
    everything must be bit-equal. With curv_tol_ms > 0 (the rotation model, see YAW_TOL_MS) every sub-frame must hold the same
    multiset of points (x, y, z, intensity) as the checker's, with curvatures, end_ms and t_beg within that tolerance position by
    position; points whose times are that close may come out of the sort in another order inside a sub-frame. Returns (curvatures
    not bit-equal, positions holding another point)."""
    assert len(got) == len(want), (len(got), len(want))
    off = moved = 0
    for g, p12, w in zip(got, got_pts, want):
        assert g["n"] == w["n"] and len(p12) == w["n"]
        p5 = np.stack([p12[:, 0], p12[:, 1], p12[:, 2], p12[:, 8], p12[:, 9]], 1)
        a, b = np.ascontiguousarray(p5[:, 0:4]).view(np.uint32), np.ascontiguousarray(w["pts"][:, 0:4]).view(np.uint32)
        if curv_tol_ms == 0.0:
            np.testing.assert_array_equal(a, b)
        else:
            np.testing.assert_array_equal(_rows(p5[:, 0:4]), _rows(w["pts"][:, 0:4]))   # same composition of this sub-frame
        moved += int((a != b).any(axis=1).sum())
        # an absolute tolerance, not one ulp of the re-timed value: a boundary time one ulp off shifts last_frame_end_time, and with
        # it every re-timed curvature of the later sub-frames, by that absolute amount (YAW_TOL_MS)
        d = np.abs(p5[:, 4].astype(np.float64) - w["pts"][:, 4])
        assert d.max(initial=0.0) <= curv_tol_ms, d.max()
        off += int((p5[:, 4].view(np.uint32) != w["pts"][:, 4].view(np.uint32)).sum())
        assert abs(float(g["end_ms"]) - float(w["end_ms"])) <= curv_tol_ms
        assert abs(g["t_beg"] - w["t_beg"]) <= curv_tol_ms * len(want) * 1e-3
        assert (p12[:, 3] == 1.0).all() and (p12[:, 4:8] == 0.0).all() and (p12[:, 10:12] == 0.0).all()
    return off, moved


# The rotation model's offset times lie below 256 ms, where one float32 ulp is 2^-16 ms. The reference takes atan2 of two floats,
# i.e. the C library's atan2f, which is not correctly rounded (glibc 2.39: it differs from the correctly rounded value for about 16%
# of random arguments); the device rounds a double atan2 once. A time may therefore be one ulp off, and the re-timing adds one more
# rounding.
YAW_TOL_MS = 2.0 ** -15
