"""ctypes binding of tests/cpp/output_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU checker of the node's published clouds
(pointBodyToWorld on PointType records, publish_frame_body, PCL's VoxelGrid with downsample_all_data_, the effect compaction).
Compiled on first use into a per-user temporary directory, so that the tests also run from a read-only tree; the package never
loads it. Also a reader of the binary PCD files pcd_save writes, written from the PCD v0.7 format description."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "output_oracle.cpp")
_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
_L = None


def load():
    global _L
    if _L is not None:
        return _L
    src = open(SRC, "rb").read()
    d = os.path.join(tempfile.gettempdir(), f"liinit-output-oracle-{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    lib = os.path.join(d, f"liboutput_oracle_{hashlib.sha1(src).hexdigest()[:12]}.so")
    if not os.path.exists(lib):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
        tmp = lib + f".{os.getpid()}.tmp"
        subprocess.check_call([gxx, "-O3", "-std=c++14", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC])
        os.replace(tmp, lib)
    L = C.CDLL(lib)
    L.oo_to_world.restype = None
    L.oo_to_world.argtypes = [_f32p, C.c_int, _f64p, _f64p, _f64p, _f64p, _f32p]
    L.oo_frame_body.restype = None
    L.oo_frame_body.argtypes = [_f32p, C.c_int, _f32p]
    L.oo_voxel_grid.restype = C.c_int
    L.oo_voxel_grid.argtypes = [_f32p, C.c_int, C.c_float, _f32p]
    L.oo_effect.restype = C.c_int
    L.oo_effect.argtypes = [_f32p, _u8p, C.c_int, _f64p, _f64p, _f64p, _f64p, _f32p]
    _L = L
    return L


def _r(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 12)


def _pose(R, p, RLI, TLI):
    return [np.ascontiguousarray(x, np.float64).reshape(-1) for x in (R, p, RLI, TLI)]


def records(xyz, normals=None, intensity=None, curvature=None):
    """PointType records as the preprocess makes them: data[3] = 1, padding 0."""
    n = len(xyz)
    r = np.zeros((n, 12), np.float32)
    r[:, 0:3] = xyz
    r[:, 3] = 1.0
    if normals is not None:
        r[:, 4:7] = normals
    if intensity is not None:
        r[:, 8] = intensity
    if curvature is not None:
        r[:, 9] = curvature
    return r


def to_world(rec, R, p, RLI, TLI):
    a = _r(rec)
    out = np.zeros_like(a)
    load().oo_to_world(a, len(a), *_pose(R, p, RLI, TLI), out)
    return out


def frame_body(rec):
    a = _r(rec)
    out = np.zeros_like(a)
    load().oo_frame_body(a, len(a), out)
    return out


def voxel_grid(rec, leaf):
    a = _r(rec)
    out = np.zeros_like(a)
    m = load().oo_voxel_grid(a, len(a), float(leaf), out)
    assert m >= 0, "voxel grid overflow"
    return out[:m]


def effect(down_rec, selected, R, p, RLI, TLI):
    a = _r(down_rec)
    sel = np.ascontiguousarray(selected, np.uint8)
    out = np.zeros_like(a)
    m = load().oo_effect(a, sel, len(a), *_pose(R, p, RLI, TLI), out)
    return out[:m]


def read_pcd(path):
    """A binary PCD v0.7 file -> (header dict, structured array of its fields, raw record bytes [n, point size]). The fields are laid
    out as SIZE x COUNT bytes one after the other, in the order FIELDS lists them."""
    raw = open(path, "rb").read()
    hdr, pos = {}, 0
    while True:
        e = raw.index(b"\n", pos)
        line = raw[pos:e].decode("ascii")
        pos = e + 1
        if line.startswith("#"):
            continue
        k, *v = line.split()
        hdr[k] = v
        if k == "DATA":
            break
    assert hdr["DATA"] == ["binary"]
    names, sizes, types, counts = hdr["FIELDS"], [int(x) for x in hdr["SIZE"]], hdr["TYPE"], [int(x) for x in hdr["COUNT"]]
    assert len(names) == len(sizes) == len(types) == len(counts)
    kinds = {("F", 4): "<f4", ("F", 8): "<f8", ("U", 1): "u1", ("U", 2): "<u2", ("U", 4): "<u4", ("I", 1): "i1", ("I", 2): "<i2", ("I", 4): "<i4"}
    fields, off = [], 0
    for j, (nm, sz, ty, ct) in enumerate(zip(names, sizes, types, counts)):
        fields.append((nm if nm != "_" else f"_pad{j}", kinds[(ty, sz)], (ct,) if ct > 1 else ()))
        off += sz * ct
    n = int(hdr["POINTS"][0])
    assert int(hdr["WIDTH"][0]) * int(hdr["HEIGHT"][0]) == n
    body = raw[pos:]
    assert len(body) == n * off, (len(body), n, off)
    dt = np.dtype(fields)
    assert dt.itemsize == off
    return hdr, np.frombuffer(body, dt), np.frombuffer(body, np.uint8).reshape(n, off)


# ---- shared checks of the CPU and GPU tests -----------------------------------------------------------------------------------------
def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, want, what=""):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.size == 0:
        return
    bad = np.nonzero((bits(got) != bits(want)).reshape(len(got), -1).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(got)} records differ; first {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}"


def staged_records(g, attrs12, pointtype=True):
    """The staged (undistorted) cloud as PointType records: xyz from the device, normals / intensity / time from the uploaded
    PointType points (attrs12); an upload in another layout has no attributes (zeros)."""
    xyz = g.raw_points()
    a = np.asarray(attrs12, np.float32)
    if pointtype:
        return records(xyz, a[:, 4:7], a[:, 8], a[:, 9])
    return records(xyz, curvature=a[:, 9] if a.shape[1] > 9 else None)


def check_staged(g, staged, pose):
    """REGISTERED (also against liinit_raw_download_world) and BODY of the staged cloud."""
    reg = g.cloud(1, *pose)
    assert_bits(reg, to_world(staged, *pose), "REGISTERED")
    assert_bits(reg[:, 0:3], g.raw_world(*pose), "REGISTERED xyz vs raw_download_world")
    assert_bits(g.cloud(3), frame_body(staged), "BODY")
    return reg


def check_down(g, staged, leaf, pose):
    """The voxel grid of the staged cloud, then REGISTERED_DOWN. Returns the checker's feats_down_body records."""
    nd = g.raw_downsample(leaf)
    down = voxel_grid(staged, leaf)
    assert nd == len(down)
    assert_bits(g.scan_body(), down[:, 0:3], "voxel grid xyz")
    assert_bits(g.cloud(2, *pose), to_world(down, *pose), "REGISTERED_DOWN")
    return down


def check_effect(g, down, pose):
    """EFFECT after the last pass: the count of liinit_scan_download_effect, the records of the checker on the device's flags."""
    sel = g.scan_state()["selected"]
    ori, _ = g.scan_effect()
    eff = g.cloud(4, *pose)
    assert len(eff) == len(ori) == int(sel.astype(bool).sum())
    assert_bits(eff, effect(down, sel, *pose), "EFFECT")
    assert_bits(ori, down[sel.astype(bool), 0:3], "effect points")
    return len(eff)
