"""Deterministic synthetic scenes, scans and poses (SURVEY.md section 8d).

The reference ships no input data (no rosbag, SURVEY.md section 4), so every test and
bench input is generated here from a seed:

* Scene S(M): axis-aligned "warehouse" box L x W x H with optional interior slab
  walls. Map points: one per ``ds`` cell on every surface (cell centre +
  U(-0.4 ds, 0.4 ds) in-plane, N(0, sigma^2) out-of-plane) -- the density of the
  reference's steady-state map (<= 1 point per filter_size_map voxel,
  ikd_Tree.cpp:381-456).
* Scan(N): N points uniform on the surfaces within ``det_range`` of the sensor and
  beyond ``blind``, N(0, sigma^2) range noise, expressed in the LiDAR body frame of a
  ground-truth pose; optionally a fraction of "open-air" points with no map
  neighbours (exercises the reject path of laserMapping.cpp:981-984).

Everything is numpy (host side); float32 outputs, double poses.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class Rect:
    o: np.ndarray  # origin (3,)
    u: np.ndarray  # unit edge 1
    v: np.ndarray  # unit edge 2
    a: float       # length along u
    b: float       # length along v

    @property
    def n(self):
        return np.cross(self.u, self.v)

    @property
    def area(self):
        return self.a * self.b


@dataclass
class Scene:
    rects: list = field(default_factory=list)
    L: float = 0.0
    W: float = 0.0
    H: float = 0.0

    @property
    def area(self):
        return float(sum(r.area for r in self.rects))


def box_scene(L: float, W: float, H: float, n_slabs_x: int = 0, n_slabs_y: int = 0) -> Scene:
    """Box [0,L]x[0,W]x[0,H] (floor, ceiling, 4 walls) + interior slab walls.

    Slabs are full-height walls spanning 60 % of the box, alternating sides, at
    evenly spaced x (normal along x) or y (normal along y)."""
    ex, ey, ez = np.eye(3)
    z0 = np.zeros(3)
    rs = [
        Rect(z0, ex, ey, L, W),                         # floor z=0
        Rect(np.array([0, 0, H], float), ex, ey, L, W),  # ceiling
        Rect(z0, ex, ez, L, H),                         # wall y=0
        Rect(np.array([0, W, 0], float), ex, ez, L, H),  # wall y=W
        Rect(z0, ey, ez, W, H),                         # wall x=0
        Rect(np.array([L, 0, 0], float), ey, ez, W, H),  # wall x=L
    ]
    for i in range(n_slabs_x):
        x = L * (i + 1) / (n_slabs_x + 1)
        y0 = 0.0 if i % 2 == 0 else 0.4 * W
        rs.append(Rect(np.array([x, y0, 0], float), ey, ez, 0.6 * W, H))
    for i in range(n_slabs_y):
        y = W * (i + 1) / (n_slabs_y + 1)
        x0 = 0.0 if i % 2 == 0 else 0.4 * L
        rs.append(Rect(np.array([x0, y, 0], float), ex, ez, 0.6 * L, H))
    return Scene(rs, L, W, H)


def scene_for_points(M: int, ds: float = 0.15, aspect=(300.0, 160.0, 20.0)) -> Scene:
    """Box with the given aspect ratio scaled so its surfaces hold >= M ds-cells (about 2 % more)."""
    L, W, H = aspect
    area0 = 2 * (L * W + L * H + W * H)
    s = np.sqrt(M * ds * ds * 1.02 / area0)

    def cells(sc):
        return sum(max(int(np.floor(r.a / ds)), 1) * max(int(np.floor(r.b / ds)), 1) for r in sc.rects)

    scene = box_scene(L * s, W * s, H * s)
    while cells(scene) < M:   # small scenes lose whole rows to the floor(); grow until enough
        s *= 1.01
        scene = box_scene(L * s, W * s, H * s)
    return scene


def map_points(scene: Scene, ds: float, M: int | None = None, seed: int = 1, sigma: float = 0.01,
               jitter: float = 0.4) -> np.ndarray:
    """One jittered point per ds x ds surface cell; thinned uniformly to exactly M if given."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for r in scene.rects:
        na, nb = max(int(np.floor(r.a / ds)), 1), max(int(np.floor(r.b / ds)), 1)
        ia, ib = np.meshgrid(np.arange(na), np.arange(nb), indexing="ij")
        s = (ia.ravel() + 0.5 + rng.uniform(-jitter, jitter, na * nb)) * ds
        t = (ib.ravel() + 0.5 + rng.uniform(-jitter, jitter, na * nb)) * ds
        w = rng.normal(0.0, sigma, na * nb) if sigma > 0 else np.zeros(na * nb)
        out.append(r.o[None, :] + s[:, None] * r.u[None, :] + t[:, None] * r.v[None, :] + w[:, None] * r.n[None, :])
    pts = np.concatenate(out, 0)
    if M is not None:
        if len(pts) < M:
            raise ValueError(f"scene holds {len(pts)} cells < M={M}")
        keep = rng.permutation(len(pts))[:M]
        keep.sort()
        pts = pts[keep]
    return np.ascontiguousarray(pts, dtype=np.float32)


def rot_from_rpy(r, p, y):
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def so3_exp(w):
    w = np.asarray(w, float)
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


@dataclass
class Pose:
    rot_end: np.ndarray
    pos_end: np.ndarray
    R_LI: np.ndarray
    T_LI: np.ndarray

    def copy(self):
        return Pose(self.rot_end.copy(), self.pos_end.copy(), self.R_LI.copy(), self.T_LI.copy())


def identity_extrinsic():
    return np.eye(3), np.zeros(3)


def sample_extrinsic():
    """R_LI ~ Rz(88 deg) * small, T_LI from the reference's sample result
    (result/Initialization_result.txt:2-3)."""
    R = rot_from_rpy(np.deg2rad(-0.94), np.deg2rad(-0.32), np.deg2rad(88.13))
    T = np.array([-0.0197, 0.0215, 0.1702])
    return R, T


def perturb_pose(pose: Pose, seed: int, dtheta_deg: float = 0.5, dpos: float = 0.05) -> Pose:
    """ground truth boxplus delta: delta-theta on the dtheta sphere, delta-p on the dpos sphere."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = rng.normal(size=3)
    a *= np.deg2rad(dtheta_deg) / np.linalg.norm(a)
    t = rng.normal(size=3)
    t *= dpos / np.linalg.norm(t)
    return Pose(pose.rot_end @ so3_exp(a), pose.pos_end + t, pose.R_LI.copy(), pose.T_LI.copy())


def scan_points(scene: Scene, pose: Pose, N: int, seed: int = 2, det_range: float = 450.0, blind: float = 2.0,
                sigma: float = 0.01, open_air_frac: float = 0.0, order: str = "voxel", leaf: float = 0.05) -> np.ndarray:
    """N body-frame points (float32 [N,3]).

    order: 'voxel'  = sorted by (z,y,x) leaf cell in the body frame, the order PCL's
                      VoxelGrid emits (laserMapping.cpp:917-918) -- what the reference loop sees;
           'shuffle' = random order; 'asis' = generation order (by surface)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    # LiDAR position in world: p_w = R_end (R_LI p_b + T_LI) + pos  => lidar origin:
    sensor = pose.rot_end @ pose.T_LI + pose.pos_end
    areas = np.array([r.area for r in scene.rects])
    cdf = np.cumsum(areas) / areas.sum()
    n_air = int(round(N * open_air_frac))
    n_surf = N - n_air
    got = []
    need = n_surf
    guard = 0
    while need > 0:
        guard += 1
        if guard > 200:
            raise RuntimeError("could not sample enough in-range surface points")
        k = int(need * 1.3) + 16
        ri = np.searchsorted(cdf, rng.uniform(size=k))
        s = rng.uniform(size=k)
        t = rng.uniform(size=k)
        O = np.stack([scene.rects[i].o for i in range(len(areas))])[ri]
        U = np.stack([scene.rects[i].u * scene.rects[i].a for i in range(len(areas))])[ri]
        V = np.stack([scene.rects[i].v * scene.rects[i].b for i in range(len(areas))])[ri]
        P = O + s[:, None] * U + t[:, None] * V
        d = np.linalg.norm(P - sensor[None, :], axis=1)
        ok = (d > blind) & (d < det_range)
        P, d = P[ok], d[ok]
        if sigma > 0:
            ray = (P - sensor[None, :]) / d[:, None]
            P = P + ray * rng.normal(0.0, sigma, len(P))[:, None]
        got.append(P[:need])
        need -= len(got[-1])
    Pw = np.concatenate(got, 0) if got else np.zeros((0, 3))
    if n_air > 0:
        # points floating outside the building, >= 3 m beyond the x=L wall => no map
        # neighbour within sqrt(5) m (the kNN radius, ikd_Tree.cpp:842)
        A = np.stack([scene.L + 3.0 + 7.0 * rng.uniform(size=n_air), scene.W * rng.uniform(size=n_air),
                      scene.H * rng.uniform(size=n_air)], 1)
        Pw = np.concatenate([Pw, A], 0)
    # world -> body: p_b = R_LI^T (R_end^T (p_w - pos) - T_LI)
    Pb = (pose.R_LI.T @ (pose.rot_end.T @ (Pw - pose.pos_end[None, :]).T - pose.T_LI[:, None])).T
    if order == "voxel":
        ijk = np.floor(Pb / leaf).astype(np.int64)
        ijk -= ijk.min(0, keepdims=True)
        dims = ijk.max(0) + 1
        lin = ijk[:, 0] + dims[0] * (ijk[:, 1] + dims[1] * ijk[:, 2])
        Pb = Pb[np.argsort(lin, kind="stable")]
    elif order == "morton":
        # Z-order of 0.6 m body-frame cells: what a spatial sort at upload would produce
        ijk = np.floor(Pb / 0.6).astype(np.int64)
        ijk -= ijk.min(0, keepdims=True)
        def spread(v):
            v = v & 0x3ff
            v = (v | (v << 16)) & 0x030000ff
            v = (v | (v << 8)) & 0x0300f00f
            v = (v | (v << 4)) & 0x030c30c3
            v = (v | (v << 2)) & 0x09249249
            return v
        key = spread(ijk[:, 0]) | (spread(ijk[:, 1]) << 1) | (spread(ijk[:, 2]) << 2)
        Pb = Pb[np.argsort(key, kind="stable")]
    elif order == "shuffle":
        Pb = Pb[rng.permutation(len(Pb))]
    elif order != "asis":
        raise ValueError(order)
    return np.ascontiguousarray(Pb, dtype=np.float32)


def timed_scan_points(scene: Scene, pose_at, t_beg: float, dur: float, N: int, seed: int = 2, det_range: float = 450.0,
                      blind: float = 2.0, sigma: float = 0.01) -> np.ndarray:
    """N raw points of a moving LiDAR as the driver delivers them: float32 [N, 12] in the pcl::PointXYZINormal layout
    (x, y, z at 0:3, intensity at 8, curvature at 9), ascending in time.

    Every point gets a time t uniform in [t_beg, t_beg + dur] and is expressed in the LiDAR frame of the pose at t.
    curvature = (t - t_beg) in milliseconds, the per-point offset the undistortion reads (src/preprocess.cpp).
    pose_at(t) -> (R [n,3,3], p [n,3]): the LiDAR frame's orientation and origin in the world at the times t [n].
    Surface sampling, range gate and range noise as in scan_points."""
    rng = np.random.Generator(np.random.PCG64(seed))
    areas = np.array([r.area for r in scene.rects])
    cdf = np.cumsum(areas) / areas.sum()
    O_all = np.stack([r.o for r in scene.rects])
    U_all = np.stack([r.u * r.a for r in scene.rects])
    V_all = np.stack([r.v * r.b for r in scene.rects])
    got_p, got_t = [], []
    need = N
    guard = 0
    while need > 0:
        guard += 1
        if guard > 200:
            raise RuntimeError("could not sample enough in-range surface points")
        k = int(need * 1.3) + 16
        t = t_beg + dur * rng.uniform(size=k)
        R, sensor = pose_at(t)
        ri = np.searchsorted(cdf, rng.uniform(size=k))
        s = rng.uniform(size=k)
        u = rng.uniform(size=k)
        P = O_all[ri] + s[:, None] * U_all[ri] + u[:, None] * V_all[ri]
        d = np.linalg.norm(P - sensor, axis=1)
        ok = (d > blind) & (d < det_range)
        if sigma > 0:
            ray = (P - sensor) / d[:, None]
            P = P + ray * rng.normal(0.0, sigma, k)[:, None]
        # world -> LiDAR frame at the point's own time: R^T (p_w - p)
        B = np.einsum("nji,nj->ni", R[ok], P[ok] - sensor[ok])
        got_p.append(B[:need])
        got_t.append(t[ok][:need])
        need -= len(got_p[-1])
    B = np.concatenate(got_p, 0)
    t = np.concatenate(got_t, 0)
    o = np.argsort(t, kind="stable")
    out = np.zeros((N, 12), np.float32)
    out[:, 0:3] = B[o]
    out[:, 3] = 1.0
    out[:, 8] = rng.uniform(0.0, 255.0, N)
    out[:, 9] = (t[o] - t_beg) * 1000.0
    return out


def default_sensor_pose(scene: Scene, R_LI=None, T_LI=None, yaw_deg: float = 20.0) -> Pose:
    """Ground-truth pose: sensor 1.5 m above the floor near the scene centre, mild attitude."""
    if R_LI is None:
        R_LI, T_LI = identity_extrinsic()
    R = rot_from_rpy(np.deg2rad(1.5), np.deg2rad(-2.0), np.deg2rad(yaw_deg))
    pos = np.array([0.47 * scene.L, 0.53 * scene.W, min(1.5, 0.5 * scene.H)])
    return Pose(R, pos, np.asarray(R_LI, float), np.asarray(T_LI, float))


# ---- named configurations of BASELINE.json ---------------------------------
CONFIGS = {
    # name: (N scan pts, M map pts, ds, det_range)
    "C1": (1_000, 10_000, 0.15, 450.0),
    "C2": (240_000, 5_000_000, 0.15, 450.0),
    "C3": (130_000, 10_000_000, 0.15, 100.0),
    "C4": (260_000, 5_000_000, 0.15, 150.0),
    "C5": (2_000_000, 5_000_000, 0.15, 450.0),
}


def make_config(name: str, seed: int = 1, imu_en: bool = False, open_air_frac: float = 0.01, order: str = "voxel",
                N: int | None = None, M: int | None = None):
    """Returns dict(scene, map_xyz, body_xyz, pose_gt, pose_init, ds, imu_en)."""
    n0, m0, ds, det = CONFIGS[name]
    N = n0 if N is None else N
    M = m0 if M is None else M
    if name == "C1":
        # noise-free planar scene: floor + two walls dominate; exact residuals (SURVEY 8d)
        scene = box_scene(15.0, 15.0, 6.0)
        mp = map_points(scene, ds, None, seed=seed, sigma=0.0)
        if len(mp) > M:
            rng = np.random.Generator(np.random.PCG64(seed + 100))
            keep = np.sort(rng.permutation(len(mp))[:M])
            mp = mp[keep]
        sig = 0.0
        open_air_frac = 0.0
    else:
        scene = scene_for_points(M, ds)
        mp = map_points(scene, ds, M, seed=seed)
        sig = 0.01
    R_LI, T_LI = sample_extrinsic() if imu_en else identity_extrinsic()
    gt = default_sensor_pose(scene, R_LI, T_LI)
    body = scan_points(scene, gt, N, seed=seed + 1, det_range=det, sigma=sig, open_air_frac=open_air_frac, order=order)
    init = perturb_pose(gt, seed + 2)
    return dict(scene=scene, map_xyz=mp, body_xyz=body, pose_gt=gt, pose_init=init, ds=ds, imu_en=imu_en, name=name)


# ---- driver messages for the cut-frame preprocess (liinit_frame_cut_*) -------------------------------------------------------
def livox_message(scene: Scene, pose_at, stamp: float, N: int, seed: int = 2, dur: float = 0.1, n_scans: int = 6, noise_frac: float = 0.0,
                  bad_line_frac: float = 0.0, zero_frac: float = 0.0, dup_frac: float = 0.0, tie_frac: float = 0.0, aligned: bool = False,
                  sigma: float = 0.01) -> np.ndarray:
    """A Livox CustomMsg of one 1/10 s sweep (10 Hz): N records of capi.LIVOX_POINT (19 bytes; aligned -> the 20-byte ROS struct),
    offset_time in ns from `stamp`, ascending, built from timed_scan_points. Controllable fractions of records get a noise tag
    ((tag & 0x30) = 0x20 / 0x30), a line >= n_scans, a zero (no-return) point, the previous record's coordinates (consecutive
    duplicate) or the previous record's offset_time (dual-return tie)."""
    from .capi import LIVOX_POINT, LIVOX_POINT_ALIGNED
    rng = np.random.Generator(np.random.PCG64(seed + 7919))
    pts = timed_scan_points(scene, pose_at, stamp, dur, N, seed=seed, sigma=sigma)
    m = np.zeros(N, LIVOX_POINT_ALIGNED if aligned else LIVOX_POINT)
    off = np.round(pts[:, 9].astype(np.float64) * 1e6).astype(np.uint32)
    xyz = pts[:, 0:3].copy()
    line = rng.integers(0, n_scans, N)
    tag = np.where(rng.uniform(size=N) < 0.5, 0x00, 0x10)
    u = rng.uniform(size=N)
    tag = np.where(u < noise_frac, rng.choice([0x20, 0x30], N), tag)
    u = rng.uniform(size=N)
    line = np.where(u < bad_line_frac, rng.integers(n_scans, n_scans + 3, N), line)
    u = rng.uniform(size=N)
    xyz[u < zero_frac] = 0.0
    for i in np.nonzero(rng.uniform(size=N) < dup_frac)[0]:
        if i > 0:
            xyz[i] = xyz[i - 1]
    for i in np.nonzero(rng.uniform(size=N) < tie_frac)[0]:
        if i > 0:
            off[i] = off[i - 1]
    m["offset_time"] = off
    m["x"], m["y"], m["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    m["reflectivity"] = rng.integers(0, 256, N)
    m["tag"] = tag
    m["line"] = line
    return m


# PointCloud2 point layouts of the drivers (the point structs of the reference's preprocess.h, PCL_ADD_POINT4D padding included)
PCL2_FIELDS = {
    2: dict(point_step=32, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=20, off_ring=24),   # velodyne: time f32, ring u16
    3: dict(point_step=48, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=20, off_ring=26),   # ouster: t u32, ring u8
    5: dict(point_step=48, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=24, off_ring=32),   # pandar: timestamp f64, ring u16
    6: dict(point_step=32, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=24, off_ring=18),   # robosense: intensity u8, ring u16, timestamp f64
}


def spinning_pcl2(lidar_type: int, n_rings: int, n_az: int, stamp: float = 0.0, seed: int = 3, with_time: bool = True, turns: float = 1.0,
                  nan_frac: float = 0.0, zero_frac: float = 0.0, extra_pad: int = 0, dur: float = 0.1, az0_deg: float = 30.0):
    """A spinning LiDAR's PointCloud2 (lidar_type 2 Velodyne, 3 Ouster, 5 Pandar, 6 Robosense): n_az firings of n_rings rings, ring-
    ordered within a firing, the head turning clockwise (yaw decreasing) by `turns` revolutions over `dur` seconds, ranges 2-40 m.
    with_time = False leaves the time field out of the layout (Velodyne / Robosense then take the constant-rotation model).
    Returns (data bytes as uint8 array, layout dict, n). extra_pad adds unused bytes to every point."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lay = dict(PCL2_FIELDS[lidar_type])
    lay["point_step"] += int(extra_pad)
    if not with_time:
        lay["off_time"] = -1
    n = n_rings * n_az
    j = np.repeat(np.arange(n_az), n_rings)
    ring = np.tile(np.arange(n_rings), n_az)
    t = dur * j / n_az + rng.uniform(0.0, 1e-6, n)                      # seconds from stamp
    az = np.deg2rad(az0_deg - 360.0 * turns * j / n_az + rng.normal(0.0, 0.02, n))
    el = np.deg2rad(-15.0 + 30.0 * ring / max(n_rings - 1, 1))
    r = rng.uniform(2.0, 40.0, n)
    xyz = np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], 1).astype(np.float32)
    xyz[rng.uniform(size=n) < nan_frac] = np.nan
    xyz[rng.uniform(size=n) < zero_frac] = 0.0
    buf = np.zeros((n, lay["point_step"]), np.uint8)

    def put(off, arr, dt):
        if off >= 0:
            a = np.ascontiguousarray(np.asarray(arr).astype(dt))
            buf[:, off:off + a.dtype.itemsize] = a.view(np.uint8).reshape(n, a.dtype.itemsize)

    put(lay["off_x"], xyz[:, 0], "<f4")
    put(lay["off_y"], xyz[:, 1], "<f4")
    put(lay["off_z"], xyz[:, 2], "<f4")
    put(lay["off_intensity"], rng.integers(0, 256, n), "u1" if lidar_type == 6 else "<f4")
    put(lay["off_ring"], ring, "u1" if lidar_type == 3 else "<u2")
    if lidar_type == 2:
        put(lay["off_time"], t, "<f4")
    elif lidar_type == 3:
        put(lay["off_time"], np.round(t * 1e9), "<u4")
    else:
        put(lay["off_time"], stamp + t, "<f8")
    return buf.reshape(-1), lay, n
