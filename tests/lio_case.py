"""Timed-scan lockstep of the node's loop through LidarOdometry.process_raw (test infrastructure).

Both legs see the same raw scans (scenes.timed_scan_points: every point at its own time, in the LiDAR frame of that time) and the
same IMU stream (calib_sim.make_streams). The product leg runs the host library and the device chain; the oracle leg replaces every
stage by the CPU checkers (lio_oracle: IMU propagation and pointBodyToWorld; oracle/: the undistortion loops, the voxel grid, the
restated / verbatim map)."""
import os

import numpy as np

import calib_sim
import lio_oracle

P0 = (15.0, 12.0, 2.2)   # where the rig starts in the scene (the odometry frame of a full run is the first LiDAR frame)


def angle(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


class TruePath:
    """The simulated rig in the scene: LiDAR pose (vectorised over time) and IMU pose / velocity, true time."""

    def __init__(self, seed, S, t0=100.0, p0=P0):
        self.tr = calib_sim.Trajectory(seed)
        self.S, self.t0, self.p0 = S, t0, np.asarray(p0, float)

    def lidar(self, t):
        """t [n] -> R [n,3,3], p [n,3] (calib_sim.Trajectory.R / pos evaluated for many times at once)."""
        tr = self.tr
        s = np.asarray(t, float) - self.t0 - tr.t_move
        u = np.clip(s / 2.0, 0, 1)
        ramp = u ** 4 * (35 - 84 * u + 70 * u ** 2 - 20 * u ** 3)
        ang = ramp[:, None] * np.sum(tr.aa[None] * (np.sin(2 * np.pi * tr.fa[None] * s[:, None, None] + tr.pa[None]) - np.sin(tr.pa)[None]), axis=2)
        pos = ramp[:, None] * np.sum(tr.ap[None] * (np.sin(2 * np.pi * tr.fp[None] * s[:, None, None] + tr.pp[None]) - np.sin(tr.pp)[None]), axis=2)
        c, sn = np.cos(ang), np.sin(ang)
        n = len(s)
        Rx, Ry, Rz = (np.zeros((n, 3, 3)) for _ in range(3))
        Rx[:, 0, 0] = 1; Rx[:, 1, 1] = c[:, 0]; Rx[:, 1, 2] = -sn[:, 0]; Rx[:, 2, 1] = sn[:, 0]; Rx[:, 2, 2] = c[:, 0]
        Ry[:, 1, 1] = 1; Ry[:, 0, 0] = c[:, 1]; Ry[:, 0, 2] = sn[:, 1]; Ry[:, 2, 0] = -sn[:, 1]; Ry[:, 2, 2] = c[:, 1]
        Rz[:, 2, 2] = 1; Rz[:, 0, 0] = c[:, 2]; Rz[:, 0, 1] = -sn[:, 2]; Rz[:, 1, 0] = sn[:, 2]; Rz[:, 1, 1] = c[:, 2]
        return Rz @ Ry @ Rx, pos + self.p0

    def imu(self, t):
        """IMU frame rot_end / pos_end (the state of the LIO mode) at the scalar time t."""
        R, p = self.lidar(np.array([t]))
        R_I = R[0] @ self.S["R_LI"].T
        return R_I, p[0] - R_I @ self.S["T_LI"]

    def imu_vel(self, t, h=1e-5):
        return (self.imu(t + h)[1] - self.imu(t - h)[1]) / (2 * h)


def make_oracle_odometry(orc, ds, nthreads, undistort=True, **kw):
    from lidar_imu_init_b200 import host
    from lidar_imu_init_b200.odometry import LidarOdometry

    class OracleOdometry(LidarOdometry):
        """LidarOdometry with every stage of process_raw on the CPU oracle. undistort=False skips the undistortion (negative control)."""

        def __init__(self):
            super().__init__(None, ds, **kw)
            self.om = orc.OracleMap(ds, 1 if orc.has_ikd() else 0)
            self.sc = None
            self.raw_xyz = None
            self.body = None

        def _make_imu_proc(self):
            return lio_oracle.OracleImu()

        def _undistort_cv(self, raw, state):
            xyz = raw[:, 0:3]
            self.raw_xyz = orc.undistort_cv(xyz, raw[:, 9], state[27:30], state[0:9], state[24:27]) if undistort else np.ascontiguousarray(xyz)

        def _undistort_imu(self, raw, poses, state):
            xyz = raw[:, 0:3]
            if undistort and len(poses) >= 2:
                R, p, RLI, TLI = host.state_pose(state)
                self.raw_xyz = orc.undistort_imu(xyz, raw[:, 9], poses, R, p, RLI, TLI)
            else:
                self.raw_xyz = np.ascontiguousarray(xyz, np.float32)

        def _downsample(self, leaf):
            self.body = orc.voxel_grid(self.raw_xyz, leaf)

        def _scan_body(self):
            return self.body

        def _map_build(self, world):
            self.om.build(world)

        def _scan_update_resident(self, state):
            self.sc = orc.OracleScan(self.body)
            st, iters, searches, m = self.sc.scan_update(self.om, state, self.max_iteration, self.imu_en, nthreads=nthreads)
            return st, dict(iterations=iters, search_passes=searches, effect_feat_num=m)

        def _map_incremental(self, R, p, RLI, TLI):
            self.sc.map_incremental(self.om, R, p, RLI, TLI, self.ds)

        def world_cloud(self):
            R, p, RLI, TLI = host.state_pose(self.state)
            return lio_oracle.body_to_world(self.raw_xyz, R, p, RLI, TLI)

    return OracleOdometry()


def true_result(S):
    """What LI_Initialization returns on the simulated rig, exactly (the calibration of the short runs that skip the LO leg)."""
    return dict(R_LI=S["R_LI"], T_LI=S["T_LI"], grav_L0=S["g_W"], gyro_bias=S["b_g"], acc_bias=S["b_a"], time_lag_1=S["t_off"], time_lag_2=0.0)


def run(legs, orc, seconds, points, seed=0, t_off=0.013, ds=0.15, t_start=None, scans=None, map_from_scene=False, on_scan=None):
    """Drives the odometries of `legs` (name -> LidarOdometry, built by the caller) over the same timed scans and IMU samples.

    t_start None: from the beginning, LiDAR-only mode until LI-Init fires on every leg, then the hand-over with each leg's own
    result. t_start given: the run starts at that time (seconds after the stream start) with the hand-over right after the first
    scan, using the simulator's true calibration, and the true IMU velocity. on_scan(j, legs, truth) is called after every scan.
    Returns dict(init_scan, switch_scan, res, truth)."""
    from lidar_imu_init_b200 import scenes

    S = calib_sim.make_streams(seed=seed, duration=seconds if t_start is None else t_start + seconds, t_off=t_off)
    path = TruePath(seed, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    tl = S["lidar"][0]
    j0 = 0 if t_start is None else int(np.searchsorted(tl, path.t0 + t_start))
    k_imu = int(np.searchsorted(ti, tl[j0] - 0.05))
    res = {name: None for name in legs}
    out = dict(init_scan=None, switch_scan=None, res=res, truth=S, path=path)
    if map_from_scene:
        mp = scenes.map_points(scene, ds, seed=seed + 7)
        for lo in legs.values():
            lo._map_build(mp)
            lo.map_ready = True
    n = 0
    for j in range(j0, len(tl)):
        if scans is not None and n >= scans:
            break
        t_beg = tl[j] - 0.02
        raw = scenes.timed_scan_points(scene, path.lidar, t_beg, 0.02, points, seed=1000 + j, det_range=60.0, sigma=0.01)
        t_end = t_beg + float(raw[:, 9].max()) / 1000.0
        while k_imu < len(ti) and ti[k_imu] <= t_end + 0.03:      # the IMU runs ahead of the LiDAR (sync_packages waits for it)
            for lo in legs.values():
                lo.imu_buffer.push(ti[k_imu], wi[k_imu], ai[k_imu])
                lo.push_imu(wi[k_imu], ai[k_imu], ti[k_imu])
            k_imu += 1
        if t_start is not None and n == 0:
            # start in LiDAR-only mode with the true LiDAR motion, so that the first cloud is undistorted and the state after the
            # constant-velocity propagation of the first frame (dt = 0.1) is the true pose
            R, p = path.lidar(np.array([t_end]))
            w_L = path.tr.omega_body(t_end - path.t0)
            v_L = (path.lidar(np.array([t_end + 1e-5]))[1][0] - path.lidar(np.array([t_end - 1e-5]))[1][0]) / 2e-5
            for lo in legs.values():
                s = lo.state
                s[0:9] = (R[0] @ scenes.so3_exp(-w_L * 0.1)).reshape(9)
                s[9:12] = p[0] - v_L * 0.1
                s[24:27] = v_L
                s[27:30] = w_L
        for lo in legs.values():
            lo.process_raw(raw, t_beg)
        if t_start is not None and n == 0:
            r = true_result(S)
            for name, lo in legs.items():
                lo.data_accum_finished = True
                lo.hand_over(r)
                lo.state[24:27] = path.imu_vel(t_end)
                res[name] = r
            out["init_scan"] = j
        elif t_start is None and out["init_scan"] is None and all(lo.data_accum_finished for lo in legs.values()):
            for name, lo in legs.items():
                res[name] = lo.initialize(0.0)
                lo.hand_over(res[name])
            out["init_scan"] = j
        if out["switch_scan"] is None and out["init_scan"] is not None and j > out["init_scan"]:
            out["switch_scan"] = j
        if on_scan is not None:
            on_scan(j, legs, dict(t_end=t_end, imu=path.imu(t_end), path=path, raw=raw, lio=out["init_scan"] is not None and j > out["init_scan"]))
        n += 1
    out["scans"] = n
    return out


def default_threads():
    return min(16, os.cpu_count() or 1)
