"""The node's main loop (src/laserMapping.cpp:893-1234) over the C-ABI.

process_scan: the LiDAR-only branch on a downsampled, undistorted scan -- constant-velocity propagation -> ICP / IESKF update on
the device map -> map_incremental -> LI-Init data accumulation.
process_raw: the whole loop body on a raw, timed scan, in both modes -- LiDAR-only (constant-velocity propagation, device
undistortion) and, after the hand-over of LI_Initialization, LIO (IMU propagation, device undistortion from the IMU pose table);
then the device voxel grid, the update and map_incremental.
lidar_cbk_livox / lidar_cbk_pcl2 + process_next: the node's LiDAR callbacks with the cut-frame preprocess on the device and
sync_packages: a driver message is cut into sub-frames that stay on the device until process_next stages one for the loop body.
publish= (off by default): the node's published clouds after every update of process_raw -- /cloud_registered, /cloud_registered_body,
/cloud_effected as PointCloud2-ready records built on the device -- and pcd_save's PCD files.

Host-side mirror used by the replay tool and the end-to-end tests; every step is one call into the native libraries
(libliinit_host.so: liinit_propagate_cv, liinit_imu_*, liinit_scan_update; libliinit_gpu.so: liinit_raw_* / liinit_scan_upload /
liinit_map_*; libliinit_calib.so: li_calib_*). Nothing is computed in Python.
"""
from __future__ import annotations

import os
from collections import deque
from dataclasses import dataclass

import numpy as np

from . import capi, host, pcd
from .calib import LiCalib


@dataclass
class Publish:
    """The node's publish/* and pcd_save/* parameters with its defaults (laserMapping.cpp:794-799); set them from the YAML.
    pcd_dir is where pcd_save writes (the node's root_dir + "/PCD")."""
    scan_pub_en: bool = True        # publish/scan_publish_en
    dense_pub_en: bool = True       # publish/dense_publish_en
    scan_body_pub_en: bool = True   # publish/scan_bodyframe_pub_en
    pcd_save_en: bool = False       # pcd_save/pcd_save_en
    interval: int = -1              # pcd_save/interval
    pcd_dir: str = "PCD"
    # which of the published clouds are built when their condition holds (a recording that does not keep a topic skips its download)
    clouds: tuple = ("registered", "body", "effect")


class ImuBuffer:
    """The node's imu_buffer: imu_cbk's time compensation (laserMapping.cpp:412-423) and sync_packages's selection of a measure
    group (:466-474). Rows are {stamp, gyr xyz, acc xyz}."""

    def __init__(self, timediff_imu_wrt_lidar: float = 0.0):
        self.timediff = float(timediff_imu_wrt_lidar)
        self.time_lag = 0.0             # time_lag_IMU_wtr_lidar, set at the hand-over
        self.last_stamp = -np.inf       # last_timestamp_imu
        self.rows = deque()

    def push(self, t, gyr, acc):
        stamp = float(t) - self.timediff - self.time_lag
        if stamp < self.last_stamp:     # "IMU loop back, clear IMU buffer" (:415-419)
            self.rows.clear()
        self.last_stamp = stamp
        self.rows.append(np.concatenate([[stamp], np.asarray(gyr, float), np.asarray(acc, float)]))

    def ready(self, lidar_end_time: float) -> bool:
        """sync_packages waits until an IMU sample at or after the scan end has arrived (:461-462)."""
        return self.last_stamp >= lidar_end_time

    def pop(self, lidar_end_time: float) -> np.ndarray:
        """The measure group of a scan ending at lidar_end_time: the buffered samples with stamp <= lidar_end_time (:466-474)."""
        out = []
        imu_time = self.rows[0][0] if self.rows else 0.0
        while self.rows and imu_time < lidar_end_time:
            imu_time = self.rows[0][0]
            if imu_time > lidar_end_time:
                break
            out.append(self.rows.popleft())
        return np.array(out, float).reshape(-1, 7)

    def shift(self, time_lag: float):
        """The hand-over (:1217-1220): the buffered stamps and every later one are moved by -time_lag. (Later samples are compared
        against the last stamp before the shift, so the first one after it clears the buffer when the lag exceeds a sample period,
        as imu_cbk does.)"""
        self.time_lag = float(time_lag)
        for r in self.rows:
            r[0] -= self.time_lag


class SubFrame:
    """A sub-frame held on the device (an entry of liinit_frame_cut_*), as process_raw's scan."""

    def __init__(self, entry):
        self.handle = int(entry["handle"])
        self.end_ms = np.float32(entry["end_ms"])
        self.n = int(entry["n"])


class ReplayFrame(SubFrame):
    """A sub-frame of the replay store (liinit_replay_*): stored sub-frame j, staged by liinit_replay_stage."""

    def __init__(self, j: int, end_ms, n: int):
        self.j, self.end_ms, self.n = int(j), np.float32(end_ms), int(n)


class LidarOdometry:
    def __init__(self, gpu: capi.LiInitGpu, filter_size_map: float, max_iteration: int = 4, gyr_cov: float = 0.1, acc_cov: float = 0.1,
                 orig_odom_freq: int = 10, cut_frame_num: int = 1, data_accum_length: float = 300.0, calib: LiCalib | None = None,
                 filter_size_surf: float | None = None, rot_LI_cov: float = 0.00005, trans_LI_cov: float = 0.0005, b_gyr_cov: float = 0.0001,
                 b_acc_cov: float = 0.0001, mean_acc_norm: float = 9.81, publish: Publish | dict | None = None):
        self.g = gpu
        self.ds = float(filter_size_map)
        self.max_iteration = int(max_iteration)            # "max_iteration", laserMapping.cpp:767
        self.gyr_cov, self.acc_cov = gyr_cov, acc_cov      # mapping/gyr_cov, mapping/acc_cov (:776-777)
        self.orig_odom_freq, self.cut_frame_num = int(orig_odom_freq), int(cut_frame_num)
        self.state = host.state_init()
        self.calib = calib if calib is not None else LiCalib(data_accum_length)
        self.map_ready = False
        self.first_prop = True
        self.t_last = None
        self.frame_num = 0
        self.data_accum_start = False
        self.data_accum_finished = False
        self.move_start_time = 0.0
        self.stats = None
        self.imu_en = False
        # process_raw: the voxel-grid leaf of the scan (mapping/filter_size_surf, :772), the IMU buffer and the IMU processor
        # configured as the node does it at start-up (:833-838)
        self.filter_size_surf = self.ds if filter_size_surf is None else float(filter_size_surf)
        self.mean_acc_norm = float(mean_acc_norm)
        self.imu_buffer = ImuBuffer()
        self.imu_proc = self._make_imu_proc()
        for which, v in (("gyr_cov", gyr_cov), ("acc_cov", acc_cov), ("R_LI_cov", rot_LI_cov), ("T_LI_cov", trans_LI_cov),
                         ("gyr_bias_cov", b_gyr_cov), ("acc_bias_cov", b_acc_cov)):
            self.imu_proc.set_cov(which, v)
        self.lidar_end_time = None
        self.switch_scan = None   # index (frame_num) of the scan that switched to LIO mode
        # the LiDAR callbacks (laserMapping.cpp:310-381): preprocess/* parameters with the node's defaults (:768,781-786)
        self.preprocess = dict(lidar_type=1, N_SCANS=16, blind=1.0, point_filter_num=2)
        self.scan_count = 0
        self.last_timestamp_lidar = 0.0
        self.timediff_set = False
        self.lidar_buffer = deque()   # lidar_buffer + time_buffer: sub-frame entries {handle, t_beg, end_ms, n} of liinit_frame_cut_*
        self.dropped_subframes = 0
        # the published clouds of the last process_raw: {"registered", "body", "effect"} -> [n, 12] float32 records
        self.publish = Publish(**publish) if isinstance(publish, dict) else publish
        self.published = {}
        self.pcd_wait = []            # pcl_wait_save, as the REGISTERED records of the scans since the last file
        self.scan_wait_num = 0
        self.pcd_index = 0
        self.pcd_files = []
        # a timed assessment (assess.Assessment(timed=True)): the IMU undistortion holds the staged raw cloud for the store, and
        # timing keeps (pose table, propagated state) of the last process_raw that undistorted from a table (None for any other)
        self.assess_hold = False
        self.timing = None
        # a replay of the LIO phase (assess.Replay): process_next hands it every sub-frame it processes; frozen: the update holds the
        # extrinsic constant (liinit_scan_update_frozen)
        self.replay = None
        self.frozen = False

    def push_imu(self, omg, acc, t, mean_acc_norm=9.81):
        """imu_cbk in LO mode (:428-430)."""
        if not self.data_accum_finished:
            self.calib.push_imu_all(omg, acc, t, mean_acc_norm)

    def process_scan(self, body_xyz: np.ndarray, t_beg: float, t_end: float):
        """One pass of the loop body for a downsampled, undistorted scan in the LiDAR frame. Returns the posterior state."""
        # p_imu->Process in LO mode: Forward_propagation_without_imu (IMU_Processing.hpp:212-243)
        if self.first_prop:
            dt = 0.1
            self.first_prop = False
        else:
            dt = t_beg - self.t_last
        self.t_last = t_beg
        self.state = host.propagate_cv(self.state, dt, self.gyr_cov, self.acc_cov)
        R, p, RLI, TLI = host.state_pose(self.state)
        if not self.map_ready:                              # :921-931
            if len(body_xyz) > 5:
                world = (R @ (RLI @ body_xyz.T.astype(np.float64) + TLI[:, None]) + p[:, None]).T.astype(np.float32)
                self._map_build(world)
                self.map_ready = True
            return self.state
        self.state, self.stats = self._scan_update(body_xyz, self.state)   # :936-1134
        R, p, RLI, TLI = host.state_pose(self.state)
        self._map_incremental(R, p, RLI, TLI)               # :1140
        if not self.data_accum_start and np.linalg.norm(p) > 0.05:   # :1145-1149
            self.data_accum_start = True
            self.move_start_time = t_end
        self.frame_num += 1                                 # :1160
        if not self.data_accum_finished and self.data_accum_start:   # :1190-1196
            bias_g, vel = self.state[27:30], self.state[24:27]
            self.calib.push_lidar(R, bias_g, vel, t_end)
            ok, _ = self.calib.data_sufficiency(self.frame_num, bias_g, self.orig_odom_freq, self.cut_frame_num)
            self.data_accum_finished = ok
        return self.state

    def process_raw(self, raw_pts12: np.ndarray, t_beg: float, imu_group: np.ndarray | None = None):
        """One pass of the loop body (laserMapping.cpp:893-1160) for a raw scan: raw_pts12 [n, 12] float32 in the PointType layout
        with the per-point time offset in ms in the curvature field (index 9), t_beg = lidar_beg_time. imu_group [k, 7] {stamp, gyr,
        acc}: the measure group; None -> the samples of imu_buffer with stamp <= lidar_end_time (sync_packages, :466-474).
        Returns the posterior state.

        LiDAR-only mode: constant-velocity propagation, device undistortion with omega = bias_g. LIO mode: IMU propagation, device
        undistortion from the IMU pose table. The first scan after the hand-over only switches the IMU processor: like Process, it
        neither propagates nor touches the undistorted cloud, so the cloud of the previous scan -- still staged on the device -- is
        downsampled and matched again (the reference keeps feats_undistort, :909-918)."""
        if isinstance(raw_pts12, SubFrame):
            raw = raw_pts12
            end_ms = float(raw.end_ms)
        else:
            raw = np.ascontiguousarray(raw_pts12, np.float32)
            end_ms = float(raw[:, 9].max())                 # points.back().curvature of the time-sorted cloud
        t_end = t_beg + end_ms / 1000.0                     # lidar_end_time (:455-456)
        group = self.imu_buffer.pop(t_end) if imu_group is None else np.asarray(imu_group, float).reshape(-1, 7)
        self.published = {}
        self.timing = None
        if not self.imu_en:
            # Forward_propagation_without_imu (IMU_Processing.hpp:204-267)
            if self.first_prop:
                dt = 0.1
                self.first_prop = False
            else:
                dt = t_beg - self.t_last
            self.t_last = t_beg
            self.state = host.propagate_cv(self.state, dt, self.gyr_cov, self.acc_cov)
            self._undistort_cv(raw, self.state)
        elif len(group) and not self.imu_proc.need_init:
            self.state, poses = self._propagate_imu(self.state, group, t_beg, end_ms)   # propagation_and_undist (:269-416)
            self._undistort_imu(raw, poses, self.state)
            self.timing = (poses, self.state.copy())
        elif len(group):
            self.imu_proc.switch(group)                     # Process, IMU_Processing.hpp:445-453: no propagation, cloud kept
            self.switch_scan = self.frame_num
        # (an empty group in LIO mode: Process returns at once, :423 -- nothing propagated, cloud kept)
        self._downsample(self.filter_size_surf)             # downSizeFilterSurf (:917-918)
        self.lidar_end_time = t_end
        if not self.map_ready:                              # :921-931
            body = self._scan_body()
            if len(body) > 5:
                R, p, RLI, TLI = host.state_pose(self.state)
                world = (R @ (RLI @ body.T.astype(np.float64) + TLI[:, None]) + p[:, None]).T.astype(np.float32)
                self._map_build(world)
                self.map_ready = True
            return self.state
        self.state, self.stats = self._scan_update_resident(self.state)   # :936-1134
        R, p, RLI, TLI = host.state_pose(self.state)
        self._map_incremental(R, p, RLI, TLI)               # :1140
        if not self.imu_en and not self.data_accum_start and np.linalg.norm(p) > 0.05:   # :1145-1149
            self.data_accum_start = True
            self.move_start_time = t_end
        if self.publish is not None:                        # :1152-1156
            self._publish(R, p, RLI, TLI)
        self.frame_num += 1                                 # :1160
        if not self.imu_en and not self.data_accum_finished and self.data_accum_start:   # :1190-1196
            bias_g, vel = self.state[27:30], self.state[24:27]
            self.calib.push_lidar(R, bias_g, vel, t_end)
            ok, _ = self.calib.data_sufficiency(self.frame_num, bias_g, self.orig_odom_freq, self.cut_frame_num)
            self.data_accum_finished = ok
        return self.state

    # ---- the LiDAR callbacks and sync_packages over the device cut ----
    def _lidar_cbk(self, stamp: float):
        """The part of livox_pcl_cbk / standard_pcl_cbk before the cut (:312-324)."""
        self.scan_count += 1
        if stamp < self.last_timestamp_lidar:           # "lidar loop back, clear buffer"
            self.lidar_buffer.clear()
        self.last_timestamp_lidar = stamp
        ib = self.imu_buffer
        if ib.rows and abs(ib.last_stamp - stamp) > 1.0 and not self.timediff_set:   # self sync of IMU and LiDAR clocks
            self.timediff_set = True
            ib.timediff = ib.last_stamp - stamp

    def _cut_params(self, stamp):
        return dict(self.preprocess, required_frame_num=self.cut_frame_num, scan_count=self.scan_count, stamp=float(stamp))

    def lidar_cbk_livox(self, records, stamp: float):
        """livox_pcl_cbk with cut_frame (:310-345): records = the CustomMsg points (capi.LIVOX_POINT / LIVOX_POINT_ALIGNED),
        stamp = header.stamp [s]. The sub-frames stay on the device; their entries are appended to lidar_buffer."""
        self._lidar_cbk(stamp)
        self.lidar_buffer.extend(self.g.frame_cut_livox(records, **self._cut_params(stamp)))

    def lidar_cbk_pcl2(self, data, layout, n: int, stamp: float):
        """standard_pcl_cbk with cut_frame (:347-381) for Velodyne, Ouster, Pandar and Robosense PointCloud2 messages."""
        self._lidar_cbk(stamp)
        self.lidar_buffer.extend(self.g.frame_cut_pcl2(data, layout, n, **self._cut_params(stamp)))

    def process_next(self):
        """sync_packages (:436-480) and the loop body on the oldest buffered sub-frame: sub-frames of <= 1 point are dropped; the
        sub-frame waits until an IMU stamp >= its lidar_end_time has arrived. Sub-frames whose message slot the device has reused
        (LIINIT_FRAME_SLOTS later messages have yielded sub-frames) are dropped and counted in dropped_subframes. Returns the posterior
        state, or None when nothing is ready."""
        while self.lidar_buffer:
            e = self.lidar_buffer[0]
            if e["n"] <= 1:                                 # "Too few input point cloud!"
                self.lidar_buffer.popleft()
            elif self.g.frame_size(e["handle"]) is None:
                # the device keeps the sub-frames of the last LIINIT_FRAME_SLOTS messages only: when the loop fell that far behind
                # the callbacks, the older sub-frames are gone and are skipped before any state is touched
                self.lidar_buffer.popleft()
                self.dropped_subframes += 1
            else:
                break
        if not self.lidar_buffer or not self.imu_buffer.rows:
            return None
        e = self.lidar_buffer[0]
        t_end = e["t_beg"] + float(np.float32(e["end_ms"])) / 1000.0
        if not self.imu_buffer.ready(t_end):
            return None
        self.lidar_buffer.popleft()
        group = self.imu_buffer.pop(t_end)
        if self.replay is not None:
            self.replay.record_frame(e)
        return self.process_raw(SubFrame(e), e["t_beg"], group)

    def _publish(self, R, p, RLI, TLI):
        """The "Publish points" block of the loop (:1152-1156) with the posterior: publish_frame_world (:561-614) when scan_pub_en or
        pcd_save_en, publish_frame_body (:616-623) when scan_pub_en and scan_body_pub_en, publish_effect_world (:625-636) always;
        each only when it is in Publish.clouds. The records land in self.published; pcd_save accumulates the REGISTERED records on the
        host."""
        c = self.publish
        out = {}
        reg = None
        if c.scan_pub_en and "registered" in c.clouds:
            which = capi.CLOUD_REGISTERED if c.dense_pub_en else capi.CLOUD_REGISTERED_DOWN
            out["registered"] = self.g.cloud(which, R, p, RLI, TLI)
            if c.dense_pub_en:
                reg = out["registered"]
        if c.pcd_save_en:
            self._pcd_save(reg if reg is not None else self.g.cloud(capi.CLOUD_REGISTERED, R, p, RLI, TLI))
        if c.scan_pub_en and c.scan_body_pub_en and "body" in c.clouds:
            out["body"] = self.g.cloud(capi.CLOUD_BODY)
        if "effect" in c.clouds:
            out["effect"] = self.g.cloud(capi.CLOUD_EFFECT, R, p, RLI, TLI)
        self.published = out

    def _pcd_save(self, reg):
        """pcd_save (:594-613): feats_undistort in the world frame is appended to pcl_wait_save; with interval > 0 every interval-th
        scan writes PCD<k>.pcd and starts over."""
        self.pcd_wait.append(reg)
        self.scan_wait_num += 1
        if sum(len(a) for a in self.pcd_wait) > 0 and self.publish.interval > 0 and self.scan_wait_num >= self.publish.interval:
            self.pcd_index += 1
            self._pcd_write(f"PCD{self.pcd_index}.pcd")
            self.pcd_wait = []
            self.scan_wait_num = 0

    def _pcd_write(self, name):
        os.makedirs(self.publish.pcd_dir, exist_ok=True)
        path = os.path.join(self.publish.pcd_dir, name)
        pcd.write_binary(path, np.concatenate(self.pcd_wait) if self.pcd_wait else np.zeros((0, 12), np.float32))
        self.pcd_files.append(path)

    def close(self):
        """The node's shutdown (SigHandle, :183-187): with pcd_save_en and interval < 0 everything accumulated goes to PCD_all.pcd
        (nothing is written when no point has been accumulated: PCL refuses an empty cloud)."""
        c = self.publish
        if c is not None and c.pcd_save_en and c.interval < 0 and sum(len(a) for a in self.pcd_wait) > 0:
            self._pcd_write("PCD_all.pcd")
            self.pcd_wait = []

    def world_cloud(self):
        """The undistorted raw cloud of the last process_raw in the world frame with the current state (publish_frame_world with
        dense_publish_en, pcd_save; laserMapping.cpp:560-603), [n, 3] float32 in upload order."""
        R, p, RLI, TLI = host.state_pose(self.state)
        return self.g.raw_world(R, p, RLI, TLI)

    # the calls into the hot path; a test substitutes the CPU oracle here to drive the SAME loop from the other side
    def _map_build(self, world):
        self.g.map_build(world)

    def _scan_update(self, body_xyz, state):
        self.g.scan_upload(body_xyz)
        return host.scan_update(self.g, state, self.max_iteration, self.imu_en)

    def _map_incremental(self, R, p, RLI, TLI):
        self.g.map_incremental(R, p, RLI, TLI, self.ds)

    # process_raw's stages
    def _make_imu_proc(self):
        return host.ImuProcess()

    def _propagate_imu(self, state, group, t_beg, end_ms):
        return self.imu_proc.propagate(state, group, t_beg, end_ms)

    def _stage(self, raw):
        """Stage the raw cloud of the scan: an uploaded PointType array, or a sub-frame the device already holds (in a message slot or
        in the replay store)."""
        if isinstance(raw, ReplayFrame):
            self.g.replay_stage(raw.j)
        elif isinstance(raw, SubFrame):
            self.g.frame_stage(raw.handle)
        else:
            self.g.raw_upload(raw, 9)

    def _undistort_cv(self, raw, state):
        self._stage(raw)
        self.g.raw_undistort_cv(state[27:30], state[0:9], state[24:27])   # omega = bias_g, rot_end / vel_end propagated

    def _undistort_imu(self, raw, poses, state):
        self._stage(raw)
        if self.assess_hold:
            self.g.assess_hold()
        if len(poses) >= 2:   # (one pose: the back-propagation loop of the reference runs zero times)
            R, p, RLI, TLI = host.state_pose(state)
            self.g.raw_undistort_imu(poses, R, p, RLI, TLI)

    def _downsample(self, leaf):
        self.g.raw_downsample(leaf)

    def _scan_body(self):
        return self.g.scan_body()

    def _scan_update_resident(self, state):
        return host.scan_update(self.g, state, self.max_iteration, self.imu_en, frozen=self.frozen)

    def hand_over(self, res):
        """laserMapping.cpp:1198-1222 after LI_Initialization: the pose is re-expressed in the IMU frame with the calibrated extrinsic,
        gravity / biases are taken over and the filter continues with the 12-column Jacobian (imu_en = true)."""
        R, p, _, _ = host.state_pose(self.state)
        R_LI, T_LI = np.asarray(res["R_LI"], float).reshape(3, 3), np.asarray(res["T_LI"], float)
        s = self.state
        s[12:21] = R_LI.reshape(9)                          # offset_R_L_I = Init_LI->get_R_LI() (:1204)
        s[21:24] = T_LI                                     # offset_T_L_I (:1205)
        s[9:12] = p - R @ R_LI.T @ T_LI                     # pos_end = -rot_end * R_LI^T * T_LI + pos_end (:1206)
        s[0:9] = (R @ R_LI.T).reshape(9)                    # rot_end = rot_end * R_LI^T (:1207)
        s[33:36] = np.asarray(res["grav_L0"], float)        # gravity (:1208)
        s[27:30] = np.asarray(res["gyro_bias"], float)      # bias_g (:1209)
        s[30:33] = np.asarray(res["acc_bias"], float)       # bias_a (:1210)
        self.imu_en = True
        if self.preprocess["lidar_type"] != 1:             # spinning sensors continue at two sub-frames per message (:1214-1215)
            self.cut_frame_num = 2
        # (:1217-1228) the buffered IMU stamps move by the total time lag; the IMU processor switches at its next scan
        self.imu_buffer.shift(float(res["time_lag_1"]) + float(res["time_lag_2"]))
        self.imu_proc.set_mean_acc_norm(self.mean_acc_norm)
        for which, v in (("gyr_cov", 0.1), ("acc_cov", 0.1), ("gyr_bias_cov", 0.0001), ("acc_bias_cov", 0.0001)):
            self.imu_proc.set_cov(which, v)

    def initialize(self, timediff_imu_wrt_lidar: float = 0.0):
        """LI_Initialization on what has been accumulated (:1198); returns the calibration dict of calib.LiCalib."""
        return self.calib.initialize(self.orig_odom_freq, self.cut_frame_num, timediff_imu_wrt_lidar, self.move_start_time, from_groups=False)
