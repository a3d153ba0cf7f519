"""The node's main() (laserMapping.cpp:891-1244) over LidarOdometry, without ROS: the IMU and LiDAR callbacks, the loop body after every
delivered message, the LI-Init trigger and hand-over, the online-refinement clock, and the node's result files:

  <out>/result/Initialization_result.txt   fileout_calib_result (:708-725) after "Initialization result:" / "Refinement result:"
  <out>/Log/mat_out.txt                    the fout_out row of every update (:1162-1166)
  <out>/result/trajectory.txt              one TUM line per update, the pose of /aft_mapped_to_init (set_posestamp, :647-663)
  <out>/PCD/                               pcd_save (LidarOdometry's Publish path)
  <out>/Log/<six LI-Init logs>             with open_debug_logs(): LI_Init's logs (LI_init.cpp:11-16), written at the trigger

and, with a Recorder in Node.recorder, the node's published topics in a bag (bagwrite); with an Assessment in Node.assess, the LIO
scans it scores the calibration on (assess).

Delivery model: after every delivered message the loop body runs until sync_packages has nothing ready (LidarOdometry.process_next
returns None), i.e. a node that always keeps up with playback (DESIGN §4b). The node's spinOnce batching, which depends on timing, is
not reproduced.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

from . import config as cfgmod
from . import host, pubmsg, rosmsg
from .odometry import LidarOdometry


# ---- formatting of the node's streams ------------------------------------------------------------------------------------------------
def rot_to_euler(R) -> np.ndarray:
    """RotMtoEuler (include/so3_math.h:110-131)."""
    R = np.asarray(R, float)
    sy = math.sqrt(R[0, 0] * R[0, 0] + R[1, 0] * R[1, 0])
    if sy >= 1e-6:
        return np.array([math.atan2(R[2, 1], R[2, 2]), math.atan2(-R[2, 0], sy), math.atan2(R[1, 0], R[0, 0])])
    return np.array([math.atan2(-R[1, 2], R[1, 1]), math.atan2(-R[2, 0], sy), 0.0])


def quat_from_rpy(roll, pitch, yaw) -> np.ndarray:
    """tf::createQuaternionMsgFromRollPitchYaw (tf::Quaternion::setRPY) -> [x, y, z, w]."""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def _fixed6(v):
    return "%.6f" % v


def _general6(v):
    return "%.6g" % v


def eigen_str(m, fmt) -> str:
    """Eigen's default operator<< of a matrix (IOFormat(): stream precision, aligned columns): every coefficient right-aligned to the
    widest coefficient of the whole object, coefficients separated by one space, rows by a newline. A 1-D array is a row (a
    transposed vector)."""
    m = np.atleast_2d(np.asarray(m, float))
    s = [[fmt(v) for v in row] for row in m]
    w = max(len(x) for row in s for x in row)
    return "\n".join(" ".join(x.rjust(w) for x in row) for row in s)


def calib_result_text(euler_deg, T_LI, time_lag, bias_g, bias_a, gravity, R_LI) -> str:
    """fileout_calib_result (laserMapping.cpp:708-725) with the stream in fixed, precision 6. euler_deg = RotMtoEuler(R_LI) * 57.3 and
    time_lag = time_lag_IMU_wtr_lidar + timediff_imu_wrt_lidar, as printed."""
    T = np.eye(4)
    T[0:3, 0:3] = np.asarray(R_LI, float).reshape(3, 3)
    T[0:3, 3] = T_LI
    return ("Rotation LiDAR to IMU (degree)     = " + eigen_str(euler_deg, _fixed6) + "\n"
            "Translation LiDAR to IMU (meter)   = " + eigen_str(T_LI, _fixed6) + "\n"
            "Time Lag IMU to LiDAR (second)     = " + _fixed6(time_lag) + "\n"
            "Bias of Gyroscope  (rad/s)         = " + eigen_str(bias_g, _fixed6) + "\n"
            "Bias of Accelerometer (meters/s^2) = " + eigen_str(bias_a, _fixed6) + "\n"
            "Gravity in World Frame(meters/s^2) = " + eigen_str(gravity, _fixed6) + "\n\n"
            "Homogeneous Transformation Matrix from LiDAR to IMU: \n" + eigen_str(T, _fixed6) + "\n\n\n")


def state_calib_values(state, time_lag) -> dict:
    """The arguments of calib_result_text for a state."""
    R, _, RLI, TLI = host.state_pose(state)
    return dict(euler_deg=rot_to_euler(RLI) * 57.3, T_LI=TLI, time_lag=time_lag, bias_g=state[27:30], bias_a=state[30:33],
                gravity=state[33:36], R_LI=RLI)


def mat_out_row(euler_deg, pos, ext_deg, T_LI, vel, bias_g, bias_a_scaled, gravity, total_distance) -> str:
    """The fout_out row (laserMapping.cpp:1162-1166) in the stream's default format (6 significant digits), the reference's double
    space before bias_g included; bias_a_scaled = bias_a * 0.9822 / 9.81 and the angles in degrees, as printed."""
    e = lambda v: eigen_str(v, _general6)   # noqa: E731
    return (e(euler_deg) + " " + e(pos) + " " + e(ext_deg) + " " + e(T_LI) + " " + e(vel) + " " + " " + e(bias_g) + " " + e(bias_a_scaled)
            + " " + e(gravity) + " " + _general6(total_distance) + "\n")


def state_mat_out_row(state, euler_cur, total_distance) -> str:
    R, p, RLI, TLI = host.state_pose(state)
    return mat_out_row(euler_cur * 57.3, p, rot_to_euler(RLI) * 57.3, TLI, state[24:27], state[27:30], state[30:33] * 0.9822 / 9.81, state[33:36],
                       total_distance)


# LI_Init's logs (LI_init.cpp:11-16, in the constructor's order): file -> (calib.LiCalib.log_rows table, the stream's precision,
# coefficients of each object the row streams: an Eigen row vector (transpose()) or a scalar, separated by one space)
DEBUG_LOGS = {
    "LiDAR_meas.txt": ("LiDAR_meas", 12, (3, 1, 3, 3, 1)),                 # :151-156
    "IMU_meas.txt": ("IMU_meas", 12, (3, 1, 3, 3, 1)),                     # :135-139
    "IMU_before_filter.txt": ("IMU_before_filter", 15, (3, 1, 3, 1)),      # :45-46
    "Lidar_before_filter.txt": ("Lidar_before_filter", 15, (3, 1, 1)),     # :49-50
    "acc_cost.txt": ("acc_cost", 10, (3, 3, 1, 1)),                        # :483-484
    "Lidar_omg_after_rot.txt": ("Lidar_omg_after_rot", 12, (3, 1)),        # :398-399
}


def log_row(values, precision: int, groups) -> str:
    """One row of an LI_Init log: the stream's default float format at `precision` significant digits, each Eigen object's
    coefficients right-aligned to its widest one (eigen_str)."""
    fmt = lambda v: "%.*g" % (precision, v)   # noqa: E731
    out, i = [], 0
    for g in groups:
        out.append(eigen_str(values[i:i + g], fmt))
        i += g
    return " ".join(out) + "\n"


def refine_result_lines(state, time_lag) -> list:
    """print_refine_result (laserMapping.cpp:727-743), without the terminal colours."""
    v = state_calib_values(state, time_lag)
    f = lambda x: eigen_str(x, _fixed6)    # noqa: E731
    return ["[Final Result] Rotation LiDAR to IMU    = " + f(v["euler_deg"]) + " deg",
            "[Final Result] Translation LiDAR to IMU = " + f(v["T_LI"]) + " m",
            "[Final Result] Time Lag IMU to LiDAR    = %.8f s " % time_lag,
            "[Final Result] Bias of Gyroscope        = " + f(v["bias_g"]) + " rad/s",
            "[Final Result] Bias of Accelerometer    = " + f(v["bias_a"]) + " m/s^2",
            "[Final Result] Gravity in World Frame   = " + f(v["gravity"]) + " m/s^2"]


def refine_tick(frame_num: int, orig_odom_freq: int, cut_frame_num: int) -> bool:
    """The refinement clock's condition `frame_num % orig_odom_freq * cut_frame_num == 0` (:1169) with C++ precedence:
    (frame_num % orig_odom_freq) * cut_frame_num == 0."""
    return (frame_num % orig_odom_freq) * cut_frame_num == 0


class Log:
    """Progress and warnings on stderr; colour only on a terminal."""

    def __init__(self, stream=None, quiet=False):
        self.s = sys.stderr if stream is None else stream
        self.quiet = quiet
        self.color = hasattr(self.s, "isatty") and self.s.isatty()

    def info(self, msg, color="36"):
        if not self.quiet:
            self.s.write((f"\x1b[1;{color}m{msg}\x1b[0m" if self.color else msg) + "\n")
            self.s.flush()

    def warn(self, msg):
        self.info("[WARN] " + msg, "33")


class Recorder:
    """The node's publishers (laserMapping.cpp:561-706) into a bag writer (bagwrite), called after every update with the update's
    lidar_end_time, the set_posestamp pose and LidarOdometry.published. In the order of the loop (:1137-1157): /aft_mapped_to_init and
    its /tf transform (publish_odometry), then /cloud_registered, /cloud_registered_body and /cloud_effected as far as they were
    published, then /path on every 5th call (publish_path's static counter), a growing list of PoseStamped whose header keeps the stamp
    set once at start-up (:804, lidar_end_time = 0 then). Every other stamp is lidar_end_time, and so is every record time. /Laser_map
    has no message: publish_map has no caller. Only `topics` are written."""
    FRAME, CHILD = "camera_init", "aft_mapped"

    def __init__(self, writer, cfg: cfgmod.Config, topics=cfgmod.RECORD_TOPICS):
        self.w, self.topics, self.path_en = writer, frozenset(topics), cfg.path_en
        self.path_calls = 0
        self.path_poses = []
        self.path_stamp = pubmsg.ros_time(0.0)

    def update(self, t: float, pos, quat, published: dict):
        stamp, enc, topics, F = pubmsg.ros_time(t), self.w.encoding, self.topics, self.FRAME

        def put(topic, type_, data):
            self.w.write(topic, type_, stamp, data)
        if "/aft_mapped_to_init" in topics:
            put("/aft_mapped_to_init", pubmsg.ODOMETRY, pubmsg.odometry(stamp, F, self.CHILD, pos, quat, enc))
        if "/tf" in topics:
            put("/tf", pubmsg.TF_MESSAGE, pubmsg.tf_message(stamp, F, self.CHILD, pos, quat, enc))
        for key, topic in cfgmod.CLOUD_TOPICS.items():
            if key in published and topic in topics:
                put(topic, pubmsg.POINTCLOUD2, pubmsg.pointcloud2(stamp, F, published[key], enc))
        if self.path_en:
            self.path_calls += 1
            if self.path_calls % 5 == 0:
                self.path_poses.append((stamp, F, tuple(pos), tuple(quat)))
                if "/path" in topics:
                    put("/path", pubmsg.PATH, pubmsg.path(self.path_stamp, F, self.path_poses, enc))

    def close(self):
        self.w.close()


class Node:
    """laserMapping's main(): node.imu_cbk / node.livox_cbk / node.pcl2_cbk deliver messages, each followed by node.spin(); node.run(bag)
    does both over a bag; node.close() ends the run (pcd_save's last file, the end-of-run report)."""

    def __init__(self, cfg: cfgmod.Config, odom: LidarOdometry, out_dir: str, log: Log | None = None):
        self.cfg, self.odom, self.log = cfg, odom, log or Log()
        odom.preprocess = cfgmod.preprocess(cfg)
        self.out_dir = out_dir
        for d in ("result", "Log"):
            os.makedirs(os.path.join(out_dir, d), exist_ok=True)
        self.f_result = open(os.path.join(out_dir, "result", "Initialization_result.txt"), "w")
        self.f_mat = open(os.path.join(out_dir, "Log", "mat_out.txt"), "w")
        self.f_traj = open(os.path.join(out_dir, "result", "trajectory.txt"), "w")
        # imu_cbk's statics (:388-389)
        self.imu_cnt, self.mean_acc, self.imu_period, self.last_time_msg_in = 0, np.zeros(3), 0.0, 0.0
        self.total_distance, self.position_last = 0.0, np.zeros(3)   # :79,131
        self.online_calib_starts_time, self.online_calib_finish, self.refine_print = 0.0, False, False
        self.init_scan = self.refine_scan = None    # frame_num of the trigger scan / of the scan that completed the refinement
        self.init_result = None                     # LI_Initialization's result (calib.LiCalib.initialize)
        self.init_state = self.refine_state = None  # the states written under "Initialization result:" / "Refinement result:"
        self.updates = 0
        self.on_update = None                       # callback(node) after every update's output rows, for tests and tools
        self.recorder = None                        # a Recorder: the published topics of every update go to its bag
        self.assess = None                          # an assess.Assessment: every LIO update but the switch scan stores its cloud
        self.replay = None                          # an assess.Replay: captures the hand-over, records the LIO phase's input and updates
        self.debug_logs = None                      # open_debug_logs(): {file name: open file} of LI_Init's logs
        self.closed = False

    def open_debug_logs(self):
        """Create LI_Init's six logs in <out>/Log/, empty until the trigger writes them (LI_init.cpp:11-16)."""
        self.debug_logs = {name: open(os.path.join(self.out_dir, "Log", name), "w") for name in DEBUG_LOGS}

    def _write_debug_logs(self):
        calib = self.odom.calib
        for name, f in self.debug_logs.items():
            table, precision, groups = DEBUG_LOGS[name]
            f.write("".join(log_row(r, precision, groups) for r in calib.log_rows(table)))
            f.flush()

    @property
    def time_lag(self) -> float:
        """time_lag_IMU_wtr_lidar + timediff_imu_wrt_lidar"""
        return self.odom.imu_buffer.time_lag + self.odom.imu_buffer.timediff

    # ---- callbacks ----
    def imu_cbk(self, stamp: float, gyr, acc):
        """imu_cbk (:384-434). The time compensation and the loop-back clear of imu_buffer are ImuBuffer.push; the running statistics,
        the clear of the calibration's IMU samples and the push into the calibration are here."""
        if self.imu_cnt < 100:
            self.imu_cnt += 1
            self.mean_acc += (np.asarray(acc, float) - self.mean_acc) / self.imu_cnt
            if self.imu_cnt > 1:
                self.imu_period += (stamp - self.last_time_msg_in - self.imu_period) / (self.imu_cnt - 1)
            if self.imu_cnt == 99:
                self.log.info("Acceleration norm  : %g" % np.linalg.norm(self.mean_acc))
                if self.imu_period > 0.01:
                    self.log.info("IMU data frequency : %g Hz" % (1 / self.imu_period))
                    self.log.warn("IMU data frequency too low. Higher than 150 Hz is recommended.")
        self.last_time_msg_in = stamp
        o, ib = self.odom, self.odom.imu_buffer
        t = float(stamp) - ib.timediff - ib.time_lag
        if t < ib.last_stamp:
            self.log.warn("IMU loop back, clear IMU buffer.")
            o.calib.clear_imu_all()                 # Init_LI->IMU_buffer_clear() (:420)
        ib.push(stamp, gyr, acc)
        if self.replay is not None:
            self.replay.record_imu(stamp, gyr, acc)
        if not o.imu_en and not o.data_accum_finished:
            o.push_imu(gyr, acc, ib.last_stamp, self.cfg.mean_acc_norm)   # push_ALL_IMU_CalibState (:428-430)

    def livox_cbk(self, stamp: float, points):
        had = self.odom.timediff_set
        self.odom.lidar_cbk_livox(points, stamp)
        self._note_sync(had)

    def pcl2_cbk(self, stamp: float, data, layout, n: int):
        had = self.odom.timediff_set
        self.odom.lidar_cbk_pcl2(data, layout, n, stamp)
        self._note_sync(had)

    def _note_sync(self, had):
        if self.odom.timediff_set and not had:
            self.log.info("Self sync IMU and LiDAR, HARD time lag is %.10f" % self.odom.imu_buffer.timediff)

    # ---- the loop ----
    def spin(self):
        """The loop body on every sub-frame sync_packages can deliver now."""
        o = self.odom
        while True:
            frame_num = o.frame_num
            if o.process_next() is None:
                return
            if o.frame_num != frame_num:            # an update ran (the map-building scan returns before it, :921-931)
                self._after_update()

    def _after_update(self):
        o, s = self.odom, self.odom.state
        R, p, RLI, TLI = host.state_pose(s)
        self.updates += 1
        # the covariance update of the last iteration (:1110-1127): flg_EKF_inited is always true and liinit_scan_update always
        # leaves through that branch, so total_distance / position_last / geoQuat follow every update
        self.total_distance += float(np.linalg.norm(p - self.position_last))
        self.position_last = p
        euler_cur = rot_to_euler(R)                 # euler_cur of the last iteration (:1099)
        if not o.imu_en:
            q = quat_from_rpy(*euler_cur)
            pos = p
        else:                                       # the LiDAR's pose (:1120-1125, set_posestamp :651-656)
            q = quat_from_rpy(*rot_to_euler(R @ RLI))
            pos = R @ TLI + p
        t = o.lidar_end_time
        self.f_traj.write("%.9f %s %s\n" % (t, " ".join("%.9g" % v for v in pos), " ".join("%.9g" % v for v in q)))
        self.f_mat.write(state_mat_out_row(s, euler_cur, self.total_distance))
        if self.recorder is not None:
            self.recorder.update(t, pos, q, o.published)
        # (the switch scan re-filters the previous scan's cloud; LiDAR-only updates have no extrinsic in the model)
        if self.assess is not None and o.imu_en and o.switch_scan != o.frame_num - 1:
            timing = getattr(o, "timing", None)
            if getattr(self.assess, "timed", False) and timing is not None and len(timing[0]) >= 2:
                self.assess.append_timed(R, p, RLI, TLI, *timing)   # the scan's raw cloud, pose table and propagated state
            else:
                self.assess.append(R, p, RLI, TLI)
        if self.replay is not None:
            self.replay.record_update(s)
        if self.on_update is not None:               # the posterior of the update, before the hand-over of a trigger scan
            self.on_update(self)
        # the refinement clock (:1169-1187)
        if o.imu_en and refine_tick(o.frame_num, o.orig_odom_freq, o.cut_frame_num) and not self.online_calib_finish:
            comp = t - self.online_calib_starts_time
            comp = comp if comp < self.cfg.online_refine_time else self.cfg.online_refine_time
            if self.cfg.online_refine_time > 0.1:
                self.log.info("[Refinement] Online Refinement: %3d%%" % int(comp / self.cfg.online_refine_time * 100), "35")
            if not self.refine_print and comp > self.cfg.online_refine_time - 1e-6:
                self.refine_print = self.online_calib_finish = True
                self.refine_scan = o.frame_num
                self.refine_state = s.copy()
                print("\n".join(refine_result_lines(s, self.time_lag)), flush=True)
                self.f_result.write("Refinement result:\n" + calib_result_text(**state_calib_values(s, self.time_lag)))
                self.f_result.flush()
                self.log.info("Initialization and refinement result is written to " +
                              os.path.join(self.out_dir, "result", "Initialization_result.txt"), "32")
        # the trigger (:1190-1233): LidarOdometry has pushed the scan and assessed the data; LI_Initialization and the hand-over run now
        if not o.imu_en and o.data_accum_finished:
            self.init_result = res = o.initialize(o.imu_buffer.timediff)
            if self.debug_logs is not None:
                self._write_debug_logs()
            self.online_calib_starts_time = t
            if self.replay is not None:
                self.replay.capture(o, res)         # the LiDAR-only state and the map as LI-Init found them
            o.hand_over(res)
            self.init_scan = o.frame_num
            self.init_state = o.state.copy()
            self.log.info("[Initialization] LI-Init done at %.6f s; online refinement of %g s starts" % (t, self.cfg.online_refine_time), "32")
            self.f_result.write("Initialization result:\n" + calib_result_text(**state_calib_values(o.state, self.time_lag)))
            self.f_result.flush()
        if not o.imu_en and o.data_accum_start and self.updates % 50 == 0:
            self.log.info("[Initialization] data accumulation, frame %d" % o.frame_num)

    def run(self, bag):
        """Deliver every message of the configured LiDAR and IMU topics in playback order, each followed by spin(). bag: a
        rosbag.Bag or a rosbag2.Bag2; its `format` picks the decoders (rosmsg.decoders)."""
        c = self.cfg
        if c.lid_topic == c.imu_topic:
            raise cfgmod.ConfigError(f"common/lid_topic and common/imu_topic are both {c.lid_topic!r}")
        dec = rosmsg.decoders(bag.format, c.lidar_type)
        wanted = cfgmod.wanted_topics(c, bag.format)
        total = bag.count(wanted)
        types = bag.topics()
        self.log.info(f"{bag.path}: {total} messages on {c.lid_topic} [{types[c.lid_topic]}] and {c.imu_topic} [{types[c.imu_topic]}]")
        lidar_cbk = self.livox_cbk if c.lidar_type == 1 else self.pcl2_cbk
        for i, m in enumerate(bag.messages(wanted)):
            try:
                if m.topic == c.imu_topic:
                    self.imu_cbk(*dec.imu(m.data))
                else:
                    lidar_cbk(*dec.lidar(m.data))
            except rosmsg.MsgError as e:
                raise rosmsg.MsgError(f"{bag.path}: message {i} on {m.topic} at record time {m.sec}.{m.nsec:09d}: {e}") from None
            self.spin()
        return self

    def close(self, report: bool = True):
        """The end of the run (:1236-1244, SigHandle's pcd_save): the refinement report, with a warning when it did not finish."""
        if self.closed:
            return
        self.closed = True
        self.odom.close()
        for f in (self.f_result, self.f_mat, self.f_traj, *(self.debug_logs or {}).values()):
            f.close()
        if self.recorder is not None:
            self.recorder.close()
        if not report:
            return
        if self.init_result is None:
            self.log.warn("LI-Init did not run: the data accumulated did not reach the excitation it needs (data_accum_length "
                          f"{self.cfg.data_accum_length:g}); Initialization_result.txt is empty")
        if not self.online_calib_finish:
            self.log.warn("Online refinement not finished yet.")
            print("\n".join(refine_result_lines(self.odom.state, self.time_lag)), flush=True)
