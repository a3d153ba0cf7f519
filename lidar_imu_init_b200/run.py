"""Run LI-Init on a recorded ROS1 or ROS 2 bag, without ROS:

    python -m lidar_imu_init_b200.run --config avia.yaml --bag rec.bag [--out DIR] [--param name=value ...] [--device N]
                                      [--max-map-points N] [--record PATH [--record-format ros1|ros2]
                                      [--record-compression none|bz2] [--record-topics a,b,...]] [--debug-logs]
                                      [--assess] [--assess-cloud PATH [--assess-cloud-leaf L]] [--assess-radius R]
                                      [--assess-max-points N] [--assess-time] [--assess-replay] [--assess-replay-max-points N]
                                      [--refine [--refine-max-replays N] [--profile]]

--bag is a ROS1 bag (v2.0), a rosbag2 directory (sqlite3 storage) or one of its .db3 files, told apart by the file's first bytes. The
LiDAR topic carries livox_ros_driver/CustomMsg or livox_ros_driver2/CustomMsg (lidar_type 1) or sensor_msgs/PointCloud2 in a ROS1
bag, and livox_ros_driver2/msg/CustomMsg or sensor_msgs/msg/PointCloud2 in a ROS 2 bag.

The config is one of the reference's config/*.yaml as it ships; --param sets a launch-file <param> (point_filter_num, max_iteration,
cube_side_length) or any other node parameter. Writes DIR/result/Initialization_result.txt, DIR/Log/mat_out.txt,
DIR/result/trajectory.txt and, with pcd_save_en, DIR/PCD/. Prints print_refine_result's lines on stdout; progress goes to stderr.
Exits 0 on success, 1 on a bag, message, config or library error, with a message that says what was wrong and where.

--record PATH writes the node's published topics (/cloud_registered, /cloud_registered_body, /cloud_effected, /aft_mapped_to_init,
/tf, /path; --record-topics chooses some) under the node's publish/* parameters into a new bag: a ROS1 bag for a ROS1 input, a rosbag2
directory for a ROS 2 input, or as --record-format says. --debug-logs writes LI-Init's six logs to DIR/Log/.

--assess stores the LIO scans on the device and, at the end of the run, scores the calibration by how sharp a map it builds: the mean
map entropy and plane variance of the as-run, final and perturbed extrinsics, written to DIR/result/assessment.txt (assess).
--assess-cloud PATH (with or without --assess) writes where the as-run map is blurred: the entropy and plane variance of every stored
point, averaged over cubic leaves of --assess-cloud-leaf metres (0: every point), as a binary PCD.
--assess-time also keeps each LIO scan's raw cloud and IMU pose table, re-undistorts the scans for every candidate, and scores the
time lag too: the 14 candidates and a lag profile around the run's lag, written to DIR/result/assessment_time.txt.
--assess-replay keeps the map at the hand-over and the LIO phase's sub-frames and IMU samples, and runs the LIO phase again for every
candidate with the candidate extrinsic held constant: the run itself, LI-Init's result, the final extrinsic, its 12 perturbations and
the final extrinsic at lag shifts of -+5 ms, each scored by the sharpness of the map its replay builds, written to
DIR/result/assessment_replay.txt (stores the LIO scans like --assess).
--refine records the LIO phase as --assess-replay does and searches, by replay, for the lag shift and then the extrinsic whose map is
sharpest, starting from the better of LI-Init's result and the final extrinsic, within --refine-max-replays replays (default 120). It
writes every replay, the end condition of each axis and the refined calibration, in the format of Initialization_result.txt, to
DIR/result/refinement.txt, and leaves Initialization_result.txt as it is.
--profile (with --refine) then replays a profile through the refined calibration along each of its seven parameters (rotation about
each IMU axis, translation along it, the lag), 6 steps each side, and fits where each profile has its minimum: a verdict and an
interval per parameter in degrees, metres and milliseconds, written to DIR/result/profile.txt (profiles.py).
"""
from __future__ import annotations

import argparse
import os
import sys
import time

from . import assess as assessmod
from . import bagwrite
from . import config as cfgmod
from . import profiles as profilesmod
from . import refine as refinemod
from . import rosbag, rosbag2, rosmsg


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m lidar_imu_init_b200.run", description=__doc__.split("\n\n")[0],
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config", required=True, help="a reference config YAML (config/avia.yaml, ouster.yaml, ...)")
    ap.add_argument("--bag", required=True, help="ROS1 bag (v2.0), rosbag2 directory or .db3 file with the LiDAR and IMU topics of "
                    "the config")
    ap.add_argument("--out", default=".", help="output directory, laid out like the node's package directory (default: .)")
    ap.add_argument("--param", action="append", default=[], metavar="NAME=VALUE",
                    help="a node parameter, e.g. max_iteration=5 point_filter_num=2 cube_side_length=2000 (repeatable)")
    ap.add_argument("--device", type=int, default=0, help="CUDA device (default 0)")
    ap.add_argument("--max-map-points", type=int, default=6_000_000, help="capacity of the device map (default 6000000)")
    ap.add_argument("--max-scan-points", type=int, default=300_000, help="capacity of a scan on the device (default 300000)")
    ap.add_argument("--quiet", action="store_true", help="no progress on stderr")
    ap.add_argument("--record", metavar="PATH", help="record the node's published topics into a new bag at PATH")
    ap.add_argument("--record-format", choices=bagwrite.FORMATS, help="ros1 (a .bag file) or ros2 (a rosbag2 directory); default: "
                    "the format of --bag")
    ap.add_argument("--record-compression", choices=bagwrite.COMPRESSIONS, default="none", help="chunk compression of a ROS1 "
                    "recording (default none)")
    ap.add_argument("--record-topics", metavar="TOPIC,...", help="the topics to record, comma-separated (default: all of "
                    + ", ".join(cfgmod.RECORD_TOPICS) + ")")
    ap.add_argument("--debug-logs", action="store_true", help="write LI-Init's logs (LiDAR_meas.txt, IMU_meas.txt, ...) to DIR/Log/")
    ap.add_argument("--assess", action="store_true", help="score the calibration by the sharpness of the map of the LIO scans: "
                    "DIR/result/assessment.txt")
    ap.add_argument("--assess-radius", type=float, default=assessmod.RADIUS, metavar="R",
                    help=f"neighbourhood radius of the assessment [m] (default {assessmod.RADIUS:g})")
    ap.add_argument("--assess-cloud", metavar="PATH", help="write the per-point map entropy and plane variance of the as-run map, "
                    "thinned to leaves, as a binary PCD at PATH (stores the LIO scans like --assess)")
    ap.add_argument("--assess-cloud-leaf", type=float, default=assessmod.CLOUD_LEAF, metavar="L",
                    help=f"leaf edge of --assess-cloud [m] (default {assessmod.CLOUD_LEAF:g}; 0: one record per stored point)")
    ap.add_argument("--assess-max-points", type=int, default=assessmod.MAX_POINTS, metavar="N",
                    help=f"LIO points the assessment stores on the device (default {assessmod.MAX_POINTS}); later scans are skipped")
    ap.add_argument("--assess-time", action="store_true", help="score the time lag too, re-undistorting the stored LIO scans for every "
                    "candidate: DIR/result/assessment_time.txt (stores the LIO scans like --assess)")
    ap.add_argument("--assess-replay", action="store_true", help="run the LIO phase again for every candidate calibration, extrinsic "
                    "held constant, and score the map each replay builds: DIR/result/assessment_replay.txt (stores the LIO scans like "
                    "--assess)")
    ap.add_argument("--assess-replay-max-points", type=int, default=assessmod.REPLAY_MAX_POINTS, metavar="N",
                    help=f"raw LIO-phase points the replay keeps on the device (default {assessmod.REPLAY_MAX_POINTS}); a run that "
                    "outgrows it is not replayed")
    ap.add_argument("--refine", action="store_true", help="search, by LIO replay, for the lag and extrinsic whose map is sharpest and "
                    "write the refined calibration: DIR/result/refinement.txt (records the replay like --assess-replay)")
    ap.add_argument("--refine-max-replays", metavar="N", help=f"replays the refinement may spend (default {refinemod.MAX_REPLAYS})")
    ap.add_argument("--profile", action="store_true", help="after --refine, replay a profile through the refined calibration along "
                    "each parameter and fit where its minimum lies: DIR/result/profile.txt")
    ap.add_argument("--replay-jobs", metavar="K", help="replays of --assess-replay and --refine run at once, each on its own device "
                    "context sharing the recorded replay (default 1)")
    return ap.parse_args(argv)


def replay_jobs(args) -> int:
    """--replay-jobs as a positive integer (1 when it is not given)."""
    if args.replay_jobs is None:
        return 1
    try:
        n = int(args.replay_jobs)
    except ValueError:
        n = 0
    if n < 1:
        raise cfgmod.ConfigError(f"--replay-jobs {args.replay_jobs!r}: must be a positive integer")
    return n


def refine_max_replays(args) -> int:
    """--refine-max-replays as a positive integer (refine.MAX_REPLAYS when it is not given)."""
    if args.refine_max_replays is None:
        return refinemod.MAX_REPLAYS
    try:
        n = int(args.refine_max_replays)
    except ValueError:
        n = 0
    if n < 1:
        raise cfgmod.ConfigError(f"--refine-max-replays {args.refine_max_replays!r}: must be a positive integer")
    return n


def record_topics(args) -> tuple:
    """The topics --record-topics names (all the node publishes when it is not given)."""
    if args.record_topics is None:
        return cfgmod.RECORD_TOPICS
    topics = tuple(dict.fromkeys(t.strip() for t in args.record_topics.split(",") if t.strip()))
    bad = [t for t in topics if t not in cfgmod.RECORD_TOPICS]
    if bad or not topics:
        raise cfgmod.ConfigError(f"--record-topics {args.record_topics!r}: {'unknown topic ' + repr(bad[0]) if bad else 'no topic'}; "
                                 f"the node publishes {', '.join(cfgmod.RECORD_TOPICS)}")
    return topics


def make_node(args, cfg, log):
    from . import capi
    from .node import Node
    from .odometry import LidarOdometry
    g = capi.LiInitGpu(cfg.filter_size_map, max_map_points=args.max_map_points, max_scan_points=args.max_scan_points, device_id=args.device)
    kw = cfgmod.odometry_kwargs(cfg, pcd_dir=os.path.join(args.out, "PCD"), record_topics=record_topics(args) if args.record else None)
    odom = LidarOdometry(g, **kw)
    return Node(cfg, odom, args.out, log)


def play(args, log, on_node=None, jobs: int = 1):
    """Plays args.bag through a new Node with what args asks it to store (--assess*, --refine, --record, --debug-logs) and closes the
    node, which writes its result files. Returns (node, wall seconds of the bag): the node's context, assessment store and replay stay
    open for the caller to use and close. on_node(node), when given, is called before the bag is played; jobs: the replay's jobs of
    Replay.write and write_refinement. On an error the node and the recording are closed and the error is raised."""
    from .node import Recorder
    node = writer = None
    try:
        cfg = cfgmod.load(args.config, args.param)
        topics = record_topics(args)
        replaying = args.assess_replay or args.refine
        assessing = args.assess or args.assess_cloud is not None or args.assess_time or replaying
        if assessing and not (args.assess_radius > 0 and args.assess_radius < float("inf")):
            raise cfgmod.ConfigError(f"--assess-radius {args.assess_radius!r}: must be a positive number of metres")
        if args.assess_cloud is not None and not (args.assess_cloud_leaf >= 0 and args.assess_cloud_leaf < float("inf")):
            raise cfgmod.ConfigError(f"--assess-cloud-leaf {args.assess_cloud_leaf!r}: must be zero or a positive number of metres")
        if assessing and args.assess_max_points < 1:
            raise cfgmod.ConfigError(f"--assess-max-points {args.assess_max_points}: must be positive")
        if replaying and args.assess_replay_max_points < 1:
            raise cfgmod.ConfigError(f"--assess-replay-max-points {args.assess_replay_max_points}: must be positive")
        with rosbag2.open_bag(args.bag) as bag:
            bag.check_topics(cfgmod.wanted_topics(cfg, bag.format))
            if args.record:
                fmt = args.record_format or ("ros1" if bag.format == "ros1" else "ros2")
                writer = bagwrite.open_writer(args.record, fmt, args.record_compression)
            log.info(f"lidar_type: {cfg.lidar_type} ({cfgmod.LIDAR_NAMES[cfg.lidar_type]}); LiDAR-only odometry starts.")
            node = make_node(args, cfg, log)
            if writer is not None:
                node.recorder = Recorder(writer, cfg, topics)
            if args.debug_logs:
                node.open_debug_logs()
            if assessing:
                node.assess = assessmod.Assessment(node.odom.g, args.assess_max_points, args.assess_radius, timed=args.assess_time)
                node.odom.assess_hold = args.assess_time
            if replaying:
                node.replay = node.odom.replay = assessmod.Replay(node.odom.g, node.assess, args.assess_replay_max_points)
                node.replay.jobs = jobs
            if on_node is not None:
                on_node(node)
            t0 = time.perf_counter()
            node.run(bag)
            wall = time.perf_counter() - t0
        node.close()
        return node, wall
    except BaseException:
        # an interrupted run (Ctrl-C) still closes its files and its recording, so the bag it leaves is complete
        _abort(node, writer)
        raise


def main(argv=None, on_node=None) -> int:
    """The command line; on_node(node), when given, is called with the Node before the bag is played (for tools and tests)."""
    from . import host
    from .node import Log
    args = parse_args(argv)
    log = Log(quiet=args.quiet)
    try:
        max_replays = refine_max_replays(args) if args.refine else None
        if args.profile and not args.refine:
            raise cfgmod.ConfigError("--profile profiles the refined calibration: it needs --refine")
        jobs = replay_jobs(args)
        replaying = args.assess_replay or args.refine
        node, wall = play(args, log, on_node, jobs)      # (closed: the error paths below have nothing left to close)
        if args.assess:
            t0 = time.perf_counter()
            node.assess.write(os.path.join(args.out, "result", "assessment.txt"))
            log.info(f"assessment written to {os.path.join(args.out, 'result', 'assessment.txt')} in {time.perf_counter() - t0:.1f} s")
        if args.assess_time:
            t0 = time.perf_counter()
            path = os.path.join(args.out, "result", "assessment_time.txt")
            node.assess.write_time(path, node.time_lag)
            log.info(f"time assessment written to {path} in {time.perf_counter() - t0:.1f} s")
        if args.assess_cloud is not None:
            t0 = time.perf_counter()
            got = node.assess.write_cloud(args.assess_cloud, args.assess_cloud_leaf)
            if got is None:
                log.warn(f"{args.assess_cloud} not written: {assessmod.NOTHING.strip()}")
            else:
                log.info(f"assessment cloud written to {args.assess_cloud}: {got[0]} records, full-resolution MME {got[1]['mme']:.6f} over "
                         f"{got[1]['valid']} of {got[1]['points']} points, in {time.perf_counter() - t0:.1f} s")
        if args.assess_replay:
            # (last: every replay refills the assessment store)
            t0 = time.perf_counter()
            path = os.path.join(args.out, "result", "assessment_replay.txt")
            _, _, R_final, T_final = host.state_pose(node.odom.state)
            node.replay.write(path, R_final, T_final)
            log.info(f"replay assessment written to {path} in {time.perf_counter() - t0:.1f} s ({jobs} replay job{'s' if jobs > 1 else ''})")
        if args.refine:
            # (after --assess-replay: every replay refills the assessment store)
            path = os.path.join(args.out, "result", "refinement.txt")
            _, _, R_final, T_final = host.state_pose(node.odom.state)
            ref = node.replay.write_refinement(path, R_final, T_final, max_replays)
            if ref is None:
                log.warn(f"{path}: {assessmod.NOTHING.strip()}")
            else:
                log.info(refine_summary(path, ref, jobs))
            if args.profile:
                path = os.path.join(args.out, "result", "profile.txt")
                prof = node.replay.write_profile(path, ref)
                if prof is None:
                    log.warn(f"{path}: {assessmod.NOTHING.strip()}")
                else:
                    log.info(profile_summary(path, prof, jobs))
        if replaying:
            node.replay.close()
        node.odom.g.close()
        log.info(f"{node.updates} updates in {wall:.1f} s; {node.odom.dropped_subframes} sub-frames dropped")
        return 0
    except errors() as e:
        sys.stderr.write(f"error: {e}\n")
        return 1


def errors() -> tuple:
    """The errors the command line reports with a message and exit code 1."""
    from . import calib, capi
    return cfgmod.ConfigError, rosbag.BagError, rosmsg.MsgError, capi.LiInitError, calib.CalibError, assessmod.ReplayError, OSError


def refine_summary(path: str, ref: dict, jobs: int = 1) -> str:
    """The refinement's summary line: the replays and jobs, the lag, extrinsic change and MME from the start candidate to the refined
    one."""
    import numpy as np
    s = ref["trace"][[r["stage"] for r in ref["trace"]].index(ref["start"])]
    c = np.clip((np.trace(ref["R"] @ s["R"].T) - 1.0) / 2.0, -1.0, 1.0)
    return (f"refinement written to {path}: {len(ref['trace'])} replays in {ref['wall_s']:.1f} s ({ref['status']}, {jobs} replay "
            f"job{'s' if jobs > 1 else ''}); lag "
            f"{ref['lag0'] * 1000.0:.3f} -> {ref['time_lag'] * 1000.0:.3f} ms; from {ref['start']}: rotation {np.degrees(np.arccos(c)):.4f} deg, "
            f"translation {np.linalg.norm(ref['T'] - s['T']) * 1000.0:.2f} mm; MME {s['mme']:.6f} -> {ref['mme']:.6f}")


def profile_summary(path: str, prof: dict, jobs: int = 1) -> str:
    """The profile's summary line: the replays and jobs, then per parameter its verdict and the interval of its minimum in its unit;
    a `pinned` fit whose minimum lies a step or more from the profile's lowest point (profiles.off_lowest) says so."""
    parts = []
    for p, f in prof["fits"].items():
        unit = profilesmod.UNITS[p.split("_")[0]]
        iv = f" [{f['lo_phys']:.4f}, {f['hi_phys']:.4f}] {unit}" if f["verdict"] in ("pinned", "edge") else ""
        if f["verdict"] == "pinned" and profilesmod.off_lowest(f):
            iv += f" (off the profile's lowest point, k {f['lower_k']:+d}: the parabola misfits)"
        parts.append(f"{p} {f['verdict']}{iv}")
    return (f"profile written to {path}: {prof['replays']} replays in {prof['wall_s']:.1f} s ({jobs} replay job{'s' if jobs > 1 else ''}); "
            + ", ".join(parts))


def _abort(node, writer):
    if node is not None and not node.closed:
        node.close(report=False)                    # closes the recording too
    elif node is None and writer is not None:
        writer.close()


if __name__ == "__main__":
    sys.exit(main())
