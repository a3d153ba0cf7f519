"""ROS 2 bags and livox_ros_driver2 recordings on the H100: `python -m lidar_imu_init_b200.run` (as a function call) on a ROS 2 bag and
on its ROS1 twin (the same messages, the same record times) must run bit-identically.

Livox: the 60 s scenario of tests/test_gpu_bag.py as a rosbag2 directory of livox_ros_driver2/msg/CustomMsg (three split files, short
and padded messages), and as a ROS1 bag typed livox_ros_driver2/CustomMsg, each against the livox_ros_driver ROS1 bag. Ouster: the
10 s LiDAR-only PointCloud2 scenario, with and without the `t` field, as ROS 2 and as ROS1."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_bag2_node as t2  # noqa: E402  (the rosbag2 writer, the CDR serializers)
import test_bag_node as tb  # noqa: E402
import test_gpu_bag as tg  # noqa: E402  (the CLI runner and the Ouster scenario)

OUT_FILES = t2.OUT_FILES


def _same_run(a, b, out_a, out_b):
    """Bit-identical states at every update, the same trigger, calibration and refinement, byte-identical result files."""
    na, nb = a["node"], b["node"]
    assert len(a["states"]) == len(b["states"]) > 0
    for j, (x, y) in enumerate(zip(a["states"], b["states"])):
        np.testing.assert_array_equal(x, y, err_msg=f"update {j}")
    assert a["end_times"] == b["end_times"]
    assert (na.init_scan, na.refine_scan, na.updates) == (nb.init_scan, nb.refine_scan, nb.updates)
    if na.init_result is not None:
        for key in ("R_LI", "T_LI", "grav_L0", "gyro_bias", "acc_bias", "time_lag_1", "time_lag_2"):
            np.testing.assert_array_equal(na.init_result[key], nb.init_result[key])
    assert na.odom.dropped_subframes == nb.odom.dropped_subframes == 0
    for d, f in OUT_FILES:
        assert open(os.path.join(out_a, d, f), "rb").read() == open(os.path.join(out_b, d, f), "rb").read(), f


@pytest.fixture(scope="module")
def livox_ros1(gpu_lib, tmp_path_factory):
    """The 60 s Livox scenario as the livox_ros_driver ROS1 bag of tests/test_gpu_bag.py, run through the CLI."""
    from lidar_imu_init_b200 import _build
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("livox")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    out = str(tmp / "out_ros1")
    seen = tg._run_cli(str(tmp / "sim.yaml"), bag, out)
    print(f"ROS1 livox_ros_driver: {len(seen['states'])} updates, trigger at frame {seen['node'].init_scan}, refinement done at frame "
          f"{seen['node'].refine_scan}", flush=True)
    assert seen["node"].init_scan is not None and seen["node"].refine_scan is not None and len(seen["states"]) > 2000
    return dict(tmp=tmp, ev=ev, seen=seen, out=out)


@pytest.mark.gpu
def test_livox_ros2_bag_sixty_seconds(livox_ros1):
    tmp, ev = livox_ros1["tmp"], livox_ros1["ev"]
    d = str(tmp / "livox_ros2")
    paths = t2.write_event_bag2(d, ev, files=3)
    assert len(paths) == 3
    out = str(tmp / "out_ros2")
    seen = tg._run_cli(str(tmp / "sim.yaml"), d, out)
    _same_run(livox_ros1["seen"], seen, livox_ros1["out"], out)


@pytest.mark.gpu
def test_livox2_ros1_bag_sixty_seconds(livox_ros1):
    tmp, ev = livox_ros1["tmp"], livox_ros1["ev"]
    bag = str(tmp / "livox2.bag")
    t2.write_event_bag_livox2(bag, ev)
    out = str(tmp / "out_livox2")
    seen = tg._run_cli(str(tmp / "sim.yaml"), bag, out)
    _same_run(livox_ros1["seen"], seen, livox_ros1["out"], out)


@pytest.mark.gpu
@pytest.mark.parametrize("with_time", [True, False])
def test_ouster_ros2_bag_lidar_only(gpu_lib, tmp_path, with_time):
    from lidar_imu_init_b200 import _build, rosmsg
    _build.build_host()
    _build.build_calib()
    ev, _ = tg._ouster_events(10.0, 20_000, with_time)
    text = ("common:\n  lid_topic: /ouster/points\n  imu_topic: /imu/data\npreprocess:\n  lidar_type: 3\n  scan_line: 16\n  blind: 0.5\n"
            "initialization:\n  cut_frame_num: 2\n  orig_odom_freq: 10\n  mean_acc_norm: 9.81\n  online_refine_time: 15\n  data_accum_length: 100000\n"
            "  Rot_LI_cov: [0.00005, 0.00005, 0.00005]\n  Trans_LI_cov: [0.0001, 0.0001, 0.0001]\n"
            "mapping:\n  filter_size_surf: 0.15\n  filter_size_map: 0.15\n  gyr_cov: 0.1\n  acc_cov: 0.1\n")
    (tmp_path / "ouster.yaml").write_text(text)
    recs = t2.event_records(ev)
    bag1 = str(tmp_path / "ouster.bag")
    r1 = [(0, t // 10**9, t % 10**9, tb.ser_imu(sec, nsec, *pl)) if kind == "imu" else
          (1, t // 10**9, t % 10**9, tb.ser_pcl2(sec, nsec, pl[1], pl[2], pl[0], pl[3])) for kind, sec, nsec, pl, t in recs]
    tb.write_bag(bag1, {0: ("/imu/data", rosmsg.IMU_TYPE), 1: ("/ouster/points", rosmsg.PCL2_TYPE)},
                 [(("bz2", "none")[j % 2], r1[i:i + 200]) for j, i in enumerate(range(0, len(r1), 200))])
    bag2 = str(tmp_path / "ouster_ros2")
    r2 = [(1, t, t2.cdr_imu(sec, nsec, *pl)) if kind == "imu" else (2, t, t2.cdr_pcl2(sec, nsec, pl[1], pl[2], pl[0], pl[3], frame="os_sensor"))
          for kind, sec, nsec, pl, t in recs]
    t2.write_bag2(bag2, {1: ("/imu/data", rosmsg.IMU_TYPE_ROS2), 2: ("/ouster/points", rosmsg.PCL2_TYPE_ROS2)}, [r2[:len(r2) // 2], r2[len(r2) // 2:]])
    outs = [str(tmp_path / "out1"), str(tmp_path / "out2")]
    a = tg._run_cli(str(tmp_path / "ouster.yaml"), bag1, outs[0])
    b = tg._run_cli(str(tmp_path / "ouster.yaml"), bag2, outs[1])
    print(f"Ouster, time field {with_time}: {len(a['states'])} updates", flush=True)
    assert len(a["states"]) > 150 and a["node"].init_result is None
    _same_run(a, b, *outs)
