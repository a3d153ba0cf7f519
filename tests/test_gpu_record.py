"""Recording what the node publishes, on the H100: `python -m lidar_imu_init_b200.run --record` (as a function call) on the 60 s Livox
scenario of tests/test_gpu_bag.py, once into a ROS1 bag (with --debug-logs) and once into a rosbag2 directory, and on the 10 s Ouster
PointCloud2 scenario with dense_publish_en false. Each run is bit-identical to the same run without recording; read back, the
recorded clouds of sampled updates are the records liinit_cloud_download returned, and every /cloud_effected has the update's
effective-point count."""
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_bag2_node as t2  # noqa: E402
import test_bag_node as tb  # noqa: E402
import test_gpu_bag as tg  # noqa: E402
import test_gpu_bag2 as tg2  # noqa: E402

SAMPLE = 37   # every SAMPLE-th update keeps its published records for the comparison


def _run(cfg_path, bag, out, *extra):
    """tg._run_cli with extra arguments, keeping the published records of sampled updates and every effective-point count."""
    from lidar_imu_init_b200 import run
    seen = dict(states=[], end_times=[], pub={}, eff=[])

    def on_node(nd):
        seen["node"] = nd

        def upd(n):
            k = len(seen["states"])
            seen["states"].append(n.odom.state.copy())
            seen["end_times"].append(n.odom.lidar_end_time)
            seen["eff"].append(int(n.odom.stats["effect_feat_num"]))
            if k % SAMPLE == 0:
                seen["pub"][k] = {key: v.copy() for key, v in n.odom.published.items()}
        nd.on_update = upd
    argv = ["--config", cfg_path, "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet", *extra]
    assert run.main(argv, on_node=on_node) == 0
    return seen


def _width(data, enc):
    """PointCloud2 width of a message with frame_id camera_init"""
    return int(np.frombuffer(bytes(data[:64]), "<u4", 1, (31 if enc == "ros1" else 4 + 28))[0])


def _check_recording(path, seen, clouds):
    from lidar_imu_init_b200 import config, pubmsg, rosbag2
    n = len(seen["states"])
    with rosbag2.open_bag(path) as bag:
        enc = bag.format
        topics = bag.topics()
        counts = {t: 0 for t in topics}
        for m in bag.messages(topics):
            k = counts[m.topic]
            counts[m.topic] += 1
            if m.topic == "/cloud_effected":
                assert _width(m.data, enc) == seen["eff"][k], k
            if m.topic in [config.CLOUD_TOPICS[c] for c in clouds] and k in seen["pub"]:
                key = next(c for c in clouds if config.CLOUD_TOPICS[c] == m.topic)
                rec = seen["pub"][k][key]
                assert bytes(m.data) == pubmsg.pointcloud2((m.sec, m.nsec), "camera_init", rec, enc), (m.topic, k)
    want = {"/aft_mapped_to_init": n, "/tf": n, "/path": n // 5, **{config.CLOUD_TOPICS[c]: n for c in clouds}}
    assert counts == want
    return enc


@pytest.fixture(scope="module")
def livox(gpu_lib, tmp_path_factory):
    from lidar_imu_init_b200 import _build
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("rec")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    out = str(tmp / "out_plain")
    seen = tg._run_cli(str(tmp / "sim.yaml"), bag, out)
    assert seen["node"].init_scan is not None and len(seen["states"]) > 2000
    return dict(tmp=tmp, bag=bag, seen=seen, out=out)


@pytest.mark.gpu
def test_livox_record_ros1_with_debug_logs(livox):
    from lidar_imu_init_b200 import node
    tmp = livox["tmp"]
    rec, out = str(tmp / "rec1.bag"), str(tmp / "out_rec1")
    seen = _run(str(tmp / "sim.yaml"), livox["bag"], out, "--record", rec, "--debug-logs")
    tg2._same_run(livox["seen"], seen, livox["out"], out)
    size = os.path.getsize(rec)
    assert _check_recording(rec, seen, ("registered", "body", "effect")) == "ros1"
    print(f"ROS1 recording of {len(seen['states'])} updates: {size / 1e6:.1f} MB", flush=True)
    os.remove(rec)
    # LI-Init's logs: written at the trigger from the calibration's tables; the plain run has none of them
    calib = seen["node"].odom.calib
    for name, (table, precision, groups) in node.DEBUG_LOGS.items():
        rows = calib.log_rows(table)
        assert len(rows) > 100, (name, len(rows))
        assert open(os.path.join(out, "Log", name)).read() == "".join(node.log_row(r, precision, groups) for r in rows)
        assert not os.path.exists(os.path.join(livox["out"], "Log", name))


@pytest.mark.gpu
def test_livox_record_ros2(livox):
    tmp = livox["tmp"]
    rec, out = str(tmp / "rec2"), str(tmp / "out_rec2")
    seen = _run(str(tmp / "sim.yaml"), livox["bag"], out, "--record", rec, "--record-format", "ros2", "--record-topics",
                "/cloud_registered,/cloud_effected,/aft_mapped_to_init,/tf,/path")
    tg2._same_run(livox["seen"], seen, livox["out"], out)
    assert all(set(p) == {"registered", "effect"} for p in seen["pub"].values())
    assert _check_recording(rec, seen, ("registered", "effect")) == "cdr"
    shutil.rmtree(rec)


@pytest.mark.gpu
def test_ouster_record_downsampled_clouds(gpu_lib, tmp_path):
    """The Ouster PointCloud2 scenario with publish/dense_publish_en false: /cloud_registered carries REGISTERED_DOWN."""
    from lidar_imu_init_b200 import _build, rosmsg
    _build.build_host()
    _build.build_calib()
    ev, _ = tg._ouster_events(10.0, 20_000, True)
    text = ("common:\n  lid_topic: /ouster/points\n  imu_topic: /imu/data\npreprocess:\n  lidar_type: 3\n  scan_line: 16\n  blind: 0.5\n"
            "initialization:\n  cut_frame_num: 2\n  orig_odom_freq: 10\n  mean_acc_norm: 9.81\n  online_refine_time: 15\n  data_accum_length: 100000\n"
            "  Rot_LI_cov: [0.00005, 0.00005, 0.00005]\n  Trans_LI_cov: [0.0001, 0.0001, 0.0001]\n"
            "mapping:\n  filter_size_surf: 0.15\n  filter_size_map: 0.15\n  gyr_cov: 0.1\n  acc_cov: 0.1\npublish:\n  dense_publish_en: false\n")
    (tmp_path / "ouster.yaml").write_text(text)
    recs = t2.event_records(ev)
    bag = str(tmp_path / "ouster.bag")
    r1 = [(0, t // 10**9, t % 10**9, tb.ser_imu(sec, nsec, *pl)) if kind == "imu" else
          (1, t // 10**9, t % 10**9, tb.ser_pcl2(sec, nsec, pl[1], pl[2], pl[0], pl[3])) for kind, sec, nsec, pl, t in recs]
    tb.write_bag(bag, {0: ("/imu/data", rosmsg.IMU_TYPE), 1: ("/ouster/points", rosmsg.PCL2_TYPE)},
                 [(("bz2", "none")[j % 2], r1[i:i + 200]) for j, i in enumerate(range(0, len(r1), 200))])
    cfg = str(tmp_path / "ouster.yaml")
    a = tg._run_cli(cfg, bag, str(tmp_path / "out_plain"))
    rec = str(tmp_path / "ouster_rec.bag")
    b = _run(cfg, bag, str(tmp_path / "out_rec"), "--record", rec)
    tg2._same_run(a, b, str(tmp_path / "out_plain"), str(tmp_path / "out_rec"))
    assert len(b["states"]) > 150 and b["node"].init_result is None
    # the downsampled cloud: fewer points than the body cloud of the same scan
    for p in b["pub"].values():
        assert 0 < len(p["registered"]) < len(p["body"])
    _check_recording(rec, b, ("registered", "body", "effect"))
