"""The bag runner on the H100: `python -m lidar_imu_init_b200.run` (as a function call) on written bags against the same messages
pushed straight into LidarOdometry.

Livox: the 60 s scenario of test_gpu_frame's three-leg run as a bag (IMU and CustomMsg connections, bz2 and uncompressed chunks,
record times that keep that run's delivery order). Ouster: 10 s of LiDAR-only PointCloud2 messages with and without the `t` field."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_bag_node as tb  # noqa: E402  (the bag writer, the message serializers and the scenario)


def _run_cli(cfg_path, bag, out, **kw):
    from lidar_imu_init_b200 import run
    seen = {}

    def on_node(nd):
        seen["node"] = nd
        seen["states"] = []
        seen["end_times"] = []

        def upd(n):
            seen["states"].append(n.odom.state.copy())
            seen["end_times"].append(n.odom.lidar_end_time)
        nd.on_update = upd
    argv = ["--config", cfg_path, "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet"]
    for k, v in kw.items():
        argv += ["--" + k.replace("_", "-"), str(v)]
    assert run.main(argv, on_node=on_node) == 0
    return seen


def _parse_result(path):
    text = open(path).read()
    blocks = {}
    for title in ("Initialization result:", "Refinement result:"):
        assert text.count(title + "\n") == 1, title
        L = text.split(title + "\n")[1].splitlines()
        v = lambda line: np.array([float(x) for x in line.split("=")[1].split()])   # noqa: E731
        blocks[title] = dict(euler_deg=v(L[0]), T_LI=v(L[1]), time_lag=float(L[2].split("=")[1]), bias_g=v(L[3]), bias_a=v(L[4]),
                             gravity=v(L[5]), R_LI=np.array([[float(x) for x in L[i].split()] for i in range(8, 11)])[:, :3])
    return text, blocks


@pytest.mark.gpu
def test_livox_bag_sixty_seconds(gpu_lib, tmp_path):
    from lidar_imu_init_b200 import _build, config, node
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_host()
    _build.build_calib()
    cfg = tb.sim_config(tmp_path, online_refine_time=10.0)
    ev, path = tb.livox_events(60.0, 20_000)
    bag = str(tmp_path / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    out = str(tmp_path / "out")
    seen = _run_cli(str(tmp_path / "sim.yaml"), bag, out)
    nd = seen["node"]

    # leg 1 of test_gpu_frame, driven directly on the same messages, with the refinement clock restated
    d = LidarOdometry(gpu_lib.LiInitGpu(cfg.filter_size_map, max_map_points=3_000_000, max_scan_points=300_000), **config.odometry_kwargs(cfg))
    d.preprocess = config.preprocess(cfg)
    direct = dict(states=[], init_scan=None, res=None, refine_scan=None, start=None, lio=[])

    def on_state(o):
        direct["states"].append(o.state.copy())
        if o.imu_en:
            direct["lio"].append((o.lidar_end_time, o.state.copy()))
            if (direct["refine_scan"] is None and node.refine_tick(o.frame_num, o.orig_odom_freq, o.cut_frame_num)
                    and min(o.lidar_end_time - direct["start"], cfg.online_refine_time) > cfg.online_refine_time - 1e-6):
                direct["refine_scan"] = o.frame_num
        elif o.data_accum_finished:
            direct["init_scan"], direct["start"] = o.frame_num, o.lidar_end_time

    orig_hand_over = d.hand_over

    def hand_over(res):
        direct["res"] = res
        orig_hand_over(res)
    d.hand_over = hand_over
    tb.drive_direct(d, ev, cfg.mean_acc_norm, on_state)

    states = seen["states"]
    print(f"{len(states)} updates, trigger at frame {nd.init_scan}, refinement done at frame {nd.refine_scan}, "
          f"{nd.odom.dropped_subframes} dropped", flush=True)
    assert len(states) == len(direct["states"]) > 2000
    for j, (a, b) in enumerate(zip(states, direct["states"])):
        np.testing.assert_array_equal(a, b, err_msg=f"update {j}")
    assert nd.init_scan == direct["init_scan"] is not None
    for key in ("R_LI", "T_LI", "grav_L0", "gyro_bias", "acc_bias", "time_lag_1", "time_lag_2"):
        np.testing.assert_array_equal(nd.init_result[key], direct["res"][key])
    assert nd.odom.dropped_subframes == 0
    assert nd.refine_scan == direct["refine_scan"] is not None

    # the result file: both blocks parse back to the states, to print precision
    text, blocks = _parse_result(os.path.join(out, "result", "Initialization_result.txt"))
    lag = nd.time_lag
    want_text = ""
    for title, st in (("Initialization result:", nd.init_state), ("Refinement result:", nd.refine_state)):
        v = node.state_calib_values(st, lag)
        want_text += title + "\n" + node.calib_result_text(**v)
        got = blocks[title]
        for key in ("euler_deg", "T_LI", "bias_g", "bias_a", "gravity", "R_LI"):
            assert np.abs(got[key] - np.asarray(v[key])).max() <= 5.1e-7, (title, key)
        assert abs(got["time_lag"] - lag) <= 5.1e-7
    assert text == want_text
    assert np.array_equal(nd.init_state[12:21], nd.init_result["R_LI"].reshape(9))

    # one mat_out row and one trajectory line per update; the LIO positions are the LiDAR's, within 4 cm of the simulated truth
    rows = open(os.path.join(out, "Log", "mat_out.txt")).read().splitlines()
    traj = np.loadtxt(os.path.join(out, "result", "trajectory.txt"))
    assert len(rows) == len(traj) == len(states)
    np.testing.assert_allclose(traj[:, 0], np.array(seen["end_times"]), rtol=0, atol=1e-9)
    import lio_case
    p0 = np.array(lio_case.P0)
    lio_lines = [k for k, s in enumerate(states) if not np.array_equal(s[12:21], np.eye(3).reshape(9))]
    errs = []
    for k in lio_lines[1:]:                      # the switch scan re-matches the previous cloud: skip it
        R_t, p_t = path.lidar(np.array([traj[k, 0]]))
        s = states[k]
        np.testing.assert_allclose(traj[k, 1:4], s[0:9].reshape(3, 3) @ s[21:24] + s[9:12], rtol=0, atol=1e-7)
        errs.append(float(np.linalg.norm(traj[k, 1:4] - (p_t[0] - p0))))
    print(f"LIO trajectory: {len(errs)} lines, max error against truth {max(errs):.4f} m", flush=True)
    assert len(errs) > 1000 and max(errs) < 0.04


def _ouster_events(seconds, n_pts, with_time, seed=0):
    import calib_sim
    import lio_case
    from lidar_imu_init_b200 import scenes
    S = calib_sim.make_streams(seed=seed, duration=seconds, t_off=0.013)
    path = lio_case.TruePath(seed, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    step, fields = tb.DRIVER_FIELDS[3]
    if not with_time:
        fields = [f for f in fields if f[0] != "t"]
    lay = dict(point_step=step, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=20 if with_time else -1, off_ring=26)
    ev, k_imu = [], 0
    for k in range(int(seconds * 10) - 1):
        stamp = path.t0 + 0.1 * k
        pts = scenes.timed_scan_points(scene, path.lidar, stamp, 0.1, n_pts, seed=2000 + k, sigma=0.01)
        buf = np.zeros((n_pts, step), np.uint8)
        put = lambda off, a: buf.__setitem__((slice(None), slice(off, off + a.dtype.itemsize)), a.view(np.uint8).reshape(n_pts, -1))   # noqa: E731
        put(0, np.ascontiguousarray(pts[:, 0]))
        put(4, np.ascontiguousarray(pts[:, 1]))
        put(8, np.ascontiguousarray(pts[:, 2]))
        put(16, np.ascontiguousarray(pts[:, 8]) + np.float32(10.0))
        if with_time:
            put(20, np.round(pts[:, 9].astype(np.float64) * 1e6).astype("<u4"))
        put(26, (np.arange(n_pts) % 16).astype(np.uint8))
        while k_imu < len(ti) and ti[k_imu] <= stamp + 0.13:
            ev.append(("imu", *tb.split_time(ti[k_imu]), (wi[k_imu], ai[k_imu])))
            k_imu += 1
        sec, nsec = tb.split_time(stamp)
        ev.append(("lidar", sec, nsec, (buf.reshape(-1), fields, step, n_pts)))
    return ev, lay


@pytest.mark.gpu
@pytest.mark.parametrize("with_time", [True, False])
def test_ouster_bag_lidar_only(gpu_lib, tmp_path, with_time):
    from lidar_imu_init_b200 import _build, config, rosmsg
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_host()
    _build.build_calib()
    ev, lay = _ouster_events(10.0, 20_000, with_time)
    text = ("common:\n  lid_topic: /ouster/points\n  imu_topic: /imu/data\npreprocess:\n  lidar_type: 3\n  scan_line: 16\n  blind: 0.5\n"
            "initialization:\n  cut_frame_num: 2\n  orig_odom_freq: 10\n  mean_acc_norm: 9.81\n  online_refine_time: 15\n  data_accum_length: 100000\n"
            "  Rot_LI_cov: [0.00005, 0.00005, 0.00005]\n  Trans_LI_cov: [0.0001, 0.0001, 0.0001]\n"
            "mapping:\n  filter_size_surf: 0.15\n  filter_size_map: 0.15\n  gyr_cov: 0.1\n  acc_cov: 0.1\n")
    (tmp_path / "ouster.yaml").write_text(text)
    cfg = config.load(str(tmp_path / "ouster.yaml"))
    conns = {0: ("/imu/data", rosmsg.IMU_TYPE), 1: ("/ouster/points", rosmsg.PCL2_TYPE)}
    recs = []
    for kind, sec, nsec, pl in ev:
        if kind == "imu":
            recs.append((0, sec, nsec, tb.ser_imu(sec, nsec, *pl)))
        else:
            rs, rn = max(tb.split_time(sec + 1e-9 * nsec + 0.13), recs[-1][1:3])   # after the IMU samples delivered before it
            recs.append((1, rs, rn, tb.ser_pcl2(sec, nsec, pl[1], pl[2], pl[0], pl[3])))
    bag = str(tmp_path / "ouster.bag")
    tb.write_bag(bag, conns, [(("bz2", "none")[j % 2], recs[i:i + 200]) for j, i in enumerate(range(0, len(recs), 200))])
    seen = _run_cli(str(tmp_path / "ouster.yaml"), bag, str(tmp_path / "out"))
    nd = seen["node"]

    d = LidarOdometry(gpu_lib.LiInitGpu(cfg.filter_size_map, max_map_points=3_000_000, max_scan_points=300_000), **config.odometry_kwargs(cfg))
    d.preprocess = config.preprocess(cfg)
    states = []
    for kind, sec, nsec, pl in ev:
        t = sec + 1e-9 * nsec
        if kind == "imu":
            d.imu_buffer.push(t, *pl)
            d.push_imu(pl[0], pl[1], t, cfg.mean_acc_norm)
            continue
        d.lidar_cbk_pcl2(pl[0], lay, pl[3], t)
        while True:
            f = d.frame_num
            if d.process_next() is None:
                break
            if d.frame_num != f:
                states.append(d.state.copy())
    print(f"Ouster, time field {with_time}: {len(states)} updates", flush=True)
    assert len(seen["states"]) == len(states) > 150
    for a, b in zip(seen["states"], states):
        np.testing.assert_array_equal(a, b)
    assert nd.init_result is None and not nd.odom.imu_en and nd.odom.dropped_subframes == 0
