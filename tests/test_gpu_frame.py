"""The cut-frame preprocess on the H100 (liinit_frame_cut_livox / _pcl2, liinit_frame_stage / _download) against the literal CPU
checker (tests/cpp/frame_oracle.cpp): random Livox messages bit for bit, the four PointCloud2 types with and without a time field,
staging into the raw chain, the error paths, and 60 s of the whole LI-Init run driven by the device front end against the same
product loop and the oracle loop fed the checker's sub-frames."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import frame_oracle as fo  # noqa: E402


def _subframes(g, got):
    return [g.frame_download(s["handle"]) for s in got]


@pytest.mark.gpu
def test_livox_random_messages_bit_equal(gpu_lib):
    g = gpu_lib.LiInitGpu(0.5, max_map_points=100_000, max_scan_points=50_000)
    rng = np.random.Generator(np.random.PCG64(fo.LIVOX_SEED))
    n_msgs, n_sub, n_pts, degenerate = 400, 0, 0, 0
    for _ in range(n_msgs):
        m, prm = fo.random_livox(rng)
        want = fo.cut_livox(m, **prm)
        got = g.frame_cut_livox(m, **prm)
        fo.compare(got, _subframes(g, got), want)
        n_sub += len(got)
        n_pts += sum(s["n"] for s in got)
        degenerate += int(len(m) < 20)
    print(f"{n_msgs} Livox messages ({degenerate} degenerate sizes): {n_sub} sub-frames, {n_pts} points, all bit-equal")
    assert n_sub > n_msgs and degenerate > 50
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lidar_type", [2, 3, 5, 6])
@pytest.mark.parametrize("with_time", [True, False])
def test_pcl2_types(gpu_lib, lidar_type, with_time):
    """Given times: bit-equal. The rotation model (Velodyne / Robosense without a time field): same sub-frame sizes and points, curvature
    within fo.YAW_TOL_MS, at most 1% of the points in another order among near-equal times; the counts are printed. Ouster / Pandar
    without a time field read times 0."""
    from lidar_imu_init_b200 import scenes
    g = gpu_lib.LiInitGpu(0.5, max_map_points=100_000, max_scan_points=300_000)
    rotation = not with_time and lidar_type in (2, 6)
    total = moved = npts = 0
    for seed, (rings, az, pad) in enumerate(((16, 1800, 0), (32, 1024, 5), (128, 1800, 3))):
        data, lay, n = scenes.spinning_pcl2(lidar_type, rings, az, stamp=50.0 + seed, seed=seed + 10 * lidar_type, with_time=with_time,
                                            turns=1.02, nan_frac=0.02, zero_frac=0.02, extra_pad=pad)
        prm = dict(N_SCANS=min(rings - 2, 100), blind=0.8, point_filter_num=1 + seed, required_frame_num=3, scan_count=19 + seed, stamp=50.0 + seed)
        want = fo.cut_pcl2(data, lay, n, lidar_type, **prm)
        got = g.frame_cut_pcl2(data, lay, n, lidar_type, **prm)
        a, b = fo.compare(got, _subframes(g, got), want, curv_tol_ms=fo.YAW_TOL_MS if rotation else 0.0)
        total, moved, npts = total + a, moved + b, npts + sum(s["n"] for s in got)
    print(f"lidar_type {lidar_type}, time field {with_time}: {npts} points, {total} curvatures not bit-equal, {moved} in another order")
    if not rotation:
        assert total == 0 and moved == 0
    else:
        assert moved <= npts // 100
    g.close()


@pytest.mark.gpu
def test_stage_equals_raw_upload_and_errors(gpu_lib):
    """liinit_frame_stage of a sub-frame leaves what liinit_raw_upload(its PointType points, 12, 9) leaves: raw download, CV undistortion
    and voxel grid bit-identical. A message above the staging capacity and bad parameters change nothing; a handle older than the
    slot ring is refused."""
    from lidar_imu_init_b200 import scenes
    g = gpu_lib.LiInitGpu(0.5, max_map_points=500_000, max_scan_points=60_000)
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 10.0, 24_000, seed=4, dup_frac=0.02, tie_frac=0.1)
    prm = dict(N_SCANS=6, blind=0.5, point_filter_num=1, required_frame_num=5, scan_count=9, stamp=10.0)
    got = g.frame_cut_livox(m, **prm)
    want = fo.cut_livox(m, **prm)
    fo.compare(got, _subframes(g, got), want)
    k = 2
    h = got[k]["handle"]
    p12 = np.zeros((want[k]["n"], 12), np.float32)
    p12[:, 0:3] = want[k]["pts"][:, 0:3]
    p12[:, 3] = 1.0
    p12[:, 8] = want[k]["pts"][:, 3]
    p12[:, 9] = want[k]["pts"][:, 4]
    np.testing.assert_array_equal(g.frame_download(h), p12)
    omega, R, v = np.array([0.01, -0.02, 0.3]), np.eye(3), np.array([0.5, 0.1, 0.0])
    res = []
    for stage in (lambda: g.frame_stage(h), lambda: g.raw_upload(p12, 9)):
        stage()
        a = g.raw_points()
        g.raw_undistort_cv(omega, R, v)
        b = g.raw_points()
        nd = g.raw_downsample(0.3)
        res.append((a, b, nd, g.scan_body()))
    for x, y in zip(res[0], res[1]):
        np.testing.assert_array_equal(x, y)
    # errors change nothing
    before = g.frame_download(h)
    with pytest.raises(gpu_lib.LiInitError) as e:
        g.frame_cut_livox(np.zeros((1 << 20) + 1, m.dtype), **prm)
    assert e.value.code == -3
    with pytest.raises(gpu_lib.LiInitError) as e:
        g.frame_cut_livox(m, **dict(prm, lidar_type=2))
    assert e.value.code == -1
    data = np.zeros((4, 32), np.uint8)                   # the rotation model meets ring 128
    data[:, 0:4] = np.frombuffer(np.float32(5.0).tobytes(), np.uint8)
    data[1, 24:26] = np.frombuffer(np.uint16(128).tobytes(), np.uint8)
    with pytest.raises(gpu_lib.LiInitError) as e:
        g.frame_cut_pcl2(data.reshape(-1), dict(point_step=32, off_x=0, off_y=4, off_z=8, off_intensity=16, off_time=-1, off_ring=24), 4, 2,
                         N_SCANS=4)
    assert e.value.code == -1
    np.testing.assert_array_equal(g.frame_download(h), before)
    g.frame_stage(h)
    np.testing.assert_array_equal(g.raw_points(), res[0][0])
    # four more messages reuse every slot: the first handle is gone, the latest ones work
    for i in range(4):
        last = g.frame_cut_livox(m, **dict(prm, stamp=11.0 + i))
    with pytest.raises(gpu_lib.LiInitError) as e:
        g.frame_stage(h)
    assert e.value.code == -1
    g.frame_stage(last[-1]["handle"])
    g.close()


@pytest.mark.gpu
def test_sixty_seconds_of_livox_messages_three_legs(gpu_lib, oracle_mod):
    """60 s of 10 Hz Livox messages (20k points each, cut_frame_num 5 -> 50 Hz once scan_count reaches 5) with the IMU stream of
    calib_sim, through the whole LI-Init run: LiDAR-only mode, the trigger, LI_Initialization, the hand-over, the switch scan, LIO.
    Leg 1: LidarOdometry through the device front end (lidar_cbk_livox + process_next). Leg 2: the same product odometry fed the
    checker's sub-frames through process_raw. Leg 3: the oracle loop of lio_case fed the checker's sub-frames. Legs 1 and 2: bit-
    identical states at every scan, the same trigger scan and calibration. Legs 1 and 3: the bounds of test_gpu_lio (1e-3 m / 1e-3 rad
    per scan in both modes, same trigger scan, calibration within 1e-3, extrinsic of the LIO leg within 1e-3)."""
    import calib_sim
    import lio_case
    from lidar_imu_init_b200 import _build, host, scenes
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_host()
    _build.build_calib()
    ds, per_msg, seconds = 0.15, 20_000, 60.0
    kw = dict(max_iteration=4, orig_odom_freq=10, cut_frame_num=5)
    front = LidarOdometry(gpu_lib.LiInitGpu(ds, max_map_points=3_000_000, max_scan_points=per_msg + 16), ds, **kw)
    raw = LidarOdometry(gpu_lib.LiInitGpu(ds, max_map_points=3_000_000, max_scan_points=per_msg + 16), ds, **kw)
    orc = lio_case.make_oracle_odometry(oracle_mod, ds, lio_case.default_threads(), **kw)
    legs = (front, raw, orc)
    for o in legs:
        o.preprocess = dict(lidar_type=1, N_SCANS=6, blind=0.5, point_filter_num=1)
    S = calib_sim.make_streams(seed=0, duration=seconds, t_off=0.013)
    path = lio_case.TruePath(0, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    k_imu, scans, init_scan, switch_ok = 0, 0, None, None
    st = dict(lo_dp=0.0, lo_dr=0.0, lio_dp=0.0, lio_dr=0.0, lio_dT=0.0, lio_dRLI=0.0, dm_max=0, lio_scans=0)

    def next_raw(o):
        e = o.lidar_buffer.popleft()
        return o.process_raw(e["p12"], e["t_beg"])

    for k in range(int(seconds * 10) - 1):
        stamp = path.t0 + 0.1 * k
        m = scenes.livox_message(scene, path.lidar, stamp, per_msg, seed=1000 + k, dup_frac=0.01, tie_frac=0.05, noise_frac=0.01,
                                 bad_line_frac=0.01)
        while k_imu < len(ti) and ti[k_imu] <= stamp + 0.13:    # the IMU runs ahead of the LiDAR (sync_packages waits for it)
            for o in legs:
                o.imu_buffer.push(ti[k_imu], wi[k_imu], ai[k_imu])
                o.push_imu(wi[k_imu], ai[k_imu], ti[k_imu])
            k_imu += 1
        front.lidar_cbk_livox(m, stamp)
        for o in (raw, orc):
            o._lidar_cbk(stamp)
        want = fo.cut_livox(m, **{a: v for a, v in raw._cut_params(stamp).items() if a != "lidar_type"})
        for w in want:
            p12 = np.zeros((w["n"], 12), np.float32)
            p12[:, 0:3], p12[:, 3], p12[:, 8], p12[:, 9] = w["pts"][:, 0:3], 1.0, w["pts"][:, 3], w["pts"][:, 4]
            for o in (raw, orc):
                o.lidar_buffer.append(dict(p12=p12, t_beg=w["t_beg"], end_ms=w["end_ms"], n=w["n"]))
        while True:
            sa = front.process_next()
            if sa is None:
                assert not raw.lidar_buffer or not raw.imu_buffer.ready(raw.lidar_buffer[0]["t_beg"] + float(raw.lidar_buffer[0]["end_ms"]) / 1000.0)
                break
            sb = next_raw(raw)
            next_raw(orc)
            np.testing.assert_array_equal(sa, sb)
            Rg, pg, RLg, TLg = host.state_pose(front.state)
            Ro, po, RLo, TLo = host.state_pose(orc.state)
            if front.stats is not None and orc.stats is not None:
                st["dm_max"] = max(st["dm_max"], abs(front.stats["effect_feat_num"] - orc.stats["effect_feat_num"]))
            if not front.imu_en:
                assert front.data_accum_finished == raw.data_accum_finished == orc.data_accum_finished, scans
                st["lo_dp"] = max(st["lo_dp"], float(np.abs(pg - po).max()))
                st["lo_dr"] = max(st["lo_dr"], lio_case.angle(Rg, Ro))
                assert st["lo_dp"] <= 1e-3 and st["lo_dr"] <= 1e-3, (scans, st)
                if front.data_accum_finished:
                    res = [o.initialize(0.0) for o in legs]
                    for o, r in zip(legs, res):
                        o.hand_over(r)
                    init_scan = scans
                    for key in ("R_LI", "T_LI", "grav_L0", "gyro_bias", "acc_bias", "time_lag_1", "time_lag_2"):
                        np.testing.assert_array_equal(res[0][key], res[1][key])
                    assert lio_case.angle(res[0]["R_LI"], res[2]["R_LI"]) <= 1e-3
                    for key in ("T_LI", "grav_L0", "gyro_bias", "acc_bias"):
                        assert np.abs(np.asarray(res[0][key]) - np.asarray(res[2][key])).max() <= 1e-3, key
                    assert abs(res[0]["time_lag_1"] + res[0]["time_lag_2"] - res[2]["time_lag_1"] - res[2]["time_lag_2"]) <= 1e-3
            else:
                st["lio_dp"] = max(st["lio_dp"], float(np.abs(pg - po).max()))
                st["lio_dr"] = max(st["lio_dr"], lio_case.angle(Rg, Ro))
                st["lio_dT"] = max(st["lio_dT"], float(np.abs(TLg - TLo).max()))
                st["lio_dRLI"] = max(st["lio_dRLI"], lio_case.angle(RLg, RLo))
                assert max(st["lio_dp"], st["lio_dr"], st["lio_dT"], st["lio_dRLI"]) <= 1e-3, (scans, st)
                if switch_ok is None:
                    switch_ok = front.switch_scan == raw.switch_scan == orc.switch_scan
                st["lio_scans"] += 1
            scans += 1
    print(f"three legs: {scans} scans, trigger at scan {init_scan}, {st}, front end dropped {front.dropped_subframes} sub-frames, "
          f"map {front.g.map_validnum()} / {orc.om.validnum()}", flush=True)
    assert init_scan is not None and switch_ok and st["lio_scans"] > 1000
    assert st["dm_max"] <= 3 and front.dropped_subframes == 0
    assert front.g.map_validnum() == raw.g.map_validnum()
    assert abs(front.g.map_validnum() - orc.om.validnum()) <= 1e-3 * orc.om.validnum()
