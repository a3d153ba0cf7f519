"""The node's published clouds on the H100 (liinit_cloud_download) against the literal CPU checker (tests/cpp/output_oracle.cpp), bit for
bit: a 230k-point 128-ring PointCloud2 message with times, a 24k-point Livox message, IMU undistortion of PointType uploads; a 300-scan
slice of the Livox LI-Init run with publishing and pcd_save on, checked at every scan against the checker applied to the device's own
staged inputs and state; and with two GPUs, REGISTERED and EFFECT identical to the one-GPU result on every rank."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import frame_oracle as fo  # noqa: E402
import output_oracle as oo  # noqa: E402

pytestmark = pytest.mark.gpu


def _pose(rng, big=False):
    from lidar_imu_init_b200 import scenes
    return (scenes.so3_exp(rng.normal(size=3)), rng.normal(size=3) * (100.0 if big else 5.0), scenes.so3_exp(rng.normal(size=3) * 0.05),
            rng.normal(size=3) * 0.1)


def _check_subframe(g, handle, leaf, pose, undistort):
    """map of the scan itself (it takes the staging buffer: first), then stage, undistort, every cloud"""
    p12 = g.frame_download(handle)

    def stage():
        g.frame_stage(handle)
        undistort()
    stage()
    g.map_build(oo.to_world(oo.voxel_grid(oo.staged_records(g, p12), leaf), *pose)[:, 0:3])
    stage()
    staged = oo.staged_records(g, p12)
    oo.check_staged(g, staged, pose)
    down = oo.check_down(g, staged, leaf, pose)
    g.icp_iterate(*pose, False, True)
    m = oo.check_effect(g, down, pose)
    return len(staged), len(down), m


def test_pcl2_230k_message(gpu_lib):
    from lidar_imu_init_b200 import scenes
    rng = np.random.default_rng(1)
    g = gpu_lib.LiInitGpu(0.5, max_map_points=2_000_000, max_scan_points=300_000)
    data, lay, n = scenes.spinning_pcl2(3, 128, 1800, stamp=50.0, seed=3, with_time=True, nan_frac=0.01, zero_frac=0.01)
    assert n == 230_400
    got = g.frame_cut_pcl2(data, lay, n, 3, N_SCANS=128, blind=0.5, point_filter_num=1, required_frame_num=1, scan_count=25, stamp=50.0)
    assert len(got) == 1 and got[0]["n"] > 200_000
    pose = _pose(rng, big=True)
    n_st, n_dn, m = _check_subframe(g, got[0]["handle"], 0.5, pose,
                                    lambda: g.raw_undistort_cv(np.array([0.01, 0.02, 0.4]), np.eye(3), np.array([1.0, 0.2, 0.0])))
    print(f"PointCloud2 230k: {n_st} staged, {n_dn} downsampled, {m} effect points, all bit-equal")
    assert n_st > 200_000 and m > 10_000
    g.close()


def test_livox_24k_message(gpu_lib):
    from lidar_imu_init_b200 import scenes
    rng = np.random.default_rng(2)
    g = gpu_lib.LiInitGpu(0.3, max_map_points=1_000_000, max_scan_points=60_000)
    m = scenes.livox_message(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 10.0, 24_000, seed=4, dup_frac=0.02, tie_frac=0.1)
    got = g.frame_cut_livox(m, N_SCANS=6, blind=0.5, point_filter_num=1, required_frame_num=1, scan_count=9, stamp=10.0)
    assert len(got) == 1
    pose = _pose(rng)
    n_st, n_dn, k = _check_subframe(g, got[0]["handle"], 0.3, pose,
                                    lambda: g.raw_undistort_cv(np.array([0.01, 0.02, -0.2]), np.eye(3), np.array([0.3, 0.0, 0.1])))
    print(f"Livox 24k: {n_st} staged, {n_dn} downsampled, {k} effect points, all bit-equal")
    assert n_st > 20_000 and k > 1000
    g.close()


def test_imu_undistortion_pointtype_upload(gpu_lib):
    from lidar_imu_init_b200 import scenes
    rng = np.random.default_rng(3)
    g = gpu_lib.LiInitGpu(0.3, max_map_points=1_000_000, max_scan_points=120_000)
    n = 100_000
    raw = scenes.timed_scan_points(scenes.box_scene(15.0, 15.0, 6.0), fo._pose_at, 10.0, 0.1, n, seed=21, det_range=60.0, sigma=0.01)
    nv = rng.normal(size=(n, 3))
    raw[:, 4:7] = nv / np.linalg.norm(nv, axis=1, keepdims=True)
    poses = np.zeros((21, 22))
    poses[:, 0] = np.linspace(0, 0.1, 21)
    poses[:, 1:13] = rng.normal(size=(21, 12)) * 0.2
    for k in range(21):
        poses[k, 13:22] = scenes.so3_exp(rng.normal(size=3) * 0.05).reshape(9)
    upose = _pose(rng)
    pose = _pose(rng, big=True)

    def stage():
        g.raw_upload(raw, 9)
        g.raw_undistort_imu(poses, *upose)
    stage()
    g.map_build(oo.to_world(oo.voxel_grid(oo.staged_records(g, raw), 0.3), *pose)[:, 0:3])
    stage()
    staged = oo.staged_records(g, raw)
    oo.check_staged(g, staged, pose)
    down = oo.check_down(g, staged, 0.3, pose)
    g.icp_iterate(*pose, True, True)
    m = oo.check_effect(g, down, pose)
    print(f"IMU-undistorted PointType upload: {n} staged, {len(down)} downsampled, {m} effect points, all bit-equal")
    g.close()


def test_livox_run_slice_publishes(gpu_lib, tmp_path):
    """300 scans of the Livox LI-Init run of test_gpu_frame (10 Hz messages of 20k points, cut_frame_num 5) through the device front
    end with publishing and pcd_save (interval 10): at every scan the three clouds equal the checker applied to the staged sub-frame,
    the device's undistorted cloud and flags and the posterior; every PCD<k>.pcd holds the REGISTERED records of its ten scans."""
    import calib_sim
    import lio_case
    from lidar_imu_init_b200 import _build, host, scenes
    from lidar_imu_init_b200.odometry import LidarOdometry, Publish
    _build.build_host()
    _build.build_calib()

    class Front(LidarOdometry):
        def _stage(self, raw):
            self.staged_handle = raw.handle
            super()._stage(raw)

    ds, per_msg = 0.15, 20_000
    o = Front(gpu_lib.LiInitGpu(ds, max_map_points=3_000_000, max_scan_points=per_msg + 16), ds, max_iteration=4, orig_odom_freq=10,
              cut_frame_num=5, publish=Publish(pcd_save_en=True, interval=10, pcd_dir=str(tmp_path / "PCD")))
    o.preprocess = dict(lidar_type=1, N_SCANS=6, blind=0.5, point_filter_num=1)
    S = calib_sim.make_streams(seed=0, duration=8.0, t_off=0.013)
    path = lio_case.TruePath(0, S)
    scene = scenes.box_scene(40.0, 25.0, 6.0, n_slabs_x=2, n_slabs_y=1)
    ti, wi, ai = S["imu"]
    k_imu, scans, regs, eff = 0, 0, [], 0
    for k in range(75):
        stamp = path.t0 + 0.1 * k
        m = scenes.livox_message(scene, path.lidar, stamp, per_msg, seed=1000 + k, dup_frac=0.01, tie_frac=0.05, noise_frac=0.01,
                                 bad_line_frac=0.01)
        while k_imu < len(ti) and ti[k_imu] <= stamp + 0.13:
            o.imu_buffer.push(ti[k_imu], wi[k_imu], ai[k_imu])
            o.push_imu(wi[k_imu], ai[k_imu], ti[k_imu])
            k_imu += 1
        o.lidar_cbk_livox(m, stamp)
        while scans < 300 and o.process_next() is not None:
            pub = o.published
            if not pub:                      # the map-build scan publishes nothing
                assert scans == 0
                scans += 1
                continue
            g = o.g
            pose = host.state_pose(o.state)
            staged = oo.staged_records(g, g.frame_download(o.staged_handle))
            oo.assert_bits(pub["registered"], oo.to_world(staged, *pose), f"REGISTERED at scan {scans}")
            oo.assert_bits(pub["body"], oo.frame_body(staged), f"BODY at scan {scans}")
            down = oo.voxel_grid(staged, o.filter_size_surf)
            sel = g.scan_state()["selected"]
            oo.assert_bits(pub["effect"], oo.effect(down, sel, *pose), f"EFFECT at scan {scans}")
            assert len(pub["effect"]) == o.stats["effect_feat_num"]
            regs.append(pub["registered"])
            eff += len(pub["effect"])
            scans += 1
    o.close()
    print(f"Livox run: {scans} scans published, {sum(len(r) for r in regs)} registered points, {eff} effect points, all bit-equal")
    assert scans == 300 and o.dropped_subframes == 0
    files = sorted(os.listdir(tmp_path / "PCD"), key=lambda f: int(f[3:-4]))
    assert files == [f"PCD{k}.pcd" for k in range(1, len(regs) // 10 + 1)]
    for k, f in enumerate(files):
        np.testing.assert_array_equal(oo.read_pcd(str(tmp_path / "PCD" / f))[2].view(np.float32), np.concatenate(regs[10 * k:10 * k + 10]))


# ---- two GPUs ------------------------------------------------------------------------------------------------------------------------
def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _clouds(g):
    from lidar_imu_init_b200 import scenes
    c = scenes.make_config("C2", N=30001, M=200000, open_air_frac=0.02, imu_en=True)
    p = c["pose_init"]
    pose = (p.rot_end, p.pos_end, p.R_LI, p.T_LI)
    rng = np.random.default_rng(9)
    raw = oo.records(c["body_xyz"], rng.normal(size=(len(c["body_xyz"]), 3)), rng.uniform(0, 255, len(c["body_xyz"])),
                     rng.uniform(0, 100, len(c["body_xyz"])))
    g.map_build(c["map_xyz"])
    g.raw_upload(raw, 9)
    g.raw_downsample(0.1)
    g.icp_iterate(*pose, True, True)
    return dict(registered=g.cloud(1, *pose), effect=g.cloud(4, *pose))


def _worker(rank, world, port, out_dir):
    import torch
    import torch.distributed as dist
    from lidar_imu_init_b200 import capi, sharding
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = capi.LiInitGpu(0.5, max_map_points=400000, max_scan_points=40000, device_id=rank)
    sharding.attach_comm(g, rank, world)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **_clouds(g))
    g.close()
    dist.destroy_process_group()


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_two_gpus_every_rank_gets_the_whole_frame(tmp_path, gpu_lib):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    g = gpu_lib.LiInitGpu(0.5, max_map_points=400000, max_scan_points=40000)
    one = _clouds(g)
    g.close()
    assert len(one["effect"]) > 1000
    for r in range(2):
        got = np.load(tmp_path / f"rank{r}.npz")
        for k in ("registered", "effect"):
            oo.assert_bits(got[k], one[k], f"{k} on rank {r}")
