"""The device-pointer twins on the H100, fed with torch CUDA tensors through the binding: every result bit-identical to the host twin's,
at the C2 size and at the strided frame size of test_gpu_strided_pass.py (num_sms * 3072 + 37 points), for both knn indexes; the
stand-alone search over more queries than one staging chunk holds; an odometry loop of 40 raw timed scans uploaded from the device;
inputs written by torch on its current stream right before the call, with no synchronise in between."""
import numpy as np
import pytest

from lidar_imu_init_b200 import scenes

BRICKS, CELLS = 1, 2
pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _world(body, p):
    return np.ascontiguousarray((p.rot_end @ (p.R_LI @ body.T.astype(np.float64) + p.T_LI[:, None]) + p.pos_end[:, None]).T, np.float32)


def _same_set(a, b):
    return sorted(map(bytes, np.ascontiguousarray(a, np.float32))) == sorted(map(bytes, np.ascontiguousarray(b, np.float32)))


def _strided(xyz, stride):
    a = np.full((len(xyz), stride), 7.5, np.float32)
    a[:, :3] = xyz
    return a


def _pass_eq(rh, sh, rd, sd, tag):
    for a, b, name in zip(rh, rd, ("HtH", "Htr", "m", "res_sq")):
        assert np.array_equal(np.asarray(a), np.asarray(b)), (tag, name)
    for k in ("world", "near_xyz", "near_cnt", "selected"):
        assert np.array_equal(sh[k], sd[k]), (tag, k)
    sel = sh["selected"].astype(bool)
    assert np.array_equal(sh["normvec"][sel], sd["normvec"][sel]), tag


@pytest.fixture(scope="module")
def frames():
    torch = _torch()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"C2": scenes.make_config("C2", seed=3), "strided": scenes.make_config("C2", seed=3, N=sms * 3072 + 37, M=2_000_000,
                                                                                   open_air_frac=0.02)}


@pytest.mark.parametrize("index", [BRICKS, CELLS], ids=["bricks", "cells"])
@pytest.mark.parametrize("size", ["C2", "strided"])
def test_device_twins_bit_identical(gpu_lib, frames, size, index):
    """map_build into two contexts (same live set); then on one map -- so that neighbours at exactly equal distances are settled by
    the same pool order -- scan_upload (stride 4 in place, stride 12, a misaligned stride-4 view) through search / reuse / search passes,
    the published clouds, the raw chain and the live map: device twins against host twins"""
    torch = _torch()
    c = frames[size]
    N = len(c["body_xyz"])
    p, p2 = c["pose_init"], scenes.perturb_pose(c["pose_init"], 77, dtheta_deg=0.05, dpos=0.01)
    mk = lambda: gpu_lib.LiInitGpu(c["ds"], max_map_points=max(2_200_000, 2 * len(c["map_xyz"])), max_scan_points=N + 16,  # noqa: E731
                                   knn_index=index)
    hb, g = mk(), mk()
    hb.map_build(c["map_xyz"])
    g.map_build(torch.from_numpy(np.ascontiguousarray(c["map_xyz"])).cuda())
    assert g.map_validnum() == hb.map_validnum() and g.map_stats()["bricks"] == hb.map_stats()["bricks"]
    assert _same_set(g.map_download(), hb.map_download())
    hb.close()
    body4 = _strided(c["body_xyz"], 4)
    flat = torch.from_numpy(np.concatenate([[0.0], body4.reshape(-1)]).astype(np.float32)).cuda()
    uploads = {"stride 4": torch.from_numpy(body4).cuda(), "stride 12": torch.from_numpy(_strided(c["body_xyz"], 12)).cuda(),
               "stride 4, misaligned": flat[1:].view(N, 4)}
    assert uploads["stride 4, misaligned"].data_ptr() % 16 == 4
    passes = ((p, True), (p2, False), (c["pose_gt"], True))
    g.scan_upload(c["body_xyz"])
    ref = [(g.icp_iterate(q.rot_end, q.pos_end, q.R_LI, q.T_LI, False, s), g.scan_state()) for q, s in passes]
    gt = c["pose_gt"]
    pose = (gt.rot_end, gt.pos_end, gt.R_LI, gt.T_LI)
    eff = g.cloud(4, *pose)
    for tag, t in uploads.items():
        g.scan_upload(t)
        for (q, s), (rh, sh) in zip(passes, ref):
            _pass_eq(rh, sh, g.icp_iterate(q.rot_end, q.pos_end, q.R_LI, q.T_LI, False, s), g.scan_state(), tag)
        eff_d = g.cloud(4, *pose, device=True)
        assert eff_d.is_cuda and np.array_equal(eff_d.cpu().numpy(), eff), tag
    g.map_incremental(*pose, c["ds"])
    live = g.map_download(device=True)
    assert live.is_cuda and _same_set(live.cpu().numpy(), g.map_download())
    # the raw chain: PointType records with attributes -> voxel grid -> the three other clouds
    rng = np.random.default_rng(4)
    raw = _strided(c["body_xyz"], 12)
    raw[:, 4:7] = rng.normal(size=(N, 3))
    raw[:, 8] = rng.uniform(0, 255, N)
    raw[:, 9] = np.sort(rng.uniform(0, 100, N))
    got = {}
    for src in (raw, torch.from_numpy(raw).cuda()):
        dev = not isinstance(src, np.ndarray)
        g.raw_upload(src, 9)
        for which in (1, 3):
            got[which, dev] = g.cloud(which, *pose, device=True).cpu().numpy() if dev else g.cloud(which, *pose)
        got["n", dev] = g.raw_downsample(0.5)
        got[2, dev] = g.cloud(2, *pose, device=True).cpu().numpy() if dev else g.cloud(2, *pose)
    for k in (1, 2, 3, "n"):
        assert np.array_equal(got[k, False], got[k, True]), k
    assert np.any(got[2, True][:, 4:7] != 0)
    g.close()


@pytest.mark.parametrize("index", [BRICKS, CELLS], ids=["bricks", "cells"])
def test_nearest_search_device_over_two_chunks(gpu_lib, frames, index):
    """2^20 + 4099 device queries in one asynchronous call, against the host twin that stages them in two chunks"""
    torch = _torch()
    c = frames["strided"]
    nq = (1 << 20) + 4099
    N = len(c["body_xyz"])
    poses = [c["pose_init"], c["pose_gt"]] + [scenes.perturb_pose(c["pose_gt"], 90 + i, 0.3, 0.05) for i in range(nq // N)]
    q = np.ascontiguousarray(np.concatenate([_world(c["body_xyz"], p) for p in poses])[:nq])
    g = gpu_lib.LiInitGpu(c["ds"], max_map_points=2_200_000, max_scan_points=N + 16, knn_index=index)
    g.map_build(c["map_xyz"])
    hx, hd, hc = g.nearest_search(q)
    dx, dd, dc = g.nearest_search(torch.from_numpy(q).cuda())
    assert dx.is_cuda and dx.shape == (nq, 5, 3) and dc.dtype == torch.int32
    assert np.array_equal(dc.cpu().numpy(), hc) and np.array_equal(dd.cpu().numpy(), hd) and np.array_equal(dx.cpu().numpy(), hx)
    g.close()


def test_stream_order_without_synchronise(gpu_lib, frames):
    """inputs produced by torch kernels on the current stream immediately before the calls, outputs consumed by torch right after:
    the binding's event handshake orders them, no synchronise anywhere"""
    torch = _torch()
    c = frames["C2"]
    p = c["pose_init"]
    mk = lambda: gpu_lib.LiInitGpu(c["ds"], max_map_points=2 * len(c["map_xyz"]), max_scan_points=len(c["body_xyz"]) + 16)  # noqa: E731
    dev = mk()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):                        # a non-default current stream, as a pipeline would have
        big = torch.from_numpy(np.ascontiguousarray(c["map_xyz"])).pin_memory().cuda(non_blocking=True)
        m = (big * 3.0 - 1.0)                            # a chain of torch kernels the upload has to wait for
        m = (m + 1.0) / 3.0                              # (not x again in float32: the host twin gets what torch made)
        dev.map_build(m)
        body = torch.from_numpy(np.ascontiguousarray(c["body_xyz"])).pin_memory().cuda(non_blocking=True) * 1.0
        dev.scan_upload(body)
        got = dev.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
        qx, qd, qc = dev.nearest_search(m[:50000] + 0.0)
        s = qd.sum() + qc.sum()                          # consumed by torch at once, on the same stream
        del big, body                                    # their memory may go back to torch's allocator right away
    side.synchronize()
    # the map the device twin built holds exactly what torch computed (a second context, compared as a set) ...
    host = mk()
    host.map_build(m.cpu().numpy())
    assert dev.map_validnum() == host.map_validnum() and _same_set(dev.map_download(), host.map_download())
    host.close()
    # ... and on that map (one pool order for exact-distance ties) the host twins reproduce the device twins' results
    dev.scan_upload(c["body_xyz"])
    want = dev.icp_iterate(p.rot_end, p.pos_end, p.R_LI, p.T_LI, False, True)
    wx, wd, wc = dev.nearest_search(m[:50000].cpu().numpy())
    assert want[2] > 0 and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(want, got))
    assert np.array_equal(qx.cpu().numpy(), wx) and np.array_equal(qd.cpu().numpy(), wd) and np.array_equal(qc.cpu().numpy(), wc)
    assert s.item() == (torch.from_numpy(wd).cuda().sum() + torch.from_numpy(wc).cuda().sum()).item()
    dev.close()


def test_odometry_loop_raw_upload_device(gpu_lib):
    """40 raw timed scans through the LiDAR-only loop of odometry.LidarOdometry (undistortion, voxel grid, IESKF, map update), once
    with host uploads and once staging every scan from a CUDA tensor: the same state at every scan, bit for bit"""
    torch = _torch()
    import frame_oracle as fo
    from lidar_imu_init_b200 import odometry

    class DeviceOdometry(odometry.LidarOdometry):
        def _stage(self, raw):
            self.g.raw_upload(torch.from_numpy(np.ascontiguousarray(raw)).cuda(), 9)

    scene = scenes.box_scene(15.0, 15.0, 6.0, 2, 2)
    ds = 0.3
    mk = lambda: gpu_lib.LiInitGpu(ds, max_map_points=2_000_000, max_scan_points=120_000)  # noqa: E731
    gh, gd = mk(), mk()
    oh, od = odometry.LidarOdometry(gh, ds), DeviceOdometry(gd, ds)
    for k in range(40):
        t0 = 10.0 + 0.1 * k
        raw = scenes.timed_scan_points(scene, fo._pose_at, t0, 0.1, 60_000, seed=100 + k, det_range=60.0, sigma=0.01)
        sh = np.array(oh.process_raw(raw, t0))
        sd = np.array(od.process_raw(raw, t0))
        assert np.array_equal(sh, sd), k
    assert oh.frame_num == od.frame_num == 39 and gh.map_validnum() == gd.map_validnum()
    gh.close()
    gd.close()


def test_other_device_refused(gpu_lib, frames):
    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    c = frames["C2"]
    g = gpu_lib.LiInitGpu(c["ds"], max_map_points=2 * len(c["map_xyz"]), max_scan_points=len(c["body_xyz"]) + 16, device_id=0)
    g.map_build(c["map_xyz"])
    n = g.map_validnum()
    with pytest.raises(gpu_lib.LiInitError) as e:
        g.map_build(torch.from_numpy(np.ascontiguousarray(c["map_xyz"])).to("cuda:1"))
    assert e.value.code == -1 and "device 1" in str(e.value)
    assert g.map_validnum() == n
    g.close()


def test_communicator_refused(gpu_lib, frames):
    """under a communicator (here one rank) the device twins refuse, and the host twins still work"""
    torch = _torch()
    c = frames["C2"]
    g = gpu_lib.LiInitGpu(c["ds"], max_map_points=2 * len(c["map_xyz"]), max_scan_points=len(c["body_xyz"]) + 16)
    try:
        g.comm_init(gpu_lib.LiInitGpu.comm_unique_id(), 1, 0)
    except gpu_lib.LiInitError as e:
        g.close()
        pytest.skip(f"no NCCL communicator: {e}")
    g.map_build(c["map_xyz"])
    n, launches = g.map_validnum(), g.launch_count()
    for call in (lambda t: g.map_build(t), lambda t: g.scan_upload(t), lambda t: g.raw_upload(t, -1), lambda t: g.nearest_search(t)):
        with pytest.raises(gpu_lib.LiInitError) as e:
            call(torch.from_numpy(np.ascontiguousarray(c["body_xyz"])).cuda())
        assert e.value.code == -1 and "communicator" in str(e.value)
    assert g.map_validnum() == n and g.launch_count() == launches
    g.close()
