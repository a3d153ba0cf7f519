"""CPU tests of the LIO mode of the loop: the IMU branch of ImuProcess in the host library (liinit_imu_*) against a literal restatement
(tests/cpp/lio_oracle.cpp) and a closed form, the switch scan, the pose-table capacity, the world-frame export of the undistorted raw cloud and a
short LIO lockstep of LidarOdometry.process_raw on the CPU build of the device library (tests/emul)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


@pytest.fixture(scope="module")
def host_mod():
    from lidar_imu_init_b200 import _build, host
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    return host


def _random_case(rng, host, orc, n, before_last_end=False):
    s = host.state_init()
    s[0:9] = orc.so3_exp(rng.normal(size=3)).reshape(9)
    s[9:12] = rng.normal(size=3) * 5
    s[12:21] = orc.so3_exp(rng.normal(size=3) * 0.1).reshape(9)
    s[21:24] = rng.normal(size=3) * 0.1
    s[24:27] = rng.normal(size=3)
    s[27:30] = rng.normal(size=3) * 0.01
    s[30:33] = rng.normal(size=3) * 0.05
    g = rng.normal(size=3)
    s[33:36] = g / np.linalg.norm(g) * 9.81
    A = rng.normal(size=(24, 24)) * 0.1
    s[36:] = (A @ A.T + np.eye(24) * 1e-4).reshape(-1)
    t0 = 50.0 + rng.uniform()
    ts = t0 + np.arange(n) / 200.0
    mean_norm = rng.uniform(9.6, 10.0)
    smp = np.concatenate([ts[:, None], rng.normal(size=(n, 3)) * 0.5, rng.normal(size=(n, 3)) * 2 + [0, 0, mean_norm]], 1)
    last_imu = np.concatenate([[t0 - 0.005], rng.normal(size=3) * 0.5, rng.normal(size=3) * 2 + [0, 0, mean_norm]])
    # last_lidar_end_time_: after the first samples (pairs skipped, the first kept one measured from it) or before all of them
    last_end = t0 + rng.uniform(0.0, min(n, 6) / 200.0) if before_last_end else t0 - rng.uniform(0.0, 0.004)
    angvel_last, acc_s_last = rng.normal(size=3), rng.normal(size=3)
    return s, smp, last_imu, last_end, mean_norm, angvel_last, acc_s_last


def _product_imu(host, last_imu, last_end, mean_norm, angvel_last, acc_s_last, covs):
    p = host.ImuProcess()
    for k, v in covs.items():
        p.set_cov(k, v)
    p.set_mean_acc_norm(mean_norm)
    p.switch(last_imu[None])
    p.m.last_lidar_end_time = last_end
    for i in range(3):
        p.m.angvel_last[i] = angvel_last[i]
        p.m.acc_s_last[i] = acc_s_last[i]
    return p


def _oracle_imu(orc, last_imu, last_end, mean_norm, angvel_last, acc_s_last, covs):
    import lio_oracle
    o = lio_oracle.OracleImu()
    for k, v in covs.items():
        o.set_cov(k, v)
    o.set_mean_acc_norm(mean_norm)
    o.switch(last_imu[None])
    o.m[13] = last_end
    o.m[7:10] = angvel_last
    o.m[10:13] = acc_s_last
    return o


def test_imu_propagation_matches_oracle_restatement(host_mod, oracle_mod):
    """Random groups of 1..25 samples at 200 Hz, random biases / gravity / mean_acc_norm / covariances; groups that start before
    last_lidar_end_time_; scan ends after the last sample (note = +1) and before it (note = -1). State, 24x24 covariance, pose table
    and the updated members agree within 1e-12 relative."""
    host, orc = host_mod, oracle_mod
    rng = np.random.default_rng(7)
    notes = set()
    skipped = 0
    for trial in range(300):
        n = int(rng.integers(1, 26))
        s, smp, last_imu, last_end, mn, wl, al = _random_case(rng, host, orc, n, before_last_end=trial % 3 == 0)
        covs = {k: rng.uniform(1e-5, 1.0, 3) for k in ("gyr_cov", "acc_cov", "R_LI_cov", "T_LI_cov", "gyr_bias_cov", "acc_bias_cov")}
        p = _product_imu(host, last_imu, last_end, mn, wl, al, covs)
        o = _oracle_imu(orc, last_imu, last_end, mn, wl, al, covs)
        beg = smp[0, 0] - rng.uniform(0.0, 0.01)
        end_ms = (smp[-1, 0] - beg + rng.uniform(-0.004, 0.004)) * 1000.0
        notes.add(beg + end_ms / 1000.0 > smp[-1, 0])
        sp, pp = p.propagate(s, smp, beg, end_ms)
        so, po = o.propagate(s, smp, beg, end_ms)
        skipped += n + 1 - len(po)
        assert pp.shape == po.shape and len(pp) >= 1
        np.testing.assert_allclose(sp[:36], so[:36], rtol=1e-12, atol=1e-12 * np.abs(so[:36]).max())
        np.testing.assert_allclose(sp[36:], so[36:], rtol=1e-12, atol=1e-12 * np.abs(so[36:]).max())
        np.testing.assert_allclose(pp, po, rtol=1e-12, atol=1e-12 * max(np.abs(po).max(), 1.0))
        np.testing.assert_allclose(np.array(p.m.angvel_last[:] + p.m.acc_s_last[:]), o.m[7:13], rtol=1e-12, atol=1e-12)
        assert p.m.last_lidar_end_time == o.m[13] == beg + end_ms / 1000.0
        assert list(p.m.last_imu) == list(smp[-1])
    assert notes == {True, False} and skipped > 50


def test_imu_propagation_closed_form(host_mod):
    """Constant rate and a specific force along the rotation axis: the world acceleration R a + g is constant, so the discrete
    scheme of propagation_and_undist is exact -- R = R0 Exp(w t), p = p0 + v0 t + a t^2 / 2 -- and the pose table holds the same
    closed form at every sample. Forward extrapolation (note = +1) is exact too; backward (note = -1) keeps the reference's sign of
    the quadratic term (p_last - v_last dt - a dt^2 / 2). One covariance step against numpy's dense F P F^T + Q."""
    host = host_mod
    from lidar_imu_init_b200 import scenes
    w_true = np.array([0.3, -0.2, 0.5])
    axis = w_true / np.linalg.norm(w_true)
    bg, ba, g = np.array([0.01, -0.02, 0.005]), np.array([0.1, 0.05, -0.08]), np.array([0.3, -0.4, -9.79])
    mean_norm = 9.7
    f = 2.5 * axis                                             # specific force (bias-free, in m/s^2)
    R0 = scenes.rot_from_rpy(0.1, -0.2, 0.7)
    p0, v0 = np.array([1.0, 2.0, 3.0]), np.array([0.5, -0.3, 0.2])
    s = host.state_from_pose(R0, p0, np.eye(3), np.zeros(3))
    s[24:27], s[27:30], s[30:33], s[33:36] = v0, bg, ba, g
    t0 = 10.0
    n = 9
    reading = np.concatenate([w_true + bg, (f + ba) * mean_norm / 9.81])
    smp = np.concatenate([(t0 + 0.005 * (1 + np.arange(n)))[:, None], np.tile(reading, (n, 1))], 1)
    A = R0 @ f + g

    def expect(t):
        return R0 @ scenes.so3_exp(w_true * t), p0 + v0 * t + 0.5 * A * t * t, v0 + A * t

    for note, end in ((1, smp[-1, 0] + 0.0032), (-1, smp[-1, 0] - 0.0021)):
        p = host.ImuProcess()
        p.set_mean_acc_norm(mean_norm)
        p.switch(np.concatenate([[t0], reading])[None])
        beg = t0 + 0.001
        sp, poses = p.propagate(s, smp, beg, (end - beg) * 1000.0)
        assert len(poses) == n + 1
        np.testing.assert_array_equal(poses[0, 7:10], v0)
        for k in range(1, n + 1):
            R, pos, vel = expect(smp[k - 1, 0] - t0)
            assert abs(poses[k, 0] - (smp[k - 1, 0] - beg)) < 1e-15
            np.testing.assert_allclose(poses[k, 13:22].reshape(3, 3), R, atol=1e-12)
            np.testing.assert_allclose(poses[k, 10:13], pos, atol=1e-12)
            np.testing.assert_allclose(poses[k, 7:10], vel, atol=1e-12)
            np.testing.assert_allclose(poses[k, 1:4], A, atol=1e-12)
            np.testing.assert_allclose(poses[k, 4:7], w_true, atol=1e-12)
        R, pos, vel = expect(end - t0)
        np.testing.assert_allclose(sp[0:9].reshape(3, 3), R, atol=1e-12)
        np.testing.assert_allclose(sp[24:27], vel, atol=1e-12)
        if note == 1:
            np.testing.assert_allclose(sp[9:12], pos, atol=1e-12)
        else:
            dt = smp[-1, 0] - end
            _, pl, vl = expect(smp[-1, 0] - t0)
            np.testing.assert_allclose(sp[9:12], pl - vl * dt - 0.5 * A * dt * dt, atol=1e-12)
            assert np.abs(sp[9:12] - pos).max() > 1e-6

    # covariance: one pair, against the dense product
    P = np.random.default_rng(3).normal(size=(24, 24))
    P = P @ P.T
    s[36:] = P.reshape(-1)
    p = host.ImuProcess()
    p.set_mean_acc_norm(mean_norm)
    p.switch(np.concatenate([[t0], reading])[None])
    dt = 0.005
    sp, _ = p.propagate(s, smp[:1], t0, dt * 1000.0)
    acc = f                                                     # bias-corrected, rescaled mean specific force
    K = np.array([[0, -acc[2], acc[1]], [acc[2], 0, -acc[0]], [-acc[1], acc[0], 0]])
    F = np.eye(24)
    F[0:3, 0:3] = scenes.so3_exp(-w_true * dt)
    F[0:3, 15:18] = -np.eye(3) * dt
    F[3:6, 12:15] = np.eye(3) * dt
    F[12:15, 0:3] = -R0 @ K * dt
    F[12:15, 18:21] = -R0 * dt
    F[12:15, 21:24] = np.eye(3) * dt
    Q = np.zeros((24, 24))
    Q[0:3, 0:3] = np.eye(3) * 0.1 * dt * dt
    Q[6:9, 6:9] = np.eye(3) * 1e-5 * dt * dt
    Q[9:12, 9:12] = np.eye(3) * 1e-4 * dt * dt
    Q[12:15, 12:15] = R0 @ (np.eye(3) * 0.1) @ R0.T * dt * dt
    Q[15:18, 15:18] = np.eye(3) * 1e-4 * dt * dt
    Q[18:21, 18:21] = np.eye(3) * 1e-4 * dt * dt
    np.testing.assert_allclose(sp[36:].reshape(24, 24), F @ P @ F.T + Q, rtol=1e-11, atol=1e-11 * np.abs(P).max())


def test_switch_scan(host_mod):
    """Process after LI_init_done (IMU_Processing.hpp:445-453): the first group only records its last sample and takes the
    covariance scales; the state is not touched (not even an argument) and propagation is refused before it."""
    host = host_mod
    from lidar_imu_init_b200 import capi
    p = host.ImuProcess()
    assert p.need_init and p.m.mean_acc_norm == 9.81 and list(p.m.cov_acc) == [0.1] * 3
    assert list(p.m.acc_s_last) == [0.0] * 3 and p.m.last_lidar_end_time == 0.0
    s = host.state_init()
    grp = np.array([[1.0, 0.1, 0.2, 0.3, 0.0, 0.0, 9.8], [1.005, 0.4, 0.5, 0.6, 0.1, 0.2, 9.7]])
    with pytest.raises(capi.LiInitError) as e:
        p.propagate(s, grp, 0.99, 10.0)
    assert e.value.code == -1
    p.switch(np.zeros((0, 7)))                                  # an empty group changes nothing
    assert p.need_init
    p.set_cov("acc_cov", [2.0, 3.0, 4.0])
    p.set_cov("gyr_cov", 50.0)
    p.switch(grp)
    assert not p.need_init and list(p.m.last_imu) == list(grp[-1])
    assert list(p.m.cov_acc) == [2.0, 3.0, 4.0] and list(p.m.cov_gyr) == [50.0] * 3
    sp, poses = p.propagate(s, grp[:0], 1.0, 10.0)              # an empty group: nothing happens
    assert len(poses) == 0 and np.array_equal(sp, s)


def test_pose_table_capacity(host_mod):
    """A table longer than the device's 4096 poses is refused before anything changes; 4096 poses are accepted."""
    host = host_mod
    from lidar_imu_init_b200 import capi
    n = host.MAX_IMU_POSES
    smp = np.zeros((n, 7))
    smp[:, 0] = 1.0 + np.arange(n) * 0.005
    smp[:, 6] = 9.81
    p = host.ImuProcess()
    p.switch(np.array([[0.995, 0, 0, 0, 0, 0, 9.81]]))
    before = bytes(p.m)
    s = host.state_init()
    with pytest.raises(capi.LiInitError) as e:
        p.propagate(s, smp, 1.0, 1000.0)
    assert e.value.code == -3 and bytes(p.m) == before
    sp, poses = p.propagate(s, smp[:n - 1], 1.0, 1000.0)
    assert len(poses) == n
    p2 = host.ImuProcess()
    p2.switch(np.array([[0.995, 0, 0, 0, 0, 0, 9.81]]))
    p2.m.last_lidar_end_time = smp[10, 0] + 1e-4                # pairs older than the previous scan end do not count
    _, poses = p2.propagate(s, smp, 1.0, 1000.0)
    assert len(poses) == n + 1 - 11


def _emul():
    import liinit_emul as le
    if not le.available():
        pytest.skip("g++ or the CUDA vector-type headers are missing")
    L = le.load()
    L.liinit_raw_download_world.argtypes = [le.vp, le._f64, le._f64, le._f64, le._f64, le.vp, C.c_int, C.POINTER(C.c_int)]

    class EmulGpu(le.EmulGpu):
        def raw_world(self, rot_end, pos_end, R_LI, T_LI):
            n = C.c_int()
            a = (le._c64(rot_end).reshape(9), le._c64(pos_end), le._c64(R_LI).reshape(9), le._c64(T_LI))
            self._ck(self.L.liinit_raw_download_world(self.h, *a, None, 0, C.byref(n)))
            out = np.zeros((n.value, 3), np.float32)
            self._ck(self.L.liinit_raw_download_world(self.h, *a, out.ctypes.data_as(le.vp), n.value, C.byref(n)))
            return out
    return le, EmulGpu


def test_world_export_on_the_cpu_build(host_mod, oracle_mod):
    """liinit_raw_download_world on the CPU build of the library: bit-equal to the oracle's pointBodyToWorld of the staged
    (IMU-undistorted) cloud, in upload order; the kernel reaches the emulation through the launch rewrite."""
    import lio_oracle
    orc = oracle_mod
    le, EmulGpu = _emul()
    gen = open(os.path.join(ROOT, "tests", "emul", "_gen", "liinit_gpu_emul.cpp")).read()
    assert "(k_raw_to_world)(" in gen and "k_raw_to_world<<<" not in gen
    rng = np.random.default_rng(5)
    g = EmulGpu(0.15, max_scan_points=4000)
    n = 3000
    raw = np.zeros((n, 12), np.float32)
    raw[:, 0:3] = rng.uniform(-30, 30, (n, 3))
    raw[:, 9] = np.sort(rng.uniform(0, 100, n)).astype(np.float32)
    rng.shuffle(raw)                                            # upload order is not time order
    g.raw_upload(raw, 9)
    with pytest.raises(le.EmulError):                           # capacity: fewer slots than staged points
        m = C.c_int()
        z = np.zeros((10, 3), np.float32)
        g._ck(g.L.liinit_raw_download_world(g.h, np.eye(3).reshape(9), np.zeros(3), np.eye(3).reshape(9), np.zeros(3),
                                            z.ctypes.data_as(le.vp), 10, C.byref(m)))
    poses = np.zeros((6, 22))
    poses[:, 0] = np.linspace(0, 0.1, 6)
    poses[:, 1:13] = rng.normal(size=(6, 12))
    for k in range(6):
        poses[k, 13:22] = orc.so3_exp(rng.normal(size=3) * 0.1).reshape(9)
    R, p = orc.so3_exp([0.3, -0.2, 1.1]), np.array([5.0, -3.0, 1.5])
    RLI, TLI = orc.so3_exp([0.01, 0.02, 1.5]), np.array([-0.02, 0.03, 0.15])
    g.raw_undistort_imu(poses, R, p, RLI, TLI)
    staged = g.raw_points()
    np.testing.assert_array_equal(staged, orc.undistort_imu(raw[:, 0:3], raw[:, 9], poses, R, p, RLI, TLI))
    R2, p2 = orc.so3_exp([-0.5, 0.1, 0.4]), np.array([100.25, -40.5, 3.0])
    w = g.raw_world(R2, p2, RLI, TLI)
    assert w.shape == (n, 3)
    np.testing.assert_array_equal(w, lio_oracle.body_to_world(staged, R2, p2, RLI, TLI))
    g.close()


def _lio_legs(oracle_mod, points, undistort=True, with_product=True):
    import lio_case
    from lidar_imu_init_b200.odometry import LidarOdometry
    kw = dict(max_iteration=4, orig_odom_freq=10, cut_frame_num=5)
    legs = {"oracle": lio_case.make_oracle_odometry(oracle_mod, 0.15, lio_case.default_threads(), undistort=undistort, **kw)}
    if with_product:
        le, EmulGpu = _emul()

        class EmulOdometry(LidarOdometry):
            def _scan_update_resident(self, state):
                return le.scan_update(self.g, state, self.max_iteration, self.imu_en)

        legs["product"] = EmulOdometry(EmulGpu(0.15, max_map_points=400_000, max_scan_points=points + 16), 0.15, **kw)
    return legs


def test_lio_lockstep_on_the_cpu_build(host_mod, oracle_mod):
    """About 30 scans of 300 timed points from the hand-over on (true calibration, map from the scene): one LiDAR-only scan, the
    switch scan, then LIO scans -- IMU propagation in the host library, the raw chain and the update on the CPU build of the device
    library -- in lockstep with the oracle leg. Poses, extrinsic and world clouds agree within 1e-6 scan after scan."""
    import lio_case
    legs = _lio_legs(oracle_mod, 300)
    diffs = dict(dp=0.0, dr=0.0, dT=0.0, dRLI=0.0, dw=0.0, lio=0)

    def on_scan(j, legs, truth):
        from lidar_imu_init_b200 import host
        Rg, pg, RLg, TLg = host.state_pose(legs["product"].state)
        Ro, po, RLo, TLo = host.state_pose(legs["oracle"].state)
        diffs["dp"] = max(diffs["dp"], float(np.abs(pg - po).max()))
        diffs["dr"] = max(diffs["dr"], lio_case.angle(Rg, Ro))
        diffs["dT"] = max(diffs["dT"], float(np.abs(TLg - TLo).max()))
        diffs["dRLI"] = max(diffs["dRLI"], lio_case.angle(RLg, RLo))
        diffs["dw"] = max(diffs["dw"], float(np.abs(legs["product"].world_cloud() - legs["oracle"].world_cloud()).max()))
        diffs["lio"] += int(truth["lio"])

    out = lio_case.run(legs, oracle_mod, seconds=0.7, points=300, t_start=8.0, scans=30, map_from_scene=True, on_scan=on_scan)
    assert out["switch_scan"] == out["init_scan"] + 1 and diffs["lio"] == 29
    assert legs["product"].switch_scan == legs["oracle"].switch_scan == 1
    assert max(diffs["dp"], diffs["dr"], diffs["dT"], diffs["dRLI"]) <= 1e-6, diffs
    assert diffs["dw"] <= 1e-4, diffs


def test_lio_negative_control_on_the_oracle_half(oracle_mod, host_mod):
    """The same LIO scans on the oracle half, once with the IMU undistortion and once with it skipped: the error against the
    simulated truth is several times larger without it -- the scans are distorted enough for the lockstep to test the undistortion."""
    import lio_case
    err = {}
    for undistort in (True, False):
        legs = _lio_legs(oracle_mod, 300, undistort=undistort, with_product=False)
        e = dict(dp=[], dr=[])

        def on_scan(j, legs, truth):
            from lidar_imu_init_b200 import host
            if truth["lio"]:
                R, p, _, _ = host.state_pose(legs["oracle"].state)
                R_t, p_t = truth["imu"]
                e["dp"].append(float(np.linalg.norm(p - p_t)))
                e["dr"].append(lio_case.angle(R, R_t))

        lio_case.run(legs, oracle_mod, seconds=0.7, points=300, t_start=8.0, scans=30, map_from_scene=True, on_scan=on_scan)
        err[undistort] = (np.mean(e["dp"]), np.mean(e["dr"]))
    print("mean error vs truth with / without undistortion:", err)
    assert err[False][0] > 3 * err[True][0] or err[False][1] > 3 * err[True][1], err
