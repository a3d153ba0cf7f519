"""The map assessment on the H100, on the 60 s Livox scenario of tests/test_gpu_bag.py (true extrinsic: tests/calib_sim.py): `run --assess`
leaves every other result file byte-identical; the as-run placement equals the published REGISTERED records of sampled updates; the
per-query values of the whole stored LIO phase match the numpy restatement on a query sample and repeat bit for bit; the measure
ranks perturbed and grossly wrong extrinsics above the final one. Plus (CPU: nvcc only) ptxas reports no spills for the new kernels."""
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import assess_oracle as ao  # noqa: E402
from lidar_imu_init_b200 import _build, assess  # noqa: E402

SAMPLE_EVERY = 40   # stored updates whose REGISTERED records are kept for the placement check


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("assess")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"samples": []}

    def on_node(nd):
        g = nd.odom.g
        seen["g"] = g
        seen["assessment"] = nd.assess
        g.close = lambda: None                      # kept open for the tests below; closed at teardown
        real = nd.assess.append

        def append(R, p, RLI, TLI):
            k = g.assess_info()["scans"]
            off = g.assess_info()["points"]
            if k % SAMPLE_EVERY == 0:
                seen["samples"].append((off, g.cloud(capi.CLOUD_REGISTERED, R, p, RLI, TLI)[:, :3].copy()))
            real(R, p, RLI, TLI)
        nd.assess.append = append
    outs = []
    for i, extra in enumerate(([], ["--assess"])):
        out = str(tmp / f"out{i}")
        argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet"] + extra
        assert run.main(argv, on_node=on_node if extra else None) == 0
        outs.append(out)
    seen["outs"] = outs
    yield seen
    capi.LiInitGpu.close(seen["g"])


@pytest.mark.gpu
def test_runner_files_identical_and_report_parses(runs):
    a, b = runs["outs"]
    files = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    assert "result/Initialization_result.txt" in files and "result/assessment.txt" not in files
    for f in files:
        assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read(), f
    text = open(os.path.join(b, "result", "assessment.txt")).read()
    print(text, flush=True)
    rep = assess.parse_report(text)
    info = runs["g"].assess_info()
    assert rep["header"]["scans"] == info["scans"] > 500 and rep["header"]["skipped"] == 0 and rep["header"]["points"] == info["points"]
    assert rep["header"]["queries"] <= 2_000_000 and len(rep["rows"]) == 14 and len(rep["axes"]) == 6


@pytest.mark.gpu
def test_as_run_placement_equals_registered_records(runs):
    g = runs["g"]
    g.assess_evaluate(radius=0.3, min_neighbors=10, as_run=True)
    w = g.assess_placed()
    assert len(runs["samples"]) > 10
    for off, rec in runs["samples"]:
        np.testing.assert_array_equal(w[off:off + len(rec)], rec)


@pytest.mark.gpu
def test_parity_with_restatement_and_determinism(runs):
    g = runs["g"]
    R, T = _final(runs)
    res = g.assess_evaluate(R, T, radius=0.3, min_neighbors=10)
    h, v, n = g.assess_download()
    w = g.assess_placed()
    print(f"final: {res}", flush=True)
    assert res["points"] > 5_000_000 and res["queries"] <= 2_000_000 and res["valid"] > 0.5 * res["queries"]
    # a query sample against the restatement: candidates from a kd-tree (radius + 1 mm), the definitions applied to them exactly
    from scipy.spatial import cKDTree
    s = res["stride"]
    sample = np.linspace(0, res["queries"] - 1, 3000).astype(np.int64)
    tree = cKDTree(w.astype(np.float64))
    on, oh, ov = ao.evaluate_sample(w, tree, sample * s, 0.3, 10)
    np.testing.assert_array_equal(n[sample], on)
    np.testing.assert_array_equal(np.isnan(h[sample]), np.isnan(oh))
    ok = ~np.isnan(oh)
    np.testing.assert_allclose(h[sample][ok], oh[ok], rtol=0, atol=1e-9)
    np.testing.assert_allclose(v[sample][ok], ov[ok], rtol=1e-9, atol=0)
    valid = ~np.isnan(h)
    assert res["valid"] == valid.sum() and res["sparse"] == (n < 10).sum()
    assert res["mme"] == pytest.approx(h[valid].mean(), abs=1e-9)
    res2 = g.assess_evaluate(R, T, radius=0.3, min_neighbors=10)
    h2, v2, n2 = g.assess_download()
    assert res2 == res and h2.tobytes() == h.tobytes() and v2.tobytes() == v.tobytes() and n2.tobytes() == n.tobytes()


def _final(runs):
    """the extrinsic of the last stored scan"""
    return runs["assessment"].final


@pytest.mark.gpu
def test_discrimination(runs):
    """At 1 deg and 5 cm the perturbations of the final extrinsic score a higher MME, a grossly wrong extrinsic (3 deg yaw, 10 cm) scores
    clearly higher, and the simulated true extrinsic scores within a small margin of the final one.

    Finding on this scene (H100, 9.69 M stored points): T_x does not separate towards -x. Moving T_x by -5 cm LOWERS the MME by 0.0054
    (+5 cm raises it by 0.043); every other perturbation raises it by 0.0095 (T_z) to 0.18 (rotations). The stored poses were estimated
    together with the run's extrinsic, so the final extrinsic is self-consistent with them; the true one (5 mm off in T_x) scores 0.0059
    worse than final. The test pins this instead of hiding it: trans_x- is asserted to be the only perturbation that does not separate."""
    import calib_sim
    g = runs["g"]
    R0, T0 = _final(runs)
    ev = lambda R, T: g.assess_evaluate(R, T, radius=0.3, min_neighbors=10)["mme"]   # noqa: E731
    f = ev(R0, T0)
    d = {}
    for name, R, T in assess.candidates(R0, T0, dtheta_deg=1.0, dt=0.05)[2:]:
        d[name] = ev(R, T) - f
    gross = ev(assess.rot_exp([0, 0, math.radians(3.0)]) @ R0, T0 + [0.1, 0.0, 0.0]) - f
    S = calib_sim.make_streams(seed=0, duration=60.0, t_off=0.013)
    true = ev(S["R_LI"], S["T_LI"]) - f
    print(f"MME final {f:.6f}; differences: " + ", ".join(f"{k} {x:+.6f}" for k, x in d.items()) + f"; gross {gross:+.6f}; true {true:+.6f}",
          flush=True)
    assert [k for k, x in d.items() if not x > 0] == ["trans_x-"], d
    assert gross > 2 * max(d.values()), (gross, d)
    rot = min(x for k, x in d.items() if k.startswith("rot"))
    assert abs(true) < 0.1 * rot, (true, d)


# ---- registers (nvcc cross-compiles sm_90a; no GPU needed) ----
_ENTRY = re.compile(r"Compiling entry function '(\w+)'")
_PROPS = re.compile(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
_NEW = re.compile(r"_Z\d+(k_as_\w+?|k_rs_gather_hi)P")


def test_assess_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    flags = [f for f in _build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-shared")]
    r = subprocess.run([nvcc] + flags + ["-cubin", "-Xptxas", "-v", "-o", str(tmp_path / "l.cubin"), os.path.join(_build.CSRC, "liinit_gpu.cu")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    report, name = {}, None
    for line in r.stderr.splitlines():
        m = _ENTRY.search(line)
        if m:
            name = m.group(1)
            continue
        m = _PROPS.search(line)
        if m and name and _NEW.match(name):
            report[name] = tuple(int(x) for x in m.groups())
    names = {_NEW.match(k).group(1) for k in report}
    assert names == {"k_as_store", "k_as_place", "k_as_key", "k_as_gather", "k_as_mark", "k_as_index", "k_as_task_count", "k_as_task_emit",
                     "k_as_moments", "k_as_reduce", "k_rs_gather_hi"}, sorted(names)
    bad = {k: v for k, v in report.items() if any(v)}
    assert not bad, bad
