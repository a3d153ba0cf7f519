"""The assessment cloud on the H100, on the 60 s Livox scenario of tests/test_gpu_assess.py: `run --assess-cloud` leaves every other result
file byte-identical and writes the as-run leaf records; every stored point is scored, bit-equal to the strided evaluation's queries and
from call to call; a point sample matches the numpy restatement; the leaf records equal the restatement from the per-point records.
Printed for information: the full-resolution MME next to the strided one, and how many points a gross perturbation blurs. Plus (CPU:
nvcc only) ptxas reports no spills for the cloud's kernels."""
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

import assess_cloud_oracle as aco  # noqa: E402
import assess_oracle as ao  # noqa: E402
from lidar_imu_init_b200 import _build, assess  # noqa: E402


@pytest.fixture(scope="module")
def runs(tmp_path_factory, gpu_lib):
    import test_bag_node as tb
    from lidar_imu_init_b200 import capi, run
    _build.build_host()
    _build.build_calib()
    tmp = tmp_path_factory.mktemp("assess_cloud")
    tb.sim_config(tmp, online_refine_time=10.0)
    ev, _ = tb.livox_events(60.0, 20_000)
    bag = str(tmp / "livox.bag")
    tb.write_event_bag(bag, ev, chunk_msgs=300)
    seen = {"pcd": str(tmp / "assess.pcd"), "cache": {}}

    def on_node(nd):
        seen["g"] = nd.odom.g
        seen["assessment"] = nd.assess
        nd.odom.g.close = lambda: None              # kept open for the tests below; closed at teardown
    outs = []
    for i, extra in enumerate((["--assess"], ["--assess", "--assess-cloud", seen["pcd"]])):
        out = str(tmp / f"out{i}")
        argv = ["--config", str(tmp / "sim.yaml"), "--bag", bag, "--out", out, "--max-map-points", "3000000", "--quiet"] + extra
        assert run.main(argv, on_node=on_node if i else None) == 0
        outs.append(out)
    seen["outs"] = outs
    yield seen
    capi.LiInitGpu.close(seen["g"])


def _cloud(runs, which, leaf=0.0):
    """(records, totals) of the as-run or the final extrinsic, computed once per module"""
    key = (which, leaf)
    if key not in runs["cache"]:
        g = runs["g"]
        if which == "as-run":
            runs["cache"][key] = g.assess_cloud(radius=0.3, min_neighbors=10, leaf=leaf, as_run=True)
        else:
            R, T = runs["assessment"].final
            runs["cache"][key] = g.assess_cloud(R, T, radius=0.3, min_neighbors=10, leaf=leaf)
    return runs["cache"][key]


@pytest.mark.gpu
def test_runner_writes_the_as_run_cloud(runs):
    a, b = runs["outs"]
    files = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    assert "result/assessment.txt" in files
    assert files == sorted(os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs)
    for f in files:
        assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read(), f
    header, body = aco.read_assess_pcd(runs["pcd"])
    rec, tot = _cloud(runs, "as-run", 0.1)
    assert body.tobytes() == rec.tobytes()
    assert body[:, 6].sum() == runs["g"].assess_info()["points"] == tot["points"]


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["as-run", "final"])
def test_every_point_bit_equal_to_strided_evaluation(runs, which):
    g = runs["g"]
    rec, tot = _cloud(runs, which)
    info = g.assess_info()
    assert len(rec) == tot["points"] == tot["queries"] == info["points"] > 9_000_000 and tot["stride"] == 1
    assert tot["valid"] + tot["sparse"] + tot["degenerate"] == len(rec)
    R, T = runs["assessment"].final
    res = g.assess_evaluate(radius=0.3, min_neighbors=10, as_run=True) if which == "as-run" else \
        g.assess_evaluate(R, T, radius=0.3, min_neighbors=10)
    s = res["stride"]
    assert s > 1 and res["queries"] == len(rec[::s])
    h, v, n = g.assess_download()
    assert rec[::s, 3].tobytes() == h.astype(np.float32).tobytes()
    assert rec[::s, 4].tobytes() == v.astype(np.float32).tobytes()
    assert rec[::s, 5].tobytes() == n.astype(np.float32).tobytes()
    assert tot["valid"] == int(rec[:, 7].sum())
    assert tot["mme"] == pytest.approx(float(rec[rec[:, 7] == 1, 3].astype(np.float64).mean()), abs=1e-6)
    text = open(os.path.join(runs["outs"][1], "result", "assessment.txt")).read()
    row = assess.parse_report(text)["rows"][which]
    print(f"{which}: full-resolution MME {tot['mme']:.6f} over {tot['valid']} of {tot['points']} points; assessment.txt (stride {s}) "
          f"{row['mme']:.6f}; MPV {tot['mpv']:.6e} vs {row['mpv']:.6e}", flush=True)
    if which == "final":
        rec2, tot2 = g.assess_cloud(R, T, radius=0.3, min_neighbors=10, leaf=0.0)
        assert rec2.tobytes() == rec.tobytes() and tot2 == tot


def _f32_close(dev, ref):
    ref = np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(dev), np.isnan(ref))
    ok = ~np.isnan(ref)
    r32 = ref[ok].astype(np.float32)
    d = np.abs(dev[ok].astype(np.float64) - r32.astype(np.float64))
    assert (d <= np.spacing(np.abs(r32)).astype(np.float64)).all(), d.max()


@pytest.mark.gpu
def test_point_sample_matches_restatement(runs):
    """2,000 stored points of the final extrinsic's cloud against the restatement (kd-tree candidates, then the definitions): counts
    exact, h and v the float32 of values within 1e-9 of the restatement's."""
    from scipy.spatial import cKDTree
    rec, _ = _cloud(runs, "final")
    w = rec[:, :3].copy()
    k = np.linspace(0, len(rec) - 1, 2000).astype(np.int64)
    on, oh, ov = ao.evaluate_sample(w, cKDTree(w.astype(np.float64)), k, 0.3, 10)
    np.testing.assert_array_equal(rec[k, 5], on.astype(np.float32))
    _f32_close(rec[k, 3], oh)
    _f32_close(rec[k, 4], ov)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["as-run", "final"])
def test_leaf_records_equal_restatement(runs, which):
    rec0, _ = _cloud(runs, which)
    recL, _ = _cloud(runs, which, 0.1)
    ref = aco.leaf_records(rec0, 0.1)
    np.testing.assert_array_equal(recL, ref)
    print(f"{which}: {len(rec0)} points in {len(recL)} leaves of 0.1 m; {int((recL[:, 7] == 0).sum())} leaves without a valid point",
          flush=True)


@pytest.mark.gpu
def test_gross_perturbation_share(runs):
    """Information: with the final extrinsic turned by 3 deg in yaw and moved 10 cm along x, the share of points valid under both whose
    entropy rises."""
    g = runs["g"]
    R, T = runs["assessment"].final
    rec0, tot0 = _cloud(runs, "final")
    rec1, tot1 = g.assess_cloud(assess.rot_exp([0, 0, math.radians(3.0)]) @ R, T + [0.1, 0.0, 0.0], radius=0.3, min_neighbors=10,
                                leaf=0.0)
    both = (rec0[:, 7] == 1) & (rec1[:, 7] == 1)
    share = float((rec1[both, 3] > rec0[both, 3]).mean())
    print(f"3 deg yaw / 10 cm: MME {tot0['mme']:.6f} -> {tot1['mme']:.6f}; h rises at {100 * share:.1f} % of the {int(both.sum())} "
          f"points valid under both", flush=True)
    assert 0.0 <= share <= 1.0


# ---- registers (nvcc cross-compiles sm_90a; no GPU needed) ----
_ENTRY = re.compile(r"Compiling entry function '(\w+)'")
_PROPS = re.compile(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
_NEW = re.compile(r"_Z\d+(k_ac_\w+?)P")


def test_assess_cloud_kernels_do_not_spill(tmp_path):
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
    assert names == {"k_ac_point_rec", "k_ac_point_pack", "k_ac_leaf_mark", "k_ac_leaf_index", "k_ac_leaf_rec"}, sorted(names)
    bad = {k: v for k, v in report.items() if any(v)}
    assert not bad, bad
