"""Register budget of the ICP hot path (CPU: nvcc cross-compiles sm_90a without a GPU).

The 5-NN search kernel is latency bound and the plane kernel of a search pass runs at its 128-register cap; a spill puts local-memory
round trips into both. ptxas (-Xptxas -v, the library's own flags) must report no stack frame and no spill bytes for:
  * every k_knn_scan instantiation at G = 4 and 8 (first pass, seeded later pass, attached host scan);
  * the lidar-only plane kernels of a search pass, k_icp_plane<false, true, *> (the metric's pass).
"""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_imu_init_b200 import _build  # noqa: E402

_ENTRY = re.compile(r"Compiling entry function '(\w+)'")
_PROPS = re.compile(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
_REGS = re.compile(r"Used (\d+) registers")
_KNN = re.compile(r"_Z10k_knn_scanILi(\d+)ELb([01])ELb([01])EE")
_PLANE = re.compile(r"_Z11k_icp_planeILb([01])ELb([01])ELb([01])EE")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    # device code only (-cubin): ptxas sees the same PTX as in the shared library build
    flags = [f for f in _build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-shared")]
    out = str(tmp_path_factory.mktemp("ptxas") / "liinit_gpu.cubin")
    r = subprocess.run([nvcc] + flags + ["-cubin", "-Xptxas", "-v", "-o", out, os.path.join(_build.CSRC, "liinit_gpu.cu")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    report, name = {}, None
    for line in r.stderr.splitlines():
        m = _ENTRY.search(line)
        if m:
            name = m.group(1)
            continue
        m = _PROPS.search(line)
        if m and name:
            report[name] = {"stack": int(m.group(1)), "spill_st": int(m.group(2)), "spill_ld": int(m.group(3))}
            continue
        m = _REGS.search(line)
        if m and name in report:
            report[name]["regs"] = int(m.group(1))
    return report


def _select(report, pattern, want):
    return {n: v for n, v in report.items() if (m := pattern.match(n)) and want(m)}


def test_search_kernels_do_not_spill(ptxas_report):
    ks = _select(ptxas_report, _KNN, lambda m: int(m.group(1)) in (4, 8))
    assert len(ks) == 6, sorted(ks)
    bad = {n: v for n, v in ks.items() if v["stack"] or v["spill_st"] or v["spill_ld"]}
    assert not bad, bad


def test_search_pass_plane_kernels_do_not_spill(ptxas_report):
    ks = _select(ptxas_report, _PLANE, lambda m: m.group(1) == "0" and m.group(2) == "1")
    assert len(ks) == 2, sorted(ks)
    bad = {n: v for n, v in ks.items() if v["stack"] or v["spill_st"] or v["spill_ld"]}
    assert not bad, bad
