"""Refining one calibration from several recordings (joint.search, joint.refine_replays, python -m lidar_imu_init_b200.joint) without a
GPU: with one recording the joint search is refine.search, bit for bit; two recordings that each leave a different axis flat pin every
axis together; each recording replays the shift L - lambda_b of a common total lag L; a NaN never wins; the budget counts candidates;
the report round-trips; on the emulated library the joint search over one recording is Replay.refine, its trace does not depend on the
replay jobs, and the runner writes each recording's files as `run` does and refuses bad arguments."""
import math
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lidar_imu_init_b200 import assess, joint, node, refine  # noqa: E402
from test_refine import R_STAR, R_START, T_STAR, T_START, Bowl  # noqa: E402

T_INIT = T_STAR + [0.05, 0, 0]


def _scorer(fs, calls=None):
    """score_many of joint.search over per-recording scorers fs[b](R, T, shift_b)"""
    def score_many(items):
        if calls is not None:
            calls.append(list(items))
        return [fs[b](R, T, s) for b, R, T, s in items]
    return score_many


def _rows(r, labels=None):
    labels = labels or {}
    return [(labels.get(x["stage"], x["stage"]), x["R"].tobytes(), x["T"].tobytes(), x["shift_ms"], np.float64(x["mme"]).tobytes())
            for x in r["trace"]]


def _same_as_single(j, s):
    """a joint search over one recording against refine.search / Replay.refine with the (final, li-init) start pair"""
    assert _rows(j, {"final:0": "final", "li-init:0": "li-init"}) == _rows(s)
    assert {"final:0": "final", "li-init:0": "li-init"}[j["start"]] == s["start"]
    for k in ("status", "at_edge", "best", "steps", "shift_ms", "shift_s"):
        assert j[k] == s[k], k
    assert j["R"].tobytes() == s["R"].tobytes() and j["T"].tobytes() == s["T"].tobytes()
    assert np.float64(j["mme"]).tobytes() == np.float64(s["mme"]).tobytes()
    assert list(j["axes"]) == list(s["axes"])
    for k in j["axes"]:
        assert np.array(j["axes"][k]).tobytes() == np.array(s["axes"][k]).tobytes() == np.array(j["axes_rec"][0][k]).tobytes(), k


@pytest.mark.parametrize("budget", [1, 2, 9, 40, 1000])
def test_one_recording_is_the_single_search(budget):
    f = Bowl(7.0)
    s = refine.search(f, R_START, T_START, max_replays=budget, R_init=R_STAR, T_init=T_INIT)
    j = joint.search(_scorer([f]), [-0.00297], [("final:0", R_START, T_START), ("li-init:0", R_STAR, T_INIT)], budget)
    _same_as_single(j, s)
    assert j["lag0"] == -0.00297 and j["time_lag"] == -0.00297 + j["shift_s"] and j["offsets"] == [0.0]


def test_complementary_recordings_pin_every_axis():
    """Recording 0 does not see trans_x, recording 1 not trans_y: each single search keeps its flat axis at the start's value and calls
    it flat; the joint search reaches the minimum on both and calls every axis constrained."""
    fs = [Bowl(4.0, flat=0), Bowl(4.0, flat=1)]
    for b, f in enumerate(fs):
        r = refine.search(f, R_START, T_START, max_replays=2000)
        assert r["status"] == "converged" and r["T"][b] == T_START[b]
        assert refine.axis_verdict(*r["axes"][f"trans_{'xy'[b]}"][1:]) == "flat"
    j = joint.search(_scorer(fs), [0.0, 0.0], [("final:0", R_START, T_START), ("final:1", R_START, T_START)], 2000)
    assert j["status"] == "converged"
    assert np.abs(j["T"] - T_STAR).max() <= refine.DT_MIN_M
    assert all(refine.axis_verdict(dp, dm) == "constrained" for _, dp, dm in j["axes"].values())
    # per recording: the axis a recording does not see is flat in its own differences
    assert refine.axis_verdict(*j["axes_rec"][0]["trans_x"][1:]) == "flat"
    assert refine.axis_verdict(*j["axes_rec"][1]["trans_y"][1:]) == "flat"
    assert refine.axis_verdict(*j["axes_rec"][0]["trans_y"][1:]) == "constrained"


def test_each_recording_replays_its_own_lag_shift():
    """Recordings handed over at different lags, all with their minimum at the same total lag L*: recording b is scored at L - lambda_b
    for every candidate, and the search finds L*."""
    lags, L_star = [-0.003, 0.004, 0.0105], 0.013
    fs = [Bowl((L_star - lam) * 1000.0) for lam in lags]
    calls = []
    j = joint.search(_scorer(fs, calls), lags, [(f"final:{b}", R_START, T_START) for b in range(3)], 1000)
    assert j["status"] == "converged" and j["lag0"] == (-0.003 + 0.004 + 0.0105) / 3
    assert abs(j["time_lag"] - L_star) <= refine.LAG_TOL_MS / 1000.0
    seen = set()
    for batch in calls:
        assert len(batch) % 3 == 0 and [b for b, *_ in batch] == [0, 1, 2] * (len(batch) // 3)
        seen |= {(b, R.tobytes(), T.tobytes(), s) for b, R, T, s in batch}
    for row in j["trace"]:
        for b in range(3):
            s_b = row["shift_ms"] / 1000.0 + j["offsets"][b]
            assert (b, row["R"].tobytes(), row["T"].tobytes(), s_b) in seen
            assert s_b == pytest.approx(row["lag"] - lags[b], abs=1e-15)


def test_one_recordings_nan_never_wins():
    f0, f1 = Bowl(0.0), Bowl(0.0)
    fs = [f0, lambda R, T, s: math.nan if s > 0 else f1(R, T, s)]
    j = joint.search(_scorer(fs), [0.0, 0.0], [("final:0", R_START, T_START), ("final:1", R_START, T_START)], 1000)
    assert j["mme"] == j["mme"] and j["shift_ms"] <= 0.0
    assert any(r["mme"] != r["mme"] for r in j["trace"])     # NaN candidates were scored and not taken


@pytest.mark.parametrize("budget", [1, 3, 17, 60])
def test_budget_counts_candidates(budget):
    fs = [Bowl(12.0), Bowl(12.0, flat=2)]
    calls = []
    j = joint.search(_scorer(fs, calls), [0.001, -0.001], [("final:0", R_START, T_START), ("li-init:0", R_STAR, T_INIT),
                                                           ("final:1", R_START, T_START), ("li-init:1", R_STAR, T_INIT)], budget)
    n = sum(len(c) for c in calls)
    assert len(j["trace"]) <= budget and n == 2 * len(j["trace"]) <= 2 * budget
    assert all(len(r["mmes"]) == 2 for r in j["trace"])


def _fake(rng, B=2, n=9):
    fs = [Bowl(4.0), Bowl(3.0, flat=1)][:B]
    lags = [-0.00297, 0.0011][:B]
    starts = [s for b in range(B) for s in ((f"final:{b}", R_START, T_START), (f"li-init:{b}", R_STAR, T_STAR))]
    r = joint.search(_scorer(fs), lags, starts, n)
    r["wall_s"] = 12.5
    states = []
    for b in range(B):
        s = np.zeros(612)
        s[12:21] = r["R"].reshape(9)
        s[21:24] = r["T"]
        s[27:36] = rng.normal(size=9)
        states.append(s)
    r["calibs"] = [node.state_calib_values(s, r["time_lag"]) for s in states]
    recs = [dict(bag=f"/data/run {b}.bag", subframes=100 + b, skipped=0, lag=lags[b], R_init=R_STAR, T_init=T_STAR, R_final=R_START,
                 T_final=T_START) for b in range(B)]
    return r, recs


@pytest.mark.parametrize("B", [1, 2])
def test_joint_report_round_trip(B):
    rng = np.random.default_rng(3)
    ref, recs = _fake(rng, B)
    text = assess.joint_report_text(recs, ref, 0.3, 10)
    rep = assess.parse_joint_report(text)
    h = rep["header"]
    assert (h["recordings"], h["candidates"], h["replays"], h["start"], h["status"], h["n_min"]) == (B, 9, 9 * B, ref["start"], "budget", 10)
    assert h["lag0_ms"] == pytest.approx(ref["lag0"] * 1000, abs=1e-6) and h["lag_ms"] == pytest.approx(ref["time_lag"] * 1000, abs=1e-6)
    for b, r in enumerate(rep["recs"]):
        assert r["bag"] == recs[b]["bag"] and r["subframes"] == 100 + b and r["lag_ms"] == pytest.approx(recs[b]["lag"] * 1000, abs=1e-6)
        assert r["final"][3:] == pytest.approx(tuple(T_START), abs=1e-6)
        assert r["li_init"][:3] == pytest.approx(tuple(np.degrees(node.rot_to_euler(R_STAR))), abs=1e-6)
    assert len(rep["rows"]) == 9
    for got, row in zip(rep["rows"], ref["trace"]):
        assert got["stage"] == row["stage"] and got["lag_ms"] == pytest.approx(row["lag"] * 1000, abs=1e-6)
        assert (got["t_x"], got["t_y"], got["t_z"]) == pytest.approx(tuple(row["T"]), abs=1e-6)
        assert got["mme"] == pytest.approx(row["mme"], abs=1e-9) and got["mmes"] == pytest.approx(row["mmes"], abs=1e-9)
    assert list(rep["axes"]) == ["joint"] + list(range(B))
    for who, axes in [("joint", ref["axes"])] + list(enumerate(ref["axes_rec"])):
        for axis, (step, dp, dm) in axes.items():
            v, s, p, m = rep["axes"][who][axis]
            assert v == refine.axis_verdict(dp, dm) and s == pytest.approx(step, abs=1e-6)
            assert (p == pytest.approx(dp, abs=1e-9) or (p != p and dp != dp)) and (m == pytest.approx(dm, abs=1e-9) or (m != m and dm != dm))
    assert rep["result"] == [node.calib_result_text(**c) for c in ref["calibs"]]


# ---- on the emulated library -----------------------------------------------------------------------------------------------------------
EMUL_RADIUS = 1.5   # [m] (as in test_refine: the short runs store a few thousand points)


@pytest.fixture(scope="module")
def two_runs(tmp_path_factory):
    import test_assess_replay_emul as tr
    import test_replay_jobs_emul as tj
    out = []
    for b, trigger in enumerate((6, 7)):
        nd, rp, _, _ = tr._emul_run(tmp_path_factory.mktemp(f"rec{b}"), trigger_at=trigger, seconds=1.2)
        rp.assessment.radius = EMUL_RADIUS
        tj._use_emul(rp, ((float(nd.odom.ds),), dict(max_map_points=400_000, max_scan_points=1_000)))
        out.append((nd, rp))
    yield out
    for _, rp in out:
        rp.close()


def _finals(runs):
    return [assess.host_pose(nd.odom.state)[2:] for nd, _ in runs]


def test_one_emulated_recording_is_replay_refine(two_runs):
    import test_assess_replay_emul as tr
    (nd, rp), = two_runs[:1]
    R_fin, T_fin = _finals(two_runs)[0]
    s = rp.refine(R_fin, T_fin, max_replays=4)
    j = joint.refine_replays([rp], [(R_fin, T_fin)], max_candidates=4)
    _same_as_single(j, s)
    for x, y in zip(j["trace"], s["trace"]):
        assert tr._same(x["results"][0], y["result"])
    assert j["states"][0].tobytes() == s["state"].tobytes() and j["time_lag"] == s["time_lag"] and j["lag0"] == s["lag0"]
    assert node.calib_result_text(**j["calibs"][0]) == node.calib_result_text(**s["calib"])


def test_two_emulated_recordings_do_not_depend_on_the_jobs(two_runs):
    import test_assess_replay_emul as tr
    rps, finals = [rp for _, rp in two_runs], _finals(two_runs)
    a = joint.refine_replays(rps, finals, max_candidates=3)
    b = joint.refine_replays(rps, finals, max_candidates=3, jobs=2)
    assert len(a["trace"]) == 3 and [r["stage"] for r in a["trace"]][:3] == ["final:0", "li-init:0", "final:1"]
    assert _rows(a) == _rows(b) and [r["mmes"] for r in a["trace"]] == [r["mmes"] for r in b["trace"]]
    for x, y in zip(a["trace"], b["trace"]):
        assert all(tr._same(p, q) for p, q in zip(x["results"], y["results"]))
    assert all(p.tobytes() == q.tobytes() for p, q in zip(a["states"], b["states"]))
    assert (a["status"], a["best"], a["start"], a["time_lag"]) == (b["status"], b["best"], b["start"], b["time_lag"])
    assert str(a["axes_rec"]) == str(b["axes_rec"])
    assert all(len(rp.workers) == 1 for rp in rps)


def _joint_runner(tmp_path, monkeypatch):
    """joint.main on the emulated library (the runner of test_refine, with replay workers); jmain(out, bags, extra, trigger_at)"""
    import test_replay_jobs_emul as tj
    import test_refine as trf
    from lidar_imu_init_b200 import capi, run
    rmain = trf._runner(tmp_path, monkeypatch)
    made = run.make_node

    def make(args, c, log):
        nd = made(args, c, log)
        cls = type(nd.odom.g)
        cls.replay_share = capi.LiInitGpu.replay_share
        cls.replay_unshare = capi.LiInitGpu.replay_unshare
        cls.twin = lambda self: cls(c.filter_size_map, max_map_points=400_000, max_scan_points=1_000)
        return nd
    monkeypatch.setattr(run, "make_node", make)
    H = tj._emul_host()
    real_replay = assess.Replay

    def replay(*a, **k):
        rp = real_replay(*a, **k)
        rp.host_lib, rp.threads = H, 1
        return rp
    monkeypatch.setattr(assess, "Replay", replay)
    shutil.copy(tmp_path / "rec.bag", tmp_path / "rec2.bag")
    bags = [str(tmp_path / "rec.bag"), str(tmp_path / "rec2.bag")]

    def jmain(out, bags, extra, trigger_at=6):
        def on_node(nd):
            def on_update(n):
                if n.updates == trigger_at:
                    n.odom.data_accum_finished = True
            nd.on_update = on_update
        argv = ["--config", str(tmp_path / "sim.yaml"), "--out", str(out), "--assess-max-points", "500000", "--assess-radius",
                str(EMUL_RADIUS), "--assess-replay-max-points", "2000000"]
        for bag in bags:
            argv += ["--bag", bag]
        return joint.main(argv + extra, on_node=on_node)
    return rmain, jmain, bags


def test_runner_writes_each_recordings_files_and_the_joint_report(tmp_path, monkeypatch, capsys):
    rmain, jmain, bags = _joint_runner(tmp_path, monkeypatch)
    assert jmain(tmp_path / "j", bags, ["--replay-jobs", "2", "--max-candidates", "2", "--devices", "0"]) == 0
    err = capsys.readouterr().err
    assert "joint refinement written to" in err and "2 candidates, 4 replays of 2 recordings" in err
    assert err.count("device memory ") == 2
    plain = tmp_path / "plain"                   # (run on bags[0]; bags[1] is a copy of it)
    assert rmain(plain, ["--quiet"]) == 0
    files = sorted(os.path.relpath(os.path.join(d, f), plain) for d, _, fs in os.walk(plain) for f in fs)
    assert {"result/Initialization_result.txt", "Log/mat_out.txt", "result/trajectory.txt"} <= set(files)
    for b in range(2):
        got = tmp_path / "j" / f"rec{b}"
        assert files == sorted(os.path.relpath(os.path.join(d, f), got) for d, _, fs in os.walk(got) for f in fs)
        for f in files:
            assert open(plain / f, "rb").read() == open(got / f, "rb").read(), (b, f)
    rep = assess.parse_joint_report(open(tmp_path / "j" / "result" / "refinement_joint.txt").read())
    assert rep["header"]["candidates"] == 2 and rep["header"]["replays"] == 4 and [r["bag"] for r in rep["recs"]] == bags
    assert len(rep["result"]) == 2 and all(x.startswith("Rotation LiDAR to IMU (degree)     = ") for x in rep["result"])


def test_runner_refusals(tmp_path, monkeypatch, capsys):
    _, jmain, bags = _joint_runner(tmp_path, monkeypatch)
    capsys.readouterr()
    cases = [([bags[0], bags[0]], [], "given twice")]
    cases += [(bags, ["--devices", d], "--devices") for d in ("a", "-1", "0,0", "", "0,,1")]
    cases += [(bags, ["--replay-jobs", j], "--replay-jobs") for j in ("0", "-2", "x", "1.5")]
    cases += [(bags, ["--max-candidates", n], "--max-candidates") for n in ("0", "-1", "x")]
    cases += [(bags, ["--assess-replay-max-points", "500"], "truncated")]
    for bg, extra, msg in cases:
        assert jmain(tmp_path / "bad", bg, ["--quiet"] + extra) == 1, extra
        e = capsys.readouterr().err
        assert msg in e, (extra, e)
    assert jmain(tmp_path / "none", bags, ["--quiet"], trigger_at=-1) == 1
    e = capsys.readouterr().err
    assert "recording 0" in e and bags[0] in e and "hand-over" in e
