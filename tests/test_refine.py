"""The refinement by LIO replay (refine.search, assess.Replay.refine, run --refine) without a GPU: the search on synthetic bowls with a
known minimum (its tolerances, the lag bracket inside and beyond the steps and at the cap, a flat axis, the cache, the budget, its
determinism); the report round-trips; on the emulated library every trace row is the score of an independent replay of its candidate;
the runner's --refine."""
import math
import os
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lidar_imu_init_b200 import assess, node, refine  # noqa: E402

R_STAR = assess.rot_exp([0.02, -0.01, 1.2])
T_STAR = np.array([0.05, -0.03, 0.10])
R_START = assess.rot_exp(np.radians([0.7, -0.4, 0.3])) @ R_STAR
T_START = T_STAR + [0.02, -0.015, 0.01]


def _angle_deg(R, R_ref) -> float:
    return float(np.degrees(np.linalg.norm(Rotation.from_matrix(R @ R_ref.T).as_rotvec())))


class Bowl:
    """A smooth bowl with its minimum -5 at (R_STAR, T_STAR, s_star): 1 per 0.5 deg, per 2 cm and per 5 ms from it. `flat`: a translation
    axis the score does not depend on. Counts its calls."""

    def __init__(self, s_star_ms, flat=None):
        self.s_star, self.flat, self.calls = s_star_ms, flat, 0

    def __call__(self, R, T, shift_s):
        self.calls += 1
        w = np.degrees(Rotation.from_matrix(R @ R_STAR.T).as_rotvec()) / 0.5
        t = (np.asarray(T) - T_STAR) / 0.02
        if self.flat is not None:
            t[self.flat] = 0.0
        s = (shift_s * 1000.0 - self.s_star) / 5.0
        return -5.0 + float(w @ w + t @ t + s * s)


@pytest.mark.parametrize("s_star", [3.0, -27.0, 60.0])   # inside the first steps, beyond +-20 ms on the negative side, beyond the cap
def test_search_finds_the_minimum_of_a_bowl(s_star):
    f = Bowl(s_star)
    r = refine.search(f, R_START, T_START, max_replays=1000, R_init=assess.rot_exp([0.0, 0.0, 0.05]) @ R_STAR, T_init=T_STAR + [0.1, 0, 0])
    assert r["status"] == "converged" and r["start"] == "final"
    assert [row["stage"] for row in r["trace"][:2]] == ["final", "li-init"]
    assert _angle_deg(r["R"], R_STAR) <= refine.DTHETA_MIN_DEG
    assert np.abs(r["T"] - T_STAR).max() <= refine.DT_MIN_M
    if s_star > refine.LAG_CAP_MS:
        assert r["at_edge"] and r["shift_ms"] == refine.LAG_CAP_MS
    else:
        assert not r["at_edge"] and abs(r["shift_ms"] - s_star) <= refine.LAG_TOL_MS
    assert r["shift_s"] == r["shift_ms"] / 1000.0
    # the end condition: every neighbour at the final step scores at or above the refined candidate
    assert r["steps"][0] <= refine.DTHETA_MIN_DEG and r["steps"][1] <= refine.DT_MIN_M
    for axis, (step, dp, dm) in r["axes"].items():
        assert step == r["steps"][0 if axis.startswith("rot") else 1] and dp >= 0 and dm >= 0, axis
    # the cache: one call per row, no candidate twice; the result is the best row
    assert f.calls == len(r["trace"])
    assert len({refine.key(x["R"], x["T"], x["shift_ms"] / 1000.0) for x in r["trace"]}) == len(r["trace"])
    best = r["trace"][r["best"]]
    assert best["mme"] == min(x["mme"] for x in r["trace"]) == r["mme"]
    assert best["R"].tobytes() == r["R"].tobytes() and best["T"].tobytes() == r["T"].tobytes() and best["shift_ms"] == r["shift_ms"]


def test_search_starts_from_the_lower_candidate():
    r = refine.search(Bowl(0.0), R_START, T_START, max_replays=1000, R_init=R_STAR, T_init=T_STAR)
    assert r["start"] == "li-init" and r["trace"][1]["stage"] == "li-init" and r["trace"][1]["mme"] < r["trace"][0]["mme"]
    assert _angle_deg(r["R"], R_STAR) <= refine.DTHETA_MIN_DEG and np.abs(r["T"] - T_STAR).max() <= refine.DT_MIN_M
    # no LI-Init candidate: the final one is the start
    assert refine.search(Bowl(0.0), R_START, T_START, max_replays=5)["start"] == "final"


def test_flat_axis_keeps_its_value_and_is_reported():
    f = Bowl(1.0, flat=2)
    r = refine.search(f, R_START, T_START, max_replays=1000)
    assert r["status"] == "converged"
    assert r["T"][2] == T_START[2]                                     # the start's value, bit for bit
    step, dp, dm = r["axes"]["trans_z"]
    assert dp == 0.0 and dm == 0.0 and refine.axis_verdict(dp, dm) == "flat"
    assert all(refine.axis_verdict(dp, dm) == "constrained" for a, (_, dp, dm) in r["axes"].items() if a != "trans_z")
    assert np.abs(r["T"][:2] - T_STAR[:2]).max() <= refine.DT_MIN_M


@pytest.mark.parametrize("budget", [1, 2, 7, 40])
def test_budget_is_never_exceeded(budget):
    f = Bowl(12.0)
    r = refine.search(f, R_START, T_START, max_replays=budget, R_init=R_STAR, T_init=T_STAR + [0.05, 0, 0])
    assert f.calls == len(r["trace"]) == budget and r["status"] == "budget"
    best = r["trace"][r["best"]]
    assert r["mme"] == best["mme"] == min(x["mme"] for x in r["trace"])
    if budget < 12:   # the compass has not scored around the result: its differences are unknown
        assert all(refine.axis_verdict(dp, dm) == "unmeasured" for _, dp, dm in r["axes"].values())
    # enough budget: the same search converges
    assert refine.search(Bowl(12.0), R_START, T_START, max_replays=1000)["status"] == "converged"


@pytest.mark.parametrize("bad", [0, -3, 2.5, True])
def test_bad_budget_is_refused(bad):
    with pytest.raises(ValueError, match="max_replays"):
        refine.search(Bowl(0.0), R_START, T_START, max_replays=bad)


def test_search_is_deterministic():
    a = refine.search(Bowl(-8.0), R_START, T_START, max_replays=1000, R_init=R_STAR, T_init=T_START)
    b = refine.search(Bowl(-8.0), R_START, T_START, max_replays=1000, R_init=R_STAR, T_init=T_START)
    assert len(a["trace"]) == len(b["trace"])
    for x, y in zip(a["trace"], b["trace"]):
        assert (x["stage"], x["R"].tobytes(), x["T"].tobytes(), x["shift_ms"], x["mme"]) == (y["stage"], y["R"].tobytes(), y["T"].tobytes(),
                                                                                              y["shift_ms"], y["mme"])


def test_nan_scores_are_never_best():
    """A candidate with no valid query (MME NaN) never becomes the result."""
    f = Bowl(0.0)

    def score(R, T, s):
        return math.nan if s > 0 else f(R, T, s)
    r = refine.search(score, R_START, T_START, max_replays=1000)
    assert r["mme"] == r["mme"] and r["shift_ms"] <= 0.0


# ---- the report ------------------------------------------------------------------------------------------------------------------------
def _fake_ref(rng, n=9):
    r = refine.search(Bowl(4.0), R_START, T_START, max_replays=n, R_init=R_STAR, T_init=T_STAR)
    for row in r["trace"]:
        row["result"] = dict(valid=int(rng.integers(1, 10**6)), sparse=int(rng.integers(0, 1000)), degenerate=int(rng.integers(0, 100)),
                             mme=row["mme"], mpv=float(rng.uniform(1e-6, 1e-3)))
        row["seconds"] = float(rng.uniform(0.5, 3.0))
    state = np.zeros(612)
    state[12:21] = r["R"].reshape(9)
    state[21:24] = r["T"]
    state[27:36] = rng.normal(size=9)
    r.update(wall_s=123.456, lag0=-0.00297, time_lag=-0.00297 + r["shift_s"], state=state,
             calib=node.state_calib_values(state, -0.00297 + r["shift_s"]))
    return r


def test_refine_report_round_trip():
    rng = np.random.default_rng(5)
    ref = _fake_ref(rng)
    text = assess.refine_report_text(dict(frames=2498, skipped=0, points=9_700_000), ref, 0.3, 10)
    rep = assess.parse_refine_report(text)
    assert rep["header"] == dict(subframes=2498, skipped=0, start="li-init", replays=9, wall_s=123.456, status="budget", at_edge=0, lag0_ms=-2.97,
                                 shift_ms=pytest.approx(ref["shift_ms"], abs=1e-6), lag_ms=pytest.approx(ref["time_lag"] * 1000, abs=1e-6),
                                 radius=0.3, n_min=10)
    assert len(rep["rows"]) == len(ref["trace"]) == 9
    for got, row in zip(rep["rows"], ref["trace"]):
        e = np.degrees(node.rot_to_euler(row["R"]))
        assert got["stage"] == row["stage"] and got["shift_ms"] == pytest.approx(row["shift_ms"], abs=1e-6)
        assert (got["roll_deg"], got["pitch_deg"], got["yaw_deg"]) == pytest.approx(tuple(e), abs=1e-6)
        assert (got["t_x"], got["t_y"], got["t_z"]) == pytest.approx(tuple(row["T"]), abs=1e-6)
        res = row["result"]
        assert (got["valid"], got["sparse"], got["degenerate"]) == (res["valid"], res["sparse"], res["degenerate"])
        assert got["mme"] == pytest.approx(res["mme"], abs=1e-9) and got["mpv"] == pytest.approx(res["mpv"], rel=1e-9)
        assert got["seconds"] == pytest.approx(row["seconds"], abs=1e-3)
    assert list(rep["axes"]) == ["rot_x", "rot_y", "rot_z", "trans_x", "trans_y", "trans_z"]
    for axis, (step, dp, dm) in ref["axes"].items():
        v, s, p, m = rep["axes"][axis]
        assert v == refine.axis_verdict(dp, dm) and s == pytest.approx(step, abs=1e-6)
        assert (p == pytest.approx(dp, abs=1e-9) or (p != p and dp != dp)) and (m == pytest.approx(dm, abs=1e-9) or (m != m and dm != dm))
    assert rep["result"] == node.calib_result_text(**ref["calib"])
    assert text.endswith(assess.REFINED + "\n" + node.calib_result_text(**ref["calib"]))
    assert assess.parse_refine_report(assess.NOTHING) == {"nothing": True}


# ---- on the emulated library -----------------------------------------------------------------------------------------------------------
EMUL_RADIUS = 1.5   # [m] the short emulated runs store a few thousand points: at 0.3 m no query has 10 neighbours


def test_refine_on_the_emulated_replay(tmp_path):
    """Replay.refine over a short emulated run: every trace row's MME is bit-equal to an independent frozen replay of its candidate, the
    refined MME is at or below the start's, and the refined extrinsic, lag and state are the best row's."""
    import test_assess_replay_emul as tr
    nd, rp, _, _ = tr._emul_run(tmp_path, trigger_at=6, seconds=1.2)
    rp.assessment.radius = EMUL_RADIUS
    _, _, R_fin, T_fin = assess.host_pose(nd.odom.state)
    ref = rp.refine(R_fin, T_fin, max_replays=3)
    assert len(ref["trace"]) == 3 and ref["status"] == "budget"
    assert all(r["result"]["valid"] > 0 for r in ref["trace"])
    assert [r["stage"] for r in ref["trace"][:2]] == ["final", "li-init"]
    for row in ref["trace"]:
        again = rp.run(row["R"], row["T"], row["shift_ms"] / 1000.0, frozen=True)["result"]
        assert tr._same(again, row["result"]) and np.float64(again["mme"]).tobytes() == np.float64(row["mme"]).tobytes(), row["stage"]
    start = next(r for r in ref["trace"] if r["stage"] == ref["start"])
    assert ref["mme"] <= start["mme"]
    best = ref["trace"][ref["best"]]
    assert ref["R"].tobytes() == best["R"].tobytes() and ref["T"].tobytes() == best["T"].tobytes()
    assert ref["lag0"] == nd.odom.imu_buffer.timediff + float(rp.res["time_lag_1"]) + float(rp.res["time_lag_2"])
    assert ref["time_lag"] == ref["lag0"] + best["shift_ms"] / 1000.0
    # the refined result's extrinsic is the candidate's, bit for bit (the replay was frozen); its biases and gravity the replay's
    assert ref["state"][12:21].tobytes() == best["R"].reshape(9).tobytes() and ref["state"][21:24].tobytes() == best["T"].tobytes()
    assert ref["calib"]["time_lag"] == ref["time_lag"] and ref["calib"]["gravity"].tobytes() == ref["state"][33:36].tobytes()


# ---- the runner ------------------------------------------------------------------------------------------------------------------------
def _runner(tmp_path, monkeypatch):
    """run.main on the emulated library, LI-Init's result forced to the simulated truth; handover(argv, trigger_at) runs it."""
    import lio_case
    import test_assess_replay_emul as tr
    import test_bag_node as tb
    from lidar_imu_init_b200 import _build, config, run
    from lidar_imu_init_b200.odometry import LidarOdometry
    _build.build_gpu()
    _build.build_host()
    _build.build_calib()
    cfg = tb.sim_config(tmp_path)
    G = tr._frames_cls()
    ev, path = tb.livox_events(1.2, 400)
    bag = str(tmp_path / "rec.bag")
    tb.write_event_bag(bag, ev)
    res = lio_case.true_result(path.S)

    class EmulOdometry(LidarOdometry):
        def _scan_update_resident(self, state):
            return tr.scan_update(self.g, state, self.max_iteration, self.imu_en, self.frozen)

        def initialize(self, timediff_imu_wrt_lidar=0.0):
            return dict(res)

    def make(args, c, log):
        o = EmulOdometry(G(cfg.filter_size_map, max_map_points=400_000, max_scan_points=1_000), **config.odometry_kwargs(cfg))
        return node.Node(c, o, args.out, log)
    monkeypatch.setattr(run, "make_node", make)

    def main(out, extra, trigger_at=6):
        def on_node(nd):
            def on_update(n):
                if n.updates == trigger_at:
                    n.odom.data_accum_finished = True
            nd.on_update = on_update
        return run.main(["--config", str(tmp_path / "sim.yaml"), "--bag", bag, "--out", str(out), "--assess-max-points", "500000",
                         "--assess-radius", str(EMUL_RADIUS), "--assess-replay-max-points", "2000000"] + extra, on_node=on_node)
    return main


def test_runner_refine(tmp_path, monkeypatch, capsys):
    """run --refine writes a refinement.txt that parses, and every other file byte-identical to a run without it; a run that never
    hands over writes NOTHING; a bad --refine-max-replays exits 1 with a message."""
    main = _runner(tmp_path, monkeypatch)
    assert main(tmp_path / "plain", ["--quiet"]) == 0
    assert main(tmp_path / "ref", ["--refine", "--refine-max-replays", "3"]) == 0
    err = capsys.readouterr().err
    assert "refinement written to" in err and "replays" in err and "MME" in err
    rep = assess.parse_refine_report(open(tmp_path / "ref" / "result" / "refinement.txt").read())
    assert rep["header"]["replays"] == len(rep["rows"]) == 3 and rep["header"]["status"] == "budget"
    assert rep["result"].startswith("Rotation LiDAR to IMU (degree)     = ")
    best = min(rep["rows"], key=lambda r: r["mme"])
    assert rep["header"]["shift_ms"] == best["shift_ms"]
    plain = tmp_path / "plain"
    files = sorted(os.path.relpath(os.path.join(d, f), plain) for d, _, fs in os.walk(plain) for f in fs)
    assert "result/Initialization_result.txt" in files
    assert open(plain / "result" / "Initialization_result.txt").read().startswith("Initialization result:")
    for f in files:
        assert open(plain / f, "rb").read() == open(tmp_path / "ref" / f, "rb").read(), f
    # no hand-over: NOTHING
    assert main(tmp_path / "none", ["--quiet", "--refine"], trigger_at=-1) == 0
    assert assess.parse_refine_report(open(tmp_path / "none" / "result" / "refinement.txt").read()) == {"nothing": True}
    for bad in ("0", "-2", "abc", "1.5"):
        capsys.readouterr()
        assert main(tmp_path / "bad", ["--quiet", "--refine", "--refine-max-replays", bad]) == 1
        assert "--refine-max-replays" in capsys.readouterr().err


def test_runner_refine_refuses_a_truncated_store(tmp_path, monkeypatch, capsys):
    """A replay store that overflowed: run --refine exits 1 and says so."""
    main = _runner(tmp_path, monkeypatch)
    assert main(tmp_path / "o", ["--quiet", "--refine", "--refine-max-replays", "3", "--assess-replay-max-points", "500"]) == 1
    assert "truncated" in capsys.readouterr().err
