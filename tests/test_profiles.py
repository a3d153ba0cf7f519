"""Profiles of a refined calibration (profiles.profile, assess.Replay.profile, joint.profile_replays, run --profile, joint --profile)
without a GPU: the candidates are one step from the centre each, scored in one call; the fit, restated in numpy, on synthetic scorers
(an exact quadratic is pinned at its minimum, a constant is flat, a minimum beyond the profile is at the edge, a NaN is unmeasured, a
point below the centre is reported); the interval's coverage over seeded noise; the t table; the reports round-trip; on the emulated
library the profile does not depend on the jobs, a row is an independent replay of its candidate, the centre is the refinement's best
row; the joint profile over one recording is Replay.profile; the runners write the profiles and leave every other file alone."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lidar_imu_init_b200 import assess, joint, profiles  # noqa: E402
from test_refine import R_STAR, T_STAR  # noqa: E402

SHIFT = 0.01743
LAG0 = -0.002965


def _u(R, T, s):
    """the profile coordinates [steps] of a candidate around (R_STAR, T_STAR, SHIFT): rotation vector of R R_STAR^T, T - T_STAR, the
    shift, each over its step"""
    from scipy.spatial.transform import Rotation
    w = np.degrees(Rotation.from_matrix(R @ R_STAR.T).as_rotvec()) / profiles.H_ROT_DEG
    t = (np.asarray(T) - T_STAR) / profiles.H_TRANS_M
    return np.concatenate([w, t, [(s - SHIFT) * 1000.0 / profiles.H_LAG_MS]])


def _scorer(f, calls=None):
    """score_many over a function of the seven coordinates"""
    def score_many(cands):
        if calls is not None:
            calls.append(list(cands))
        return [f(_u(*c)) for c in cands]
    return score_many


def _restated(u, y):
    """the fit as the module documents it, in plain numpy: (c, s, u*, se, lo, hi, verdict) of y over u [steps]"""
    n = (len(u) - 1) // 2
    X = np.stack([np.ones_like(u), u, u * u], axis=1)
    c = np.linalg.lstsq(X, y, rcond=None)[0]
    dof = len(u) - 3
    s2 = float(np.sum((y - X @ c) ** 2)) / dof
    C = s2 * np.linalg.inv(X.T @ X)
    us = -c[1] / (2 * c[2])
    g = np.array([0.0, -1.0 / (2 * c[2]), c[1] / (2 * c[2] ** 2)])
    se = math.sqrt(g @ C @ g)
    t = profiles.T975[dof]
    v = "flat" if c[2] <= t * math.sqrt(C[2, 2]) else "edge" if abs(us) > n else "pinned"
    return c, math.sqrt(s2), us, se, us - t * se, us + t * se, v


def test_t_table_matches_scipy():
    from scipy.stats import t
    assert sorted(profiles.T975) == [2 * n - 2 for n in range(profiles.MIN_STEPS, profiles.MAX_STEPS + 1)]
    for dof, q in profiles.T975.items():
        assert q == pytest.approx(float(t.ppf(0.975, dof)), rel=1e-12), dof


@pytest.mark.parametrize("steps", [2, 6, 16])
def test_candidates_are_one_step_from_the_centre_and_scored_once(steps):
    calls = []
    out = profiles.profile(_scorer(lambda u: float(u @ u), calls), R_STAR, T_STAR, SHIFT, -1.0, steps, lag0=LAG0)
    assert len(calls) == 1 and len(calls[0]) == 7 * 2 * steps == len(out["rows"])
    ks = [k for k in range(-steps, steps + 1) if k != 0]
    want = []
    for a in range(3):
        want += [(f"rot_{'xyz'[a]}", k, assess.rot_exp(k * math.radians(0.1) * np.eye(3)[a]) @ R_STAR, T_STAR, SHIFT) for k in ks]
    for a in range(3):
        want += [(f"trans_{'xyz'[a]}", k, R_STAR, T_STAR + k * 0.005 * np.eye(3)[a], SHIFT) for k in ks]
    want += [("lag", k, R_STAR, T_STAR, SHIFT + k * 0.0005) for k in ks]
    centre = (R_STAR.tobytes(), T_STAR.tobytes(), np.float64(SHIFT).tobytes())
    for (p, k, R, T, s), (Rc, Tc, sc), row in zip(want, calls[0], out["rows"]):
        got = (Rc.tobytes(), Tc.tobytes(), np.float64(sc).tobytes())
        assert got == (R.tobytes(), np.asarray(T, np.float64).tobytes(), np.float64(s).tobytes()), (p, k)
        assert got != centre and (row["param"], row["k"]) == (p, k)
        assert row["R"].tobytes() == got[0] and row["T"].tobytes() == got[1]
    # offsets in the parameters' units: degrees from the centre, absolute metres, the absolute total lag in ms
    r = {(x["param"], x["k"]): x["offset"] for x in out["rows"]}
    assert r["rot_y", 2] == pytest.approx(0.2) and r["trans_z", -1] == pytest.approx(T_STAR[2] - 0.005)
    assert r["lag", 1] == pytest.approx((LAG0 + SHIFT) * 1000.0 + 0.5)


@pytest.mark.parametrize("steps", [2, 6, 16])
def test_exact_quadratics_are_pinned_at_their_minimum(steps):
    m = np.array([0.7, -1.3, 0.0, 1.9, -0.4, 0.25, -1.75])      # minima [steps], within the profile
    a = np.array([2e-3, 1e-3, 5e-4, 3e-3, 1e-4, 7e-4, 0.03])
    out = profiles.profile(_scorer(lambda u: -4.8 + float(a @ (u - m) ** 2)), R_STAR, T_STAR, SHIFT, -4.8 + float(a @ m ** 2), steps,
                           lag0=LAG0)
    u = np.arange(-steps, steps + 1, dtype=float)
    for i, p in enumerate(profiles.PARAMS):
        f = out["fits"][p]
        assert f["verdict"] == "pinned" and f["u"] == pytest.approx(m[i], abs=1e-9), p
        ys = [r["mme"] for r in out["rows"] if r["param"] == p]
        y = np.array(ys[:steps] + [out["centre"]["mme"]] + ys[steps:])
        c, s, us, se, lo, hi, v = _restated(u, y)
        assert f["c"] == pytest.approx(tuple(c), rel=1e-9, abs=1e-12) and us == pytest.approx(f["u"], abs=1e-9) and v == f["verdict"]
        assert f["se"] < 1e-6 and f["lo"] <= f["u"] <= f["hi"] and (m[i] == 0.0 or not f["centre_inside"])
    assert not any(profiles.off_lowest(f) for f in out["fits"].values())
    assert out["fits"]["rot_x"]["u_phys"] == pytest.approx(0.07, abs=1e-9)
    assert out["fits"]["trans_x"]["u_phys"] == pytest.approx(T_STAR[0] + 1.9 * 0.005, abs=1e-9)
    assert out["fits"]["lag"]["u_phys"] == pytest.approx((LAG0 + SHIFT) * 1000.0 - 1.75 * 0.5, abs=1e-9)


def test_flat_edge_unmeasured_and_lower_points():
    """rot_x constant: flat; rot_y minimum 9 steps out of 6: edge; trans_x one NaN: unmeasured; trans_y lowest at k = -2 below the
    centre: reported; the others exact quadratics around the centre: pinned, nothing lower."""
    centre = -4.8
    fs = dict(rot_x=lambda k: centre, rot_y=lambda k: centre + 1e-3 * ((k - 9.0) ** 2 - 81.0),
              trans_x=lambda k: math.nan if k == 4 else centre + 1e-3 * k * k, trans_y=lambda k: centre + 1e-3 * ((k + 2.0) ** 2 - 4.0))

    def score_many(cands):
        order = profiles.candidates(R_STAR, T_STAR, SHIFT, 6)
        assert [c[0].tobytes() for c in cands] == [c[2].tobytes() for c in order]
        return [fs.get(p, lambda k: centre + 1e-3 * k * k)(k) for p, k, *_ in order]
    out = profiles.profile(score_many, R_STAR, T_STAR, SHIFT, centre, 6)
    v = {p: out["fits"][p]["verdict"] for p in profiles.PARAMS}
    assert v == dict(rot_x="flat", rot_y="edge", rot_z="pinned", trans_x="unmeasured", trans_y="pinned", trans_z="pinned", lag="pinned")
    fx = out["fits"]["rot_x"]
    assert fx["c"][2] == 0.0 and fx["lower_k"] == 0 and fx["lower_dmme"] == 0.0
    assert out["fits"]["rot_y"]["u"] == pytest.approx(9.0, abs=1e-9) and out["fits"]["rot_y"]["lower_k"] == 6
    assert math.isnan(out["fits"]["trans_x"]["u"]) and not out["fits"]["trans_x"]["centre_inside"]
    ty = out["fits"]["trans_y"]
    assert ty["lower_k"] == -2 and ty["lower_dmme"] == pytest.approx(-4e-3, abs=1e-12) and not ty["centre_inside"]
    assert all(out["fits"][p]["lower_k"] == 0 and abs(out["fits"][p]["u"]) < 1e-9 for p in ("rot_z", "trans_z", "lag"))
    for p in ("rot_x", "rot_y", "trans_y"):
        ys = [r["mme"] for r in out["rows"] if r["param"] == p]
        c, s, us, se, lo, hi, vv = _restated(np.arange(-6, 7, dtype=float), np.array(ys[:6] + [centre] + ys[6:]))
        assert vv == v[p], p


def test_asymmetric_v_is_flagged_off_its_lowest_point():
    """A V-shaped profile with its minimum at the centre, twice as steep below as above, plus a little seeded noise: the parabola's
    vertex moves to the shallow side, a step or more from the lowest point (the centre), and its `pinned` interval excludes the centre.
    off_lowest says so, and so does the summary line; a parabola through the same minimum is not flagged."""
    from lidar_imu_init_b200 import run
    rng = np.random.default_rng(1)
    u = np.arange(-6, 7, dtype=float)
    y = -4.8 + np.where(u < 0, -0.012 * u, 0.006 * u) + rng.normal(0.0, 3e-4, u.size)
    y[6] = -4.8
    f = profiles.fit(list(y[:6]) + list(y[7:]), y[6], 6)
    assert f["verdict"] == "pinned" and f["lower_k"] == 0 and not f["centre_inside"] and f["u"] >= 1.0
    assert profiles.off_lowest(f)
    g = profiles.fit(list(-4.8 + 1e-3 * u[:6] ** 2) + list(-4.8 + 1e-3 * u[7:] ** 2), -4.8, 6)
    assert g["verdict"] == "pinned" and not profiles.off_lowest(g)

    def score_many(cands):
        return [-4.8 + (float(y[k + 6]) + 4.8 if p == "lag" else 1e-3 * k * k) for p, k, *_ in profiles.candidates(R_STAR, T_STAR, SHIFT)]
    prof = dict(profiles.profile(score_many, R_STAR, T_STAR, SHIFT, -4.8, lag0=LAG0), replays=84, wall_s=1.0)
    line = run.profile_summary("profile.txt", prof, 2)
    assert line.count("off the profile's lowest point") == 1 and "lag pinned [" in line and "k +0: the parabola misfits" in line


def test_noisy_fit_restated_and_interval_coverage():
    """A quadratic of curvature 0.01 per step^2 with its minimum uniform in [-2, 2] steps, plus i.i.d. normal noise of 0.01, at n = 6,
    over 2000 seeded trials. Each fit agrees with the numpy restatement. The fraction of intervals that contain the true minimum is
    within [0.93, 0.97]: at a true coverage of 0.95 its standard deviation over 2000 trials is sqrt(0.95 * 0.05 / 2000) = 0.0049, so the
    band is about four standard deviations each side, wide enough for the delta method's small bias at this curvature to noise ratio
    and narrow enough that a t quantile off by one degree of freedom or a z quantile in its place would fail it."""
    rng = np.random.default_rng(20261018)
    n, trials, hits = 6, 2000, 0
    u = np.arange(-n, n + 1, dtype=float)
    for i in range(trials):
        m = rng.uniform(-2.0, 2.0)
        y = -4.8 + 0.01 * (u - m) ** 2 + rng.normal(0.0, 0.01, u.size)
        f = profiles.fit(list(y[:n]) + list(y[n + 1:]), y[n], n)
        if i < 200:
            c, s, us, se, lo, hi, v = _restated(u, y)
            assert f["c"] == pytest.approx(tuple(c), rel=1e-9, abs=1e-12) and f["s"] == pytest.approx(s, rel=1e-9)
            assert (f["u"], f["se"], f["lo"], f["hi"]) == pytest.approx((us, se, lo, hi), rel=1e-9, abs=1e-12) and f["verdict"] == v
        hits += f["lo"] <= m <= f["hi"]
    assert 0.93 <= hits / trials <= 0.97, hits / trials


@pytest.mark.parametrize("bad", [1, 17, 2.5, True])
def test_bad_steps_are_refused(bad):
    with pytest.raises(ValueError, match="steps"):
        profiles.profile(_scorer(lambda u: 0.0), R_STAR, T_STAR, SHIFT, 0.0, bad)


# ---- the reports -----------------------------------------------------------------------------------------------------------------------
def _fake(joint_B=None, steps=3):
    """a profile dict with results and seconds per row: NaN scores on trans_x (unmeasured), a flat rot_x; joint_B recordings"""
    rng = np.random.default_rng(7)

    def f(u):
        return math.nan if u[3] > 1.5 else -4.8 + 1e-3 * float(np.sum(u[1:] ** 2)) + rng.normal(0, 1e-5)
    out = profiles.profile(_scorer(f), R_STAR, T_STAR, SHIFT, -4.8, steps, lag0=LAG0)
    B = joint_B or 1
    for row in out["rows"]:
        res = [dict(valid=int(rng.integers(0, 10**6)), sparse=0, degenerate=0, mme=row["mme"] + 1e-4 * b, mpv=1e-4) for b in range(B)]
        secs = [float(rng.uniform(0.5, 3.0)) for _ in range(B)]
        if joint_B:
            row.update(results=res, seconds=secs, mmes=[r["mme"] for r in res])
        else:
            row.update(result=res[0], seconds=secs[0])
    out.update(wall_s=81.25, jobs=4, status="budget", replays=len(out["rows"]) * B)
    if joint_B:
        out["centre"]["mmes"] = [-4.8 + 1e-4 * b for b in range(B)]
        out["recs"] = [profiles.fit_all([r["mmes"][b] for r in out["rows"]], out["centre"]["mmes"][b], T_STAR, out["centre"]["lag_s"], steps)
                       for b in range(B)]
    return out


def _same_fit(got, f, p):
    assert got["verdict"] == f["verdict"] and got["unit"] == profiles.UNITS[p.split("_")[0]]
    want = (*f["c"], f["s"], f["u"], f["se"], f["u_phys"], f["lo_phys"], f["hi_phys"])
    for k, w in zip(("c0", "c1", "c2", "s", "u_star", "se", "min", "lo", "hi"), want):
        assert (math.isnan(got[k]) and math.isnan(w)) or got[k] == pytest.approx(w, rel=1e-9, abs=1e-15), (p, k)
    assert (got["centre_inside"], got["lower_k"]) == (f["centre_inside"], f["lower_k"])
    assert got["lower_dmme"] == pytest.approx(f["lower_dmme"], rel=1e-9, abs=1e-15)


def test_profile_report_round_trip():
    prof = _fake()
    text = assess.profile_report_text(prof)
    rep = assess.parse_profile_report(text)
    assert rep["header"] == dict(replays=42, jobs=4, wall_s=81.25, status="budget", steps=3, h_rot_deg=0.1, h_trans_m=0.005, h_lag_ms=0.5)
    c = rep["centre"]
    assert c["t_m"] == pytest.approx(tuple(T_STAR), abs=1e-6) and c["mme"] == -4.8
    assert c["lag_ms"] == pytest.approx((LAG0 + SHIFT) * 1000.0, abs=1e-6) and c["shift_ms"] == pytest.approx(SHIFT * 1000.0, abs=1e-6)
    assert len(rep["rows"]) == 42
    for got, row in zip(rep["rows"], prof["rows"]):
        assert (got["param"], got["k"], got["valid"]) == (row["param"], row["k"], row["result"]["valid"])
        assert got["offset"] == pytest.approx(row["offset"], abs=1e-9) and got["seconds"] == pytest.approx(row["seconds"], abs=1e-3)
        assert (math.isnan(got["mme"]) and math.isnan(row["mme"])) or got["mme"] == pytest.approx(row["mme"], abs=1e-9)
    assert any(math.isnan(r["mme"]) for r in rep["rows"])
    assert list(rep["fits"]) == list(profiles.PARAMS)
    assert rep["fits"]["trans_x"]["verdict"] == "unmeasured"
    for p, f in prof["fits"].items():
        _same_fit(rep["fits"][p], f, p)
    assert assess.parse_profile_report(assess.NOTHING) == {"nothing": True}


@pytest.mark.parametrize("B", [1, 2])
def test_joint_profile_report_round_trip(B):
    prof = _fake(B)
    rep = assess.parse_profile_report(assess.profile_report_text(prof))
    h = rep["header"]
    assert (h["recordings"], h["candidates"], h["replays"], h["jobs"]) == (B, 42, 42 * B, 4)
    assert rep["centre"]["mmes"] == pytest.approx(prof["centre"]["mmes"], abs=1e-9)
    for got, row in zip(rep["rows"], prof["rows"]):
        assert (got["param"], got["k"]) == (row["param"], row["k"]) and got["valid"] == [r["valid"] for r in row["results"]]
        assert str(np.round(got["mmes"], 9)) == str(np.round(row["mmes"], 9)) and got["seconds"] == pytest.approx(row["seconds"], abs=1e-3)
    assert list(rep["fits"]) == ["joint"] + list(range(B))
    for who, fits in [("joint", prof["fits"])] + list(enumerate(prof["recs"])):
        assert list(rep["fits"][who]) == list(profiles.PARAMS)
        for p, f in fits.items():
            _same_fit(rep["fits"][who][p], f, p)


# ---- on the emulated library -----------------------------------------------------------------------------------------------------------
EMUL_RADIUS = 1.5   # [m] (as in test_refine: the short runs store a few thousand points)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    import test_assess_replay_emul as tr
    import test_replay_jobs_emul as tj
    nd, rp, _, _ = tr._emul_run(tmp_path_factory.mktemp("run"), trigger_at=6, seconds=1.2)
    rp.assessment.radius = EMUL_RADIUS
    tj._use_emul(rp, ((float(nd.odom.ds),), dict(max_map_points=400_000, max_scan_points=1_000)))
    _, _, R_fin, T_fin = assess.host_pose(nd.odom.state)
    ref = rp.refine(R_fin, T_fin, max_replays=3)
    prof = rp.profile(ref, 1, steps=2)
    yield rp, ref, prof
    rp.close()


def _rows(prof):
    return [(r["param"], r["k"], r["R"].tobytes(), r["T"].tobytes(), np.float64(r["shift_s"]).tobytes(), np.float64(r["mme"]).tobytes())
            for r in prof["rows"]]


def test_emulated_profile_does_not_depend_on_the_jobs(emul):
    import test_assess_replay_emul as tr
    rp, ref, a = emul
    b = rp.profile(ref, 3, steps=2)
    assert len(a["rows"]) == a["replays"] == 28 and len(rp.workers) == 2
    assert all(r["result"]["valid"] > 0 for r in a["rows"])
    assert _rows(a) == _rows(b) and all(tr._same(x["result"], y["result"]) for x, y in zip(a["rows"], b["rows"]))
    assert str(a["fits"]) == str(b["fits"])


def test_emulated_rows_and_centre_are_replays_of_their_candidates(emul):
    import test_assess_replay_emul as tr
    rp, ref, prof = emul
    row = next(r for r in prof["rows"] if r["param"] == "rot_y" and r["k"] == -1)
    again = rp.run(row["R"], row["T"], row["shift_s"], frozen=True)["result"]
    assert tr._same(again, row["result"]) and np.float64(again["mme"]).tobytes() == np.float64(row["mme"]).tobytes()
    centre = rp.run(ref["R"], ref["T"], ref["shift_s"], frozen=True)["result"]["mme"]
    assert np.float64(centre).tobytes() == np.float64(ref["mme"]).tobytes() == np.float64(prof["centre"]["mme"]).tobytes()
    assert prof["centre"]["lag_s"] == rp.lag + ref["shift_s"] and prof["status"] == ref["status"]


class _FakeReplay(assess.Replay):
    """a Replay whose replays are a synthetic function of the candidate: its lag, contexts and results without a device"""
    lag = -0.002965

    def __init__(self, f):
        self.f, self.workers, self.threads = f, [], 1

    def pool(self, jobs):
        return [None] * jobs

    def run(self, R_LI=None, T_LI=None, lag_shift=0.0, frozen=True):
        m = self.f(_u(R_LI, T_LI, lag_shift))
        return dict(result=dict(valid=1000, sparse=0, degenerate=0, mme=m, mpv=1e-4), states=[], seconds=0.5)

    def run_native(self, *c, g=None):
        return self.run(*c)


@pytest.mark.parametrize("jobs", [1, 3])
def test_joint_profile_of_one_recording_is_replay_profile(jobs):
    """joint.profile_replays over one recording: the rows, their MMEs and the fits of Replay.profile bit for bit, and the recording's
    own fits the joint ones"""
    rng = np.random.default_rng(4)
    a = rng.uniform(1e-4, 1e-3, 7)

    def f(u):
        return -4.8 + float(a @ (u - 0.3) ** 2) + 1e-5 * math.sin(float(np.sum(u * [1.1, 2.3, 3.7, 5.3, 7.1, 11.3, 13.7])))
    rp = _FakeReplay(f)
    ref = dict(R=R_STAR, T=T_STAR, shift_s=SHIFT, mme=f(np.zeros(7)), status="converged")
    single = rp.profile(ref, jobs)
    jref = dict(ref, lag0=joint.mean_lag([rp.lag]), offsets=[0.0], mmes=[ref["mme"]])
    j = joint.profile_replays([rp], jref, jobs)
    assert _rows(j) == _rows(single) and len(j["rows"]) == 84 == j["replays"] == single["replays"]
    assert [np.float64(r["mmes"][0]).tobytes() for r in j["rows"]] == [np.float64(r["mme"]).tobytes() for r in single["rows"]]
    assert str(j["fits"]) == str(single["fits"]) == str(j["recs"][0])
    assert j["centre"]["lag_s"] == single["centre"]["lag_s"] == rp.lag + SHIFT
    assert {p: x["verdict"] for p, x in single["fits"].items()} == dict.fromkeys(profiles.PARAMS, "pinned")


# ---- the runners -----------------------------------------------------------------------------------------------------------------------
def _cheap_replays(monkeypatch):
    """Each Replay's first replay real, every later one that replay with a synthetic MME of how far its candidate lies from the first:
    the runners' wiring without 14n emulated replays of about 15 s each (the replays themselves are checked above)."""
    def stub(real):
        def replay(self, R_LI=None, T_LI=None, lag_shift=0.0, frozen=True, **kw):
            if getattr(self, "_first", None) is None:
                self._first = (real(self, R_LI, T_LI, lag_shift, frozen, **kw), np.array(R_LI), np.array(T_LI), lag_shift)
                return self._first[0]
            r, R0, T0, s0 = self._first
            d = float(np.sum((R_LI - R0) ** 2)) + float(np.sum((T_LI - T0) ** 2)) + (lag_shift - s0) ** 2
            return dict(r, result=dict(r["result"], mme=r["result"]["mme"] + 10.0 * d))
        return replay
    monkeypatch.setattr(assess.Replay, "run", stub(assess.Replay.run))
    monkeypatch.setattr(assess.Replay, "run_native", stub(assess.Replay.run_native))


def _files(d):
    return sorted(os.path.relpath(os.path.join(r, f), d) for r, _, fs in os.walk(d) for f in fs)


def test_runner_profile(tmp_path, monkeypatch, capsys):
    """run --refine --profile writes a profile.txt that parses, centred on the refinement's best row, and every file a plain run writes
    byte-identical; --profile without --refine exits 1 with a message; a run that never hands over writes NOTHING to refinement.txt
    and profile.txt."""
    import test_refine as trf
    main = trf._runner(tmp_path, monkeypatch)
    _cheap_replays(monkeypatch)
    assert main(tmp_path / "plain", ["--quiet"]) == 0
    assert main(tmp_path / "prof", ["--refine", "--refine-max-replays", "2", "--profile"]) == 0
    err = capsys.readouterr().err
    assert "profile written to" in err and "84 replays" in err and "lag " in err
    rep = assess.parse_profile_report(open(tmp_path / "prof" / "result" / "profile.txt").read())
    ref = assess.parse_refine_report(open(tmp_path / "prof" / "result" / "refinement.txt").read())
    assert rep["header"]["replays"] == len(rep["rows"]) == 84 and rep["header"]["steps"] == 6 and rep["header"]["status"] == "budget"
    assert list(rep["fits"]) == list(profiles.PARAMS) and all(r["valid"] > 0 for r in rep["rows"])
    assert rep["centre"]["mme"] == pytest.approx(min(r["mme"] for r in ref["rows"]), abs=1e-9)
    assert rep["centre"]["lag_ms"] == pytest.approx(ref["header"]["lag_ms"], abs=1e-6)
    plain = tmp_path / "plain"
    files = _files(plain)
    assert "result/Initialization_result.txt" in files and set(_files(tmp_path / "prof")) == set(files) | {"result/refinement.txt",
                                                                                                         "result/profile.txt"}
    for f in files:
        assert open(plain / f, "rb").read() == open(tmp_path / "prof" / f, "rb").read(), f
    assert main(tmp_path / "alone", ["--quiet", "--profile"]) == 1
    assert "--profile" in capsys.readouterr().err and not os.path.exists(tmp_path / "alone")
    assert main(tmp_path / "none", ["--quiet", "--refine", "--profile"], trigger_at=-1) == 0
    for f in ("refinement.txt", "profile.txt"):
        assert open(tmp_path / "none" / "result" / f).read() == assess.NOTHING, f


def test_joint_runner_profile(tmp_path, monkeypatch, capsys):
    """joint --profile writes profile_joint.txt with a fit block for the joint score and one per recording."""
    import test_joint as tj
    _cheap_replays(monkeypatch)
    _, jmain, bags = tj._joint_runner(tmp_path, monkeypatch)
    assert jmain(tmp_path / "j", bags, ["--max-candidates", "1", "--profile"]) == 0
    assert "profile written to" in capsys.readouterr().err
    rep = assess.parse_profile_report(open(tmp_path / "j" / "result" / "profile_joint.txt").read())
    h = rep["header"]
    assert (h["recordings"], h["candidates"], h["replays"]) == (2, 84, 168) and len(rep["rows"]) == 84
    assert list(rep["fits"]) == ["joint", 0, 1] and all(list(f) == list(profiles.PARAMS) for f in rep["fits"].values())
    assert all(f["verdict"] == "pinned" for fits in rep["fits"].values() for f in fits.values())
    for r in rep["rows"]:
        m = r["mmes"]
        assert r["mme"] == pytest.approx((m[0] + m[1]) / 2.0, abs=2e-9)
