"""Concurrent replays without a GPU (liinit_replay_share / _unshare, liinit_replay_run, assess.Replay.run_many, refine.search's batches,
run --replay-jobs): a worker that shares a lead's replay store and map snapshot restores and stages what the lead does; every refusal
of the sharing rule; the native loop of a replay is bit-equal to Replay.run; the batched search has the one-at-a-time search's trace at
every budget; the runner's files do not depend on the number of replay jobs. The CPU build of the kernels keeps its SIMT block state in
globals, so the batches here run on one thread (Replay.threads = 1), driving the contexts in turn."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from lidar_imu_init_b200 import assess, capi, host, refine  # noqa: E402

emul = pytest.importorskip("liinit_emul")
import test_assess_replay_emul as tr  # noqa: E402
import test_refine as trf  # noqa: E402

INVALID = -1
EMUL_RADIUS = 1.5   # [m] (as in test_refine: the short runs store a few thousand points)


def _sharing_cls(cfg_args):
    """the emulated context class with the sharing calls and a twin of the given configuration"""
    G = tr._frames_cls()
    G.replay_share = capi.LiInitGpu.replay_share
    G.replay_unshare = capi.LiInitGpu.replay_unshare
    G.twin = lambda self: type(self)(*cfg_args[0], **cfg_args[1])
    return G


def _emul_host():
    H = emul.host_lib()
    host.set_replay_run_argtypes(H)
    return H


def _use_emul(rp, cfg_args):
    """a Replay of an emulated run driven through the emulated library: its native loop, its workers, one thread"""
    cls = type(rp.g)
    cls.replay_share = capi.LiInitGpu.replay_share
    cls.replay_unshare = capi.LiInitGpu.replay_unshare
    cls.twin = lambda self: cls(*cfg_args[0], **cfg_args[1])
    rp.host_lib = _emul_host()
    rp.threads = 1


# ---- sharing ---------------------------------------------------------------------------------------------------------------------------
def _lead(G, rng):
    g = G(0.15, max_map_points=60_000, max_scan_points=5_000)
    g.map_build(tr._cloud(rng, 8000))
    g.map_add_points(tr._cloud(rng, 3000, (0.5, 0.2, 0.0)), True)
    subs = tr._subframes(g, rng)
    g.frame_stage(subs[0]["handle"])
    g.raw_n = subs[0]["n"]
    g.replay_reserve(sum(e["n"] for e in subs), 64)
    for e in subs:
        g.replay_append(e["handle"], e["t_beg"], e["end_ms"])
    g.map_snapshot()
    return g, subs


def test_worker_restores_and_stages_what_the_lead_does():
    """A worker's restore gives the lead's map download, stats, live count, 5-NN results and staged cloud bit for bit; its
    replay_stage(j) stages the lead's cloud; its own map changes leave the lead's alone."""
    rng = np.random.default_rng(11)
    G = _sharing_cls(((0.15,), dict(max_map_points=60_000, max_scan_points=5_000)))
    g, subs = _lead(G, rng)
    q = tr._cloud(rng, 400, (0.1, 0.1, 0.0))
    g.map_restore()
    want = tr._view(g, q)
    w = g.twin()
    w.assess_reserve(1000, 8)
    w.replay_share(g)
    assert w.replay_info() == g.replay_info()
    w.map_restore()
    assert tr._view(w, q) == want
    for j in (0, len(subs) - 1, 2):
        g.replay_stage(j)
        w.replay_stage(j)
        assert tr._staged(w) == tr._staged(g), j
        assert w.replay_frame(j) == g.replay_frame(j)
    w.map_add_points(tr._cloud(rng, 2000, (1.0, -0.5, 0.3)), True)   # the worker's map is its own
    g.map_restore()
    assert tr._view(g, q) == want
    w.close()


def _refused(call):
    with pytest.raises(emul.EmulError) as ex:
        call()
    assert ex.value.code == INVALID
    return str(ex.value)


def test_sharing_refusals():
    rng = np.random.default_rng(12)
    G = _sharing_cls(((0.15,), dict(max_map_points=60_000, max_scan_points=5_000)))
    g, subs = _lead(G, rng)
    w = g.twin()
    assert "own" in _refused(lambda: w.replay_share(w))
    assert "own" in _refused(lambda: g.replay_share(g))
    # configurations that differ: filter_size_map, capacities, brick cells, cell directory
    for args, kw in (((0.2,), dict(max_map_points=60_000, max_scan_points=5_000)), ((0.15,), dict(max_map_points=70_000, max_scan_points=5_000)),
                     ((0.15,), dict(max_map_points=60_000, max_scan_points=6_000)),
                     ((0.15,), dict(max_map_points=60_000, max_scan_points=5_000, brick_cells_log2=2)),
                     ((0.15,), dict(max_map_points=60_000, max_scan_points=5_000, knn_index=2))):
        other = G(*args, **kw)
        assert "configuration" in _refused(lambda: other.replay_share(g))
        other.close()
    # a lead without a snapshot, without a store
    bare = g.twin()
    assert "snapshot" in _refused(lambda: w.replay_share(bare))
    bare.map_snapshot()
    assert "replay store" in _refused(lambda: w.replay_share(bare))
    bare.close()
    # shared: the store and the snapshot stay as they are, and the lead stays alive
    w.replay_share(g)
    assert "already" in _refused(lambda: w.replay_share(g))
    third = g.twin()
    assert "lead" in _refused(lambda: third.replay_share(w))      # a worker is no lead
    assert "lead" in _refused(lambda: g.replay_share(third))       # a lead is no worker
    for ctx in (g, w):
        _refused(lambda: ctx.map_snapshot())
        _refused(lambda: ctx.replay_reserve(10, 4))
        _refused(lambda: ctx.replay_append(subs[0]["handle"], 0.0, 1.0))
    assert g.L.liinit_destroy(g.h) == INVALID and "unshare" in g.L.liinit_last_error(g.h).decode()
    assert g.replay_info()["frames"] == len(subs)
    # unshare ends it; so does destroying the worker
    w.replay_unshare()
    assert "does not share" in _refused(lambda: w.replay_unshare())
    third.replay_share(g)
    w.replay_share(g)
    w.close()
    _refused(lambda: g.map_snapshot())           # third still shares
    third.close()
    g.map_snapshot()
    g.replay_reserve(10, 4)
    assert g.L.liinit_destroy(g.h) == 0
    g.h = None


# ---- the native loop and run_many ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul_run(tmp_path_factory):
    nd, rp, _, _ = tr._emul_run(tmp_path_factory.mktemp("run"), trigger_at=6, seconds=1.2)
    rp.assessment.radius = EMUL_RADIUS
    cfg = nd.odom
    _use_emul(rp, ((float(cfg.ds),), dict(max_map_points=400_000, max_scan_points=1_000)))
    yield nd, rp
    rp.close()


def _same_replay(a, b):
    assert [j for j, _ in a["states"]] == [j for j, _ in b["states"]]
    for (_, x), (_, y) in zip(a["states"], b["states"]):
        assert x.tobytes() == y.tobytes()
    assert tr._same(a["result"], b["result"])
    assert a["R_LI"].tobytes() == b["R_LI"].tobytes() and a["T_LI"].tobytes() == b["T_LI"].tobytes()
    assert np.float64(a["rms_m"]).tobytes() == np.float64(b["rms_m"]).tobytes()


def test_native_replays_on_a_worker_pool_equal_the_python_replay(emul_run):
    """run_many at jobs=2 (the lead and one worker, in turn) with the native loop: every posterior state, the end extrinsic, every field
    of the evaluation and rms_m are bit-equal to Replay.run -- unfrozen with LI-Init's extrinsic, frozen at a perturbed one, and at lag
    shifts of -+5 ms and -+20 ms."""
    nd, rp = emul_run
    R0, T0 = np.asarray(rp.res["R_LI"], float), np.asarray(rp.res["T_LI"], float)
    Rp, Tp = assess.rot_exp([0.0, np.radians(0.5), 0.0]) @ R0, T0 + [0.0, 0.02, 0.0]
    cands = [(None, None, 0.0, False), (Rp, Tp, 0.0, True), (Rp, Tp, -0.005, True), (Rp, Tp, 0.005, True), (R0, T0, -0.02, True),
             (R0, T0, 0.02, True)]
    got = rp.run_many(cands, jobs=2)
    assert len(rp.workers) == 1
    for c, r in zip(cands, got):
        want = rp.run(*c)
        assert len(want["states"]) >= 4
        _same_replay(r, want)
    # the run's own hand-over, natively on the lead: the run's states bit for bit
    own = rp.run_native(frozen=False)
    assert [j for j, _ in own["states"]] == [j for j, _ in rp.run_states]
    assert all(a.tobytes() == b.tobytes() for (_, a), (_, b) in zip(own["states"], rp.run_states)) and own["rms_m"] == 0.0


def test_sweep_and_refine_do_not_depend_on_the_jobs(emul_run):
    """Replay.refine at jobs=2 has the trace and the refined result of jobs=1."""
    nd, rp = emul_run
    _, _, R_fin, T_fin = assess.host_pose(nd.odom.state)
    a = rp.refine(R_fin, T_fin, max_replays=4)
    b = rp.refine(R_fin, T_fin, max_replays=4, jobs=2)
    assert len(a["trace"]) == len(b["trace"]) == 4
    for x, y in zip(a["trace"], b["trace"]):
        assert (x["stage"], x["R"].tobytes(), x["T"].tobytes(), x["shift_ms"]) == (y["stage"], y["R"].tobytes(), y["T"].tobytes(), y["shift_ms"])
        assert tr._same(x["result"], y["result"])
    assert a["state"].tobytes() == b["state"].tobytes() and a["calib"].keys() == b["calib"].keys()
    assert (a["status"], a["best"], a["shift_ms"]) == (b["status"], b["best"], b["shift_ms"])


def test_bad_jobs_are_refused(emul_run):
    _, rp = emul_run
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="jobs"):
            rp.run_many([(None, None, 0.0, True)], jobs=bad)


# ---- the batched search ----------------------------------------------------------------------------------------------------------------
def _rows(r):
    return [(x["stage"], x["R"].tobytes(), x["T"].tobytes(), x["shift_ms"], np.float64(x["mme"]).tobytes()) for x in r["trace"]]


def _same_search(a, b):
    assert _rows(a) == _rows(b)
    for k in ("status", "start", "at_edge", "best", "steps", "shift_ms"):
        assert a[k] == b[k], k
    assert a["R"].tobytes() == b["R"].tobytes() and a["T"].tobytes() == b["T"].tobytes()
    assert np.float64(a["mme"]).tobytes() == np.float64(b["mme"]).tobytes()
    assert list(a["axes"]) == list(b["axes"])
    for k in a["axes"]:
        assert np.array(a["axes"][k]).tobytes() == np.array(b["axes"][k]).tobytes(), k


@pytest.mark.parametrize("nan", [False, True])
def test_batched_search_equals_the_sequential_one_at_every_budget(nan):
    """search with score_many on the bowls: for every budget from 1 to past convergence (so the budget also runs out inside a batch), the
    trace field by field, the result, the status and the axes are those of the one-at-a-time search; no batch exceeds 12 candidates;
    with a NaN-scoring half of the lag axis too."""
    f = trf.Bowl(7.0)

    def score(R, T, s):
        return math.nan if nan and s > 0 else f(R, T, s)
    sizes = []

    def score_many(cands):
        sizes.append(len(cands))
        return [score(*c) for c in cands]
    kw = dict(R_init=trf.R_STAR, T_init=trf.T_STAR + [0.05, 0, 0])
    full = refine.search(score, trf.R_START, trf.T_START, max_replays=10_000, **kw)
    assert full["status"] == "converged"
    n = len(full["trace"])
    for budget in range(1, n + 3):
        a = refine.search(score, trf.R_START, trf.T_START, max_replays=budget, **kw)
        b = refine.search(score, trf.R_START, trf.T_START, max_replays=budget, score_many=score_many, **kw)
        _same_search(a, b)
    assert max(sizes) == 12 and all(1 <= s <= 12 for s in sizes)


# ---- the runner ------------------------------------------------------------------------------------------------------------------------
def test_runner_replay_jobs(tmp_path, monkeypatch, capsys):
    """run --assess-replay --refine --replay-jobs 2 writes assessment_replay.txt and refinement.txt equal to --replay-jobs 1 but for the
    wall times and seconds; the summary names the jobs; a bad --replay-jobs exits 1 with a message."""
    from lidar_imu_init_b200 import run
    main = trf._runner(tmp_path, monkeypatch)
    made = run.make_node

    def make(args, c, log):
        nd = made(args, c, log)
        cls = type(nd.odom.g)
        cls.replay_share = capi.LiInitGpu.replay_share
        cls.replay_unshare = capi.LiInitGpu.replay_unshare
        cls.twin = lambda self: cls(c.filter_size_map, max_map_points=400_000, max_scan_points=1_000)
        return nd
    monkeypatch.setattr(run, "make_node", make)
    H = _emul_host()
    real_replay = assess.Replay

    def replay(*a, **k):
        rp = real_replay(*a, **k)
        rp.host_lib, rp.threads = H, 1
        return rp
    monkeypatch.setattr(assess, "Replay", replay)
    texts = {}
    for jobs in ("1", "2"):
        out = tmp_path / f"j{jobs}"
        assert main(out, ["--assess-replay", "--refine", "--refine-max-replays", "3", "--replay-jobs", jobs]) == 0
        err = capsys.readouterr().err
        assert f"{jobs} replay job" in err
        texts[jobs] = [open(out / "result" / f).read() for f in ("assessment_replay.txt", "refinement.txt")]
    a, b = (assess.parse_replay_report(texts[j][0]) for j in ("1", "2"))
    assert str(a["rows"]) == str(b["rows"]) and str(a["axes"]) == str(b["axes"]) and str(a["lag"]) == str(b["lag"])   # (NaN-safe)
    assert {k: v for k, v in a["header"].items() if k != "replay_s"} == {k: v for k, v in b["header"].items() if k != "replay_s"}
    a, b = (assess.parse_refine_report(texts[j][1]) for j in ("1", "2"))
    assert str([{k: v for k, v in r.items() if k != "seconds"} for r in a["rows"]]) == str([{k: v for k, v in r.items() if k != "seconds"}
                                                                                           for r in b["rows"]])
    assert str(a["axes"]) == str(b["axes"]) and a["result"] == b["result"]   # (an unmeasured axis has NaN differences)
    assert {k: v for k, v in a["header"].items() if k != "wall_s"} == {k: v for k, v in b["header"].items() if k != "wall_s"}
    for bad in ("0", "-2", "abc", "1.5"):
        assert main(tmp_path / "bad", ["--quiet", "--refine", "--replay-jobs", bad]) == 1
        assert "--replay-jobs" in capsys.readouterr().err
