"""GPU: the total (weighted) tardiness (SB_FLAG_DUE, solve(objective="tardiness", due=...)) — bit-exact scores on
every kernel path against the fp32 oracle, unweighted and weighted, d = 0 equal to the completion objectives,
unchanged schedules, arg-min keys, the refusals, incremental rounds, the stop at zero, and solve()'s plans."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_tardiness as RT
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1


def _w(J, seed):
    return np.random.default_rng(seed).uniform(0.1, 12.0, size=J).astype(np.float32)


def _setup(engine, tab, opt, prio, weighted, seed, nodes=1):
    """Due dates spread from before t = 0 to past a typical completion (a mix of late and early jobs), and the
    weights; returns (objective, w or None, d)."""
    J = tab.shape[0]
    o, p = opt[:1].cpu().numpy(), prio[:1].cpu().numpy()
    mean = float(RT.c_evaluate(tab, o, p, np.zeros(J), True, np.float64, nodes=nodes)[0]) / J
    d = (np.random.default_rng(seed).uniform(-0.2, 2.0, size=J) * mean).astype(np.float32)
    engine.set_due(d)
    w = None
    if weighted:
        w = _w(J, seed + 1)
        engine.set_weights(w)
    return ("weighted_tardiness" if weighted else "tardiness"), w, d


def _ref(tab, opt, prio, ints, d, w, nodes=1):
    return RT.c_evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), d, ints, np.float32, threads=8, nodes=nodes,
                         weights=w)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _check_runs(engine, opt, prio, ref, objective, runs, **common):
    """Every run: the tardiness equals the oracle bit for bit with the arg-min key, and some jobs are late; with
    d = 0 it equals the (weighted) completion objective's score.  Leaves the due dates set."""
    d = engine.due.copy()
    assert (ref > 0).any() and (ref < np.inf).all()
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, objective, **common, **kw)
        assert path is None or p == path, kw
        assert got.tobytes() == ref.tobytes(), kw
        assert key == _key_of(ref, 11), kw
    completion = objective.replace("tardiness", "completion")
    engine.set_due(np.zeros(engine.J, np.float32))
    for kw, path in runs:
        got = _eval(engine, opt, prio, objective, **common, **kw)[0]
        assert got.tobytes() == _eval(engine, opt, prio, completion, **common, **kw)[0].tobytes(), kw
    engine.set_due(d)


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_tardiness_on_the_tile_and_generic_paths(engine, J, S, B, ints, weighted):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities, and sb_eval_host."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    objective, w, d = _setup(engine, tab, opt, prio, weighted, J)
    ref = _ref(tab, opt, prio, ints, d, w)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, objective, runs, integer_starts=ints)
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), objective, integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective=objective)
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_tardiness_with_large_tables(engine, ints, weighted):
    """J = 1024 with the full 8-strategy table: paths 9, 4 and 0 on job-indexed rows; J = 256: the position-major
    kernel with its table in shared memory (5), split over a CTA pair (7) and in global memory (8)."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    objective, w, d = _setup(engine, tab, opt, prio, weighted, 5)
    ref = _ref(tab, opt, prio, ints, d, w)
    _check_runs(engine, opt, prio, ref, objective, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)],
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    objective, w, d = _setup(engine, tab, opt, prio, weighted, 9)
    ref = _ref(tab, opt, prio, ints, d, w)
    obp = opt_by_position(opt, prio)
    _check_runs(engine, obp, prio, ref, objective, [({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)],
                integer_starts=ints, by_position=True)
    got, key, p = _eval(engine, opt, prio, objective, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref) and key == _key_of(ref, 11)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_tardiness_multi_node_and_decode(engine, J, nodes, B, ints, weighted):
    """1..4 nodes: every path equals the oracle; sb_eval_full and sb_decode give the same starts and slot masks as
    the makespan call, and their score is the tardiness."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    objective, w, d = _setup(engine, tab, opt, prio, weighted, J + nodes, nodes)
    ref = _ref(tab, opt, prio, ints, d, w, nodes)
    runs = [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, objective, runs, integer_starts=ints, reduced=True)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=objective)
    mk, start_m, mask_m = engine.eval_full(opt, prio, integer_starts=ints, reduced=True)
    assert np.array_equal(tot.cpu().numpy(), ref)
    assert torch.equal(start, start_m) and torch.equal(mask, mask_m)
    b = B // 3
    o, p = opt[b].cpu().numpy(), prio[b].cpu().numpy()
    d1 = engine.decode(o, p, integer_starts=ints, reduced=True, objective=objective)
    d0 = engine.decode(o, p, integer_starts=ints, reduced=True)
    assert d1["makespan"] == float(ref[b]) and d0["makespan"] == float(mk[b])
    for k in ("start", "slotmask", "strategy", "gpus", "node"):
        assert np.array_equal(d1[k], d0[k]), k


def test_refusals(engine):
    """DUE without SUM (SB_ERR_ARG), before set_due and after set_table cleared them (SB_ERR_STATE), set_due with
    the wrong J or a bad value, and the alternate shape."""
    from saturn_b200 import _lib
    from saturn_b200._lib import SaturnB200Error, check
    from saturn_b200.solver import SolverError
    import ctypes as C
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE) == -3        # no due dates yet
    with pytest.raises(SolverError, match="set_due"):                                            # the engine's check
        engine.eval(opt, prio, objective="tardiness")
    engine.set_due(np.zeros(J))
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_DUE) == -1                                   # without SUM
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE) == 0
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_WEIGHTED) == -3
    with pytest.raises(SaturnB200Error, match="ALT_WARPSCAN"):
        engine.eval(opt, prio, alt_shape=True, objective="tardiness")
    engine.set_table(T)                                                                           # clears them
    assert engine.due is None
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE) == -3
    for call in (lambda: engine.eval(opt, prio, objective="tardiness"),
                 lambda: engine.search_init(256, reduced=True, objective="tardiness"),
                 lambda: engine.search_run(256, 4, reduced=True, objective="weighted_tardiness")):
        with pytest.raises(SolverError, match="set_due"):
            call()
    for bad in ([np.nan] + [1.0] * (J - 1), [np.inf] + [1.0] * (J - 1), [2.0 ** 24] + [1.0] * (J - 1)):
        d = np.array(bad, np.float32)
        assert engine._lib.sb_set_due(engine._h, C.c_void_p(d.ctypes.data), J) == -1
    d = np.zeros(J + 1, np.float32)
    assert engine._lib.sb_set_due(engine._h, C.c_void_p(d.ctypes.data), J + 1) == -1
    with pytest.raises(SolverError):
        engine.set_due(np.zeros(J - 1))
    check(engine._lib.sb_set_due(engine._h, None, 0))


def _cases():
    with open(os.path.join(HERE, "golden", "tardiness_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, _ = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    return [p[0] + p[2] for p in plan]                                   # completion time per task


def _device_table(tuples):
    tab, om = R.table_from_tuples(tuples)
    tab32 = np.where(np.isfinite(tab), tab.astype(np.float32), np.inf)
    up = tab32.astype(np.float64) < tab
    tab32[up] = np.nextafter(tab32[up], np.float32(np.inf))
    return tab32, om


def test_solve_reaches_the_tardiness_fixture_optimum():
    """On every fixture HiGHS proved optimal, solve(objective="tardiness", due=..., weights=...) returns a feasible
    plan whose weighted tardiness equals the MILP's optimum; the device's score is the oracle's fp32 score of that
    plan; last_stats holds the plan's tardiness and late tasks."""
    from saturn_b200 import solver as S
    n = 0
    for rec in _cases():
        if not rec["milp"]["proven_optimal"]:
            continue
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        w, d = rec["weights"], rec["due"]
        out = S.solve(tasks, None, chains=8192, rounds=60, objective="tardiness", due=d, weights=w)
        comp = _plan(tasks, out)
        ww = w if w is not None else [1.0] * len(comp)
        total = sum(wi * max(0.0, c - di) for wi, c, di in zip(ww, comp, d))
        assert S.last_stats["weighted_tardiness"] == pytest.approx(total, rel=1e-12, abs=1e-9)
        assert S.last_stats["late_tasks"] == sum(1 for c, di in zip(comp, d) if c > di)
        assert total == pytest.approx(rec["milp"]["weighted_tardiness"], rel=1e-9, abs=1e-9), rec["name"]
        tab32, om = _device_table(tuples)
        plan = R.plan_from_arrays(tuples, out[0], out[1], out[2], out[3])
        opt = [om[t][plan[t][4]] for t in range(len(tuples))]
        boa = out[4]
        order = sorted(range(len(tuples)), key=lambda t: sum(1 for a in range(len(tuples)) if a != t and boa[a][t] == 1))
        dev = RT.list_schedule(tab32, opt, order, d, True, np.float32, weights=w)[0]
        assert S.last_stats["device_makespan"] == dev, rec["name"]
        n += 1
    assert n >= 15


def test_solve_reaches_the_exhaustive_optimum_on_random_small_instances():
    """Random 2..5-task instances with random due dates, unweighted and weighted, on one and two nodes: the
    device's fp32 tardiness equals the fp32 exhaustive optimum and the plan is feasible."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(23)
    for trial in range(16):
        nodes = 1 if trial % 2 == 0 else 2
        J = int(rng.integers(2, 6 if nodes == 1 else 5))
        tuples = []
        for _ in range(J):
            ks = sorted(rng.choice([1, 2, 4, 8], size=int(rng.integers(1, 3 if nodes > 1 else 4)), replace=False).tolist())
            base = float(rng.uniform(20, 900))
            tuples.append([(int(k), base * float(rng.uniform(1, 1.3)) / k ** float(rng.uniform(0.4, 1.0))) for k in ks])
        d = rng.integers(-50, 900, size=J).astype(float)
        w = rng.uniform(0.2, 6.0, size=J) if trial % 4 >= 2 else None
        tasks = tasks_from_tuples(tuples)
        out = S.solve(tasks, None, chains=4096, rounds=64, nodes=nodes, seed=trial, objective="tardiness", due=d,
                      weights=w)
        assert R.milp_constraints_hold(tuples, *out) == [], trial
        tab32, om = _device_table(tuples)
        if nodes > 1:
            tab32 = R.reduce_table(tab32)[0][:, None, :]
            om = [[o & 7 for o in ops] for ops in om]
        best = RT.brute_force(tab32, om, d, True, dtype=np.float32, nodes=nodes,
                              weights=None if w is None else w.astype(np.float32))[0]
        assert S.last_stats["device_makespan"] == best, (trial, J, nodes, tuples, d, w)


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
def test_incremental_rounds_with_due_dates(engine, J):
    """The verify hook recomputes every incremental score from position 0: no mismatch with the running tardiness
    stored in the snapshots.  Fused and unfused rounds return valid plans that re-score to the reported value."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    w = _w(J, 200 + J)
    engine.set_weights(w)
    # due dates a quarter of the way into a typical plan: most jobs late, so the search never reaches zero
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    d = (np.random.default_rng(J).uniform(0.0, 0.25, size=J) * horizon).astype(np.float32)
    engine.set_due(d)
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective="weighted_tardiness")
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    assert b.makespan > 0
    for r in (a, b):
        assert float(RT.list_schedule(tmin, r.opt, r.prio, d, True, np.float32, weights=w)[0]) == r.makespan
    for fused in (True, False):
        kw2 = dict(kw, chains=4096 if J <= 300 else 2048, rounds=24)
        r = run_search(engine, _no_fused=not fused, **kw2)
        assert engine.search_is_fused() == fused
        assert sorted(r.prio.tolist()) == list(range(J))
        assert float(RT.list_schedule(tmin, r.opt, r.prio, d, True, np.float32, weights=w)[0]) == r.makespan


def test_loose_due_dates_stop_the_search_at_zero(engine):
    """Due dates past any plan's completion: the library's loop and the Python driver stop with stop_reason 3 and
    a score of +0 long before the round budget."""
    from saturn_b200.search import run_search
    J = 64
    T, valid = R.synth_table(J, 3, 8, seed=4)
    engine.set_table(T)
    engine.set_due(np.full(J, 2.0 ** 24 - 1, np.float32))
    r = engine.search_run(4096, 400, seed=1, reduced=True, sync_every=8, objective="tardiness")
    assert r["stop_reason"] == 3 and r["makespan"] == 0.0 and r["rounds"] < 400
    p = run_search(engine, chains=4096, rounds=400, seed=1, reduced=True, use_dist=False, exchange_every=8,
                   objective="tardiness", _python_driver=True)
    assert p.stop_reason == 3 and p.makespan == 0.0 and p.rounds < 400


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_tardiness_plan_beats_the_other_objectives_and_is_reproducible():
    """J = 256 with seeded due dates: the tardiness plan's tardiness is no larger than the completion plan's and the
    makespan plan's; the same call twice returns the identical plan."""
    from saturn_b200 import solver as S
    tasks = _tasks256()
    J = len(tasks)
    kw = dict(chains=16384, rounds=200, seed=1)
    mk_plan = S.solve(tasks, None, **kw)
    c_mk = _plan(tasks, mk_plan)
    c_plan = _plan(tasks, S.solve(tasks, None, objective="completion", **kw))
    d = np.random.default_rng(5).integers(0, int(max(c_plan)), size=J).astype(float)
    a = S.solve(tasks, None, objective="tardiness", due=d, **kw)
    ta = S.last_stats["weighted_tardiness"]
    ca = _plan(tasks, a)
    assert ta == pytest.approx(sum(max(0.0, c - di) for c, di in zip(ca, d)), rel=1e-12)
    for other in (c_mk, c_plan):
        assert ta <= sum(max(0.0, c - di) for c, di in zip(other, d))
    a2 = S.solve(tasks, None, objective="tardiness", due=d, **kw)
    assert all(x == y for x, y in zip(a[:5], a2[:5])) and a2[5] == a[5]
    assert S.last_stats["weighted_tardiness"] == ta


def test_orchestrate_with_due_dates_keyed_by_task():
    """A due-date mapping keyed by Task survives orchestrate()'s shrinking task list: the loop runs to completion in
    simulated time."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    due = {t: float(1000 * (i + 1)) for i, t in enumerate(tasks)}
    launched = []
    recs = orchestrate(tasks, interval=1000, execute_fn=lambda rtt, btr, itv, npt, tdd: launched.append(len(rtt)),
                       solver_kwargs={"chains": 4096, "rounds": 25, "objective": "tardiness", "due": due},
                       max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)
    assert len(recs) >= 2 and sum(launched) >= 8


def test_multiple_devices_equal_single_device_runs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200.engine import Engine, MultiEngine
    J, S = 96, 4
    T, valid = R.synth_table(J, S, 8, seed=2)
    w = _w(J, 2)
    d = np.random.default_rng(3).uniform(0, 2000, size=J).astype(np.float32)
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_weights(w)
        e.set_due(d)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16,
                                    objective="weighted_tardiness"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_weights(w)
    me.set_due(d)
    r = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="weighted_tardiness")
    best = min(singles, key=lambda x: x["key"])
    assert r["key"] == best["key"] and r["makespan"] == best["makespan"]
    assert np.array_equal(r["opt"], best["opt"]) and np.array_equal(r["prio"], best["prio"])
    me.close()
