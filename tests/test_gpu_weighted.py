"""GPU: the weighted sum of completion times (SB_FLAG_WEIGHTED, solve(objective="completion", weights=...)) —
bit-exact scores on every kernel path against the fp32 oracle, unit weights equal to the unweighted objective and
doubled weights to twice it, unchanged schedules, arg-min keys, the refusals, incremental rounds, and solve()'s
plans."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_weighted as RW
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1


def _w(J, seed):
    return np.random.default_rng(seed).uniform(0.1, 12.0, size=J).astype(np.float32)


def _ref(tab, opt, prio, ints, w, nodes=1):
    return RW.c_evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32, threads=8, nodes=nodes,
                         weights=w)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective="weighted_completion", **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _check_runs(engine, opt, prio, ref, runs, **common):
    """Every run: the weighted score equals the oracle bit for bit with the arg-min key; with unit weights it equals
    the completion objective's score, with weights of 2 exactly twice it.  Leaves `ref`'s weights set."""
    w = engine.weights.copy()
    J = engine.J
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, **common, **kw)
        assert path is None or p == path, kw
        assert got.tobytes() == ref.tobytes(), kw
        assert key == _key_of(ref, 11), kw
    plain = {}
    for i, (kw, path) in enumerate(runs):
        plain[i] = _eval(engine, opt, prio, objective="completion", **common, **kw)[0]
    for scale in (1.0, 2.0):
        engine.set_weights(np.full(J, scale, np.float32))
        for i, (kw, path) in enumerate(runs):
            got, _, p = _eval(engine, opt, prio, **common, **kw)
            assert got.tobytes() == (plain[i] * np.float32(scale)).astype(np.float32).tobytes(), kw
    engine.set_weights(w)


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
def test_weighted_scores_on_the_tile_and_generic_paths(engine, J, S, B, ints):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities, and sb_eval_host."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    w = _w(J, J)
    engine.set_weights(w)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    ref = _ref(tab, opt, prio, ints, w)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, runs, integer_starts=ints)
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective="weighted_completion")
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
def test_weighted_scores_with_large_tables(engine, ints):
    """J = 1024 with the full 8-strategy table: paths 9, 4 and 0 on job-indexed rows; J = 256: the position-major
    kernel on rows in schedule order with its table in shared memory (5), split over a CTA pair (7) and in global
    memory (8)."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    w = _w(J, 5)
    engine.set_weights(w)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    ref = _ref(tab, opt, prio, ints, w)
    _check_runs(engine, opt, prio, ref, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)],
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    w = _w(J, 9)
    engine.set_weights(w)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    ref = _ref(tab, opt, prio, ints, w)
    obp = opt_by_position(opt, prio)
    _check_runs(engine, obp, prio, ref, [({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)],
                integer_starts=ints, by_position=True)
    got, key, p = _eval(engine, opt, prio, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref) and key == _key_of(ref, 11)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
def test_weighted_multi_node_and_decode(engine, J, nodes, B, ints):
    """1..4 nodes: every path equals the oracle; sb_eval_full and sb_decode give the same starts and slot masks with
    and without the weights, and their score is the weighted sum."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    w = _w(J, J + nodes)
    engine.set_weights(w)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    ref = _ref(tab, opt, prio, ints, w, nodes)
    runs = [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, runs, integer_starts=ints, reduced=True)
    got, _, _ = _eval(engine, opt.contiguous(), prio.contiguous(), integer_starts=ints, reduced=True)
    assert np.array_equal(got, ref)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective="weighted_completion")
    mk, start_m, mask_m = engine.eval_full(opt, prio, integer_starts=ints, reduced=True)
    assert np.array_equal(tot.cpu().numpy(), ref)
    assert torch.equal(start, start_m) and torch.equal(mask, mask_m)
    plain = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective="completion")[0]
    engine.set_weights(np.ones(J, np.float32))
    one = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective="weighted_completion")[0]
    assert torch.equal(one, plain)
    engine.set_weights(w)
    b = B // 3
    o, p = opt[b].cpu().numpy(), prio[b].cpu().numpy()
    d1 = engine.decode(o, p, integer_starts=ints, reduced=True, objective="weighted_completion")
    d0 = engine.decode(o, p, integer_starts=ints, reduced=True)
    assert d1["makespan"] == float(ref[b]) and d0["makespan"] == float(mk[b])
    for k in ("start", "slotmask", "strategy", "gpus", "node"):
        assert np.array_equal(d1[k], d0[k]), k


def test_refusals(engine):
    """WEIGHTED without SUM (SB_ERR_ARG), before set_weights and after set_table cleared them (SB_ERR_STATE),
    set_weights with the wrong J or a weight that is not finite and > 0, and the alternate shape."""
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
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_WEIGHTED) == -3   # no weights yet
    with pytest.raises(SaturnB200Error, match="sb_set_weights"):
        engine.eval(opt, prio, objective="weighted_completion")
    engine.set_weights(np.ones(J))
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_WEIGHTED) == -1                             # without SUM
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_WEIGHTED) == 0
    with pytest.raises(SaturnB200Error, match="ALT_WARPSCAN"):
        engine.eval(opt, prio, alt_shape=True, objective="weighted_completion")
    engine.set_table(T)                                                                           # clears them
    assert engine.weights is None
    with pytest.raises(SaturnB200Error, match="sb_set_weights"):
        engine.eval(opt, prio, objective="weighted_completion")
    with pytest.raises(SaturnB200Error, match="sb_set_weights"):
        engine.search_init(256, reduced=True, objective="weighted_completion")
    for bad in ([1.0, 0.0] + [1.0] * (J - 2), [1.0, -1.0] + [1.0] * (J - 2), [np.nan] * J):
        w = np.array(bad, np.float32)
        assert engine._lib.sb_set_weights(engine._h, C.c_void_p(w.ctypes.data), J) == -1
    w = np.ones(J + 1, np.float32)
    assert engine._lib.sb_set_weights(engine._h, C.c_void_p(w.ctypes.data), J + 1) == -1
    with pytest.raises(SolverError):
        engine.set_weights(np.ones(J - 1))
    with pytest.raises(SolverError):
        engine.set_weights([1e-50] * J)
    check(engine._lib.sb_set_weights(engine._h, None, 0))


def _weighted_cases():
    with open(os.path.join(HERE, "golden", "weighted_completion_cases.json")) as f:
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


def test_solve_reaches_the_weighted_fixture_optimum():
    """On every fixture HiGHS proved optimal, solve(objective="completion", weights=...) returns a feasible plan
    whose weighted sum equals the MILP's optimum; the device's score is the oracle's fp32 score of that plan."""
    from saturn_b200 import solver as S
    n = 0
    for rec in _weighted_cases():
        if not rec["milp"]["proven_optimal"]:
            continue
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        w = rec["weights"]
        out = S.solve(tasks, None, chains=8192, rounds=60, objective="completion", weights=w)
        comp = _plan(tasks, out)
        total = sum(wi * c for wi, c in zip(w, comp))
        assert S.last_stats["weighted_completion"] == pytest.approx(total, rel=1e-12)
        assert S.last_stats["total_completion"] == pytest.approx(sum(comp), rel=1e-12)
        assert total == pytest.approx(rec["milp"]["weighted_completion"], rel=1e-9), rec["name"]
        tab32, om = _device_table(tuples)
        plan = R.plan_from_arrays(tuples, out[0], out[1], out[2], out[3])
        opt = [om[t][plan[t][4]] for t in range(len(tuples))]
        boa = out[4]
        order = sorted(range(len(tuples)), key=lambda t: sum(1 for a in range(len(tuples)) if a != t and boa[a][t] == 1))
        dev = RW.list_schedule(tab32, opt, order, True, np.float32, weights=w)[0]
        assert S.last_stats["device_makespan"] == dev, rec["name"]
        n += 1
    assert n >= 15


def test_solve_reaches_the_exhaustive_optimum_on_random_small_instances():
    """Random 2..5-task instances with random weights on one and two nodes: the device's fp32 weighted sum equals the
    fp32 exhaustive optimum and the plan is feasible."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(17)
    for trial in range(14):
        nodes = 1 if trial % 2 == 0 else 2
        J = int(rng.integers(2, 6 if nodes == 1 else 5))
        tuples = []
        for _ in range(J):
            ks = sorted(rng.choice([1, 2, 4, 8], size=int(rng.integers(1, 3 if nodes > 1 else 4)), replace=False).tolist())
            base = float(rng.uniform(20, 900))
            tuples.append([(int(k), base * float(rng.uniform(1, 1.3)) / k ** float(rng.uniform(0.4, 1.0))) for k in ks])
        w = rng.uniform(0.2, 6.0, size=J)
        tasks = tasks_from_tuples(tuples)
        out = S.solve(tasks, None, chains=4096, rounds=64, nodes=nodes, seed=trial, objective="completion", weights=w)
        assert R.milp_constraints_hold(tuples, *out) == [], trial
        tab32, om = _device_table(tuples)
        if nodes > 1:
            tab32 = R.reduce_table(tab32)[0][:, None, :]
            om = [[o & 7 for o in ops] for ops in om]
        best = RW.brute_force(tab32, om, True, dtype=np.float32, nodes=nodes, weights=w.astype(np.float32))[0]
        assert S.last_stats["device_makespan"] == best, (trial, J, nodes, tuples, w)


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
def test_incremental_rounds_with_weights(engine, J):
    """The verify hook recomputes every incremental score from position 0: no mismatch with the weighted running sum
    stored in the snapshots.  Fused and unfused rounds return valid plans that re-score to the reported sum."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    w = _w(J, 200 + J)
    engine.set_weights(w)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective="weighted_completion")
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    for r in (a, b):
        assert float(RW.list_schedule(tmin, r.opt, r.prio, True, np.float32, weights=w)[0]) == r.makespan
    assert b.history[-1][2] < b.history[0][2] or J <= 40
    for fused in (True, False):
        kw2 = dict(kw, chains=4096 if J <= 300 else 2048, rounds=24)
        r = run_search(engine, _no_fused=not fused, **kw2)
        assert engine.search_is_fused() == fused
        assert sorted(r.prio.tolist()) == list(range(J))
        assert float(RW.list_schedule(tmin, r.opt, r.prio, True, np.float32, weights=w)[0]) == r.makespan


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_unit_weights_reproduce_the_completion_plan():
    """J = 256: weights of 1 give the same plan, device score and sum of completion times as the unweighted
    completion objective with the same seed (the weighted path runs; it is not short-circuited)."""
    from saturn_b200 import solver as S
    tasks = _tasks256()
    kw = dict(chains=16384, rounds=200, seed=1, objective="completion")
    a = S.solve(tasks, None, **kw)
    sa = dict(S.last_stats)
    b = S.solve(tasks, None, weights=[1.0] * len(tasks), **kw)
    sb = dict(S.last_stats)
    assert all(x == y for x, y in zip(a[:5], b[:5])) and a[5] == b[5]
    assert sa["device_makespan"] == sb["device_makespan"] and sa["total_completion"] == sb["total_completion"]
    assert sb["weighted_completion"] == sb["total_completion"]


def test_heavy_tasks_finish_earlier_and_the_plan_is_reproducible():
    """J = 256, 32 tasks of weight 8 and the rest 1: the weighted plan's weighted sum is no larger than the unweighted
    completion plan's and than every WSPT seed's; the heavy tasks' mean completion time drops; the same call twice
    returns the identical plan."""
    from saturn_b200 import solver as S
    from saturn_b200.search import lpt_seeds
    tasks = _tasks256()
    J = len(tasks)
    heavy = set(range(0, J, J // 32))
    w = [8.0 if j in heavy else 1.0 for j in range(J)]
    kw = dict(chains=16384, rounds=200, seed=1, objective="completion")
    u = S.solve(tasks, None, **kw)
    cu = _plan(tasks, u)
    a = S.solve(tasks, None, weights=w, **kw)
    wc_a = S.last_stats["weighted_completion"]
    ca = _plan(tasks, a)
    assert wc_a == pytest.approx(sum(wi * c for wi, c in zip(w, ca)), rel=1e-12)
    assert wc_a <= sum(wi * c for wi, c in zip(w, cu))
    assert np.mean([ca[j] for j in heavy]) < np.mean([cu[j] for j in heavy])
    Tdev, usable, _ = S.build_table(tasks)
    Tdev = np.where(usable[:, None, :] | ~usable.any(axis=1)[:, None, None], Tdev, np.inf)
    for col, order in lpt_seeds(Tdev[:, 0, :], sentinel=np.inf, objective="weighted_completion",
                                weights=np.array(w, np.float32)):
        wspt = RW.list_schedule(Tdev.astype(np.float64), col, order, True, np.float64, weights=w)[0]
        assert wc_a <= wspt * (1 + 1e-6)
    a2 = S.solve(tasks, None, weights=w, **kw)
    assert all(x == y for x, y in zip(a[:5], a2[:5])) and a2[5] == a[5]
    assert S.last_stats["weighted_completion"] == wc_a


def test_orchestrate_with_weights_keyed_by_task():
    """A mapping keyed by Task survives orchestrate()'s shrinking task list: the loop runs to completion in
    simulated time."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    weights = {t: (5.0 if i % 3 == 0 else 1.0) for i, t in enumerate(tasks)}
    launched = []
    recs = orchestrate(tasks, interval=1000, execute_fn=lambda rtt, btr, itv, npt, tdd: launched.append(len(rtt)),
                       solver_kwargs={"chains": 4096, "rounds": 25, "objective": "completion", "weights": weights},
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
    chains, rounds = 4096, 32
    singles = []
    for d in range(2):
        e = Engine(d, stream=torch.cuda.current_stream(torch.device("cuda", d)))
        e.set_table(T)
        e.set_weights(w)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=d * chains, reduced=True, sync_every=16,
                                    objective="weighted_completion"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_weights(w)
    r = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="weighted_completion")
    best = min(singles, key=lambda x: x["key"])
    assert r["key"] == best["key"] and r["makespan"] == best["makespan"]
    assert np.array_equal(r["opt"], best["opt"]) and np.array_equal(r["prio"], best["prio"])
    me.close()
