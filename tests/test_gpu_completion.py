"""GPU: the sum-of-completion-times objective (SB_FLAG_SUM_COMPLETION, objective="completion") — bit-exact scores on
every kernel path against the fp32 oracle, unchanged schedules, arg-min keys, the exact optimum on small instances,
incremental rounds, and solve()'s plans."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import tasks_from_tuples
from oracle import ref_completion as RC, ref_eval as R
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1


def _ref(tab, opt, prio, ints, nodes=1):
    return RC.c_evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32, threads=8, nodes=nodes)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))                                        # first index of the minimum
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective="completion", best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
def test_completion_scores_on_the_tile_and_generic_paths(engine, J, S, B, ints):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities: the device's sum equals the oracle's left
    fold bit for bit, and the best key is the arg-min of the sums."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    ref = _ref(tab, opt, prio, ints)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, integer_starts=ints, **kw)
        assert p == path, kw
        assert np.array_equal(got, ref), kw
        assert key == _key_of(ref, 11), kw
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    mk = engine.eval(opt, prio, integer_starts=ints).cpu().numpy()
    assert np.all(ref >= mk) and not np.array_equal(ref, mk)       # the makespan path is untouched by the flag
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective="completion")
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
def test_completion_scores_with_large_tables(engine, ints):
    """J = 1024 with the full 8-strategy table: path 9 (opt rows re-ordered on the device, position-major kernel),
    path 4 (tile kernel, table in global memory) and the generic kernel; then the position-major kernel on
    caller rows in schedule order with its table in shared memory (5), split over a CTA pair (7) and in global
    memory (8)."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    ref = _ref(tab, opt, prio, ints)
    for kw, path in (({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)):
        got, key, p = _eval(engine, opt, prio, integer_starts=ints, **kw)
        assert p == path and np.array_equal(got, ref) and key == _key_of(ref, 11), kw
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    ref = _ref(tab, opt, prio, ints)
    obp = opt_by_position(opt, prio)
    for kw, path in (({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)):
        got, key, p = _eval(engine, obp, prio, integer_starts=ints, by_position=True, **kw)
        assert p == path and np.array_equal(got, ref) and key == _key_of(ref, 11), kw
    got, key, p = _eval(engine, opt, prio, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
def test_completion_multi_node_and_decode(engine, J, nodes, B, ints):
    """1..4 nodes: every path equals the oracle; sb_eval_full and sb_decode give the same starts and slot masks with
    and without the flag, and their score is the sum."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    ref = _ref(tab, opt, prio, ints, nodes)
    for kw in ({}, {"_no_stream": True}, {"_force_generic": True}):
        got, key, _ = _eval(engine, opt, prio, integer_starts=ints, reduced=True, **kw)
        assert np.array_equal(got, ref) and key == _key_of(ref, 11), kw
    got, _, _ = _eval(engine, opt.contiguous(), prio.contiguous(), integer_starts=ints, reduced=True)
    assert np.array_equal(got, ref)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective="completion")
    mk, start_m, mask_m = engine.eval_full(opt, prio, integer_starts=ints, reduced=True)
    assert np.array_equal(tot.cpu().numpy(), ref)
    assert torch.equal(start, start_m) and torch.equal(mask, mask_m)
    b = B // 3
    o, p = opt[b].cpu().numpy(), prio[b].cpu().numpy()
    d1 = engine.decode(o, p, integer_starts=ints, reduced=True, objective="completion")
    d0 = engine.decode(o, p, integer_starts=ints, reduced=True)
    assert d1["makespan"] == float(ref[b]) and d0["makespan"] == float(mk[b])
    for k in ("start", "slotmask", "strategy", "gpus", "node"):
        assert np.array_equal(d1[k], d0[k]), k


def test_alternate_shape_refuses_the_completion_objective(engine):
    from saturn_b200._lib import SaturnB200Error
    from saturn_b200.solver import SolverError
    T, valid = R.synth_table(32, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    with pytest.raises(SaturnB200Error, match="ALT_WARPSCAN"):
        engine.eval(opt, prio, alt_shape=True, objective="completion")
    with pytest.raises(SolverError):
        engine.eval(opt, prio, objective="tardiness")


def _completion_cases():
    with open(os.path.join(HERE, "golden", "completion_cases.json")) as f:
        return json.load(f)["cases"]


def _check_plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, mk2 = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0 and mk2 == pytest.approx(mk, rel=1e-12)
    return sum(p[0] + p[2] for p in plan)


def _device_table(tuples):
    """The fp32 table solve() hands the device: every runtime rounded UP to the next fp32 (build_table)."""
    tab, om = R.table_from_tuples(tuples)
    tab32 = np.where(np.isfinite(tab), tab.astype(np.float32), np.inf)
    up = tab32.astype(np.float64) < tab
    tab32[up] = np.nextafter(tab32[up], np.float32(np.inf))
    return tab32, om


def test_solve_reaches_the_fixture_optimum():
    """On every fixture HiGHS proved optimal for the sum of completion times, solve(objective="completion") returns a
    feasible plan whose sum equals the MILP's optimum; the device's fp32 score is the oracle's fp32 score of that plan
    on the device's table (runtimes rounded up to fp32, so not the fixture's round-to-nearest fp32 optimum)."""
    from saturn_b200 import solver as S
    n = 0
    for rec in _completion_cases():
        if not rec["milp"]["proven_optimal"]:
            continue
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        out = S.solve(tasks, None, chains=8192, rounds=60, objective="completion")
        total = _check_plan(tasks, out)
        assert S.last_stats["objective"] == "completion"
        assert S.last_stats["total_completion"] == pytest.approx(total, rel=1e-12)
        assert total == pytest.approx(rec["milp"]["total_completion"], rel=1e-9), rec["name"]
        tab32, om = _device_table(tuples)
        plan = R.plan_from_arrays(tuples, out[0], out[1], out[2], out[3])
        opt = [om[t][plan[t][4]] for t in range(len(tuples))]
        boa = out[4]                                               # boa[a][b] == 1: a is scheduled before b
        order = sorted(range(len(tuples)), key=lambda t: sum(1 for a in range(len(tuples)) if a != t and boa[a][t] == 1))
        dev = RC.list_schedule(tab32, opt, order, True, np.float32)[0]
        assert S.last_stats["device_makespan"] == dev, rec["name"]
        n += 1
    assert n >= 15


def test_solve_reaches_the_exhaustive_optimum_on_random_small_instances():
    """Random 2..5-task instances on one and two nodes: solve(objective="completion")'s fp32 score equals the fp32
    exhaustive optimum and its plan is feasible."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(7)
    for trial in range(14):
        nodes = 1 if trial % 2 == 0 else 2
        J = int(rng.integers(2, 6 if nodes == 1 else 5))
        tuples = []
        for _ in range(J):
            ks = sorted(rng.choice([1, 2, 4, 8], size=int(rng.integers(1, 3 if nodes > 1 else 4)), replace=False).tolist())
            base = float(rng.uniform(20, 900))
            tuples.append([(int(k), base * float(rng.uniform(1, 1.3)) / k ** float(rng.uniform(0.4, 1.0))) for k in ks])
        tasks = tasks_from_tuples(tuples)
        out = S.solve(tasks, None, chains=4096, rounds=64, nodes=nodes, seed=trial, objective="completion")
        assert R.milp_constraints_hold(tuples, *out) == [], trial
        tab32, om = _device_table(tuples)
        if nodes > 1:
            tab32 = R.reduce_table(tab32)[0][:, None, :]
            om = [[o & 7 for o in ops] for ops in om]
        best = RC.brute_force(tab32, om, True, dtype=np.float32, nodes=nodes)[0]
        assert S.last_stats["device_makespan"] == best, (trial, J, nodes, tuples)


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
def test_incremental_rounds_in_completion_mode(engine, J):
    """The verify hook recomputes every incremental score from position 0: no mismatch with the running sum stored in
    the snapshots.  Fused and unfused rounds both return valid plans that re-score to the reported sum."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective="completion")
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    for r in (a, b):
        assert float(RC.list_schedule(tmin, r.opt, r.prio, True, np.float32)[0]) == r.makespan
    assert b.history[-1][2] < b.history[0][2] or J <= 40
    for fused in (True, False):
        kw2 = dict(kw, chains=4096 if J <= 300 else 2048, rounds=24)
        r = run_search(engine, _no_fused=not fused, **kw2)
        assert engine.search_is_fused() == fused
        assert sorted(r.prio.tolist()) == list(range(J))
        assert float(RC.list_schedule(tmin, r.opt, r.prio, True, np.float32)[0]) == r.makespan


def test_the_objective_changes_the_plan_and_is_reproducible():
    """A fixed J = 256 instance: the completion plan's sum of completion times is no larger than the makespan plan's
    and than every shortest-processing-time seed's; the same call twice returns the identical plan.  Hysteresis is
    refused with the completion objective."""
    from saturn_b200 import solver as S
    from saturn_b200.search import lpt_seeds
    from saturn_b200.synth import synth_table
    from saturn_b200.solver import SolverError, strategies_from_table
    from conftest import DuckTask
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    tasks = [DuckTask("t%d" % j, strategies[j]) for j in range(J)]
    kw = dict(chains=16384, rounds=200, seed=1)
    a = S.solve(tasks, None, objective="completion", **kw)
    tc_a = S.last_stats["total_completion"]
    assert _check_plan(tasks, a) == pytest.approx(tc_a, rel=1e-12)
    a2 = S.solve(tasks, None, objective="completion", **kw)
    assert all(x == y for x, y in zip(a[:5], a2[:5])) and a2[5] == a[5] and S.last_stats["total_completion"] == tc_a
    m = S.solve(tasks, None, **kw)
    assert S.last_stats["objective"] == "makespan"
    tc_m = S.last_stats["total_completion"]
    assert tc_a <= tc_m
    Tdev, usable, _ = S.build_table(tasks)
    Tdev = np.where(usable[:, None, :] | ~usable.any(axis=1)[:, None, None], Tdev, np.inf)
    for col, order in lpt_seeds(Tdev[:, 0, :], sentinel=np.inf, objective="completion"):
        spt = RC.list_schedule(Tdev.astype(np.float64), col, order, True, np.float64)[0]
        assert tc_a <= spt * (1 + 1e-6)
    with pytest.raises(SolverError):
        S.solve(tasks, None, objective="completion", hysteresis=True, chains=64, rounds=2)
    with pytest.raises(SolverError):
        S.solve(tasks, None, objective="throughput", chains=64, rounds=2)


def test_multiple_devices_equal_single_device_runs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200.engine import Engine, MultiEngine
    J, S = 96, 4
    T, valid = R.synth_table(J, S, 8, seed=2)
    chains, rounds = 4096, 32
    singles = []
    for d in range(2):
        e = Engine(d, stream=torch.cuda.current_stream(torch.device("cuda", d)))
        e.set_table(T)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=d * chains, reduced=True, sync_every=16,
                                    objective="completion"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    r = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="completion")
    best = min(singles, key=lambda x: x["key"])
    assert r["key"] == best["key"] and r["makespan"] == best["makespan"]
    assert np.array_equal(r["opt"], best["opt"]) and np.array_equal(r["prio"], best["prio"])
    me.close()
