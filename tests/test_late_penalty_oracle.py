"""CPU: the late-penalty objective (SB_FLAG_LATE_PENALTY, solve(objective="late_penalty")) in the oracle — the Python
schedule and fold against the C port (oracle/ref_late_penalty.c) bit for bit, p = 0 against the tardiness oracle, the
exact check on the tie-heavy and boundary inputs of test_exact_edges, absent cells, the MILP fixtures
(tests/golden/late_penalty_cases.json, oracle/gen_late_penalty.py), the lexicographic limit of large penalties, the
seeds, solve() / solve_table() / orchestrate() handling without a device, and the flag and setter against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_exact as X, ref_late_penalty as LP, ref_late_tasks as LT, ref_release as RR

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _candidates(J, S, B, nodes, seed):
    if nodes == 1:
        T, valid = R.synth_table(J, S, 8, seed=seed)
        tab = R.canon_table(T, range(1, 9))
        opt, prio = R.synth_candidates(J, B, valid, seed=seed + 1)
        return tab, opt, prio
    T, valid = R.synth_table(J, 1, 8, seed=seed, masked=False)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = R.synth_candidates(J, B, valid, seed=seed + 1)
    rng = np.random.default_rng(seed + 2)
    return tab, (opt | (rng.integers(0, nodes, size=opt.shape) << 3)).astype(np.uint8), prio


def _due(J, seed, scale):
    return np.random.default_rng(seed).uniform(-0.3, 1.2, size=J) * scale


def _weights(J, seed):
    return np.random.default_rng(seed).choice([0.25, 0.5, 1.0, 1.5, 3.0, 7.0, 0.1], size=J)


def _penalty(J, seed, scale):
    """Real penalties with about a quarter at 0 and one -0.0."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0, 1, size=J) * scale
    p[rng.random(J) < 0.25] = 0.0
    p[0] = -0.0
    return p


@pytest.mark.parametrize("J,S,nodes,B", [(7, 3, 1, 30000), (40, 4, 1, 20000), (23, 1, 2, 60), (12, 1, 4, 60)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_python_fold_equals_c_port(J, S, nodes, B, ints, released, weighted):
    """The C port (schedule and fold in C) gives the same bits as the Python schedule with the numpy fold, scores,
    starts and slot masks, in fp32 and fp64: integer and real-valued starts, 1 to 4 nodes, with and without release
    dates, unit and real rates."""
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 7 * nodes)
    scale = 2000.0 * J / 8
    d = _due(J, J + 1, scale)
    p = _penalty(J, J + 4, scale)
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    w = _weights(J, J + 3) if weighted else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = LP.c_evaluate(tab, opt, prio, d, p, r, ints, dtype, want_plan=True, threads=8, nodes=nodes,
                                  weights=w)
        py, ps, pm = LP.evaluate(tab, opt, prio, d, p, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True,
                                 weights=w)
        assert c.dtype == dtype and c.tobytes() == py.tobytes()
        assert np.array_equal(cs, ps) and np.array_equal(cm, pm)
        assert (c >= 0).all() and not np.signbit(c).any() and len(np.unique(c)) > 1


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_zero_penalties_are_the_tardiness(nodes, ints, released, weighted):
    """With p = 0 (and with p = -0.0, stored as +0) every score equals the tardiness oracle's bit for bit, in fp32 and
    fp64; penalties change the score exactly where a job is late."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 500, nodes, seed=41)
    d = _due(J, 42, 6000.0)
    r = np.random.default_rng(43).uniform(-10, 3000, size=J) if released else None
    w = _weights(J, 44) if weighted else None
    obj = "weighted_tardiness" if weighted else "tardiness"
    for dtype in (np.float32, np.float64):
        td = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, dtype, nodes=nodes, objective=obj,
                           weights=w, due=d)
        for zero in (np.zeros(J), np.full(J, -0.0)):
            got = LP.c_evaluate(tab, opt, prio, d, zero, r, ints, dtype, nodes=nodes, weights=w)
            assert got.tobytes() == td.tobytes()
        late = LP.c_evaluate(tab, opt, prio, d, np.full(J, 5.0), r, ints, dtype, nodes=nodes, weights=w)
        assert (late >= td).all() and (late > td).any()


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_absent_cells_score_inf(nodes, ints, released):
    """A candidate that gives a job an option it does not have (rt = +inf) scores +inf in the C port and the Python
    fold, on exactly the candidates the makespan oracle finds infeasible, whatever that job's penalty; every other
    candidate stays finite."""
    J, B = 24, 400
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, B, nodes, seed=17)
    tab = np.array(tab, dtype=np.float32)
    tab[5, :, 2] = np.inf                                        # job 5 has no 3-GPU option anywhere
    rng = np.random.default_rng(18)
    bad = rng.random(B) < 0.3
    opt = opt.copy()
    for b in range(B):
        o = int(opt[b, 5])
        row = tab[5, 0 if nodes > 1 else o >> 3]
        cols = [c for c in range(8) if np.isfinite(row[c])]
        opt[b, 5] = (o & 0xF8) | (2 if bad[b] else (o & 7 if (o & 7) in cols else cols[0]))
    d = _due(J, 19, 2000.0 * J / 8)
    p = _penalty(J, 22, 500.0)
    p[5] = 0.0
    r = np.random.default_rng(20).uniform(0, 3000, size=J) if released else None
    w = _weights(J, 21)
    for dtype in (np.float32, np.float64):
        c = LP.c_evaluate(tab, opt, prio, d, p, r, ints, dtype, threads=8, nodes=nodes, weights=w)
        py = LP.evaluate(tab, opt, prio, d, p, r, ints, dtype, nodes=nodes, use_c=False, weights=w)
        mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, dtype, nodes=nodes)
        assert c.tobytes() == py.tobytes()
        assert np.array_equal(np.isinf(c), bad) and np.array_equal(np.isinf(mk), bad)
        assert np.isfinite(c[~bad]).all() and (c[~bad] > 0).any()


# the inputs of test_exact_edges.test_exact_reference_agrees_with_both_oracles (the squared form's list), on which
# every term p + w x and every partial sum stays exact in fp32 with small integer and dyadic penalties
EDGE_CASES = [(1, 1, "equal", True), (2, 8, "zeros", False), (7, 3, "small", True), (31, 1, "dyadic", False),
              (33, 5, "equal", True), (128, 7, "zeros", True)]
PENALTIES = np.array([0.0, -0.0, 1.0, 2.0, 0.5, 8.0, 0.25])


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: "J%d-n%d-%s-%s" % (c[0], c[1], c[2], "int" if c[3] else "real"))
@pytest.mark.parametrize("rel", [None, "ready", "nonpos"])
@pytest.mark.parametrize("weighted", [False, True])
def test_exact_check_on_edge_inputs(case, rel, weighted):
    """On the tie-heavy and boundary inputs of test_exact_edges (equal, zero, -0.0 and dyadic runtimes; due dates at
    a completion, one step before it, -0.0, negative and beyond every completion; release dates at slot times and
    non-positive) fp32 rounds nothing: the fp32 C port and the float64 fold equal sum [C > d] (p + w (C - d)) in exact
    arithmetic, and the starts are ref_exact's.  A job that completes exactly at its due date pays nothing."""
    import test_exact_edges as E
    J, nodes, fam, ints = case
    S = 1 if nodes > 1 else 3
    seed = J * 101 + nodes
    tab = E.rt_table(fam, J, S, seed)
    opt, prio = E.candidates(J, 15, nodes if nodes > 1 else S, seed + 1)
    r = E.release_dates(rel, tab, opt, prio, ints, nodes, seed + 2)
    d = E.due_dates(tab, opt, prio, ints, nodes, r, seed + 4)
    w = E.WEIGHTS[np.random.default_rng(seed + 3).integers(0, 5, J)].astype(np.float32) if weighted else None
    p = PENALTIES[np.random.default_rng(seed + 5).integers(0, len(PENALTIES), J)]
    c32, cst, _ = LP.c_evaluate(tab, opt, prio, d, p, r, ints, np.float32, want_plan=True, threads=8, nodes=nodes,
                                weights=w)
    s64 = LP.evaluate(tab, opt, prio, d, p, r, ints, np.float64, nodes=nodes, use_c=False, weights=w)
    _, xst, _ = X.batch(tab, opt, prio, r, ints, nodes, "makespan")
    for b in range(len(opt)):
        ex = LP.exact(tab, opt[b], prio[b], d, p, r, ints, nodes, weights=w)
        assert float(ex) == s64[b] == float(c32[b]), (b, ex, s64[b], c32[b])
        assert np.array_equal(xst[b], cst[b].astype(np.float64))


def test_on_time_at_the_due_date():
    """A job that completes exactly at its due date pays neither its penalty nor any tardiness; one unit later it pays
    both."""
    tab = np.full((1, 1, 8), 5.0, np.float32)
    o, pr = np.array([[7]], np.uint8), np.array([[0]], np.uint8)
    for dtype in (np.float32, np.float64):
        assert float(LP.c_evaluate(tab, o, pr, [5.0], [100.0], dtype=dtype)[0]) == 0.0
        assert float(LP.c_evaluate(tab, o, pr, [4.0], [100.0], dtype=dtype, weights=[3.0])[0]) == 103.0
    assert LP.exact(tab, o[0], pr[0], [5.0], [100.0]) == 0 and LP.exact(tab, o[0], pr[0], [4.0], [100.0]) == 101


def test_exact_refuses_a_sum_that_fp32_would_round():
    """exact() asserts that p + w x is exact in fp32: a penalty of 2^24 plus a tardiness of 1 is not."""
    tab = np.full((1, 1, 8), 5.0, np.float32)
    with pytest.raises(X.NotExact):
        LP.exact(tab, np.array([7], np.uint8), np.array([0], np.uint8), [4.0], [2.0 ** 24])


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "late_penalty_cases.json")) as f:
        return json.load(f)["cases"]


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum; where HiGHS stopped at its time limit
    with an incumbent, the exhaustive optimum is no worse than it.  Every MILP plan is feasible and its score is its
    objective value, the fp32 and fp64 optima agree, and the fixtures include weighted instances, instances with
    release dates, zero and dominant penalties, and instances whose optimum beats both the tardiness optimum and the
    late-count optimum."""
    proven = 0
    for rec in cases:
        m, bf = rec["milp"], rec["bruteforce_f64"]["score"]
        assert rec["bruteforce_f32"]["score"] == bf, rec["name"]      # integer data: fp32 rounds nothing here
        if m["start"] is None:
            assert not m["proven_optimal"], rec["name"]
            continue
        assert m["feasible"] and m["overlaps"] == 0, rec["name"]
        assert m["score"] == pytest.approx(m["objective_value"], rel=1e-6, abs=1e-6), rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), rec["name"]
        else:
            assert bf <= m["score"] * (1 + 1e-9), rec["name"]
    assert len(cases) == 24 and proven >= len(cases) // 2
    assert sum(rec["weights"] is not None for rec in cases) >= 10
    assert sum(rec["release"] is not None for rec in cases) >= 4
    assert sum(0.0 in rec["penalty"] for rec in cases) >= 10
    assert sum(max(rec["penalty"]) >= 10000 for rec in cases) >= 8
    both = sum(rec["tardiness_optimum"]["differs"] and rec["late_count_optimum"]["differs"] for rec in cases)
    assert both >= 3


def test_fixture_plans_rescore_to_their_recorded_values(cases):
    """The recorded optima and the rescored tardiness and late-count optima re-derive from the oracle, and each
    `differs` flag says whether that plan is worse than the optimum; every runtime, due date and penalty is an
    integer."""
    for rec in cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        assert all(float(rt).is_integer() for t in tuples for _k, rt in t)
        assert all(float(x).is_integer() and x >= 0 for x in rec["penalty"])
        assert all(float(x).is_integer() for x in rec["due"])
        tab, _ = R.table_from_tuples(tuples)
        for key, dtype in (("bruteforce_f64", np.float64), ("bruteforce_f32", np.float32)):
            b = rec[key]
            got = LP.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), rec["due"],
                              rec["penalty"], rec["release"], True, dtype, weights=rec["weights"])[0]
            assert float(got) == b["score"], (rec["name"], key)
        best = rec["bruteforce_f64"]["score"]
        for key in ("tardiness_optimum", "late_count_optimum"):
            t = rec[key]
            got = LP.evaluate(tab, np.array([t["opt"]], np.uint8), np.array([t["prio"]], np.uint8), rec["due"],
                              rec["penalty"], rec["release"], True, np.float64, weights=rec["weights"])[0]
            assert float(got) == t["score"] >= best and t["differs"] == (t["score"] > best), (rec["name"], key)


@pytest.mark.parametrize("seed", range(6))
def test_large_penalties_give_the_late_count_then_the_tardiness(seed):
    """In float64 with one penalty above any total tardiness the horizon allows, the late-penalty optimum has the
    late-count optimum's count, and the least (weighted) tardiness among the plans with that count."""
    rng = np.random.default_rng(300 + seed)
    J = 4
    tuples = [[(k, float(rng.integers(5, 60)) / k) for k in (1, 2, 4)] for _ in range(J)]
    tab, optmap = R.table_from_tuples(tuples)
    due = [float(x) for x in rng.integers(0, 40, J)]
    w = [float(x) for x in rng.choice([1.0, 2.0, 3.0], J)] if seed % 2 else None
    big = 1e7
    opts = np.array(np.meshgrid(*optmap, indexing="ij")).reshape(J, -1).T.astype(np.uint8)
    import itertools
    perms = np.array(list(itertools.permutations(range(J))), np.uint8)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    count = LT.evaluate(tab, opt, prio, due, None, True, np.float64)
    tard = LP.evaluate(tab, opt, prio, due, np.zeros(J), None, True, np.float64, weights=w)
    score = LP.evaluate(tab, opt, prio, due, np.full(J, big), None, True, np.float64, weights=w)
    i = int(np.argmin(score))
    least = count.min()
    assert count[i] == least == LT.brute_force(tab, optmap, due, None, True, np.float64)[0]
    assert tard[i] == tard[count == least].min()
    assert tard.max() < big
    assert LP.brute_force(tab, optmap, due, np.full(J, big), None, True, np.float64, weights=w)[0] == score[i]


def test_lpt_seeds_are_the_tardiness_seeds():
    """lpt_seeds(objective="late_penalty" / "weighted_late_penalty") plants the EDD seeds of "tardiness" /
    "weighted_tardiness" unchanged (ties by rt / w with weights), on 1 and 3 nodes, with and without release dates."""
    from saturn_b200.search import lpt_seeds
    for nodes in (1, 3):
        for released in (False, True):
            rng = np.random.default_rng(5 + nodes)
            J = 64
            tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
            d = np.round(rng.uniform(0, 3, size=J)).astype(np.float32) * 1000  # many equal due dates: ties matter
            r = rng.uniform(0, 500, size=J).astype(np.float32) if released else None
            w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32)
            for obj, base in (("late_penalty", "tardiness"), ("weighted_late_penalty", "weighted_tardiness")):
                a = lpt_seeds(tmin, objective=obj, due=d, release=r, nodes=nodes, weights=w)
                b = lpt_seeds(tmin, objective=base, due=d, release=r, nodes=nodes, weights=w)
                for (ca, oa), (cb, ob) in zip(a, b):
                    assert np.array_equal(ca, cb) and np.array_equal(oa, ob)


class _Strat:
    def __init__(self, runtime, executor="x"):
        self.runtime, self.executor = runtime, executor


class _Task:
    def __init__(self, name, runtimes=(100.0, 60.0)):
        self.name = name
        self.strategies = {g: _Strat(rt) for g, rt in zip((1, 2), runtimes)}


D3 = [1.0, 2.0, 3.0]
P3 = [5.0, 0.0, 2.0]


@pytest.mark.parametrize("objective,kw,match", [
    ("late_penalty", {"penalty": P3}, "needs due dates"),
    ("late_penalty", {"due": D3}, "penalty=\\.\\.\\."),
    ("late_penalty", {"due": D3, "penalty": [1.0, 2.0]}, "one value per task"),
    ("late_penalty", {"due": D3, "penalty": [1.0, -1.0, 2.0]}, "finite and >= 0"),
    ("late_penalty", {"due": D3, "penalty": [1.0, float("nan"), 2.0]}, "finite and >= 0"),
    ("late_penalty", {"due": D3, "penalty": [1.0, float("inf"), 2.0]}, "finite and >= 0"),
    ("late_penalty", {"due": D3, "penalty": [1.0, 1e39, 2.0]}, "2\\^126"),
    ("late_penalty", {"due": D3, "penalty": [1.0, 3e37, 2.0]}, "2\\^126"),
    ("late_penalty", {"due": D3, "penalty": ["a", 1.0, 2.0]}, "numbers"),
    ("late_penalty", {"due": D3, "penalty": P3, "hysteresis": True}, "hysteresis"),
    ("late_penalty", {"due": D3, "penalty": P3, "weights": [1.0, 0.0, 1.0]}, "finite and > 0"),
    ("late_penalty", {"due": D3, "penalty": P3, "release": [0.0, float("inf"), 1.0]}, None),
    ("tardiness", {"due": D3, "penalty": P3}, "late_penalty' only"),
    ("late_tasks", {"due": D3, "penalty": P3}, "late_penalty' only"),
    ("makespan", {"penalty": P3}, "late_penalty' only"),
    ("squared_tardiness", {"due": D3, "penalty": P3}, "late_penalty' only"),
])
def test_solver_refusals_before_any_device_call(objective, kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one): a
    missing `due` or `penalty`, `penalty` under any other objective, a wrong length, a negative, NaN, inf or
    non-numeric penalty, penalties whose fp32 sum could overflow (3 tasks * 3e37 >= 2^126), hysteresis, a bad weight,
    a bad release date."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective=objective, engine=object(), **kw)
    if "hysteresis" not in kw:  # solve_table has no hysteresis
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [100.0, 60.0]
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective=objective, engine=object(), **kw)


def test_penalty_mapping_in_solve():
    """solve() takes `penalty` as a mapping Task -> number too; a task missing from it, or a mapping in solve_table,
    raises SolverError before any device call."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    p64, p32 = S._resolve_penalty({tasks[2]: 3.0, tasks[0]: 1.0, tasks[1]: -0.0}, "late_penalty", 3, tasks)
    assert p64 == [1.0, -0.0, 3.0] and p32.dtype == np.float32 and p32.tolist() == [1.0, 0.0, 3.0]
    assert not np.signbit(p32).any()
    with pytest.raises(S.SolverError, match="no entry for task"):
        S.solve(tasks, None, objective="late_penalty", engine=object(), due=D3, penalty={tasks[0]: 1.0})
    T = np.full((3, 1, 8), np.inf, dtype=np.float32)
    T[:, 0, :2] = [100.0, 60.0]
    with pytest.raises(S.SolverError, match="sequence aligned"):
        S.solve_table(T, objective="late_penalty", engine=object(), due=D3, penalty={0: 1.0})
    assert S._resolve_penalty(None, "tardiness", 3) == (None, None)


def test_overflow_guard_boundary():
    """The guard refuses J * max(p) >= 2^126 on the fp32 penalties, and nothing below it."""
    from saturn_b200.engine import penalty_f32
    from saturn_b200.solver import SolverError
    J = 4
    ok = float(np.nextafter(np.float32(2.0 ** 124), np.float32(0)))
    assert penalty_f32([0.0, ok, 1.0, 2.0], J)[1] == np.float32(ok)
    with pytest.raises(SolverError, match="2\\^126"):
        penalty_f32([0.0, 2.0 ** 124, 1.0, 2.0], J)
    penalty_f32(np.zeros(1 << 20), 1 << 20)


def test_late_penalty_stats_and_set_objective():
    """The stats are float64 sums over the late tasks only, with weighted_tardiness and late_tasks; _set_objective
    hands the penalties to the engine and picks the weighted form with weights."""
    from saturn_b200 import solver as S
    st = S._late_penalty_stats([0.0, 10.0, 20.0], [3.0, 4.0, 5.0], [2.0, 1.0, 0.5], [5.0, 11.0, 20.0],
                               [100.0, 7.0, 1.5])
    assert st == {"late_penalty": 7.0 + 3.0 + 1.5 + 0.5 * 5.0, "weighted_tardiness": 3.0 + 2.5, "late_tasks": 2}
    assert S._late_penalty_stats([0.0], [3.0], None, [3.0], [9.0])["late_penalty"] == 0.0

    class Eng:
        def __init__(self):
            self.calls = []

        def __getattr__(self, name):
            return lambda *a, **k: self.calls.append(name)
    w = np.ones(3, np.float32)
    d = np.zeros(3, np.float32)
    p = np.ones(3, np.float32)
    e = Eng()
    assert S._set_objective(e, "late_penalty", None, d, None, p) == "late_penalty" and "set_penalty" in e.calls
    assert S._set_objective(Eng(), "late_penalty", w, d, None, p) == "weighted_late_penalty"
    e = Eng()
    S._set_objective(e, "tardiness", None, d)
    assert "set_penalty" not in e.calls


def test_engine_objective_table():
    """OBJECTIVES keeps its ten forms; the late-penalty pair has its own tuple, its flags and per-job arrays, reads the
    penalties (no other form does), needs due dates and penalties, and the name check accepts it."""
    from saturn_b200 import _lib
    from saturn_b200.engine import (OBJECTIVES, PENALTY_OBJECTIVES, SQUARED_OBJECTIVES, _OBJECTIVES, _require_due,
                                    _require_penalty, objective_flag, objective_reads_penalty, objective_spec)
    from saturn_b200.solver import SolverError
    assert OBJECTIVES == ("makespan", "completion", "weighted_completion", "tardiness", "weighted_tardiness",
                          "max_lateness", "late_tasks", "weighted_late_tasks", "max_tardiness",
                          "weighted_max_tardiness")
    assert PENALTY_OBJECTIVES == ("late_penalty", "weighted_late_penalty")
    assert set(_OBJECTIVES) == set(OBJECTIVES) | set(SQUARED_OBJECTIVES) | set(PENALTY_OBJECTIVES)
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_LATE_PENALTY
    assert objective_flag("late_penalty") == base
    assert objective_flag("weighted_late_penalty") == base | _lib.FLAG_WEIGHTED
    assert objective_spec("late_penalty") == (base, False, True)
    assert objective_spec("weighted_late_penalty") == (base | _lib.FLAG_WEIGHTED, True, True)
    assert {o for o in _OBJECTIVES if objective_reads_penalty(o)} == set(PENALTY_OBJECTIVES)
    for obj in PENALTY_OBJECTIVES:
        with pytest.raises(SolverError):
            _require_due(None, obj)
        with pytest.raises(SolverError, match="set_penalty"):
            _require_penalty(None, obj)
        _require_penalty(np.zeros(1, np.float32), obj)
    for obj in OBJECTIVES + SQUARED_OBJECTIVES:
        _require_penalty(None, obj)
    with pytest.raises(SolverError, match="weighted_late_penalty"):
        objective_spec("penalty")


def test_orchestrate_passes_penalties_through(monkeypatch):
    """orchestrate() hands every solve the same `penalty` mapping while it shifts the due dates, and refuses a
    sequence `penalty` before any solve."""
    from saturn_b200 import orchestrator as O
    from saturn_b200.solver import SolverError

    class Strat:
        def __init__(self, runtime):
            self.runtime = runtime

    class Task:
        def __init__(self, name, batches, per_batch):
            self.name, self.total_batches = name, batches
            self.strategies = {1: Strat(per_batch * batches)}
            self.selected_strategy = self.strategies[1]

    tasks = [Task("a", 1, 500.0), Task("b", 3, 900.0)]
    due = {tasks[0]: 800.0, tasks[1]: 4000.0}
    penalty = {tasks[0]: 50.0, tasks[1]: 0.0}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), kw["objective"], kw["due"], kw["penalty"]))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "late_penalty", "due": due, "penalty": penalty})
    assert [n for n, _, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got_due, got_p) in enumerate(seen):
        assert obj == "late_penalty" and got_due == {t: d - n * 1000 for t, d in due.items()}
        assert got_p == penalty
    seen.clear()
    with pytest.raises(SolverError, match="mapping"):
        O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "late_penalty", "due": due,
                                                           "penalty": [50.0, 0.0]})
    assert not seen


def test_flag_and_setter_match_the_header():
    """SB_FLAG_LATE_PENALTY is 16384 in the header and in _lib, shares no bit with any other flag or test hook, and is
    in the hooks' static_assert; sb_set_penalty is declared as the other per-job setters are and is in SYMBOLS."""
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_LATE_PENALTY\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_LATE_PENALTY == 16384
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_LATE_PENALTY"]
    assert all(f & _lib.FLAG_LATE_PENALTY == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_LATE_PENALTY == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_LATE_PENALTY" in f.read().split("the test hooks share no bit")[0]
    assert re.search(r"\bint sb_set_penalty\(sb_handle\* h, const float\* p, int J\);", header)
    assert "sb_set_penalty" in _lib.SYMBOLS
    assert re.search(r"#define\s+SB_ABI_VERSION\s+1\b", header)
