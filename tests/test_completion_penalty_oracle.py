"""CPU: the completion-penalty objective (SB_FLAG_COMPLETION_PENALTY, solve(objective="completion_penalty")) in the
oracle — the Python schedule and fold against the C port (oracle/ref_completion_penalty.c) bit for bit, p = 0 against
the weighted-completion oracles, the exact check on the tie-heavy and boundary inputs of test_exact_edges, absent
cells, the MILP and front fixtures (tests/golden/completion_penalty_cases.json, oracle/gen_completion_penalty.py),
the cap limit of large penalties, the seeds, solve() / solve_front() / orchestrate() handling without a device, and
the flag against the header."""
import itertools
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_completion_penalty as CP, ref_eval as R, ref_exact as X, ref_release as RR, ref_weighted as RW

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
    dates, unit and real weights."""
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 7 * nodes)
    scale = 2000.0 * J / 8
    d = _due(J, J + 1, scale)
    p = _penalty(J, J + 4, scale)
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    w = _weights(J, J + 3) if weighted else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = CP.c_evaluate(tab, opt, prio, d, p, r, ints, dtype, want_plan=True, threads=8, nodes=nodes,
                                  weights=w)
        py, ps, pm = CP.evaluate(tab, opt, prio, d, p, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True,
                                 weights=w)
        assert c.dtype == dtype and c.tobytes() == py.tobytes()
        assert np.array_equal(cs, ps) and np.array_equal(cm, pm)
        assert (c > 0).all() and len(np.unique(c)) > 1


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_zero_penalties_are_the_weighted_completion(nodes, ints, released, weighted):
    """With p = 0 (and with p = -0.0, stored as +0) every score equals the (weighted) completion oracle's bit for
    bit, in fp32 and fp64 (ref_weighted without release dates, ref_release's completion folds with them); penalties
    add to the score exactly where a job is late."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 500, nodes, seed=41)
    d = _due(J, 42, 6000.0)
    r = np.random.default_rng(43).uniform(-10, 3000, size=J) if released else None
    w = _weights(J, 44) if weighted else None
    for dtype in (np.float32, np.float64):
        if r is None:
            wc = RW.c_evaluate(tab, opt, prio, ints, dtype, nodes=nodes, weights=w)
        else:
            wc = RR.c_evaluate(tab, opt, prio, r, ints, dtype, nodes=nodes,
                               objective="weighted_completion" if weighted else "completion", weights=w)
        for zero in (np.zeros(J), np.full(J, -0.0)):
            got = CP.c_evaluate(tab, opt, prio, d, zero, r, ints, dtype, nodes=nodes, weights=w)
            assert got.tobytes() == wc.tobytes()
        late = CP.c_evaluate(tab, opt, prio, d, np.full(J, 5.0), r, ints, dtype, nodes=nodes, weights=w)
        never = CP.c_evaluate(tab, opt, prio, np.full(J, 1e9), np.full(J, 5.0), r, ints, dtype, nodes=nodes, weights=w)
        assert (late >= wc).all() and (late > wc).any() and never.tobytes() == wc.tobytes()


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_absent_cells_score_inf(nodes, ints, released):
    """A candidate that gives a job an option it does not have (rt = +inf) scores +inf in the C port and the Python
    fold, on exactly the candidates the makespan oracle finds infeasible; every other candidate stays finite."""
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
    r = np.random.default_rng(20).uniform(0, 3000, size=J) if released else None
    w = _weights(J, 21)
    for dtype in (np.float32, np.float64):
        c = CP.c_evaluate(tab, opt, prio, d, p, r, ints, dtype, threads=8, nodes=nodes, weights=w)
        py = CP.evaluate(tab, opt, prio, d, p, r, ints, dtype, nodes=nodes, use_c=False, weights=w)
        mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, dtype, nodes=nodes)
        assert c.tobytes() == py.tobytes()
        assert np.array_equal(np.isinf(c), bad) and np.array_equal(np.isinf(mk), bad)
        assert np.isfinite(c[~bad]).all()


# the inputs of test_exact_edges.test_exact_reference_agrees_with_both_oracles, on which every term w e + p and every
# partial sum stays exact in fp32 with small integer and dyadic penalties
EDGE_CASES = [(1, 1, "equal", True), (2, 8, "zeros", False), (7, 3, "small", True), (31, 1, "dyadic", False),
              (33, 5, "equal", True), (128, 7, "zeros", True)]
PENALTIES = np.array([0.0, -0.0, 1.0, 2.0, 0.5, 8.0, 0.25])


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: "J%d-n%d-%s-%s" % (c[0], c[1], c[2], "int" if c[3] else "real"))
@pytest.mark.parametrize("rel", [None, "ready", "nonpos"])
@pytest.mark.parametrize("weighted", [False, True])
def test_exact_check_on_edge_inputs(case, rel, weighted):
    """On the tie-heavy and boundary inputs of test_exact_edges (equal, zero, -0.0 and dyadic runtimes; due dates at
    a completion, one step before it, -0.0, negative and beyond every completion; release dates at slot times and
    non-positive) fp32 rounds nothing: the fp32 C port and the float64 fold equal sum (w C + [C > d] p) in exact
    arithmetic, and the starts are ref_exact's."""
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
    c32, cst, _ = CP.c_evaluate(tab, opt, prio, d, p, r, ints, np.float32, want_plan=True, threads=8, nodes=nodes,
                                weights=w)
    s64 = CP.evaluate(tab, opt, prio, d, p, r, ints, np.float64, nodes=nodes, use_c=False, weights=w)
    _, xst, _ = X.batch(tab, opt, prio, r, ints, nodes, "makespan")
    for b in range(len(opt)):
        ex = CP.exact(tab, opt[b], prio[b], d, p, r, ints, nodes, weights=w)
        assert float(ex) == s64[b] == float(c32[b]), (b, ex, s64[b], c32[b])
        assert np.array_equal(xst[b], cst[b].astype(np.float64))


def test_on_time_at_the_due_date():
    """A job that completes exactly at its due date pays only its completion time; one unit later it pays the penalty
    too."""
    tab = np.full((1, 1, 8), 5.0, np.float32)
    o, pr = np.array([[7]], np.uint8), np.array([[0]], np.uint8)
    for dtype in (np.float32, np.float64):
        assert float(CP.c_evaluate(tab, o, pr, [5.0], [100.0], dtype=dtype)[0]) == 5.0
        assert float(CP.c_evaluate(tab, o, pr, [4.0], [100.0], dtype=dtype, weights=[3.0])[0]) == 115.0
    assert CP.exact(tab, o[0], pr[0], [5.0], [100.0]) == 5 and CP.exact(tab, o[0], pr[0], [4.0], [100.0]) == 105


def test_exact_refuses_a_sum_that_fp32_would_round():
    """exact() asserts that w e + p is exact in fp32: a penalty of 2^24 plus a completion of 5 is not."""
    tab = np.full((1, 1, 8), 5.0, np.float32)
    with pytest.raises(X.NotExact):
        CP.exact(tab, np.array([7], np.uint8), np.array([0], np.uint8), [4.0], [2.0 ** 24])


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "completion_penalty_cases.json")) as f:
        return json.load(f)["cases"]


def _check_milp(m, bf, name):
    if m["start"] is None:
        assert not m["proven_optimal"], name
        return 0
    assert m["feasible"] and m["overlaps"] == 0, name
    assert m["score"] == pytest.approx(m["objective_value"], rel=1e-6, abs=1e-6), name
    if m["proven_optimal"]:
        assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), name
        return 1
    assert bf <= m["score"] * (1 + 1e-9), name
    return 0


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum, for the instances' own due dates and
    penalties and for their cap variants; where HiGHS stopped at its time limit with an incumbent, the exhaustive
    optimum is no worse than it.  Every MILP plan is feasible and its score is its objective value, and the fp32 and
    fp64 optima agree (integer data).  The cap variant's optimum is the exhaustive minimum of sum w C under the cap,
    and the fixtures include weighted instances and instances with release dates."""
    proven = 0
    for rec in cases:
        for v in (rec, rec["cap"]):
            bf = v["bruteforce_f64"]["score"]
            assert v["bruteforce_f32"]["score"] == bf, rec["name"]
            proven += _check_milp(v["milp"], bf, rec["name"])
        assert rec["cap"]["bruteforce_f64"]["score"] == rec["cap"]["front_at_cap"], rec["name"]
    assert len(cases) == 24 and proven >= len(cases)
    assert sum(rec["weights"] is not None for rec in cases) >= 10
    assert sum(rec["release"] is not None for rec in cases) >= 4


def test_fixture_plans_and_fronts_rescore(cases):
    """The recorded optima re-derive from the oracle; every front is non-dominated (makespan ascending, sum strictly
    descending) and is the exhaustive front; the cap lies within it and P is a power of two above sum w * H."""
    for rec in cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        assert all(float(rt).is_integer() for t in tuples for _k, rt in t)
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        cap, P = rec["cap"]["cap"], rec["cap"]["P"]
        for v, d, p in ((rec, rec["due"], rec["penalty"]), (rec["cap"], [cap] * J, [P] * J)):
            for key, dtype in (("bruteforce_f64", np.float64), ("bruteforce_f32", np.float32)):
                b = v[key]
                got = CP.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), d, p,
                                  rec["release"], True, dtype, weights=rec["weights"])[0]
                assert float(got) == b["score"], (rec["name"], key)
        fr = rec["front"]
        assert all(a[0] < b[0] and a[1] > b[1] for a, b in zip(fr, fr[1:]))
        assert fr[0][0] <= cap <= fr[-1][0]
        assert math_pow2(P) and P >= (sum(rec["weights"]) if rec["weights"] else J) * (
            max([0.0] + (rec["release"] or [])) + sum(max(rt for _k, rt in t) for t in tuples))
        again = CP.front_brute_force(tab, optmap, [cap], rec["release"], True, weights=rec["weights"])
        assert again["front"] == fr and again["at_cap"] == [rec["cap"]["front_at_cap"]]


def math_pow2(x):
    m, _e = np.frexp(x)
    return m == 0.5


@pytest.mark.parametrize("seed", range(6))
def test_large_penalties_give_the_cap_constrained_completion(seed):
    """One due date H for every job and penalties above any sum w C: the completion-penalty optimum is the least
    sum w C among the plans whose makespan is <= H, and front_brute_force finds the same minimum."""
    rng = np.random.default_rng(400 + seed)
    J = 4
    tuples = [[(k, float(rng.integers(5, 60)) / k) for k in (1, 2, 4)] for _ in range(J)]
    tab, optmap = R.table_from_tuples(tuples)
    w = [float(x) for x in rng.choice([1.0, 2.0, 3.0], J)] if seed % 2 else None
    opts = np.array(np.meshgrid(*optmap, indexing="ij")).reshape(J, -1).T.astype(np.uint8)
    perms = np.array(list(itertools.permutations(range(J))), np.uint8)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    wc = CP.evaluate(tab, opt, prio, np.full(J, np.inf), np.zeros(J), None, True, np.float64, weights=w)
    mk = RR.c_evaluate(tab, opt, prio, np.zeros(J), True, np.float64)
    H = float(np.quantile(mk, 0.3))
    big = 1e7
    score = CP.evaluate(tab, opt, prio, np.full(J, H), np.full(J, big), None, True, np.float64, weights=w)
    i = int(np.argmin(score))
    assert mk[i] <= H and wc[i] == wc[mk <= H].min() and wc.max() < big
    assert CP.front_brute_force(tab, optmap, [H], weights=w)["at_cap"] == [wc[mk <= H].min()]


def test_lpt_seeds_are_the_completion_seeds():
    """lpt_seeds(objective="completion_penalty" / "weighted_completion_penalty") plants the SPT / WSPT seeds of
    "completion" / "weighted_completion", not EDD, on 1 and 3 nodes, with and without release dates."""
    from saturn_b200.search import lpt_seeds
    for nodes in (1, 3):
        for released in (False, True):
            rng = np.random.default_rng(5 + nodes)
            J = 64
            tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
            d = np.round(rng.uniform(0, 3, size=J)).astype(np.float32) * 1000
            r = rng.uniform(0, 500, size=J).astype(np.float32) if released else None
            w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32)
            for obj, base in (("completion_penalty", "completion"),
                              ("weighted_completion_penalty", "weighted_completion")):
                a = lpt_seeds(tmin, objective=obj, due=d, release=r, nodes=nodes, weights=w)
                b = lpt_seeds(tmin, objective=base, release=r, nodes=nodes, weights=w)
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


@pytest.mark.parametrize("kw,match", [
    ({"penalty": P3}, "needs due dates"),
    ({"due": D3}, "penalty=\\.\\.\\."),
    ({"due": D3, "penalty": [1.0, 2.0]}, "one value per task"),
    ({"due": D3, "penalty": [1.0, -1.0, 2.0]}, "finite and >= 0"),
    ({"due": D3, "penalty": [1.0, float("nan"), 2.0]}, "finite and >= 0"),
    ({"due": D3, "penalty": [1.0, 3e37, 2.0]}, "2\\^126"),
    ({"due": D3, "penalty": P3, "hysteresis": True}, "hysteresis"),
    ({"due": D3, "penalty": P3, "weights": [1.0, 0.0, 1.0]}, "finite and > 0"),
    ({"due": [1.0, float("nan"), 3.0], "penalty": P3}, "finite"),
    ({"due": D3, "penalty": P3, "release": [0.0, float("inf"), 1.0]}, None),
])
def test_solver_refusals_before_any_device_call(kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one),
    with the late penalty's rules."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective="completion_penalty", engine=object(), **kw)
    if "hysteresis" not in kw:
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [100.0, 60.0]
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective="completion_penalty", engine=object(), **kw)


@pytest.mark.parametrize("kw,match", [
    ({"points": 1}, "points >= 2"),
    ({"points": 0}, "points >= 2"),
    ({"points": 2.5}, "points >= 2"),
    ({"due": D3}, "no due"),
    ({"penalty": P3}, "no penalty"),
    ({"hysteresis": True}, "no hysteresis"),
    ({"presolved": (None,) * 6}, "no presolved"),
    ({"weights": [1.0, -1.0, 1.0]}, "finite and > 0"),
    ({"release": [0.0, float("nan"), 1.0]}, "finite"),
    ({"weights": [1e37, 1.0, 1.0]}, "2\\^126"),
])
def test_solve_front_refusals_before_any_device_call(kw, match):
    """solve_front refuses fewer than two points, the arguments it sets itself, bad weights or release dates, and
    weights whose penalty P would break sb_set_penalty's bound, before any device call."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve_front(tasks, engine=object(), **kw)
    with pytest.raises(TypeError):
        S.solve_front(tasks, engine=object(), objective="makespan")


def test_front_helpers_on_a_plan():
    """_plan_candidate recovers the exact list order from boa and the reduced opt bytes from bss / bna (several
    nodes: the node in bits 3 and up), and _device_makespan is max fp32(start + rt) over the fp32 table cells."""
    from saturn_b200 import solver as S
    tasks = [_Task("a", (100.0, 60.5)), _Task("b", (30.0, 20.0)), _Task("c", (7.0, 5.0))]
    T, _u, _o = S.build_table(tasks)
    position = [2, 0, 1]
    plan = S.plan_to_arrays([2, 2, 2], [1, 0, 0], [20.0, 0.0, 0.0], [0b11, 0b1, 0b100], position, nodes=2,
                            node_of=[1, 1, 0]) + (80.5,)
    opt, order = S._plan_candidate(tasks, plan, nodes=2)
    assert order.tolist() == [1, 2, 0] and opt.tolist() == [1 | 8, 0 | 8, 0]
    opt1, _ = S._plan_candidate(tasks, plan, nodes=1)
    assert opt1.tolist() == [1, 0, 0]
    assert S._device_makespan(tasks, plan, T) == 80.5


def test_completion_penalty_stats_and_set_objective():
    """The stats are float64 sums: every task's w C, plus the penalty of the late ones; _set_objective hands the
    penalties to the engine and picks the weighted form with weights."""
    from saturn_b200 import solver as S
    st = S._completion_penalty_stats([0.0, 10.0, 20.0], [3.0, 4.0, 5.0], [2.0, 1.0, 0.5], [5.0, 11.0, 25.0],
                                     [100.0, 7.0, 1.5])
    assert st == {"completion_penalty": 6.0 + 14.0 + 12.5 + 7.0, "weighted_completion": 6.0 + 14.0 + 12.5,
                  "late_tasks": 1, "penalty_paid": 7.0}
    assert S._completion_penalty_stats([0.0], [3.0], None, [3.0], [9.0])["completion_penalty"] == 3.0

    class Eng:
        def __init__(self):
            self.calls = []

        def __getattr__(self, name):
            return lambda *a, **k: self.calls.append(name)
    w = np.ones(3, np.float32)
    d = np.zeros(3, np.float32)
    p = np.ones(3, np.float32)
    e = Eng()
    assert S._set_objective(e, "completion_penalty", None, d, None, p) == "completion_penalty"
    assert "set_penalty" in e.calls and "set_due" in e.calls
    assert S._set_objective(Eng(), "completion_penalty", w, d, None, p) == "weighted_completion_penalty"


def test_engine_objective_table():
    """The completion-penalty pair has its own table, leaves the other tables as they are, carries its flags and
    per-job arrays, reads the penalties, needs due dates and penalties, and the name checks accept it."""
    from saturn_b200 import _lib
    from saturn_b200.engine import (COMPLETION_PENALTY_OBJECTIVES, OBJECTIVES, PENALTY_OBJECTIVES, _OBJECTIVES,
                                    _require_due, _require_penalty, objective_flag, objective_reads_penalty,
                                    objective_spec)
    from saturn_b200.solver import SolverError
    assert set(COMPLETION_PENALTY_OBJECTIVES) == {"completion_penalty", "weighted_completion_penalty"}
    assert not set(COMPLETION_PENALTY_OBJECTIVES) & set(_OBJECTIVES)
    assert len(_OBJECTIVES) == 14 and PENALTY_OBJECTIVES == ("late_penalty", "weighted_late_penalty")
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_COMPLETION_PENALTY
    assert objective_flag("completion_penalty") == base
    assert objective_flag("weighted_completion_penalty") == base | _lib.FLAG_WEIGHTED
    assert objective_spec("completion_penalty") == (base, False, True)
    assert objective_spec("weighted_completion_penalty") == (base | _lib.FLAG_WEIGHTED, True, True)
    for obj in COMPLETION_PENALTY_OBJECTIVES:
        assert objective_reads_penalty(obj)
        with pytest.raises(SolverError):
            _require_due(None, obj)
        with pytest.raises(SolverError, match="set_penalty"):
            _require_penalty(None, obj)
        _require_penalty(np.zeros(1, np.float32), obj)
    for obj in OBJECTIVES:
        _require_penalty(None, obj)
    with pytest.raises(SolverError, match="weighted_completion_penalty"):
        objective_spec("penalty")


def test_orchestrate_passes_penalties_through(monkeypatch):
    """orchestrate() shifts the due dates of objective="completion_penalty" with every interval and hands every solve
    the same `penalty` mapping."""
    from saturn_b200 import orchestrator as O

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
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "completion_penalty", "due": due,
                                                       "penalty": penalty})
    assert [n for n, _, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got_due, got_p) in enumerate(seen):
        assert obj == "completion_penalty" and got_due == {t: d - n * 1000 for t, d in due.items()}
        assert got_p == penalty


def test_flag_matches_the_header():
    """SB_FLAG_COMPLETION_PENALTY is 32768 in the header and in _lib, shares no bit with any other flag or test hook,
    and is in the hooks' static_assert; solve_front is exported from saturn_b200 but not from the saturn alias."""
    import saturn_b200
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_COMPLETION_PENALTY\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_COMPLETION_PENALTY == 32768
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_COMPLETION_PENALTY"]
    assert all(f & _lib.FLAG_COMPLETION_PENALTY == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_COMPLETION_PENALTY == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_COMPLETION_PENALTY" in f.read().split("the test hooks share no bit")[0]
    assert "solve_front" in saturn_b200.__all__ and saturn_b200.solve_front is saturn_b200.solver.solve_front
    with open(os.path.join(ROOT, "saturn", "solver", "__init__.py")) as f:
        assert "solve_front" not in f.read()
