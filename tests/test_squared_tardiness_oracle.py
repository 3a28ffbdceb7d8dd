"""CPU: the squared-tardiness objective (SB_FLAG_SQUARED, solve(objective="squared_tardiness" / "squared_flow")) in
the oracle — the Python schedule and fold against the C port (oracle/ref_squared_tardiness.c) bit for bit, the exact
check on the tie-heavy and boundary inputs of test_exact_edges, absent cells, the unit-weight, doubled-weight and
on-time identities, the MILP fixtures (tests/golden/squared_tardiness_cases.json, oracle/gen_squared_tardiness.py), the
seeds, solve() / solve_table() / orchestrate() handling without a device, and the flag against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_exact as X, ref_release as RR, ref_squared_tardiness as SQ

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
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    w = _weights(J, J + 3) if weighted else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = SQ.c_evaluate(tab, opt, prio, d, r, ints, dtype, want_plan=True, threads=8, nodes=nodes, weights=w)
        py, ps, pm = SQ.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True,
                                 weights=w)
        assert c.dtype == dtype and c.tobytes() == py.tobytes()
        assert np.array_equal(cs, ps) and np.array_equal(cm, pm)
        assert (c >= 0).all() and len(np.unique(c)) > 1


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
    r = np.random.default_rng(20).uniform(0, 3000, size=J) if released else None
    w = _weights(J, 21)
    for dtype in (np.float32, np.float64):
        c = SQ.c_evaluate(tab, opt, prio, d, r, ints, dtype, threads=8, nodes=nodes, weights=w)
        py = SQ.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, weights=w)
        mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, dtype, nodes=nodes)
        assert c.tobytes() == py.tobytes()
        assert np.array_equal(np.isinf(c), bad) and np.array_equal(np.isinf(mk), bad)
        assert np.isfinite(c[~bad]).all() and (c[~bad] > 0).any()


# the inputs of test_exact_edges.test_exact_reference_agrees_with_both_oracles whose squares and sums of squares stay
# exact in fp32 under every release family, with and without weights (the others square tardiness of hundreds in 1/8
# steps, or sum squares past 2^24, which fp32 rounds; exact() would refuse them)
EDGE_CASES = [(1, 1, "equal", True), (2, 8, "zeros", False), (7, 3, "small", True), (31, 1, "dyadic", False),
              (33, 5, "equal", True), (128, 7, "zeros", True)]


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: "J%d-n%d-%s-%s" % (c[0], c[1], c[2], "int" if c[3] else "real"))
@pytest.mark.parametrize("rel", [None, "ready", "nonpos"])
@pytest.mark.parametrize("weighted", [False, True])
def test_exact_check_on_edge_inputs(case, rel, weighted):
    """On the tie-heavy and boundary inputs of test_exact_edges (equal, zero, -0.0 and dyadic runtimes; due dates at
    a completion, one step before it, -0.0, negative and beyond every completion; release dates at slot times and
    non-positive) fp32 rounds nothing: the fp32 C port and the float64 fold equal sum w max(0, C - d)^2 in exact
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
    c32, cst, _ = SQ.c_evaluate(tab, opt, prio, d, r, ints, np.float32, want_plan=True, threads=8, nodes=nodes,
                                weights=w)
    s64 = SQ.evaluate(tab, opt, prio, d, r, ints, np.float64, nodes=nodes, use_c=False, weights=w)
    _, xst, _ = X.batch(tab, opt, prio, r, ints, nodes, "makespan")
    for b in range(len(opt)):
        ex = SQ.exact(tab, opt[b], prio[b], d, r, ints, nodes, weights=w)
        assert float(ex) == s64[b] == float(c32[b]), (b, ex, s64[b], c32[b])
        assert np.array_equal(xst[b], cst[b].astype(np.float64))


def test_exact_refuses_a_square_that_fp32_would_round():
    """exact() asserts that t * t is exact in fp32: a tardiness of 2^12 + 1 squares to 2^24 + 2^13 + 1, which is not."""
    tab = np.full((1, 1, 8), 4097.0, np.float32)
    with pytest.raises(X.NotExact):
        SQ.exact(tab, np.array([7], np.uint8), np.array([0], np.uint8), [0.0])


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_unit_doubled_weights_and_on_time(nodes, ints, released):
    """w = 1 gives exactly the unweighted fold and w = 2 exactly twice it; due dates at or past every completion give
    +0; d = 0 with unit weights gives the sum of fp32(C * C) in schedule order."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 300, nodes, seed=3)
    r = np.random.default_rng(4).uniform(-10, 3000, size=J) if released else None
    d = _due(J, 6, 6000.0)
    one = SQ.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.ones(J))
    two = SQ.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.full(J, 2.0))
    unit = SQ.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes)
    assert one.tobytes() == unit.tobytes() and two.tobytes() == (one * np.float32(2)).tobytes()
    assert (one > 0).all()
    _, start, _ = SQ.evaluate(tab, opt, prio, np.zeros(J), r, ints, np.float32, nodes=nodes, want_plan=True)
    rt = np.asarray(tab, np.float32)[np.arange(J)[None, :], 0 if nodes > 1 else opt >> 3, opt & 7]
    e = (start + rt).astype(np.float32)
    late = np.full(J, float(e.max()))                             # the latest fp32 completion
    zero = SQ.evaluate(tab, opt, prio, late, r, ints, np.float32, nodes=nodes, weights=_weights(J, 5))
    assert zero.tobytes() == np.zeros(len(opt), np.float32).tobytes()
    got = SQ.evaluate(tab, opt, prio, np.zeros(J), r, ints, np.float32, nodes=nodes)
    want = np.zeros(len(opt), np.float32)
    for i in range(J):
        x = e[np.arange(len(opt)), prio[:, i].astype(np.int64)]
        want = (want + (x * x).astype(np.float32)).astype(np.float32)
    assert got.tobytes() == want.tobytes()


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "squared_tardiness_cases.json")) as f:
        return json.load(f)["cases"]


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum to 1e-9 relative; where HiGHS stopped at
    its time limit with an incumbent, the exhaustive optimum is no worse than it.  Every MILP plan is feasible and its
    score is its objective value (the tangent cuts are exact on these integer instances), the fp32 and fp64 optima
    agree to fp32 rounding, and the fixtures include weighted instances, instances with release dates and squared-flow
    instances."""
    proven = 0
    for rec in cases:
        m, bf = rec["milp"], rec["bruteforce_f64"]["score"]
        assert rec["bruteforce_f32"]["score"] == pytest.approx(bf, rel=1e-6), rec["name"]
        if m["start"] is None:                       # stopped at the time limit before it found a plan
            assert not m["proven_optimal"], rec["name"]
            continue
        assert m["feasible"] and m["overlaps"] == 0, rec["name"]
        assert m["score"] == pytest.approx(m["objective_value"], rel=1e-6, abs=1e-6), rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), rec["name"]
        else:
            assert bf <= m["score"] * (1 + 1e-9), rec["name"]
    assert proven >= len(cases) // 2
    assert sum(rec["weights"] is not None and not rec["flow"] for rec in cases) >= 10
    assert sum(rec["release"] is not None for rec in cases) >= 4
    assert sum(rec["flow"] for rec in cases) >= 6


def test_fixture_plans_rescore_to_their_recorded_values(cases):
    """The recorded exhaustive optima and the tardiness-optimal flags re-derive from the oracle; every runtime is an
    integer; a squared-flow instance's due dates are max(r, 0)."""
    from oracle.gen_squared_tardiness import flow_due
    for rec in cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        assert all(float(rt).is_integer() for t in tuples for _k, rt in t)
        tab, optmap = R.table_from_tuples(tuples)
        for key, dtype in (("bruteforce_f64", np.float64), ("bruteforce_f32", np.float32)):
            b = rec[key]
            got = SQ.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), rec["due"],
                              rec["release"], True, dtype, weights=rec["weights"])[0]
            assert float(got) == b["score"], (rec["name"], key)
        best = rec["bruteforce_f64"]["score"]
        t = rec["tardiness_optimum"]
        assert t["is_optimal"] == (t["score"] <= best * (1 + 1e-9) + 1e-12) and t["score"] >= best * (1 - 1e-9)
        if rec["flow"]:
            assert rec["due"] == flow_due(len(tuples), rec["release"]) and best > 0


def test_lpt_seeds_are_the_tardiness_seeds():
    """lpt_seeds(objective="squared_tardiness" / "weighted_squared_tardiness") plants the EDD seeds of "tardiness" /
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
            for obj, base in (("squared_tardiness", "tardiness"), ("weighted_squared_tardiness", "weighted_tardiness")):
                a = lpt_seeds(tmin, objective=obj, due=d, release=r, nodes=nodes, weights=w)
                b = lpt_seeds(tmin, objective=base, due=d, release=r, nodes=nodes, weights=w)
                for (ca, oa), (cb, ob) in zip(a, b):
                    assert np.array_equal(ca, cb) and np.array_equal(oa, ob)


def test_squared_flow_seed_is_shortest_first_on_one_machine():
    """All jobs released at 0 on one machine (every job on all 8 GPUs): under squared_flow every due date is 0, so the
    EDD seed falls back to its runtime tie-break, shortest first, and that order's sum of C^2 is the exhaustive
    optimum (the adjacent-interchange argument of DESIGN.md)."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(21)
    for _ in range(8):
        J = 6
        p = rng.integers(1, 40, size=J).astype(np.float32)
        tab = np.full((J, 1, 8), np.inf, dtype=np.float32)
        tab[:, 0, 7] = p
        tmin = np.full((J, 8), np.inf, dtype=np.float32)
        tmin[:, 7] = p
        (ob, order), = lpt_seeds(tmin, objective="squared_tardiness", due=np.zeros(J, np.float32))[:1]
        assert np.array_equal(order, np.lexsort((np.arange(J), p)))
        best, _, _ = SQ.brute_force(tab, [[7]] * J, np.zeros(J))
        got = SQ.evaluate(tab, ob[None, :].astype(np.uint8), order[None, :].astype(np.uint8), np.zeros(J), None,
                          True, np.float64)
        assert float(got[0]) == best


class _Strat:
    def __init__(self, runtime, executor="x"):
        self.runtime, self.executor = runtime, executor


class _Task:
    def __init__(self, name, runtimes=(100.0, 60.0)):
        self.name = name
        self.strategies = {g: _Strat(rt) for g, rt in zip((1, 2), runtimes)}


@pytest.mark.parametrize("objective,kw,match", [
    ("squared_tardiness", {}, "needs due dates"),
    ("squared_tardiness", {"due": [1.0, 2.0]}, "one value per task"),
    ("squared_tardiness", {"due": [1.0, 2.0, 3.0], "hysteresis": True}, "hysteresis"),
    ("squared_tardiness", {"due": [1.0, 2.0, 3.0], "weights": [1.0, 0.0, 1.0]}, "finite and > 0"),
    ("squared_tardiness", {"due": [1.0, 2.0, 3.0], "weights": [1.0, 3.0e23, 1.0]}, "2\\^50"),
    ("squared_flow", {"due": [1.0, 2.0, 3.0]}, "takes no due dates"),
    ("squared_flow", {"hysteresis": True}, "hysteresis"),
    ("squared_flow", {"weights": [1.0, 2.0e23, 1.0]}, "2\\^50"),
    ("squared_flow", {"release": [0.0, float("inf"), 1.0]}, None),
])
def test_solver_refusals_before_any_device_call(objective, kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one): a
    missing or malformed `due`, `due` under squared_flow, hysteresis, a bad weight, weights past the overflow guard
    (3 tasks * 2e23 * 2^50 >= FLT_MAX), a bad release date."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective=objective, engine=object(), **kw)
    if "hysteresis" not in kw:  # solve_table has no hysteresis
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [100.0, 60.0]
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective=objective, engine=object(), **kw)


def test_overflow_guard_boundary():
    """The guard refuses J * max(w) * 2^50 >= FLT_MAX in float64 on the fp32 weights, and nothing below it: unit
    weights pass at any task count."""
    from saturn_b200 import solver as S
    fmax = float(np.finfo(np.float32).max)
    J = 3
    ok = float(np.float32(fmax / 2.0 ** 50 / J / 2))
    w64, w32 = S._resolve_weights([1.0, ok, 1.0], "squared_tardiness", J)
    assert w32.dtype == np.float32 and w64[1] == ok
    big = float(np.nextafter(np.float32(fmax / 2.0 ** 50 / J), np.float32(np.inf)))
    for obj in ("squared_tardiness", "squared_flow"):
        with pytest.raises(S.SolverError, match="2\\^50"):
            S._resolve_weights([1.0, big, 1.0], obj, J)
    S._resolve_weights([big, big, big], "tardiness", J)           # the other objectives have no such bound
    S._resolve_weights(np.ones(1 << 20), "squared_flow", 1 << 20)


def test_squared_flow_due_dates_and_stats():
    """squared_flow runs against max(r32, +0) (+0 without release dates), the due dates max_stretch builds; the stats
    are float64 sums of squares."""
    from saturn_b200 import solver as S
    r32 = np.array([-5.0, 0.0, 12.5, -0.0], np.float32)
    d = S._release_due(r32, 4)
    assert d.dtype == np.float32 and d.tolist() == [0.0, 0.0, 12.5, 0.0] and not np.signbit(d).any()
    assert S._release_due(None, 3).tolist() == [0.0, 0.0, 0.0]
    Tdev = np.full((4, 1, 8), np.inf, np.float32)
    Tdev[:, 0, 0] = [3.0, 4.0, 5.0, 6.0]
    assert S._stretch_form(Tdev, r32)[2].tolist() == d.tolist()
    st = S._squared_flow_stats([0.0, 10.0, 20.0], [3.0, 4.0, 5.0], [2.0, 1.0, 0.5], [-5.0, 0.0, 12.5])
    flow = [3.0, 14.0, 12.5]
    assert st["total_flow_time"] == sum(flow)
    assert st["squared_flow"] == 2.0 * 9.0 + 196.0 + 0.5 * 12.5 ** 2
    assert S._squared_flow_stats([1.0], [2.0], None, None) == {"squared_flow": 9.0, "total_flow_time": 3.0}
    sq = S._squared_stats([0.0, 10.0, 20.0], [3.0, 4.0, 5.0], None, [5.0, 11.0, 20.0])
    assert sq == {"squared_tardiness": 9.0 + 25.0, "weighted_tardiness": 8.0, "late_tasks": 2}

    class Eng:
        def __getattr__(self, name):
            return lambda *a, **k: None
    w = np.ones(3, np.float32)
    for obj in ("squared_tardiness", "squared_flow"):
        assert S._set_objective(Eng(), obj, None, d) == "squared_tardiness"
        assert S._set_objective(Eng(), obj, w, d) == "weighted_squared_tardiness"


def test_engine_objective_table():
    """The engine's table has both squared forms with their flags and per-job arrays; they need due dates, and the
    name check accepts them."""
    from saturn_b200 import _lib
    from saturn_b200.engine import SQUARED_OBJECTIVES, _OBJECTIVES, _require_due, objective_flag, objective_spec
    from saturn_b200.solver import SolverError
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_SQUARED
    assert objective_flag("squared_tardiness") == base
    assert objective_flag("weighted_squared_tardiness") == base | _lib.FLAG_WEIGHTED
    assert objective_spec("squared_tardiness") == (base, False, True)
    assert objective_spec("weighted_squared_tardiness") == (base | _lib.FLAG_WEIGHTED, True, True)
    assert set(SQUARED_OBJECTIVES) == {o for o, s in _OBJECTIVES.items() if s.flags & _lib.FLAG_SQUARED}
    for obj in SQUARED_OBJECTIVES:
        with pytest.raises(SolverError):
            _require_due(None, obj)
    with pytest.raises(SolverError, match="squared_tardiness"):
        objective_spec("squared")


@pytest.mark.parametrize("objective", ["squared_tardiness", "squared_flow"])
def test_orchestrate_shifts_due_and_release_dates(monkeypatch, objective):
    """orchestrate() hands the solve for interval n the due dates d - n * interval (squared_tardiness) and the release
    dates r - n * interval (both)."""
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
    release = {tasks[0]: 0.0, tasks[1]: 1500.0}
    due = {tasks[0]: 800.0, tasks[1]: 4000.0}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), kw["objective"], dict(kw["release"]), kw.get("due")))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
    kw = {"objective": objective, "release": release}
    if objective == "squared_tardiness":
        kw["due"] = due
    O.orchestrate(tasks, interval=1000, solver_kwargs=kw)
    assert [n for n, _, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got, got_due) in enumerate(seen):
        assert obj == objective and got == {t: r - n * 1000 for t, r in release.items()}
        if objective == "squared_tardiness":
            assert got_due == {t: d - n * 1000 for t, d in due.items()}
        else:
            assert got_due is None


def test_flag_squared_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_SQUARED\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_SQUARED == 8192
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_SQUARED"]
    assert all(f & _lib.FLAG_SQUARED == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_SQUARED == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_SQUARED" in f.read().split("the test hooks share no bit")[0]
