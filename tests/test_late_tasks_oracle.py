"""CPU: the late-count objective (SB_FLAG_LATE_COUNT, solve(objective="late_tasks")) in the oracle — the Python
schedule and count fold against the C port (oracle/ref_late_tasks.c) bit for bit, the exact check on tie-heavy inputs
with completions on their due dates, the boundary due dates, doubled weights, the Moore-Hodgson seeds against the
exhaustive optimum and against their restatement, the MILP fixtures (tests/golden/late_tasks_cases.json,
oracle/gen_late_tasks.py), solve() / solve_table() / orchestrate() handling without a device, and the flag against
the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_exact as X, ref_late_tasks as LT

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


def _due(J, seed, scale, integer=False):
    d = np.random.default_rng(seed).uniform(-0.3, 1.2, size=J) * scale
    return np.round(d) if integer else d


def _weights(J, seed):
    return np.random.default_rng(seed).choice([0.25, 0.5, 1.0, 1.5, 3.0, 7.0, 0.1], size=J)


@pytest.mark.parametrize("J,S,nodes,B", [(7, 3, 1, 30000), (40, 4, 1, 20000), (23, 1, 2, 60), (12, 1, 4, 60)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_python_fold_equals_c_port(J, S, nodes, B, ints, released, weighted):
    """The C port (schedule and count fold in C) gives the same bits as the Python schedule with the numpy fold,
    scores, starts and slot masks, in fp32 and fp64: integer and real-valued starts, 1 to 4 nodes, with and without
    release dates, unit and real weights (over 1e5 candidates in all)."""
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 7 * nodes)
    scale = 2000.0 * J / 8
    d = _due(J, J + 1, scale)
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    w = _weights(J, J + 3) if weighted else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = LT.c_evaluate(tab, opt, prio, d, r, ints, dtype, want_plan=True, threads=8, nodes=nodes, weights=w)
        py, ps, pm = LT.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True,
                                 weights=w)
        assert c.dtype == dtype and c.tobytes() == py.tobytes()
        assert np.array_equal(cs, ps) and np.array_equal(cm, pm)
        assert (c >= 0).all() and len(np.unique(c)) > 1


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_absent_cells_score_inf(nodes, ints, released):
    """A candidate that gives a job an option it does not have (rt = +inf) is infeasible: the C port and the Python
    fold both score it +inf, on the same candidates as the makespan oracle, and every other candidate keeps its
    finite count, which is not changed by the absent cells of other candidates."""
    from oracle import ref_release as RR
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
        c = LT.c_evaluate(tab, opt, prio, d, r, ints, dtype, threads=8, nodes=nodes, weights=w)
        py = LT.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, weights=w)
        mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, dtype, nodes=nodes)
        assert c.tobytes() == py.tobytes()
        assert np.array_equal(np.isinf(c), bad) and np.array_equal(np.isinf(mk), bad)
        assert np.isfinite(c[~bad]).all() and (c[~bad] > 0).any()


def _tie_heavy(J, seed, released):
    """Integer runtimes in {1, 2, 3} on a one-strategy table; due dates set to the completions of candidate 0 for a
    third of the jobs (C = d exactly there), the rest integers, some equal, some negative."""
    rng = np.random.default_rng(seed)
    tab = rng.integers(1, 4, size=(J, 1, 8)).astype(np.float32)
    opt = rng.integers(0, 8, size=(64, J)).astype(np.uint8)
    prio = np.argsort(rng.random((64, J)), axis=1).astype(np.uint8)
    r = rng.integers(-2, J, size=J).astype(np.float64) if released else None
    d = rng.integers(-3, 2 * J, size=J).astype(np.float64)
    _, start, _ = X.schedule(tab, opt[0], prio[0], r)
    on = rng.permutation(J)[: max(1, J // 3)]
    for j in on:
        d[j] = float(start[j] + int(tab[j, 0, opt[0, j] & 7]))
    return tab, opt, prio, d, r, on


@pytest.mark.parametrize("J", [1, 5, 16, 33])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_exact_check_on_tie_heavy_inputs(J, released, weighted):
    """On integer data fp32 rounds nothing: the fp32 fold equals sum w [C > d] in exact arithmetic (starts from
    ref_exact), and a job that completes exactly at its due date is on time."""
    tab, opt, prio, d, r, on = _tie_heavy(J, J, released)
    w = np.random.default_rng(J).integers(1, 5, size=J).astype(np.float64) if weighted else None
    got = LT.evaluate(tab, opt, prio, d, r, True, np.float32, weights=w)
    for b in range(len(opt)):
        assert float(LT.exact(tab, opt[b], prio[b], d, r, weights=w)) == float(got[b]), b
    # candidate 0 completes the jobs of `on` exactly at their due dates: they do not count
    _, start, _ = X.schedule(tab, opt[0], prio[0], r)
    late = [j for j in range(J) if start[j] + int(tab[j, 0, opt[0, j] & 7]) > d[j]]
    assert not set(late) & set(on.tolist())
    wj = np.ones(J) if w is None else w
    assert float(got[0]) == float(sum(wj[j] for j in late))


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_boundary_due_dates_and_doubled_weights(nodes, ints, released):
    """Due dates at or past every completion give +0; due dates below every completion give sum w; w = 2 gives
    exactly twice w = 1."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 300, nodes, seed=3)
    r = np.random.default_rng(4).uniform(-10, 3000, size=J) if released else None
    w = _weights(J, 5)
    _, start, _ = LT.evaluate(tab, opt, prio, np.zeros(J), r, ints, np.float32, nodes=nodes, want_plan=True)
    rt = np.asarray(tab, np.float32)[np.arange(J)[None, :], 0 if nodes > 1 else opt >> 3, opt & 7]
    late = np.full(J, float((start + rt).astype(np.float32).max()))  # the latest fp32 completion
    zero = LT.evaluate(tab, opt, prio, late, r, ints, np.float32, nodes=nodes, weights=w)
    assert zero.tobytes() == np.zeros(len(opt), np.float32).tobytes()
    below = np.full(J, -1.0)
    allw = LT.evaluate(tab, opt, prio, below, r, ints, np.float32, nodes=nodes, weights=w)
    assert np.all(allw == LT.fold(tab, opt, prio, np.zeros_like(start), below, np.float32, nodes, w))
    assert np.all(LT.evaluate(tab, opt, prio, below, r, ints, np.float32, nodes=nodes) == np.float32(J))
    d = _due(J, 6, 6000.0)
    one = LT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.ones(J))
    two = LT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.full(J, 2.0))
    unit = LT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes)
    assert two.tobytes() == (one * np.float32(2)).tobytes() and one.tobytes() == unit.tobytes()


def test_moore_hodgson_seed_is_optimal_on_one_machine():
    """With every job on all 8 GPUs (one machine), one node and unit weights, the repaired EDD order is
    Moore-Hodgson's algorithm: its count equals the exhaustive optimum."""
    rng = np.random.default_rng(11)
    counts = []
    for _ in range(12):
        J = 6
        tab = np.full((J, 1, 8), np.inf, dtype=np.float32)
        tab[:, 0, 7] = rng.integers(1, 20, size=J)
        d = rng.integers(5, 50, size=J).astype(np.float64)
        best, _, _ = LT.brute_force(tab, [[7]] * J, d)
        edd = np.lexsort((np.arange(J), tab[:, 0, 7], d))
        seq = LT.moore_hodgson_seed(edd, [8] * J, tab[:, 0, 7], d)
        got = LT.evaluate(tab, np.full((1, J), 7, np.uint8), np.array([seq], np.uint8), d, None, True, np.float64)
        assert float(got[0]) == best
        counts.append(best)
    assert min(counts) < max(counts) and max(counts) > 0


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("objective", ["late_tasks", "weighted_late_tasks"])
@pytest.mark.parametrize("ints", [True, False])
def test_lpt_seeds_repair_the_tardiness_seeds(nodes, released, objective, ints):
    """lpt_seeds(objective="late_tasks" / "weighted_late_tasks") plants the options and node fill of the tardiness
    seeds, with each order repaired as oracle.ref_late_tasks.moore_hodgson_seed restates it; the repair moves jobs."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(5 + nodes)
    J = 64
    tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
    d = rng.uniform(0, 3000, size=J).astype(np.float32)
    r = rng.uniform(0, 500, size=J).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32)
    base = "weighted_tardiness" if objective.startswith("weighted") else "tardiness"
    a = lpt_seeds(tmin, objective=objective, due=d, release=r, nodes=nodes, weights=w, integer_starts=ints)
    b = lpt_seeds(tmin, objective=base, due=d, release=r, nodes=nodes, weights=w, integer_starts=ints)
    moved = 0
    usable = np.where(tmin < 1.0e6, tmin, np.inf)
    rel = None if r is None else (np.ceil(r) if ints else r)
    for (ca, oa), (cb, ob) in zip(a, b):
        assert np.array_equal(ca, cb) and sorted(oa.tolist()) == list(range(J))
        col = ca & 7
        want = LT.moore_hodgson_seed(ob, col.astype(int) + 1, usable[np.arange(J), col], d,
                                     node=ca >> 3 if nodes > 1 else None, nodes=nodes,
                                     weights=w if objective.startswith("weighted") else None, release=rel,
                                     integer_starts=ints)
        assert oa.tolist() == want
        moved += int((oa != ob).any())
    assert moved > 0


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "late_tasks_cases.json")) as f:
        return json.load(f)["cases"]


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum to 1e-9; where HiGHS stopped at its
    time limit, the exhaustive optimum is no worse than the incumbent.  Every MILP plan is feasible, its count is its
    objective value, the fp32 and fp64 optima agree, and the fixtures include weighted instances and instances with
    release dates."""
    proven = 0
    for rec in cases:
        m, bf = rec["milp"], rec["bruteforce_f64"]["score"]
        assert m["start"] is not None and m["feasible"] and m["overlaps"] == 0, rec["name"]
        assert m["score"] == pytest.approx(m["objective_value"], abs=1e-6), rec["name"]
        assert rec["bruteforce_f32"]["score"] == bf, rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), rec["name"]
        else:
            assert bf <= m["score"] + 1e-9, rec["name"]
    assert proven >= len(cases) // 2
    assert sum(rec["weights"] is not None for rec in cases) >= 10
    assert sum(rec["release"] is not None for rec in cases) >= 4
    assert sum(not rec["tardiness_optimum"]["is_count_optimal"] for rec in cases) >= len(cases) // 2


def test_fixture_plans_rescore_to_their_recorded_counts(cases):
    """The recorded exhaustive optimum and the tardiness-, L_max- and makespan-optimal flags re-derive from the
    oracle."""
    for rec in cases:
        tab, optmap = R.table_from_tuples([[tuple(x) for x in t] for t in rec["gpu_time_tuples"]])
        b = rec["bruteforce_f64"]
        got = LT.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), rec["due"],
                          rec["release"], True, np.float64, weights=rec["weights"])[0]
        assert got == pytest.approx(b["score"], abs=1e-9)
        if rec["due_qualifies"]:
            assert b["score"] > 0 and not rec["tardiness_optimum"]["is_count_optimal"]
        for k in ("tardiness_optimum", "max_lateness_optimum", "makespan_optimum"):
            assert rec[k]["is_count_optimal"] == (rec[k]["late"] <= b["score"] + 1e-9)
            assert rec[k]["late"] >= b["score"] - 1e-9


class _Task:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("kw", [
    {},                                                     # no due dates
    {"due": [1.0, 2.0]},                                    # wrong length
    {"due": [1.0, float("nan"), 2.0]},
    {"due": [1.0, 2.0 ** 24, 2.0]},
    {"due": [1.0, 2.0, 3.0], "weights": [1.0, 0.0, 1.0]},
    {"due": [1.0, 2.0, 3.0], "weights": [1.0, 1e-46, 1.0]},  # > 0, but 0 in fp32
    {"due": [1.0, 2.0, 3.0], "weights": [1.0, 1.0]},
    {"due": [1.0, 2.0, 3.0], "hysteresis": True},
    {"due": [1.0, 2.0, 3.0], "release": [0.0, float("inf"), 1.0]},
    {"due": "abc"},
])
def test_solver_refusals_before_any_device_call(kw):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one)."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="late_tasks", engine=object(), **kw)
    if kw and "hysteresis" not in kw:  # solve_table has no hysteresis
        T = np.ones((3, 1, 8), dtype=np.float32)
        with pytest.raises(S.SolverError):
            S.solve_table(T, objective="late_tasks", engine=object(), **kw)
    with pytest.raises(S.SolverError, match="no entry"):
        S.solve(tasks, None, objective="late_tasks", due={tasks[0]: 1.0}, engine=object())


@pytest.mark.parametrize("objective", ["makespan", "max_lateness"])
def test_weights_and_due_refused_under_other_objectives(objective):
    """`due` belongs to the due-date objectives and `weights` to completion, tardiness and the late count."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective=objective, due=[1.0, 2.0, 3.0], weights=[1.0, 1.0, 1.0], engine=object())
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="completion", due=[1.0, 2.0, 3.0], engine=object())


def test_engine_objective_flags():
    from saturn_b200 import _lib
    from saturn_b200.engine import OBJECTIVES, _require_due, objective_flag
    from saturn_b200.solver import SolverError
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_LATE_COUNT
    assert objective_flag("late_tasks") == base
    assert objective_flag("weighted_late_tasks") == base | _lib.FLAG_WEIGHTED
    assert {"late_tasks", "weighted_late_tasks"} <= set(OBJECTIVES)
    for obj in ("late_tasks", "weighted_late_tasks"):
        with pytest.raises(SolverError):
            _require_due(None, obj)


def test_set_objective_picks_the_weighted_count():
    from saturn_b200 import solver as S

    class Eng:
        def __getattr__(self, name):
            return lambda *a, **k: None
    d32 = np.zeros(3, np.float32)
    assert S._set_objective(Eng(), "late_tasks", None, d32) == "late_tasks"
    assert S._set_objective(Eng(), "late_tasks", np.ones(3, np.float32), d32) == "weighted_late_tasks"
    stats = S._late_count_stats([0.0, 5.0, 1.0], [2.0, 1.0, 1.0], [1.0, 3.0, 0.5], [2.0, 5.0, 1.5])
    assert stats == {"weighted_tardiness": 3.0 + 0.25, "late_tasks": 2, "weighted_late_tasks": 3.5}


def test_orchestrate_shifts_due_dates_under_late_tasks(monkeypatch):
    """orchestrate() hands the solve for interval n the due dates d - n * interval under objective="late_tasks"."""
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
    due = {tasks[0]: 700.0, tasks[1]: 2500.0}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), kw["objective"], dict(kw["due"])))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "late_tasks", "due": due})
    assert [n for n, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got) in enumerate(seen):
        assert obj == "late_tasks" and got == {t: d - n * 1000 for t, d in due.items()}


def test_flag_late_count_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_LATE_COUNT\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_LATE_COUNT == 2048
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_LATE_COUNT"]
    assert all(f & _lib.FLAG_LATE_COUNT == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_LATE_COUNT == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_LATE_COUNT" in f.read().split("the test hooks share no bit")[0]
