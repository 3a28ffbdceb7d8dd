"""CPU: the maximum-lateness objective (SB_FLAG_MAX_LATENESS, solve(objective="max_lateness")) in the oracle — the
Python schedule and tail fold against the C port (oracle/ref_max_lateness.c) bit for bit, the exact check on
tie-heavy inputs, d = c giving the makespan, shifted due dates giving the same scores, the exhaustive optimum against
Jackson's rule and against the MILP fixtures (tests/golden/max_lateness_cases.json, oracle/gen_max_lateness.py), the
seeds, solve() / solve_table() / orchestrate() handling without a device, and the flag against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_exact as X, ref_max_lateness as ML, ref_release as RR

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


@pytest.mark.parametrize("J,S,nodes,B", [(7, 3, 1, 30000), (40, 4, 1, 20000), (23, 1, 2, 60), (12, 1, 4, 60)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_python_fold_equals_c_port(J, S, nodes, B, ints, released):
    """The C port (schedule and tail fold in C) gives the same bits as the Python schedule with the numpy tail fold,
    scores, starts and slot masks, in fp32 and fp64: integer and real-valued starts, 1 to 4 nodes, with and without
    release dates (over 1e5 candidates in all)."""
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 7 * nodes)
    scale = 2000.0 * J / 8
    d = _due(J, J + 1, scale)
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = ML.c_evaluate(tab, opt, prio, d, r, ints, dtype, want_plan=True, threads=8, nodes=nodes)
        py, ps, pm = ML.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True)
        assert c.dtype == dtype and c.tobytes() == py.tobytes()
        assert np.array_equal(cs, ps) and np.array_equal(cm, pm)
        assert (c >= 0).all()
        if released:  # the tails matter: the fold is not the makespan's
            mk = RR.c_evaluate(tab, opt, prio, r, ints, dtype, nodes=nodes)
            assert (c != mk).any()


def _tie_heavy(J, seed):
    """Integer runtimes in {1, 2, 3} on a one-strategy table, integer due dates, some equal, some negative."""
    rng = np.random.default_rng(seed)
    tab = rng.integers(1, 4, size=(J, 1, 8)).astype(np.float32)
    opt = rng.integers(0, 8, size=(64, J)).astype(np.uint8)
    prio = np.argsort(rng.random((64, J)), axis=1).astype(np.uint8)
    d = rng.integers(-3, 2 * J, size=J).astype(np.float64)
    d[: J // 3] = d[0]
    return tab, opt, prio, d


@pytest.mark.parametrize("J", [1, 5, 16, 33])
@pytest.mark.parametrize("released", [False, True])
def test_exact_check_on_tie_heavy_inputs(J, released):
    """On integer data fp32 rounds nothing: the fp32 fold equals max(C + q) in exact arithmetic (starts from
    ref_exact), and subtracting D gives max(C - d)."""
    tab, opt, prio, d = _tie_heavy(J, J)
    r = np.random.default_rng(J + 1).integers(-2, J, size=J).astype(np.float64) if released else None
    got = ML.evaluate(tab, opt, prio, d, r, True, np.float32)
    _, D = ML.tails(d)
    for b in range(len(opt)):
        ex = ML.exact(tab, opt[b], prio[b], d, r)
        assert float(ex) == float(got[b]), b
        _, start, _ = X.schedule(tab, opt[b], prio[b], r)
        lmax = max(start[j] + int(tab[j, 0, opt[b, j] & 7]) - int(d[j]) for j in range(J))
        assert float(lmax) == float(got[b]) - D


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("c", [0.0, -17.5, 1234.0])
def test_equal_due_dates_give_the_makespan(nodes, ints, c):
    """d = c for every job: q = +0, and the tail fold is the makespan fold bit for bit."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 200, nodes, seed=3)
    r = np.random.default_rng(4).uniform(-10, 3000, size=J)
    for rel in (None, r):
        got = ML.evaluate(tab, opt, prio, np.full(J, c), rel, ints, np.float32, nodes=nodes)
        mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if rel is None else rel, ints, np.float32, nodes=nodes)
        assert got.tobytes() == mk.tobytes()


@pytest.mark.parametrize("shift", [1.0, -250.0, 4096.0])
def test_shifted_due_dates_give_the_same_scores(shift):
    """Integer due dates shifted by an integer: the tails, hence every score, are unchanged."""
    J = 40
    tab, opt, prio = _candidates(J, 4, 500, 1, seed=9)
    d = _due(J, 10, 5000.0, integer=True)
    a = ML.evaluate(tab, opt, prio, d, None, True, np.float32)
    b = ML.evaluate(tab, opt, prio, d + shift, None, True, np.float32)
    assert a.tobytes() == b.tobytes()
    assert np.array_equal(ML.tails(d)[0], ML.tails(d + shift)[0])


def test_exhaustive_optimum_on_one_gpu_count_is_jacksons_rule():
    """With every job on all 8 GPUs (one machine), EDD order is optimal for L_max (Jackson's rule): the exhaustive
    optimum equals the EDD schedule's L_max, and it can be negative."""
    rng = np.random.default_rng(11)
    bests = []
    for _ in range(6):
        J = 5
        tab = np.full((J, 1, 8), np.inf, dtype=np.float32)
        tab[:, 0, 7] = rng.integers(1, 20, size=J)
        d = rng.integers(5, 60, size=J).astype(np.float64)
        best, _, _ = ML.brute_force(tab, [[7]] * J, d)
        edd = np.argsort(d, kind="stable").astype(np.uint8)
        c = np.cumsum(tab[edd, 0, 7].astype(np.float64))
        assert best == float(np.max(c - d[edd]))
        bests.append(best)
    assert min(bests) < 0 < max(bests)


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "max_lateness_cases.json")) as f:
        return json.load(f)["cases"]


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum to 1e-9; where HiGHS stopped at its
    time limit, the exhaustive optimum is no worse than the incumbent.  Every MILP plan is feasible, its L_max is its
    objective value, and the fixtures include instances with L_max* < 0 (tardiness flat at zero) and with release
    dates."""
    proven = 0
    for rec in cases:
        m, bf = rec["milp"], rec["bruteforce_f64"]["score"]
        assert m["start"] is not None and m["feasible"] and m["overlaps"] == 0, rec["name"]
        assert m["score"] == pytest.approx(m["objective_value"], abs=1e-6), rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), rec["name"]
        else:
            assert bf <= m["score"] + 1e-9, rec["name"]
    assert proven >= len(cases) // 2
    assert sum(rec["bruteforce_f64"]["score"] < 0 for rec in cases) >= 4
    assert sum(rec["release"] is not None for rec in cases) >= 4


def test_fixture_plans_rescore_to_their_recorded_lateness(cases):
    """The recorded exhaustive optimum and the tardiness- and makespan-optimal flags re-derive from the oracle."""
    for rec in cases:
        tab, optmap = R.table_from_tuples([[tuple(x) for x in t] for t in rec["gpu_time_tuples"]])
        b = rec["bruteforce_f64"]
        got = ML.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), rec["due"],
                          rec["release"], True, np.float64)[0] - ML.tails(rec["due"], np.float64)[1]
        assert got == pytest.approx(b["score"], abs=1e-9)
        for k in ("tardiness_optimum", "makespan_optimum"):
            assert rec[k]["is_lmax_optimal"] == (rec[k]["max_lateness"] <= b["score"] + 1e-9)
            assert rec[k]["max_lateness"] >= b["score"] - 1e-9


def test_max_lateness_seeds_are_the_tardiness_seeds():
    """lpt_seeds(objective="max_lateness") plants the unit-weight EDD orders of "tardiness", re-sorted by release."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(5)
    J = 48
    tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
    d = rng.integers(0, 5, size=J).astype(np.float32) * 100
    r = rng.integers(0, 3, size=J).astype(np.float32) * 50
    for rel in (None, r):
        a = lpt_seeds(tmin, objective="max_lateness", due=d, release=rel, nodes=2)
        b = lpt_seeds(tmin, objective="tardiness", due=d, release=rel, nodes=2)
        for (ca, oa), (cb, ob) in zip(a, b):
            assert np.array_equal(ca, cb) and np.array_equal(oa, ob)
    with pytest.raises(ValueError):
        lpt_seeds(tmin, objective="max_lateness")


class _Task:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("kw", [
    {},                                                     # no due dates
    {"due": [1.0, 2.0]},                                    # wrong length
    {"due": [1.0, float("nan"), 2.0]},
    {"due": [1.0, 2.0 ** 24, 2.0]},
    {"due": [-2.0 ** 23 - 1, 0.0, 2.0 ** 23]},              # spread >= 2^24
    {"due": [1.0, 2.0, 3.0], "weights": [1.0, 1.0, 1.0]},
    {"due": [1.0, 2.0, 3.0], "hysteresis": True},
    {"due": [1.0, 2.0, 3.0], "release": [0.0, float("inf"), 1.0]},
    {"due": "abc"},
])
def test_solver_refusals_before_any_device_call(kw):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one)."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="max_lateness", engine=object(), **kw)
    if kw and "hysteresis" not in kw:  # solve_table has no hysteresis
        T = np.ones((3, 1, 8), dtype=np.float32)
        with pytest.raises(S.SolverError):
            S.solve_table(T, objective="max_lateness", engine=object(), **kw)
    with pytest.raises(S.SolverError, match="no entry"):
        S.solve(tasks, None, objective="max_lateness", due={tasks[0]: 1.0}, engine=object())


def test_horizon_guard_counts_the_tails():
    """The pre-check refuses a table whose tail makespan bound max_t (min_k rt + q_t) reaches 2^24, even when the
    makespan bound alone would pass."""
    from saturn_b200 import solver as S
    T = np.ones((3, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError, match="2\\^24"):
        S.solve_table(T, objective="max_lateness", due=[2.0 ** 24 - 1, 0.5, 0.0], engine=object())


def test_engine_objective_flag():
    from saturn_b200 import _lib
    from saturn_b200.engine import OBJECTIVES, _require_due, objective_flag
    from saturn_b200.solver import SolverError
    assert "max_lateness" in OBJECTIVES and objective_flag("max_lateness") == _lib.FLAG_MAX_LATENESS
    with pytest.raises(SolverError):
        _require_due(None, "max_lateness")


def test_orchestrate_shifts_due_dates_under_max_lateness(monkeypatch):
    """orchestrate() hands the solve for interval n the due dates d - n * interval under objective="max_lateness"."""
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
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "max_lateness", "due": due})
    assert [n for n, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got) in enumerate(seen):
        assert obj == "max_lateness" and got == {t: d - n * 1000 for t, d in due.items()}


def test_flag_max_lateness_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_MAX_LATENESS\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_MAX_LATENESS == 1024
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_MAX_LATENESS"]
    assert all(f & _lib.FLAG_MAX_LATENESS == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_MAX_LATENESS == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_MAX_LATENESS" in f.read().split("the test hooks share no bit")[0]
