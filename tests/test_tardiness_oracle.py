"""CPU: the weighted tardiness (SB_FLAG_DUE) in the oracle — the Python fold against its C port bit for bit, the
identities against the completion folds, the tardiness MILP fixtures (tests/golden/tardiness_cases.json,
oracle/gen_tardiness.py), the dominance of list schedules on their plans, solve() / solve_table() / orchestrate()
due-date handling without a device, and the flag's value against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_completion as RC, ref_eval as R, ref_tardiness as RT, ref_weighted as RW

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def tardiness_cases():
    with open(os.path.join(HERE, "golden", "tardiness_cases.json")) as f:
        return json.load(f)["cases"]


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


def _due(tab, opt, prio, nodes, seed):
    """Real due dates spread over the candidates' completions, some negative: a mix of late and early jobs."""
    horizon = float(RW.c_evaluate(tab, opt[:1], prio[:1], True, np.float64, nodes=nodes, weights=np.ones(
        opt.shape[1]))[0]) / max(1, opt.shape[1])
    return np.random.default_rng(seed).uniform(-0.2, 2.5, size=opt.shape[1]) * horizon


@pytest.mark.parametrize("J,S,nodes", [(1, 1, 1), (7, 3, 1), (40, 4, 1), (300, 2, 1), (23, 1, 2), (64, 1, 3),
                                       (9, 1, 4)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("weighted", [False, True])
def test_python_fold_equals_c_port(J, S, nodes, ints, dtype, weighted):
    """e = s + rt, l = e - d, t = max(l, +0), acc = acc + (w * t), each step rounded, gives the same bits in Python
    and in C, fp32 and fp64, on one node and on several, with integer and real-valued starts, unit and random
    real weights."""
    B = 48
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 3 * nodes)
    d = _due(tab, opt, prio, nodes, seed=J)
    w = np.random.default_rng(J + 1).uniform(0.05, 20.0, size=J) if weighted else None
    tot = RT.c_evaluate(tab, opt, prio, d, ints, dtype, nodes=nodes, weights=w)
    wd = np.ones(J, dtype) if w is None else w.astype(dtype)
    dd = d.astype(dtype)
    assert (tot > 0).any()
    for b in range(B):
        got, start, _, _ = RT.list_schedule(tab, opt[b], prio[b], d, ints, dtype, nodes=nodes, weights=w)
        assert dtype(got).tobytes() == tot[b].tobytes()
        acc = dtype(0.0)
        for j in prio[b]:
            e = dtype(dtype(start[j]) + dtype(tab[j][0 if nodes > 1 else opt[b][j] >> 3][opt[b][j] & 7]))
            acc = dtype(acc + dtype(wd[j] * max(dtype(e - dd[j]), dtype(0.0))))
        assert acc == tot[b]
    if nodes == 1:
        assert np.array_equal(RT.list_schedule_batch(tab, opt, prio, d, ints, dtype, weights=w), tot)


@pytest.mark.parametrize("ints", [True, False])
def test_c_port_at_scale(ints):
    """About 1e5 candidates: the C fold equals the vectorised Python fold bit for bit in fp32 and fp64."""
    J, B = 48, 100_000
    tab, opt, prio = _candidates(J, 3, B, 1, seed=77)
    d = _due(tab, opt, prio, 1, seed=78)
    w = np.random.default_rng(79).uniform(0.05, 20.0, size=J)
    for dt in (np.float32, np.float64):
        c = RT.c_evaluate(tab, opt, prio, d, ints, dt, weights=w, threads=8)
        py = RT.list_schedule_batch(tab, opt, prio, d, ints, dt, weights=w)
        assert np.array_equal(c, py)


@pytest.mark.parametrize("J,S,nodes", [(40, 4, 1), (300, 2, 1), (64, 1, 3)])
def test_identities(J, S, nodes):
    """d = 0 gives the weighted-completion fold, and with unit weights the unweighted one, bit for bit; due dates at
    or past every completion give +0; w = 2 gives exactly twice w = 1."""
    B = 256
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J)
    w = np.random.default_rng(J).uniform(0.05, 20.0, size=J)
    d = _due(tab, opt, prio, nodes, seed=J + 1)
    zero = np.zeros(J)
    for ints in (True, False):
        for dt in (np.float32, np.float64):
            assert RT.c_evaluate(tab, opt, prio, zero, ints, dt, nodes=nodes).tobytes() == \
                RC.c_evaluate(tab, opt, prio, ints, dt, nodes=nodes).tobytes()
            assert RT.c_evaluate(tab, opt, prio, zero, ints, dt, nodes=nodes, weights=w).tobytes() == \
                RW.c_evaluate(tab, opt, prio, ints, dt, nodes=nodes, weights=w).tobytes()
            loose = RT.c_evaluate(tab, opt, prio, np.full(J, 2.0 ** 24 - 1), ints, dt, nodes=nodes, weights=w)
            assert (loose == 0).all() and not np.signbit(loose).any()
            one = RT.c_evaluate(tab, opt, prio, d, ints, dt, nodes=nodes)
            two = RT.c_evaluate(tab, opt, prio, d, ints, dt, nodes=nodes, weights=np.full(J, 2.0))
            assert two.tobytes() == (one * dt(2)).astype(dt).tobytes()
            py = [RT.list_schedule(tab, opt[b], prio[b], zero, ints, dt, nodes=nodes)[0] for b in range(8)]
            assert np.array_equal(np.array(py, dtype=dt), RC.c_evaluate(tab, opt[:8], prio[:8], ints, dt, nodes=nodes))


def test_tardiness_fixtures_match_the_milp(tardiness_cases):
    """On every instance HiGHS proved optimal the exhaustive fp64 optimum equals the tardiness MILP's optimum (1e-9
    relative); on a time-limited one it is no worse than the MILP's incumbent.  The MILP's plans are feasible; the
    weights and due dates are exact in fp32; half the instances have unit weights; the recorded facts hold."""
    assert len(tardiness_cases) >= 18
    assert sum(r["weights"] is None for r in tardiness_cases) == len(tardiness_cases) // 2
    proven = 0
    for rec in tardiness_cases:
        w, d = rec["weights"], rec["due"]
        assert w is None or all(float(np.float32(x)) == x and x > 0 for x in w)
        assert all(float(np.float32(x)) == x and x == int(x) for x in d)
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        bf = rec["bruteforce_f64"]["weighted_tardiness"]
        again = RT.list_schedule(tab, rec["bruteforce_f64"]["opt"], rec["bruteforce_f64"]["prio"], d, True,
                                 np.float64, weights=w)[0]
        assert again == bf, rec["name"]
        f32 = RT.list_schedule(tab, rec["bruteforce_f32"]["opt"], rec["bruteforce_f32"]["prio"], d, True, np.float32,
                               weights=w)[0]
        assert f32 == rec["bruteforce_f32"]["weighted_tardiness"] and f32 == pytest.approx(bf, rel=1e-6)
        assert rec["positive"] == (bf > 0)
        assert rec["differs"] == (rec["completion_optimum_tardiness"] > bf * (1 + 1e-12))
        m = rec["milp"]
        if m["start"] is None:
            continue
        assert m["feasible"] and m["overlaps"] == 0, rec["name"]
        J = len(tuples)
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        assert R.check_plan(m["start"], m["mask"], rt, k)[0]
        if m["proven_optimal"]:
            proven += 1
            assert bf == pytest.approx(m["weighted_tardiness"], rel=1e-9, abs=1e-9), rec["name"]
            assert m["objective_value"] == pytest.approx(m["weighted_tardiness"], rel=1e-6, abs=1e-6), rec["name"]
        else:
            assert bf <= m["weighted_tardiness"] * (1 + 1e-9), rec["name"]
    assert proven >= 15
    assert sum(r["positive"] and r["differs"] for r in tardiness_cases) >= len(tardiness_cases) // 2


def test_list_schedules_dominate_the_tardiness_milp_plans(tardiness_cases):
    """DESIGN.md §3.1: ordering a feasible plan's jobs by start and running the list rule with its options finishes
    every job no later, so the weighted tardiness (non-decreasing in every completion) does not grow."""
    n = 0
    for rec in tardiness_cases:
        m = rec["milp"]
        if m["start"] is None:
            continue
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        opt = [optmap[t][m["opt_idx"][t]] for t in range(J)]
        order = sorted(range(J), key=lambda t: (m["start"][t], t))
        score, start, _, _ = RT.list_schedule(tab, opt, order, rec["due"], True, np.float64, weights=rec["weights"])
        for t in range(J):
            assert start[t] <= m["start"][t] + 1e-9, (rec["name"], t)
        assert score <= m["weighted_tardiness"] * (1 + 1e-12) + 1e-9
        n += 1
    assert n >= 15


class _Task:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("due", [[1.0, 2.0], [1.0, 2.0, 3.0, 4.0], [1.0, float("nan"), 2.0],
                                 [1.0, float("inf"), 2.0], [1.0, 2.0 ** 24, 2.0], [1.0, -2.0 ** 24, 2.0], "abc", 3.0])
def test_solver_validates_due_dates_before_any_device_call(due):
    """solve() and solve_table() refuse malformed due dates with SolverError before they touch a device (this runs
    without one): wrong length, not finite, |d| >= 2^24, not a sequence."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="tardiness", due=due, engine=object())
    T = np.ones((3, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError):
        S.solve_table(T, objective="tardiness", due=due, engine=object())


def test_solver_refusals():
    """A missing `due`, `due` under another objective, a task missing from the mapping, a mapping for solve_table,
    a bad weight and hysteresis=True all raise SolverError before any device call."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b")]
    T = np.ones((2, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError, match="due"):
        S.solve(tasks, None, objective="tardiness", engine=object())
    with pytest.raises(S.SolverError, match="due"):
        S.solve_table(T, objective="tardiness", engine=object())
    for objective in ("makespan", "completion"):
        with pytest.raises(S.SolverError, match="tardiness"):
            S.solve(tasks, None, objective=objective, due=[1.0, 2.0], engine=object())
        with pytest.raises(S.SolverError, match="tardiness"):
            S.solve_table(T, objective=objective, due=[1.0, 2.0], engine=object())
    with pytest.raises(S.SolverError, match="no entry"):
        S.solve(tasks, None, objective="tardiness", due={tasks[0]: 1.0}, engine=object())
    with pytest.raises(S.SolverError):
        S.solve_table(T, objective="tardiness", due={0: 1.0, 1: 2.0}, engine=object())
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="tardiness", due=[1.0, 2.0], weights=[1.0, 0.0], engine=object())
    with pytest.raises(S.SolverError, match="hysteresis"):
        S.solve(tasks, None, objective="tardiness", due=[1.0, 2.0], hysteresis=True, engine=object())


def test_orchestrate_shifts_due_dates_by_the_interval(monkeypatch):
    """orchestrate() hands the solve for interval n the due dates d - n * interval (the plan's t = 0 moves forward,
    the deadlines do not), and refuses a sequence `due`, whose alignment its shrinking task list would break."""
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

    tasks = [Task("a", 1, 500.0), Task("b", 3, 900.0)]  # "a" finishes in interval 0, "b" in interval 2
    due = {tasks[0]: 500.0, tasks[1]: 4000.0}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), dict(kw["due"])))
        assert kw["objective"] == "tardiness"
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    def fake_convert(task_list, *a):
        return {}, {}, [0.0] * len(task_list)

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", fake_convert)
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "tardiness", "due": due})
    assert [n for n, _ in seen] == [2, 1, 1]
    for n, (_, got) in enumerate(seen):
        assert got == {t: d - n * 1000 for t, d in due.items()}
    with pytest.raises(SolverError):
        O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "tardiness", "due": [1.0, 2.0]})


def test_flag_due_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_DUE\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_DUE == 256
    assert "sb_set_due" in _lib.SYMBOLS and re.search(r"int\s+sb_set_due\s*\(", header)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_DUE == 0 for h in hooks)


def test_edd_seeds():
    """lpt_seeds(objective="tardiness") orders by due date, ties by runtime, then by job index;
    "weighted_tardiness" breaks ties by runtime / weight."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(3)
    J = 40
    tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
    tmin[:, 5:] = np.inf
    tmin[:10] = tmin[10:20]                       # equal runtimes: the job index decides
    d = rng.integers(0, 6, size=J).astype(np.float32)
    w = rng.choice([0.5, 1.0, 2.0, 8.0], size=J).astype(np.float32)
    for col, order in lpt_seeds(tmin, objective="tardiness", due=d):
        rt = tmin[np.arange(J), col].astype(np.float64)
        keys = [(d[j], rt[j], j) for j in order]
        assert keys == sorted(keys)
    for col, order in lpt_seeds(tmin, objective="weighted_tardiness", due=d, weights=w):
        ratio = tmin[np.arange(J), col].astype(np.float64) / w.astype(np.float64)
        keys = [(d[j], ratio[j], j) for j in order]
        assert keys == sorted(keys)
    with pytest.raises(ValueError):
        lpt_seeds(tmin, objective="tardiness")
