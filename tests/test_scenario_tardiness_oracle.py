"""CPU: the worst- and mean-tardiness objectives over runtime scenarios (SB_FLAG_WORST_TARDINESS /
SB_FLAG_MEAN_TARDINESS; solve(objective="worst_tardiness" | "mean_tardiness" | "worst_completion" |
"mean_completion", scenarios=...)) in the oracle — the fp32 fold against the float64 fold and the C port
(oracle/ref_scenario_tardiness.c), K = 1 with unit factors against ref_release's tardiness and completion folds bit for
bit, d = 0 against the completion folds bit for bit, the fixtures (tests/golden/scenario_tardiness_cases.json,
oracle/gen_scenario_tardiness.py), solve() / solve_table() / orchestrate() handling without a device, the engine table
and the flags against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_release as RR, ref_scenario_tardiness as ST

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TARDINESS = ("worst_tardiness", "mean_tardiness")
COMPLETION = ("worst_completion", "mean_completion")


def _candidates(J, B, nodes, seed, S=3):
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


def _factors(K, J, seed):
    return np.random.default_rng(seed).lognormal(0.0, 0.3, size=(K, J))


def _release(J, seed, scale=3000.0):
    return np.random.default_rng(seed).uniform(-200.0, scale, size=J)


def _due(J, seed, scale=20000.0):
    return np.random.default_rng(seed).uniform(0.0, scale, size=J)


def _weights(J, seed):
    return np.random.default_rng(seed).uniform(0.25, 4.0, size=J)


def _per_job(obj, J, weighted, seed):
    return (_due(J, seed) if obj in TARDINESS else None), (_weights(J, seed + 1) if weighted else None)


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("rel", [False, True])
def test_fp32_fold_tracks_float64(nodes, ints, rel):
    """On the same fp32 scenario tables the fp32 scores agree with the float64 fold to within 1e-5 relative (a sum of
    J terms per scenario, then K more adds), weighted and unweighted."""
    J, B, K = 24, 400, 4
    tab, opt, prio = _candidates(J, B, nodes, seed=11)
    f = _factors(K, J, 3)
    r = _release(J, 5) if rel else None
    for obj in ST.OBJECTIVES:
        for weighted in (False, True):
            d, w = _per_job(obj, J, weighted, 7)
            s32 = ST.evaluate(tab, opt, prio, f, obj, d, w, r, ints, np.float32, nodes)
            s64 = ST.evaluate(tab, opt, prio, f, obj, d, w, r, ints, np.float64, nodes)
            ok = np.isfinite(s64) & (s64 > 0)
            assert np.array_equal(np.isfinite(s32), np.isfinite(s64))
            assert ok.sum() > B // 2
            assert np.max(np.abs(s32[ok] - s64[ok]) / s64[ok]) <= 1e-5


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("rel", [False, True])
def test_c_port_is_bit_equal(nodes, ints, rel):
    """The C port of the fp32 rule equals the Python fold (tables, schedules and both folds) bit for bit, scores and
    every S_k, u8 and u16 priorities, weighted and unweighted: 1e5 candidates at J = 30."""
    for J, B in ((30, 100000), (300, 100)):
        tab, opt, prio = _candidates(J, B, nodes, seed=51 + J)
        if J > 256:
            prio = prio.astype(np.uint16)
        f = _factors(5, J, 7)
        r = _release(J, 8) if rel else None
        for obj in ST.OBJECTIVES:
            for weighted in (False, True):
                if B > 1000 and weighted != (obj in TARDINESS):
                    continue  # the 1e5 sweep takes each weighting once per fold
                d, w = _per_job(obj, J, weighted, 9)
                s, S = ST.evaluate(tab, opt, prio, f, obj, d, w, r, ints, np.float32, nodes, want_totals=True)
                cs, cS = ST.c_evaluate(tab, opt, prio, f, obj, d, w, r, ints, nodes)
                assert np.array_equal(cs.view(np.uint32), s.view(np.uint32))
                assert np.array_equal(cS.view(np.uint32), S.view(np.uint32))


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("rel", [False, True])
def test_one_unit_scenario_is_the_tardiness(nodes, ints, rel):
    """K = 1 with f = 1: both tardiness scores are ref_release's tardiness / weighted-tardiness fold bit for bit."""
    J, B = 20, 500
    tab, opt, prio = _candidates(J, B, nodes, seed=21)
    r = _release(J, 22) if rel else None
    rel_ = np.zeros(J) if r is None else r
    d = _due(J, 23)
    for w, form in ((None, "tardiness"), (_weights(J, 24), "weighted_tardiness")):
        ref = RR.c_evaluate(tab, opt, prio, rel_, ints, np.float32, nodes=nodes, objective=form, weights=w, due=d)
        for obj in TARDINESS:
            s = ST.c_evaluate(tab, opt, prio, np.ones((1, J)), obj, d, w, r, ints, nodes)[0]
            assert np.array_equal(s.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
def test_zero_due_dates_are_the_completion_time(nodes, ints):
    """With every d = 0 the per-scenario tardiness total is ref_release's completion / weighted-completion fold bit
    for bit on every scenario table, release dates negative and positive included: every completion is >= +0, so
    max(C - 0, 0) is C."""
    J, B, K = 20, 500, 3
    tab, opt, prio = _candidates(J, B, nodes, seed=31)
    f = _factors(K, J, 32)
    tabs = ST.scale_tables(tab, f)
    for r in (None, _release(J, 33, scale=-1.0) - 500.0, _release(J, 34)):
        rel_ = np.zeros(J) if r is None else r
        for w, form in ((None, "completion"), (_weights(J, 35), "weighted_completion")):
            for obj in ST.OBJECTIVES:
                d = np.zeros(J) if obj in TARDINESS else None
                _, S = ST.c_evaluate(tab, opt, prio, f, obj, d, w, r, ints, nodes)
                for k in range(K):
                    ref = RR.c_evaluate(tabs[k], opt, prio, rel_, ints, np.float32, nodes=nodes, objective=form,
                                        weights=w)
                    assert np.array_equal(S[:, k].view(np.uint32), ref.view(np.uint32))


def test_worst_is_not_the_per_job_maximum():
    """worst_tardiness is the largest TOTAL over the scenarios: two late jobs in one scenario add up."""
    tab = np.full((2, 1, 8), np.inf, np.float32)
    tab[:, 0, 7] = [10.0, 10.0]
    opt = np.array([[7, 7]], np.uint8)
    prio = np.array([[0, 1]], np.uint8)
    s, S = ST.evaluate(tab, opt, prio, [[1.0, 1.0], [2.0, 1.0]], "worst_tardiness", due=[5.0, 5.0],
                       want_totals=True)
    # scenario 0: completions 10, 20 -> 5 + 15; scenario 1: 20, 30 -> 15 + 25
    assert S.tolist() == [[20.0, 40.0]] and s[0] == 40.0
    m = ST.evaluate(tab, opt, prio, [[1.0, 1.0], [2.0, 1.0]], "mean_tardiness", due=[5.0, 5.0])
    assert m[0] == 60.0


def _cases():
    with open(os.path.join(HERE, "golden", "scenario_tardiness_cases.json")) as f:
        return json.load(f)["cases"]


def test_fixtures_recheck():
    """Every fixture's optima re-check: the stored fp32 optimum scores its stored value and its per-scenario totals,
    the brute force finds the same optimum again (J <= 5), and the fp64 optimum is no worse than the fp32 plan
    rescored.  The fixtures are the instances of scenario_cases.json with due dates and weights added."""
    cases = _cases()
    assert len(cases) == 20
    with open(os.path.join(HERE, "golden", "scenario_cases.json")) as f:
        base = json.load(f)["cases"]
    assert [c["factors"] for c in cases] == [c["factors"] for c in base]
    assert {c["nodes"] for c in cases} == {1, 2} and any(c["release"] for c in cases)
    assert any(c["weights"] for c in cases) and any(c["weights"] is None for c in cases)
    assert any(c["worst_tardiness_f32"]["score"] > 0 for c in cases)
    for c in cases:
        tab, optmap = R.table_from_tuples([[tuple(x) for x in t] for t in c["gpu_time_tuples"]])
        for obj in ST.OBJECTIVES:
            d = c["due"] if obj in TARDINESS else None
            rec = c[obj + "_f32"]
            opt, prio = np.array([rec["opt"]], np.uint8), np.array([rec["prio"]], np.uint8)
            s, S = ST.evaluate(tab, opt, prio, c["factors"], obj, d, c["weights"], c["release"], True, np.float32,
                               c["nodes"], want_totals=True)
            assert float(s[0]) == rec["score"] and [float(x) for x in S[0]] == rec["totals"]
            if len(c["gpu_time_tuples"]) <= 5:
                again = ST.brute_force(tab, optmap, c["factors"], obj, d, c["weights"], c["release"], True,
                                       np.float32, c["nodes"])
                assert again[0] == rec["score"]
            s64 = ST.evaluate(tab, opt, prio, c["factors"], obj, d, c["weights"], c["release"], True, np.float64,
                              c["nodes"])
            assert c[obj + "_f64"]["score"] <= float(s64[0])


class _Strat:
    def __init__(self, runtime, executor="x"):
        self.runtime, self.executor = runtime, executor


class _Task:
    def __init__(self, name, runtimes=(100.0, 60.0)):
        self.name = name
        self.strategies = {g: _Strat(rt) for g, rt in zip((1, 2), runtimes)}


F3 = [[1.0, 1.5], [0.8, 1.2], [1.0, 1.0]]
D3 = [500.0, 300.0, 200.0]


@pytest.mark.parametrize("objective,kw,match", [
    ("worst_tardiness", {"due": D3}, "scenarios=\\.\\.\\."),
    ("mean_tardiness", {"due": D3}, "scenarios=\\.\\.\\."),
    ("worst_completion", {}, "scenarios=\\.\\.\\."),
    ("mean_completion", {"weights": [1.0, 2.0, 3.0]}, "scenarios=\\.\\.\\."),
    ("worst_tardiness", {"scenarios": F3}, "due=\\.\\.\\."),
    ("mean_tardiness", {"scenarios": F3, "weights": [1.0, 2.0, 3.0]}, "due=\\.\\.\\."),
    ("worst_completion", {"scenarios": F3, "due": D3}, "no due dates"),
    ("mean_completion", {"scenarios": F3, "due": D3}, "no due dates"),
    ("tardiness", {"scenarios": F3, "due": D3}, "scenarios apply"),
    ("completion", {"scenarios": F3}, "scenarios apply"),
    ("worst_tardiness", {"scenarios": F3, "due": D3, "penalty": [1.0] * 3}, "penalties apply"),
    ("mean_completion", {"scenarios": F3, "penalty": [1.0] * 3}, "penalties apply"),
    ("worst_tardiness", {"scenarios": F3, "due": D3, "hysteresis": True}, "hysteresis"),
    ("mean_completion", {"scenarios": F3, "hysteresis": True}, "hysteresis"),
    ("mean_tardiness", {"scenarios": F3[:2], "due": D3}, "one row per task"),
    ("worst_completion", {"scenarios": [[1.0, 1.5], [0.8], [1.0, 1.0]]}, "same number"),
    ("mean_completion", {"scenarios": [[1.0] * 9] * 3}, "1 <= K <= 8"),
    ("worst_tardiness", {"scenarios": [[1.0, 0.0], [1.0, 1.0], [1.0, 1.0]], "due": D3}, "finite and > 0"),
    ("mean_tardiness", {"scenarios": F3, "due": D3, "weights": [1.0, 0.0, 1.0]}, "finite and > 0"),
    ("worst_completion", {"scenarios": [[1.0, 1e6], [1.0, 1.0], [1.0, 1.0]]}, "2\\^24"),
    ("mean_tardiness", {"scenarios": F3, "due": [1.0, float("nan"), 2.0]}, "due"),
])
def test_solver_refusals_before_any_device_call(objective, kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one):
    missing scenarios or due dates, due dates on the completion forms, scenarios on the nominal objectives, penalties,
    hysteresis, ragged or out-of-range K, bad factors or weights, and a scenario table beyond the 2^24 horizon."""
    from saturn_b200 import solver as S
    tasks = [_Task("a", (1e5, 6e4)), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective=objective, engine=object(), **kw)
    if "hysteresis" not in kw:
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [[1e5, 6e4], [100.0, 60.0], [100.0, 60.0]]
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective=objective, engine=object(), **kw)


def test_engine_objective_per_solve_objective():
    """The engine objective each solve() objective runs: the tardiness forms by name, weighted with weights, and the
    completion forms as the tardiness forms on due dates of +0."""
    from saturn_b200 import solver as S

    class Eng:
        def __getattr__(self, name):
            return lambda *a, **k: None

    w = np.ones(3, np.float32)
    d = np.zeros(3, np.float32)
    assert S._set_objective(Eng(), "worst_tardiness", None, d) == "worst_tardiness"
    assert S._set_objective(Eng(), "mean_tardiness", w, d) == "weighted_mean_tardiness"
    d64, d32 = S._resolve_due(None, "mean_completion", 3)
    assert d64 == [0.0] * 3 and d32.dtype == np.float32 and not d32.any() and not np.signbit(d32).any()
    assert S._set_objective(Eng(), "worst_completion", None, d32) == "worst_tardiness"
    assert S._set_objective(Eng(), "mean_completion", w, d32) == "weighted_mean_tardiness"


@pytest.mark.parametrize("objective", ST.OBJECTIVES)
def test_scenario_stats_match_the_oracle(objective):
    """_scenario_stats re-runs the list rule per scenario in float64 from a plan's options and order: on integer
    runtimes, integer due dates and weights and power-of-two factors its tardiness (or completion) totals equal the
    oracle's fp64 totals, with and without release dates and on two nodes."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(5)
    J, K = 9, 3
    rts = rng.integers(50, 500, size=J).astype(np.float64)
    gpus = rng.choice([1, 2, 4, 8], size=J)
    f = 2.0 ** rng.integers(-2, 3, size=(K, J))
    what = "tardiness" if objective in TARDINESS else "completion"
    for nodes in (1, 2):
        node = rng.integers(0, nodes, size=J)
        prio = rng.permutation(J)
        tab = np.full((J, 1, 8), np.inf)
        tab[np.arange(J), 0, gpus - 1] = rts
        opt = ((gpus - 1) | (node << 3 if nodes > 1 else 0)).astype(np.uint8)
        for rel in (None, rng.integers(0, 900, size=J).astype(np.float64)):
            for w in (None, rng.integers(1, 5, size=J).astype(np.float64)):
                d = rng.integers(0, 2000, size=J).astype(np.float64) if what == "tardiness" else None
                st = S._scenario_stats(rts, gpus, node, prio, f, True, rel, w, d, objective)
                Sk = ST.totals(tab, opt[None], prio[None].astype(np.uint8), f, d, w, rel, True, np.float64, nodes,
                               objective)[0]
                assert st["scenario_" + what] == [float(x) for x in Sk]
                assert st["worst_" + what] == max(Sk) and st["mean_" + what] == sum(Sk) / K
                assert len(st["scenario_makespans"]) == K


def test_orchestrate_passes_scenarios_and_shifted_due_dates(monkeypatch):
    """orchestrate() hands every solve the same `scenarios` mapping, and under the tardiness forms the due dates
    shifted to each interval's t = 0."""
    from saturn_b200 import orchestrator as O

    class Strat:
        def __init__(self, runtime):
            self.runtime = runtime

    class Task:
        def __init__(self, name, batches, per_batch):
            self.name, self.total_batches = name, batches
            self.strategies = {1: Strat(per_batch * batches)}
            self.selected_strategy = self.strategies[1]

    for objective in ST.OBJECTIVES:
        tasks = [Task("a", 1, 500.0), Task("b", 3, 900.0)]
        scen = {tasks[0]: [1.0, 1.3], tasks[1]: [0.9, 1.1]}
        due = {tasks[0]: 800.0, tasks[1]: 2500.0} if objective in TARDINESS else None
        seen = []

        def fake_solve(task_list, presolved, **kw):
            seen.append((len(task_list), kw["objective"], kw["scenarios"], kw.get("due")))
            return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

        monkeypatch.setattr(O, "solve", fake_solve)
        monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
        kw = {"objective": objective, "scenarios": scen}
        if due is not None:
            kw["due"] = due
        O.orchestrate(tasks, interval=1000, solver_kwargs=kw)
        assert [n for n, _, _, _ in seen] == [2, 1, 1]
        assert all(obj == objective and got is scen for _, obj, got, _ in seen)
        if due is None:
            assert all(d is None for _, _, _, d in seen)
        else:
            assert [d[tasks[1]] for _, _, _, d in seen] == [2500.0, 1500.0, 500.0]


def test_engine_objective_table():
    """The four engine forms have a table of their own, with the flags of the header; the makespan pair's table is
    unchanged, and the name checks accept the new names."""
    from saturn_b200 import _lib
    from saturn_b200.engine import (COMPLETION_PENALTY_OBJECTIVES, SCENARIO_OBJECTIVES, SCENARIO_TARDINESS_OBJECTIVES,
                                    _OBJECTIVES, objective_flag, objective_spec)
    from saturn_b200.solver import SolverError
    assert set(SCENARIO_OBJECTIVES) == {"worst_makespan", "mean_makespan"}
    assert set(SCENARIO_TARDINESS_OBJECTIVES) == {"worst_tardiness", "weighted_worst_tardiness", "mean_tardiness",
                                                  "weighted_mean_tardiness"}
    assert not set(SCENARIO_TARDINESS_OBJECTIVES) & (set(_OBJECTIVES) | set(COMPLETION_PENALTY_OBJECTIVES) |
                                                     set(SCENARIO_OBJECTIVES))
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE
    assert objective_flag("worst_tardiness") == base | _lib.FLAG_WORST_TARDINESS
    assert objective_spec("weighted_mean_tardiness") == (base | _lib.FLAG_MEAN_TARDINESS | _lib.FLAG_WEIGHTED, True,
                                                         True)
    with pytest.raises(SolverError, match="weighted_mean_tardiness"):
        objective_spec("robust_tardiness")


def test_engine_refuses_without_scenarios_or_due_dates():
    """Engine._flags refuses the new forms, before any device call, without scenarios or without due dates."""
    from saturn_b200.engine import Engine
    from saturn_b200.solver import SolverError
    eng = Engine.__new__(Engine)
    eng.due, eng.penalty, eng.release, eng.scenarios = np.zeros(2, np.float32), None, None, None
    for name in ("worst_tardiness", "weighted_mean_tardiness"):
        with pytest.raises(SolverError, match="set_scenarios"):
            eng._flags(True, True, name)
    eng.due, eng.scenarios = None, np.ones((1, 2), np.float32)
    with pytest.raises(SolverError, match="set_due"):
        eng._flags(True, True, "mean_tardiness")


def test_flags_match_the_header():
    """SB_FLAG_WORST_TARDINESS and SB_FLAG_MEAN_TARDINESS are 262144 and 524288 in the header and in _lib, share no bit
    with any other flag or test hook, are in the hooks' static_assert, and end just below the lowest hook."""
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        internal = f.read()
    for name, val in (("WORST_TARDINESS", 262144), ("MEAN_TARDINESS", 524288)):
        m = re.search(r"#define\s+SB_FLAG_%s\s+(\d+)u" % name, header)
        assert m and int(m.group(1)) == getattr(_lib, "FLAG_" + name) == val
        others = [v for k, v in vars(_lib).items() if (k.startswith("FLAG_") or k.startswith("HOOK_"))
                  and k != "FLAG_" + name]
        assert all(o & val == 0 for o in others)
        assert "SB_FLAG_" + name in internal.split("the test hooks share no bit")[0]
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert min(hooks) == _lib.FLAG_MEAN_TARDINESS << 1
