"""CPU: the worst- and mean-makespan objectives over runtime scenarios (SB_FLAG_WORST_MAKESPAN / SB_FLAG_MEAN_MAKESPAN,
solve(objective="worst_makespan" | "mean_makespan", scenarios=...)) in the oracle — the fp32 fold against the float64
fold and the C port (oracle/ref_scenarios.c), K = 1 with unit factors against ref_eval bit for bit, exact scaling by
powers of two, the bounds of both scores, the fixtures (tests/golden/scenario_cases.json, oracle/gen_scenarios.py),
solve() / solve_table() / orchestrate() handling without a device, and the flags against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import c_oracle, ref_eval as R, ref_scenarios as SC

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


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


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("rel", [False, True])
def test_fp32_fold_tracks_float64(nodes, ints, rel):
    """On the same fp32 scenario tables the fp32 scores agree with the float64 fold to within the makespan bars of
    test_oracle (integer starts: one rounding of the final completion per scenario; real starts: 2e-6 relative)."""
    J, B, K = 24, 400, 4
    tab, opt, prio = _candidates(J, B, nodes, seed=11)
    f = _factors(K, J, 3)
    r = _release(J, 5) if rel else None
    for obj in SC.OBJECTIVES:
        s32 = SC.evaluate(tab, opt, prio, f, obj, r, ints, np.float32, nodes)
        s64 = SC.evaluate(tab, opt, prio, f, obj, r, ints, np.float64, nodes)
        ok = np.isfinite(s64)
        assert np.array_equal(np.isfinite(s32), ok)
        bar = 2.0 ** -22 if ints else 2e-6
        assert np.max(np.abs(s32[ok] - s64[ok]) / s64[ok]) <= bar


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
def test_one_unit_scenario_is_the_makespan(nodes, ints):
    """K = 1 with f = 1: both scores equal ref_eval's makespan bit for bit (the anchor to the pinned oracle)."""
    J, B = 20, 600
    tab, opt, prio = _candidates(J, B, nodes, seed=21)
    ref = c_oracle.evaluate(tab, opt, prio, ints, np.float32, nodes=nodes) if nodes > 1 else \
        c_oracle.evaluate(tab, opt, prio, ints, np.float32)
    for obj in SC.OBJECTIVES:
        s = SC.evaluate(tab, opt, prio, np.ones((1, J)), obj, None, ints, np.float32, nodes)
        assert np.array_equal(s.view(np.uint32), np.asarray(ref, np.float32).view(np.uint32))
        cs, _M = SC.c_evaluate(tab, opt, prio, np.ones((1, J)), obj, None, ints, nodes)
        assert np.array_equal(cs.view(np.uint32), s.view(np.uint32))


@pytest.mark.parametrize("n", [-3, 1, 4])
def test_power_of_two_scales_every_makespan(n):
    """Without integer starts, a uniform factor 2^n scales every M_k exactly (every sum and max commutes with it)."""
    J, B = 16, 300
    tab, opt, prio = _candidates(J, B, 1, seed=31)
    base = SC.makespans(tab, opt, prio, np.ones((1, J)), None, False, np.float32)[:, 0]
    M = SC.makespans(tab, opt, prio, np.full((3, J), 2.0 ** n), None, False, np.float32)
    for k in range(3):
        assert np.array_equal(M[:, k], (base * np.float32(2.0 ** n)).astype(np.float32))


@pytest.mark.parametrize("K", [1, 3, 8])
def test_score_bounds(K):
    """worst >= M_k >= 0 for every k, and the mean (the sum / K) lies between the smallest and the largest M_k."""
    J, B = 12, 500
    tab, opt, prio = _candidates(J, B, 1, seed=41)
    f = _factors(K, J, 9)
    worst, M = SC.evaluate(tab, opt, prio, f, "worst_makespan", want_makespans=True)
    total = SC.evaluate(tab, opt, prio, f, "mean_makespan")
    ok = np.isfinite(worst)
    assert (M >= 0).all()
    assert (worst[:, None] >= M).all()
    mean = total[ok].astype(np.float64) / K
    assert (mean >= M[ok].min(axis=1) * (1 - 1e-6)).all() and (mean <= M[ok].max(axis=1) * (1 + 1e-6)).all()


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("rel", [False, True])
def test_c_port_is_bit_equal(nodes, ints, rel):
    """The C port of the fp32 rule equals the Python fold (tables, schedules and fold) bit for bit, scores and every
    M_k, u8 and u16 priorities."""
    for J, B in ((30, 3000), (300, 200)):
        tab, opt, prio = _candidates(J, B, nodes, seed=51 + J)
        if J > 256:
            prio = prio.astype(np.uint16)
        f = _factors(5, J, 7)
        r = _release(J, 8) if rel else None
        for obj in SC.OBJECTIVES:
            s, M = SC.evaluate(tab, opt, prio, f, obj, r, ints, np.float32, nodes, want_makespans=True)
            cs, cM = SC.c_evaluate(tab, opt, prio, f, obj, r, ints, nodes)
            assert np.array_equal(cs.view(np.uint32), s.view(np.uint32))
            assert np.array_equal(cM.view(np.uint32), M.view(np.uint32))


def test_absent_cells_stay_absent():
    """An option without a runtime (+inf) stays +inf under every factor: a candidate that selects one scores +inf."""
    tab = np.full((2, 1, 8), np.inf, np.float32)
    tab[:, 0, 0] = [10.0, 20.0]
    opt = np.array([[0, 0], [1, 0]], np.uint8)
    prio = np.array([[0, 1], [0, 1]], np.uint8)
    s = SC.evaluate(tab, opt, prio, [[0.5, 2.0], [1.5, 1.0]], "worst_makespan")
    assert s[0] == 40.0 and np.isinf(s[1])


def _cases():
    with open(os.path.join(HERE, "golden", "scenario_cases.json")) as f:
        return json.load(f)["cases"]


def test_fixtures_recheck():
    """Every fixture's optima re-check: the stored fp32 optimum scores its stored value and its scenario makespans,
    the brute force finds the same optimum again, and the fp64 optimum is no worse than the fp32 plan rescored."""
    cases = _cases()
    assert len(cases) == 20
    assert {c["nodes"] for c in cases} == {1, 2} and any(c["release"] for c in cases)
    assert {len(c["factors"]) for c in cases} == {2, 4, 8}
    for c in cases:
        tab, optmap = R.table_from_tuples([[tuple(x) for x in t] for t in c["gpu_time_tuples"]])
        for obj in SC.OBJECTIVES:
            rec = c[obj + "_f32"]
            opt, prio = np.array([rec["opt"]], np.uint8), np.array([rec["prio"]], np.uint8)
            s, M = SC.evaluate(tab, opt, prio, c["factors"], obj, c["release"], True, np.float32, c["nodes"],
                               want_makespans=True)
            assert float(s[0]) == rec["score"] and [float(x) for x in M[0]] == rec["makespans"]
            if len(c["gpu_time_tuples"]) <= 5:
                again = SC.brute_force(tab, optmap, c["factors"], obj, c["release"], True, np.float32, c["nodes"])
                assert again[0] == rec["score"]
            s64 = SC.evaluate(tab, opt, prio, c["factors"], obj, c["release"], True, np.float64, c["nodes"])
            assert c[obj + "_f64"]["score"] <= float(s64[0])


class _Strat:
    def __init__(self, runtime, executor="x"):
        self.runtime, self.executor = runtime, executor


class _Task:
    def __init__(self, name, runtimes=(100.0, 60.0)):
        self.name = name
        self.strategies = {g: _Strat(rt) for g, rt in zip((1, 2), runtimes)}


F3 = [[1.0, 1.5], [0.8, 1.2], [1.0, 1.0]]


@pytest.mark.parametrize("objective,kw,match", [
    ("worst_makespan", {}, "scenarios=\\.\\.\\."),
    ("mean_makespan", {}, "scenarios=\\.\\.\\."),
    ("makespan", {"scenarios": F3}, "scenarios apply"),
    ("completion", {"scenarios": F3}, "scenarios apply"),
    ("worst_makespan", {"scenarios": F3[:2]}, "one row per task"),
    ("worst_makespan", {"scenarios": [[1.0, 1.5], [0.8], [1.0, 1.0]]}, "same number"),
    ("worst_makespan", {"scenarios": [[1.0] * 9] * 3}, "1 <= K <= 8"),
    ("mean_makespan", {"scenarios": [[], [], []]}, "1 <= K <= 8"),
    ("worst_makespan", {"scenarios": [[1.0, 0.0], [1.0, 1.0], [1.0, 1.0]]}, "finite and > 0"),
    ("worst_makespan", {"scenarios": [[1.0, -1.0], [1.0, 1.0], [1.0, 1.0]]}, "finite and > 0"),
    ("mean_makespan", {"scenarios": [[1.0, float("nan")], [1.0, 1.0], [1.0, 1.0]]}, "finite and > 0"),
    ("mean_makespan", {"scenarios": [[1.0, float("inf")], [1.0, 1.0], [1.0, 1.0]]}, "finite and > 0"),
    ("worst_makespan", {"scenarios": [[1.0, 1e-46], [1.0, 1.0], [1.0, 1.0]]}, "fp32"),
    ("worst_makespan", {"scenarios": [[1.0, 1e6], [1.0, 1.0], [1.0, 1.0]]}, "2\\^24"),
    ("worst_makespan", {"scenarios": F3, "hysteresis": True}, "hysteresis"),
])
def test_solver_refusals_before_any_device_call(objective, kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one):
    missing or unwanted scenarios, ragged or out-of-range K, bad factors, hysteresis, and a scenario table that breaks
    the integer-start horizon."""
    from saturn_b200 import solver as S
    tasks = [_Task("a", (1e5, 6e4)), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective=objective, engine=object(), **kw)
    if "hysteresis" not in kw:
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [[1e5, 6e4], [100.0, 60.0], [100.0, 60.0]]
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective=objective, engine=object(), **kw)


def test_scenarios_as_a_mapping():
    """solve() takes scenarios as a mapping Task -> K factors too, and a task missing from it raises."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    f64, f32 = S._resolve_scenarios({t: F3[i] for i, t in enumerate(tasks)}, "worst_makespan", 3, tasks)
    assert f64.shape == (2, 3) and f32.dtype == np.float32 and f64[1].tolist() == [1.5, 1.2, 1.0]
    with pytest.raises(S.SolverError, match="no entry"):
        S._resolve_scenarios({tasks[0]: [1.0]}, "worst_makespan", 3, tasks)


def test_scenario_stats_match_the_oracle():
    """_scenario_stats re-runs the list rule per scenario in float64 from a plan's options and order: on integer
    runtimes and power-of-two factors it equals the oracle's fp64 makespans, with and without release dates and on
    two nodes."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(5)
    J, K = 9, 3
    rts = rng.integers(50, 500, size=J).astype(np.float64)
    gpus = rng.choice([1, 2, 4, 8], size=J)
    f = 2.0 ** rng.integers(-2, 3, size=(K, J))
    for nodes in (1, 2):
        node = rng.integers(0, nodes, size=J)
        prio = rng.permutation(J)
        tab = np.full((J, 1, 8), np.inf)
        tab[np.arange(J), 0, gpus - 1] = rts
        opt = ((gpus - 1) | (node << 3 if nodes > 1 else 0)).astype(np.uint8)
        for rel in (None, rng.integers(0, 900, size=J).astype(np.float64)):
            st = S._scenario_stats(rts, gpus, node, prio, f, True, rel)
            M = SC.makespans(tab, opt[None], prio[None].astype(np.uint8), f, rel, True, np.float64, nodes)[0]
            assert st["scenario_makespans"] == [float(x) for x in M]
            assert st["worst_makespan"] == max(M) and st["mean_makespan"] == sum(M) / K


def test_orchestrate_passes_scenarios_through(monkeypatch):
    """orchestrate() hands every solve the same `scenarios` mapping and refuses a sequence."""
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
    scen = {tasks[0]: [1.0, 1.3], tasks[1]: [0.9, 1.1]}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), kw["objective"], kw["scenarios"]))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "worst_makespan", "scenarios": scen})
    assert [n for n, _, _ in seen] == [2, 1, 1]
    assert all(obj == "worst_makespan" and got is scen for _, obj, got in seen)
    with pytest.raises(SolverError, match="mapping"):
        O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "worst_makespan", "scenarios": [[1.0]] * 2})


def test_engine_objective_table():
    """The scenario pair has its own table, leaves the other tables as they are, and the name checks accept it."""
    from saturn_b200 import _lib
    from saturn_b200.engine import (COMPLETION_PENALTY_OBJECTIVES, SCENARIO_OBJECTIVES, _OBJECTIVES, objective_flag,
                                    objective_spec, scenarios_f32)
    from saturn_b200.solver import SolverError
    assert set(SCENARIO_OBJECTIVES) == {"worst_makespan", "mean_makespan"}
    assert not set(SCENARIO_OBJECTIVES) & (set(_OBJECTIVES) | set(COMPLETION_PENALTY_OBJECTIVES))
    assert objective_flag("worst_makespan") == _lib.FLAG_WORST_MAKESPAN
    assert objective_spec("mean_makespan") == (_lib.FLAG_MEAN_MAKESPAN, False, False)
    with pytest.raises(SolverError, match="mean_makespan"):
        objective_spec("robust")
    assert scenarios_f32([[1.0, 2.0]], 2).shape == (1, 2)
    with pytest.raises(SolverError):
        scenarios_f32([[1.0, 2.0]], 3)


def test_flags_match_the_header():
    """SB_FLAG_WORST_MAKESPAN and SB_FLAG_MEAN_MAKESPAN are 65536 and 131072 in the header and in _lib, share no bit
    with any other flag or test hook, are in the hooks' static_assert, and the two new entry points are declared."""
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    for name, val in (("WORST_MAKESPAN", 65536), ("MEAN_MAKESPAN", 131072)):
        m = re.search(r"#define\s+SB_FLAG_%s\s+(\d+)u" % name, header)
        assert m and int(m.group(1)) == getattr(_lib, "FLAG_" + name) == val
        others = [v for k, v in vars(_lib).items() if (k.startswith("FLAG_") or k.startswith("HOOK_"))
                  and k != "FLAG_" + name]
        assert all(o & val == 0 for o in others)
        with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
            assert "SB_FLAG_" + name in f.read().split("the test hooks share no bit")[0]
    for sym in ("sb_set_scenarios", "sb_eval_scenarios"):
        assert sym in _lib.SYMBOLS and re.search(r"int\s+%s\s*\(" % sym, header)
