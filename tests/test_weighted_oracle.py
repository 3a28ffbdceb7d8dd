"""CPU: the weighted sum of completion times (SB_FLAG_WEIGHTED) in the oracle — the Python fold against its C port
bit for bit, unit and doubled weights against the unweighted fold, the weighted MILP fixtures
(tests/golden/weighted_completion_cases.json, oracle/gen_weighted.py), the dominance of list schedules on their plans, solve() /
solve_table() weight validation without a device, and the flag's value against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_weighted as RW

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def weighted_cases():
    with open(os.path.join(HERE, "golden", "weighted_completion_cases.json")) as f:
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


def _weights(J, seed):
    return np.random.default_rng(seed).uniform(0.05, 20.0, size=J)


@pytest.mark.parametrize("J,S,nodes", [(1, 1, 1), (7, 3, 1), (40, 4, 1), (300, 2, 1), (23, 1, 2), (64, 1, 3),
                                       (9, 1, 4)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_python_fold_equals_c_port(J, S, nodes, ints, dtype):
    """acc = acc + (w * (start + rt)) with two roundings gives the same bits in Python and in C, fp32 and fp64, on
    one node and on several, with integer and real-valued starts and random real weights."""
    B = 48
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 3 * nodes)
    w = _weights(J, J)
    tot = RW.c_evaluate(tab, opt, prio, ints, dtype, nodes=nodes, weights=w)
    wd = w.astype(dtype)
    for b in range(B):
        got, start, _, _ = RW.list_schedule(tab, opt[b], prio[b], ints, dtype, nodes=nodes, weights=w)
        assert dtype(got).tobytes() == tot[b].tobytes()
        acc = dtype(0.0)
        for j in prio[b]:
            c = dtype(dtype(start[j]) + dtype(tab[j][0 if nodes > 1 else opt[b][j] >> 3][opt[b][j] & 7]))
            acc = dtype(acc + dtype(wd[j] * c))
        assert acc == tot[b]
    if nodes == 1:
        assert np.array_equal(RW.list_schedule_batch(tab, opt, prio, ints, dtype, weights=w), tot)


@pytest.mark.parametrize("ints", [True, False])
def test_c_port_at_scale(ints):
    """About 1e5 candidates: the C fold equals the vectorised Python fold bit for bit in fp32 and fp64."""
    J, B = 48, 100_000
    tab, opt, prio = _candidates(J, 3, B, 1, seed=77)
    w = _weights(J, 78)
    for dt in (np.float32, np.float64):
        c = RW.c_evaluate(tab, opt, prio, ints, dt, weights=w, threads=8)
        py = RW.list_schedule_batch(tab, opt, prio, ints, dt, weights=w)
        assert np.array_equal(c, py)


@pytest.mark.parametrize("J,S,nodes", [(40, 4, 1), (300, 2, 1), (64, 1, 3)])
def test_unit_weights_give_the_unweighted_fold_and_doubled_weights_twice_it(J, S, nodes):
    B = 256
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J)
    for ints in (True, False):
        for dt in (np.float32, np.float64):
            plain = RW.c_evaluate(tab, opt, prio, ints, dt, nodes=nodes)
            one = RW.c_evaluate(tab, opt, prio, ints, dt, nodes=nodes, weights=np.ones(J))
            two = RW.c_evaluate(tab, opt, prio, ints, dt, nodes=nodes, weights=np.full(J, 2.0))
            assert one.tobytes() == plain.tobytes()
            assert two.tobytes() == (plain * dt(2)).astype(dt).tobytes()
            py = [RW.list_schedule(tab, opt[b], prio[b], ints, dt, nodes=nodes, weights=np.ones(J))[0]
                  for b in range(8)]
            assert np.array_equal(np.array(py, dtype=dt), plain[:8])


def test_oracle_refuses_bad_weights():
    tab, optmap = R.table_from_tuples([[(1, 10.0)], [(2, 5.0)]])
    for w in ([1.0], [1.0, 0.0], [1.0, -2.0], [1.0, np.inf], [1.0, np.nan]):
        with pytest.raises(ValueError):
            RW.list_schedule(tab, [0, 0], [0, 1], weights=w)
    with pytest.raises(ValueError):
        RW.c_evaluate(tab, np.zeros((1, 2), np.uint8), np.array([[0, 1]], np.uint8), weights=[1.0, 0.0])


def test_weighted_fixtures_match_the_milp(weighted_cases):
    """On every instance HiGHS proved optimal the exhaustive fp64 optimum equals the weighted MILP's optimum (1e-9
    relative); the MILP's plans are feasible under the MILP's constraints; the weights are exact in fp32; most
    instances have an optimum the unweighted objective does not pick."""
    assert len(weighted_cases) >= 18
    proven = 0
    for rec in weighted_cases:
        w = rec["weights"]
        assert all(float(np.float32(x)) == x and x > 0 for x in w)
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        bf = rec["bruteforce_f64"]["weighted_completion"]
        again = RW.list_schedule(tab, rec["bruteforce_f64"]["opt"], rec["bruteforce_f64"]["prio"], True, np.float64,
                                 weights=w)[0]
        assert again == bf, rec["name"]
        f32 = RW.list_schedule(tab, rec["bruteforce_f32"]["opt"], rec["bruteforce_f32"]["prio"], True, np.float32,
                               weights=w)[0]
        assert f32 == rec["bruteforce_f32"]["weighted_completion"] and f32 == pytest.approx(bf, rel=1e-6)
        assert rec["differs"] == (rec["unweighted_optimum_weighted"] > bf * (1 + 1e-12))
        m = rec["milp"]
        if m["start"] is None:
            continue
        assert m["feasible"] and m["overlaps"] == 0, rec["name"]
        J = len(tuples)
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        bss = [[1 if s == m["opt_idx"][t] else 0 for s in range(len(tuples[t]))] for t in range(J)]
        tga = [[[(m["mask"][t] >> g) & 1 for g in range(R.NSLOT)]] for t in range(J)]
        sta = [[[m["start"][t] if tga[t][0][g] else 0.0 for t in range(J)] for g in range(R.NSLOT)]]
        bna = [[1] for _ in range(J)]
        boa = [[1 if a != b and (m["start"][a], a) < (m["start"][b], b) else 0 for b in range(J)] for a in range(J)]
        assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, max(s + r for s, r in zip(m["start"], rt))) == []
        assert R.check_plan(m["start"], m["mask"], rt, k)[0]
        if m["proven_optimal"]:
            proven += 1
            assert bf == pytest.approx(m["weighted_completion"], rel=1e-9), rec["name"]
            assert m["objective_value"] == pytest.approx(m["weighted_completion"], rel=1e-6), rec["name"]
        else:
            assert bf <= m["weighted_completion"] * (1 + 1e-9), rec["name"]
    assert proven >= 15
    assert sum(r["differs"] for r in weighted_cases) >= len(weighted_cases) // 2


def test_list_schedules_dominate_the_weighted_milp_plans(weighted_cases):
    """DESIGN.md §3.1: ordering a feasible plan's jobs by start and running the list rule with its options finishes
    every job no later, so the weighted sum (non-negative weights) does not grow."""
    n = 0
    for rec in weighted_cases:
        m = rec["milp"]
        if m["start"] is None:
            continue
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        opt = [optmap[t][m["opt_idx"][t]] for t in range(J)]
        order = sorted(range(J), key=lambda t: (m["start"][t], t))
        score, start, _, _ = RW.list_schedule(tab, opt, order, True, np.float64, weights=rec["weights"])
        for t in range(J):
            rt = tuples[t][m["opt_idx"][t]][1]
            assert start[t] + rt <= m["start"][t] + rt + 1e-9, (rec["name"], t)
        assert score <= m["weighted_completion"] * (1 + 1e-12)
        n += 1
    assert n >= 15


class _Task:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("weights", [[1.0, 2.0], [1.0, 2.0, 3.0, 4.0], [1.0, 2.0, 0.0], [1.0, -1.0, 2.0],
                                     [1.0, float("nan"), 2.0], [1.0, float("inf"), 2.0], [1.0, 1e-50, 2.0],
                                     [1.0, 1e300, 2.0], "abc", 3.0])
def test_solver_validates_weights_before_any_device_call(weights):
    """solve() and solve_table() refuse malformed weights with SolverError before they touch a device (this runs
    without one): wrong length, not finite and > 0, 0 or inf once in fp32, not a sequence."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="completion", weights=weights, engine=object())
    T = np.ones((3, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError):
        S.solve_table(T, objective="completion", weights=weights, engine=object())


def test_solver_refuses_weights_without_the_completion_objective_and_incomplete_mappings():
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b")]
    with pytest.raises(S.SolverError, match="completion"):
        S.solve(tasks, None, weights=[1.0, 2.0], engine=object())
    with pytest.raises(S.SolverError, match="completion"):
        S.solve_table(np.ones((2, 1, 8), dtype=np.float32), weights=[1.0, 2.0], engine=object())
    with pytest.raises(S.SolverError, match="no entry"):
        S.solve(tasks, None, objective="completion", weights={tasks[0]: 1.0}, engine=object())
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="completion", weights={tasks[0]: 1.0, tasks[1]: 0.0}, engine=object())
    with pytest.raises(S.SolverError):
        S.solve_table(np.ones((2, 1, 8), dtype=np.float32), objective="completion", weights={0: 1.0, 1: 2.0},
                      engine=object())
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="completion", weights=[1.0, 2.0], hysteresis=True, engine=object())


def test_flag_weighted_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_WEIGHTED\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_WEIGHTED == 128
    assert "sb_set_weights" in _lib.SYMBOLS and re.search(r"int\s+sb_set_weights\s*\(", header)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_WEIGHTED == 0 for h in hooks)


def test_wspt_seeds_follow_smiths_rule():
    """lpt_seeds(objective="weighted_completion") orders by rt / w ascending, ties by job index; unit weights give
    exactly the shortest-processing-time orders."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(3)
    J = 40
    tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
    tmin[:, 5:] = np.inf
    spt = lpt_seeds(tmin, objective="completion")
    unit = lpt_seeds(tmin, objective="weighted_completion", weights=np.ones(J, np.float32))
    for (c0, o0), (c1, o1) in zip(spt, unit):
        assert np.array_equal(c0, c1) and np.array_equal(o0, o1)
    w = rng.choice([0.5, 1.0, 2.0, 8.0], size=J).astype(np.float32)
    for col, order in lpt_seeds(tmin, objective="weighted_completion", weights=w):
        ratio = tmin[np.arange(J), col].astype(np.float64) / w.astype(np.float64)
        keys = [(ratio[j], j) for j in order]
        assert keys == sorted(keys)
    with pytest.raises(ValueError):
        lpt_seeds(tmin, objective="weighted_completion")
