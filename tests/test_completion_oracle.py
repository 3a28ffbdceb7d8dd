"""CPU: the sum-of-completion-times objective in the oracle — the Python restatement against its C port (fp32,
bit for bit), against the MILP restated for that objective (tests/golden/completion_cases.json), the dominance of
list schedules checked on the MILP's own plans, and the makespan objective left as it was."""
import json
import os

import numpy as np
import pytest

from oracle import c_oracle, ref_completion as RC, ref_eval as R

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def completion_cases():
    with open(os.path.join(HERE, "golden", "completion_cases.json")) as f:
        return json.load(f)["cases"]


def _multi_node_candidates(J, B, nodes, seed):
    T, valid = R.synth_table(J, 1, 8, seed=seed, masked=False)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = R.synth_candidates(J, B, valid, seed=seed + 1)
    rng = np.random.default_rng(seed + 2)
    opt = (opt | (rng.integers(0, nodes, size=opt.shape) << 3)).astype(np.uint8)
    return tab, opt, prio


@pytest.mark.parametrize("J,S,nodes", [(1, 1, 1), (7, 3, 1), (40, 4, 1), (300, 2, 1), (23, 1, 2), (64, 1, 3),
                                       (9, 1, 4)])
@pytest.mark.parametrize("ints", [True, False])
def test_python_oracle_equals_c_port_fp32(J, S, nodes, ints):
    """The left fold acc = acc + (start + rt) in schedule order gives the same fp32 bits in Python and in C, on one
    node and on several, with integer and real-valued starts; the starts and masks are those of the makespan rule."""
    B = 64
    if nodes == 1:
        T, valid = R.synth_table(J, S, 8, seed=J + S)
        tab = R.canon_table(T, range(1, 9))
        opt, prio = R.synth_candidates(J, B, valid, seed=J)
    else:
        tab, opt, prio = _multi_node_candidates(J, B, nodes, seed=J)
    tot, start, mask = RC.c_evaluate(tab, opt, prio, ints, np.float32, want_plan=True, nodes=nodes)
    mk, start_m, mask_m = c_oracle.evaluate(tab, opt, prio, ints, np.float32, want_plan=True, nodes=nodes)
    assert np.array_equal(start, start_m) and np.array_equal(mask, mask_m)
    for b in range(B):
        got, st, mk_b, _ = RC.list_schedule(tab, opt[b], prio[b], ints, np.float32, nodes=nodes)
        assert np.float32(got) == tot[b] and np.float32(got).tobytes() == tot[b].tobytes()
        assert [np.float32(x) for x in st] == list(start[b])
        # the fold is sequential: the same values summed in another order may differ in fp32, this one never does
        acc = np.float32(0.0)
        for j in prio[b]:
            acc = np.float32(acc + np.float32(np.float32(start[b][j]) + np.float32(tab[j][0 if nodes > 1 else opt[b][j] >> 3][opt[b][j] & 7])))
        assert acc == tot[b]
    if nodes == 1:
        batch = RC.list_schedule_batch(tab, opt, prio, ints, np.float32)
        assert np.array_equal(batch, tot)
    tot64 = RC.c_evaluate(tab, opt, prio, ints, np.float64, nodes=nodes)
    assert np.allclose(tot64, tot, rtol=1e-5)
    assert np.all(tot >= mk)                                       # a sum of completions is at least their max


def test_completion_fixtures_match_the_restated_milp(completion_cases):
    """On every instance HiGHS closed to a zero gap the exhaustive list-schedule optimum equals the MILP's optimum
    (1e-9 relative); on a time-limited one it is no worse than the incumbent.  The MILP's plans are feasible."""
    assert len(completion_cases) >= 18
    proven = 0
    for rec in completion_cases:
        m = rec["milp"]
        bf = rec["bruteforce_f64"]["total_completion"]
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        # the recorded exhaustive optimum is what its recorded candidate scores
        again = RC.list_schedule(tab, rec["bruteforce_f64"]["opt"], rec["bruteforce_f64"]["prio"], True, np.float64)[0]
        assert again == bf, rec["name"]
        f32 = RC.list_schedule(tab, rec["bruteforce_f32"]["opt"], rec["bruteforce_f32"]["prio"], True, np.float32)[0]
        assert f32 == rec["bruteforce_f32"]["total_completion"]
        assert f32 == pytest.approx(bf, rel=1e-6)
        if m["total_completion"] is None:
            continue
        assert m["feasible"] and m["overlaps"] == 0, rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert bf == pytest.approx(m["total_completion"], rel=1e-9), rec["name"]
            assert m["objective_value"] == pytest.approx(m["total_completion"], rel=1e-6), rec["name"]
        else:
            assert bf <= m["total_completion"] * (1 + 1e-9), rec["name"]
    assert proven >= 15


def test_list_schedules_dominate_the_milp_plans(completion_cases):
    """DESIGN.md §3: take a feasible plan, order its jobs by start and run the list rule with the plan's options —
    every job finishes no later than in the plan.  Checked on every MILP plan of the fixtures."""
    n = 0
    for rec in completion_cases:
        m = rec["milp"]
        if m["start"] is None:
            continue
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        opt = [optmap[t][m["opt_idx"][t]] for t in range(J)]
        order = sorted(range(J), key=lambda t: (m["start"][t], t))
        _, start, _, _ = RC.list_schedule(tab, opt, order, True, np.float64)
        for t in range(J):
            rt = tuples[t][m["opt_idx"][t]][1]
            assert start[t] + rt <= m["start"][t] + rt + 1e-9, (rec["name"], t)
        n += 1
    assert n >= 15


def test_makespan_objective_is_unchanged(golden):
    """objective="makespan" in the completion module is the makespan evaluator itself: the recorded exhaustive
    optima of the makespan fixtures, and the same batch results as ref_eval and its C port."""
    n = 0
    for rec in golden["cases"]:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, _ = R.table_from_tuples(tuples)
        bf = rec["bruteforce_int"]
        a = R.list_schedule(tab, bf["opt"], bf["prio"], True, np.float64)
        b = RC.list_schedule(tab, bf["opt"], bf["prio"], True, np.float64, objective="makespan")
        assert a[0] == b[0] == bf["makespan"] and a[1] == b[1] and a[2] == b[2]
        n += 1
    assert n > 10
    T, valid = R.synth_table(50, 3, 8, seed=4)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = R.synth_candidates(50, 200, valid, seed=5)
    for ints in (True, False):
        ref = c_oracle.evaluate(tab, opt, prio, ints, np.float32)
        assert np.array_equal(ref, R.list_schedule_batch(tab, opt, prio, ints, np.float32))
        assert np.array_equal(ref, RC.list_schedule_batch(tab, opt, prio, ints, np.float32, objective="makespan"))


def test_exhaustive_optimum_small(completion_cases):
    """brute_force(objective="completion") on a 3-task fixture gives the recorded optimum, and differs from the
    makespan optimum's own sum of completions only in the direction it must (never worse)."""
    rec = next(r for r in completion_cases if len(r["gpu_time_tuples"]) == 3)
    tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
    tab, optmap = R.table_from_tuples(tuples)
    best = RC.brute_force(tab, optmap, True)
    assert best[0] == rec["bruteforce_f64"]["total_completion"]
    mk_best = RC.brute_force(tab, optmap, True, objective="makespan")
    assert mk_best[0] == R.brute_force(tab, optmap, True)[0]
    assert best[0] <= RC.list_schedule(tab, mk_best[1], mk_best[2], True)[0]


def test_unknown_objective_is_refused():
    tab, optmap = R.table_from_tuples([[(1, 10.0)]])
    with pytest.raises(ValueError):
        RC.list_schedule(tab, [0], [0], objective="tardiness")
    with pytest.raises(ValueError):
        RC.brute_force(tab, [[0]], objective="mean")
