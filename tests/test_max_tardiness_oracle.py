"""CPU: the maximum-tardiness objective (SB_FLAG_MAX_TARDINESS, solve(objective="max_stretch")) in the oracle — the
Python schedule and max fold against the C port (oracle/ref_max_tardiness.c) bit for bit, the exact check on
tie-heavy inputs, absent cells, the makespan and doubled-weight identities, the agreement with the maximum lateness on
integer data, the MILP fixtures (tests/golden/max_tardiness_cases.json, oracle/gen_max_tardiness.py), the seeds,
solve() / solve_table() / orchestrate() handling without a device, and the flag against the header."""
import json
import os
import re

import numpy as np
import pytest

from oracle import ref_eval as R, ref_exact as X, ref_max_lateness as ML, ref_max_tardiness as MT, ref_release as RR

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
    """The C port (schedule and max fold in C) gives the same bits as the Python schedule with the numpy fold,
    scores, starts and slot masks, in fp32 and fp64: integer and real-valued starts, 1 to 4 nodes, with and without
    release dates, unit and real weights."""
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 7 * nodes)
    scale = 2000.0 * J / 8
    d = _due(J, J + 1, scale)
    r = np.random.default_rng(J + 2).uniform(-0.1, 0.8, size=J) * scale if released else None
    w = _weights(J, J + 3) if weighted else None
    for dtype in (np.float32, np.float64):
        c, cs, cm = MT.c_evaluate(tab, opt, prio, d, r, ints, dtype, want_plan=True, threads=8, nodes=nodes, weights=w)
        py, ps, pm = MT.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, want_plan=True,
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
        c = MT.c_evaluate(tab, opt, prio, d, r, ints, dtype, threads=8, nodes=nodes, weights=w)
        py = MT.evaluate(tab, opt, prio, d, r, ints, dtype, nodes=nodes, use_c=False, weights=w)
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
    """On integer data fp32 rounds nothing: the fp32 fold equals max w max(0, C - d) in exact arithmetic (starts from
    ref_exact), and with unit weights the maximum is that of the jobs whose completion is past their due date."""
    tab, opt, prio, d, r, on = _tie_heavy(J, J, released)
    w = np.random.default_rng(J).integers(1, 5, size=J).astype(np.float64) if weighted else None
    got = MT.evaluate(tab, opt, prio, d, r, True, np.float32, weights=w)
    for b in range(len(opt)):
        assert float(MT.exact(tab, opt[b], prio[b], d, r, weights=w)) == float(got[b]), b
    _, start, _ = X.schedule(tab, opt[0], prio[0], r)
    wj = np.ones(J) if w is None else w
    late = [wj[j] * (start[j] + int(tab[j, 0, opt[0, j] & 7]) - d[j]) for j in range(J)]
    assert float(got[0]) == float(max([0.0] + [float(x) for x in late]))


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_makespan_boundary_and_doubled_weights(nodes, ints, released):
    """d = 0 with unit weights gives the makespan fold bit for bit; due dates at or past every completion give +0;
    w = 2 gives exactly twice w = 1, and w = 1 exactly the unweighted fold."""
    J = 30
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, 300, nodes, seed=3)
    r = np.random.default_rng(4).uniform(-10, 3000, size=J) if released else None
    mk = RR.c_evaluate(tab, opt, prio, np.zeros(J) if r is None else r, ints, np.float32, nodes=nodes)
    got = MT.evaluate(tab, opt, prio, np.zeros(J), r, ints, np.float32, nodes=nodes)
    assert got.tobytes() == mk.tobytes()
    _, start, _ = MT.evaluate(tab, opt, prio, np.zeros(J), r, ints, np.float32, nodes=nodes, want_plan=True)
    rt = np.asarray(tab, np.float32)[np.arange(J)[None, :], 0 if nodes > 1 else opt >> 3, opt & 7]
    late = np.full(J, float((start + rt).astype(np.float32).max()))  # the latest fp32 completion
    zero = MT.evaluate(tab, opt, prio, late, r, ints, np.float32, nodes=nodes, weights=_weights(J, 5))
    assert zero.tobytes() == np.zeros(len(opt), np.float32).tobytes()
    d = _due(J, 6, 6000.0)
    one = MT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.ones(J))
    two = MT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes, weights=np.full(J, 2.0))
    unit = MT.evaluate(tab, opt, prio, d, r, ints, np.float32, nodes=nodes)
    assert two.tobytes() == (one * np.float32(2)).tobytes() and one.tobytes() == unit.tobytes()
    assert (one > 0).all()


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("released", [False, True])
def test_unweighted_maximum_is_the_clipped_max_lateness(nodes, released):
    """With integer data the unweighted maximum tardiness is max(+0, L_max), L_max from ref_max_lateness (its tail
    makespan minus max d)."""
    J = 20
    T, valid = R.synth_table(J, 1, 8, seed=9, masked=False)
    tab = np.ceil(R.canon_table(T, range(1, 9))).astype(np.float32)
    opt, prio = R.synth_candidates(J, 500, valid, seed=10)
    if nodes > 1:
        opt = (opt | (np.random.default_rng(11).integers(0, nodes, size=opt.shape) << 3)).astype(np.uint8)
    d = _due(J, 12, 2000.0 * J / 8, integer=True)
    r = np.round(np.random.default_rng(13).uniform(-10, 3000, size=J)) if released else None
    signs = set()
    for shift in (0.0, 6.0e4, 2.0e5):                             # late, mixed, and every candidate on time
        got = MT.evaluate(tab, opt, prio, d + shift, r, True, np.float32, nodes=nodes)
        lmax = ML.evaluate(tab, opt, prio, d + shift, r, True, np.float32, nodes=nodes).astype(np.float64) - \
            float((d + shift).max())
        assert np.array_equal(got.astype(np.float64), np.maximum(lmax, 0.0))
        signs |= set(np.sign(lmax).tolist())
    assert {-1.0, 1.0} <= signs


@pytest.fixture(scope="module")
def cases():
    with open(os.path.join(HERE, "golden", "max_tardiness_cases.json")) as f:
        return json.load(f)["cases"]


def test_milp_fixtures_match_the_exhaustive_optimum(cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum to 1e-9 relative; where HiGHS stopped at
    its time limit, the exhaustive optimum is no worse than the incumbent.  Every MILP plan is feasible and its score
    is its objective value, the fp32 and fp64 optima agree to fp32 rounding, and the fixtures include weighted
    instances, instances with release dates and stretch instances."""
    proven = 0
    for rec in cases:
        m, bf = rec["milp"], rec["bruteforce_f64"]["score"]
        assert m["start"] is not None and m["feasible"] and m["overlaps"] == 0, rec["name"]
        assert m["score"] == pytest.approx(m["objective_value"], rel=1e-6, abs=1e-6), rec["name"]
        assert rec["bruteforce_f32"]["score"] == pytest.approx(bf, rel=1e-6), rec["name"]
        if m["proven_optimal"]:
            proven += 1
            assert abs(m["score"] - bf) <= 1e-9 * max(1.0, abs(bf)), rec["name"]
        else:
            assert bf <= m["score"] * (1 + 1e-9), rec["name"]
    assert proven >= len(cases) // 2
    assert sum(rec["weights"] is not None and not rec["stretch"] for rec in cases) >= 10
    assert sum(rec["release"] is not None for rec in cases) >= 4
    assert sum(rec["stretch"] for rec in cases) >= 8


def test_fixture_plans_rescore_to_their_recorded_values(cases):
    """The recorded exhaustive optima and the tardiness- and makespan-optimal flags re-derive from the oracle; a
    stretch instance's weights and due dates are fp32(1 / p*) and max(r, 0), and its optimum is >= 1."""
    from oracle.gen_max_tardiness import stretch_form
    for rec in cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        for key, dtype in (("bruteforce_f64", np.float64), ("bruteforce_f32", np.float32)):
            b = rec[key]
            got = MT.evaluate(tab, np.array([b["opt"]], np.uint8), np.array([b["prio"]], np.uint8), rec["due"],
                              rec["release"], True, dtype, weights=rec["weights"])[0]
            assert float(got) == b["score"], (rec["name"], key)
        best = rec["bruteforce_f64"]["score"]
        for k in ("tardiness_optimum", "makespan_optimum"):
            assert rec[k]["is_optimal"] == (rec[k]["score"] <= best * (1 + 1e-9) + 1e-12)
            assert rec[k]["score"] >= best * (1 - 1e-9)
        if rec["stretch"]:
            w, d = stretch_form(tuples, rec["release"])
            assert rec["weights"] == w and rec["due"] == d
            assert best >= 1.0 - 1e-6


def test_lpt_seeds_are_the_tardiness_seeds():
    """lpt_seeds(objective="max_tardiness" / "weighted_max_tardiness") plants the EDD seeds of "tardiness" /
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
            for obj, base in (("max_tardiness", "tardiness"), ("weighted_max_tardiness", "weighted_tardiness")):
                a = lpt_seeds(tmin, objective=obj, due=d, release=r, nodes=nodes, weights=w)
                b = lpt_seeds(tmin, objective=base, due=d, release=r, nodes=nodes, weights=w)
                for (ca, oa), (cb, ob) in zip(a, b):
                    assert np.array_equal(ca, cb) and np.array_equal(oa, ob)
            u = lpt_seeds(tmin, objective="max_tardiness", due=d, release=r, nodes=nodes, weights=w)
            v = lpt_seeds(tmin, objective="weighted_max_tardiness", due=d, release=r, nodes=nodes, weights=w)
            if not released:  # distinct release dates decide the whole order
                assert any(not np.array_equal(x[1], y[1]) for x, y in zip(u, v))


def test_stretch_seed_is_shortest_first_on_one_machine():
    """All jobs released at 0 on one machine (every job on all 8 GPUs): the weighted EDD seed with w = 1 / p* and
    d = 0 orders by ascending rt * p* = p*^2, i.e. shortest first, and that order's max stretch is the exhaustive
    optimum (the adjacent-exchange argument of DESIGN.md)."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(21)
    for _ in range(8):
        J = 6
        p = rng.integers(1, 40, size=J).astype(np.float32)
        tab = np.full((J, 1, 8), np.inf, dtype=np.float32)
        tab[:, 0, 7] = p
        w = (1.0 / p.astype(np.float64)).astype(np.float32)
        tmin = np.full((J, 8), np.inf, dtype=np.float32)
        tmin[:, 7] = p
        (ob, order), = lpt_seeds(tmin, objective="weighted_max_tardiness", due=np.zeros(J, np.float32), weights=w)[:1]
        assert np.array_equal(order, np.lexsort((np.arange(J), p)))
        best, _, _ = MT.brute_force(tab, [[7]] * J, np.zeros(J), weights=w)
        got = MT.evaluate(tab, ob[None, :].astype(np.uint8), order[None, :].astype(np.uint8), np.zeros(J), None,
                          True, np.float64, weights=w)
        assert float(got[0]) == best


class _Strat:
    def __init__(self, runtime, executor="x"):
        self.runtime, self.executor = runtime, executor


class _Task:
    def __init__(self, name, runtimes=(100.0, 60.0), sentinel=()):
        self.name = name
        self.strategies = {g: _Strat(rt, None if g in sentinel else "x") for g, rt in zip((1, 2), runtimes)}


@pytest.mark.parametrize("kw,match", [
    ({"weights": [1.0, 1.0, 1.0]}, "takes no weights"),
    ({"due": [1.0, 2.0, 3.0]}, "takes no due dates"),
    ({"hysteresis": True}, "hysteresis"),
    ({"runtimes": (0.0, 60.0)}, "undefined"),
    ({"runtimes": (1e-36, 60.0)}, "overflows"),
    ({"release": [0.0, float("inf"), 1.0]}, None),
])
def test_solver_refusals_before_any_device_call(kw, match):
    """solve() and solve_table() refuse these with SolverError before they touch a device (this runs without one):
    weights, due dates, hysteresis, a fastest runtime of 0, a reciprocal that overflows fp32 at 2^24, a bad release."""
    from saturn_b200 import solver as S
    kw = dict(kw)
    runtimes = kw.pop("runtimes", (100.0, 60.0))
    tasks = [_Task("a"), _Task("b", runtimes), _Task("c")]
    with pytest.raises(S.SolverError, match=match):
        S.solve(tasks, None, objective="max_stretch", engine=object(), **kw)
    if "hysteresis" not in kw:  # solve_table has no hysteresis
        T = np.full((3, 1, 8), np.inf, dtype=np.float32)
        T[:, 0, :2] = [100.0, 60.0]
        T[1, 0, :2] = runtimes
        with pytest.raises(S.SolverError, match=match):
            S.solve_table(T, objective="max_stretch", engine=object(), **kw)


def test_stretch_form_and_stats():
    """p* is the smallest cell the search may propose (a sentinel-only task keeps its sentinel cell), the weights are
    fp32(1 / p*) from float64, the due dates max(r32, +0); the stats are float64 stretches."""
    from saturn_b200 import solver as S
    Tdev = np.full((3, 2, 8), np.inf, dtype=np.float32)
    Tdev[0, 0, :3] = [300.0, 170.0, 3.0e5]
    Tdev[0, 1, 1] = 150.0                                         # a second strategy is faster
    Tdev[1, 0, 0] = 1.0e6                                         # sentinel only: it is what the search uses
    Tdev[2, 1, 7] = 7.0
    pstar, w32, d32 = S._stretch_form(Tdev, np.array([-5.0, 0.0, 12.5], np.float32))
    assert pstar.tolist() == [150.0, 1.0e6, 7.0]
    assert w32.dtype == np.float32 and w32.tolist() == [float(np.float32(1.0 / p)) for p in (150.0, 1.0e6, 7.0)]
    assert d32.dtype == np.float32 and d32.tolist() == [0.0, 0.0, 12.5] and not np.signbit(d32).any()
    _, _, dz = S._stretch_form(Tdev, None)
    assert dz.tolist() == [0.0, 0.0, 0.0]
    st = S._stretch_stats([0.0, 10.0, 20.0], [150.0, 1.0e6, 7.0], pstar, [-5.0, 0.0, 12.5])
    want = [1.0, (10.0 + 1.0e6) / 1.0e6, (27.0 - 12.5) / 7.0]
    assert st["max_stretch"] == max(want) and st["mean_stretch"] == pytest.approx(sum(want) / 3, rel=1e-15)

    class Eng:
        def __getattr__(self, name):
            return lambda *a, **k: None
    assert S._set_objective(Eng(), "max_stretch", w32, d32) == "weighted_max_tardiness"


def test_engine_objective_flags():
    from saturn_b200 import _lib
    from saturn_b200.engine import OBJECTIVES, _require_due, objective_flag
    from saturn_b200.solver import SolverError
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE | _lib.FLAG_MAX_TARDINESS
    assert objective_flag("max_tardiness") == base
    assert objective_flag("weighted_max_tardiness") == base | _lib.FLAG_WEIGHTED
    assert {"max_tardiness", "weighted_max_tardiness"} <= set(OBJECTIVES)
    for obj in ("max_tardiness", "weighted_max_tardiness"):
        with pytest.raises(SolverError):
            _require_due(None, obj)


def test_orchestrate_shifts_release_dates_under_max_stretch(monkeypatch):
    """orchestrate() hands the solve for interval n the release dates r - n * interval under objective="max_stretch"."""
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
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), kw["objective"], dict(kw["release"]), "due" in kw))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", lambda task_list, *a: ({}, {}, [0.0] * len(task_list)))
    O.orchestrate(tasks, interval=1000, solver_kwargs={"objective": "max_stretch", "release": release})
    assert [n for n, _, _, _ in seen] == [2, 1, 1]
    for n, (_, obj, got, has_due) in enumerate(seen):
        assert obj == "max_stretch" and not has_due and got == {t: r - n * 1000 for t, r in release.items()}


def test_flag_max_tardiness_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_MAX_TARDINESS\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_MAX_TARDINESS == 4096
    flags = [v for k, v in vars(_lib).items() if k.startswith("FLAG_") and k != "FLAG_MAX_TARDINESS"]
    assert all(f & _lib.FLAG_MAX_TARDINESS == 0 for f in flags)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_MAX_TARDINESS == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_MAX_TARDINESS" in f.read().split("the test hooks share no bit")[0]
