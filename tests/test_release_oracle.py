"""CPU: release dates (SB_FLAG_RELEASE) in the oracle — the Python schedule and folds against the C port bit for bit,
the r <= 0 identities against the existing oracles, plan feasibility and start >= r, the release MILP fixtures
(tests/golden/release_cases.json, oracle/gen_release.py), the dominance of list schedules on their plans, the
seed orders, solve() / solve_table() / orchestrate() release handling without a device, and the flag against the
header."""
import json
import math
import os
import re

import numpy as np
import pytest

from oracle import ref_completion as RC, ref_eval as R, ref_release as RR, ref_tardiness as RT, ref_weighted as RW

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FOLDS = RR.OBJECTIVES


@pytest.fixture(scope="module")
def release_cases():
    with open(os.path.join(HERE, "golden", "release_cases.json")) as f:
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


def _per_job(J, fold, seed, scale):
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 20.0, size=J) if fold.startswith("weighted") else None
    d = rng.uniform(-0.2, 2.0, size=J) * scale if fold.endswith("tardiness") else None
    return w, d


def _release(J, seed, scale):
    """Real release dates over the schedule's span, a few negative (already released)."""
    return np.random.default_rng(seed).uniform(-0.1, 1.0, size=J) * scale


@pytest.mark.parametrize("J,S,nodes", [(7, 3, 1), (40, 4, 1), (23, 1, 3)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("fold", FOLDS)
def test_python_equals_c_port(J, S, nodes, ints, dtype, fold):
    """The release schedule and every score fold give the same bits in Python and in C: fp32 and fp64, one node and
    three, integer and real-valued starts."""
    B = 24
    tab, opt, prio = _candidates(J, S, B, nodes, seed=J + 5 * nodes)
    scale = 2000.0 * J / 8
    r = _release(J, J + 1, scale)
    w, d = _per_job(J, fold, J + 2, scale)
    tot, start, mask = RR.c_evaluate(tab, opt, prio, r, ints, dtype, nodes=nodes, want_plan=True, objective=fold,
                                     weights=w, due=d)
    for b in range(B):
        s, st, m, _ = RR.list_schedule(tab, opt[b], prio[b], r, ints, dtype, nodes=nodes, objective=fold, weights=w,
                                       due=d)
        assert np.asarray(s, dtype).tobytes() == np.asarray(tot[b], dtype).tobytes(), (b, s, tot[b])
        assert np.array_equal(np.asarray(st, dtype), start[b])
        assert np.array_equal(np.asarray(m, np.uint32), mask[b])
    if nodes == 1:
        bt, bs, bm = RR.list_schedule_batch(tab, opt, prio, r, ints, dtype, want_plan=True, objective=fold, weights=w,
                                            due=d)
        assert np.array_equal(bt, tot) and np.array_equal(bs, start) and np.array_equal(bm, mask)


@pytest.mark.parametrize("nodes", [1, 3])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("sign", [0.0, -1.0])
def test_released_jobs_change_nothing(nodes, ints, dtype, sign):
    """r = 0 and all-negative r give exactly the scores of ref_eval (makespan), ref_completion, ref_weighted and
    ref_tardiness, and their starts and slot masks."""
    J, B = 19, 32
    tab, opt, prio = _candidates(J, 1 if nodes > 1 else 3, B, nodes, seed=11 * nodes)
    r = sign * np.random.default_rng(4).uniform(0.5, 5000.0, size=J)
    w = np.random.default_rng(5).uniform(0.1, 9.0, size=J)
    d = np.random.default_rng(6).uniform(-100.0, 3000.0, size=J)
    mk, st, m = R.list_schedule(tab, opt[0], prio[0], ints, dtype, nodes=nodes)[:3]
    got = RR.list_schedule(tab, opt[0], prio[0], r, ints, dtype, nodes=nodes)
    assert got[0] == mk and list(got[1]) == list(st) and list(got[2]) == list(m)
    ref = {"completion": RC.c_evaluate(tab, opt, prio, ints, dtype, nodes=nodes),
           "weighted_completion": RW.c_evaluate(tab, opt, prio, ints, dtype, nodes=nodes, weights=w),
           "tardiness": RT.c_evaluate(tab, opt, prio, d, ints, dtype, nodes=nodes),
           "weighted_tardiness": RT.c_evaluate(tab, opt, prio, d, ints, dtype, nodes=nodes, weights=w)}
    for fold, want in ref.items():
        got = RR.c_evaluate(tab, opt, prio, r, ints, dtype, nodes=nodes, objective=fold,
                            weights=w if fold.startswith("weighted") else None, due=d)
        assert got.tobytes() == want.astype(dtype).tobytes(), fold
    if nodes == 1:
        mkb = R.list_schedule_batch(tab, opt, prio, ints, dtype)
        assert RR.list_schedule_batch(tab, opt, prio, r, ints, dtype).tobytes() == mkb.tobytes()


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("fractional", [False, True])
def test_plans_are_feasible_and_start_after_release(ints, fractional):
    """Every oracle plan passes check_plan (fp32 with real-valued starts aside: its slot times are rounded), and every
    start is >= r (>= ceil(r) with integer starts)."""
    J, B = 12, 40
    tab, opt, prio = _candidates(J, 3, B, 1, seed=21)
    rng = np.random.default_rng(22)
    r = rng.integers(0, 3000, size=J).astype(float) + (rng.uniform(0, 1, size=J) if fractional else 0.0)
    for dtype in (np.float32, np.float64):
        _tot, start, mask = RR.list_schedule_batch(tab, opt, prio, r, ints, dtype, want_plan=True)
        for b in range(B):
            k = [(int(opt[b, j]) & 7) + 1 for j in range(J)]
            rt = [float(tab[j, int(opt[b, j]) >> 3, int(opt[b, j]) & 7]) for j in range(J)]
            if ints or dtype == np.float64:  # fp32 real-valued ends round to the nearest fp32, a hair early
                ok, ov, _ = R.check_plan([float(x) for x in start[b]], mask[b], rt, k, integer_starts=ints)
                assert ok and ov == 0
            for j in range(J):
                assert float(start[b, j]) >= r[j]
                if ints:
                    assert float(start[b, j]) >= math.ceil(r[j])


def test_release_as_rounds_up():
    r = np.array([0.1, 1.0 / 3.0, 2.0 ** 23 + 0.5, -0.7, 5.0])
    r32 = RR.release_as(r, 5, np.float32, False)
    assert (r32.astype(np.float64) >= r).all()
    assert list(RR.release_as(r, 5, np.float32, True)) == [1.0, 1.0, 2.0 ** 23 + 1, 0.0, 5.0]
    assert not np.signbit(RR.release_as(r, 5, np.float32, True)).any()


def test_milp_fixtures_match_the_exhaustive_optimum(release_cases):
    """Every proven MILP optimum equals the exhaustive list-schedule optimum to 1e-9; where HiGHS stopped at its time
    limit, the exhaustive optimum is no worse than its incumbent.  Each recorded plan is feasible and starts every
    task at or after its release date."""
    proven = {o: 0 for o in ("makespan", "completion")}
    differs = {o: 0 for o in ("makespan", "completion")}
    for rec in release_cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        r = rec["release"]
        for o in proven:
            bf = RR.brute_force(tab, optmap, r, o, integer_starts=True, dtype=np.float64)[0]
            assert bf == rec[o]["bruteforce_f64"]["score"], rec["name"]
            bf32 = RR.brute_force(tab, optmap, r, o, integer_starts=True, dtype=np.float32)[0]
            assert bf32 == rec[o]["bruteforce_f32"]["score"], rec["name"]
            differs[o] += rec["differs"][o]
            m = rec[o]["milp"]
            if m["start"] is None:
                continue
            assert m["feasible"] and m["overlaps"] == 0, rec["name"]
            for t in range(J):
                assert m["start"][t] >= math.ceil(r[t]) - 1e-9, (rec["name"], t)
            if m["proven_optimal"]:
                proven[o] += 1
                assert bf == pytest.approx(m["score"], rel=1e-9, abs=1e-9), (rec["name"], o)
            else:
                assert bf <= m["score"] * (1 + 1e-9), (rec["name"], o)
    print("release fixtures: proven optimal %s of %d, differs %s" % (proven, len(release_cases), differs))
    assert len(release_cases) == 24
    assert sum(rec["fractional"] for rec in release_cases) == 4
    assert min(proven.values()) >= len(release_cases) // 2
    assert min(differs.values()) >= len(release_cases) // 2


def test_list_schedules_dominate_the_release_milp_plans(release_cases):
    """DESIGN.md §3.1, *Release dates*: ordering a feasible plan's jobs by start and running the list rule with the
    release and its options starts every job no later, so no objective here gets worse."""
    n = 0
    for rec in release_cases:
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, optmap = R.table_from_tuples(tuples)
        J = len(tuples)
        for o in ("makespan", "completion"):
            m = rec[o]["milp"]
            if m["start"] is None:
                continue
            opt = [optmap[t][m["opt_idx"][t]] for t in range(J)]
            order = sorted(range(J), key=lambda t: (m["start"][t], t))
            score, start, _, _ = RR.list_schedule(tab, opt, order, rec["release"], True, np.float64, objective=o)
            for t in range(J):
                assert start[t] <= m["start"][t] + 1e-9, (rec["name"], o, t)
            assert score <= m["score"] * (1 + 1e-12) + 1e-9
            n += 1
    assert n >= 24


def test_release_seeds_follow_the_release_order():
    """lpt_seeds(release=) re-sorts each seed's order stably by ascending release date (ceiled with integer starts):
    jobs released together keep the objective's order."""
    from saturn_b200.search import lpt_seeds
    rng = np.random.default_rng(7)
    J = 48
    tmin = rng.uniform(10, 1000, size=(J, 8)).astype(np.float32)
    tmin[:, 6:] = np.inf
    r = (rng.integers(0, 4, size=J) * 100 + rng.choice([0.0, 0.5], size=J)).astype(np.float32)
    for objective in ("makespan", "completion"):
        for ints in (True, False):
            plain = lpt_seeds(tmin, objective=objective)
            rel = np.ceil(r) if ints else r
            for (col, order), (pcol, porder) in zip(lpt_seeds(tmin, objective=objective, release=r,
                                                              integer_starts=ints), plain):
                assert np.array_equal(col, pcol)
                rank = {j: i for i, j in enumerate(porder)}
                keys = [(rel[j], rank[j]) for j in order]
                assert keys == sorted(keys)


class _Task:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("release", [[1.0, 2.0], [1.0, 2.0, 3.0, 4.0], [1.0, float("nan"), 2.0],
                                     [1.0, float("inf"), 2.0], [1.0, 2.0 ** 24, 2.0], [1.0, -2.0 ** 24, 2.0],
                                     [1.0, 2.0 ** 24 - 0.5, 2.0], "abc", 3.0])
@pytest.mark.parametrize("objective", ["makespan", "completion"])
def test_solver_validates_release_dates_before_any_device_call(release, objective):
    """solve() and solve_table() refuse malformed release dates with SolverError before they touch a device (this
    runs without one): wrong length, not finite, |r| >= 2^24 (also once rounded up to fp32), not a sequence."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b"), _Task("c")]
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective=objective, release=release, engine=object())
    T = np.ones((3, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError):
        S.solve_table(T, objective=objective, release=release, engine=object())


def test_solver_refusals():
    """A task missing from the mapping, a mapping for solve_table and hysteresis=True together with `release` raise
    SolverError before any device call."""
    from saturn_b200 import solver as S
    tasks = [_Task("a"), _Task("b")]
    T = np.ones((2, 1, 8), dtype=np.float32)
    with pytest.raises(S.SolverError, match="no entry"):
        S.solve(tasks, None, release={tasks[0]: 1.0}, engine=object())
    with pytest.raises(S.SolverError):
        S.solve_table(T, release={0: 1.0, 1: 2.0}, engine=object())
    with pytest.raises(S.SolverError, match="hysteresis"):
        S.solve(tasks, None, release=[1.0, 2.0], hysteresis=True, engine=object())
    with pytest.raises(S.SolverError):
        S.solve(tasks, None, objective="tardiness", due=[1.0, 2.0], release=[1.0, float("nan")], engine=object())


def test_release_f32_rounds_up():
    from saturn_b200.engine import release_f32
    r = [0.1, 1.0 / 3.0, -0.7, 7.0, 1e7 + 0.3]
    r32 = release_f32(r, 5)
    assert r32.dtype == np.float32
    assert (r32.astype(np.float64) >= np.asarray(r)).all()
    assert r32[3] == 7.0


def test_orchestrate_shifts_release_dates_by_the_interval(monkeypatch):
    """orchestrate() hands the solve for interval n the release dates r - n * interval, and refuses a sequence."""
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
    release = {tasks[0]: 0.0, tasks[1]: 1500.0}
    seen = []

    def fake_solve(task_list, presolved, **kw):
        seen.append((len(task_list), dict(kw["release"])))
        return [[[0.0] * len(task_list)]], None, None, None, None, 1.0

    def fake_convert(task_list, *a):
        return {}, {}, [0.0] * len(task_list)

    monkeypatch.setattr(O, "solve", fake_solve)
    monkeypatch.setattr(O, "convert_into_comprehensible", fake_convert)
    O.orchestrate(tasks, interval=1000, solver_kwargs={"release": release})
    assert [n for n, _ in seen] == [2, 1, 1]
    for n, (_, got) in enumerate(seen):
        assert got == {t: r - n * 1000 for t, r in release.items()}
    with pytest.raises(SolverError):
        O.orchestrate(tasks, interval=1000, solver_kwargs={"release": [1.0, 2.0]})


def test_flag_release_matches_the_header():
    from saturn_b200 import _lib
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    m = re.search(r"#define\s+SB_FLAG_RELEASE\s+(\d+)u", header)
    assert m and int(m.group(1)) == _lib.FLAG_RELEASE == 512
    assert "sb_set_release" in _lib.SYMBOLS and re.search(r"int\s+sb_set_release\s*\(", header)
    hooks = [v for k, v in vars(_lib).items() if k.startswith("HOOK_")]
    assert all(h & _lib.FLAG_RELEASE == 0 for h in hooks)
    with open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")) as f:
        assert "SB_FLAG_RELEASE" in f.read().split("the test hooks share no bit")[0]
