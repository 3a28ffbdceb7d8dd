"""GPU: release dates (SB_FLAG_RELEASE, solve(release=...)) — bit-exact scores on every kernel path against the fp32
oracle under every objective, r = 0 identical to the flag-less run, starts and slot masks of eval_full / decode,
arg-min keys, the refusals, incremental rounds, solve()'s plans, orchestrate() and reproducibility."""
import json
import math
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_release as RR
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1
FOLDS = RR.OBJECTIVES


def _setup(engine, tab, opt, prio, fold, seed, nodes=1):
    """fp32 release dates over the first candidate's makespan (a few negative: already released), and the weights
    and due dates the fold needs; returns (r, w, d)."""
    J = tab.shape[0]
    o, p = opt[:1].cpu().numpy(), prio[:1].cpu().numpy()
    span = float(RR.c_evaluate(tab, o, p, np.zeros(J), True, np.float64, nodes=nodes)[0])
    rng = np.random.default_rng(seed)
    r = (rng.uniform(-0.1, 0.8, size=J) * span).astype(np.float32)
    w = rng.uniform(0.1, 12.0, size=J).astype(np.float32) if fold.startswith("weighted") else None
    d = (rng.uniform(0.0, 1.5, size=J) * span).astype(np.float32) if fold.endswith("tardiness") else None
    engine.set_release(r)
    if w is not None:
        engine.set_weights(w)
    if d is not None:
        engine.set_due(d)
    return r, w, d


def _ref(tab, opt, prio, ints, fold, r, w, d, nodes=1, want_plan=False):
    return RR.c_evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), r, ints, np.float32, threads=8, nodes=nodes,
                         objective=fold, weights=w, due=d, want_plan=want_plan)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _check_runs(engine, opt, prio, ref, fold, runs, **common):
    """Every run: the score equals the oracle bit for bit on the path asked for, with the arg-min key; the release
    dates change the scores.  Then r = 0 under the flag gives exactly the flag-less run's scores, keys and path.
    Leaves the release dates set."""
    r = engine.release.copy()
    assert (ref < np.inf).all()
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, fold, **common, **kw)
        assert path is None or p == path, (kw, p)
        assert got.tobytes() == ref.tobytes(), kw
        assert key == _key_of(ref, 11), kw
    plain = {}
    engine.set_release(None)
    for i, (kw, _path) in enumerate(runs):
        plain[i] = _eval(engine, opt, prio, fold, **common, **kw)
    assert plain[0][0].tobytes() != ref.tobytes()
    engine.set_release(np.zeros(engine.J, np.float32))
    for i, (kw, _path) in enumerate(runs):
        got = _eval(engine, opt, prio, fold, **common, **kw)
        assert got[0].tobytes() == plain[i][0].tobytes() and got[1:] == plain[i][1:], kw
    engine.set_release(r)


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("fold", FOLDS)
def test_release_on_the_tile_and_generic_paths(engine, J, S, B, ints, fold):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities, and sb_eval_host."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    r, w, d = _setup(engine, tab, opt, prio, fold, J)
    ref = _ref(tab, opt, prio, ints, fold, r, w, d)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, fold, runs, integer_starts=ints)
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), fold, integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective=fold)
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("fold", ["makespan", "completion", "weighted_tardiness"])
def test_release_with_large_tables(engine, ints, fold):
    """J = 1024 with the full 8-strategy table: paths 9, 4 and 0 on job-indexed rows; J = 256: the position-major
    kernel with its table in shared memory (5), split over a CTA pair (7) and in global memory (8)."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    r, w, d = _setup(engine, tab, opt, prio, fold, 5)
    ref = _ref(tab, opt, prio, ints, fold, r, w, d)
    _check_runs(engine, opt, prio, ref, fold, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)],
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    r, w, d = _setup(engine, tab, opt, prio, fold, 9)
    ref = _ref(tab, opt, prio, ints, fold, r, w, d)
    obp = opt_by_position(opt, prio)
    _check_runs(engine, obp, prio, ref, fold, [({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)],
                integer_starts=ints, by_position=True)
    got, key, p = _eval(engine, opt, prio, fold, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref) and key == _key_of(ref, 11)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("fold", ["makespan", "completion", "weighted_tardiness"])
def test_release_multi_node_and_decode(engine, J, nodes, B, ints, fold):
    """1..4 nodes: every path equals the oracle; sb_eval_full and sb_decode give the oracle's starts and slot masks,
    every start is >= r (>= ceil(r) with integer starts), and r = 0 gives the flag-less starts and masks."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    r, w, d = _setup(engine, tab, opt, prio, fold, J + nodes, nodes)
    ref, rstart, rmask = _ref(tab, opt, prio, ints, fold, r, w, d, nodes, want_plan=True)
    runs = [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, fold, runs, integer_starts=ints, reduced=True)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=fold)
    assert np.array_equal(tot.cpu().numpy(), ref)
    assert np.array_equal(start.cpu().numpy(), rstart)
    assert np.array_equal(mask.cpu().numpy().astype(np.uint32), rmask)
    lo = np.ceil(r) if ints else r
    assert (start.cpu().numpy() >= lo[None, :]).all()
    b = B // 3
    o, p = opt[b].cpu().numpy(), prio[b].cpu().numpy()
    dec = engine.decode(o, p, integer_starts=ints, reduced=True, objective=fold)
    assert dec["makespan"] == float(ref[b])
    assert np.array_equal(dec["start"], rstart[b]) and np.array_equal(dec["slotmask"], rmask[b] & 0xffff)
    assert np.array_equal(dec["node"], (rmask[b] >> 16).astype(np.uint8))
    engine.set_release(np.zeros(J, np.float32))
    z = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=fold)
    engine.set_release(None)
    n = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=fold)
    for a, c in zip(z, n):
        assert a.cpu().numpy().tobytes() == c.cpu().numpy().tobytes()


def test_refusals(engine):
    """The flag before set_release and after set_table cleared the dates (SB_ERR_STATE), set_release with a bad
    value or the wrong J (SB_ERR_ARG), the alternate shape, and the Python refusals."""
    from saturn_b200 import _lib
    from saturn_b200._lib import SaturnB200Error, check
    from saturn_b200.solver import SolverError
    import ctypes as C
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_RELEASE) == -3                         # no release dates yet
    engine.set_release(np.arange(J, dtype=np.float32))
    for extra in (0, _lib.FLAG_SUM_COMPLETION):
        assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_RELEASE | extra) == 0
    assert raw(_lib.FLAG_RELEASE | _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE) == -3          # due dates missing
    with pytest.raises(SaturnB200Error, match="ALT_WARPSCAN"):
        engine.eval(opt, prio, alt_shape=True)
    engine.set_table(T)                                                                     # clears them
    assert engine.release is None
    assert raw(_lib.FLAG_INTEGER_STARTS | _lib.FLAG_RELEASE) == -3
    p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | _lib.FLAG_RELEASE, t_start=0.01, t_end=1e-4,
                          total_rounds=4)
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
    for bad in ([np.nan] + [1.0] * (J - 1), [np.inf] + [1.0] * (J - 1), [2.0 ** 24] + [1.0] * (J - 1),
                [-2.0 ** 24] + [1.0] * (J - 1)):
        rr = np.array(bad, np.float32)
        assert engine._lib.sb_set_release(engine._h, C.c_void_p(rr.ctypes.data), J) == -1
    rr = np.zeros(J + 1, np.float32)
    assert engine._lib.sb_set_release(engine._h, C.c_void_p(rr.ctypes.data), J + 1) == -1
    with pytest.raises(SolverError):
        engine.set_release(np.zeros(J - 1))
    with pytest.raises(SolverError):
        engine.set_release([float("nan")] * J)
    check(engine._lib.sb_set_release(engine._h, None, 0))
    from saturn_b200 import solver as S
    tasks = tasks_from_tuples([[(1, 10.0)], [(2, 20.0)]])
    with pytest.raises(SolverError, match="hysteresis"):
        S.solve(tasks, None, release=[0.0, 5.0], hysteresis=True)
    with pytest.raises(SolverError):
        S.solve(tasks, None, release=[0.0])


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
@pytest.mark.parametrize("objective", ["makespan", "completion"])
def test_incremental_rounds_with_release_dates(engine, J, objective):
    """The verify hook recomputes every incremental score from position 0: no mismatch with the running score stored
    in the snapshots.  The search returns valid plans that re-score to the reported value."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    r = (np.random.default_rng(J).uniform(0.0, 0.6, size=J) * horizon).astype(np.float32)
    engine.set_release(r)
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, **({"objective": objective} if objective != "makespan" else {}))
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    for res in (a, b):
        assert sorted(res.prio.tolist()) == list(range(J))
        assert float(RR.list_schedule(tmin, res.opt, res.prio, r, True, np.float32, objective=objective)[0]) == \
            res.makespan


def _cases():
    with open(os.path.join(HERE, "golden", "release_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, _ = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    return [p[0] for p in plan], [p[0] + p[2] for p in plan]        # start and completion time per task


def _device_table(tuples):
    tab, om = R.table_from_tuples(tuples)
    tab32 = np.where(np.isfinite(tab), tab.astype(np.float32), np.inf)
    up = tab32.astype(np.float64) < tab
    tab32[up] = np.nextafter(tab32[up], np.float32(np.inf))
    return tab32, om


@pytest.mark.parametrize("objective", ["makespan", "completion"])
def test_solve_reaches_the_release_fixture_optimum(objective):
    """On every fixture, solve(release=...) returns a feasible plan that starts no task before its release and whose
    makespan / sum of completion times equals the exhaustive optimum; last_stats holds the total flow time."""
    from saturn_b200 import solver as S
    for rec in _cases():
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        r = rec["release"]
        out = S.solve(tasks, None, chains=8192, rounds=60, objective=objective, release=r)
        start, comp = _plan(tasks, out)
        for t in range(len(tasks)):
            assert start[t] >= math.ceil(r[t])
        score = max(comp) if objective == "makespan" else sum(comp)
        assert score == pytest.approx(rec[objective]["bruteforce_f64"]["score"], rel=1e-9, abs=1e-9), rec["name"]
        assert S.last_stats["total_flow_time"] == pytest.approx(sum(c - max(x, 0.0) for c, x in zip(comp, r)),
                                                                rel=1e-12)


def test_solve_reaches_the_exhaustive_optimum_on_random_small_instances():
    """Random 2..5-task instances with random release dates under all objectives, on one and two nodes: the device's
    fp32 score equals the fp32 exhaustive optimum and the plan is feasible."""
    from saturn_b200 import solver as S
    rng = np.random.default_rng(31)
    for trial in range(16):
        nodes = 1 if trial % 2 == 0 else 2
        J = int(rng.integers(2, 6 if nodes == 1 else 5))
        tuples = []
        for _ in range(J):
            ks = sorted(rng.choice([1, 2, 4, 8], size=int(rng.integers(1, 3 if nodes > 1 else 4)), replace=False).tolist())
            base = float(rng.uniform(20, 900))
            tuples.append([(int(k), base * float(rng.uniform(1, 1.3)) / k ** float(rng.uniform(0.4, 1.0))) for k in ks])
        r = rng.integers(-50, 900, size=J).astype(float) + (0.5 if trial % 3 == 0 else 0.0)
        objective = ("makespan", "completion", "tardiness")[trial % 3]
        d = rng.integers(0, 1500, size=J).astype(float) if objective == "tardiness" else None
        tasks = tasks_from_tuples(tuples)
        out = S.solve(tasks, None, chains=4096, rounds=64, nodes=nodes, seed=trial, objective=objective, release=r,
                      due=d)
        assert R.milp_constraints_hold(tuples, *out) == [], trial
        tab32, om = _device_table(tuples)
        if nodes > 1:
            tab32 = R.reduce_table(tab32)[0][:, None, :]
            om = [[o & 7 for o in ops] for ops in om]
        best = RR.brute_force(tab32, om, r, objective, True, dtype=np.float32, nodes=nodes, due=d)[0]
        assert S.last_stats["device_makespan"] == best, (trial, J, nodes, tuples, r)


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_release_plan_is_reproducible_and_respects_the_release():
    """J = 256 with seeded release dates: every start is >= ceil(r), and the same call twice returns the identical
    plan and statistics."""
    from saturn_b200 import solver as S
    tasks = _tasks256()
    J = len(tasks)
    kw = dict(chains=16384, rounds=120, seed=1)
    plain = S.solve(tasks, None, **kw)
    r = np.random.default_rng(5).uniform(0, 0.5 * plain[5], size=J)
    a = S.solve(tasks, None, release=r, **kw)
    start, comp = _plan(tasks, a)
    assert all(s >= math.ceil(x) for s, x in zip(start, r))
    flow = S.last_stats["total_flow_time"]
    assert flow == pytest.approx(sum(c - x for c, x in zip(comp, r)), rel=1e-12)
    a2 = S.solve(tasks, None, release=r, **kw)
    assert all(x == y for x, y in zip(a[:5], a2[:5])) and a2[5] == a[5]
    assert S.last_stats["total_flow_time"] == flow


def test_orchestrate_with_release_dates_keyed_by_task(monkeypatch):
    """A release mapping keyed by Task survives orchestrate()'s shrinking task list, and no simulated launch comes
    before its task's release: a task launched in interval n at plan start st begins at n * interval + st >= r."""
    from saturn_b200 import orchestrate, orchestrator as O
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    release = {t: float(700 * i) for i, t in enumerate(tasks)}
    plans = []
    real = O.convert_into_comprehensible

    def spy(task_list, *a):
        out = real(task_list, *a)
        plans.append(dict(zip(task_list, out[2])))
        return out
    monkeypatch.setattr(O, "convert_into_comprehensible", spy)
    recs = orchestrate(tasks, interval=1000, solver_kwargs={"chains": 4096, "rounds": 25, "release": release},
                       max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)
    launched = 0
    for n, rec in enumerate(recs):
        for name in rec["launched"]:
            t = next(x for x in tasks if x.name == name)
            assert n * 1000 + plans[n][t] >= release[t] - 1e-9, (n, name)
            launched += 1
    assert launched >= 8


def test_multiple_devices_equal_single_device_runs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200.engine import Engine, MultiEngine
    J, S = 96, 4
    T, valid = R.synth_table(J, S, 8, seed=2)
    r = np.random.default_rng(3).uniform(0, 2000, size=J).astype(np.float32)
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_release(r)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_release(r)
    res = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16)
    best = min(singles, key=lambda x: x["key"])
    assert res["key"] == best["key"] and res["makespan"] == best["makespan"]
    assert np.array_equal(res["opt"], best["opt"]) and np.array_equal(res["prio"], best["prio"])
    me.close()
