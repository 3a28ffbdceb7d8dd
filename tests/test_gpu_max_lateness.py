"""GPU: the maximum-lateness objective (SB_FLAG_MAX_LATENESS, solve(objective="max_lateness")) — bit-exact tail
makespans and arg-min keys on every kernel path against the fp32 oracle (oracle/ref_max_lateness.py), d = c giving
the makespan, the tardiness sign test, eval_full / decode starts, the ABI refusals, incremental rounds and the
search population, solve() against the exhaustive optimum and the EDD seeds, shifted due dates, orchestrate() and
two devices."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_max_lateness as ML, ref_release as RR
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1
OBJ = "max_lateness"


def _setup(engine, tab, opt, prio, seed, released, nodes=1):
    """fp32 due dates around the first candidate's makespan (some negative, some past every completion) and, when
    `released`, release dates; returns (d, r)."""
    J = tab.shape[0]
    span = float(RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float64,
                               nodes=nodes)[0])
    rng = np.random.default_rng(seed)
    d = (rng.uniform(-0.2, 1.3, size=J) * span).astype(np.float32)
    r = (rng.uniform(-0.1, 0.6, size=J) * span).astype(np.float32) if released else None
    engine.set_due(d)
    engine.set_release(r)
    return d, r


def _ref(tab, opt, prio, d, r, ints, nodes=1, want_plan=False):
    return ML.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), d, r, ints, np.float32, nodes=nodes,
                       want_plan=want_plan)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective=OBJ, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _check_runs(engine, opt, prio, ref, runs, **common):
    """Every run: the tail makespan equals the oracle bit for bit on the path asked for, with the arg-min key.  Then
    d = c for every job gives exactly the makespan run's scores and keys on the same path.  Restores the due dates."""
    d = engine.due.copy()
    assert (ref < np.inf).all() and (ref >= 0).all()
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, **common, **kw)
        assert path is None or p == path, (kw, p)
        assert got.tobytes() == ref.tobytes(), kw
        assert key == _key_of(ref, 11), kw
    engine.set_due(np.full(engine.J, 321.0, np.float32))
    for kw, _path in runs:
        got = _eval(engine, opt, prio, **common, **kw)
        mk = _eval(engine, opt, prio, "makespan", **common, **kw)
        assert got[0].tobytes() == mk[0].tobytes() and got[1:] == mk[1:], kw
    engine.set_due(d)


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_tile_and_generic_paths(engine, J, S, B, ints, released):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities, and sb_eval_host."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    d, r = _setup(engine, tab, opt, prio, J, released)
    ref = _ref(tab, opt, prio, d, r, ints)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, runs, integer_starts=ints)
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective=OBJ)
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_large_tables(engine, ints, released):
    """J = 1024 with the full 8-strategy table: paths 9, 4 and 0 on job-indexed rows; J = 256: the position-major
    kernel with its table in shared memory (5), split over a CTA pair (7) and in global memory (8); S = 32: the
    route that table size selects."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    d, r = _setup(engine, tab, opt, prio, 5, released)
    ref = _ref(tab, opt, prio, d, r, ints)
    _check_runs(engine, opt, prio, ref, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)],
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    d, r = _setup(engine, tab, opt, prio, 9, released)
    ref = _ref(tab, opt, prio, d, r, ints)
    obp = opt_by_position(opt, prio)
    _check_runs(engine, obp, prio, ref, [({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)],
                integer_starts=ints, by_position=True)
    got, key, p = _eval(engine, opt, prio, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    for J, S in ((224, 32), (64, 17), (40, 9)):
        T, valid = R.synth_table(J, S, 8, seed=J + S)
        engine.set_table(T)
        tab = R.canon_table(T, range(1, 9))
        opt, prio = random_candidates(engine, 700, valid, seed=J)
        d, r = _setup(engine, tab, opt, prio, J, released)
        ref = _ref(tab, opt, prio, d, r, ints)
        _check_runs(engine, opt, prio, ref, [({}, None), ({"_force_generic": True}, 0)], integer_starts=ints)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_multi_node_eval_full_and_decode(engine, J, nodes, B, ints, released):
    """1..4 nodes on the reduced table: every path equals the oracle; sb_eval_full and sb_decode give the oracle's
    scores, starts and slot masks."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    d, r = _setup(engine, tab, opt, prio, J + nodes, released, nodes)
    ref, rstart, rmask = _ref(tab, opt, prio, d, r, ints, nodes, want_plan=True)
    _check_runs(engine, opt, prio, ref, [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)],
                integer_starts=ints, reduced=True)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=OBJ)
    assert tot.cpu().numpy().tobytes() == ref.tobytes()
    assert np.array_equal(start.cpu().numpy(), rstart)
    assert np.array_equal(mask.cpu().numpy().astype(np.uint32), rmask)
    b = B // 3
    dec = engine.decode(opt[b].cpu().numpy(), prio[b].cpu().numpy(), integer_starts=ints, reduced=True, objective=OBJ)
    assert dec["makespan"] == float(ref[b])
    assert np.array_equal(dec["start"], rstart[b]) and np.array_equal(dec["slotmask"], rmask[b] & 0xffff)


def test_full_table_decode_and_tardiness_sign(engine):
    """On integer data (integer runtimes and due dates) a candidate's total tardiness is +0 exactly when its tail
    makespan is <= D = max d; eval_full on the full table matches the oracle."""
    J, B = 60, 4000
    rng = np.random.default_rng(2)
    T, valid = R.synth_table(J, 3, 8, seed=2)
    T = np.ceil(T)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=3)
    span = float(RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float64)[0])
    d = np.round(rng.uniform(0.6, 2.5, size=J) * span).astype(np.float32)
    engine.set_due(d)
    score = _eval(engine, opt, prio)[0]
    tard = _eval(engine, opt, prio, "tardiness")[0]
    D = float(d.max())
    assert ((tard == 0) == (score <= D)).all()
    assert (tard == 0).any() and (tard > 0).any()
    tot, _, _ = engine.eval_full(opt, prio, objective=OBJ)
    assert tot.cpu().numpy().tobytes() == _ref(tab, opt, prio, d, None, True).tobytes()


def test_refusals(engine):
    """The flag without due dates (SB_ERR_STATE), with another objective flag or a due-date spread >= 2^24
    (SB_ERR_ARG), the alternate shape (SB_ERR_UNSUPPORTED), and sb_set_due still accepting that spread."""
    from saturn_b200 import _lib
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    ML_ = _lib.FLAG_MAX_LATENESS

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)
    assert raw(ML_) == -3                                                            # no due dates
    p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | ML_, t_start=0.01, t_end=1e-4, total_rounds=4)
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
    engine.set_due(np.arange(J, dtype=np.float32))
    assert raw(ML_) == 0 and raw(ML_ | _lib.FLAG_INTEGER_STARTS) == 0
    engine.set_weights(np.ones(J, np.float32))
    for other in (_lib.FLAG_SUM_COMPLETION, _lib.FLAG_SUM_COMPLETION | _lib.FLAG_WEIGHTED,
                  _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE):
        assert raw(ML_ | other) == -1
    assert raw(ML_ | _lib.FLAG_ALT_WARPSCAN) == -4
    wide = np.zeros(J, np.float32)
    wide[0], wide[1] = -9.0e6, 9.0e6                                                 # spread 1.8e7 >= 2^24
    assert engine._lib.sb_set_due(engine._h, C.c_void_p(wide.ctypes.data), J) == 0
    assert raw(ML_) == -1
    assert raw(_lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE) == 0                        # tardiness still takes it
    engine.set_table(T)                                                              # clears the due dates
    assert raw(ML_) == -3


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
@pytest.mark.parametrize("released", [False, True])
def test_incremental_rounds_and_population(engine, J, released):
    """The verify hook recomputes every incremental score from position 0: no mismatch.  After seeding, rounds and
    a resample, every chain's stored score is the oracle's tail makespan of its rows, and the search's result
    re-scores to the reported value."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    rng = np.random.default_rng(J)
    d = (rng.uniform(-0.2, 1.2, size=J) * horizon).astype(np.float32)
    r = (rng.uniform(0.0, 0.6, size=J) * horizon).astype(np.float32) if released else None
    engine.set_due(d)
    engine.set_release(r)
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective=OBJ)
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    for res in (a, b):
        assert sorted(res.prio.tolist()) == list(range(J))
        assert float(ML.evaluate(tmin, res.opt[None], res.prio[None], d, r)[0]) == res.makespan
    chains = 2048
    engine.search_init(chains, seed=3, reduced=True, t_start=0.01, t_end=1e-4, total_rounds=40, objective=OBJ)

    def check_population(what):
        opt, prio, score, _layout = engine.debug_search_population()
        ref = ML.evaluate(tmin, opt, prio, d, r)
        assert score.tobytes() == ref.tobytes(), what
    check_population("init")
    engine.search_seed_lpt()
    check_population("seeds")
    for n in (1, 3, 16, 17):
        engine.search_round(n)
        check_population("rounds %d" % n)


def _completion_cases():
    with open(os.path.join(HERE, "golden", "completion_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, _ = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    return [p[0] for p in plan], [p[0] + p[2] for p in plan]        # start and completion time per task


def test_solve_reaches_the_exhaustive_optimum():
    """The 20 completion fixtures with seeded integer due dates (some all met: L_max < 0), with and without release
    dates: solve() returns a feasible plan whose L_max, recomputed in float64, is the exhaustive optimum's, and
    last_stats reports it, the late tasks and the device score minus max d."""
    from saturn_b200 import solver as S
    negative = 0
    for i, rec in enumerate(_completion_cases()):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        J = len(tasks)
        rng = np.random.default_rng(1000 + i)
        scale = sum(min(rt for _, rt in t) for t in tuples)
        d = np.round(rng.uniform(0.2, 1.6, size=J) * scale).astype(float)
        for r in (None, np.round(rng.uniform(0, 0.4, size=J) * scale)):
            out = S.solve(tasks, None, chains=4096, rounds=60, seed=i, objective=OBJ, due=list(d),
                          release=None if r is None else list(r))
            start, comp = _plan(tasks, out)
            lmax = max(c - x for c, x in zip(comp, d))
            tab, om = R.table_from_tuples(tuples)
            best = ML.brute_force(tab, om, d, r, True, dtype=np.float64)[0]
            assert lmax == pytest.approx(best, rel=1e-6, abs=1e-6), (rec["name"], r is None)
            assert S.last_stats["max_lateness"] == pytest.approx(lmax, abs=1e-9)
            assert S.last_stats["late_tasks"] == sum(1 for c, x in zip(comp, d) if c - x > 0)
            assert S.last_stats["device_makespan"] == pytest.approx(lmax, rel=1e-5, abs=1e-3)
            assert out[5] == pytest.approx(max(comp), rel=1e-12)
            if r is not None:
                assert "total_flow_time" in S.last_stats
            negative += best < 0
    assert negative >= 3


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_solve_256_tasks_beats_the_edd_seeds_and_shifts_with_the_due_dates():
    """J = 256 with seeded integer due dates: the plan passes check_plan, its L_max is no worse than the best EDD seed's
    (the search starts from them), and due dates shifted by an integer give the same plan with L_max shifted by it."""
    from saturn_b200 import solver as S
    from saturn_b200.search import lpt_seeds
    tasks = _tasks256()
    J = len(tasks)
    kw = dict(chains=16384, rounds=120, seed=1)
    plain = S.solve(tasks, None, **kw)
    d = np.round(np.random.default_rng(7).uniform(0.1, 1.1, size=J) * plain[5])
    a = S.solve(tasks, None, objective=OBJ, due=list(d), **kw)
    _plan(tasks, a)
    la = S.last_stats["max_lateness"]
    eng = S._engine()
    tmin, _args = eng.reduced_table()
    seeds = lpt_seeds(tmin, objective=OBJ, due=eng.due)
    seed_scores = [ML.evaluate(tmin[:, None, :], col[None], order.astype(np.uint8)[None], eng.due)[0] for col, order
                   in seeds]
    assert la <= float(min(seed_scores)) - eng.due_shift + 1e-5 * abs(eng.due_shift) + 1e-3
    b = S.solve(tasks, None, objective=OBJ, due=list(d + 5000.0), **kw)
    assert all(x == y for x, y in zip(a[:5], b[:5])) and a[5] == b[5]
    assert S.last_stats["max_lateness"] == pytest.approx(la - 5000.0, abs=1e-9)


def test_orchestrate_runs_max_lateness_in_simulated_time():
    """orchestrate() with a due mapping keyed by Task under objective="max_lateness" runs every task to completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    due = {t: float(1500 * i) for i, t in enumerate(tasks)}
    recs = orchestrate(tasks, interval=1000, solver_kwargs={"chains": 4096, "rounds": 25, "objective": OBJ,
                                                             "due": due}, max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)
    assert sum(len(rec["launched"]) for rec in recs) >= 8


def test_multiple_devices_equal_single_device_runs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200.engine import Engine, MultiEngine
    J, S = 96, 4
    T, valid = R.synth_table(J, S, 8, seed=2)
    d = np.random.default_rng(3).uniform(0, 2000, size=J).astype(np.float32)
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_due(d)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16,
                                    objective=OBJ))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_due(d)
    res = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective=OBJ)
    best = min(singles, key=lambda x: x["key"])
    assert res["key"] == best["key"] and res["makespan"] == best["makespan"]
    me.close()
