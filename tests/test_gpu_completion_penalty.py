"""GPU: the completion-penalty objective (SB_FLAG_COMPLETION_PENALTY, solve(objective="completion_penalty")) and
solve_front — bit-exact scores and arg-min keys on every kernel path against the fp32 oracle
(oracle/ref_completion_penalty.py), weighted and unweighted, with and without release dates; eval_full / decode starts,
p = 0 against the weighted-completion kernels, absent cells, the ABI refusals, incremental rounds and the search
population, the seeds of the C driver against lpt_seeds, solve() with p = 0 against objective="completion", solve()
and solve_table() against the exhaustive optimum, warm starts, orchestrate(), two devices, and solve_front against the
exhaustive front and on the 256-task set."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_completion_penalty as CP, ref_eval as R, ref_release as RR
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1


def _setup(engine, tab, opt, prio, seed, released, weighted, nodes=1):
    """fp32 due dates around the first candidate's makespan (some negative, some past every completion), penalties
    (a quarter of them 0), weights when `weighted` and release dates when `released`; returns (objective, w, d, r, p)."""
    J = tab.shape[0]
    span = float(RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float64,
                               nodes=nodes)[0])
    rng = np.random.default_rng(seed)
    d = (rng.uniform(-0.2, 1.3, size=J) * span).astype(np.float32)
    r = (rng.uniform(-0.1, 0.6, size=J) * span).astype(np.float32) if released else None
    w = rng.choice([0.25, 0.5, 1.0, 1.5, 3.0, 8.0, 0.1], size=J).astype(np.float32) if weighted else None
    p = (rng.uniform(0, 0.5, size=J) * span).astype(np.float32)
    p[rng.random(J) < 0.25] = 0.0
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    engine.set_penalty(p)
    return ("weighted_completion_penalty" if weighted else "completion_penalty"), w, d, r, p


def _ref(tab, opt, prio, d, r, w, p, ints, nodes=1, want_plan=False):
    return CP.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), d, p, r, ints, np.float32, nodes=nodes,
                       want_plan=want_plan, weights=w)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=11, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _check_runs(engine, opt, prio, ref, runs, objective, infeasible=False, **common):
    """Every run: the score equals the oracle bit for bit on the path asked for, with the arg-min key (`infeasible`:
    some candidates score +inf)."""
    assert ((ref < np.inf).all() or infeasible) and (ref > 0).all() and len(np.unique(ref)) > 1
    for kw, path in runs:
        got, key, p = _eval(engine, opt, prio, objective, **common, **kw)
        assert path is None or p == path, (kw, p)
        assert got.tobytes() == ref.tobytes(), kw
        assert key == _key_of(ref, 11), kw


@pytest.mark.parametrize("J,S,B", [(100, 4, 3001), (256, 8, 4000), (300, 2, 1500), (17, 2, 77)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_tile_and_generic_paths(engine, J, S, B, ints, released, weighted):
    """Paths 3 (both address forms), 2, 1 and 0, u8 and u16 priorities, and sb_eval_host."""
    T, valid = R.synth_table(J, S, 8, seed=J + S)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=J)
    obj, w, d, r, p = _setup(engine, tab, opt, prio, J, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, p, ints)
    runs = [({}, 3), ({"_plain_addr": True}, 3), ({"_no_stream": True}, 2), ({"_force_generic": True}, 0)]
    _check_runs(engine, opt, prio, ref, runs, obj, integer_starts=ints)
    if (J * (1 if J <= 256 else 2)) % 16:
        got, key, p = _eval(engine, opt.contiguous(), prio.contiguous(), obj, integer_starts=ints)
        assert p == 1 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, objective=obj)
    assert np.array_equal(host.numpy(), ref)


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_large_tables(engine, ints, released, weighted):
    """J = 1024 with the full 8-strategy table: paths 9, 4 and 0 on job-indexed rows; J = 256: the position-major
    kernel with its table in shared memory (5), split over a CTA pair (7) and in global memory (8); S > 8: the route
    that table size selects."""
    J, S, B = 1024, 8, 1500
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    obj, w, d, r, p = _setup(engine, tab, opt, prio, 5, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, p, ints)
    _check_runs(engine, opt, prio, ref, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)], obj,
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    obj, w, d, r, p = _setup(engine, tab, opt, prio, 9, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, p, ints)
    obp = opt_by_position(opt, prio)
    _check_runs(engine, obp, prio, ref, [({}, 5), ({"_table_home": 2}, 7), ({"_table_home": 1}, 8)], obj,
                integer_starts=ints, by_position=True)
    got, key, p = _eval(engine, opt, prio, obj, integer_starts=ints, _reorder=True)
    assert p == 9 and np.array_equal(got, ref) and key == _key_of(ref, 11)
    for J, S in ((224, 32), (64, 17), (40, 9)):
        T, valid = R.synth_table(J, S, 8, seed=J + S)
        engine.set_table(T)
        tab = R.canon_table(T, range(1, 9))
        opt, prio = random_candidates(engine, 700, valid, seed=J)
        obj, w, d, r, p = _setup(engine, tab, opt, prio, J, released, weighted)
        ref = _ref(tab, opt, prio, d, r, w, p, ints)
        _check_runs(engine, opt, prio, ref, [({}, None), ({"_force_generic": True}, 0)], obj, integer_starts=ints)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 3000), (100, 3, 1001), (300, 4, 700), (40, 1, 500)])
@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_multi_node_eval_full_and_decode(engine, J, nodes, B, ints, released):
    """1..4 nodes on the reduced table: every path equals the oracle; sb_eval_full and sb_decode give the oracle's
    scores, starts and slot masks (weighted on odd node counts)."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    obj, w, d, r, p = _setup(engine, tab, opt, prio, J + nodes, released, nodes % 2 == 1, nodes)
    ref, rstart, rmask = _ref(tab, opt, prio, d, r, w, p, ints, nodes, want_plan=True)
    _check_runs(engine, opt, prio, ref, [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)],
                obj, integer_starts=ints, reduced=True)
    tot, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True, objective=obj)
    assert tot.cpu().numpy().tobytes() == ref.tobytes()
    assert np.array_equal(start.cpu().numpy(), rstart)
    assert np.array_equal(mask.cpu().numpy().astype(np.uint32), rmask)
    b = B // 3
    dec = engine.decode(opt[b].cpu().numpy(), prio[b].cpu().numpy(), integer_starts=ints, reduced=True, objective=obj)
    assert dec["makespan"] == float(ref[b])
    assert np.array_equal(dec["start"], rstart[b]) and np.array_equal(dec["slotmask"], rmask[b] & 0xffff)


def test_zero_penalties_are_the_weighted_completion_kernels(engine):
    """With p = 0 (and p = -0.0, stored as +0) every path scores exactly what the completion kernels score, weighted
    and unweighted, integer and real starts, with release dates, and sb_eval_full too; due dates past every completion
    give the completion score whatever the penalties, and a penalty is paid exactly where a job is late."""
    J, B = 60, 4000
    T, valid = R.synth_table(J, 3, 8, seed=2)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=3)
    _obj, w, d, r, _p = _setup(engine, tab, opt, prio, 4, True, True)
    runs = ({}, {"_no_stream": True}, {"_force_generic": True}, {"_plain_addr": True}, {"_reorder": True})
    for zero in (np.zeros(J, np.float32), np.full(J, -0.0, np.float32)):
        engine.set_penalty(zero)
        for ints in (True, False):
            for cp, wc in (("completion_penalty", "completion"), ("weighted_completion_penalty",
                                                                  "weighted_completion")):
                want = _eval(engine, opt, prio, wc, integer_starts=ints)[0]
                for kw in runs:
                    got = _eval(engine, opt, prio, cp, integer_starts=ints, **kw)[0]
                    assert got.tobytes() == want.tobytes(), (cp, ints, kw)
                tot, _, _ = engine.eval_full(opt, prio, integer_starts=ints, objective=cp)
                assert tot.cpu().numpy().tobytes() == want.tobytes()
    engine.set_penalty(np.full(J, 1.0e6, np.float32))
    comp = _eval(engine, opt, prio, "completion")[0]
    tard = _eval(engine, opt, prio, "tardiness")[0]
    pen = _eval(engine, opt, prio, "completion_penalty")[0]
    assert ((pen > comp) == (tard > 0)).all() and (tard > 0).any()
    engine.set_due(np.full(J, 2.0 ** 23, np.float32))
    assert _eval(engine, opt, prio, "completion_penalty")[0].tobytes() == comp.tobytes()


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_absent_cells_score_inf(engine, ints, released):
    """A candidate that gives a job an option it does not have (here 3 GPUs, absent from gcount) is infeasible: every
    path scores it +inf, as the oracle says, and the arg-min key is a feasible candidate's.  The same on two nodes, in
    sb_eval_full, and for a candidate injected into the search population."""
    from saturn_b200.engine import padded_rows
    gcount = [8, 1, 4, 2]
    for J, nodes in ((100, 1), (64, 2)):
        rng = np.random.default_rng(J)
        T = rng.uniform(10, 500, size=(J, 4 if nodes == 1 else 1, 4)).astype(np.float32)
        engine.set_table(T, gcount, nodes=nodes)
        tab = R.canon_table(T, gcount)
        valid = np.ones(T.shape, dtype=bool)
        B = 2000
        opt, prio = random_candidates(engine, B, valid, seed=J, nodes=nodes)
        bad = rng.random(B) < 0.3
        bad[0] = False                                                            # _setup scales by candidate 0
        o = opt.cpu().numpy()
        o[bad, 7] = (o[bad, 7] & 0xF8) | 2                                        # 3 GPUs: no such column
        opt2 = padded_rows(B, J, torch.uint8, engine.device)
        opt2.copy_(torch.from_numpy(o))
        if nodes > 1:
            tab = R.reduce_table(tab)[0][:, None, :]
        obj, w, d, r, p = _setup(engine, tab, opt2, prio, J, released, True, nodes)
        ref = _ref(tab, opt2, prio, d, r, w, p, ints, nodes)
        assert np.array_equal(np.isinf(ref), bad) and np.isfinite(ref[~bad]).all()
        red = {"reduced": True} if nodes > 1 else {}
        runs = [({}, None), ({"_no_stream": True}, None), ({"_force_generic": True}, 0)]
        if nodes == 1:
            runs += [({"_plain_addr": True}, 3), ({"_reorder": True}, 9)]
        _check_runs(engine, opt2, prio, ref, runs, obj, infeasible=True, integer_starts=ints, **red)
        if nodes == 1:
            _check_runs(engine, opt_by_position(opt2, prio), prio, ref, [({}, 5), ({"_table_home": 1}, 8)], obj,
                        infeasible=True, integer_starts=ints, by_position=True)
        tot, _, _ = engine.eval_full(opt2, prio, integer_starts=ints, objective=obj, **red)
        assert tot.cpu().numpy().tobytes() == ref.tobytes()
    b = int(np.nonzero(bad)[0][0])
    engine.search_init(1024, seed=2, reduced=True, integer_starts=ints, objective=obj)
    engine.search_inject(o[b], prio[b].cpu().numpy(), copies=4, first=8)
    _o, _p, score, _layout = engine.debug_search_population(8, 4)
    assert np.isinf(score).all()


def test_refusals(engine):
    """The flag without both tardiness flags, or with the late penalty, the late count, the maximum tardiness, the
    squares or the maximum lateness (SB_ERR_ARG); without due dates, weights or penalties (SB_ERR_STATE, due dates
    first, then weights, then penalties, then release dates); with the alternate shape (SB_ERR_UNSUPPORTED).  With
    release dates set the flag runs like every form."""
    from saturn_b200 import _lib
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    CPF, SUM, DUE, W = _lib.FLAG_COMPLETION_PENALTY, _lib.FLAG_SUM_COMPLETION, _lib.FLAG_DUE, _lib.FLAG_WEIGHTED
    REL = _lib.FLAG_RELEASE

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)
    try:
        assert raw(CPF | SUM | DUE) == -3                                             # no due dates
        p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | CPF | SUM | DUE, t_start=0.01,
                              t_end=1e-4, total_rounds=4)
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
        engine.set_due(np.arange(J, dtype=np.float32))
        assert raw(CPF | SUM | DUE | REL) == -3                                       # no penalties
        assert "SB_FLAG_COMPLETION_PENALTY" in engine._lib.sb_last_error().decode()
        engine.set_penalty(np.ones(J, np.float32))
        assert raw(CPF | SUM | DUE) == 0
        assert raw(CPF | SUM | DUE | REL) == -3                                       # no release dates
        engine.set_release(np.arange(J, dtype=np.float32))
        assert raw(CPF | SUM | DUE | REL) == 0
        assert raw(CPF | SUM | DUE | W) == -3                                         # no weights
        engine.set_weights(np.ones(J, np.float32))
        assert raw(CPF | SUM | DUE | W) == 0
        for bad in (CPF, CPF | SUM, CPF | DUE, CPF | SUM | W, CPF | _lib.FLAG_MAX_LATENESS,
                    CPF | SUM | DUE | _lib.FLAG_LATE_PENALTY, CPF | SUM | DUE | W | _lib.FLAG_LATE_PENALTY,
                    CPF | SUM | DUE | _lib.FLAG_MAX_LATENESS, CPF | SUM | DUE | _lib.FLAG_LATE_COUNT,
                    CPF | SUM | DUE | _lib.FLAG_MAX_TARDINESS, CPF | SUM | DUE | _lib.FLAG_SQUARED,
                    CPF | SUM | DUE | W | _lib.FLAG_SQUARED):
            assert raw(bad) == -1, bad
        p.flags = _lib.FLAG_REDUCED | CPF | SUM
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -1
        assert raw(CPF | SUM | DUE | _lib.FLAG_ALT_WARPSCAN) == -4
        engine.set_table(T)                                                          # clears the penalties
        engine.set_due(np.arange(J, dtype=np.float32))
        assert raw(CPF | SUM | DUE) == -3 and raw(SUM | DUE) == 0
    finally:
        engine.set_table(T)


def _population_case(J, released, weighted):
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    rng = np.random.default_rng(J)
    d = (rng.uniform(-0.2, 1.2, size=J) * horizon).astype(np.float32)
    r = (rng.uniform(0.0, 0.6, size=J) * horizon).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32) if weighted else None
    p = (rng.uniform(0.0, 0.5, size=J) * horizon).astype(np.float32)
    p[rng.random(J) < 0.25] = 0.0
    return T, tmin, d, r, w, p


@pytest.mark.parametrize("J", [40, 256, 300, 1024])
@pytest.mark.parametrize("released", [False, True])
def test_incremental_rounds_and_population(engine, J, released):
    """The verify hook recomputes every incremental score from position 0: no mismatch.  After init, seeding, and
    rounds of 1, 3, 16 and 17, in the layout the library picks for J (fused tile or position-major) and in unfused
    propose / evaluate / accept rounds, every chain's stored score is the oracle's score of its rows, and the search's
    result re-scores to the reported value (weighted at J = 256 and 1024)."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    weighted = J in (256, 1024)
    T, tmin, d, r, w, p = _population_case(J, released, weighted)
    obj = "weighted_completion_penalty" if weighted else "completion_penalty"
    engine.set_table(T)
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    engine.set_penalty(p)
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective=obj, t_start=0.05, t_end=0.01)
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    assert a.stop_reason != 3 and b.stop_reason != 3                   # no stop at zero: the score never reaches it
    for res in (a, b):
        assert sorted(res.prio.tolist()) == list(range(J))
        assert float(CP.evaluate(tmin, res.opt[None], res.prio[None], d, p, r, weights=w)[0]) == res.makespan
    chains = 2048

    def check_population(what):
        opt, prio, score, layout = engine.debug_search_population()
        ref = CP.evaluate(tmin, opt, prio, d, p, r, weights=w)
        assert score.tobytes() == ref.tobytes(), what
        return layout
    layouts = set()
    for no_fused in (False, True):  # the library's layout for J, then propose / evaluate / accept rounds
        engine.search_init(chains, seed=3, reduced=True, t_start=0.01, t_end=1e-4, total_rounds=40, objective=obj,
                           _no_fused=no_fused)
        check_population("init")
        engine.search_seed_lpt()
        check_population("seeds")
        for n in (1, 3, 16, 17):
            engine.search_round(n)
            layouts.add(check_population("rounds %d, no_fused %s" % (n, no_fused)))
    assert 0 in layouts and len(layouts) == 2


@pytest.mark.parametrize("nodes", [1, 2, 3])
@pytest.mark.parametrize("released", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("ints", [True, False])
def test_c_seeds_equal_lpt_seeds(engine, nodes, released, weighted, ints):
    """sb_search_seed_lpt plants exactly the seeds of lpt_seeds, which are the completion seeds (SPT / WSPT), not
    the EDD seeds of the tardiness."""
    from saturn_b200.search import lpt_seeds
    J = 120
    T, valid = R.synth_table(J, 1, 8, seed=7 + nodes, masked=False)
    engine.set_table(T, nodes=nodes)
    tmin_c = R.reduce_table(R.canon_table(T, range(1, 9)))[0]
    horizon = float(tmin_c.min(axis=1).sum()) / 8 / nodes
    rng = np.random.default_rng(nodes + 10 * released)
    d = (np.round(rng.uniform(0.0, 4.0, size=J)) * horizon / 4).astype(np.float32)
    r = (rng.uniform(0.0, 0.3, size=J) * horizon).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32) if weighted else None
    obj = "weighted_completion_penalty" if weighted else "completion_penalty"
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    engine.set_penalty(rng.uniform(0, 100, size=J).astype(np.float32))
    chains = 4096
    engine.search_init(chains, seed=1, reduced=True, integer_starts=ints, objective=obj)
    engine.search_seed_lpt()
    tmin, _args = engine.reduced_table()
    seeds = lpt_seeds(tmin, nodes=nodes, objective=obj, weights=w, due=d, release=r, integer_starts=ints)
    base = lpt_seeds(tmin, nodes=nodes, objective=obj.replace("_penalty", ""), weights=w, release=r,
                     integer_starts=ints)
    if not released:  # release dates re-sort every order by release date first: then they can all coincide
        edd = lpt_seeds(tmin, nodes=nodes, objective="tardiness", due=d, integer_starts=ints)
        assert any(not np.array_equal(o, e) for (_c, o), (_ce, e) in zip(seeds, edd))
    per = chains // 8
    for i, ((col, order), (bcol, border)) in enumerate(zip(seeds, base)):
        assert np.array_equal(col, bcol) and np.array_equal(order, border)
        opt, prio, _score, _layout = engine.debug_search_population(i * per, per)
        assert (opt == col[None, :]).all() and (prio == order.astype(prio.dtype)[None, :]).all(), i


def _cases():
    with open(os.path.join(HERE, "golden", "completion_penalty_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, _ = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    return [p[0] for p in plan], [p[0] + p[2] for p in plan]        # start and completion time per task


def _device_table(tasks):
    """The fp32 table solve() hands the device."""
    from saturn_b200 import solver as S
    T, usable, _ = S.build_table(tasks)
    Tdev = T.copy()
    for j in range(len(tasks)):
        if usable[j].any():
            Tdev[j, 0, ~usable[j]] = np.inf
    return Tdev


def test_zero_penalties_solve_as_the_completion():
    """With p = 0 the search is the completion search, plan for plan: solve(objective="completion_penalty") returns
    the same plan, score and candidate count as objective="completion" for the same seed, weighted and unweighted,
    with release dates."""
    from saturn_b200 import solver as S
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 96
    T, valid = synth_table(J, 4, 8, seed=8)
    st = strategies_from_table(T, valid)
    tasks = [DuckTask("t%d" % j, st[j]) for j in range(J)]
    rng = np.random.default_rng(9)
    due = [float(x) for x in rng.integers(0, 40000, size=J)]
    release = [float(x) for x in rng.integers(0, 5000, size=J)]
    for weights in (None, [float(x) for x in rng.choice([1.0, 2.0, 3.0], size=J)]):
        kw = dict(chains=8192, rounds=80, seed=3, weights=weights, release=release)
        a = S.solve(tasks, None, objective="completion", **kw)
        sa = dict(S.last_stats)
        b = S.solve(tasks, None, objective="completion_penalty", due=due, penalty=[0.0] * J, **kw)
        sb = dict(S.last_stats)
        assert tuple(a) == tuple(b)
        assert sa["device_makespan"] == sb["device_makespan"] and sa["candidates"] == sb["candidates"]
        assert sb["penalty_paid"] == 0.0 and sb["completion_penalty"] == sb["weighted_completion"]
        want = sa["weighted_completion"] if weights is not None else sa["total_completion"]
        assert sb["weighted_completion"] == pytest.approx(want, rel=1e-12)


def test_solve_reaches_the_exhaustive_optimum():
    """Every fixture instance and its cap variant (with and without weights and release dates): solve() returns a
    feasible plan whose fp32 device score is the fp32 exhaustive optimum of the same table, weights, due dates and
    penalties; last_stats' float64 sums are the plan's and agree with the fixture's optimum; solve_table on the same
    table returns the same plan."""
    from saturn_b200 import solve_table, strategies_from_table
    from saturn_b200 import solver as S
    from saturn_b200.engine import due_f32, penalty_f32, release_f32, weights_f32
    cases = _cases()
    assert len(cases) == 24
    for i, rec in enumerate(cases):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        J = len(tasks)
        cap = rec["cap"]
        for due, pen, best64 in ((rec["due"], rec["penalty"], rec["bruteforce_f64"]["score"]),
                                 ([cap["cap"]] * J, [cap["P"]] * J, cap["bruteforce_f64"]["score"])):
            kw = {"objective": "completion_penalty", "due": due, "penalty": pen, "release": rec["release"],
                  "weights": rec["weights"]}
            out = S.solve(tasks, None, chains=4096, rounds=60, seed=i, **kw)
            _start, comp = _plan(tasks, out)
            Tdev = _device_table(tasks)
            w32 = weights_f32(rec["weights"], J) if rec["weights"] is not None else None
            r32 = release_f32(rec["release"], J) if rec["release"] is not None else None
            _tab, optmap = R.table_from_tuples(tuples)
            best32 = CP.brute_force(Tdev, [[7 & o for o in ops] for ops in optmap], due_f32(due, J),
                                    penalty_f32(pen, J), r32, True, np.float32, weights=w32)[0]
            st = S.last_stats
            assert st["device_makespan"] == best32, rec["name"]
            w = rec["weights"] if rec["weights"] is not None else [1.0] * J
            late = [c > d for c, d in zip(comp, due)]
            assert st["weighted_completion"] == pytest.approx(sum(wi * c for wi, c in zip(w, comp)), rel=1e-12)
            assert st["penalty_paid"] == sum(p for p, x in zip(pen, late) if x)
            assert st["late_tasks"] == sum(late)
            assert st["completion_penalty"] == pytest.approx(best64, rel=1e-9), rec["name"]
            T = np.full((J, 1, 8), np.inf, np.float32)
            for j, tup in enumerate(tuples):
                for g, rt in tup:
                    T[j, 0, int(g) - 1] = rt
            tb = solve_table(T, np.isfinite(T), chains=4096, rounds=60, seed=i, **kw)
            view = [DuckTask("t%d" % j, s) for j, s in enumerate(strategies_from_table(T, np.isfinite(T)))]
            sv = S.solve(view, None, chains=4096, rounds=60, seed=i, **kw)
            assert all(tb[k] == sv[k] for k in range(5)) and tb[5] == pytest.approx(sv[5], rel=1e-12), rec["name"]


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_256_task_warm_starts_never_get_worse():
    """The 256-task set with seeded due dates and penalties: completion_penalty solves warm-started with the
    completion plan and with the makespan plan each return a plan whose fp32 device score is at most the oracle's
    score of the candidate the warm start plants, since the search starts from that candidate and keeps its best."""
    from saturn_b200 import solver as S
    from saturn_b200.engine import due_f32, penalty_f32
    tasks = _tasks256()
    J = len(tasks)
    rng = np.random.default_rng(4)
    due = [float(x) for x in rng.integers(0, 200000, size=J)]
    pen = [float(x) for x in rng.integers(0, 20000, size=J)]
    d32, p32 = due_f32(due, J), penalty_f32(pen, J)
    tab = _device_table(tasks)[:, 0, :][:, None, :]

    def injected(plan):  # the candidate a warm start plants, scored by the oracle's schedule
        opt, prio = S.candidate_from_arrays(tasks, plan, 1)
        return float(CP.evaluate(tab, opt[None, :], prio[None, :].astype(np.uint8), d32, p32, None, True,
                                 np.float32)[0])
    kw = dict(rounds=200, seed=1)
    for base in ("completion", "makespan"):
        warm = S.solve(tasks, None, objective=base, **kw)
        S.solve(tasks, warm, objective="completion_penalty", due=due, penalty=pen, **kw)
        got, before = S.last_stats["device_makespan"], injected(warm)
        print(base, "warm start", before, "-> completion penalty plan", got)
        assert S.last_stats["completion_penalty"] == pytest.approx(got, rel=1e-4)
        assert got <= before, (base, got, before)


def test_orchestrate_runs_in_simulated_time():
    """orchestrate() with due, penalty and release mappings keyed by Task runs every task to completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    kw = {"chains": 4096, "rounds": 25, "objective": "completion_penalty",
          "release": {t: float(700 * i) for i, t in enumerate(tasks)},
          "due": {t: float(2500 * i + 3000) for i, t in enumerate(tasks)},
          "penalty": {t: float(500 * (i % 3)) for i, t in enumerate(tasks)}}
    recs = orchestrate(tasks, interval=1000, solver_kwargs=kw, max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)
    assert sum(len(rec["launched"]) for rec in recs) >= 8


def test_multiple_devices_equal_single_device_runs():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200.engine import Engine, MultiEngine
    J, S = 96, 4
    T, valid = R.synth_table(J, S, 8, seed=2)
    d = np.random.default_rng(3).uniform(0, 2000, size=J).astype(np.float32)
    w = np.random.default_rng(4).choice([1.0, 2.0, 3.0], size=J).astype(np.float32)
    p = np.random.default_rng(5).uniform(0, 3000, size=J).astype(np.float32)
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_due(d)
        e.set_weights(w)
        e.set_penalty(p)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16,
                                    objective="weighted_completion_penalty"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_due(d)
    me.set_weights(w)
    me.set_penalty(p)
    res = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="weighted_completion_penalty")
    best = min(singles, key=lambda x: x["key"])
    assert res["key"] == best["key"] and res["makespan"] == best["makespan"]
    me.close()


def _front_ok(front):
    """Makespan strictly ascending, completion strictly descending, every cap met in fp32."""
    assert front and all(a.makespan < b.makespan and a.completion > b.completion for a, b in zip(front, front[1:]))


def test_solve_front_against_the_exhaustive_front():
    """On every fixture instance (weights and release dates as recorded): every point but the makespan plan has the
    exhaustive minimum of sum w C under its cap, the makespan plan has the exhaustive minimum makespan, every point
    lies on or above the exhaustive front, and the returned set is non-dominated."""
    from saturn_b200 import solver as S
    for i, rec in enumerate(_cases()):
        tasks = tasks_from_tuples(rec["gpu_time_tuples"])
        front = S.solve_front(tasks, points=5, weights=rec["weights"], release=rec["release"], seed=i, chains=4096,
                              rounds=60)
        _front_ok(front)
        ex = rec["front"]
        for pt in front:
            _plan(tasks, pt.plan)
            best = min(c for m, c in ex if m <= pt.cap)
            assert pt.completion >= best - 1e-9 * best, rec["name"]
            if pt.stats["objective"] == "makespan":
                assert pt.makespan == ex[0][0] and pt.cap == ex[0][0], rec["name"]
            else:
                assert pt.completion == pytest.approx(best, rel=1e-12), (rec["name"], pt.cap)
            assert pt.makespan <= pt.cap
        assert front[-1].completion == pytest.approx(ex[-1][1], rel=1e-12), rec["name"]


def test_solve_front_on_the_256_task_set():
    """The 256-task set with the seeded release dates of the release measurement: the first point is
    solve(objective="makespan") with the same seed, every point's fp32 makespan is within its cap and its float64
    makespan within half an fp32 ulp of it, the completion falls strictly from point to point, the interior points
    ran the completion-penalty form without paying a penalty, and convert_into_comprehensible takes every plan."""
    from saturn_b200 import convert_into_comprehensible, solve_front
    from saturn_b200 import solver as S
    tasks = _tasks256()
    J = len(tasks)
    kw = dict(seed=1, rounds=200)
    mk = S.solve(tasks, None, **kw)[5]
    release = [float(x) for x in np.random.default_rng(6).integers(0, int(0.5 * mk), size=J)]
    first = S.solve(tasks, None, objective="makespan", release=release, **kw)
    front = solve_front(tasks, points=8, release=release, **kw)
    print([(p.cap, p.makespan, p.completion / J) for p in front])
    _front_ok(front)
    assert len(front) >= 3
    assert tuple(front[0].plan) == tuple(first)
    T, _u, _o = S.build_table(tasks)
    for p in front:
        assert S._device_makespan(tasks, p.plan, T) <= p.cap
        assert p.makespan <= p.cap + 0.5 * float(np.spacing(np.float32(p.cap)))
        if p.stats["objective"] == "completion_penalty":
            assert p.stats["penalty_paid"] == 0.0 and p.stats["late_tasks"] == 0
        convert_into_comprehensible(tasks, p.plan[2], p.plan[4], p.plan[1], p.plan[3], p.plan[0])
