"""GPU: the late-penalty objective (SB_FLAG_LATE_PENALTY, solve(objective="late_penalty")) — bit-exact scores and
arg-min keys on every kernel path against the fp32 oracle (oracle/ref_late_penalty.py), weighted and unweighted, with
and without release dates; eval_full / decode starts, p = 0 against the tardiness kernels, absent cells, the ABI
refusals and every combination of the objective flags against the four per-job arrays, incremental rounds and the
search population, the seeds of the C driver against lpt_seeds, solve() with p = 0 against objective="tardiness",
solve() and solve_table() against the exhaustive optimum, the 256-task warm starts, orchestrate() and two devices."""
import ctypes as C
import itertools
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_late_penalty as LP, ref_release as RR
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
    p = (rng.uniform(0, 0.05, size=J) * span).astype(np.float32)
    p[rng.random(J) < 0.25] = 0.0
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    engine.set_penalty(p)
    return ("weighted_late_penalty" if weighted else "late_penalty"), w, d, r, p


def _ref(tab, opt, prio, d, r, w, p, ints, nodes=1, want_plan=False):
    return LP.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), d, p, r, ints, np.float32, nodes=nodes,
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
    assert ((ref < np.inf).all() or infeasible) and (ref >= 0).all() and len(np.unique(ref)) > 1
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



def test_zero_penalties_are_the_tardiness_kernels(engine):
    """With p = 0 (and p = -0.0, stored as +0) every path scores exactly what the tardiness kernels score, weighted
    and unweighted, integer and real starts, with release dates, and sb_eval_full too; due dates past every completion
    score every candidate +0 whatever the penalties, and a penalty is paid exactly where the tardiness is > 0."""
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
            for lp, td in (("late_penalty", "tardiness"), ("weighted_late_penalty", "weighted_tardiness")):
                want = _eval(engine, opt, prio, td, integer_starts=ints)[0]
                for kw in runs:
                    got = _eval(engine, opt, prio, lp, integer_starts=ints, **kw)[0]
                    assert got.tobytes() == want.tobytes(), (lp, ints, kw)
                tot, _, _ = engine.eval_full(opt, prio, integer_starts=ints, objective=lp)
                assert tot.cpu().numpy().tobytes() == want.tobytes()
    engine.set_penalty(np.full(J, 100.0, np.float32))
    tard = _eval(engine, opt, prio, "tardiness")[0]
    pen = _eval(engine, opt, prio, "late_penalty")[0]
    assert ((pen > tard) == (tard > 0)).all() and (tard > 0).any()
    engine.set_due(np.full(J, 2.0 ** 23, np.float32))
    assert not _eval(engine, opt, prio, "late_penalty")[0].any()


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
    """The flag without both tardiness flags, or with the late count, the maximum tardiness, the squares or the maximum
    lateness (SB_ERR_ARG); without due dates, weights or penalties (SB_ERR_STATE); and with the alternate shape
    (SB_ERR_UNSUPPORTED).  sb_set_penalty refuses negative, NaN and inf values, a wrong J and penalties whose sum could
    overflow (SB_ERR_ARG), and answers SB_ERR_STATE before sb_set_table."""
    from saturn_b200 import _lib
    from saturn_b200.engine import Engine
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    LPF, SUM, DUE, W = _lib.FLAG_LATE_PENALTY, _lib.FLAG_SUM_COMPLETION, _lib.FLAG_DUE, _lib.FLAG_WEIGHTED

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)

    def set_p(vals, n=J):
        a = np.ascontiguousarray(vals, dtype=np.float32)
        return engine._lib.sb_set_penalty(engine._h, C.c_void_p(a.ctypes.data), n)
    assert raw(LPF | SUM | DUE) == -3                                                 # no due dates
    p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | LPF | SUM | DUE, t_start=0.01, t_end=1e-4,
                          total_rounds=4)
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
    engine.set_due(np.arange(J, dtype=np.float32))
    assert raw(LPF | SUM | DUE) == -3                                                 # no penalties
    engine.set_penalty(np.ones(J, np.float32))
    assert raw(LPF | SUM | DUE) == 0
    assert raw(LPF | SUM | DUE | W) == -3                                             # no weights
    engine.set_weights(np.ones(J, np.float32))
    assert raw(LPF | SUM | DUE | W) == 0
    for bad in (LPF, LPF | SUM, LPF | DUE, LPF | SUM | W, LPF | _lib.FLAG_MAX_LATENESS,
                LPF | SUM | DUE | _lib.FLAG_MAX_LATENESS, LPF | SUM | DUE | _lib.FLAG_LATE_COUNT,
                LPF | SUM | DUE | W | _lib.FLAG_LATE_COUNT, LPF | SUM | DUE | _lib.FLAG_MAX_TARDINESS,
                LPF | SUM | DUE | W | _lib.FLAG_MAX_TARDINESS, LPF | SUM | DUE | _lib.FLAG_SQUARED,
                LPF | SUM | DUE | W | _lib.FLAG_SQUARED):
        assert raw(bad) == -1, bad
    p.flags = _lib.FLAG_REDUCED | LPF | SUM
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -1
    assert raw(LPF | SUM | DUE | _lib.FLAG_ALT_WARPSCAN) == -4
    for v in (-1.0, np.nan, np.inf):
        vals = np.ones(J, np.float32)
        vals[3] = v
        assert set_p(vals) == -1, v
    assert raw(LPF | SUM | DUE) == 0                                                  # a refused set keeps the old ones
    assert set_p(np.ones(J - 1, np.float32), J - 1) == -1
    big = np.zeros(J, np.float32)
    big[0] = np.float32(2.0 ** 126 / J)                                                # J * max p = 2^126
    assert set_p(big) == -1
    big[0] = np.nextafter(big[0], np.float32(0))
    assert set_p(big) == 0
    assert engine._lib.sb_set_penalty(engine._h, None, 0) == 0                         # clears them
    assert raw(LPF | SUM | DUE) == -3
    engine.set_penalty(np.ones(J, np.float32))
    engine.set_table(T)                                                              # clears the penalties
    engine.set_due(np.arange(J, dtype=np.float32))
    assert raw(LPF | SUM | DUE) == -3 and raw(SUM | DUE) == 0
    fresh = Engine(0)
    try:
        a = np.ones(J, np.float32)
        assert fresh._lib.sb_set_penalty(fresh._h, C.c_void_p(a.ctypes.data), J) == -3  # before sb_set_table
    finally:
        fresh.close()


OK, ERR_ARG, ERR_STATE = 0, -1, -3


def _refused(flags, lib):
    """The combinations of the eight objective flags the ABI refuses (SB_ERR_ARG) whatever the handle holds."""
    SUM, W, DUE = flags & lib.FLAG_SUM_COMPLETION, flags & lib.FLAG_WEIGHTED, flags & lib.FLAG_DUE
    ML, LC, MT = flags & lib.FLAG_MAX_LATENESS, flags & lib.FLAG_LATE_COUNT, flags & lib.FLAG_MAX_TARDINESS
    SQF, LPF = flags & lib.FLAG_SQUARED, flags & lib.FLAG_LATE_PENALTY
    if (LC or MT or SQF or LPF) and not (SUM and DUE):
        return True                            # the late count, the maximum, the squares and the penalty modify
    if MT and (LC or ML):                      # the tardiness
        return True
    if SQF and (LC or MT or ML):
        return True
    if LPF and (LC or MT or SQF or ML):
        return True
    if ML and (SUM or W or DUE):
        return True                            # the maximum lateness is an objective of its own
    return bool((W or DUE) and not SUM)        # weights and due dates score the sum form


def _expected(flags, lib, has_w, has_d, has_r, has_p, q_exact, sq_finite):
    """The ABI's rules (include/saturn_b200.h): every refusal of a flag combination (SB_ERR_ARG) comes first, then the
    arrays the flags read (SB_ERR_STATE) in the order weights-free due dates, weights, penalties, release dates, where
    the maximum lateness also needs a due-date spread below 2^24 and the weighted squares weights with
    J * max w * 2^50 < FLT_MAX (SB_ERR_ARG) once the handle holds those arrays."""
    W, DUE, SQF = flags & lib.FLAG_WEIGHTED, flags & lib.FLAG_DUE, flags & lib.FLAG_SQUARED
    ML, REL, LPF = flags & lib.FLAG_MAX_LATENESS, flags & lib.FLAG_RELEASE, flags & lib.FLAG_LATE_PENALTY
    if _refused(flags, lib):
        return ERR_ARG
    if (ML or DUE) and not has_d:
        return ERR_STATE
    if ML and not q_exact:
        return ERR_ARG
    if W and not has_w:
        return ERR_STATE
    if SQF and W and not sq_finite:
        return ERR_ARG
    if LPF and not has_p:
        return ERR_STATE
    if REL and not has_r:
        return ERR_STATE
    return OK


def test_flag_combinations_against_handle_states(engine):
    """Every combination of the eight objective flags and SB_FLAG_RELEASE against states of the four per-job arrays
    (weights, due dates, release dates, penalties), through sb_eval (B = 0: every check, no launch), sb_search_init and
    sb_search_wave, which refuses only the combinations that can never run."""
    from saturn_b200 import _lib
    J = 24
    T, valid = R.synth_table(J, 2, 8, seed=3)
    bits = (_lib.FLAG_SUM_COMPLETION, _lib.FLAG_WEIGHTED, _lib.FLAG_DUE, _lib.FLAG_MAX_LATENESS, _lib.FLAG_LATE_COUNT,
            _lib.FLAG_MAX_TARDINESS, _lib.FLAG_SQUARED, _lib.FLAG_LATE_PENALTY, _lib.FLAG_RELEASE)
    narrow = np.arange(J, dtype=np.float32) * 3.0 - 20.0
    wide = np.zeros(J, np.float32)
    wide[0], wide[1] = -9.0e6, 9.0e6                   # spread 1.8e7 >= 2^24: the tails would round
    weights = np.linspace(0.5, 4.0, J).astype(np.float32)
    heavy = weights.copy()
    heavy[5] = 1.0e24                                  # 24 * 1e24 * 2^50 >= FLT_MAX: the squares could overflow
    release = np.linspace(-1.0, 30.0, J).astype(np.float32)
    pen = np.linspace(0.0, 50.0, J).astype(np.float32)
    # state: (weights, due dates, release dates, penalties)
    states = {
        "nothing": (None, None, None, None),
        "penalty": (None, None, None, pen),
        "weights_penalty": (weights, None, None, pen),
        "due": (None, narrow, None, None),
        "due_penalty": (None, narrow, None, pen),
        "due_release": (None, narrow, release, None),
        "wide_due_penalty": (None, wide, None, pen),
        "all_but_penalty": (weights, narrow, release, None),
        "all_but_release": (weights, narrow, None, pen),
        "all_heavy": (heavy, narrow, release, pen),
        "all": (weights, narrow, release, pen),
    }
    seen = set()
    try:
        for name, (w, d, r, p) in states.items():
            engine.set_table(T)
            engine.set_weights(w)
            engine.set_due(d)
            engine.set_release(r)
            engine.set_penalty(p)
            q_exact = d is None or float(d.max()) - float(d.min()) < 2.0 ** 24
            sq_finite = w is None or J * float(w.max()) * 2.0 ** 50 < float(np.finfo(np.float32).max)
            for pick in itertools.product((0, 1), repeat=len(bits)):
                flags = sum(b for b, on in zip(bits, pick) if on)
                want = _expected(flags, _lib, w is not None, d is not None, r is not None, p is not None, q_exact,
                                 sq_finite)
                seen.add((want, bool(flags & _lib.FLAG_LATE_PENALTY)))
                got = engine._lib.sb_eval(engine._h, None, None, 0, J, flags, None, None, 0)
                assert got == want, (name, hex(flags), "sb_eval", got, want)
                p_ = _lib.SearchParams(seed=1, chains=64, flags=_lib.FLAG_REDUCED | flags, t_start=0.01, t_end=1e-4,
                                       total_rounds=2)
                got = engine._lib.sb_search_init(engine._h, C.byref(p_), None, None)
                assert got == want, (name, hex(flags), "sb_search_init", got, want)
                n = C.c_int64(0)
                got = engine._lib.sb_search_wave(engine._h, _lib.FLAG_REDUCED | flags, C.byref(n))
                assert got == (ERR_ARG if _refused(flags, _lib) else OK), (name, hex(flags), "sb_search_wave", got)
                assert (n.value > 0) == (got == OK)
    finally:
        engine.set_table(T)                            # clears every per-job array of the shared engine
    assert seen == {(c, s) for c in (OK, ERR_ARG, ERR_STATE) for s in (False, True)}


def _population_case(J, released, weighted):
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    rng = np.random.default_rng(J)
    d = (rng.uniform(-0.2, 1.2, size=J) * horizon).astype(np.float32)
    r = (rng.uniform(0.0, 0.6, size=J) * horizon).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32) if weighted else None
    p = (rng.uniform(0.0, 0.05, size=J) * horizon).astype(np.float32)
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
    obj = "weighted_late_penalty" if weighted else "late_penalty"
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
    for res in (a, b):
        assert sorted(res.prio.tolist()) == list(range(J))
        assert float(LP.evaluate(tmin, res.opt[None], res.prio[None], d, p, r, weights=w)[0]) == res.makespan
    chains = 2048

    def check_population(what):
        opt, prio, score, layout = engine.debug_search_population()
        ref = LP.evaluate(tmin, opt, prio, d, p, r, weights=w)
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
    """sb_search_seed_lpt plants exactly the seeds of lpt_seeds, which are the EDD seeds of the tardiness."""
    from saturn_b200.search import lpt_seeds
    J = 120
    T, valid = R.synth_table(J, 1, 8, seed=7 + nodes, masked=False)
    engine.set_table(T, nodes=nodes)
    tmin_c = R.reduce_table(R.canon_table(T, range(1, 9)))[0]
    horizon = float(tmin_c.min(axis=1).sum()) / 8 / nodes
    rng = np.random.default_rng(nodes + 10 * released)
    d = (np.round(rng.uniform(0.0, 4.0, size=J)) * horizon / 4).astype(np.float32)     # ties: the rt / w rule decides
    r = (rng.uniform(0.0, 0.3, size=J) * horizon).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32) if weighted else None
    obj = "weighted_late_penalty" if weighted else "late_penalty"
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    engine.set_penalty(rng.uniform(0, 100, size=J).astype(np.float32))
    chains = 4096
    engine.search_init(chains, seed=1, reduced=True, integer_starts=ints, objective=obj)
    engine.search_seed_lpt()
    tmin, _args = engine.reduced_table()
    seeds = lpt_seeds(tmin, nodes=nodes, objective=obj, weights=w, due=d, release=r, integer_starts=ints)
    base = lpt_seeds(tmin, nodes=nodes, objective=obj.replace("late_penalty", "tardiness"), weights=w, due=d,
                     release=r, integer_starts=ints)
    per = chains // 8
    for i, ((col, order), (bcol, border)) in enumerate(zip(seeds, base)):
        assert np.array_equal(col, bcol) and np.array_equal(order, border)
        opt, prio, _score, _layout = engine.debug_search_population(i * per, per)
        assert (opt == col[None, :]).all() and (prio == order.astype(prio.dtype)[None, :]).all(), i


def _cases():
    with open(os.path.join(HERE, "golden", "late_penalty_cases.json")) as f:
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


def test_zero_penalties_solve_as_the_tardiness():
    """With p = 0 the search is the tardiness search, plan for plan: solve(objective="late_penalty") returns the same
    plan, score and key as objective="tardiness" for the same seed, weighted and unweighted, with release dates."""
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
        kw = dict(chains=8192, rounds=80, seed=3, due=due, weights=weights, release=release)
        a = S.solve(tasks, None, objective="tardiness", **kw)
        sa = dict(S.last_stats)
        b = S.solve(tasks, None, objective="late_penalty", penalty=[0.0] * J, **kw)
        sb = dict(S.last_stats)
        assert tuple(a) == tuple(b)
        assert sa["device_makespan"] == sb["device_makespan"] and sa["candidates"] == sb["candidates"]
        assert sb["late_penalty"] == pytest.approx(sb["weighted_tardiness"], rel=1e-12)
        assert sa["weighted_tardiness"] == sb["weighted_tardiness"] and sa["late_tasks"] == sb["late_tasks"]


def test_solve_reaches_the_exhaustive_optimum():
    """Every fixture instance (with and without weights and release dates, zero and dominant penalties): solve()
    returns a feasible plan whose fp32 device score is the fp32 exhaustive optimum of the same table, rates, due dates
    and penalties; last_stats' float64 sums are the plan's and agree with the fixture's optimum; solve_table on the
    same table returns the same plan."""
    from saturn_b200 import solve_table, strategies_from_table
    from saturn_b200 import solver as S
    from saturn_b200.engine import due_f32, penalty_f32, release_f32, weights_f32
    cases = _cases()
    assert len(cases) == 24
    for i, rec in enumerate(cases):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        J = len(tasks)
        kw = {"objective": "late_penalty", "due": rec["due"], "penalty": rec["penalty"], "release": rec["release"],
              "weights": rec["weights"]}
        out = S.solve(tasks, None, chains=4096, rounds=60, seed=i, **kw)
        start, comp = _plan(tasks, out)
        Tdev = _device_table(tasks)
        w32 = weights_f32(rec["weights"], J) if rec["weights"] is not None else None
        r32 = release_f32(rec["release"], J) if rec["release"] is not None else None
        _tab, optmap = R.table_from_tuples(tuples)
        best32 = LP.brute_force(Tdev, [[7 & o for o in ops] for ops in optmap], due_f32(rec["due"], J),
                                penalty_f32(rec["penalty"], J), r32, True, np.float32, weights=w32)[0]
        st = S.last_stats
        assert st["device_makespan"] == best32, rec["name"]
        w = rec["weights"] if rec["weights"] is not None else [1.0] * J
        x = [c - d for c, d in zip(comp, rec["due"])]
        assert st["late_penalty"] == pytest.approx(sum(p + wi * v for v, p, wi in zip(x, rec["penalty"], w) if v > 0),
                                                   rel=1e-12)
        assert st["weighted_tardiness"] == pytest.approx(sum(wi * max(0.0, v) for wi, v in zip(w, x)), rel=1e-12)
        assert st["late_tasks"] == sum(1 for v in x if v > 0)
        assert st["late_penalty"] == pytest.approx(rec["bruteforce_f64"]["score"], rel=1e-6), rec["name"]
        assert out[5] == pytest.approx(max(comp), rel=1e-12)
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
    """The 256-task set with seeded due dates and penalties: late_penalty solves warm-started with the tardiness plan
    and with the late-tasks plan each return a plan whose fp32 device score is at most the oracle's score of the
    candidate the warm start plants, since the search starts from that candidate and keeps its best."""
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
        return float(LP.evaluate(tab, opt[None, :], prio[None, :].astype(np.uint8), d32, p32, None, True,
                                 np.float32)[0])
    kw = dict(rounds=200, seed=1)
    for base in ("tardiness", "late_tasks"):
        warm = S.solve(tasks, None, objective=base, due=due, **kw)
        S.solve(tasks, warm, objective="late_penalty", due=due, penalty=pen, **kw)
        got, before = S.last_stats["device_makespan"], injected(warm)
        print(base, "warm start", before, "-> late penalty plan", got)
        assert S.last_stats["late_penalty"] == pytest.approx(got, rel=1e-4)
        assert got <= before, (base, got, before)


def test_orchestrate_runs_in_simulated_time():
    """orchestrate() with due, penalty and release mappings keyed by Task runs every task to completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    kw = {"chains": 4096, "rounds": 25, "objective": "late_penalty",
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
    p = np.random.default_rng(5).uniform(0, 300, size=J).astype(np.float32)
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_due(d)
        e.set_weights(w)
        e.set_penalty(p)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16,
                                    objective="weighted_late_penalty"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_due(d)
    me.set_weights(w)
    me.set_penalty(p)
    res = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="weighted_late_penalty")
    best = min(singles, key=lambda x: x["key"])
    assert res["key"] == best["key"] and res["makespan"] == best["makespan"]
    me.close()
