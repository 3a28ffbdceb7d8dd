"""GPU: the maximum-tardiness objective (SB_FLAG_MAX_TARDINESS, solve(objective="max_stretch")) — bit-exact scores
and arg-min keys on every kernel path against the fp32 oracle (oracle/ref_max_tardiness.py), weighted and unweighted,
with and without release dates; eval_full / decode starts, the makespan identity, the ABI refusals, incremental rounds
and the search population, the seeds of the C driver against lpt_seeds, solve() and solve_table() against the
exhaustive optimum, the 256-task warm starts, orchestrate() and two devices."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_max_tardiness as MT, ref_release as RR
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1


def _setup(engine, tab, opt, prio, seed, released, weighted, nodes=1):
    """fp32 due dates around the first candidate's makespan (some negative, some past every completion), weights
    when `weighted` and release dates when `released`; returns (objective, w, d, r)."""
    J = tab.shape[0]
    span = float(RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float64,
                               nodes=nodes)[0])
    rng = np.random.default_rng(seed)
    d = (rng.uniform(-0.2, 1.3, size=J) * span).astype(np.float32)
    r = (rng.uniform(-0.1, 0.6, size=J) * span).astype(np.float32) if released else None
    w = rng.choice([0.25, 0.5, 1.0, 1.5, 3.0, 8.0, 0.1], size=J).astype(np.float32) if weighted else None
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    return ("weighted_max_tardiness" if weighted else "max_tardiness"), w, d, r


def _ref(tab, opt, prio, d, r, w, ints, nodes=1, want_plan=False):
    return MT.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), d, r, ints, np.float32, nodes=nodes,
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
    obj, w, d, r = _setup(engine, tab, opt, prio, J, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, ints)
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
    obj, w, d, r = _setup(engine, tab, opt, prio, 5, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, ints)
    _check_runs(engine, opt, prio, ref, [({}, 9), ({"_reorder": False}, 4), ({"_force_generic": True}, 0)], obj,
                integer_starts=ints)
    J, S, B = 256, 8, 3000
    T, valid = R.synth_table(J, S, 8, seed=9)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=10)
    obj, w, d, r = _setup(engine, tab, opt, prio, 9, released, weighted)
    ref = _ref(tab, opt, prio, d, r, w, ints)
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
        obj, w, d, r = _setup(engine, tab, opt, prio, J, released, weighted)
        ref = _ref(tab, opt, prio, d, r, w, ints)
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
    obj, w, d, r = _setup(engine, tab, opt, prio, J + nodes, released, nodes % 2 == 1, nodes)
    ref, rstart, rmask = _ref(tab, opt, prio, d, r, w, ints, nodes, want_plan=True)
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


def test_full_table_makespan_identity_and_the_tardiness_sign(engine):
    """d = 0 with unit weights scores exactly the makespan on every path and in sb_eval_full.  On integer data a
    candidate's maximum tardiness is +0 exactly when its total tardiness is +0; due dates equal to candidate 0's
    completions score it +0.  eval_full on the full table matches the oracle."""
    J, B = 60, 4000
    T, valid = R.synth_table(J, 3, 8, seed=2)
    T = np.ceil(T)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=3)
    for ints in (True, False):
        engine.set_due(np.zeros(J, np.float32))
        mk = _eval(engine, opt, prio, "makespan", integer_starts=ints)[0]
        for kw in ({}, {"_no_stream": True}, {"_force_generic": True}, {"_plain_addr": True}):
            got = _eval(engine, opt, prio, "max_tardiness", integer_starts=ints, **kw)[0]
            assert got.tobytes() == mk.tobytes(), (ints, kw)
        tot, _, _ = engine.eval_full(opt, prio, integer_starts=ints, objective="max_tardiness")
        assert tot.cpu().numpy().tobytes() == mk.tobytes()
    _, start, _ = RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float32,
                                want_plan=True)
    o0 = opt[0].cpu().numpy()
    d = (start[0] + tab[np.arange(J), o0 >> 3, o0 & 7]).astype(np.float32)       # candidate 0 on time, to the second
    engine.set_due(d)
    score = _eval(engine, opt, prio, "max_tardiness")[0]
    tard = _eval(engine, opt, prio, "tardiness")[0]
    assert ((tard == 0) == (score == 0)).all()
    assert score[0] == 0 and tard[0] == 0 and (tard > 0).any()
    assert score.tobytes() == _ref(tab, opt, prio, d, None, None, True).tobytes()
    tot, _, _ = engine.eval_full(opt, prio, objective="max_tardiness")
    assert tot.cpu().numpy().tobytes() == score.tobytes()


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_absent_cells_score_inf(engine, ints, released):
    """A candidate that gives a job an option it does not have (here 3 GPUs, absent from gcount) is infeasible: every
    path scores it +inf, as under every other objective and as the oracle says, and the arg-min key is a feasible
    candidate's.  The same on two nodes, in sb_eval_full, and for a candidate injected into the search population."""
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
        obj, w, d, r = _setup(engine, tab, opt2, prio, J, released, True, nodes)
        ref = _ref(tab, opt2, prio, d, r, w, ints, nodes)
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
    # the search population: an injected infeasible candidate holds +inf
    b = int(np.nonzero(bad)[0][0])
    engine.search_init(1024, seed=2, reduced=True, integer_starts=ints, objective=obj)
    engine.search_inject(o[b], prio[b].cpu().numpy(), copies=4, first=8)
    _o, _p, score, _layout = engine.debug_search_population(8, 4)
    assert np.isinf(score).all()


def test_refusals(engine):
    """The flag without both tardiness flags, or with the late count or the maximum lateness (SB_ERR_ARG), without
    due dates or weights (SB_ERR_STATE), and with the alternate shape (SB_ERR_UNSUPPORTED)."""
    from saturn_b200 import _lib
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    MX, SUM, DUE, W = _lib.FLAG_MAX_TARDINESS, _lib.FLAG_SUM_COMPLETION, _lib.FLAG_DUE, _lib.FLAG_WEIGHTED

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)
    assert raw(MX | SUM | DUE) == -3                                                 # no due dates
    p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | MX | SUM | DUE, t_start=0.01, t_end=1e-4,
                          total_rounds=4)
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
    engine.set_due(np.arange(J, dtype=np.float32))
    assert raw(MX | SUM | DUE) == 0
    assert raw(MX | SUM | DUE | W) == -3                                             # no weights
    engine.set_weights(np.ones(J, np.float32))
    assert raw(MX | SUM | DUE | W) == 0
    for bad in (MX, MX | SUM, MX | DUE, MX | SUM | W, MX | _lib.FLAG_MAX_LATENESS,
                MX | SUM | DUE | _lib.FLAG_MAX_LATENESS, MX | SUM | DUE | _lib.FLAG_LATE_COUNT,
                MX | SUM | DUE | W | _lib.FLAG_LATE_COUNT):
        assert raw(bad) == -1, bad
    p.flags = _lib.FLAG_REDUCED | MX | SUM
    assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -1
    assert raw(MX | SUM | DUE | _lib.FLAG_ALT_WARPSCAN) == -4
    engine.set_table(T)                                                              # clears the due dates
    assert raw(MX | SUM | DUE) == -3


def _population_case(J, released, weighted):
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    rng = np.random.default_rng(J)
    d = (rng.uniform(-0.2, 1.2, size=J) * horizon).astype(np.float32)
    r = (rng.uniform(0.0, 0.6, size=J) * horizon).astype(np.float32) if released else None
    w = rng.choice([0.5, 1.0, 2.0, 3.0], size=J).astype(np.float32) if weighted else None
    return T, tmin, d, r, w


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
    T, tmin, d, r, w = _population_case(J, released, weighted)
    obj = "weighted_max_tardiness" if weighted else "max_tardiness"
    engine.set_table(T)
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4, objective=obj, t_start=0.05, t_end=0.01)
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, **kw)
    assert b.makespan == a.makespan and np.array_equal(b.opt, a.opt) and np.array_equal(b.prio, a.prio)
    for res in (a, b):
        assert sorted(res.prio.tolist()) == list(range(J))
        assert float(MT.evaluate(tmin, res.opt[None], res.prio[None], d, r, weights=w)[0]) == res.makespan
    chains = 2048

    def check_population(what):
        opt, prio, score, layout = engine.debug_search_population()
        ref = MT.evaluate(tmin, opt, prio, d, r, weights=w)
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
    obj = "weighted_max_tardiness" if weighted else "max_tardiness"
    engine.set_due(d)
    engine.set_release(r)
    engine.set_weights(w)
    chains = 4096
    engine.search_init(chains, seed=1, reduced=True, integer_starts=ints, objective=obj)
    engine.search_seed_lpt()
    tmin, _args = engine.reduced_table()
    seeds = lpt_seeds(tmin, nodes=nodes, objective=obj, weights=w, due=d, release=r, integer_starts=ints)
    base = lpt_seeds(tmin, nodes=nodes, objective=obj.replace("max_tardiness", "tardiness"), weights=w, due=d,
                     release=r, integer_starts=ints)
    per = chains // 8
    for i, ((col, order), (bcol, border)) in enumerate(zip(seeds, base)):
        assert np.array_equal(col, bcol) and np.array_equal(order, border)
        opt, prio, _score, _layout = engine.debug_search_population(i * per, per)
        assert (opt == col[None, :]).all() and (prio == order.astype(prio.dtype)[None, :]).all(), i


def _cases():
    with open(os.path.join(HERE, "golden", "max_tardiness_cases.json")) as f:
        return [rec for rec in json.load(f)["cases"] if rec["stretch"]]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, _ = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    return [p[0] for p in plan], [p[0] + p[2] for p in plan]        # start and completion time per task


def _device_form(tasks, release):
    """The fp32 table, weights, due dates and release dates solve(objective="max_stretch") hands the device."""
    from saturn_b200 import solver as S
    from saturn_b200.engine import release_f32
    T, usable, _ = S.build_table(tasks)
    Tdev = T.copy()
    for j in range(len(tasks)):
        if usable[j].any():
            Tdev[j, 0, ~usable[j]] = np.inf
    r32 = release_f32(release, len(tasks)) if release is not None else None
    _pstar, w32, d32 = S._stretch_form(Tdev, r32)
    return Tdev, w32, d32, r32


def test_solve_reaches_the_exhaustive_optimum():
    """Every stretch fixture instance (with and without release dates): solve(objective="max_stretch") returns a
    feasible plan whose fp32 device score is the fp32 exhaustive optimum of the same table, weights and due dates;
    last_stats' float64 max stretch is the plan's and agrees with the fixture's optimum; solve_table on the same table
    returns the same plan."""
    from saturn_b200 import solver as S
    cases = _cases()
    assert len(cases) >= 8
    for i, rec in enumerate(cases):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        r = rec["release"]
        out = S.solve(tasks, None, chains=4096, rounds=60, seed=i, objective="max_stretch", release=r)
        start, comp = _plan(tasks, out)
        Tdev, w32, d32, r32 = _device_form(tasks, r)
        _tab, optmap = R.table_from_tuples(tuples)
        best32 = MT.brute_force(Tdev, [[7 & o for o in ops] for ops in optmap], d32, r32, True, np.float32,
                                weights=w32)[0]
        st = S.last_stats
        assert st["device_makespan"] == best32, rec["name"]
        pstar = [min(rt for _g, rt in tup) for tup in tuples]
        rr = r if r is not None else [0.0] * len(tasks)
        stretch = [(c - max(x, 0.0)) / p for c, x, p in zip(comp, rr, pstar)]
        assert st["max_stretch"] == pytest.approx(max(stretch), rel=1e-12)
        assert st["mean_stretch"] == pytest.approx(sum(stretch) / len(stretch), rel=1e-12)
        assert st["max_stretch"] == pytest.approx(rec["bruteforce_f64"]["score"], rel=1e-5), rec["name"]
        assert out[5] == pytest.approx(max(comp), rel=1e-12)
        from saturn_b200 import solve_table, strategies_from_table
        T = np.full((len(tasks), 1, 8), np.inf, np.float32)
        for j, tup in enumerate(tuples):
            for g, rt in tup:
                T[j, 0, int(g) - 1] = rt
        tb = solve_table(T, np.isfinite(T), chains=4096, rounds=60, seed=i, objective="max_stretch", release=r)
        view = [DuckTask("t%d" % j, s) for j, s in enumerate(strategies_from_table(T, np.isfinite(T)))]
        sv = S.solve(view, None, chains=4096, rounds=60, seed=i, objective="max_stretch", release=r)
        assert all(tb[k] == sv[k] for k in range(5)) and tb[5] == pytest.approx(sv[5], rel=1e-12), rec["name"]


def _tasks256():
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J = 256
    T, valid = synth_table(J, 4, 8, seed=3)
    strategies = strategies_from_table(T, valid)
    return [DuckTask("t%d" % j, strategies[j]) for j in range(J)]


def test_256_task_warm_starts_never_get_worse():
    """The 256-task set with the seeded release dates of scripts/bench_objective.py: max_stretch solves warm-started
    with the completion plan and with the makespan plan each return a plan whose fp32 oracle score is at most the
    warm-start plan's, since the search starts from that candidate and keeps its best."""
    from saturn_b200 import solver as S
    tasks = _tasks256()
    J = len(tasks)
    release = [float(x) for x in np.random.default_rng(5).integers(0, 100000, size=J)]
    Tdev, w32, d32, r32 = _device_form(tasks, release)
    tab = Tdev[:, 0, :][:, None, :]

    def injected(plan):  # the candidate a warm start plants, scored by the oracle's schedule
        opt, prio = S.candidate_from_arrays(tasks, plan, 1)
        return float(MT.evaluate(tab, opt[None, :], prio[None, :].astype(np.uint8), d32, r32, True, np.float32,
                                 weights=w32)[0])

    def emitted(plan):  # the plan's own starts, folded by the oracle
        opt, prio = S.candidate_from_arrays(tasks, plan, 1)
        start, _comp = _plan(tasks, plan)
        return float(MT.fold(tab, opt[None, :], prio[None, :], np.array([start], np.float32), d32, np.float32,
                             weights=w32)[0])
    kw = dict(rounds=200, seed=1, release=release)
    for base in ("completion", "makespan"):
        warm = S.solve(tasks, None, objective=base, **kw)
        out = S.solve(tasks, warm, objective="max_stretch", **kw)
        got, before = emitted(out), injected(warm)
        print(base, "warm start", before, "-> max stretch plan", got, "max stretch", S.last_stats["max_stretch"])
        assert got == S.last_stats["device_makespan"]
        assert got <= before, (base, got, before)


def test_orchestrate_runs_max_stretch_in_simulated_time():
    """orchestrate() with a release mapping keyed by Task under objective="max_stretch" runs every task to
    completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    release = {t: float(700 * i) for i, t in enumerate(tasks)}
    recs = orchestrate(tasks, interval=1000, solver_kwargs={"chains": 4096, "rounds": 25, "objective": "max_stretch",
                                                             "release": release}, max_intervals=50)
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
    chains, rounds = 4096, 32
    singles = []
    for dev in range(2):
        e = Engine(dev, stream=torch.cuda.current_stream(torch.device("cuda", dev)))
        e.set_table(T)
        e.set_due(d)
        e.set_weights(w)
        singles.append(e.search_run(chains, rounds, seed=5, chain_base=dev * chains, reduced=True, sync_every=16,
                                    objective="weighted_max_tardiness"))
        e.close()
    me = MultiEngine([0, 1])
    me.set_table(T)
    me.set_due(d)
    me.set_weights(w)
    res = me.search_run(chains, rounds, seed=5, reduced=True, sync_every=16, objective="weighted_max_tardiness")
    best = min(singles, key=lambda x: x["key"])
    assert res["key"] == best["key"] and res["makespan"] == best["makespan"]
    me.close()
