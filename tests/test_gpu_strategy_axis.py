"""Tables of 9 to 32 strategies, checked against the oracle on every kernel route and search layout they select.

sb_set_table accepts S up to SB_MAX_STRATEGIES = 32 (five strategy bits: opt bytes up to 0xFF), and the search runs
on the full table unless asked for the reduced one.  The table's size, J * S * 32 bytes, decides the kernel shape:
the tile plan's warps per CTA, where the position-major kernel keeps the table, whether the search round is fused,
position-major or unfused.  With S <= 8 and J <= 256 the table is at most 64 KB, so those shapes never run there.

* `route_*` below restate the library's shape rules for an H100 (sharedMemPerBlockOptin = 232,448 bytes); a CPU
  test pins the shapes this file relies on to them, and every GPU run asserts the path or layout it actually took
  against them.
* CPU: the C ports of every fold equal the Python list schedule bit for bit at S in {9, 17, 32}; the first-minimum
  rule of canon_table / reduce_table at S = 32; table_from_trials, strategies_from_table and the solve_table
  refusals at 32 executors.
* GPU: the reduced table in bits; the headline tile kernel at 16, 15, 11, 4, 3 and 2 warps per CTA under every
  objective (release dates lower the warp count) with its debug options; path 4 by default, path 9, the generic
  kernel with the table in shared and in global memory, by-position paths 5 / 7 / 8, eval_host, eval_full, decode
  and validate, also under the objectives whose per-job arrays move a shape to another route; the population
  invariants of test_gpu_search_state on full-table searches of every layout, those objectives included; search_run
  against the Python driver; solve_table against solve() at 32 executors.
"""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import ref_completion as RC
from oracle import ref_eval as R
from oracle import ref_exact as X
from oracle import ref_release as RR
from oracle import ref_tardiness as RT
from oracle import ref_weighted as RW
from saturn_b200 import _lib
from saturn_b200.engine import OBJECTIVES, objective_flag
from test_exact_edges import c_ref, candidates, release_dates, rt_table
from test_exact_edges import per_job as exact_per_job
from test_gpu_search_state import case, make_table, proposable, run_script

FOLDS = OBJECTIVES
KEY_MAX = 2 ** 63 - 1
ID_BASE = 0x7ffff000          # keys of b >= 4096 carry into bit 31 of the id
PATHS_SEEN = {}               # path -> set of (J, S) that took it, at S > 8
NW_SEEN = set()               # warps per CTA of path-3 runs on u8 rows
LAYOUTS_SEEN = {}             # layout -> set of (J, S)


# --------------------------------------------------------------------------- the route rules, restated
OPTIN = 232448                # H100: cudaDeviceProp::sharedMemPerBlockOptin


def _r16(n):
    return (n + 15) & ~15


def _round_row(b):
    r = (b + 15) // 16
    return (r + (r % 2 == 0)) * 16


def job_arrays(objective, release):
    """job_arrays(flags) of sb_internal.h: the per-job fp32 arrays staged beside the table, from the objective's flag
    bits: weights and due dates with SB_FLAG_DUE (unit weights without SB_FLAG_WEIGHTED), weights alone with
    SB_FLAG_WEIGHTED, the delivery tails with SB_FLAG_MAX_LATENESS, release dates with SB_FLAG_RELEASE."""
    f = objective_flag(objective)
    return (2 if f & _lib.FLAG_DUE else 1 if f & _lib.FLAG_WEIGHTED else 0) + bool(f & _lib.FLAG_MAX_LATENESS) + bool(
        release)


def plan_tiles(J, SG, stream, arrays=0, tab_global=False, nodes=1):
    """Warps per CTA of the tile kernel (plan_tiles in sb_eval.cu)."""
    pb = 1 if J <= 256 else 2
    tab = 0 if tab_global else _r16(J * SG * 4) + arrays * _r16(J * 4)
    per_warp = 32 * (_round_row(J) + (0 if stream else _round_row(J * pb))) + (nodes * 1024 if nodes > 1 else 0)
    nw = 16 if stream else 12
    while nw > 0 and tab + 16 * ((nw + 2) // 2) + nw * per_warp > OPTIN:
        nw -= 1
    return nw


def pos_smem(J, SG, arrays=0, nodes=1):
    return _r16(J * SG * 4) + arrays * _r16(J * 4) + 16 + (16 * nodes * 1024 if nodes > 1 else 0)


def route_eval(J, S, arrays=0):
    """(path, warps) of sb_eval on job-indexed rows padded to 32 elements, one node, no hooks: 9 = re-ordered for
    the position-major kernel (its table fits nowhere in one CTA, or J >= 1024); 3 = streamed tile kernel, table in
    shared memory; 4 = the same with the table in global memory; 2 / 1 = rows staged; 0 = generic."""
    SG = S * 8
    home = 0 if pos_smem(J, SG, arrays) <= OPTIN else 1
    if J <= 6144 and (home != 0 or J >= 1024):
        return 9, 16
    nw = plan_tiles(J, SG, True, arrays)
    if nw >= 2:
        return 3, nw
    nw = plan_tiles(J, SG, True, tab_global=True)
    if nw >= 2:
        return 4, nw
    nw = plan_tiles(J, SG, False, arrays)
    return (2, nw) if nw >= 2 else (0, 4)


def route_search(J, S, arrays=0):
    """(layout, warps) of a full-table search: 1 = fused tile round (both rows of 8+ warps beside the table),
    2 = position-major (the table fits in one CTA), 0 = unfused propose / evaluate / accept rounds."""
    SG = S * 8
    nw = plan_tiles(J, SG, False, arrays)
    if nw >= 8:
        return 1, nw
    if pos_smem(J, SG, arrays) <= OPTIN:
        return 2, 16
    nw = plan_tiles(J, SG, True, arrays)
    return 0, (nw if nw >= 1 else 4)


def generic_table_in_smem(J, S):
    return J * S * 8 * 4 <= OPTIN // 2


# (J, S, arrays): (sb_eval path, warps), (search layout, warps)
ROUTE_MAP = {
    (256, 9, 0): ((3, 16), (1, 9)),
    (256, 9, 1): ((3, 16), (1, 9)),
    (256, 9, 2): ((3, 16), (1, 8)),
    (256, 10, 0): ((3, 16), (1, 8)),
    (256, 11, 0): ((3, 16), (1, 8)),
    (256, 11, 1): ((3, 16), (1, 8)),
    (256, 11, 2): ((3, 16), (1, 8)),
    (256, 11, 3): ((3, 15), (2, 16)),
    (256, 12, 0): ((3, 15), (2, 16)),
    (256, 16, 0): ((3, 11), (2, 16)),
    (256, 24, 0): ((3, 4), (2, 16)),
    (256, 24, 1): ((3, 3), (2, 16)),
    (256, 24, 2): ((3, 3), (2, 16)),
    (256, 25, 0): ((3, 3), (2, 16)),
    (256, 25, 1): ((3, 3), (2, 16)),
    (256, 25, 2): ((3, 2), (2, 16)),
    (208, 32, 0): ((3, 2), (2, 16)),
    (216, 31, 3): ((3, 2), (2, 16)),
    (200, 24, 0): ((3, 11), (2, 16)),
    (224, 32, 0): ((4, 16), (2, 16)),
    (256, 28, 0): ((4, 16), (2, 16)),
    (256, 28, 1): ((4, 16), (2, 16)),
    (256, 28, 2): ((4, 16), (2, 16)),
    (256, 28, 3): ((9, 16), (0, 4)),
    (256, 32, 0): ((9, 16), (0, 4)),
    (300, 16, 0): ((3, 8), (2, 16)),
    (1024, 8, 0): ((9, 16), (0, 4)),
}


# --------------------------------------------------------------------------- CPU
def test_route_rules_pin_the_shapes_this_file_uses():
    """A threshold change that moves one of these shapes to another route fails here first."""
    for (J, S, arrays), (ev, se) in ROUTE_MAP.items():
        assert route_eval(J, S, arrays) == ev, (J, S, arrays, route_eval(J, S, arrays))
        assert route_search(J, S, arrays) == se, (J, S, arrays, route_search(J, S, arrays))
    assert generic_table_in_smem(128, 28) and not generic_table_in_smem(128, 29)
    # one array per form of job_arrays(flags): the tails of max_lateness, weights and due dates of the late count and
    # the maximum tardiness, weighted or not
    assert [job_arrays(o, False) for o in OBJECTIVES] == [0, 0, 1, 2, 2, 1, 2, 2, 2, 2]
    assert job_arrays("late_tasks", True) == 3 and job_arrays("max_lateness", True) == 2
    # the tables of S <= 8 and J <= 256 never leave the headline shape: 16 warps, fused search
    for S in range(1, 9):
        assert route_eval(256, S) == (3, 16) and route_search(256, S)[0] == 1


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("S", [9, 17, 32])
def test_c_ports_equal_the_python_list_schedule(S):
    """Every C port of a ref_release fold equals its Python list schedule (fp32) bit for bit, scores, starts and masks,
    with opt bytes spanning 0x00..(S - 1) << 3 | 7 (0xFF at S = 32), both start modes, release dates off and on."""
    J, B = 24, 12
    rng = np.random.default_rng(S)
    tab = (rng.uniform(0.5, 40.0, (J, S, 8)) * rng.choice([1.0, 1.0, 3.0], (J, S, 8))).astype(np.float32)
    tab[rng.uniform(size=tab.shape) < 0.05] = np.float32(1e6)
    tab[rng.uniform(size=tab.shape) < 0.03] = np.inf
    opt = rng.integers(0, 8 * S, (B, J)).astype(np.uint8)
    opt[0, :8] = (S - 1) << 3 | np.arange(8)
    opt[1, :8] = np.arange(8)
    assert opt.max() == 8 * S - 1 and opt.min() == 0
    prio = np.argsort(rng.random((B, J)), axis=1).astype(np.uint8)
    w = rng.choice([0.5, 1.0, 2.0, 3.0], J).astype(np.float32)
    d = rng.uniform(-5, 150, J).astype(np.float32)
    for ints in (True, False):
        for rel in (False, True):
            r = rng.uniform(-10, 60, J).astype(np.float32) if rel else np.zeros(J, np.float32)
            for fold in RR.OBJECTIVES:
                wf = w if fold.startswith("weighted") else None
                df = d if fold.endswith("tardiness") else None
                got, gst, gm = RR.c_evaluate(tab, opt, prio, r, ints, np.float32, want_plan=True, objective=fold,
                                             weights=wf, due=df)
                ports = []
                if not rel:
                    if fold == "makespan":
                        ports.append(c_oracle.evaluate(tab, opt, prio, ints, np.float32))
                    elif fold == "completion":
                        ports.append(RC.c_evaluate(tab, opt, prio, ints, np.float32))
                    elif fold == "weighted_completion":
                        ports.append(RW.c_evaluate(tab, opt, prio, ints, np.float32, weights=wf))
                    else:
                        ports.append(RT.c_evaluate(tab, opt, prio, df, ints, np.float32, weights=wf))
                for b in range(B):
                    sc, st, m, _ = RR.list_schedule(tab, opt[b], prio[b], r, ints, np.float32, objective=fold,
                                                    weights=wf, due=df)
                    label = (S, ints, rel, fold, b)
                    assert _bits(sc)[()] == _bits(got[b])[()], label
                    assert np.array_equal(_bits(np.asarray(st, np.float32)), _bits(gst[b])), label
                    assert np.array_equal(np.asarray(m, np.uint32), gm[b]), label
                    for p in ports:
                        assert _bits(p[b])[()] == _bits(got[b])[()], label


def _first_min_tables(T, gcount):
    """canon / reduce by the stated rule, in plain loops: the first column (input order), then the first strategy,
    that no later one beats with a strict <, its bits kept."""
    J, S, G = T.shape
    tab = np.full((J, S, 8), np.inf, np.float32)
    for j in range(J):
        for s in range(S):
            for g in range(G):
                if T[j, s, g] < tab[j, s, gcount[g] - 1]:
                    tab[j, s, gcount[g] - 1] = T[j, s, g]
    tmin = np.full((J, 8), np.inf, np.float32)
    args = np.zeros((J, 8), np.uint8)
    for j in range(J):
        for c in range(8):
            for s in range(S):
                if tab[j, s, c] < tmin[j, c]:
                    tmin[j, c], args[j, c] = tab[j, s, c], s
    return tab, tmin, args


def ingest_table(S, G, seed):
    """T[J][S][G] with cross-strategy ties, 1e6 / 1e8 sentinel ties, +inf-only columns and +-0 in duplicate GPU-count
    columns and across strategies; gcount permuted with duplicates.  The last strategy is the unique minimum of
    job 0's first GPU count, so the args reach S - 1."""
    rng = np.random.default_rng(seed)
    J = 40
    gcount = np.array([3, 1, 8, 3, 5, 1, 7][:G], np.uint8)
    T = rng.choice(np.array([1.0, 2.0, 2.0, 3.0, 1e6, 1e8, np.inf, 0.0, -0.0], np.float32), (J, S, G))
    T[1] = np.inf                                   # +inf-only columns
    T[2] = rng.choice(np.array([1e6, 1e8], np.float32), (S, G))
    T[3, :, 0], T[3, :, 3] = -0.0, 0.0              # duplicate count 3: -0 first
    T[4, :, 0], T[4, :, 3] = 0.0, -0.0              # +0 first
    if G > 5:                                       # duplicate count 1
        T[5, :, 1], T[5, :, 5] = -0.0, 0.0
    T[6, ::2, 2], T[6, 1::2, 2] = 0.0, -0.0         # +-0 across strategies
    T[7, ::2, 2], T[7, 1::2, 2] = -0.0, 0.0
    T[0, :, 0], T[0, :, 3] = 5.0, 5.0
    T[0, S - 1, 0] = 4.0
    return T.astype(np.float32), gcount


@pytest.mark.parametrize("S,G", [(9, 5), (16, 7), (31, 4), (32, 6)])
def test_canon_and_reduce_follow_the_first_minimum_rule(S, G):
    T, gcount = ingest_table(S, G, S)
    tab, tmin, args = _first_min_tables(T, gcount)
    got = R.canon_table(T, gcount)
    assert np.array_equal(_bits(got), _bits(tab))
    gmin, gargs = R.reduce_table(got)
    assert np.array_equal(_bits(gmin), _bits(tmin)) and np.array_equal(gargs, args)
    assert args.max() == S - 1
    assert np.signbit(tmin[3, 2]) and not np.signbit(tmin[4, 2]) and (G <= 5 or np.signbit(tmin[5, 0]))
    assert tmin[6, 7] == 0 and not np.signbit(tmin[6, 7]) and np.signbit(tmin[7, 7])


def test_trials_and_strategies_at_32_executors():
    """table_from_trials places 32 executors' results (failures -> 1e8, outside the GPU range -> 1e6), and
    strategies_from_table keeps the first executor of a tie."""
    from saturn_b200.solver import FAILED, NOT_PROFILED, strategies_from_table, table_from_trials
    E, J = 32, 3
    ranges = [range(1, 9), range(2, 5), None]
    flat, want = [], np.full((J, E, 8), NOT_PROFILED, np.float32)
    rng = np.random.default_rng(1)
    for t in range(J):
        for g in (ranges[t] if ranges[t] is not None else range(1, 9)):
            for e in range(E):
                rt = float(rng.integers(5, 9))
                if (t + g + e) % 7 == 0:
                    flat.append((None, None))
                    want[t, e, g - 1] = FAILED
                else:
                    flat.append(({"e": e, "g": g}, rt))
                    want[t, e, g - 1] = rt
    T, mask, params = table_from_trials(J, E, ranges, flat)
    assert np.array_equal(T, want) and np.array_equal(mask, (want < NOT_PROFILED))
    assert params[0, 31, 0] == {"e": 31, "g": 1}
    ex = ["x%d" % e for e in range(E)]
    st = strategies_from_table(T, mask, executors=ex, params=params)
    for t in range(J):
        for g in range(1, 9):
            col = np.where(mask[t, :, g - 1], T[t, :, g - 1], np.inf)
            s = st[t][g]
            if mask[t, :, g - 1].any():
                e = int(np.nonzero(col == col.min())[0][0])
                assert s.executor == ex[e] and s.runtime == float(col.min())
            else:
                assert s.executor is None
    # a column of 32 equal runtimes: the first executor; the only minimum at executor 31: executor 31
    T2 = np.full((1, E, 8), 4.0, np.float32)
    T2[0, 31, 5] = 3.0
    st2 = strategies_from_table(T2, np.ones(T2.shape, bool), executors=ex)
    assert st2[0][1].executor == "x0" and st2[0][6].executor == "x31"


def test_solve_table_refusals_at_32_executors():
    """Before any device call (the engine here is a plain object): a bad gcount (duplicate, outside 1..8, wrong
    length) and negative or NaN cells, with and without a mask."""
    from saturn_b200 import solver as SV
    T = np.full((3, 32, 4), 5.0, np.float32)
    for gc in ([1, 2, 2, 4], [0, 1, 2, 3], [1, 2, 3, 9], [1, 2, 3]):
        with pytest.raises(SV.SolverError, match="gcount"):
            SV.solve_table(T, None, gcount=gc, engine=object())
    for bad in (-1.0, np.nan):
        Tb = T.copy()
        Tb[2, 31, 3] = bad
        for m in (None, np.ones(T.shape, bool)):
            with pytest.raises(SV.SolverError, match="negative or NaN"):
                SV.solve_table(Tb, m, gcount=[8, 1, 4, 2], engine=object())


# --------------------------------------------------------------------------- GPU helpers
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _note_path(path, J, S):
    if S > 8:
        PATHS_SEEN.setdefault(path, set()).add((J, S))


def _dev(engine, opt, prio):
    import torch
    from saturn_b200.engine import padded_rows
    B, J = opt.shape
    o = padded_rows(B, J, torch.uint8, engine.device)
    p = padded_rows(B, J, engine.prio_dtype, engine.device)
    o.copy_(torch.from_numpy(opt))
    p.copy_(torch.from_numpy(prio.astype(np.int32) if J > 256 else prio).to(engine.prio_dtype))
    return o, p


def _key(ref, id_base):
    i = int(np.argmin(ref))
    return (int(_bits(ref[i:i + 1])[0]) << 32) | ((id_base + i) & 0xffffffff)


def _eval(engine, o, p, ref, ints, fold, label, id_base=ID_BASE, **kw):
    """One sb_eval: scores equal `ref` bit for bit and best_key is the arg-min key with this id base.  Returns the
    path taken, or None when the library refuses the route at this shape (SB_ERR_UNSUPPORTED only)."""
    import torch
    from saturn_b200._lib import SaturnB200Error
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    try:
        got = engine.eval(o, p, integer_starts=ints, objective=fold, best_key=key, id_base=id_base, **kw)
        torch.cuda.synchronize()
    except SaturnB200Error as e:
        assert "error -4:" in str(e), (label, kw, str(e))
        return None
    path = engine.last_eval_path()
    g = got.cpu().numpy()
    assert g.tobytes() == ref.tobytes(), (label, kw, path, np.nonzero(_bits(g) != _bits(ref))[0][:5])
    assert int(key.item()) & 0xffffffffffffffff == _key(ref, id_base), (label, kw, path, hex(int(key.item())))
    return path


def _setup(engine, J, S, fam, fold, rel, B, ints, seed):
    T = rt_table(fam, J, S, seed)
    engine.set_table(T)
    opt, prio = candidates(J, B, S, seed + 1)
    r = release_dates("ready" if rel else None, T, opt, prio, ints, 1, seed + 2)
    w, d = exact_per_job(fold, T, opt, prio, ints, 1, r, seed + 3)
    if r is not None:
        engine.set_release(r)
    if w is not None:
        engine.set_weights(w)
    if d is not None:
        engine.set_due(d)
    return T, opt, prio, r, w, d


def _exact(T, opt, prio, r, ints, fold, w, d, ref, rows, label):
    xs = X.batch(T, opt, prio, r, ints, 1, fold, w, d, rows=rows)[0]
    assert np.array_equal(xs, ref[rows].astype(np.float64)), label


# --------------------------------------------------------------------------- GPU: table ingest
@pytest.mark.gpu
@pytest.mark.parametrize("S,G", [(9, 5), (16, 7), (31, 4), (32, 6)])
def test_reduced_table_equals_the_oracle_in_bits(engine, S, G):
    T, gcount = ingest_table(S, G, S)
    engine.set_table(T, gcount=gcount)
    tmin, args = engine.reduced_table()
    rmin, rargs = R.reduce_table(R.canon_table(T, gcount))
    assert np.array_equal(_bits(tmin), _bits(rmin)), np.argwhere(_bits(tmin) != _bits(rmin))[:5]
    assert np.array_equal(args, rargs), np.argwhere(args != rargs)[:5]
    assert args.max() == S - 1


# --------------------------------------------------------------------------- GPU: the evaluation sweep
# the path-3 shapes on u8 rows: (J, S) with 16, 15, 11, 4, 3 and 2 warps per CTA without per-job arrays (one or
# two arrays take (256, 24) to 3 warps and two take (256, 25) to 2)
TILE_SHAPES = [(256, 9), (256, 12), (256, 16), (256, 24), (256, 25), (208, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("J,S", TILE_SHAPES, ids=["J%d-S%d" % s for s in TILE_SHAPES])
def test_headline_kernel_at_every_warp_count(engine, J, S):
    """Every objective with release dates off and on, integer and real starts alternating, at batch sizes of one CTA's
    worth (no warp has two tiles: no stagger), one and a half waves and one tile past a wave (grid * nw tiles);
    each on the default route, with one bulk copy per row, and without the stagger, against the fp32 oracle and on
    sampled rows the exact reference."""
    for i, fold in enumerate(FOLDS):
        for k, rel in enumerate((False, True)):
            arrays = job_arrays(fold, rel)
            path, nw = route_eval(J, S, arrays)
            assert path == 3
            wave = _sms() * nw * 32
            B = [33, wave * 3 // 2 + 5, wave + 1][(2 * i + k) % 3]
            ints = (i + k) % 2 == 0
            seed = 1000 * S + 10 * i + k
            fam = ["small", "dyadic", "equal", "zeros"][(i + k + S) % 4]
            T, opt, prio, r, w, d = _setup(engine, J, S, fam, fold, rel, B, ints, seed)
            ref = c_ref(T, opt, prio, r, ints, 1, fold, w, d)
            o, p = _dev(engine, opt, prio)
            label = (J, S, fold, rel, B, nw)
            for dbg in (0, _lib.TILE_DEBUG_ROW_COPIES, _lib.TILE_DEBUG_NO_STAGGER):
                got = _eval(engine, o, p, ref, ints, fold, label + (dbg,), _tile_debug=dbg)
                assert got == 3, (label, dbg, got)
            _note_path(3, J, S)
            NW_SEEN.add(nw)
            rows = sorted({0, 1, 2, 3, 4, 7, 11, B // 2, B - 1})
            _exact(T, opt, prio, r, ints, fold, w, d, ref, rows, label)


def _every_route(engine, J, S, fold, rel, B, ints, seed, fam="small"):
    """Every route of sb_eval at one shape; returns {route: path or None}."""
    from saturn_b200.engine import opt_by_position
    T, opt, prio, r, w, d = _setup(engine, J, S, fam, fold, rel, B, ints, seed)
    ref = c_ref(T, opt, prio, r, ints, 1, fold, w, d)
    o, p = _dev(engine, opt, prio)
    op = opt_by_position(o, p)
    label = (J, S, fold, rel, B)
    out = {}
    for name, kw, rows in [("default", {}, o), ("no_reorder", {"_reorder": False}, o),
                           ("reorder", {"_reorder": True}, o), ("generic", {"_force_generic": True}, o),
                           ("no_stream", {"_no_stream": True}, o), ("plain_addr", {"_plain_addr": True}, o),
                           ("by_position", {"by_position": True}, op),
                           ("by_position_pair", {"by_position": True, "_table_home": 2}, op),
                           ("by_position_global", {"by_position": True, "_table_home": 1}, op),
                           ("alt_shape", {"alt_shape": True}, o)]:
        if name == "alt_shape" and (fold != "makespan" or rel):
            continue
        out[name] = _eval(engine, rows, p, ref, ints, fold, label + (name,), **kw)
        if out[name] is not None:
            _note_path(out[name], J, S)
    rows = sorted({0, 1, 2, 3, 4, 5, 6, 9, 13, B - 1})
    _exact(T, opt, prio, r, ints, fold, w, d, ref, rows, label)
    return out


# (J, S, fold, release): the default path the route rules predict is asserted
ROUTE_CASES = [(224, 32, "makespan", False), (256, 28, "weighted_completion", False),
               (256, 28, "tardiness", True), (256, 32, "makespan", False), (256, 32, "weighted_tardiness", True),
               (1024, 8, "completion", False), (300, 16, "makespan", True), (128, 28, "makespan", False),
               (128, 29, "weighted_tardiness", False), (216, 31, "tardiness", True), (256, 11, "makespan", False),
               (256, 24, "max_lateness", False), (256, 25, "weighted_late_tasks", False),
               (256, 11, "late_tasks", True), (256, 28, "late_tasks", True), (256, 28, "max_tardiness", False)]


@pytest.mark.gpu
@pytest.mark.parametrize("J,S,fold,rel", ROUTE_CASES, ids=["J%d-S%d-%s-%s" % (c[0], c[1], c[2], "rel" if c[3] else "norel")
                                                           for c in ROUTE_CASES])
def test_every_route_at_large_tables(engine, J, S, fold, rel):
    """Path 4 by default (the table fits the position-major kernel but not beside the tiles), path 9 (it fits
    neither), path 4 again with the re-order forbidden, the generic kernel (table in shared memory up to J * S * 32
    = 116,224 bytes, in global memory above), by-position paths 5 / 7 / 8 (opt bytes >= 64), the alternate shape
    where it fits; opt bytes spread over every strategy, id base near 2^31."""
    paths = _every_route(engine, J, S, fold, rel, 97, (J + S) % 2 == 0, 7 * J + S)
    want = route_eval(J, S, job_arrays(fold, rel))[0]
    assert paths["default"] == want, (paths, want)
    assert paths["generic"] == 0 and paths["reorder"] == 9
    assert paths["no_reorder"] == (4 if want == 9 else want)
    assert paths["by_position"] == (5 if pos_smem(J, S * 8, job_arrays(fold, rel)) <= OPTIN else 8)
    assert paths["by_position_global"] == 8


@pytest.mark.gpu
def test_eval_host_at_32_strategies(engine):
    """sb_eval_host over three chunks at J = 256, S = 32 (the tile kernel with the table in global memory)."""
    import torch
    J, S = 256, 32
    B = 2 * _sms() * 8 * 32 * 4 + 77
    T, opt, prio, r, w, d = _setup(engine, J, S, "small", "weighted_tardiness", True, B, True, 5)
    ref = c_ref(T, opt, prio, r, True, 1, "weighted_tardiness", w, d)
    got = engine.eval_host(torch.from_numpy(opt), torch.from_numpy(prio), objective="weighted_tardiness").numpy()
    assert got.tobytes() == ref.tobytes()
    assert engine.last_eval_path() == 4
    _note_path(4, J, S)


def _strategy_table(J, S, seed):
    """A table whose per-column minimum sits on a uniformly random strategy (args up to S - 1)."""
    rng = np.random.default_rng(seed)
    T = (rng.integers(1, 64, (J, S, 8)) / 4.0).astype(np.float32)
    win = rng.integers(0, S, (J, 8))
    T[np.arange(J)[:, None], win, np.arange(8)[None, :]] = 0.125
    return T


@pytest.mark.gpu
@pytest.mark.parametrize("S", [17, 32])
def test_eval_full_and_decode_report_every_strategy(engine, S):
    """eval_full's scores, starts and masks, and decode's starts, masks and strategies, on the full table (strategy
    = opt >> 3, up to S - 1) and on the reduced table (strategy = the arg-min of the chosen column)."""
    import torch
    J, B = 200, 64
    T = _strategy_table(J, S, S)
    engine.set_table(T)
    tmin, args = engine.reduced_table()
    assert args.max() == S - 1
    for reduced in (False, True):
        opt, prio = candidates(J, B, 1 if reduced else S, S + reduced)
        tab = tmin[:, None, :] if reduced else T
        ref, cst, cm = c_ref(tab, opt, prio, None, True, 1, "makespan", None, None, want_plan=True)
        o, p = _dev(engine, opt, prio)
        tot, st, m = engine.eval_full(o, p, reduced=reduced)
        torch.cuda.synchronize()
        assert tot.cpu().numpy().tobytes() == ref.tobytes()
        assert np.array_equal(st.cpu().numpy(), cst) and np.array_equal(m.cpu().numpy().astype(np.uint32), cm)
        seen = set()
        for b in range(0, B, 5):
            dec = engine.decode(opt[b], prio[b], reduced=reduced)
            want = args[np.arange(J), opt[b] & 7] if reduced else opt[b] >> 3
            assert np.array_equal(dec["strategy"], want), (reduced, b)
            assert np.array_equal(dec["gpus"], (opt[b] & 7) + 1)
            assert np.array_equal(dec["start"], cst[b]) and np.array_equal(dec["slotmask"], cm[b])
            assert dec["makespan"] == float(ref[b])
            seen |= set(want.tolist())
        assert max(seen) == S - 1, (reduced, max(seen))


@pytest.mark.gpu
def test_validate_refuses_strategies_beyond_the_table(engine):
    """S = 17: a byte with s = 17..31 is refused, s = 16 (bytes 128..135) is accepted."""
    J = 64
    T = rt_table("small", J, 17, 3)
    engine.set_table(T)
    opt, prio = candidates(J, 32, 17, 4)
    opt[:, 5] = (16 << 3) | 2
    o, p = _dev(engine, opt, prio)
    assert engine.validate(o, p) == 0
    bad = opt.copy()
    for i, s in enumerate(range(17, 32)):
        bad[2 * i, (3 * i) % J] = (s << 3) | (i % 8)
    o, p = _dev(engine, bad, prio)
    assert engine.validate(o, p) == 15


# --------------------------------------------------------------------------- GPU: search layouts
VERIFY = _lib.HOOK_VERIFY_INCREMENTAL
SEARCH_CASES = []
for _c in [
    # position-major populations on u8 rows (PB = 1)
    ("pos_S16_J256", 256, 1000, dict(S=16, warm=True, twice=True)),
    ("pos_S16_J256_tie_t0", 256, 33, dict(S=16, family="small", resample=-1, t0=True)),
    ("pos_S16_J256_noinc", 256, 1000, dict(S=16, hooks=_lib.HOOK_NO_INCREMENTAL, resample=-1)),
    ("pos_S16_J256_round1", 256, 4097, dict(S=16, hooks=_lib.HOOK_ROUND1_MOVES, family="small")),
    ("pos_S16_J256_verify", 256, 1000, dict(S=16, hooks=VERIFY, resample=-1)),
    ("pos_S24_J200", 200, "wave+17", dict(S=24, warm=True)),
    ("pos_S24_J200_tie_t0", 200, 1000, dict(S=24, family="equal", resample=-1, t0=True, hooks=VERIFY)),
    # the J = 256, S = 11 boundary: the per-job arrays move the population from the tile to position-major
    ("bound_S11_makespan", 256, 1000, dict(S=11, warm=True)),
    ("bound_S11_wtard_rel", 256, 1000, dict(S=11, objective="weighted_tardiness", release=True, resample=-1)),
    ("bound_S11_late_rel", 256, 1000, dict(S=11, objective="late_tasks", release=True, family="small", t0=True)),
    ("bound_S11_max_lateness", 256, 1000, dict(S=11, objective="max_lateness", release=True, resample=-1)),
    # unfused rounds the library falls back to by itself
    ("unfused_S32_J256", 256, 1000, dict(S=32, warm=True)),
    ("unfused_S32_J256_tie_t0", 256, 33, dict(S=32, family="small", resample=-1, t0=True)),
    ("unfused_C5_J1024_S8", 1024, 300, dict(S=8, resample=-1)),
    ("unfused_S28_late_rel", 256, 1000, dict(S=28, objective="late_tasks", release=True, warm=True)),
    # fused tile rounds at 8 and 9 warps
    ("tile_S10_J256", 256, 1000, dict(S=10, resample=-1, warm=True)),
    ("tile_S9_J256_tie_t0", 256, "wave+17", dict(S=9, family="small", resample=-1, t0=True)),
    ("tile_S9_wmax_tardiness", 256, 1000, dict(S=9, objective="weighted_max_tardiness", resample=-1, twice=True)),
    ("tile_S9_max_lateness", 256, 1000, dict(S=9, objective="max_lateness", warm=True)),
]:
    _k = dict(_c[3])
    _c_ = case(_c[0], _c[1], _c[2], reduced=False, **_k)
    _c_["seed"] = 104729 + 31 * len(SEARCH_CASES) + _c[1]
    SEARCH_CASES.append(_c_)


@pytest.mark.gpu
@pytest.mark.parametrize("c", SEARCH_CASES, ids=[c["name"] for c in SEARCH_CASES])
def test_full_table_population_invariants(engine, c):
    """I1-I9 of test_gpu_search_state after every scripted step, with the layout and the wave the route rules
    predict (tile-plan warps for the fused round, 16 for position-major)."""
    digests, layouts = run_script(engine, c)
    arrays = job_arrays(c["objective"], c["release"])
    layout, warps = route_search(c["J"], c["S"], arrays)
    assert layouts == {layout}, (c["name"], layouts, layout)
    assert engine.search_wave(reduced=False, objective=c["objective"]) == warps * 32 * _sms()
    LAYOUTS_SEEN.setdefault(layout, set()).add((c["J"], c["S"]))
    if c["hooks"] & VERIFY:
        assert engine.search_verify_count() == 0
    if c["twice"]:
        again, _ = run_script(engine, c)
        for i, (a, b) in enumerate(zip(digests, again)):
            assert a == b, (c["name"], "I8: the population differs between two identical runs at step", i)


RUN_SHAPES = [(256, 10, 1), (256, 16, 2), (256, 32, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("J,S,layout", RUN_SHAPES, ids=["layout%d" % s[2] for s in RUN_SHAPES])
def test_search_run_on_the_full_table(engine, J, S, layout):
    """Engine.search_run(reduced=False) end to end: the library loop equals the Python driver, and the oracle
    scores the returned plan at the returned score."""
    from saturn_b200.search import run_search
    T = make_table("rnd", J, S, J + S)
    engine.set_table(T, sentinel=1e6)
    assert route_search(J, S)[0] == layout
    chains = engine.search_wave(reduced=False) * 2
    kw = dict(chains=chains, rounds=24, seed=5, reduced=False, use_dist=False, exchange_every=8)
    a = run_search(engine, **kw)
    b = run_search(engine, _python_driver=True, **kw)
    assert a.makespan == b.makespan and np.array_equal(a.opt, b.opt) and np.array_equal(a.prio, b.prio)
    tab = R.canon_table(T, range(1, 9))
    assert c_oracle.evaluate(tab, a.opt[None], a.prio[None], True, np.float32)[0] == np.float32(a.makespan)
    tmin, args = engine.reduced_table()
    ok = proposable(tmin, args, reduced=False)
    assert ok[np.arange(J), a.opt].all()
    assert engine.search_validate() == 0


# --------------------------------------------------------------------------- GPU: the product entry
@pytest.mark.gpu
def test_solve_table_at_32_executors(engine):
    """solve_table with 32 executors and ties across them returns the plan solve() returns on the
    strategies_from_table view (same seed), and reports the first executor attaining each chosen cell's minimum."""
    from conftest import DuckTask
    from saturn_b200 import solve, solve_table, strategies_from_table
    from saturn_b200 import solver as SV
    J, E, G = 24, 32, 8
    T, valid = R.synth_table(J, E, G, seed=41)
    T = np.where(valid, np.round(T / 500.0) * 500.0, T).astype(np.float32)      # ties across executors
    T[:, 20:, :] = np.where(valid[:, 20:, :], T[:, 19:20, :], T[:, 20:, :])
    T[0, 31, 3], valid[0, 31, 3] = 1.0, True                                     # executor 31 wins job 0 at k = 4
    strategies = strategies_from_table(T, valid, executors=["e%d" % s for s in range(E)])
    tasks = [DuckTask("t%d" % j, strategies[j]) for j in range(J)]
    a = solve(tasks, None, chains=8192, rounds=40, seed=3, engine=engine)
    dev_a = SV.last_stats["device_makespan"]
    b = solve_table(T, valid, chains=8192, rounds=40, seed=3, engine=engine)
    assert SV.last_stats["device_makespan"] == dev_a
    assert all(a[i] == b[i] for i in range(5)) and b[5] == pytest.approx(a[5], rel=1e-12)
    for j in range(J):
        g = int(np.argmax(b[2][j]))
        col = np.where(valid[j, :, g], T[j, :, g], np.inf)
        assert b[6][j] == int(np.argmin(col)), (j, b[6][j], col)
    tmin, args = engine.reduced_table()
    assert args[0, 3] == 31


# --------------------------------------------------------------------------- GPU: coverage
@pytest.mark.gpu
def test_zz_every_route_and_layout_ran_above_8_strategies():
    """Runs after the file: paths 0, 3, 4, 5, 6, 7, 8, 9 and layouts 0, 1, 2 each ran at S > 8; path 3 ran at 16, 15,
    11, 4, 3 and 2 warps per CTA; a position-major population held u8 rows.  Skipped after a partial run."""
    if len(PATHS_SEEN) == 0 or len(LAYOUTS_SEEN) == 0:
        pytest.skip("the sweep did not run")
    print("paths at S > 8:", {p: sorted(v) for p, v in sorted(PATHS_SEEN.items())})
    print("layouts:", {lay: sorted(v) for lay, v in sorted(LAYOUTS_SEEN.items())})
    print("path-3 warps:", sorted(NW_SEEN))
    assert {0, 3, 4, 5, 6, 7, 8, 9} <= set(PATHS_SEEN), sorted(PATHS_SEEN)
    assert set(LAYOUTS_SEEN) == {0, 1, 2}
    assert {16, 15, 11, 4, 3, 2} <= NW_SEEN, sorted(NW_SEEN)
    assert any(J <= 256 for J, _ in LAYOUTS_SEEN[2])
