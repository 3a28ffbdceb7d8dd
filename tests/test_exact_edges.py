"""Every evaluation path against an EXACT reference on tie-heavy and boundary inputs.

The per-feature suites draw log-uniform non-integer runtimes and uniform random candidates, so exact ties (equal slot
ready times, a release date equal to a slot's ready time, a completion equal to its due date) almost never occur, and
their references are fp32 restatements of the same arithmetic.  Here:

* `oracle/ref_exact.py` is the list schedule in exact rational arithmetic, under every fold of the library (the ten
  objectives of saturn_b200.engine.OBJECTIVES), with and without release dates, on 1..8 nodes.  On the EXACT
  FAMILIES below fp32 rounds nothing, and the reference asserts that for every value it forms; the CPU tests pin it
  against the float64 oracle and the fp32 C port, value for value, starts and slot masks included.
* Seeded generators make the ties: equal runtimes, runtimes in {1, 2, 3}, dyadic fractions, zeros and -0.0; gang
  patterns of explicit opt rows (every job on 8, on 1, 1 and 8 alternating, k cycling 1..8, every job on 7: all three
  shifter stages); identity, reversed and random orders; release dates equal to exact slot ready times, <= 0 and
  -0.0; due dates equal to exact completions, one exact step before them (late by the smallest margin of the
  family), -0.0 (with zero runtimes: on time), negative and beyond every completion; weights in {1/4 .. 4}, and the
  same scaled by 2^-140 into the fp32 subnormal range.
* GPU: a shape sweep (J from 1 to 65535, B around one wave of the tile kernel, 1..8 nodes) runs every route a shape
  admits and checks every score against the fp32 C oracle bit for bit, the arg-min key, and on the exact families the
  exact reference's scores, starts and masks.  The kernel path of every run is recorded, and the last test asserts
  that every path occurred, under every fold.  Inputs that are not exact families (runtimes in [2^22, 2^23],
  r = 2^24 - 1, selected 1e8 and +inf cells, a due-date spread of 2^24 - 1 under the maximum lateness, late-count due
  dates at the fp32 neighbours of rounded completions, the maximum stretch's weights fp32(1 / p*)) are checked against
  the fp32 oracle only.
* GPU: short searches on tie-heavy exact tables with the incremental-score verifier.
* The table refusal: negative and NaN cells are refused by sb_set_table (host or device T) and by solve_table.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import ref_exact as X
from oracle import ref_late_tasks as LT
from oracle import ref_max_lateness as ML
from oracle import ref_max_tardiness as MT
from oracle import ref_release as RR
from saturn_b200.engine import OBJECTIVES

FOLDS = OBJECTIVES
NEW_FOLDS = FOLDS[5:]                # the folds of other oracles than ref_release's list schedule
GANGS = ("k8", "k1", "alt18", "cycle", "k7")
ORDERS = ("identity", "reversed", "random")
WEIGHTS = np.array([0.25, 0.5, 1.0, 2.0, 4.0])
KEY_MAX = 2 ** 63 - 1
ID_BASE = 7


# --------------------------------------------------------------------------- seeded input families
def rt_table(family, J, S, seed):
    """T[J][S][8] fp32 with one column per GPU count (gcount = 1..8, so it is already the canonical table).
    Exact families: "equal" (every cell 2.5), "small" ({1, 2, 3}), "dyadic" (multiples of 1/8 in (0, 2]), "zeros" (0,
    -0.0, 1 and 2).  fp32-only families: "large" (values in [2^22, 2^23]), "mid" (values in [2^16, 2^17]: sums of up
    to 128 stay below 2^24 and round), "sentinel" ({1, 2, 3} with 1e8 and +inf cells)."""
    rng = np.random.default_rng(seed)
    shape = (J, S, 8)
    if family == "equal":
        a = np.full(shape, 2.5)
    elif family == "small":
        a = rng.integers(1, 4, shape).astype(np.float64)
    elif family == "dyadic":
        a = rng.integers(1, 17, shape) / 8.0
    elif family == "zeros":
        a = np.array([0.0, -0.0, 1.0, 2.0])[rng.integers(0, 4, shape)]
    elif family == "large":
        a = rng.uniform(2.0 ** 22, 2.0 ** 23, shape)
    elif family == "mid":
        a = rng.uniform(2.0 ** 16, 2.0 ** 17, shape)
    elif family == "sentinel":
        a = rng.integers(1, 4, shape).astype(np.float64)
        pick = rng.uniform(size=shape)
        a[pick < 0.1] = 1e8
        a[pick > 0.95] = np.inf
    else:
        raise ValueError(family)
    return a.astype(np.float32)


def gang_k(pattern, J):
    i = np.arange(J)
    return {"k8": np.full(J, 8), "k1": np.ones(J, np.int64), "alt18": np.where(i % 2 == 0, 1, 8),
            "cycle": i % 8 + 1, "k7": np.full(J, 7)}[pattern].astype(np.int64)


def candidates(J, B, hi, seed):
    """opt[B][J], prio[B][J] (numpy): row b has gang pattern GANGS[b % 5] and order ORDERS[(b // 5) % 3]; the high
    bits of every opt byte (strategy, or node with several nodes) are uniform in [0, hi)."""
    rng = np.random.default_rng(seed)
    b = np.arange(B)
    K = np.stack([gang_k(g, J) for g in GANGS]).astype(np.uint8)
    opt = (rng.integers(0, hi, (B, J), dtype=np.uint8) << 3) | (K[b % 5] - 1)
    prio = np.empty((B, J), dtype=np.uint8 if J <= 256 else np.uint16)
    order = (b // 5) % 3
    prio[order == 0] = np.arange(J)
    prio[order == 1] = np.arange(J)[::-1]
    rnd = np.nonzero(order == 2)[0]
    for c0 in range(0, len(rnd), 4096):
        rows = rnd[c0:c0 + 4096]
        prio[rows] = np.argsort(rng.random((len(rows), J)), axis=1)
    return opt, prio


def release_dates(family, tab, opt, prio, ints, nodes, seed):
    """None; "ready": the exact starts of candidate 0 under the rule without release dates (each is a slot's ready
    time), with a quarter of them replaced by -0.0 and a quarter by negative multiples of 1/8; "nonpos": only values
    <= 0, -0.0 and 0 included; "huge": 2^24 - 1 on every third job (not an exact family)."""
    if family is None:
        return None
    J = len(prio[0])
    rng = np.random.default_rng(seed)
    if family == "ready":
        r = np.array([float(s) for s in X.schedule(tab, opt[0], prio[0], None, ints, nodes)[1]])
        pick = rng.integers(0, 4, J)
        r[pick == 1] = -0.0
        r[pick == 2] = -rng.integers(1, 64, J)[pick == 2] / 8.0
    elif family == "nonpos":
        r = np.array([0.0, -0.0, -0.125, -3.0])[rng.integers(0, 4, J)]
    elif family == "huge":
        r = np.zeros(J)
        r[::3] = 2.0 ** 24 - 1
    else:
        raise ValueError(family)
    return r.astype(np.float32)


def due_dates(tab, opt, prio, ints, nodes, release, seed):
    """Per job one of: the exact completion e of candidate 0 (e - d = 0 there: on time), e minus one step of the
    family (1/8, or 1 above J = 300: late by the smallest exact margin), -0.0 (a zero-runtime job at +0 is on time), a
    negative multiple of 1/8 (a negative integer above J = 300, where sums of tardiness need the whole fp32 mantissa),
    or 2^19 (beyond every completion of these tables)."""
    J = len(prio[0])
    rng = np.random.default_rng(seed)
    _, st, _ = X.schedule(tab, opt[0], prio[0], release, ints, nodes)
    e = np.array([float(st[j]) + float(tab[j][0 if nodes > 1 else opt[0][j] >> 3][opt[0][j] & 7]) for j in range(J)])
    pick = rng.integers(0, 5, J)
    step = 0.125 if J <= 300 else 1.0
    neg = -rng.integers(1, 64, J) / 8.0 if J <= 300 else -rng.integers(1, 8, J).astype(np.float64)
    d = np.select([pick == 0, pick == 1, pick == 2, pick == 3], [e, e - step, np.full(J, -0.0), neg], 2.0 ** 19)
    return d.astype(np.float32)


def per_job(fold, tab, opt, prio, ints, nodes, release, seed, tiny=False):
    """Weights in {1/4, 1/2, 1, 2, 4} ({1, 2, 4} above J = 300, where sums of weighted completions need the whole
    fp32 mantissa), scaled by 2^-140 (fp32 subnormals) with `tiny`, and due_dates(), as the fold's flag bits need
    them."""
    J = len(prio[0])
    use_w, use_d = X.needs(fold)
    w = (WEIGHTS[np.random.default_rng(seed).integers(0 if J <= 300 else 2, 5, J)] * (2.0 ** -140 if tiny else 1.0)
         ).astype(np.float32) if use_w else None
    d = due_dates(tab, opt, prio, ints, nodes, release, seed + 1) if use_d else None
    return w, d


def c_ref(tab, opt, prio, release, ints, nodes, fold, w, d, want_plan=False):
    J = opt.shape[1]
    r = np.zeros(J, np.float32) if release is None else release
    return RR.c_evaluate(tab, opt, prio, r, ints, np.float32, threads=8, nodes=nodes, objective=fold, weights=w,
                         due=d, want_plan=want_plan)


def f64_ref(tab, opt, prio, release, ints, nodes, fold, w, d):
    """(score[B], start[B][J], mask[B][J]) of the float64 restatement: ref_release's Python list schedule, or the
    fold's own oracle (use_c=False) for the folds ref_release does not know."""
    if fold in NEW_FOLDS:
        mod = {"max_lateness": ML, "late_tasks": LT, "weighted_late_tasks": LT, "max_tardiness": MT,
               "weighted_max_tardiness": MT}[fold]
        kw = {} if mod is ML else {"weights": w}
        return mod.evaluate(tab, opt, prio, d, release, ints, np.float64, nodes, use_c=False, want_plan=True, **kw)
    r64 = np.zeros(opt.shape[1]) if release is None else release
    out = [RR.list_schedule(tab, opt[b], prio[b], r64, ints, np.float64, nodes=nodes, objective=fold, weights=w, due=d)
           for b in range(len(opt))]
    return (np.array([o[0] for o in out]), np.array([o[1] for o in out], np.float64),
            np.array([o[2] for o in out], np.uint32))


# --------------------------------------------------------------------------- CPU: pin the exact reference
PIN_CASES = [(1, 1, "equal", True), (2, 8, "zeros", False), (7, 3, "small", True), (31, 1, "dyadic", False),
             (33, 5, "equal", True), (64, 2, "dyadic", True), (97, 6, "small", False), (128, 7, "zeros", True),
             (256, 8, "small", True), (300, 1, "dyadic", True), (300, 4, "equal", False)]


@pytest.mark.parametrize("case", PIN_CASES, ids=lambda c: "J%d-n%d-%s-%s" % (c[0], c[1], c[2], "int" if c[3] else "real"))
@pytest.mark.parametrize("rel", [None, "ready", "nonpos"])
@pytest.mark.parametrize("fold", FOLDS)
def test_exact_reference_agrees_with_both_oracles(case, rel, fold):
    """On exact-family inputs the exact reference, the float64 oracle and the fp32 C port agree value for value on the
    score, every start and every slot mask (15 candidates: every gang pattern under every order); weights are
    subnormal with the non-positive release dates."""
    J, nodes, fam, ints = case
    S = 1 if nodes > 1 else 3
    seed = J * 101 + nodes
    tab = rt_table(fam, J, S, seed)
    opt, prio = candidates(J, 15, nodes if nodes > 1 else S, seed + 1)
    r = release_dates(rel, tab, opt, prio, ints, nodes, seed + 2)
    w, d = per_job(fold, tab, opt, prio, ints, nodes, r, seed + 3, tiny=rel == "nonpos")
    exact, xst, xm = X.batch(tab, opt, prio, r, ints, nodes, fold, w, d)
    c32, cst, cm = c_ref(tab, opt, prio, r, ints, nodes, fold, w, d, want_plan=True)
    s64, st64, m64 = f64_ref(tab, opt, prio, r, ints, nodes, fold, w, d)
    for b in range(len(opt)):
        assert exact[b] == s64[b] == float(c32[b]), (b, exact[b], s64[b], c32[b])
        assert np.array_equal(xst[b], st64[b]) and np.array_equal(xst[b], cst[b].astype(np.float64))
        assert np.array_equal(xm[b], m64[b]) and np.array_equal(xm[b], cm[b])


def test_every_objective_has_both_references_and_every_sweep():
    """The objectives of the library, ref_exact's folds, the objectives ref_release.c_evaluate scores and the folds of
    the three sweeps (this file, test_gpu_search_state's cases, test_gpu_strategy_axis's tile sweep) are the same
    list: an objective cannot be added without joining them.  Both references agree on a small input under each, with
    the library's flag bits."""
    import test_gpu_search_state as SS
    import test_gpu_strategy_axis as SA
    from saturn_b200.engine import objective_flag
    assert X.OBJECTIVES == RR.C_OBJECTIVES == FOLDS == SA.FOLDS == OBJECTIVES
    assert {c["objective"] for c in SS.CASES} == set(OBJECTIVES)
    tab = np.array([[[1.0, 0.5] + [2.0] * 6], [[3.0] * 8]], np.float32)
    opt, prio = np.array([[1, 0]], np.uint8), np.array([[1, 0]], np.uint8)
    w, d = np.array([2.0, 0.5], np.float32), np.array([3.0, 2.0], np.float32)
    for o in OBJECTIVES:
        assert X.objective_flag(o) == objective_flag(o), o
        c32 = RR.c_evaluate(tab, opt, prio, np.zeros(2), objective=o, weights=w, due=d)
        assert float(c32[0]) == float(X.schedule(tab, opt[0], prio[0], objective=o, weights=w, due=d)[0]), o


def test_exact_reference_refuses_inputs_that_fp32_would_round():
    """A value that fp32 cannot hold exactly fails loudly instead of weakening a comparison: a runtime of 1/3, times
    past 2^24, a weight that makes w * e round, and a sum that outgrows the fp32 mantissa."""
    J = 4
    opt = np.zeros(J, np.uint8)
    prio = np.arange(J)
    with pytest.raises(X.NotExact):
        X.schedule(np.full((J, 1, 8), 1.0 / 3.0), opt, prio)
    with pytest.raises(X.NotExact):
        X.schedule(np.full((J, 1, 8), 2.0 ** 23 + 1.0), np.full(J, 7, np.uint8), prio)
    with pytest.raises(X.NotExact):
        X.schedule(np.full((J, 1, 8), 1.0 + 2.0 ** -23), opt, prio, objective="weighted_completion",
                   weights=[3.0] * J)
    tab = np.full((J, 1, 8), 2.0 ** 23 - 1.0)
    tab[0, 0, 0] = 0.5
    with pytest.raises(X.NotExact):
        X.schedule(tab, opt, np.array([0, 1, 2, 3]), objective="completion")
    # +inf stays exact: a selected absent cell makes the score +inf
    sc, st, _ = X.schedule(np.full((J, 1, 8), np.inf), opt, prio, objective="weighted_tardiness", weights=[1.0] * J,
                           due=[0.0] * J)
    assert sc == float("inf") and st[0] == 0


def test_solve_table_refuses_negative_and_nan_cells():
    """solve_table raises SolverError for a negative or NaN cell before any device call, with or without a mask
    (the engine here is a plain object: touching it would raise AttributeError instead).  -0.0 is a zero runtime and
    +inf / sentinels are legal; those reach the device call."""
    from saturn_b200 import solver as S
    T = np.full((3, 2, 8), 5.0, dtype=np.float32)
    mask = np.ones(T.shape, dtype=bool)
    for bad in (-1.0, -1e-30, np.nan):
        Tb = T.copy()
        Tb[1, 1, 3] = bad
        for m in (None, mask):
            with pytest.raises(S.SolverError, match="negative or NaN"):
                S.solve_table(Tb, m, engine=object())
    Tb = T.copy()
    Tb[0] = -1.0                                      # a task with no usable cell sent every finite cell before
    with pytest.raises(S.SolverError, match="negative or NaN"):
        S.solve_table(Tb, np.zeros(T.shape, dtype=bool), engine=object())
    for ok in (-0.0, np.inf, 1e8):
        Tb = T.copy()
        Tb[1, 1, 3] = ok
        with pytest.raises(AttributeError):
            S.solve_table(Tb, mask, engine=object())


# --------------------------------------------------------------------------- GPU helpers
def _dev(engine, opt, prio):
    import torch
    from saturn_b200.engine import padded_rows
    B, J = opt.shape
    o = padded_rows(B, J, torch.uint8, engine.device)
    p = padded_rows(B, J, engine.prio_dtype, engine.device)
    o.copy_(torch.from_numpy(opt))
    p.copy_(torch.from_numpy(prio.astype(np.int32) if J > 256 else prio).to(engine.prio_dtype))
    return o, p


def _unaligned(t):
    """The same rows at a base address one element past an aligned one: no bulk copies, plain row loads."""
    import torch
    B, J = t.shape
    buf = torch.zeros(B * J + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(B, J)
    v.copy_(t)
    return v


def _key_of(ref):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (ID_BASE + i)


COVERAGE = []          # (J, nodes, objective, release, path) of every run; path None = refused as unsupported
SWEEP_DONE = set()


def _set_per_job(engine, r, w, d):
    if r is not None:
        engine.set_release(r)
    if w is not None:
        engine.set_weights(w)
    if d is not None:
        engine.set_due(d)


def _routes(fold, released, nodes):
    """Every route of sb_eval: (name, eval kwargs, rows) with rows "job" (job-indexed, aligned), "unaligned" or
    "position" (opt in schedule order)."""
    out = [("default", {}, "job"), ("plain_addr", {"_plain_addr": True}, "job"), ("no_stream", {"_no_stream": True}, "job"),
           ("generic", {"_force_generic": True}, "job"), ("unaligned", {}, "unaligned"),
           ("by_position", {"by_position": True}, "position"),
           ("by_position_pair", {"by_position": True, "_table_home": 2}, "position"),
           ("by_position_global", {"by_position": True, "_table_home": 1}, "position"),
           ("reorder", {"_reorder": True}, "job"), ("no_reorder", {"_reorder": False}, "job")]
    if fold == "makespan" and not released and nodes == 1:
        out.append(("alt_shape", {"alt_shape": True}, "job"))
    return out


def _run_routes(engine, opt, prio, ref, ints, fold, released, nodes, label):
    """Each route: the scores equal `ref` bit for bit and the key is its arg-min; a route the library does not offer
    at this shape must be refused with SB_ERR_UNSUPPORTED.  Returns {route: path or None}."""
    import torch
    from saturn_b200._lib import SaturnB200Error
    from saturn_b200.engine import opt_by_position
    o_t, p_t = _dev(engine, opt, prio)
    rows = {"job": (o_t, p_t)}
    rows["unaligned"] = (_unaligned(o_t), _unaligned(p_t))
    rows["position"] = (opt_by_position(o_t, p_t), p_t)
    paths = {}
    for name, kw, which in _routes(fold, released, nodes):
        o, p = rows[which]
        key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
        try:
            got = engine.eval(o, p, integer_starts=ints, reduced=nodes > 1, objective=fold, best_key=key,
                              id_base=ID_BASE, **kw)
            torch.cuda.synchronize()
        except SaturnB200Error as e:
            assert "error -4:" in str(e), (label, name, str(e))
            paths[name] = None
            COVERAGE.append(label + (None,))
            continue
        path = engine.last_eval_path()
        paths[name] = path
        COVERAGE.append(label + (path,))
        g = got.cpu().numpy()
        assert g.tobytes() == ref.tobytes(), (label, name, path, np.nonzero(g != ref)[0][:5])
        assert int(key.item()) == _key_of(ref), (label, name, path)
    return paths, o_t, p_t


def _check_plan(engine, o_t, p_t, opt, prio, ints, fold, nodes, ref, cst, cm, label):
    """eval_full's scores, starts and masks and one decode equal the fp32 oracle."""
    import torch
    tot, start, mask = engine.eval_full(o_t, p_t, integer_starts=ints, reduced=nodes > 1, objective=fold)
    torch.cuda.synchronize()
    assert tot.cpu().numpy().tobytes() == ref.tobytes(), label
    st = start.cpu().numpy()
    m = mask.cpu().numpy().astype(np.uint32)
    assert np.array_equal(st, cst) and np.array_equal(m, cm), label
    b = len(opt) // 2
    dec = engine.decode(opt[b], prio[b], integer_starts=ints, reduced=nodes > 1, objective=fold)
    assert dec["makespan"] == float(ref[b]), label
    assert np.array_equal(dec["start"], cst[b]) and np.array_equal(dec["slotmask"], cm[b] & 0xffff), label
    assert np.array_equal(dec["node"], (cm[b] >> 16).astype(np.uint8)), label
    return st, m


def _check_exact(tab, opt, prio, r, ints, nodes, fold, w, d, got, st, m, rows, label):
    xs, xst, xm = X.batch(tab, opt, prio, r, ints, nodes, fold, w, d, rows=rows)
    assert np.array_equal(xs, got[rows].astype(np.float64)), (label, xs, got[rows])
    assert np.array_equal(xst, st[rows].astype(np.float64)), label
    assert np.array_equal(xm, m[rows]), label


def _subsample(B, J, seed):
    n = B if B * J <= 20000 else max(2, min(8, 200000 // (J * 4)))
    if n >= B:
        return list(range(B))
    rng = np.random.default_rng(seed)
    return sorted(set([0, B - 1] + rng.choice(B, size=n - 2, replace=False).tolist()))


def _sweep_one(engine, J, nodes, S, fam, fold, rel, B, ints, seed, tiny=False):
    """One shape: set the table and per-job data, build tie-heavy candidates, run every route against the fp32 oracle
    and the exact reference, plus eval_full and decode."""
    T = rt_table(fam, J, S, seed)
    engine.set_table(T, nodes=nodes)
    opt, prio = candidates(J, B, nodes if nodes > 1 else S, seed + 1)
    r = release_dates(rel, T, opt, prio, ints, nodes, seed + 2)
    w, d = per_job(fold, T, opt, prio, ints, nodes, r, seed + 3, tiny)
    _set_per_job(engine, r, w, d)
    ref = c_ref(T, opt, prio, r, ints, nodes, fold, w, d)
    label = (J, nodes, fold, r is not None)
    _, o_t, p_t = _run_routes(engine, opt, prio, ref, ints, fold, r is not None, nodes, label)
    n = min(B, 512)                                   # plans of the first rows (every gang pattern and order)
    _, cst, cm = c_ref(T, opt[:n], prio[:n], r, ints, nodes, fold, w, d, want_plan=True)
    st, m = _check_plan(engine, o_t[:n], p_t[:n], opt[:n], prio[:n], ints, fold, nodes, ref[:n], cst, cm, label)
    _check_exact(T, opt, prio, r, ints, nodes, fold, w, d, ref, st, m, _subsample(n, J, seed), label)


# --------------------------------------------------------------------------- GPU: the shape sweep (makespan)
SWEEP_J = [1, 2, 31, 32, 33, 95, 96, 97, 255, 256, 257, 1023, 1024, 1025, 4096, 6144, 6145, 16384, 65535]


def _wave():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 32


@pytest.mark.gpu
@pytest.mark.parametrize("J", SWEEP_J)
def test_shape_sweep_every_route(engine, J):
    """Makespan, one node (full table, S = 2) at B in {1, 33, wave - 1, wave + 1} (small B from J = 4096 on), then the
    reduced table on 2..8 nodes; integer and real starts alternate with B."""
    idx = SWEEP_J.index(J)
    fams = ["equal", "small", "dyadic", "zeros"] if J <= 300 else ["equal", "small", "zeros"]
    wave = _wave()
    Bs = [1, 33, wave - 1, wave + 1] if J <= 1025 else [1, 33]
    for i, B in enumerate(Bs):
        _sweep_one(engine, J, 1, 2, fams[(idx + i) % len(fams)], "makespan", None, B, i % 2 == 0, 1000 * idx + i)
    nodes = 2 + idx % 7
    _sweep_one(engine, J, nodes, 1, fams[idx % len(fams)], "makespan", "ready" if idx % 2 else None, 33, idx % 2 == 0,
               1000 * idx + 50)
    SWEEP_DONE.add(("sweep", J))


OBJ_J = [33, 256, 257, 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("nodes", [1, 6, 8])
@pytest.mark.parametrize("J", OBJ_J)
@pytest.mark.parametrize("fold", FOLDS)
def test_every_objective_with_and_without_release(engine, fold, J, nodes):
    """Every fold, release off and on, at J in {33, 256, 257, 1024} on 1, 6 and 8 nodes.  One node uses the full
    table with S = 8 at J = 1024 (too large to sit beside the tiles: path 4 without the re-order) and S = 4 below.
    Weights are subnormal in one of the two runs."""
    S = 1 if nodes > 1 else (8 if J == 1024 else 4)
    for k, rel in enumerate([None, "ready"]):
        seed = 7919 * OBJ_J.index(J) + 31 * nodes + 3 * FOLDS.index(fold) + k
        fam = ["small", "zeros", "equal", "dyadic"][(seed // 3) % (4 if J <= 300 else 2)]
        _sweep_one(engine, J, nodes, S, fam, fold, rel, 33 if k == 0 else 97, (seed % 2) == 0, seed,
                   tiny=(k + nodes) % 2 == 1)
    SWEEP_DONE.add((fold, J, nodes))


@pytest.mark.gpu
def test_eval_host_over_several_chunks(engine):
    """sb_eval_host over three chunks (SMs x 8 x 32 x 4 candidates each) at J = 256, weighted tardiness with release
    dates, against the fp32 oracle."""
    import torch
    J = 256
    chunk = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 32 * 4
    B = 2 * chunk + 77
    T = rt_table("small", J, 2, 5)
    engine.set_table(T)
    opt, prio = candidates(J, B, 2, 6)
    r = release_dates("ready", T, opt, prio, True, 1, 7)
    w, d = per_job("weighted_tardiness", T, opt, prio, True, 1, r, 8)
    _set_per_job(engine, r, w, d)
    ref = c_ref(T, opt, prio, r, True, 1, "weighted_tardiness", w, d)
    got = engine.eval_host(torch.from_numpy(opt), torch.from_numpy(prio.astype(np.int32) if J > 256 else prio),
                           objective="weighted_tardiness").numpy()
    assert got.tobytes() == ref.tobytes()
    COVERAGE.append((J, 1, "weighted_tardiness", True, engine.last_eval_path()))
    rows = _subsample(B, J, 9)
    xs = X.batch(T, opt, prio, r, True, 1, "weighted_tardiness", w, d, rows=rows)[0]
    assert np.array_equal(xs, got[rows].astype(np.float64))


# case: (table family, folds)
FP32_EDGES = {"large": ("large", ("makespan", "weighted_tardiness")),
              "huge_release": ("small", ("makespan", "weighted_tardiness")),
              "sentinel": ("sentinel", ("makespan", "weighted_tardiness")),
              "lateness_spread": ("dyadic", ("max_lateness",)),
              "late_neighbours": ("mid", ("late_tasks", "weighted_late_tasks")),
              "stretch_weights": ("dyadic", ("weighted_max_tardiness",))}


def _fp32_edge_per_job(case, fold, T, opt, prio, ints, seed):
    """(release, weights, due) of one fp32-only case."""
    J = T.shape[0]
    rng = np.random.default_rng(seed)
    r = w = d = None
    if case == "huge_release":
        r = release_dates("huge", T, opt, prio, ints, 1, 0)
    if fold == "weighted_tardiness":
        w = WEIGHTS[np.random.default_rng(seed).integers(0, 5, J)].astype(np.float32)
        d = (np.random.default_rng(seed).uniform(0, 2.0 ** 23, J) * (J / 8)).astype(np.float32)
        d = np.minimum(d, np.float32(2.0 ** 24 - 1))
    elif case == "lateness_spread":
        # the widest spread sb_set_due takes for the maximum lateness: the tails q = D - d are exact integers up to
        # 2^24 - 1, and e + q rounds (e is a multiple of 1/8)
        d = rng.integers(0, 2 ** 24, J).astype(np.float32)
        d[0], d[-1] = 0.0, 2.0 ** 24 - 1
    elif case == "late_neighbours":
        # per job candidate 0's fp32 completion e (on time), or its fp32 neighbour below (late) or above (on time)
        _, st, _ = c_ref(T, opt[:1], prio[:1], None, ints, 1, "makespan", None, None, want_plan=True)
        rt = T[np.arange(J), opt[0] >> 3, opt[0] & 7]
        e = (st[0] + rt).astype(np.float32)
        assert (e.astype(np.float64) != st[0].astype(np.float64) + rt).any()        # some completions rounded
        d = np.stack([e, np.nextafter(e, np.float32(-np.inf)), np.nextafter(e, np.float32(np.inf))])
        d = d[rng.integers(0, 3, J), np.arange(J)]
        if fold.startswith("weighted"):
            w = WEIGHTS[rng.integers(0, 5, J)].astype(np.float32)
    elif case == "stretch_weights":
        # solve(objective="max_stretch")'s weighted maximum tardiness: w = fp32(1 / p*), d = max(r, +0)
        from saturn_b200.solver import _stretch_form
        r = release_dates("ready", T, opt, prio, ints, 1, seed)
        _, w, d = _stretch_form(T, r)
    return r, w, d


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FP32_EDGES))
@pytest.mark.parametrize("J", [33, 97])
def test_fp32_only_edges(engine, case, J):
    """Inputs where fp32 rounds, against the fp32 oracle only, every route, integer and real starts: runtimes in
    [2^22, 2^23] (times cross 2^23, where the ulp is 1), release dates of 2^24 - 1, and selected 1e8 / +inf cells
    (+inf scores; the key is still the arg-min) under the makespan and the weighted tardiness; a due-date spread of
    2^24 - 1 under the maximum lateness; late-count due dates at the fp32 neighbours of rounded completions; the
    maximum stretch's weights fp32(1 / p*) with its due dates max(r, 0)."""
    seed = J + len(case)
    fam, folds = FP32_EDGES[case]
    T = rt_table(fam, J, 2, seed)
    for fold in folds:
        for ints in (True, False):
            engine.set_table(T)
            opt, prio = candidates(J, 200, 2, seed + 1)
            r, w, d = _fp32_edge_per_job(case, fold, T, opt, prio, ints, seed)
            _set_per_job(engine, r, w, d)
            ref, cst, cm = c_ref(T, opt, prio, r, ints, 1, fold, w, d, want_plan=True)
            if case == "sentinel":
                assert np.isinf(ref).any() and np.isfinite(ref).any() and (ref >= 1e8).any()
            label = (J, 1, fold, r is not None)
            _, o_t, p_t = _run_routes(engine, opt, prio, ref, ints, fold, r is not None, 1, label)
            _check_plan(engine, o_t, p_t, opt, prio, ints, fold, 1, ref, cst, cm, label)


# --------------------------------------------------------------------------- GPU: the table refusal
@pytest.mark.gpu
def test_set_table_refuses_negative_and_nan_cells(engine):
    """sb_set_table returns SB_ERR_ARG for a negative or NaN cell, with T in host and in device memory, and leaves the
    handle without a table (SB_ERR_STATE); -0.0, +inf and sentinel cells are accepted."""
    import torch
    J, S, G = 40, 2, 8
    T = rt_table("small", J, S, 1)
    gc = np.arange(1, G + 1, dtype=np.uint8)
    engine.set_table(T)
    opt, prio = _dev(engine, *candidates(J, 4, S, 2))
    out = torch.empty(4, dtype=torch.float32, device=engine.device)

    def raw_set(Tx):
        if isinstance(Tx, torch.Tensor):
            ptr = Tx.data_ptr()
        else:
            ptr = Tx.ctypes.data
        return engine._lib.sb_set_table(engine._h, C.c_void_p(ptr), C.c_void_p(gc.ctypes.data), J, S, G, 1)

    def raw_eval():
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 4,
                                   opt.stride(0), 1, C.c_void_p(out.data_ptr()), None, 0)

    for bad in (-1.0, -1e-30, np.nan):
        for on_device in (False, True):
            Tb = T.copy()
            Tb[J - 1, 1, 5] = bad
            Tx = torch.from_numpy(Tb).to(engine.device) if on_device else Tb
            assert raw_set(T) == 0 and raw_eval() == 0
            assert raw_set(Tx) == -1, (bad, on_device)
            assert b"negative or NaN" in engine._lib.sb_last_error()
            assert raw_eval() == -3, (bad, on_device)          # no table
    for ok in (-0.0, np.inf, 1e8):
        for on_device in (False, True):
            Tb = T.copy()
            Tb[0, 0, 0] = ok
            Tx = torch.from_numpy(Tb).to(engine.device) if on_device else Tb
            assert raw_set(Tx) == 0 and raw_eval() == 0, (ok, on_device)
    engine.set_table(T)


# --------------------------------------------------------------------------- GPU: searches on tie-heavy tables
SEARCHES = [("fused_tile", 256, 1), ("position_major", 1024, 1), ("six_nodes", 96, 6), ("eight_nodes", 200, 8),
            ("J4096", 4096, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,J,nodes", SEARCHES)
@pytest.mark.parametrize("fold", ["makespan", "weighted_tardiness", "late_tasks", "weighted_max_tardiness"])
def test_search_on_tie_heavy_tables(engine, fold, name, J, nodes):
    """Short searches with release dates under the incremental-score verifier: no mismatch, a valid population, and a
    best plan whose exact score equals the reported one.  J = 4096 may be refused as unsupported, nothing else."""
    from saturn_b200 import _lib
    from saturn_b200._lib import SaturnB200Error
    seed = J + nodes
    T = rt_table("small" if J > 300 else "dyadic", J, 1, seed)
    engine.set_table(T, nodes=nodes)
    tmin = engine.reduced_table()[0][:, None, :]
    assert np.array_equal(tmin, T)
    opt, prio = candidates(J, 1, nodes, seed + 1)
    r = release_dates("ready", T, opt, prio, True, nodes, seed + 2)
    w, d = per_job(fold, T, opt, prio, True, nodes, r, seed + 3)
    _set_per_job(engine, r, w, d)
    try:
        wave = engine.search_wave(reduced=True)
        res = engine.search_run(wave, 24, seed=3, reduced=True, sync_every=8, objective=fold,
                                _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL)
    except SaturnB200Error as e:
        assert J == 4096 and "error -4:" in str(e), str(e)
        return
    assert engine.search_verify_count() == 0
    assert engine.search_validate() == 0
    assert sorted(res["prio"].tolist()) == list(range(J))
    sc = X.schedule(T, res["opt"], res["prio"], r, True, nodes, fold, w, d)[0]
    assert float(sc) == res["makespan"], (float(sc), res["makespan"])


# --------------------------------------------------------------------------- GPU: coverage accounting
@pytest.mark.gpu
def test_zz_every_kernel_path_was_exercised():
    """Runs after the sweep: paths 0-5 and 7-9 each scored something, and path 6 under the makespan; under each fold
    of the other oracles, paths 0, 3, 4 or 9, 5, 7 and 8.  Skipped when only part of the sweep ran (a -k selection
    or an earlier failure)."""
    want = {("sweep", J) for J in SWEEP_J} | {(f, J, n) for f in FOLDS for J in OBJ_J for n in (1, 6, 8)}
    if want - SWEEP_DONE:
        pytest.skip("the sweep did not run completely")
    seen = {rec[4] for rec in COVERAGE if rec[4] is not None}
    for p in (0, 1, 2, 3, 4, 5, 7, 8, 9):
        assert p in seen, ("path never ran", p, sorted(seen))
    assert 6 in {rec[4] for rec in COVERAGE if rec[2] == "makespan"}
    for fold in NEW_FOLDS:
        paths = {rec[4] for rec in COVERAGE if rec[2] == fold and rec[4] is not None}
        print("paths under %s:" % fold, sorted(paths))
        assert {0, 3, 5, 7, 8} <= paths and paths & {4, 9}, (fold, sorted(paths))
    by = {}
    for J, nodes, fold, rel, path in COVERAGE:
        if J in (6145, 16384, 65535) or nodes == 8:
            by.setdefault((J, nodes), set()).add(path)
    print("paths at J > 6144 and at 8 nodes:", {k: sorted(v, key=str) for k, v in sorted(by.items())})
