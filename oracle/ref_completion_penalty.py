"""CPU ORACLE (test infrastructure — NOT product code): the COMPLETION PENALTY of list schedules.

    score = sum_j (w_j C_j + [C_j > d_j] p_j),  C_j = start_j + rt_j

In fp32 it is a LEFT FOLD IN SCHEDULE ORDER from +0 (SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE | SB_FLAG_COMPLETION_PENALTY):

    e = start + rt,  t = w * e,  t = e > d ? t + p : t,  acc = acc + t      (each rounded in `dtype` on its own)

with d the due date and p the penalty in `dtype` (round to nearest, -0 as +0) and w the weight (unit weights with
weights=None).  p = 0 gives the (weighted) completion fold of `oracle/ref_weighted.py` bit for bit (+0 added to a
value >= +0 is exact); a job that completes exactly at its due date is on time.  A job with no runtime (rt = +inf)
gives a +inf term, so an infeasible candidate scores +inf with no special case.

One due date H for every job and every p above any sum_j w_j C_j make the score "min sum_j w_j C_j subject to
makespan <= H": `front_brute_force` enumerates that constrained optimum, and the whole (makespan, sum w C) front.

The schedule, and so every start, is the one of `oracle/ref_release.py` (release dates optional: None means none);
the objective changes only the fold.

Here:
  * `fold` — the sum fold of candidates from their starts, in numpy;
  * `evaluate` — schedule + fold: in Python (`use_c=False`: ref_release's list_schedule_batch on one node,
    list_schedule per candidate on several, then `fold`) or in C (`use_c=True`: `c_evaluate`);
  * `c_evaluate` — the schedule and the fold in plain C (`oracle/ref_completion_penalty.c`, a library of its own);
  * `exact` — the same score in exact arithmetic from the starts of `oracle/ref_exact.py`, every intermediate asserted
    exact in fp32;
  * `brute_force` — the exhaustive list-schedule optimum (J <= ~6), scored by the C port;
  * `front_brute_force` — per makespan cap the exhaustive minimum of sum_j w_j C_j over the candidates whose fp32
    makespan is <= the cap, and the exhaustive non-dominated (fp32 makespan, sum_j w_j C_j) set;
  * `milp_solve` — ref_release's MILP (the release / completion model) plus C_t >= sta[g][t] + rt and a binary U_t
    with C_t - d_t <= M U_t, minimising sum_t w_t C_t + p_t U_t.  The objective does not decrease when a completion
    grows, so list schedules still contain an optimum (DESIGN.md §3.1).
"""
from __future__ import annotations

import ctypes
import itertools
import os
import subprocess
import time
from fractions import Fraction
from typing import Sequence

import numpy as np

from . import ref_exact as X
from . import ref_release as RR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_completion_penalty.so")
_lib = None


def _w(weights, J, dtype):
    return np.ones(J, dtype=dtype) if weights is None else np.asarray(weights, dtype=np.float64).astype(dtype)


def _d(due, dtype):
    return np.asarray(due, dtype=np.float64).astype(dtype)


def _p(penalty, dtype):
    """The penalties in `dtype`, -0 as +0 (as sb_set_penalty stores them)."""
    return (np.asarray(penalty, dtype=np.float64).astype(dtype) + dtype(0.0)).astype(dtype)


def _rts(tab, opt, nodes):
    tab = np.asarray(tab)
    opt = np.asarray(opt).astype(np.int64)
    j = np.arange(opt.shape[1])[None, :]
    return tab[j, 0 if nodes > 1 else opt >> 3, opt & 7]


def fold(tab, opt, prio, start, due, penalty, dtype=np.float32, nodes=1, weights=None):
    """Completion penalty score[B] of the candidates opt[B][J] / prio[B][J] whose job-indexed starts are start[B][J]:
    the left fold in schedule order of (e > d ? w * e + p : w * e); +inf where a completion is +inf."""
    opt = np.asarray(opt)
    B, J = opt.shape
    w, d, p = _w(weights, J, dtype), _d(due, dtype), _p(penalty, dtype)
    rt = _rts(np.asarray(tab, dtype=dtype), opt, nodes).astype(dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        e = (np.asarray(start, dtype=dtype) + rt).astype(dtype)
        t = (w[None, :] * e).astype(dtype)
        term = np.where(e > d[None, :], (t + p[None, :]).astype(dtype), t).astype(dtype)
    acc = np.zeros(B, dtype=dtype)
    rows = np.arange(B)
    prio = np.asarray(prio).astype(np.int64)
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(J):
            acc = (acc + term[rows, prio[:, i]]).astype(dtype)
    return acc


def evaluate(tab, opt, prio, due, penalty, release=None, integer_starts=True, dtype=np.float32, nodes=1, use_c=True,
             want_plan=False, weights=None):
    """Completion penalty score[B] (+ start[B][J], mask[B][J] with want_plan); an infeasible candidate scores +inf."""
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    B, J = opt.shape
    if use_c:
        return c_evaluate(tab, opt, prio, due, penalty, release, integer_starts, dtype, want_plan=want_plan,
                          threads=os.cpu_count() or 1, nodes=nodes, weights=weights)
    rel = np.zeros(J) if release is None else release
    if nodes == 1:
        mk, start, mask = RR.list_schedule_batch(tab, opt, prio, rel, integer_starts, dtype, want_plan=True)
    else:
        mk = np.empty(B, dtype=dtype)
        start = np.zeros((B, J), dtype=dtype)
        mask = np.zeros((B, J), dtype=np.uint32)
        for b in range(B):
            s, st, m, _ = RR.list_schedule(tab, opt[b], prio[b], rel, integer_starts, dtype, nodes=nodes)
            mk[b], start[b], mask[b] = s, st, m
    score = fold(tab, opt, prio, start, due, penalty, dtype, nodes, weights)
    score = np.where(np.isinf(mk), dtype(np.inf), score).astype(dtype)
    return (score, start, mask) if want_plan else score


def exact(tab, opt, prio, due, penalty, release=None, integer_starts=True, nodes=1, weights=None):
    """sum_j (w_j C_j + [C_j > d_j] p_j) of one candidate in exact arithmetic: the starts of ref_exact.schedule (which
    asserts them exact in fp32), then the fold in Fractions, asserting that every e, w * e, w * e + p and partial sum
    is exact in fp32 as well.  Returns a Fraction (or +inf)."""
    J = len(prio)
    mk, start, _ = X.schedule(tab, opt, prio, release, integer_starts, nodes, "makespan")
    if mk == X.INF:
        return X.INF
    w = [Fraction(1)] * J if weights is None else [X._q(v) for v in weights]
    d = [X._q(v) for v in due]
    p = [X._q(v) for v in penalty]
    acc = Fraction(0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        rt = X._q(tab[j][0 if nodes > 1 else o >> 3][o & 7])
        X._check(w[j], "weight[%d]" % j)
        X._check(d[j], "due[%d]" % j)
        X._check(p[j], "penalty[%d]" % j)
        e = X._check(start[j] + rt, "completion[%d]" % j)
        t = X._check(w[j] * e, "w e of job %d" % j)
        if e > d[j]:
            t = X._check(t + p[j], "w e + p of job %d" % j)
        acc = X._check(acc + t, "partial sum at job %d" % j)
    return acc


def _candidates(valid_opts, nodes):
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    return np.repeat(opts, len(perms), axis=0), np.tile(perms, (len(opts), 1))


def brute_force(tab, valid_opts: Sequence[Sequence[int]], due, penalty, release=None, integer_starts=True,
                dtype=np.float64, nodes=1, weights=None):
    """Exhaustive minimum of the completion penalty over every (option vector, permutation) candidate, the first
    minimum in the enumeration order of ref_release.brute_force.  Returns (score, opt, prio)."""
    opt, prio = _candidates(valid_opts, nodes)
    score = evaluate(tab, opt, prio, due, penalty, release, integer_starts, dtype, nodes, weights=weights)
    i = int(np.argmin(score))
    return float(score[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


def front_brute_force(tab, valid_opts: Sequence[Sequence[int]], caps, release=None, integer_starts=True, nodes=1,
                      weights=None):
    """The exhaustive trade-off between the makespan and sum_j w_j C_j (unit weights with weights=None) over every
    (option vector, permutation) candidate.  The makespan is the fp32 schedule's, max_j fp32(start_j + rt_j), the value
    the device compares a cap with; sum_j w_j C_j is the fp64 fold.  Returns dict(at_cap=[per cap: the minimum sum
    over the candidates with makespan <= cap, None where there is none], front=[[makespan, sum], ...] the
    non-dominated pairs, makespan ascending and sum strictly descending)."""
    opt, prio = _candidates(valid_opts, nodes)
    J = opt.shape[1]
    zero, never = np.zeros(J), np.full(J, np.inf)
    _s32, start32, _m = c_evaluate(tab, opt, prio, never, zero, release, integer_starts, np.float32, want_plan=True,
                                   threads=os.cpu_count() or 1, nodes=nodes, weights=weights)
    wc = c_evaluate(tab, opt, prio, never, zero, release, integer_starts, np.float64, threads=os.cpu_count() or 1,
                    nodes=nodes, weights=weights)
    rt32 = _rts(np.asarray(tab, dtype=np.float32), opt, nodes).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        mk = (start32 + rt32).astype(np.float32).max(axis=1).astype(np.float64)
    ok = np.isfinite(mk) & np.isfinite(wc)
    mk, wc = mk[ok], wc[ok]
    at_cap = []
    for c in caps:
        sel = mk <= float(c)
        at_cap.append(float(wc[sel].min()) if sel.any() else None)
    front = []
    for i in np.lexsort((wc, mk)):
        if not front or wc[i] < front[-1][1]:
            front.append([float(mk[i]), float(wc[i])])
    return {"at_cap": at_cap, "front": front}


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_completion_penalty.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        tmp = _SO + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-ffp-contract=off", src, "-o", tmp,
                               "-lm"])
        os.replace(tmp, _SO)
    return _SO


def _load():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        for name in ("ref_completion_penalty_f32", "ref_completion_penalty_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, due, penalty, release=None, integer_starts=True, dtype=np.float32, nslot=8,
               want_plan=False, threads=0, nodes=1, weights=None):
    """Completion penalty of B candidates in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, due[J], penalty[J],
    release[J] or None, weights[J] or None -> score[B] (+ start[B][J], mask[B][J] with want_plan)."""
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    assert prio.dtype in (np.uint8, np.uint16)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    d = np.ascontiguousarray(_d(due, dtype))
    p = np.ascontiguousarray(_p(penalty, dtype))
    w = np.ascontiguousarray(_w(weights, J, dtype))
    r = np.ascontiguousarray(RR.release_as(np.zeros(J) if release is None else release, J, dtype, integer_starts))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_completion_penalty_f32 if dtype == np.float32 else _load().ref_completion_penalty_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), w.ctypes.data, d.ctypes.data, r.ctypes.data, p.ctypes.data, tot.ctypes.data,
            start.ctypes.data if want_plan else None, mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_completion_penalty rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, due, penalty, release=None, weights=None, time_limit=240.0, mip_rel_gap=0.0):
    """min sum_t w_t C_t + p_t U_t subject to ref_release's model, C_t >= sta[g][t] + rt_ts - M (1 - bss[t][s]) for
    every GPU g and option s, and C_t - d_t <= M U_t with U_t binary (M the model's horizon).  Integer runtimes and
    due dates give integer completions, so there U_t = 0 exactly when C_t <= d_t.  HiGHS via scipy.  Returns
    dict(status, proven_optimal, objective_value, score, start[J], mask[J], opt_idx[J], wall_s, n_vars, n_cons);
    `score` is the decoded plan's completion penalty in float64."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from .ref_milp import G
    J = len(gpu_time_tuples)
    r = [0.0] * J if release is None else [float(x) for x in np.asarray(release, dtype=np.float64)]
    d = np.asarray(due, dtype=np.float64)
    p = np.asarray(penalty, dtype=np.float64)
    w = np.ones(J) if weights is None else np.asarray(weights, dtype=np.float64)
    Rw, integrality, lb, ub, idx = RR._build(gpu_time_tuples, r)
    M, nv = idx["M"], idx["nv"]
    comp = list(range(nv, nv + J))
    late = list(range(nv + J, nv + 2 * J))
    big = M + max(0.0, -float(d.min(initial=0.0)))  # C_t - d_t <= M - d_t <= big
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        Rw.add([comp[t], late[t]], [1.0, -big], -np.inf, d[t])
    nvt = nv + 2 * J
    integrality = np.concatenate([integrality, np.zeros(J), np.ones(J)])
    lb = np.concatenate([lb, np.zeros(2 * J)])
    ub = np.concatenate([ub, np.full(J, np.inf), np.ones(J)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nvt))
    c = np.zeros(nvt)
    c[comp] = w
    c[late] = p
    options = {"time_limit": float(time_limit), "disp": False, "mip_rel_gap": float(mip_rel_gap)}
    t0 = time.perf_counter()
    res = milp(c, constraints=LinearConstraint(A, Rw.lo, Rw.hi), integrality=integrality, bounds=Bounds(lb, ub),
               options=options)
    out = {"status": int(res.status), "proven_optimal": res.status == 0, "wall_s": time.perf_counter() - t0,
           "n_vars": nvt, "n_cons": Rw.n, "objective_value": None, "score": None, "start": None, "mask": None,
           "opt_idx": None}
    if res.x is None:
        return out
    x = res.x
    start, mask, opt_idx = [], [], []
    for t in range(J):
        o = int(np.argmax([x[v] for v in idx["bss"][t]]))
        m, first = 0, None
        for g in range(G):
            if round(x[idx["tga"][t][g]]) == 1:
                m |= 1 << g
                first = g if first is None else first
        start.append(float(round(x[idx["sta"][first][t]])) if first is not None else 0.0)
        mask.append(m)
        opt_idx.append(o)
    out.update(objective_value=float(res.fun), start=start, mask=mask, opt_idx=opt_idx,
               score=plan_completion_penalty(gpu_time_tuples, start, opt_idx, due, penalty, weights))
    return out


def plan_completion_penalty(gpu_time_tuples, start, opt_idx, due, penalty, weights=None):
    """A plan's sum_t (w_t C_t + [C_t > d_t] p_t) in float64."""
    J = len(start)
    w = [1.0] * J if weights is None else [float(x) for x in weights]
    total = 0.0
    for t in range(J):
        c = start[t] + gpu_time_tuples[t][opt_idx[t]][1]
        total += w[t] * c + (float(penalty[t]) if c > float(due[t]) else 0.0)
    return total
