"""CPU ORACLE (test infrastructure — NOT product code): the (weighted) SQUARED TARDINESS of list schedules.

    score = sum_j w_j max(0, C_j - d_j)^2,  C_j = start_j + rt_j

In fp32 it is a LEFT FOLD IN SCHEDULE ORDER from +0 (SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE | SB_FLAG_SQUARED):

    e = start + rt,  l = e - d,  t = max(l, +0),  u = t * t,  x = w * u,  acc = acc + x
                                                                    (each rounded in `dtype` on its own)

with d the due date in `dtype` (round to nearest) and w the weight (unit weights with weights=None).  t is the
tardiness fold's term before the weight, bit for bit; w = 1 gives exactly the unweighted fold (1 * u = u), due dates at
or past every completion give +0.  A job with no runtime (rt = +inf) gives a +inf term, so an infeasible candidate
scores +inf with no special case.  With d_t = max(r_t, 0) it is the squared flow time (solve(objective="squared_flow")).

The schedule, and so every start, is the one of `oracle/ref_release.py` (release dates optional: None means none);
the objective changes only the fold.

Here:
  * `fold` — the sum fold of candidates from their starts, in numpy;
  * `evaluate` — schedule + fold: in Python (`use_c=False`: ref_release's list_schedule_batch on one node,
    list_schedule per candidate on several, then `fold`) or in C (`use_c=True`: `c_evaluate`);
  * `c_evaluate` — the schedule and the fold in plain C (`oracle/ref_squared_tardiness.c`, a library of its own);
  * `exact` — the same score in exact arithmetic from the starts of `oracle/ref_exact.py`, every intermediate asserted
    exact in fp32;
  * `brute_force` — the exhaustive list-schedule optimum (J <= ~6), scored by the C port;
  * `milp_solve` — ref_release's MILP (the release / completion model) plus C_t >= sta[g][t] + rt, the tardiness rows
    t_t >= C_t - d_t, t_t >= 0, and the tangent cuts z_t >= 2 a t_t - a^2 of t^2 at every integer a in [0, H_t],
    minimising sum_t w_t z_t.  The objective does not decrease when a completion grows, so list schedules still
    contain an optimum (DESIGN.md §3.1).
"""
from __future__ import annotations

import ctypes
import itertools
import math
import os
import subprocess
import time
from fractions import Fraction
from typing import Sequence

import numpy as np

from . import ref_exact as X
from . import ref_release as RR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_squared_tardiness.so")
_lib = None


def _w(weights, J, dtype):
    return np.ones(J, dtype=dtype) if weights is None else np.asarray(weights, dtype=np.float64).astype(dtype)


def _d(due, dtype):
    return np.asarray(due, dtype=np.float64).astype(dtype)


def _rts(tab, opt, nodes):
    tab = np.asarray(tab)
    opt = np.asarray(opt).astype(np.int64)
    j = np.arange(opt.shape[1])[None, :]
    return tab[j, 0 if nodes > 1 else opt >> 3, opt & 7]


def fold(tab, opt, prio, start, due, dtype=np.float32, nodes=1, weights=None):
    """(Weighted) squared tardiness score[B] of the candidates opt[B][J] / prio[B][J] whose job-indexed starts are
    start[B][J]: the left fold in schedule order of w * (t * t), t = max(e - d, +0); +inf where a completion is
    +inf."""
    opt = np.asarray(opt)
    B, J = opt.shape
    w, d = _w(weights, J, dtype), _d(due, dtype)
    rt = _rts(np.asarray(tab, dtype=dtype), opt, nodes).astype(dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        e = (np.asarray(start, dtype=dtype) + rt).astype(dtype)
        t = np.maximum((e - d[None, :]).astype(dtype), dtype(0.0))
        x = (w[None, :] * (t * t).astype(dtype)).astype(dtype)
    acc = np.zeros(B, dtype=dtype)
    rows = np.arange(B)
    prio = np.asarray(prio).astype(np.int64)
    with np.errstate(over="ignore"):
        for i in range(J):
            acc = (acc + x[rows, prio[:, i]]).astype(dtype)
    return acc


def evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nodes=1, use_c=True,
             want_plan=False, weights=None):
    """(Weighted) squared tardiness score[B] (+ start[B][J], mask[B][J] with want_plan); an infeasible candidate
    scores +inf."""
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    B, J = opt.shape
    if use_c:
        return c_evaluate(tab, opt, prio, due, release, integer_starts, dtype, want_plan=want_plan,
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
    score = np.where(np.isinf(mk), dtype(np.inf), fold(tab, opt, prio, start, due, dtype, nodes, weights)).astype(dtype)
    return (score, start, mask) if want_plan else score


def exact(tab, opt, prio, due, release=None, integer_starts=True, nodes=1, weights=None):
    """sum_j w_j max(0, C_j - d_j)^2 of one candidate in exact arithmetic: the starts of ref_exact.schedule (which
    asserts them exact in fp32), then the fold in Fractions, asserting that every e, e - d, t * t, w * (t * t) and
    partial sum is exact in fp32 as well.  Returns a Fraction (or +inf)."""
    J = len(prio)
    mk, start, _ = X.schedule(tab, opt, prio, release, integer_starts, nodes, "makespan")
    if mk == X.INF:
        return X.INF
    w = [Fraction(1)] * J if weights is None else [X._q(x) for x in weights]
    d = [X._q(x) for x in due]
    acc = Fraction(0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        rt = X._q(tab[j][0 if nodes > 1 else o >> 3][o & 7])
        X._check(w[j], "weight[%d]" % j)
        X._check(d[j], "due[%d]" % j)
        e = X._check(start[j] + rt, "completion[%d]" % j)
        t = max(X._check(e - d[j], "e - d of job %d" % j), Fraction(0))
        x = X._check(w[j] * X._check(t * t, "t t of job %d" % j), "w t t of job %d" % j)
        acc = X._check(acc + x, "partial sum at job %d" % j)
    return acc


def brute_force(tab, valid_opts: Sequence[Sequence[int]], due, release=None, integer_starts=True,
                dtype=np.float64, nodes=1, weights=None):
    """Exhaustive minimum of the squared tardiness over every (option vector, permutation) candidate, the first
    minimum in the enumeration order of ref_release.brute_force.  Returns (score, opt, prio)."""
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    score = evaluate(tab, opt, prio, due, release, integer_starts, dtype, nodes, weights=weights)
    i = int(np.argmin(score))
    return float(score[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_squared_tardiness.c")
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
        for name in ("ref_squared_tardiness_f32", "ref_squared_tardiness_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False,
               threads=0, nodes=1, weights=None):
    """(Weighted) squared tardiness of B candidates in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, due[J],
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
    w = np.ascontiguousarray(_w(weights, J, dtype))
    r = np.ascontiguousarray(RR.release_as(np.zeros(J) if release is None else release, J, dtype, integer_starts))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_squared_tardiness_f32 if dtype == np.float32 else _load().ref_squared_tardiness_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), w.ctypes.data, d.ctypes.data, r.ctypes.data, tot.ctypes.data,
            start.ctypes.data if want_plan else None, mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_squared_tardiness rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, due, release=None, weights=None, time_limit=240.0, mip_rel_gap=0.0):
    """min sum_t w_t z_t subject to ref_release's model, C_t >= sta[g][t] + rt_ts - M (1 - bss[t][s]) for every GPU g
    and option s, t_t >= C_t - d_t, t_t >= 0, and z_t >= 2 a t_t - a^2 for every integer a in [0, H_t], H_t =
    max(0, ceil(M - d_t)) with M the model's horizon.  The cuts are the tangents of t^2 at the integers, so z_t is
    t_t^2 wherever t_t is an integer and below it (by at most 1/4) in between.  On instances with integer runtimes and
    due dates every integer-start plan has integer tardiness, so there the cuts make z_t = t_t^2 exactly and the
    model's optimum is the squared tardiness optimum.  HiGHS via scipy.  Returns dict(status, proven_optimal,
    objective_value, score, start[J], mask[J], opt_idx[J], wall_s, n_vars, n_cons); `score` is the decoded plan's
    (weighted) squared tardiness in float64."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from .ref_milp import G
    J = len(gpu_time_tuples)
    r = [0.0] * J if release is None else [float(x) for x in np.asarray(release, dtype=np.float64)]
    d = np.asarray(due, dtype=np.float64)
    w = np.ones(J) if weights is None else np.asarray(weights, dtype=np.float64)
    Rw, integrality, lb, ub, idx = RR._build(gpu_time_tuples, r)
    M, nv = idx["M"], idx["nv"]
    comp = list(range(nv, nv + J))
    tard = list(range(nv + J, nv + 2 * J))
    z = list(range(nv + 2 * J, nv + 3 * J))
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        Rw.add([tard[t], comp[t]], [1.0, -1.0], -d[t], np.inf)
        for a in range(int(max(0, math.ceil(M - d[t]))) + 1):
            Rw.add([z[t], tard[t]], [1.0, -2.0 * a], -float(a * a), np.inf)
    nvt = nv + 3 * J
    integrality = np.concatenate([integrality, np.zeros(3 * J)])
    lb = np.concatenate([lb, np.zeros(3 * J)])
    ub = np.concatenate([ub, np.full(3 * J, np.inf)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nvt))
    c = np.zeros(nvt)
    c[z] = w
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
               score=plan_squared_tardiness(gpu_time_tuples, start, opt_idx, due, weights))
    return out


def plan_squared_tardiness(gpu_time_tuples, start, opt_idx, due, weights=None):
    """A plan's sum_t w_t max(0, start_t + rt_t - d_t)^2 in float64."""
    J = len(start)
    w = [1.0] * J if weights is None else [float(x) for x in weights]
    return sum(w[t] * max(0.0, start[t] + gpu_time_tuples[t][opt_idx[t]][1] - float(due[t])) ** 2 for t in range(J))
