"""CPU ORACLE (test infrastructure — NOT product code): the MAXIMUM LATENESS of list schedules.

L_max = max_j (C_j - d_j) with C_j = start_j + rt_j may be negative.  The library scores the equivalent tail makespan
(SB_FLAG_MAX_LATENESS), which is never negative:

    D   = max_t d_t
    q_j = D - d_j                                   (>= +0, formed once in `dtype`)
    e   = start + rt,  x = e + q                    (each rounded in `dtype`)
    score = max_j x, a max fold from +0             = L_max + D

The schedule, and so every start, is the one of `oracle/ref_release.py` (release dates optional: None means none);
the objective changes only the fold.  Integer due dates shifted by an integer give the same q and the same scores.

Here:
  * `tails` — q and D as the device forms them;
  * `fold` — the tail fold of candidates from their starts, in numpy;
  * `evaluate` — schedule + fold: in Python (`use_c=False`: ref_release's list_schedule_batch on one node,
    list_schedule per candidate on several, then `fold`) or in C (`use_c=True`: `c_evaluate`);
  * `c_evaluate` — the schedule and the tail fold in plain C (`oracle/ref_max_lateness.c`, a library of its own);
  * `exact` — the same score in exact arithmetic from the starts of `oracle/ref_exact.py`;
  * `brute_force` — the exhaustive list-schedule optimum (J <= ~6), scored by the C port;
  * `milp_solve` — ref_release's MILP (the release / completion model) plus C_t >= sta[g][t] + rt and
    L >= C_t - d_t with L free, minimising L.
"""
from __future__ import annotations

import ctypes
import itertools
import os
import subprocess
import time
from typing import Sequence

import numpy as np

from . import ref_exact as X
from . import ref_release as RR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_max_lateness.so")
_lib = None


def tails(due, dtype=np.float32):
    """(q[J], D): the delivery tails D - d_j in `dtype` (D - d_j = +0 where d_j = D) and D = max_j d_j."""
    d = np.asarray(due, dtype=np.float64).astype(dtype)
    D = d.max()
    return (D - d).astype(dtype), float(D)


def _rts(tab, opt, nodes):
    tab = np.asarray(tab)
    opt = np.asarray(opt).astype(np.int64)
    j = np.arange(opt.shape[1])[None, :]
    return tab[j, 0 if nodes > 1 else opt >> 3, opt & 7]


def fold(tab, opt, start, due, dtype=np.float32, nodes=1):
    """Tail makespan score[B] of the candidates opt[B][J] whose job-indexed starts are start[B][J]."""
    q, _ = tails(due, dtype)
    rt = _rts(np.asarray(tab, dtype=dtype), opt, nodes).astype(dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        e = (np.asarray(start, dtype=dtype) + rt).astype(dtype)
        x = (e + q[None, :]).astype(dtype)
    return np.maximum(x.max(axis=1), dtype(0.0)).astype(dtype)


def evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nodes=1, use_c=True,
             want_plan=False):
    """Tail makespan score[B] (+ start[B][J], mask[B][J] with want_plan); an infeasible candidate scores +inf."""
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    B, J = opt.shape
    rel = np.zeros(J) if release is None else release
    if use_c:
        return c_evaluate(tab, opt, prio, due, release, integer_starts, dtype, want_plan=want_plan,
                          threads=os.cpu_count() or 1, nodes=nodes)
    if nodes == 1:
        mk, start, mask = RR.list_schedule_batch(tab, opt, prio, rel, integer_starts, dtype, want_plan=True)
    else:
        mk = np.empty(B, dtype=dtype)
        start = np.zeros((B, J), dtype=dtype)
        mask = np.zeros((B, J), dtype=np.uint32)
        for b in range(B):
            s, st, m, _ = RR.list_schedule(tab, opt[b], prio[b], rel, integer_starts, dtype, nodes=nodes)
            mk[b], start[b], mask[b] = s, st, m
    score = np.where(np.isinf(mk), dtype(np.inf), fold(tab, opt, start, due, dtype, nodes)).astype(dtype)
    return (score, start, mask) if want_plan else score


def exact(tab, opt, prio, due, release=None, integer_starts=True, nodes=1):
    """max_j (C_j + (D - d_j)) of one candidate in exact arithmetic: ref_exact.schedule's max_lateness fold, which
    asserts that every input and intermediate (the schedule, the tails and every C + q) is exact in fp32.  Returns a
    Fraction (or +inf)."""
    return X.schedule(tab, opt, prio, release, integer_starts, nodes, "max_lateness", due=due)[0]


def brute_force(tab, valid_opts: Sequence[Sequence[int]], due, release=None, integer_starts=True,
                dtype=np.float64, nodes=1):
    """Exhaustive minimum of the tail makespan over every (option vector, permutation) candidate, the first minimum
    in the enumeration order of ref_release.brute_force.  Returns (L_max, opt, prio): the score minus D."""
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    score = evaluate(tab, opt, prio, due, release, integer_starts, dtype, nodes)
    i = int(np.argmin(score))
    return float(score[i]) - tails(due, dtype)[1], tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_max_lateness.c")
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
        for name in ("ref_max_lateness_f32", "ref_max_lateness_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False,
               threads=0, nodes=1):
    """Tail makespans of B candidates in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, due[J], release[J] or
    None -> score[B] (+ start[B][J], mask[B][J] with want_plan)."""
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    assert prio.dtype in (np.uint8, np.uint16)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    q = np.ascontiguousarray(tails(due, dtype)[0])
    r = np.ascontiguousarray(RR.release_as(np.zeros(J) if release is None else release, J, dtype, integer_starts))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_max_lateness_f32 if dtype == np.float32 else _load().ref_max_lateness_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), q.ctypes.data, r.ctypes.data, tot.ctypes.data,
            start.ctypes.data if want_plan else None, mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_max_lateness rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, due, release=None, time_limit=240.0, mip_rel_gap=0.0):
    """min L subject to ref_release's model (ref_milp's model with the release rows and the big-M horizon raised by
    the latest release), C_t >= sta[g][t] + rt_ts - M (1 - bss[t][s]) for every GPU g and option s, and
    L >= C_t - d_t, L free.  HiGHS via scipy.  Returns dict(status, proven_optimal, objective_value, score, start[J],
    mask[J], opt_idx[J], wall_s, n_vars, n_cons); `score` is the decoded plan's L_max in float64."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from .ref_milp import G
    J = len(gpu_time_tuples)
    r = [0.0] * J if release is None else [float(x) for x in np.asarray(release, dtype=np.float64)]
    d = np.asarray(due, dtype=np.float64)
    Rw, integrality, lb, ub, idx = RR._build(gpu_time_tuples, r)
    M, nv = idx["M"], idx["nv"]
    comp = list(range(nv, nv + J))
    L = nv + J
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        Rw.add([L, comp[t]], [1.0, -1.0], -d[t], np.inf)
    nvt = nv + J + 1
    integrality = np.concatenate([integrality, np.zeros(J + 1)])
    lb = np.concatenate([lb, np.zeros(J), [-np.inf]])
    ub = np.concatenate([ub, np.full(J + 1, np.inf)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nvt))
    c = np.zeros(nvt)
    c[L] = 1.0
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
               score=plan_lmax(gpu_time_tuples, start, opt_idx, due))
    return out


def plan_lmax(gpu_time_tuples, start, opt_idx, due):
    """A plan's L_max = max_t (start_t + rt_t - d_t) in float64."""
    return max(start[t] + gpu_time_tuples[t][opt_idx[t]][1] - float(due[t]) for t in range(len(start)))
