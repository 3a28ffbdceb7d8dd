"""CPU ORACLE (test infrastructure — NOT product code): the (weighted) NUMBER OF LATE TASKS of list schedules.

    total = sum_j w_j [C_j > d_j],  C_j = start_j + rt_j

A task that completes exactly at its due date is on time, as its tardiness max(C - d, 0) is 0.  In fp32 the score is
a LEFT FOLD IN SCHEDULE ORDER from +0 (SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE | SB_FLAG_LATE_COUNT):

    e = start + rt                                  (rounded in `dtype`, as the tardiness fold forms it)
    acc = acc + (e > d ? w : +0)                    (one rounding per job)

with d the due date in `dtype` (round to nearest) and w the weight (unit weights with weights=None).  Unit weights,
and integer weights with sum w < 2^24, give an exact sum whatever the order.  Due dates at or past every completion
give +0, due dates below every completion give sum w, w = 2 gives exactly twice w = 1.  A candidate that gives a job
an option it does not have (rt = +inf) is infeasible and scores +inf, as under every other objective, although the
fold alone would add only that job's weight.

The schedule, and so every start, is the one of `oracle/ref_release.py` (release dates optional: None means none);
the objective changes only the fold.

Here:
  * `fold` — the count fold of candidates from their starts, in numpy;
  * `evaluate` — schedule + fold: in Python (`use_c=False`: ref_release's list_schedule_batch on one node,
    list_schedule per candidate on several, then `fold`) or in C (`use_c=True`: `c_evaluate`);
  * `c_evaluate` — the schedule and the count fold in plain C (`oracle/ref_late_tasks.c`, a library of its own);
  * `exact` — the same score in exact arithmetic from the starts of `oracle/ref_exact.py`;
  * `brute_force` — the exhaustive list-schedule optimum (J <= ~6), scored by the C port;
  * `moore_hodgson_seed` — the seed repair of the search (sb_search_seed_lpt, search.lpt_seeds), restated;
  * `milp_solve` — ref_release's MILP (the release / completion model) plus C_t >= sta[g][t] + rt and binary U_t with
    C_t - d_t <= M_U U_t, minimising sum_t w_t U_t.  The objective does not decrease when a completion grows, so list
    schedules still contain an optimum (DESIGN.md §3.1).
"""
from __future__ import annotations

import ctypes
import itertools
import math
import os
import subprocess
import time
from typing import Sequence

import numpy as np

from . import ref_exact as X
from . import ref_release as RR

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_late_tasks.so")
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
    """Late-count score[B] of the candidates opt[B][J] / prio[B][J] whose job-indexed starts are start[B][J]: the left
    fold in schedule order; +inf where a completion is +inf (a job without a runtime)."""
    opt = np.asarray(opt)
    B, J = opt.shape
    w, d = _w(weights, J, dtype), _d(due, dtype)
    rt = _rts(np.asarray(tab, dtype=dtype), opt, nodes).astype(dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        e = (np.asarray(start, dtype=dtype) + rt).astype(dtype)
    acc = np.zeros(B, dtype=dtype)
    rows = np.arange(B)
    prio = np.asarray(prio).astype(np.int64)
    for i in range(J):
        j = prio[:, i]
        acc = (acc + np.where(e[rows, j] > d[j], w[j], dtype(0.0))).astype(dtype)
    return np.where(np.isinf(e).any(axis=1), dtype(np.inf), acc).astype(dtype)


def evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nodes=1, use_c=True,
             want_plan=False, weights=None):
    """Late-count score[B] (+ start[B][J], mask[B][J] with want_plan); an infeasible candidate scores +inf."""
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
    """sum_j w_j [C_j > d_j] of one candidate in exact arithmetic: ref_exact.schedule's late_tasks fold
    (weighted_late_tasks with weights), which asserts that every input and intermediate is exact in fp32.  Returns a
    Fraction (or +inf)."""
    obj = "late_tasks" if weights is None else "weighted_late_tasks"
    return X.schedule(tab, opt, prio, release, integer_starts, nodes, obj, weights, due)[0]


def brute_force(tab, valid_opts: Sequence[Sequence[int]], due, release=None, integer_starts=True,
                dtype=np.float64, nodes=1, weights=None):
    """Exhaustive minimum of the late count over every (option vector, permutation) candidate, the first minimum in
    the enumeration order of ref_release.brute_force.  Returns (score, opt, prio)."""
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


def moore_hodgson_seed(order, k, rt, due, node=None, nodes=1, weights=None, release=None, integer_starts=True):
    """The search's seed repair, restated.  `order` is a seed's job order, job j runs on k[j] GPUs of node[j] for
    rt[j] (fp32 values; release[j] as the schedule uses it, ceiled under integer starts).  Simulated in float64: the
    on-time sequence is list-scheduled from scratch after every removal; at its first late job (C > d), the job with
    the largest k rt / w up to and including it (the latest on ties) moves to the late list.  Returns the on-time
    sequence followed by the late jobs in `order`'s order."""
    J = len(order)
    node = [0] * J if node is None else [int(x) for x in node]
    w = [1.0] * J if weights is None else [float(np.float32(x)) for x in weights]
    d = [float(np.float32(x)) for x in due]
    seq, late = [int(j) for j in order], []
    while True:
        ready = [[0.0] * 8 for _ in range(nodes)]
        first_late = None
        for q, j in enumerate(seq):
            f = sorted(ready[node[j]])
            s = f[k[j] - 1]
            if release is not None:
                s = max(s, float(release[j]))
            r = float(rt[j])
            f[:k[j]] = [s + (math.ceil(r) if integer_starts and math.isfinite(r) else r)] * k[j]
            ready[node[j]] = f
            if s + r > d[j]:
                first_late = q
                break
        if first_late is None:
            break
        ratios = [k[j] * float(rt[j]) / w[j] for j in seq[:first_late + 1]]
        best = max(ratios)
        out = max(q for q, x in enumerate(ratios) if x == best)
        late.append(seq.pop(out))
    pos = {int(j): q for q, j in enumerate(order)}
    return seq + sorted(late, key=pos.__getitem__)


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_late_tasks.c")
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
        for name in ("ref_late_tasks_f32", "ref_late_tasks_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, due, release=None, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False,
               threads=0, nodes=1, weights=None):
    """Late counts of B candidates in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, due[J], release[J] or None,
    weights[J] or None -> score[B] (+ start[B][J], mask[B][J] with want_plan)."""
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
    fn = _load().ref_late_tasks_f32 if dtype == np.float32 else _load().ref_late_tasks_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), w.ctypes.data, d.ctypes.data, r.ctypes.data, tot.ctypes.data,
            start.ctypes.data if want_plan else None, mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_late_tasks rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, due, release=None, weights=None, time_limit=240.0, mip_rel_gap=0.0):
    """min sum_t w_t U_t subject to ref_release's model, C_t >= sta[g][t] + rt_ts - M (1 - bss[t][s]) for every GPU g
    and option s, and C_t - d_t <= M_U U_t with U_t binary.  M bounds every start (ref_release's big-M horizon), so the
    smallest feasible C_t is at most M + max rt, and M_U = M + max rt - min(d, 0) + 1 never cuts off U_t = 1.  HiGHS
    via scipy.  Returns dict(status, proven_optimal, objective_value, score, start[J], mask[J], opt_idx[J], wall_s,
    n_vars, n_cons); `score` is the decoded plan's late count in float64."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from .ref_milp import G
    J = len(gpu_time_tuples)
    r = [0.0] * J if release is None else [float(x) for x in np.asarray(release, dtype=np.float64)]
    d = np.asarray(due, dtype=np.float64)
    w = np.ones(J) if weights is None else np.asarray(weights, dtype=np.float64)
    Rw, integrality, lb, ub, idx = RR._build(gpu_time_tuples, r)
    M, nv = idx["M"], idx["nv"]
    max_rt = max(rt for tup in gpu_time_tuples for _k, rt in tup if np.isfinite(rt))
    MU = M + max_rt - min(float(d.min()), 0.0) + 1.0
    comp = list(range(nv, nv + J))
    late = list(range(nv + J, nv + 2 * J))
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        Rw.add([comp[t], late[t]], [1.0, -MU], -np.inf, d[t])
    nvt = nv + 2 * J
    integrality = np.concatenate([integrality, np.zeros(J), np.ones(J)])
    lb = np.concatenate([lb, np.zeros(2 * J)])
    ub = np.concatenate([ub, np.full(J, np.inf), np.ones(J)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nvt))
    c = np.zeros(nvt)
    c[late] = w
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
               score=plan_late(gpu_time_tuples, start, opt_idx, due, weights))
    return out


def plan_late(gpu_time_tuples, start, opt_idx, due, weights=None):
    """A plan's sum_t w_t [start_t + rt_t > d_t] in float64."""
    J = len(start)
    w = [1.0] * J if weights is None else [float(x) for x in weights]
    return sum(w[t] for t in range(J) if start[t] + gpu_time_tuples[t][opt_idx[t]][1] > float(due[t]))
