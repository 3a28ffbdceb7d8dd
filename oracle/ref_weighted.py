"""CPU ORACLE (test infrastructure — NOT product code): the WEIGHTED sum of completion times.

The schedule of a candidate does not depend on the objective: `oracle/ref_eval.py` defines it (starts, slot masks)
and this module only scores it,

    total = sum_j w_j (start_j + rt_j)

In fp32 the sum is a LEFT FOLD IN SCHEDULE ORDER with TWO roundings per job, acc = acc + (w_j * (start_j + rt_j))
from +0: the product is rounded, then the sum, never one fused multiply-add (numpy cannot express a fused one, and
the kernels use __fmul_rn / __fadd_rn for SB_FLAG_WEIGHTED).  Weights are finite and > 0.  weights=None is the
unweighted fold of `oracle/ref_completion.py` (delegation, nothing restated); with w = 1 the two agree bit for bit,
with w = 2 the weighted sum is exactly twice the unweighted one.

Also here:
  * `c_evaluate` — the same fold in plain C (`oracle/ref_weighted.c`, a library of its own beside
    `ref_completion.c`) for batches of 1e5 candidates;
  * `milp_solve` — the completion MILP of `oracle/ref_completion.py` (the model of `oracle/ref_milp.py` plus one
    continuous C[t] >= 0 per task, C[t] >= sta[g][t] + rt[t][s] - M(1 - bss[t][s])) with the objective
    sum_t w_t C[t].  Non-negative weights keep the objective non-decreasing in every completion time, so list
    schedules still contain an optimum (DESIGN.md §3.1) and ref_milp's M still bounds the starts.
"""
from __future__ import annotations

import ctypes
import itertools
import os
import subprocess
import time
from typing import Sequence

import numpy as np

from . import ref_completion as RC
from . import ref_eval as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_weighted.so")
_lib = None


def weights_as(weights, J, dtype):
    """weights (length J, finite and > 0) in `dtype`; ValueError otherwise."""
    w = np.asarray(weights, dtype=np.float64)
    if w.shape != (J,) or not (np.isfinite(w).all() and (w > 0).all()):
        raise ValueError("weights must be J finite values > 0")
    return w.astype(dtype)


def _rt(tab, opt_byte, j, nodes):
    return tab[j][0 if nodes > 1 else opt_byte >> 3][opt_byte & 7]


# --------------------------------------------------------------------------- evaluator
def list_schedule(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, nodes=1, weights=None):
    """One candidate.  Returns (score, start[J], mask[J], ready) as ref_eval.list_schedule does; the score is the
    weighted sum of completion times (the unweighted sum of ref_completion with weights=None)."""
    if weights is None:
        return RC.list_schedule(tab, opt, prio, integer_starts, dtype, nslot, nodes)
    w = weights_as(weights, len(prio), dtype)
    mk, start, mask, ready = R.list_schedule(tab, opt, prio, integer_starts, dtype, nslot, nodes)
    if not np.isfinite(mk):
        return mk, start, mask, ready          # an infeasible candidate scores inf
    f = dtype
    acc = f(0.0)
    for i in range(len(prio)):
        j = int(prio[i])
        c = f(start[j] + f(_rt(tab, int(opt[j]), j, nodes)))
        acc = f(acc + f(w[j] * c))
    return float(acc), start, mask, ready


def list_schedule_batch(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, want_plan=False,
                        weights=None):
    """Vectorised over candidates (one node), as ref_eval.list_schedule_batch; score = the weighted sum in fold
    order."""
    if weights is None:
        return RC.list_schedule_batch(tab, opt, prio, integer_starts, dtype, nslot, want_plan)
    mk, start, mask = R.list_schedule_batch(tab, opt, prio, integer_starts, dtype, nslot, want_plan=True)
    tab = np.asarray(tab).astype(dtype)
    opt = np.asarray(opt)
    prio = np.asarray(prio).astype(np.int64)
    B, J = prio.shape
    w = weights_as(weights, J, dtype)
    ar = np.arange(B)
    acc = np.zeros(B, dtype=dtype)
    with np.errstate(invalid="ignore"):
        for i in range(J):
            j = prio[:, i]
            o = opt[ar, j].astype(np.int64)
            rt = tab[j, o >> 3, np.minimum(o & 7, nslot - 1)]
            c = (start[ar, j] + rt).astype(dtype)
            acc = (acc + (w[j] * c).astype(dtype)).astype(dtype)
    acc = np.where(np.isfinite(mk), acc, np.inf).astype(dtype)
    return (acc, start, mask) if want_plan else acc


def brute_force(tab, valid_opts: Sequence[Sequence[int]], integer_starts=True, nslot=R.NSLOT, dtype=np.float64,
                nodes=1, weights=None):
    """Exhaustive minimum of the weighted sum over all (option vector, permutation) candidates (J <= ~6), as
    ref_eval.brute_force.  Returns (score, opt, prio)."""
    if weights is None:
        return RC.brute_force(tab, valid_opts, integer_starts, nslot, dtype, nodes)
    J = len(valid_opts)
    weights_as(weights, J, dtype)
    best = (R.INF, None, None)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    for ov in itertools.product(*valid_opts):
        for perm in itertools.permutations(range(J)):
            v = list_schedule(tab, ov, perm, integer_starts, dtype, nslot, nodes, weights=weights)[0]
            if v < best[0]:
                best = (v, tuple(ov), tuple(perm))
    return best


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_weighted.c")
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
        for name in ("ref_weighted_f32", "ref_weighted_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False, threads=0, nodes=1,
               weights=None):
    """Weighted sum of completion times of B candidates in C, same arguments as ref_completion.c_evaluate plus
    weights[J]: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16 -> total[B] (+ start, mask)."""
    if weights is None:
        return RC.c_evaluate(tab, opt, prio, integer_starts, dtype, nslot, want_plan, threads, nodes)
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    assert prio.dtype in (np.uint8, np.uint16)
    prio = np.ascontiguousarray(prio)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    w = np.ascontiguousarray(weights_as(weights, J, dtype))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_weighted_f32 if dtype == np.float32 else _load().ref_weighted_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), w.ctypes.data, tot.ctypes.data, start.ctypes.data if want_plan else None,
            mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_weighted rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, weights, time_limit=60.0, mip_rel_gap=None):
    """The completion MILP (see the module doc) with the objective sum_t w_t C[t], HiGHS via scipy.
    Returns dict(status, proven_optimal, objective_value, weighted_completion, total_completion, makespan, start[J],
    mask[J], opt_idx[J], wall_s, n_vars, n_cons); the last three sums are recomputed from the decoded plan.
    mip_rel_gap: HiGHS' relative gap at which the search stops (None = its default, 1e-4)."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from . import ref_milp
    Rw, integrality, lb, ub, idx = ref_milp.build(gpu_time_tuples)
    J, M, G = idx["J"], idx["M"], ref_milp.G
    w = weights_as(weights, J, np.float64)
    comp = list(range(idx["nv"], idx["nv"] + J))
    nv = idx["nv"] + J
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):                                 # C[t] in the form of family (i)
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
    integrality = np.concatenate([integrality, np.zeros(J)])
    lb = np.concatenate([lb, np.zeros(J)])
    ub = np.concatenate([ub, np.full(J, np.inf)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nv))
    c = np.zeros(nv)
    c[comp] = w
    options = {"time_limit": float(time_limit), "disp": False}
    if mip_rel_gap is not None:
        options["mip_rel_gap"] = float(mip_rel_gap)
    t0 = time.perf_counter()
    res = milp(c, constraints=LinearConstraint(A, Rw.lo, Rw.hi), integrality=integrality, bounds=Bounds(lb, ub),
               options=options)
    out = {"status": int(res.status), "proven_optimal": res.status == 0, "wall_s": time.perf_counter() - t0,
           "n_vars": nv, "n_cons": Rw.n, "objective_value": None, "weighted_completion": None,
           "total_completion": None, "makespan": None, "start": None, "mask": None, "opt_idx": None}
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
    done = [start[t] + gpu_time_tuples[t][opt_idx[t]][1] for t in range(J)]
    out.update(objective_value=float(res.fun), start=start, mask=mask, opt_idx=opt_idx,
               weighted_completion=sum(float(w[t]) * done[t] for t in range(J)), total_completion=sum(done),
               makespan=max(done))
    return out
