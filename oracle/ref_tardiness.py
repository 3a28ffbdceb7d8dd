"""CPU ORACLE (test infrastructure — NOT product code): the total WEIGHTED TARDINESS.

The schedule of a candidate does not depend on the objective: `oracle/ref_eval.py` defines it (starts, slot masks)
and this module only scores it,

    total = sum_j w_j max(0, start_j + rt_j - d_j)

In fp32 the score is a LEFT FOLD IN SCHEDULE ORDER from +0 with these steps per job, each rounded on its own:
e = start_j + rt_j, l = e - d_j, t = max(l, +0), acc = acc + (w_j * t) — never a fused multiply-add, nothing
reassociated (the kernels use __fsub_rn / __fmul_rn / __fadd_rn for SB_FLAG_DUE).  Weights are finite and > 0
(weights=None: unit weights), due dates finite.  d = 0 gives the weighted fold of `oracle/ref_weighted.py` bit for
bit (e >= 0), due dates at or past every completion give +0, w = 2 gives exactly twice w = 1.

Also here:
  * `c_evaluate` — the same fold in plain C (`oracle/ref_tardiness.c`, a library of its own);
  * `brute_force` — the exhaustive list-schedule optimum (every option vector and permutation, scored by the C port);
  * `milp_solve` — the completion MILP of `oracle/ref_weighted.py` plus a continuous U[t] >= C[t] - d[t], U[t] >= 0
    per task, with the objective sum_t w_t U[t].  The objective does not decrease when a completion time grows, so
    list schedules still contain an optimum (DESIGN.md §3.1), and ref_milp's M still bounds the starts.
"""
from __future__ import annotations

import ctypes
import itertools
import os
import subprocess
import time
from typing import Sequence

import numpy as np

from . import ref_eval as R
from .ref_weighted import weights_as

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_tardiness.so")
_lib = None


def due_as(due, J, dtype):
    """due dates (length J, finite) in `dtype` (round to nearest); ValueError otherwise."""
    d = np.asarray(due, dtype=np.float64)
    if d.shape != (J,) or not np.isfinite(d).all():
        raise ValueError("due dates must be J finite values")
    return d.astype(dtype)


def _w(weights, J, dtype):
    return np.ones(J, dtype=dtype) if weights is None else weights_as(weights, J, dtype)


def _rt(tab, opt_byte, j, nodes):
    return tab[j][0 if nodes > 1 else opt_byte >> 3][opt_byte & 7]


# --------------------------------------------------------------------------- evaluator
def list_schedule(tab, opt, prio, due, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, nodes=1, weights=None):
    """One candidate.  Returns (score, start[J], mask[J], ready) as ref_eval.list_schedule does; the score is the
    weighted tardiness (unit weights with weights=None)."""
    J = len(prio)
    w, d = _w(weights, J, dtype), due_as(due, J, dtype)
    mk, start, mask, ready = R.list_schedule(tab, opt, prio, integer_starts, dtype, nslot, nodes)
    if not np.isfinite(mk):
        return mk, start, mask, ready          # an infeasible candidate scores inf
    f = dtype
    acc = f(0.0)
    for i in range(J):
        j = int(prio[i])
        e = f(start[j] + f(_rt(tab, int(opt[j]), j, nodes)))
        t = max(f(e - d[j]), f(0.0))
        acc = f(acc + f(w[j] * t))
    return float(acc), start, mask, ready


def list_schedule_batch(tab, opt, prio, due, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, want_plan=False,
                        weights=None):
    """Vectorised over candidates (one node), as ref_eval.list_schedule_batch; score = the weighted tardiness in
    fold order."""
    mk, start, mask = R.list_schedule_batch(tab, opt, prio, integer_starts, dtype, nslot, want_plan=True)
    tab = np.asarray(tab).astype(dtype)
    opt = np.asarray(opt)
    prio = np.asarray(prio).astype(np.int64)
    B, J = prio.shape
    w, d = _w(weights, J, dtype), due_as(due, J, dtype)
    ar = np.arange(B)
    acc = np.zeros(B, dtype=dtype)
    zero = dtype(0.0)
    with np.errstate(invalid="ignore"):
        for i in range(J):
            j = prio[:, i]
            o = opt[ar, j].astype(np.int64)
            rt = tab[j, o >> 3, np.minimum(o & 7, nslot - 1)]
            e = (start[ar, j] + rt).astype(dtype)
            t = np.maximum((e - d[j]).astype(dtype), zero)
            acc = (acc + (w[j] * t).astype(dtype)).astype(dtype)
    acc = np.where(np.isfinite(mk), acc, np.inf).astype(dtype)
    return (acc, start, mask) if want_plan else acc


def brute_force(tab, valid_opts: Sequence[Sequence[int]], due, integer_starts=True, nslot=R.NSLOT, dtype=np.float64,
                nodes=1, weights=None):
    """Exhaustive minimum of the weighted tardiness over all (option vector, permutation) candidates (J <= ~6), the
    first minimum in the enumeration order of ref_eval.brute_force, scored by the C port (which the tests hold to
    the Python fold bit for bit).  Returns (score, opt, prio)."""
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    tot = c_evaluate(tab, opt, prio, due, integer_starts, dtype, nslot, threads=os.cpu_count() or 1, nodes=nodes,
                     weights=weights)
    i = int(np.argmin(tot))
    return float(tot[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_tardiness.c")
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
        for name in ("ref_tardiness_f32", "ref_tardiness_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, due, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False, threads=0,
               nodes=1, weights=None):
    """Weighted tardiness of B candidates in C, same arguments as ref_weighted.c_evaluate plus due[J]:
    tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16 -> total[B] (+ start, mask).  weights=None: unit weights."""
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    assert prio.dtype in (np.uint8, np.uint16)
    prio = np.ascontiguousarray(prio)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    w = np.ascontiguousarray(_w(weights, J, dtype))
    d = np.ascontiguousarray(due_as(due, J, dtype))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_tardiness_f32 if dtype == np.float32 else _load().ref_tardiness_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), w.ctypes.data, d.ctypes.data, tot.ctypes.data, start.ctypes.data if want_plan else None,
            mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_tardiness rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, due, weights=None, time_limit=60.0, mip_rel_gap=None):
    """The tardiness MILP (see the module doc), HiGHS via scipy.  Returns dict(status, proven_optimal,
    objective_value, weighted_tardiness, late_tasks, start[J], mask[J], opt_idx[J], wall_s, n_vars, n_cons); the
    weighted tardiness and the late tasks are recomputed from the decoded plan.
    mip_rel_gap: HiGHS' relative gap at which the search stops (None = its default, 1e-4)."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from . import ref_milp
    Rw, integrality, lb, ub, idx = ref_milp.build(gpu_time_tuples)
    J, M, G = idx["J"], idx["M"], ref_milp.G
    w = _w(weights, J, np.float64)
    d = due_as(due, J, np.float64)
    comp = list(range(idx["nv"], idx["nv"] + J))
    late = list(range(idx["nv"] + J, idx["nv"] + 2 * J))
    nv = idx["nv"] + 2 * J
    for t, tup in enumerate(gpu_time_tuples):
        for s, (_k, rt) in enumerate(tup):
            for g in range(G):                                 # C[t] in the form of family (i), as ref_weighted
                Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        Rw.add([late[t], comp[t]], [1.0, -1.0], -d[t], np.inf)  # U[t] >= C[t] - d[t]
    integrality = np.concatenate([integrality, np.zeros(2 * J)])
    lb = np.concatenate([lb, np.zeros(2 * J)])                    # C[t] >= 0, U[t] >= 0
    ub = np.concatenate([ub, np.full(2 * J, np.inf)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nv))
    c = np.zeros(nv)
    c[late] = w
    options = {"time_limit": float(time_limit), "disp": False}
    if mip_rel_gap is not None:
        options["mip_rel_gap"] = float(mip_rel_gap)
    t0 = time.perf_counter()
    res = milp(c, constraints=LinearConstraint(A, Rw.lo, Rw.hi), integrality=integrality, bounds=Bounds(lb, ub),
               options=options)
    out = {"status": int(res.status), "proven_optimal": res.status == 0, "wall_s": time.perf_counter() - t0,
           "n_vars": nv, "n_cons": Rw.n, "objective_value": None, "weighted_tardiness": None, "late_tasks": None,
           "start": None, "mask": None, "opt_idx": None}
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
    lateness = [start[t] + gpu_time_tuples[t][opt_idx[t]][1] - d[t] for t in range(J)]
    out.update(objective_value=float(res.fun), start=start, mask=mask, opt_idx=opt_idx,
               weighted_tardiness=sum(float(w[t]) * max(0.0, lateness[t]) for t in range(J)),
               late_tasks=sum(1 for x in lateness if x > 0))
    return out
