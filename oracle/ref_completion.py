"""CPU ORACLE (test infrastructure — NOT product code): the sum-of-completion-times objective.

The schedule of a candidate does not depend on the objective: `oracle/ref_eval.py` defines it (starts, slot
masks) and this module only scores it differently,

    total = sum_j (start_j + rt_j)

In fp32 the sum is a LEFT FOLD IN SCHEDULE ORDER, acc = acc + (start + rt) from +0, one add per job, never paired
or reassociated — the order the kernels add in (SB_FLAG_SUM_COMPLETION), so that the two agree bit for bit.
objective="makespan" everywhere here is exactly `ref_eval` (delegation, nothing restated).

Also here:
  * `c_evaluate` — the same fold in plain C (`oracle/ref_completion.c`, a separate library next to the makespan
    port `ref_eval.c`) for batches of 1e5 candidates;
  * `milp_solve` — the MILP of `oracle/ref_milp.py` with the completion objective: one continuous C[t] >= 0 per
    task with  C[t] >= sta[g][t] + rt[t][s] - M(1 - bss[t][s])  for every g and s (the form of family (i)),
    minimising sum_t C[t].  The reference's own completion-time branch (saturn/solver/milp.py:89,174-182,
    makespan_opt=False) is unreachable from solve() (milp.py:372 always passes True) and bounds each
    completion by the start alone, without the runtime; it is not restated.  M is ref_milp's: every start of a
    plan that is optimal for the sum is at most H (list schedules dominate, DESIGN.md §3.1).

List schedules contain an optimum for either objective (DESIGN.md §3.1 has the dominance argument;
tests/test_completion_oracle.py checks it on the MILP's plans).
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

OBJECTIVES = ("makespan", "completion")
_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_completion.so")
_lib = None


def _check(objective):
    if objective not in OBJECTIVES:
        raise ValueError("objective must be 'makespan' or 'completion', not %r" % (objective,))
    return objective == "completion"


def _rt(tab, opt_byte, j, nodes):
    return tab[j][0 if nodes > 1 else opt_byte >> 3][opt_byte & 7]


# --------------------------------------------------------------------------- evaluator
def list_schedule(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, nodes=1,
                  objective="completion"):
    """One candidate.  Returns (score, start[J], mask[J], ready) as ref_eval.list_schedule does; the score is the
    sum of completion times (objective="completion") or the makespan ("makespan": ref_eval unchanged)."""
    total = _check(objective)
    mk, start, mask, ready = R.list_schedule(tab, opt, prio, integer_starts, dtype, nslot, nodes)
    if not total or not np.isfinite(mk):
        return mk, start, mask, ready          # the makespan; an infeasible candidate is inf under both objectives
    f = dtype
    acc = f(0.0)
    for i in range(len(prio)):
        j = int(prio[i])
        c = f(start[j] + f(_rt(tab, int(opt[j]), j, nodes)))
        acc = f(acc + c)
    return float(acc), start, mask, ready


def list_schedule_batch(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, want_plan=False,
                        objective="completion"):
    """Vectorised over candidates (one node), as ref_eval.list_schedule_batch; score = the sum in fold order."""
    total = _check(objective)
    if not total:
        return R.list_schedule_batch(tab, opt, prio, integer_starts, dtype, nslot, want_plan)
    mk, start, mask = R.list_schedule_batch(tab, opt, prio, integer_starts, dtype, nslot, want_plan=True)
    tab = np.asarray(tab).astype(dtype)
    opt = np.asarray(opt)
    prio = np.asarray(prio).astype(np.int64)
    B, J = prio.shape
    ar = np.arange(B)
    acc = np.zeros(B, dtype=dtype)
    with np.errstate(invalid="ignore"):
        for i in range(J):
            j = prio[:, i]
            o = opt[ar, j].astype(np.int64)
            rt = tab[j, o >> 3, np.minimum(o & 7, nslot - 1)]
            acc = (acc + (start[ar, j] + rt).astype(dtype)).astype(dtype)
    acc = np.where(np.isfinite(mk), acc, np.inf).astype(dtype)
    return (acc, start, mask) if want_plan else acc


def brute_force(tab, valid_opts: Sequence[Sequence[int]], integer_starts=True, nslot=R.NSLOT, dtype=np.float64,
                nodes=1, objective="completion"):
    """Exhaustive minimum of the objective over all (option vector, permutation) candidates (J <= ~6), as
    ref_eval.brute_force.  Returns (score, opt, prio)."""
    if not _check(objective):
        return R.brute_force(tab, valid_opts, integer_starts, nslot, dtype, nodes)
    J = len(valid_opts)
    best = (R.INF, None, None)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    for ov in itertools.product(*valid_opts):
        for perm in itertools.permutations(range(J)):
            v = list_schedule(tab, ov, perm, integer_starts, dtype, nslot, nodes)[0]
            if v < best[0]:
                best = (v, tuple(ov), tuple(perm))
    return best


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_completion.c")
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
        for name in ("ref_completion_f32", "ref_completion_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False, threads=0, nodes=1):
    """Sum of completion times of B candidates in C, same arguments as c_oracle.evaluate:
    tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16 -> total[B] (+ start, mask)."""
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    assert prio.dtype in (np.uint8, np.uint16)
    prio = np.ascontiguousarray(prio)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_completion_f32 if dtype == np.float32 else _load().ref_completion_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), tot.ctypes.data, start.ctypes.data if want_plan else None,
            mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_completion rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def milp_solve(gpu_time_tuples, time_limit=60.0, mip_rel_gap=None):
    """The MILP of oracle/ref_milp.py with the objective sum_t C[t] (see the module doc), HiGHS via scipy.
    Returns dict(status, proven_optimal, objective_value, total_completion, makespan, start[J], mask[J],
    opt_idx[J], wall_s, n_vars, n_cons); total_completion / makespan are recomputed from the decoded plan.
    mip_rel_gap: HiGHS' relative gap at which the search stops (None = its default, 1e-4)."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from . import ref_milp
    Rw, integrality, lb, ub, idx = ref_milp.build(gpu_time_tuples)
    J, M, G = idx["J"], idx["M"], ref_milp.G
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
    c[comp] = 1.0
    options = {"time_limit": float(time_limit), "disp": False}
    if mip_rel_gap is not None:
        options["mip_rel_gap"] = float(mip_rel_gap)
    t0 = time.perf_counter()
    res = milp(c, constraints=LinearConstraint(A, Rw.lo, Rw.hi), integrality=integrality, bounds=Bounds(lb, ub),
               options=options)
    out = {"status": int(res.status), "proven_optimal": res.status == 0, "wall_s": time.perf_counter() - t0,
           "n_vars": nv, "n_cons": Rw.n, "objective_value": None, "total_completion": None, "makespan": None,
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
    done = [start[t] + gpu_time_tuples[t][opt_idx[t]][1] for t in range(J)]
    out.update(objective_value=float(res.fun), start=start, mask=mask, opt_idx=opt_idx, total_completion=sum(done),
               makespan=max(done))
    return out
