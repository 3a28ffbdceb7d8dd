"""CPU ORACLE (test infrastructure — NOT product code): list schedules with RELEASE DATES.

The rule of `oracle/ref_eval.py` with one change: a job starts no earlier than its release date,

    sel   = k slots of the job's node with smallest (ready, slot)      (ties -> lowest slot)
    start = max(max(ready[sel]), r_j)
    ready[sel] = start + (integer_starts ? ceil(rt) : rt)

With integer starts the release enters as ceil(r_j) (a start >= r with an integer start is a start >= ceil(r)), so
every start stays an integer.  `release_as` gives the values the device uses: rounded UP to fp32 (the engine's
release_f32) when dtype is fp32, then ceiled under integer starts, and -0 stored as +0 (as sb_set_release
does).  r <= 0 changes nothing (ready >= +0).

Every score fold of the other oracles runs on this schedule, step for step as they fold it:
  * "makespan"             mk = max(mk, start + rt)                                  (ref_eval)
  * "completion"           acc = acc + (start + rt)                                  (ref_completion)
  * "weighted_completion"  acc = acc + (w * (start + rt))                            (ref_weighted)
  * "tardiness" / "weighted_tardiness"
                           acc = acc + (w * max((start + rt) - d, +0))              (ref_tardiness, unit w)
in schedule order from +0, each step rounded on its own.

Also here:
  * `c_evaluate` — the same schedule and folds in plain C (`oracle/ref_release.c`, a library of its own), and the
    other five objectives of the library (`C_OBJECTIVES`) through the C ports of ref_max_lateness, ref_late_tasks and
    ref_max_tardiness;
  * `brute_force` — the exhaustive list-schedule optimum (every option vector and permutation, scored by the C port);
  * `milp_solve` — the MILPs of ref_milp / ref_completion / ref_weighted / ref_tardiness plus
    sta[g][t] - r_t * tga[t][g] >= 0 for every g, with the big-M horizon raised to
    max_t ceil(r_t) + sum_t ceil(max rt) + 1 (and M3 = 8 M).  List schedules still contain an optimum
    (DESIGN.md §3.1, *Release dates*).
"""
from __future__ import annotations

import ctypes
import importlib
import itertools
import math
import os
import subprocess
import time
from typing import Sequence

import numpy as np

from . import ref_eval as R

OBJECTIVES = ("makespan", "completion", "weighted_completion", "tardiness", "weighted_tardiness")
_CODE = {o: i for i, o in enumerate(OBJECTIVES)}
# the objectives c_evaluate scores through another oracle's C port (ref_release.c folds OBJECTIVES only)
_PORTS = {"max_lateness": "ref_max_lateness", "late_tasks": "ref_late_tasks", "weighted_late_tasks": "ref_late_tasks",
          "max_tardiness": "ref_max_tardiness", "weighted_max_tardiness": "ref_max_tardiness"}
C_OBJECTIVES = OBJECTIVES + tuple(_PORTS)          # every objective c_evaluate accepts, in the library's order
_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_release.so")
_lib = None


def release_as(release, J, dtype, integer_starts):
    """The release dates the schedule uses, in `dtype`: fp32 rounds UP (so start >= r holds in float64 too), fp64
    keeps the values; then ceil under integer starts.  Values must be finite."""
    r = np.asarray(release, dtype=np.float64)
    if r.shape != (J,) or not np.isfinite(r).all():
        raise ValueError("release dates must be J finite values")
    out = r.astype(dtype)
    low = out.astype(np.float64) < r
    out[low] = np.nextafter(out[low], dtype(np.inf))
    out = np.ceil(out).astype(dtype) if integer_starts else out
    return (out + dtype(0.0)).astype(dtype)        # -0 -> +0, as sb_set_release stores it


def _per_job(objective, J, dtype, weights, due):
    if objective not in OBJECTIVES:
        raise ValueError("objective must be one of %s, not %r" % (OBJECTIVES, objective))
    w = np.ones(J, dtype=dtype) if weights is None else np.asarray(weights, dtype=np.float64).astype(dtype)
    d = np.zeros(J, dtype=dtype)
    if objective.endswith("tardiness"):
        if due is None:
            raise ValueError("objective=%r needs due dates" % objective)
        d = np.asarray(due, dtype=np.float64).astype(dtype)
    return w, d


def _rt(tab, opt_byte, j, nodes):
    return tab[j][0 if nodes > 1 else opt_byte >> 3][opt_byte & 7]


# --------------------------------------------------------------------------- evaluator
def list_schedule(tab, opt, prio, release, integer_starts=True, dtype=np.float64, nslot=R.NSLOT, nodes=1,
                  objective="makespan", weights=None, due=None):
    """One candidate.  Returns (score, start[J], mask[J], ready) as ref_eval.list_schedule does (mask[j] =
    (node << 16) | gpu bits); an infeasible candidate scores inf."""
    f = dtype
    J = len(prio)
    r = release_as(release, J, dtype, integer_starts)
    w, d = _per_job(objective, J, dtype, weights, due)
    ready = [[f(0.0)] * nslot for _ in range(nodes)]
    start = [f(0.0)] * J
    mask = [0] * J
    acc = f(0.0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        k = (o & 7) + 1
        n = (o >> 3) if nodes > 1 else 0
        rt = f(_rt(tab, o, j, nodes))
        if k > nslot or n >= nodes:
            return float("inf"), start, mask, ready
        rd = ready[n]
        sel = sorted(range(nslot), key=lambda g: (rd[g], g))[:k]
        s = max(rd[sel[-1]], r[j])
        hold = f(math.ceil(rt)) if (integer_starts and math.isfinite(rt)) else rt
        nxt = f(s + hold)
        m = 0
        for g in sel:
            rd[g] = nxt
            m |= 1 << g
        start[j] = s
        mask[j] = (n << 16) | m if nodes > 1 else m
        e = f(s + rt)
        if objective == "makespan":
            if e > acc:
                acc = e
        elif objective == "completion":
            acc = f(acc + e)
        elif objective == "weighted_completion":
            acc = f(acc + f(w[j] * e))
        else:
            acc = f(acc + f(w[j] * max(f(e - d[j]), f(0.0))))
    return float(acc), start, mask, ready


def list_schedule_batch(tab, opt, prio, release, integer_starts=True, dtype=np.float64, nslot=R.NSLOT,
                        want_plan=False, objective="makespan", weights=None, due=None):
    """Vectorised over candidates (one node).  Returns score[B] (and start[B][J], mask[B][J] if want_plan)."""
    tab = np.asarray(tab).astype(dtype)
    opt = np.asarray(opt)
    prio = np.asarray(prio).astype(np.int64)
    B, J = prio.shape
    r = release_as(release, J, dtype, integer_starts)
    w, d = _per_job(objective, J, dtype, weights, due)
    ar = np.arange(B)
    ready = np.zeros((B, nslot), dtype=dtype)
    acc = np.zeros(B, dtype=dtype)
    bad = np.zeros(B, dtype=bool)
    start = np.zeros((B, J), dtype=dtype)
    mask = np.zeros((B, J), dtype=np.uint32)
    bits = (1 << np.arange(nslot)).astype(np.uint32)
    zero = dtype(0.0)
    for i in range(J):
        j = prio[:, i]
        o = opt[ar, j].astype(np.int64)
        km1 = o & 7
        rt = tab[j, o >> 3, np.minimum(km1, nslot - 1)]
        bad |= km1 >= nslot
        km1c = np.minimum(km1, nslot - 1)
        order = np.argsort(ready, axis=1, kind="stable")
        s = np.maximum(np.take_along_axis(ready, order, axis=1)[ar, km1c], r[j]).astype(dtype)
        rank = np.empty_like(order)
        np.put_along_axis(rank, order, np.arange(nslot)[None, :].repeat(B, 0), axis=1)
        sel = rank <= km1c[:, None]
        with np.errstate(invalid="ignore"):
            hold = np.where(np.isfinite(rt), np.ceil(rt), rt).astype(dtype) if integer_starts else rt
            nxt = (s + hold).astype(dtype)
            e = (s + rt).astype(dtype)
            if objective == "makespan":
                acc = np.maximum(acc, e)
            elif objective == "completion":
                acc = (acc + e).astype(dtype)
            elif objective == "weighted_completion":
                acc = (acc + (w[j] * e).astype(dtype)).astype(dtype)
            else:
                t = np.maximum((e - d[j]).astype(dtype), zero)
                acc = (acc + (w[j] * t).astype(dtype)).astype(dtype)
        ready = np.where(sel, nxt[:, None], ready)
        start[ar, j] = s
        mask[ar, j] = (sel * bits[None, :]).sum(axis=1).astype(np.uint32)
    acc = np.where(bad, np.inf, acc).astype(dtype)
    return (acc, start, mask) if want_plan else acc


def brute_force(tab, valid_opts: Sequence[Sequence[int]], release, objective="makespan", integer_starts=True,
                nslot=R.NSLOT, dtype=np.float64, nodes=1, weights=None, due=None):
    """Exhaustive minimum over all (option vector, permutation) candidates (J <= ~6), the first minimum in the
    enumeration order of ref_eval.brute_force, scored by the C port.  Returns (score, opt, prio)."""
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    opt = np.repeat(opts, len(perms), axis=0)
    prio = np.tile(perms, (len(opts), 1))
    tot = c_evaluate(tab, opt, prio, release, integer_starts, dtype, nslot, threads=os.cpu_count() or 1, nodes=nodes,
                     objective=objective, weights=weights, due=due)
    i = int(np.argmin(tot))
    return float(tot[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_release.c")
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
        for name in ("ref_release_f32", "ref_release_f64"):
            fn = getattr(_lib, name)
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                           ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, release, integer_starts=True, dtype=np.float32, nslot=8, want_plan=False, threads=0,
               nodes=1, objective="makespan", weights=None, due=None):
    """Scores of B candidates in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, release[J] -> score[B]
    (+ start, mask).  `objective` is any of C_OBJECTIVES."""
    if objective in _PORTS:
        port = importlib.import_module("." + _PORTS[objective], __package__)
        kw = {} if objective == "max_lateness" else {"weights": weights}
        return port.c_evaluate(tab, opt, prio, due, release, integer_starts, dtype, nslot, want_plan, threads, nodes,
                               **kw)
    tab = np.ascontiguousarray(tab, dtype=dtype)
    J, S, W = tab.shape
    assert W == 8
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    assert prio.dtype in (np.uint8, np.uint16)
    prio = np.ascontiguousarray(prio)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    r = np.ascontiguousarray(release_as(release, J, dtype, integer_starts))
    w, d = (np.ascontiguousarray(x) for x in _per_job(objective, J, dtype, weights, due))
    tot = np.empty(B, dtype=dtype)
    start = np.zeros((B, J), dtype=dtype) if want_plan else None
    mask = np.zeros((B, J), dtype=np.uint32) if want_plan else None
    fn = _load().ref_release_f32 if dtype == np.float32 else _load().ref_release_f64
    rc = fn(tab.ctypes.data, J, S, opt.ctypes.data, prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
            nslot, int(nodes), _CODE[objective], w.ctypes.data, d.ctypes.data, r.ctypes.data, tot.ctypes.data,
            start.ctypes.data if want_plan else None, mask.ctypes.data if want_plan else None, int(threads))
    if rc != 0:
        raise RuntimeError("ref_release rc=%d" % rc)
    return (tot, start, mask) if want_plan else tot


# --------------------------------------------------------------------------- MILP
def _build(gpu_time_tuples, release):
    """ref_milp.build's model with the big-M horizon raised by max_t ceil(r_t) (the latest release)."""
    from .ref_milp import G, _Rows
    J = len(gpu_time_tuples)
    M = float(max(0, max(math.ceil(x) for x in release)) +
              sum(math.ceil(max(rt for (_k, rt) in tup)) for tup in gpu_time_tuples) + 1)
    M3 = 8.0 * M
    off = 0
    bss = []
    for tup in gpu_time_tuples:
        bss.append(list(range(off, off + len(tup))))
        off += len(tup)
    bna = list(range(off, off + J)); off += J
    sta = [[off + g * J + t for t in range(J)] for g in range(G)]; off += G * J
    mk = off; off += 1
    tga = [[off + t * G + g for g in range(G)] for t in range(J)]; off += J * G
    boa = {}
    for a in range(J):
        for b in range(J):
            if a != b:
                boa[(a, b)] = off
                off += 1
    nv = off
    Rw = _Rows()
    inf = np.inf
    for t in range(J):
        Rw.add(bss[t], [1.0] * len(bss[t]), 1.0, 1.0)
        Rw.add([bna[t]], [1.0], 1.0, 1.0)
    for t, tup in enumerate(gpu_time_tuples):
        for s, (k, rt) in enumerate(tup):
            for g in range(G):
                Rw.add([mk, sta[g][t], bss[t][s]], [1.0, -1.0, -M], rt - M, inf)
            cols = tga[t] + [bss[t][s], bna[t]]
            Rw.add(cols, [1.0] * G + [-M, -M], k - 2 * M, inf)
            Rw.add(cols, [1.0] * G + [M, M], -inf, k + 2 * M)
            for g in range(G):
                coef = {sta[gg][t]: 1.0 / k for gg in range(G)}
                coef[sta[g][t]] -= 1.0
                cols3 = list(coef.keys()) + [tga[t][g], bss[t][s], bna[t]]
                Rw.add(cols3, list(coef.values()) + [M3, M3, M3], -inf, 3 * M3)
                Rw.add(cols3, list(coef.values()) + [-M3, -M3, -M3], -3 * M3, inf)
        for g in range(G):                                     # the release: sta[g][t] >= r_t on an occupied GPU
            Rw.add([sta[g][t], tga[t][g]], [1.0, -float(release[t])], 0.0, inf)
    for g in range(G):
        for t in range(J):
            for p in range(J):
                if p == t:
                    continue
                b = boa[(p, t)]
                for s, (_k, rt) in enumerate(gpu_time_tuples[t]):
                    Rw.add([sta[g][t], sta[g][p], tga[p][g], tga[t][g], b, bss[t][s]],
                           [1.0, -1.0, M, M, -M, M], -inf, -rt + 3 * M)
                for s, (_k, rt) in enumerate(gpu_time_tuples[p]):
                    Rw.add([sta[g][t], sta[g][p], tga[t][g], tga[p][g], b, bss[p][s]],
                           [1.0, -1.0, -M, -M, -M, -M], rt - 4 * M, inf)
    integrality = np.ones(nv)
    integrality[mk] = 0
    lb = np.zeros(nv)
    ub = np.ones(nv)
    for g in range(G):
        for t in range(J):
            ub[sta[g][t]] = M
    ub[mk] = np.inf
    return Rw, integrality, lb, ub, dict(bss=bss, bna=bna, sta=sta, mk=mk, tga=tga, boa=boa, nv=nv, M=M, J=J)


def milp_solve(gpu_time_tuples, release, objective, weights=None, due=None, time_limit=60.0, mip_rel_gap=None):
    """The release-date MILP (see the module doc) under HiGHS via scipy.  objective: "makespan", "completion" (with
    `weights`: the weighted sum) or "tardiness" (with `due`, and `weights` optionally).  Returns dict(status,
    proven_optimal, objective_value, score, start[J], mask[J], opt_idx[J], wall_s, n_vars, n_cons); `score` is
    recomputed in float64 from the decoded plan."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    from scipy.sparse import csr_matrix
    from .ref_milp import G
    if objective not in ("makespan", "completion", "tardiness"):
        raise ValueError("objective must be 'makespan', 'completion' or 'tardiness'")
    J = len(gpu_time_tuples)
    r = [float(x) for x in np.asarray(release, dtype=np.float64)]
    Rw, integrality, lb, ub, idx = _build(gpu_time_tuples, r)
    M = idx["M"]
    w = np.ones(J) if weights is None else np.asarray(weights, dtype=np.float64)
    d = np.zeros(J) if due is None else np.asarray(due, dtype=np.float64)
    nv = idx["nv"]
    c_extra = 0
    if objective != "makespan":
        comp = list(range(nv, nv + J))
        c_extra = J
        for t, tup in enumerate(gpu_time_tuples):
            for s, (_k, rt) in enumerate(tup):
                for g in range(G):
                    Rw.add([comp[t], idx["sta"][g][t], idx["bss"][t][s]], [1.0, -1.0, -M], rt - M, np.inf)
        if objective == "tardiness":
            late = list(range(nv + J, nv + 2 * J))
            c_extra = 2 * J
            for t in range(J):
                Rw.add([late[t], comp[t]], [1.0, -1.0], -d[t], np.inf)
    nvt = nv + c_extra
    integrality = np.concatenate([integrality, np.zeros(c_extra)])
    lb = np.concatenate([lb, np.zeros(c_extra)])
    ub = np.concatenate([ub, np.full(c_extra, np.inf)])
    A = csr_matrix((Rw.v, (Rw.r, Rw.c)), shape=(Rw.n, nvt))
    c = np.zeros(nvt)
    if objective == "makespan":
        c[idx["mk"]] = 1.0
    elif objective == "completion":
        c[comp] = w
    else:
        c[late] = w
    options = {"time_limit": float(time_limit), "disp": False}
    if mip_rel_gap is not None:
        options["mip_rel_gap"] = float(mip_rel_gap)
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
               score=plan_score(gpu_time_tuples, start, opt_idx, objective, weights, due))
    return out


def plan_score(gpu_time_tuples, start, opt_idx, objective, weights=None, due=None):
    """A plan's objective in float64: the makespan, sum_t w_t C_t, or sum_t w_t max(0, C_t - d_t)."""
    J = len(start)
    C = [start[t] + gpu_time_tuples[t][opt_idx[t]][1] for t in range(J)]
    w = [1.0] * J if weights is None else [float(x) for x in weights]
    if objective == "makespan":
        return max(C)
    if objective == "completion":
        return sum(w[t] * C[t] for t in range(J))
    return sum(w[t] * max(0.0, C[t] - float(due[t])) for t in range(J))
