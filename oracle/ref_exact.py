"""CPU ORACLE (test infrastructure — NOT product code): the list schedule in EXACT arithmetic.

The rule of `oracle/ref_release.py` (ref_eval's list schedule with release dates, and every score fold), computed
with `fractions.Fraction` instead of floating point:

    sel   = k slots of the job's node with smallest (ready, slot)      (ties -> lowest slot)
    start = max(max(ready[sel]), r_j)            (r_j -> ceil(r_j) with integer starts)
    ready[sel] = start + (integer_starts ? ceil(rt) : rt)
    e = start + rt
    makespan                  mk  = max(mk, e)
    completion                acc = acc + e
    weighted_completion       acc = acc + w e
    (weighted) tardiness      acc = acc + w max(e - d, 0)
    max_lateness              q = D - d (D = max_t d_t),  acc = max(acc, e + q)   (the device's tail score L_max + D)
    (weighted) late_tasks     acc = acc + (e > d ? w : 0)
    (weighted) max_tardiness  acc = max(acc, w max(e - d, 0))

On an input where fp32 rounds nothing, every floating-point restatement (the fp32 and float64 oracles, the
kernels) must reproduce this value for value.  `schedule(..., exact32=True)` asserts that: every input and every
intermediate it forms (starts, slot times, completions, e - d, tails q and e + q, products, partial sums) must be
exactly representable in fp32, so an input that breaks exactness fails loudly instead of weakening a comparison.
+inf (an absent or selected sentinel cell) is carried as float('inf'); it is exact.  The objectives and their flag
bits are those of saturn_b200.engine, restated here so that the oracle loads no library.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

NSLOT = 8
# saturn_b200.engine.OBJECTIVES, in its order
OBJECTIVES = ("makespan", "completion", "weighted_completion", "tardiness", "weighted_tardiness", "max_lateness",
              "late_tasks", "weighted_late_tasks", "max_tardiness", "weighted_max_tardiness")
INF = float("inf")
# saturn_b200._lib's flag bits, restated so that the oracle loads no library
FLAG_SUM_COMPLETION, FLAG_WEIGHTED, FLAG_DUE, FLAG_MAX_LATENESS, FLAG_LATE_COUNT, FLAG_MAX_TARDINESS = (
    64, 128, 256, 1024, 2048, 4096)


def objective_flag(objective):
    """The SB_FLAG_* objective bits of saturn_b200.engine.objective_flag, restated."""
    if objective not in OBJECTIVES:
        raise ValueError("objective must be one of %s, not %r" % (OBJECTIVES, objective))
    if objective == "makespan":
        return 0
    if objective == "max_lateness":
        return FLAG_MAX_LATENESS
    late = objective.endswith("late_tasks")
    return FLAG_SUM_COMPLETION | (FLAG_WEIGHTED if objective.startswith("weighted_") else 0) | (
        FLAG_DUE if objective.endswith("tardiness") or late else 0) | (FLAG_LATE_COUNT if late else 0) | (
        FLAG_MAX_TARDINESS if objective.endswith("max_tardiness") else 0)


def needs(objective):
    """(weights, due dates): whether the objective reads per-job weights (SB_FLAG_WEIGHTED) and due dates
    (SB_FLAG_DUE, or SB_FLAG_MAX_LATENESS for the tails)."""
    f = objective_flag(objective)
    return bool(f & FLAG_WEIGHTED), bool(f & (FLAG_DUE | FLAG_MAX_LATENESS))


class NotExact(AssertionError):
    """A value of the schedule is not exactly representable in fp32."""


def _q(x):
    """An input value as an exact Fraction (+inf stays a float)."""
    x = float(x)
    if math.isnan(x) or x == -INF:
        raise ValueError("values must be numbers or +inf, got %r" % x)
    return INF if x == INF else Fraction(x)


def _check(x, what):
    if x == INF:
        return x
    if Fraction(float(np.float32(float(x)))) != x:
        raise NotExact("%s = %s is not exactly representable in fp32" % (what, x))
    return x


def _ceil(x):
    return x if x == INF else Fraction(math.ceil(x))


def schedule(tab, opt, prio, release=None, integer_starts=True, nodes=1, objective="makespan", weights=None,
             due=None, exact32=True):
    """One candidate.  tab[J][S][8] (S = 1 when nodes > 1), opt[J] bytes, prio[J] the schedule order; release,
    weights and due are J values or None (no release dates; unit weights; no due dates).  Returns (score, start[J],
    mask[J]) with Fractions (or +inf), mask[j] = (node << 16) | slot bits when nodes > 1."""
    _, use_due = needs(objective)
    f = objective_flag(objective)
    J = len(prio)
    chk = _check if exact32 else (lambda x, what: x)
    r = [Fraction(0)] * J if release is None else [_q(x) for x in release]
    if integer_starts:
        r = [_ceil(x) for x in r]
    w = [Fraction(1)] * J if weights is None else [_q(x) for x in weights]
    if use_due and due is None:
        raise ValueError("objective=%r needs due dates" % objective)
    d = [_q(x) for x in due] if use_due else [Fraction(0)] * J
    for j in range(J):
        chk(r[j], "release[%d]" % j)
        chk(w[j], "weight[%d]" % j)
        chk(d[j], "due[%d]" % j)
    if f & FLAG_MAX_LATENESS:                         # the delivery tails take the due dates' place
        D = max(d)
        d = [chk(D - x, "tail q[%d]" % j) for j, x in enumerate(d)]
    ready = [[Fraction(0)] * NSLOT for _ in range(nodes)]
    start = [Fraction(0)] * J
    mask = [0] * J
    acc = Fraction(0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        k = (o & 7) + 1
        n = (o >> 3) if nodes > 1 else 0
        if n >= nodes:
            return INF, start, mask
        rt = chk(_q(tab[j][0 if nodes > 1 else o >> 3][o & 7]), "rt[%d]" % j)
        rd = ready[n]
        sel = sorted(range(NSLOT), key=lambda g: (rd[g], g))[:k]
        s = chk(max(rd[sel[-1]], r[j]), "start[%d]" % j)
        nxt = chk(s + (_ceil(rt) if integer_starts else rt), "slot time after job %d" % j)
        m = 0
        for g in sel:
            rd[g] = nxt
            m |= 1 << g
        start[j] = s
        mask[j] = (n << 16) | m if nodes > 1 else m
        e = chk(s + rt, "completion[%d]" % j)
        if objective == "makespan":
            acc = max(acc, e)
        elif f & FLAG_MAX_LATENESS:
            acc = max(acc, chk(e + d[j], "e + q of job %d" % j))
        elif f & FLAG_LATE_COUNT:
            acc = INF if e == INF else chk(acc + w[j], "partial sum at job %d" % j) if e > d[j] else acc
        elif not f & FLAG_DUE:
            acc = chk(acc + (chk(w[j] * e, "w e of job %d" % j) if f & FLAG_WEIGHTED else e),
                      "partial sum at job %d" % j)
        else:
            x = chk(w[j] * max(chk(e - d[j], "e - d of job %d" % j), Fraction(0)), "w t of job %d" % j)
            acc = max(acc, x) if f & FLAG_MAX_TARDINESS else chk(acc + x, "partial sum at job %d" % j)
    return acc, start, mask


def batch(tab, opt, prio, release=None, integer_starts=True, nodes=1, objective="makespan", weights=None, due=None,
          rows=None, exact32=True):
    """schedule() of the candidates `rows` (default: all) of opt[B][J], prio[B][J] -> (score[n] float64,
    start[n][J] float64, mask[n][J] uint32); every value is exact (asserted to be fp32 when exact32)."""
    opt = np.asarray(opt)
    prio = np.asarray(prio)
    rows = range(opt.shape[0]) if rows is None else rows
    out_s, out_st, out_m = [], [], []
    for b in rows:
        sc, st, m = schedule(tab, opt[b], prio[b], release, integer_starts, nodes, objective, weights, due, exact32)
        out_s.append(float(sc))
        out_st.append([float(x) for x in st])
        out_m.append(m)
    return (np.array(out_s, dtype=np.float64), np.array(out_st, dtype=np.float64).reshape(len(out_s), -1),
            np.array(out_m, dtype=np.uint32).reshape(len(out_s), -1))
