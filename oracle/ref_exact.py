"""CPU ORACLE (test infrastructure — NOT product code): the list schedule in EXACT arithmetic.

The rule of `oracle/ref_release.py` (ref_eval's list schedule with release dates, and every score fold), computed
with `fractions.Fraction` instead of floating point:

    sel   = k slots of the job's node with smallest (ready, slot)      (ties -> lowest slot)
    start = max(max(ready[sel]), r_j)            (r_j -> ceil(r_j) with integer starts)
    ready[sel] = start + (integer_starts ? ceil(rt) : rt)
    e = start + rt
    makespan             mk  = max(mk, e)
    completion           acc = acc + e
    weighted_completion  acc = acc + w e
    (weighted) tardiness acc = acc + w max(e - d, 0)

On an input where fp32 rounds nothing, every floating-point restatement (the fp32 and float64 oracles, the
kernels) must reproduce this value for value.  `schedule(..., exact32=True)` asserts that: every input and every
intermediate it forms (starts, slot times, completions, e - d, products, partial sums) must be exactly representable
in fp32, so an input that breaks exactness fails loudly instead of weakening a comparison.  +inf (an absent or
selected sentinel cell) is carried as float('inf'); it is exact.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

NSLOT = 8
OBJECTIVES = ("makespan", "completion", "weighted_completion", "tardiness", "weighted_tardiness")
INF = float("inf")


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
    if objective not in OBJECTIVES:
        raise ValueError("objective must be one of %s" % (OBJECTIVES,))
    J = len(prio)
    chk = _check if exact32 else (lambda x, what: x)
    r = [Fraction(0)] * J if release is None else [_q(x) for x in release]
    if integer_starts:
        r = [_ceil(x) for x in r]
    w = [Fraction(1)] * J if weights is None else [_q(x) for x in weights]
    tardy = objective.endswith("tardiness")
    if tardy and due is None:
        raise ValueError("objective=%r needs due dates" % objective)
    d = [_q(x) for x in due] if tardy else [Fraction(0)] * J
    for j in range(J):
        chk(r[j], "release[%d]" % j)
        chk(w[j], "weight[%d]" % j)
        chk(d[j], "due[%d]" % j)
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
        elif objective == "completion":
            acc = chk(acc + e, "partial sum at job %d" % j)
        elif objective == "weighted_completion":
            acc = chk(acc + chk(w[j] * e, "w e of job %d" % j), "partial sum at job %d" % j)
        else:
            late = max(chk(e - d[j], "e - d of job %d" % j), Fraction(0))
            acc = chk(acc + chk(w[j] * late, "w t of job %d" % j), "partial sum at job %d" % j)
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
