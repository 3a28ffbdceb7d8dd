"""CPU ORACLE (test infrastructure — NOT product code): the WORST and MEAN total (weighted) TARDINESS of list schedules
over runtime scenarios, and with every due date 0 the worst and mean (weighted) COMPLETION time.

A scenario k is the table of `oracle/ref_scenarios.py`, T_k[j][c] = fl32(f[k][j] * T[j][c]).  A candidate (opt, prio)
keeps its options and its order in every scenario; its score S_k on scenario k is the tardiness fold of
`oracle/ref_release.py` re-run on T_k (release dates optional, several nodes allowed):

    S_k = acc = acc + fl(w_j * max(fl(C_jk - d_j), 0)), in schedule order from +0 (each add rounded in `dtype`)

with unit weights for the unweighted forms.  The two scores (SB_FLAG_WORST_TARDINESS, SB_FLAG_MEAN_TARDINESS):

    worst = max_k S_k                          (an exact max)
    mean  = acc = acc + S_k, k = 0 .. K-1      (a left fold from +0, each add rounded in `dtype`: K times the mean)

"worst_tardiness" is the largest TOTAL tardiness over the scenarios, not the per-job maximum tardiness.  Every
completion is >= +0, so with d = 0 the term is w_j * C_jk bit for bit and the scores are the worst and mean (weighted)
completion time ("worst_completion", "mean_completion"); with K = 1 and f = 1 they are ref_release's tardiness (or
completion) fold.

Here:
  * `totals` — S[B][K] of B candidates on the fp32 scenario tables (the device's tables), by ref_release's C port
    in `dtype` arithmetic (float32: the device's rule; float64: the same tables scheduled in float64);
  * `fold` — the two scores from S[B][K] in `dtype`;
  * `evaluate` — totals + fold;
  * `c_evaluate` — the fp32 rule in plain C (`oracle/ref_scenario_tardiness.c`, a library of its own): tables,
    schedules and both folds in one pass, for parity checks at 1e5 candidates;
  * `brute_force` — the exhaustive list-schedule optimum of either score (J <= ~6).
"""
from __future__ import annotations

import ctypes
import itertools
import os
import subprocess
from typing import Sequence

import numpy as np

from . import ref_release as RR
from .ref_scenarios import factors_as, scale_tables

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_scenario_tardiness.so")
_lib = None
# the scores, and what each folds per scenario: the tardiness forms, and the completion forms (d = 0)
OBJECTIVES = ("worst_tardiness", "mean_tardiness", "worst_completion", "mean_completion")


def _due(due, J, objective):
    if objective.endswith("completion"):
        assert due is None, "the completion forms take no due dates"
        return np.zeros(J)
    assert due is not None, "objective=%r needs due dates" % objective
    return np.asarray(due, dtype=np.float64)


def totals(tab, opt, prio, factors, due=None, weights=None, release=None, integer_starts=True, dtype=np.float32,
           nodes=1, objective="worst_tardiness") -> np.ndarray:
    """S[B][K]: each candidate's total (weighted) tardiness on every scenario table (ref_release's C port in `dtype`
    arithmetic; d = 0 for the completion forms)."""
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    B, J = opt.shape
    tabs = scale_tables(tab, factors, np.float32)
    rel = np.zeros(J) if release is None else release
    d = _due(due, J, objective)
    form = "tardiness" if weights is None else "weighted_tardiness"
    S = np.empty((B, tabs.shape[0]), dtype=dtype)
    for k in range(tabs.shape[0]):
        S[:, k] = RR.c_evaluate(tabs[k], opt, prio, rel, integer_starts, dtype, threads=os.cpu_count() or 1,
                                nodes=nodes, objective=form, weights=weights, due=d)
    return S


def fold(S, objective, dtype=np.float32) -> np.ndarray:
    """score[B] from S[B][K]: the max, or the left fold acc + S_k from +0 in scenario order (each add in `dtype`)."""
    S = np.asarray(S, dtype=dtype)
    assert objective in OBJECTIVES, objective
    if objective.startswith("worst"):
        return S.max(axis=1).astype(dtype)
    acc = np.zeros(S.shape[0], dtype=dtype)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(S.shape[1]):
            acc = (acc + S[:, k]).astype(dtype)
    return acc


def evaluate(tab, opt, prio, factors, objective, due=None, weights=None, release=None, integer_starts=True,
             dtype=np.float32, nodes=1, want_totals=False):
    """score[B] (and S[B][K] with want_totals)."""
    S = totals(tab, opt, prio, factors, due, weights, release, integer_starts, dtype, nodes, objective)
    s = fold(S, objective, dtype)
    return (s, S) if want_totals else s


def _candidates(valid_opts, nodes):
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    return np.repeat(opts, len(perms), axis=0), np.tile(perms, (len(opts), 1))


def brute_force(tab, valid_opts: Sequence[Sequence[int]], factors, objective, due=None, weights=None, release=None,
                integer_starts=True, dtype=np.float32, nodes=1):
    """Exhaustive minimum of the score over every (option vector, permutation) candidate, the first minimum in the
    enumeration order of ref_release.brute_force.  Returns (score, opt, prio, S_k of the optimum)."""
    opt, prio = _candidates(valid_opts, nodes)
    s, S = evaluate(tab, opt, prio, factors, objective, due, weights, release, integer_starts, dtype, nodes,
                    want_totals=True)
    i = int(np.argmin(s))
    return float(s[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i]), [float(x) for x in S[i]]


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_scenario_tardiness.c")
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
        fn = _lib.ref_scenario_tardiness_f32
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                       ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, factors, objective, due=None, weights=None, release=None, integer_starts=True, nodes=1,
               threads=0):
    """The fp32 rule in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, factors[K][J] -> (score[B], S[B][K])."""
    tab = np.ascontiguousarray(tab, dtype=np.float32)
    J, S_, W = tab.shape
    assert W == 8
    f = np.ascontiguousarray(factors_as(factors, np.float32))
    K = f.shape[0]
    assert f.shape == (K, J)
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    assert prio.dtype in (np.uint8, np.uint16)
    B = opt.shape[0]
    assert opt.shape == (B, J) and prio.shape == (B, J)
    r = np.ascontiguousarray(RR.release_as(np.zeros(J) if release is None else release, J, np.float32,
                                           integer_starts))
    w = np.ascontiguousarray(np.ones(J, dtype=np.float32) if weights is None
                             else np.asarray(weights, dtype=np.float64).astype(np.float32))
    d = np.ascontiguousarray(_due(due, J, objective).astype(np.float32))
    score = np.empty(B, dtype=np.float32)
    S = np.empty((B, K), dtype=np.float32)
    rc = _load().ref_scenario_tardiness_f32(tab.ctypes.data, J, S_, f.ctypes.data, K, opt.ctypes.data,
                                            prio.ctypes.data, prio.dtype.itemsize, B, int(bool(integer_starts)),
                                            int(nodes), r.ctypes.data, w.ctypes.data, d.ctypes.data,
                                            0 if objective.startswith("worst") else 1, score.ctypes.data,
                                            S.ctypes.data, int(threads or os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError("ref_scenario_tardiness rc=%d" % rc)
    return score, S
