"""CPU ORACLE (test infrastructure — NOT product code): the WORST and MEAN MAKESPAN of list schedules over runtime
scenarios.

A scenario k is one alternative runtime table: every cell of job j's row is multiplied by one factor f[k][j] > 0,

    T_k[j][c] = fl(f[k][j] * T[j][c])          (one product, rounded to nearest in `dtype`; +inf stays +inf)

A candidate (opt, prio) keeps its options and its order in every scenario; its makespan M_k on scenario k is the list
schedule of `oracle/ref_release.py` (release dates optional, several nodes allowed) re-run on T_k, so gang
placements and starts may differ between scenarios.  The two scores (SB_FLAG_WORST_MAKESPAN, SB_FLAG_MEAN_MAKESPAN):

    worst = max_k M_k                          (an exact max)
    mean  = acc = acc + M_k, k = 0 .. K-1      (a left fold from +0, each add rounded in `dtype`: K times the mean)

Both are >= +0.  With K = 1 and f = 1, T_0 = T bit for bit, and both scores are ref_eval's makespan.

Here:
  * `scale_tables` — the K scenario tables;
  * `makespans` — M[B][K] of B candidates on the fp32 scenario tables (the device's tables), by ref_release's C port
    in `dtype` arithmetic (float32: the device's rule; float64: the same tables scheduled in float64);
  * `fold` — the two scores from M[B][K] in `dtype`;
  * `evaluate` — makespans + fold;
  * `c_evaluate` — the fp32 fold in plain C (`oracle/ref_scenarios.c`, a library of its own): tables, schedules and
    fold in one pass, for parity checks at 1e5 candidates;
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

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libref_scenarios.so")
_lib = None
OBJECTIVES = ("worst_makespan", "mean_makespan")


def factors_as(factors, dtype=np.float32) -> np.ndarray:
    """The factors [K][J] in `dtype`; asserts 1 <= K <= 8 and every factor finite and > 0."""
    f = np.asarray(factors, dtype=np.float64)
    assert f.ndim == 2 and 1 <= f.shape[0] <= 8, f.shape
    assert np.isfinite(f).all() and (f > 0).all()
    return f.astype(dtype)


def scale_tables(tab, factors, dtype=np.float32) -> np.ndarray:
    """tab[J][S][8], factors[K][J] -> T[K][J][S][8], T[k][j] = fl(f[k][j] * tab[j]) in `dtype`."""
    t = np.asarray(tab, dtype=dtype)
    f = factors_as(factors, dtype)
    assert f.shape[1] == t.shape[0]
    with np.errstate(over="ignore", invalid="ignore"):
        return (f[:, :, None, None] * t[None]).astype(dtype)


def makespans(tab, opt, prio, factors, release=None, integer_starts=True, dtype=np.float32, nodes=1) -> np.ndarray:
    """M[B][K]: each candidate's makespan on every scenario table (ref_release's C port, `dtype` arithmetic)."""
    opt = np.ascontiguousarray(opt, dtype=np.uint8)
    prio = np.ascontiguousarray(prio)
    B, J = opt.shape
    tabs = scale_tables(tab, factors, np.float32)
    rel = np.zeros(J) if release is None else release
    M = np.empty((B, tabs.shape[0]), dtype=dtype)
    for k in range(tabs.shape[0]):
        M[:, k] = RR.c_evaluate(tabs[k], opt, prio, rel, integer_starts, dtype, threads=os.cpu_count() or 1,
                                nodes=nodes, objective="makespan")
    return M


def fold(M, objective, dtype=np.float32) -> np.ndarray:
    """score[B] from M[B][K]: the max, or the left fold acc + M_k from +0 in scenario order (each add in `dtype`)."""
    M = np.asarray(M, dtype=dtype)
    if objective == "worst_makespan":
        return M.max(axis=1).astype(dtype)
    assert objective == "mean_makespan", objective
    acc = np.zeros(M.shape[0], dtype=dtype)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(M.shape[1]):
            acc = (acc + M[:, k]).astype(dtype)
    return acc


def evaluate(tab, opt, prio, factors, objective, release=None, integer_starts=True, dtype=np.float32, nodes=1,
             want_makespans=False):
    """score[B] (and M[B][K] with want_makespans)."""
    M = makespans(tab, opt, prio, factors, release, integer_starts, dtype, nodes)
    s = fold(M, objective, dtype)
    return (s, M) if want_makespans else s


def _candidates(valid_opts, nodes):
    J = len(valid_opts)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    opts = np.array(list(itertools.product(*valid_opts)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    return np.repeat(opts, len(perms), axis=0), np.tile(perms, (len(opts), 1))


def brute_force(tab, valid_opts: Sequence[Sequence[int]], factors, objective, release=None, integer_starts=True,
                dtype=np.float32, nodes=1):
    """Exhaustive minimum of the score over every (option vector, permutation) candidate, the first minimum in the
    enumeration order of ref_release.brute_force.  Returns (score, opt, prio)."""
    opt, prio = _candidates(valid_opts, nodes)
    s = evaluate(tab, opt, prio, factors, objective, release, integer_starts, dtype, nodes)
    i = int(np.argmin(s))
    return float(s[i]), tuple(int(x) for x in opt[i]), tuple(int(x) for x in prio[i])


# --------------------------------------------------------------------------- C port
def build(force=False):
    src = os.path.join(_HERE, "ref_scenarios.c")
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
        fn = _lib.ref_scenarios_f32
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                       ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                       ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return _lib


def c_evaluate(tab, opt, prio, factors, objective, release=None, integer_starts=True, nodes=1, threads=0):
    """The fp32 rule in C: tab[J][S][8], opt[B][J] u8, prio[B][J] u8/u16, factors[K][J] -> (score[B], M[B][K])."""
    tab = np.ascontiguousarray(tab, dtype=np.float32)
    J, S, W = tab.shape
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
    score = np.empty(B, dtype=np.float32)
    M = np.empty((B, K), dtype=np.float32)
    rc = _load().ref_scenarios_f32(tab.ctypes.data, J, S, f.ctypes.data, K, opt.ctypes.data, prio.ctypes.data,
                                   prio.dtype.itemsize, B, int(bool(integer_starts)), int(nodes), r.ctypes.data,
                                   OBJECTIVES.index(objective), score.ctypes.data, M.ctypes.data,
                                   int(threads or os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError("ref_scenarios rc=%d" % rc)
    return score, M
