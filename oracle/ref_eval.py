"""CPU ORACLE (test infrastructure — NOT product code).

Restatement of what a SPASE plan *is* according to the reference MILP
(`saturn/solver/milp.py`), as a list-scheduling evaluator over candidates
``(opt[J], prio[J])`` plus an independent checker of the reference's own
constraint set.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import this
module; the product (``saturn_b200``) never does.

Parity status: the reference ships no tests / golden vectors for this path
(SURVEY §4) — the oracle is pinned instead against outputs of the reference
itself, run unmodified in the build container on ``pulp``/``ray`` shims
(``oracle/gen_golden.py`` -> ``tests/golden/milp_*.json``), see DESIGN.md §3.

Reference semantics restated here (file:line under /root/reference):
  * input  = per task an ordered list of (gpu_count, runtime) options,
             dict-insertion order                      saturn/solver/milp.py:77-81
  * exactly one option per task                         milp.py:108-111
  * exactly one node per task                           milp.py:134-137
  * a task occupies exactly gpu_count GPUs of its node  milp.py:209-227
  * all occupied GPUs share ONE start, which is an
    Integer variable >= 0                               milp.py:139-149, 233-256
  * two tasks sharing a GPU do not overlap in time;
    boa[a][b] == 1  <=>  a runs before b                milp.py:263-319
  * makespan >= start + runtime(selected option)        milp.py:162-177
  * T semantics, min over executors, sentinels 1e6/1e8  saturn/trial_runner/PerformanceEvaluator.py:24-26,96-115

Canonical encodings shared with the CUDA path (include/saturn_b200.h):
  tab[J][S][8]   float   runtime of job j with strategy s on k = col+1 GPUs,
                         +inf where the option does not exist
  opt[j]         uint8   (s << 3) | (k - 1)
  prio[i]        uintN   job scheduled i-th (a permutation of 0..J-1)

List scheduling rule (one node of G <= 8 GPU slots):
  ready[0..G) = 0
  for i in 0..J-1:
      j = prio[i]; k = (opt[j] & 7) + 1; rt = tab[j][opt[j] >> 3][k - 1]
      sel   = the k slots with smallest (ready[slot], slot)   # ties -> lowest slot
      start = max(ready[sel])
      ready[sel] = start + (ceil(rt) if integer_starts else rt)
      completion[j] = start + rt
  makespan = max_j completion[j]

With ``integer_starts`` every start is an integer (the MILP's start variables
are ``cat="Integer"``, milp.py:142-143): a slot that finishes at a fractional
time becomes usable at the next integer, so the slot state can be kept as that
integer (start + ceil(rt)); the task's real completion start + rt is what the
makespan constraint milp.py:170-177 sees.
"""
from __future__ import annotations

import itertools
import math
from typing import List, Sequence, Tuple

import numpy as np

NSLOT = 8  # GPUs per node, hard-coded in the reference: milp.py:62
INF = float("inf")


# --------------------------------------------------------------------------- tables
def canon_table(T: np.ndarray, gcount: Sequence[int]) -> np.ndarray:
    """T[J][S][G] + gcount[G] -> canonical tab[J][S][8] (column = k-1, +inf if absent).

    If two input columns carry the same GPU count the smaller runtime is kept; on equal runtimes the earlier
    column's value, so -0.0 and +0.0 keep the sign of the first of them (as sb_set_table does).
    """
    T = np.asarray(T)
    J, S, G = T.shape
    tab = np.full((J, S, NSLOT), np.inf, dtype=T.dtype)
    for g in range(G):
        k = int(gcount[g])
        if not 1 <= k <= NSLOT:
            raise ValueError("gpu count %d outside 1..8" % k)
        tab[:, :, k - 1] = np.where(T[:, :, g] < tab[:, :, k - 1], T[:, :, g], tab[:, :, k - 1])
    return tab


def reduce_table(tab: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """min over the strategy axis, first (lowest s) minimum wins.

    Restates the per-(task, gpu_count) executor reduction of
    PerformanceEvaluator.py:101-115 (`if runtime < chosen_runtime` keeps the
    first executor that attains the minimum).
    """
    args = tab.argmin(axis=1).astype(np.uint8)  # numpy argmin returns first occurrence
    # the value of that strategy: a min() reduction may return either zero of a -0.0 / +0.0 tie
    tmin = np.take_along_axis(tab, args[:, None, :].astype(np.intp), axis=1)[:, 0, :]
    return tmin, args


def table_from_tuples(gpu_time_tuples) -> Tuple[np.ndarray, List[List[int]]]:
    """Reference solver input (milp.py:77-81) -> (tab[J][S][8] float64, optmap).

    Each task's options are (gpu_count, runtime) in dict order.  Several
    options with the same gpu_count land on successive strategy rows.
    optmap[j][o] is the canonical opt byte of the task's o-th option.
    """
    J = len(gpu_time_tuples)
    per_k_rows = []
    for tup in gpu_time_tuples:
        cnt = {}
        for (k, _rt) in tup:
            cnt[k] = cnt.get(k, 0) + 1
        per_k_rows.append(max(cnt.values()) if cnt else 1)
    S = max(per_k_rows) if per_k_rows else 1
    tab = np.full((J, S, NSLOT), np.inf, dtype=np.float64)
    optmap: List[List[int]] = []
    for j, tup in enumerate(gpu_time_tuples):
        used = {}
        row = []
        for (k, rt) in tup:
            s = used.get(k, 0)
            used[k] = s + 1
            tab[j, s, k - 1] = rt
            row.append((s << 3) | (k - 1))
        optmap.append(row)
    return tab, optmap


# --------------------------------------------------------------------------- evaluator
def list_schedule(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=NSLOT, nodes=1):
    """One candidate, pure Python loops.  Returns (makespan, start[J], mask[J], ready).

    `dtype` selects the arithmetic (np.float64 = exact restatement,
    np.float32 = the arithmetic of the CUDA path, bit-for-bit).

    nodes > 1 (multi-node, reference milp.py:117-137,209-227: a task runs on exactly ONE node and
    its gang takes GPUs of that node only): the table must be the reduced one (S = 1) and the opt
    byte reads (node << 3) | (k - 1); mask[j] = (node << 16) | gpu bitmask within the node; a node
    index >= nodes makes the candidate infeasible (inf).
    """
    f = dtype
    J = len(prio)
    if nodes > 1:
        return _list_schedule_nodes(tab, opt, prio, integer_starts, f, nslot, nodes)
    ready = [f(0.0)] * nslot
    start = [f(0.0)] * J
    mask = [0] * J
    mk = f(0.0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        k = (o & 7) + 1
        rt = f(tab[j][o >> 3][o & 7])
        if k > nslot:
            return float("inf"), start, mask, ready
        order = sorted(range(nslot), key=lambda g: (ready[g], g))
        sel = order[:k]
        s = ready[sel[-1]]
        hold = f(math.ceil(rt)) if (integer_starts and math.isfinite(rt)) else rt
        nxt = f(s + hold)
        m = 0
        for g in sel:
            ready[g] = nxt
            m |= 1 << g
        start[j] = s
        mask[j] = m
        c = f(s + rt)
        if c > mk:
            mk = c
    return float(mk), start, mask, ready


def _list_schedule_nodes(tab, opt, prio, integer_starts, f, nslot, nodes):
    J = len(prio)
    ready = [[f(0.0)] * nslot for _ in range(nodes)]
    start = [f(0.0)] * J
    mask = [0] * J
    mk = f(0.0)
    for i in range(J):
        j = int(prio[i])
        o = int(opt[j])
        k = (o & 7) + 1
        n = o >> 3
        rt = f(tab[j][0][o & 7])
        if k > nslot or n >= nodes:
            return float("inf"), start, mask, ready
        rd = ready[n]
        order = sorted(range(nslot), key=lambda g: (rd[g], g))
        sel = order[:k]
        s = rd[sel[-1]]
        hold = f(math.ceil(rt)) if (integer_starts and math.isfinite(rt)) else rt
        nxt = f(s + hold)
        m = 0
        for g in sel:
            rd[g] = nxt
            m |= 1 << g
        start[j] = s
        mask[j] = (n << 16) | m
        c = f(s + rt)
        if c > mk:
            mk = c
    return float(mk), start, mask, ready


def list_schedule_batch(tab, opt, prio, integer_starts=True, dtype=np.float64, nslot=NSLOT,
                        want_plan=False):
    """Vectorised over candidates (numpy).  opt[B][J] u8, prio[B][J] int.

    Returns makespan[B] (and start[B][J], mask[B][J] if want_plan).
    Same rule as `list_schedule`; a stable argsort gives the (ready, slot) order.
    """
    tab = np.asarray(tab).astype(dtype)
    opt = np.asarray(opt)
    prio = np.asarray(prio).astype(np.int64)
    B, J = prio.shape
    ar = np.arange(B)
    ready = np.zeros((B, nslot), dtype=dtype)
    mk = np.zeros(B, dtype=dtype)
    bad = np.zeros(B, dtype=bool)
    if want_plan:
        start = np.zeros((B, J), dtype=dtype)
        mask = np.zeros((B, J), dtype=np.uint32)
    bits = (1 << np.arange(nslot)).astype(np.uint32)
    for i in range(J):
        j = prio[:, i]
        o = opt[ar, j].astype(np.int64)
        km1 = o & 7
        rt = tab[j, o >> 3, km1]
        bad |= km1 >= nslot
        km1c = np.minimum(km1, nslot - 1)
        order = np.argsort(ready, axis=1, kind="stable")
        srt = np.take_along_axis(ready, order, axis=1)
        s = srt[ar, km1c]
        rank = np.empty_like(order)
        np.put_along_axis(rank, order, np.arange(nslot)[None, :].repeat(B, 0), axis=1)
        sel = rank <= km1c[:, None]
        with np.errstate(invalid="ignore"):
            hold = np.where(np.isfinite(rt), np.ceil(rt), rt).astype(dtype) if integer_starts else rt
            nxt = (s + hold).astype(dtype)
            comp = (s + rt).astype(dtype)
        ready = np.where(sel, nxt[:, None], ready)
        mk = np.maximum(mk, comp)
        if want_plan:
            start[ar, j] = s
            mask[ar, j] = (sel * bits[None, :]).sum(axis=1).astype(np.uint32)
    mk = np.where(bad, np.inf, mk)
    if want_plan:
        return mk, start, mask
    return mk


def brute_force(tab, valid_opts: Sequence[Sequence[int]], integer_starts=True, nslot=NSLOT,
                dtype=np.float64, nodes=1):
    """Exhaustive minimum over all (option vector, permutation) candidates (J <= ~6).
    With nodes > 1 every option byte (k - 1) is combined with every node index."""
    J = len(valid_opts)
    best = (INF, None, None)
    if nodes > 1:
        valid_opts = [[(n << 3) | (o & 7) for o in ops for n in range(nodes)] for ops in valid_opts]
    for ov in itertools.product(*valid_opts):
        for perm in itertools.permutations(range(J)):
            mk, _, _, _ = list_schedule(tab, ov, perm, integer_starts, dtype, nslot, nodes)
            if mk < best[0]:
                best = (mk, tuple(ov), tuple(perm))
    return best


# --------------------------------------------------------------------------- plan checkers
def check_plan(start, mask, rt, k, nslot=NSLOT, integer_starts=True, tol=1e-6):
    """Independent feasibility check of a plan given per task (start, slot mask, runtime, k).

    Restates milp.py constraints (ii) gang size :209-227, (iii) a single integer
    start :139-149/:233-256 and (iv) mutual exclusion :277-319 without reusing
    the scheduler above.  Returns (ok, n_overlaps, makespan).
    """
    J = len(start)
    ok = True
    for t in range(J):
        if bin(int(mask[t])).count("1") != int(k[t]):
            ok = False
        if int(mask[t]) >> nslot:
            ok = False
        if start[t] < -tol:
            ok = False
        if integer_starts and abs(start[t] - round(start[t])) > tol:
            ok = False
    overlaps = 0
    for a in range(J):
        for b in range(a + 1, J):
            if int(mask[a]) & int(mask[b]):
                a0, a1 = start[a], start[a] + rt[a]
                b0, b1 = start[b], start[b] + rt[b]
                if a0 < b1 - tol and b0 < a1 - tol:
                    overlaps += 1
    mk = max((start[t] + rt[t] for t in range(J)), default=0.0)
    return ok and overlaps == 0, overlaps, mk


def milp_constraints_hold(gpu_time_tuples, sta, tga, bss, bna, boa, makespan, tol=1e-6):
    """Evaluate the reference MILP's constraints literally on returned arrays.

    Arrays have the shapes `saturn.solver.solve` returns (milp.py:445):
    sta[N][G][J], tga[J][N][G], bss[J][S_t], bna[J][N], boa[J][J].
    Uses a *sound* big-M (sum of max runtimes + 1) in place of milp.py:163's 1e10
    (SURVEY §8c hazard O1).  Returns a list of violated-constraint strings (empty = feasible).
    """
    J = len(gpu_time_tuples)
    N = len(sta)
    viol = []
    M = sum(max(rt for (_k, rt) in tup) for tup in gpu_time_tuples) + 1.0 + max(
        (max(max(g) for g in n) for n in sta), default=0.0)
    M = max(M, 16.0)

    def rnd(x):
        return int(round(x))

    for t in range(J):
        if sum(rnd(x) for x in bss[t]) != 1:
            viol.append("one-strategy t=%d" % t)           # milp.py:110-111
        if sum(rnd(x) for x in bna[t]) != 1:
            viol.append("one-node t=%d" % t)               # milp.py:136-137
    for n in range(N):
        for g in range(len(sta[n])):
            for t in range(J):
                v = sta[n][g][t]
                if v < -tol or abs(v - round(v)) > tol:
                    viol.append("integer-start n=%d g=%d t=%d" % (n, g, t))   # milp.py:142-143
                for s_idx, (_k, rt) in enumerate(gpu_time_tuples[t]):
                    if makespan < v + rt - M * (1 - rnd(bss[t][s_idx])) - tol * max(1.0, abs(makespan)):
                        viol.append("makespan n=%d g=%d t=%d s=%d" % (n, g, t, s_idx))  # milp.py:170-177
    for t in range(J):
        for n in range(N):
            occ = sum(rnd(x) for x in tga[t][n])
            on = rnd(bna[t][n])
            for s_idx, (k, _rt) in enumerate(gpu_time_tuples[t]):
                if rnd(bss[t][s_idx]) == 1 and on == 1 and occ != k:
                    viol.append("gang-size t=%d n=%d" % (t, n))                # milp.py:221-224
            if on == 0 and occ != 0:
                viol.append("off-node t=%d n=%d" % (t, n))                     # milp.py:226-227
            # start consistency, milp.py:233-256
            if on == 1:
                for s_idx, (k, _rt) in enumerate(gpu_time_tuples[t]):
                    if rnd(bss[t][s_idx]) != 1:
                        continue
                    target = sum(sta[n][g][t] for g in range(len(sta[n]))) / k
                    for g in range(len(sta[n])):
                        if rnd(tga[t][n][g]) == 1 and abs(target - sta[n][g][t]) > tol * max(1.0, abs(target)):
                            viol.append("gang-start t=%d n=%d g=%d" % (t, n, g))
    # exclusion, milp.py:277-319
    for n in range(N):
        for g in range(len(sta[n])):
            for t in range(J):
                if rnd(tga[t][n][g]) != 1:
                    continue
                rt_t = [rt for s_idx, (_k, rt) in enumerate(gpu_time_tuples[t]) if rnd(bss[t][s_idx]) == 1][0]
                for tp in range(J):
                    if tp == t or rnd(tga[tp][n][g]) != 1:
                        continue
                    rt_p = [rt for s_idx, (_k, rt) in enumerate(gpu_time_tuples[tp]) if rnd(bss[tp][s_idx]) == 1][0]
                    b = boa[tp][t]
                    if b is None:
                        viol.append("boa-none t=%d tp=%d" % (t, tp))
                        continue
                    st, sp = sta[n][g][t], sta[n][g][tp]
                    eps = tol * max(1.0, abs(st), abs(sp))
                    if rnd(b) == 0 and not (st <= sp - rt_t + eps):      # t before tp, milp.py:304-306
                        viol.append("excl-before n=%d g=%d t=%d tp=%d" % (n, g, t, tp))
                    if rnd(b) == 1 and not (st >= sp + rt_p - eps):      # t after tp, milp.py:317-319
                        viol.append("excl-after n=%d g=%d t=%d tp=%d" % (n, g, t, tp))
    return viol


def plan_from_arrays(gpu_time_tuples, sta, tga, bss, bna):
    """Decode solver arrays into per-task (start, mask, rt, k, option index).

    Same reading of the arrays as the reference decoder milp.py:470-496
    (argmax of bna / bss, round(tga) == 1, start of the first blocked GPU).
    Single-node masks only (node index returned separately).
    """
    J = len(gpu_time_tuples)
    out = []
    for t in range(J):
        n = int(np.argmax(bna[t]))
        o = int(np.argmax(bss[t]))
        k, rt = gpu_time_tuples[t][o]
        gl = [g for g, v in enumerate(tga[t][n]) if round(v) == 1]
        m = 0
        for g in gl:
            m |= 1 << g
        st = sta[n][gl[0]][t] if gl else 0.0
        out.append((st, m, rt, k, o, n))
    return out


# --------------------------------------------------------------------------- synthetic inputs
def synth_table(J, S, G, seed=0, masked=True, dtype=np.float32):
    """Deterministic synthetic T[J][S][G] of SURVEY §8d / BASELINE.md §3.

    base_j ~ LogUniform(600, 36000) s; alpha ~ U(.55,.95); beta ~ U(1,1.5);
    T[j][s][g-1] = base_j*beta/g**alpha.  Mask: strategy 0 only at g=1, the
    others only at g>=2, 10% random failures at g<=2 -> sentinel 1e8
    (PerformanceEvaluator.py:106).  A job is never left without a valid cell.
    """
    rng = np.random.default_rng(seed)
    base = np.exp(rng.uniform(np.log(600.0), np.log(36000.0), size=J))
    alpha = rng.uniform(0.55, 0.95, size=(J, S))
    beta = rng.uniform(1.0, 1.5, size=(J, S))
    g = np.arange(1, G + 1, dtype=np.float64)
    T = base[:, None, None] * beta[:, :, None] / g[None, None, :] ** alpha[:, :, None]
    valid = np.ones((J, S, G), dtype=bool)
    if masked:
        if S > 1:
            valid[:, 0, 1:] = False
            valid[:, 1:, 0] = False
        oom = rng.uniform(size=(J, S, G)) < 0.10
        oom[:, :, 2:] = False
        valid &= ~oom
        for j in range(J):
            if not valid[j].any():
                valid[j, 0, 0] = True
    T = np.where(valid, T, 1e8)
    return T.astype(dtype), valid


def synth_candidates(J, B, valid, seed=0, gcount=None):
    """opt[B][J] ~ U{valid options of j} in canonical bytes, prio[B] = random permutations."""
    rng = np.random.default_rng(seed)
    _, S, G = valid.shape
    if gcount is None:
        gcount = list(range(1, G + 1))
    opt = np.zeros((B, J), dtype=np.uint8)
    for j in range(J):
        cells = [(s << 3) | (int(gcount[g]) - 1) for s in range(S) for g in range(G) if valid[j, s, g]]
        cells = np.asarray(cells, dtype=np.uint8)
        opt[:, j] = cells[rng.integers(0, len(cells), size=B)]
    keys = rng.random((B, J))
    prio = np.argsort(keys, axis=1)
    prio = prio.astype(np.uint8 if J <= 256 else np.uint16)
    return opt, prio
