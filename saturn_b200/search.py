"""Search driver: rounds of device-side Metropolis search with one MIN all-reduce per round.

This is the host loop around the C ABI's sb_search_* calls.  With `torch.distributed`
initialised (one process per GPU, NCCL) the population is sharded by global chain id: rank r
owns chains [r*chains, (r+1)*chains); after every round the ranks exchange ONE packed
uint64 — (fp32 makespan bits << 32) | global chain id — with all_reduce(MIN), which is an
arg-min because non-negative floats order like their bit patterns (SURVEY §8e).  The winning
encoding is broadcast from its owner when the search ends (and when elites are re-seeded).
There is no reference counterpart: the reference solver is a single-process CPU MILP.
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .engine import Engine, objective_flag, objective_spec


@dataclass
class SearchResult:
    opt: np.ndarray
    prio: np.ndarray
    makespan: float
    evaluated: int          # candidates scored by all ranks
    rounds: int
    wall_s: float
    history: List[Tuple[float, int, float]] = field(default_factory=list)  # (wall s, evaluated, best makespan)
    owner_rank: int = 0
    stop_reason: int = 0    # as sb_search_result: 0 rounds, 1 time budget, 2 patience, 3 target (or tardiness 0)


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


def key_makespan(key: int) -> float:
    return float(np.array([(key >> 32) & 0xffffffff], dtype=np.uint32).view(np.float32)[0])


def lpt_seeds(tmin: np.ndarray, sentinel: float = 1.0e6, nodes: int = 1, objective: str = "makespan",
              weights: Optional[np.ndarray] = None, due: Optional[np.ndarray] = None,
              release: Optional[np.ndarray] = None, integer_starts: bool = True):
    """Heuristic warm candidates in the reduced encoding (opt byte = k-1, plus node << 3 when there
    are several nodes), longest-processing-time order: (a) every job on its fastest option,
    (b) every job on its least GPU-seconds option, (c) in between.  Nodes are filled greedily by
    accumulated GPU-seconds.  objective="completion": shortest-processing-time order instead (ascending
    runtime of the chosen option), the order that favours the sum of completion times; same options and
    node fill (sb_search_seed_lpt plants the same seeds).  objective="weighted_completion" with the fp32 job
    `weights`: WSPT order (Smith's rule), ascending runtime / weight in float64, ties by job index — for unit
    weights exactly the shortest-processing-time order.  objective="tardiness" / "weighted_tardiness" with the fp32
    `due` dates: EDD order (earliest due date first), ties by runtime (by runtime / weight when weighted), then by
    job index; objective="max_lateness" the unit-weight EDD order of "tardiness" (Jackson's rule, optimal for the
    maximum lateness on one machine).  With the fp32 `release` dates (any objective) each order is then re-sorted stably by ascending
    release date (ceiled when `integer_starts`, as the device schedules them), so jobs released together keep the
    objective's order.  objective="late_tasks" / "weighted_late_tasks": the EDD orders of "tardiness" /
    "weighted_tardiness", each repaired by Moore-Hodgson's rule after the node fill (moore_hodgson).
    objective="max_tardiness" / "weighted_max_tardiness", "squared_tardiness" / "weighted_squared_tardiness" and
    "late_penalty" / "weighted_late_penalty": the EDD orders of "tardiness" / "weighted_tardiness" unchanged.
    objective="completion_penalty" / "weighted_completion_penalty": the orders of "completion" /
    "weighted_completion" (SPT / WSPT), not EDD: the due dates there are a barrier on the completion time."""
    spec = objective_spec(objective)
    if spec.weighted:
        if weights is None:
            raise ValueError("objective=%r needs the job weights" % objective)
        w64 = np.asarray(weights, dtype=np.float32).astype(np.float64)
    late = bool(spec.flags & _lib.FLAG_LATE_COUNT)
    completion_penalty = bool(spec.flags & _lib.FLAG_COMPLETION_PENALTY)
    edd = spec.due and not completion_penalty
    if edd:
        if due is None:
            raise ValueError("objective=%r needs the job due dates" % objective)
        d32 = np.asarray(due, dtype=np.float32)
    if release is not None:
        rel = np.asarray(release, dtype=np.float32)
        if integer_starts:
            rel = np.ceil(rel)
    J = tmin.shape[0]
    # the cells the search proposes: those below the sentinel, and for a job without one only its cheapest finite
    # cell (the first minimum; column 0 when it has none)
    usable = np.where(tmin < sentinel, tmin, np.inf)
    bare = ~(tmin < sentinel).any(axis=1)
    cheapest = np.argmin(tmin, axis=1)
    usable[bare, cheapest[bare]] = tmin[bare, cheapest[bare]]
    k = np.arange(1, 9, dtype=np.float64)[None, :]
    seeds = []
    for area_weight in (0.0, 1.0, 0.5):
        cost = usable.astype(np.float64) * (k ** area_weight)
        col = np.argmin(cost, axis=1)
        rt = usable[np.arange(J), col]
        if edd:
            tie = rt.astype(np.float64) / w64 if spec.weighted else rt.astype(np.float64)
            order = np.lexsort((np.arange(J), tie, d32))
        elif objective in ("weighted_completion", "weighted_completion_penalty"):
            order = np.argsort(rt.astype(np.float64) / w64, kind="stable")
        elif objective in ("completion", "completion_penalty"):
            order = np.argsort(rt, kind="stable")
        else:
            order = np.argsort(-rt * (col + 1) ** 0.5, kind="stable")
        if release is not None:
            order = order[np.argsort(rel[order], kind="stable")]
        ob = col.astype(np.uint8)
        if nodes > 1:
            load = np.zeros(nodes)
            ob = ob.copy()
            for j in order:
                n = int(np.argmin(load))
                load[n] += float(rt[j]) * (int(col[j]) + 1)
                ob[j] |= n << 3
        if late:
            order = moore_hodgson(order, col, rt, ob >> 3 if nodes > 1 else np.zeros(J, dtype=np.int64), nodes,
                                  w64 if spec.weighted else None, d32,
                                  rel if release is not None else None, integer_starts)
        seeds.append((ob, order))
    return seeds


def moore_hodgson(order, col, rt, node, nodes, weights, due, release, integer_starts):
    """Moore-Hodgson's repair of a seed order for the late count (sb_search_seed_lpt's rule, decision for decision).
    The on-time sequence, at first `order`, is list-scheduled in float64 on the fp32 inputs by the device's rule: job j
    takes the k = col[j] + 1 slots of node[j] that are free first, starts when the k-th is free (and not before its
    release), holds them for rt[j] (ceil(rt[j]) with `integer_starts`) and completes at start + rt[j].  At the first
    job that completes after its due date, the job with the largest k * rt / w among it and the jobs before it (the
    later one on ties) moves to a late list, and the schedule resumes from that job's position, until no job of the
    sequence is late.  Returns the on-time sequence followed by the late list in `order`'s order.  With one gang size,
    one node and unit weights this is Moore-Hodgson's algorithm (a minimum number of late jobs)."""
    k = [int(c) + 1 for c in col]
    rt64 = [float(x) for x in rt]
    hold = [math.ceil(x) if integer_starts and math.isfinite(x) else x for x in rt64]
    d64 = [float(x) for x in due]
    r64 = [float(x) for x in release] if release is not None else None
    w = [float(x) for x in weights] if weights is not None else [1.0] * len(rt64)
    ratio = [k[j] * rt64[j] / w[j] for j in range(len(rt64))]
    nd = [int(x) for x in node]
    seq = [int(j) for j in order]
    pos = {j: q for q, j in enumerate(seq)}
    snap = [[[0.0] * 8 for _ in range(nodes)]]  # snap[q]: the slots' free times (ascending per node) before position q
    late = []
    q = 0
    while q < len(seq):
        j = seq[q]
        state = [list(f) for f in snap[q]]
        f = state[nd[j]]
        st = f[k[j] - 1]
        if r64 is not None:
            st = max(st, r64[j])
        v = st + hold[j]
        f[:k[j]] = [v] * k[j]
        f.sort()
        del snap[q + 1:]
        snap.append(state)
        if st + rt64[j] > d64[j]:
            out, best = 0, -math.inf
            for p in range(q + 1):
                if ratio[seq[p]] >= best:
                    out, best = p, ratio[seq[p]]
            late.append(seq.pop(out))
            q = out
            continue
        q += 1
    if not late:
        return np.asarray(order)
    late.sort(key=pos.__getitem__)
    return np.asarray(seq + late, dtype=np.asarray(order).dtype)


def run_search(engine: Engine, chains: int = 1 << 16, rounds: int = 200, seed: int = 0,
               integer_starts: bool = True, reduced: bool = False, time_budget_s: Optional[float] = None,
               patience: Optional[int] = None, t_start: float = 5e-4, t_end: float = 1e-6,
               warm: Optional[Tuple[np.ndarray, np.ndarray]] = None, use_dist: bool = True,
               target_makespan: Optional[float] = None, reseed_every: int = 0, resample_every: Optional[int] = None,
               record_history: bool = False, heuristic_seeds: bool = True,
               exchange_every: int = 16, _no_fused: bool = False, _python_driver: bool = False,
               _extra_flags: int = 0, objective: str = "makespan") -> SearchResult:
    """Run the search on `engine` (table already set).  Returns the best candidate found by any rank.
    objective="completion" minimises the sum of completion times; the result's `makespan`, the history and
    `target_makespan` then hold / target that sum.  objective="weighted_completion" minimises the sum weighted by
    the engine's set_weights.  objective="tardiness" / "weighted_tardiness" minimises the total (weighted) tardiness
    against the engine's set_due, and stops as soon as the incumbent's tardiness is 0, which no plan can beat.
    objective="max_lateness" minimises the maximum lateness against the engine's set_due; every score holds
    L_max + engine.due_shift, and there is no stop at zero (L_max has no floor).  objective="late_tasks" /
    "weighted_late_tasks" minimises the (weighted) number of tasks that complete after their due date, and stops at
    0 like the tardiness.  objective="max_tardiness" / "weighted_max_tardiness" minimises the largest (weighted)
    tardiness, and stops at 0 like the tardiness.  objective="squared_tardiness" / "weighted_squared_tardiness"
    minimises the (weighted) sum of squared tardiness, and stops at 0 like the tardiness.  objective="late_penalty" /
    "weighted_late_penalty" minimises the engine's set_penalty penalty plus the (weighted) tardiness of every late
    task, and stops at 0 like the tardiness.  objective="completion_penalty" / "weighted_completion_penalty" minimises
    the (weighted) sum of completion times plus the set_penalty penalty of every late task, with no stop at 0 (the
    score of a non-empty plan is > 0).

    `rounds` device rounds are issued in groups of `exchange_every` (tournament resampling every
    `resample_every` rounds inside a group is only another launch); after each group the ranks exchange
    their best key (one MIN) and the stopping rules are evaluated, so the host synchronises once per
    group rather than once per round."""
    objective_flag(objective)
    if resample_every is None:
        resample_every = -1          # the library's choice: 2 inside the tile kernel, 4 where it costs a copy
    dist = _dist() if use_dist else None
    if dist is None and not reseed_every and not _python_driver and hasattr(engine, "search_run"):
        # one process, one GPU: the same loop runs inside the library (sb_search_run)
        r = engine.search_run(chains, rounds, seed=seed, integer_starts=integer_starts, reduced=reduced,
                              t_start=t_start, t_end=t_end, warm=warm, resample_every=resample_every,
                              sync_every=exchange_every, patience=patience or 0, time_budget_s=time_budget_s or 0.0,
                              target_makespan=target_makespan or 0.0, heuristic_seeds=heuristic_seeds,
                              record_history=record_history, _no_fused=_no_fused, _extra_flags=_extra_flags,
                              **({"objective": objective} if objective != "makespan" else {}))
        return SearchResult(opt=r["opt"], prio=r["prio"], makespan=r["makespan"], evaluated=r["evaluated"],
                            rounds=r["rounds"], wall_s=r["wall_s"], history=r["history"], owner_rank=0,
                            stop_reason=r["stop_reason"])
    rank = dist.get_rank() if dist else 0
    world = dist.get_world_size() if dist else 1
    J = engine.J
    pdt = np.uint8 if J <= 256 else np.uint16
    t0 = time.perf_counter()
    engine.search_init(chains, seed=seed, chain_base=rank * chains, integer_starts=integer_starts,
                       reduced=reduced, t_start=t_start, t_end=t_end, total_rounds=max(rounds, 1), warm=warm,
                       resample_every=resample_every, **({"_no_fused": True} if _no_fused else {}),
                       **({"_extra_flags": _extra_flags} if _extra_flags else {}),
                       **({"objective": objective} if objective != "makespan" else {}))
    if heuristic_seeds:
        # every rank plants the longest-processing-time seeds in an eighth of its population each;
        # the rest stays random (diversity), tournament resampling then concentrates the population
        tmin, args = engine.reduced_table()
        per = max(1, chains // 8)
        nodes = getattr(engine, "nodes", 1)
        for i, (col, order) in enumerate(lpt_seeds(tmin, nodes=nodes, objective=objective,
                                                   weights=getattr(engine, "weights", None),
                                                   due=getattr(engine, "due", None),
                                                   release=getattr(engine, "release", None),
                                                   integer_starts=integer_starts)):
            opt = col if reduced else ((args[np.arange(J), col & 7].astype(np.uint8) << 3) | col)
            first = min(i * per, max(0, chains - per))
            engine.search_inject(opt.astype(np.uint8), order.astype(pdt), copies=min(per, chains), first=first)
    local_key = engine.search_best_key()          # aliases device memory
    KEY_MAX = 0x7fffffffffffffff
    gkey = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    history: List[Tuple[float, int, float]] = []
    best_seen = None
    stale = 0
    done_rounds = 0
    stop = torch.zeros(1, dtype=torch.int32, device=engine.device)

    if dist and not getattr(engine, "has_xchg", False) and hasattr(engine, "xchg_init") \
            and dist.get_backend() == "nccl":
        engine.xchg_init(dist)              # NVLink peer-memory mailboxes; collectively False -> NCCL on all ranks
    use_xchg = bool(dist) and getattr(engine, "has_xchg", False)

    def exchange() -> int:
        if use_xchg:
            # NVLink peer-memory MIN: every rank publishes its key in its own mailbox, a one-warp kernel
            # folds all mailboxes.  A wait that times out (a peer seconds late: a dead rank) leaves the
            # preset maximum in gkey and raises here — a loud failure, never a stale key as the owner id.
            gkey.fill_(KEY_MAX)
            engine.xchg_post(local_key)
            engine.xchg_reduce(gkey)
            engine.xchg_check()             # synchronises; raises SaturnB200Error on a timed-out wait
            k = int(gkey.item())
            if k == KEY_MAX:
                raise RuntimeError("peer exchange produced no key")
            return k
        engine.sync()
        gkey.copy_(local_key)
        if dist:
            dist.all_reduce(gkey, op=dist.ReduceOp.MIN)
        return int(gkey.item())

    key = exchange()
    best_seen = key
    if record_history:
        history.append((time.perf_counter() - t0, chains * world, key_makespan(key)))
    exchange_every = max(1, int(exchange_every))
    # a tardiness, late count or maximum tardiness (the SB_FLAG_DUE forms) of +0 (key bits 0) cannot be beaten; the
    # completion penalty, also an SB_FLAG_DUE form, counts every completion time and never reaches +0
    flags = objective_flag(objective)
    at_zero = bool(flags & _lib.FLAG_DUE) and not (flags & _lib.FLAG_COMPLETION_PENALTY)
    reason = 3 if at_zero and (best_seen >> 32) == 0 else 0
    while reason == 0 and done_rounds < rounds:
        # one group of rounds, no host synchronisation; the library resamples on its own cadence
        step = min(exchange_every, rounds - done_rounds)
        engine.search_round(step)
        done_rounds += step
        r = done_rounds - 1
        key = exchange()
        if key < best_seen:
            best_seen = key
            stale = 0
        else:
            stale += step
        if record_history:
            history.append((time.perf_counter() - t0, chains * world * (done_rounds + 1), key_makespan(key)))
        # stopping decisions must be identical on every rank: derive them from rank 0's clock
        want_stop = 0
        if time_budget_s is not None and time.perf_counter() - t0 > time_budget_s:
            want_stop = 1
        elif patience is not None and stale >= patience:
            want_stop = 2
        elif target_makespan is not None and key_makespan(best_seen) <= target_makespan:
            want_stop = 3
        elif at_zero and (best_seen >> 32) == 0:
            want_stop = 3
        if dist:
            stop.fill_(want_stop)
            dist.broadcast(stop, src=0)
            want_stop = int(stop.item())
        if want_stop:
            reason = want_stop
            break
        if reseed_every and (r + 1) % reseed_every == 0 and r + 1 < rounds:
            opt, prio = _gather_best(engine, best_seen, chains, dist, rank)
            engine.search_inject(opt, prio, copies=max(1, chains // 64), first=-1)
    opt, prio = _gather_best(engine, best_seen, chains, dist, rank)
    ev, _ = engine.search_stats()
    total_ev = ev
    if dist:
        evt = torch.tensor([ev], dtype=torch.int64, device=engine.device)
        dist.all_reduce(evt, op=dist.ReduceOp.SUM)
        total_ev = int(evt.item())
    return SearchResult(opt=opt, prio=prio, makespan=key_makespan(best_seen), evaluated=total_ev,
                        rounds=done_rounds, wall_s=time.perf_counter() - t0, history=history,
                        owner_rank=int((best_seen & 0xffffffff) // chains) if world > 1 else 0, stop_reason=reason)


def _gather_best(engine: Engine, key: int, chains: int, dist, rank: int):
    """Fetch the encoding that produced `key` from the rank that owns it."""
    J = engine.J
    opt, prio, _mk, lkey = engine.search_best()
    if dist is None:
        return opt, prio
    owner = int((key & 0xffffffff) // chains)
    dev = engine.device
    pdt = torch.uint8 if J <= 256 else torch.int32
    o = torch.from_numpy(opt.copy()).to(dev)
    p = torch.from_numpy(prio.astype(np.int32) if J > 256 else prio.copy()).to(dev).to(pdt)
    dist.broadcast(o, src=owner)
    dist.broadcast(p, src=owner)
    return o.cpu().numpy().astype(np.uint8), p.cpu().numpy().astype(np.uint8 if J <= 256 else np.uint16)
