"""`saturn.solver` drop-in: solve() and convert_into_comprehensible().

Same call shapes, argument meaning and return structure as the reference
(saturn/solver/milp.py:23 and :448, re-exported by saturn/solver/__init__.py:1-2), so
`saturn.orchestrate` (orchestrator.py:21-23,55-61,69-75) and user code keep working:

    sta, tga, bss, bna, boa, makespan = solve(task_list, presolved, gurobi=..., threads=...,
                                               interval=..., timeout=...)
    node_per_task, task_dependency_dict, start_times = convert_into_comprehensible(
        task_list, bss, boa, tga, bna, sta)

Instead of building the MILP of milp.py:96-319 and shelling out to Gurobi/CBC (milp.py:321-327),
solve() uploads the (gpu_count, runtime) table the MILP would have been built from
(milp.py:77-81), searches list-schedule candidates on the GPU (saturn_b200.search) and emits the
winner in exactly the nested-list layout milp.py:330-352,445 returns.  `gurobi` and `threads` are
accepted and ignored.  `timeout` bounds the wall-clock of the search, as it bounded the MILP.

There is no CPU fallback: without the CUDA library / a GPU this raises.
"""
from __future__ import annotations

import math
import os
import time
from collections import defaultdict
from collections.abc import Mapping
from typing import List, NamedTuple, Optional, Sequence

import numpy as np

NSLOT = 8            # GPUs per node, reference milp.py:62 (DEBUG = True -> 8 per node)
REPLAN_THRESHOLD = 500.0   # milp.py:363


class SolverError(RuntimeError):
    pass


# ------------------------------------------------------------------------------------------ inputs
def gpu_time_tuples_of(task_list) -> List[List[tuple]]:
    """[(gpu_count, runtime), ...] per task in dict-insertion order — milp.py:77-81."""
    out = []
    for task in task_list:
        out.append([(g_count, strat.runtime) for g_count, strat in task.strategies.items()])
    return out


def build_table(task_list):
    """Task.strategies -> (T[J][1][8] fp32 by gpu_count column, usable[J][8], optindex[J][8]).

    optindex[j][k-1] = position of the gpu_count-k option in task j's strategies dict (the index
    `bss` is expressed in, milp.py:96-111,477-486), -1 if the task has no such option.
    Options that cannot fit one node (gpu_count > 8, milp.py:62,209-227) are dropped; options whose
    executor is None are the profiler's sentinels (PerformanceEvaluator.py:99,106) and are kept in
    the table but never proposed unless a task has nothing else.
    """
    J = len(task_list)
    # one pass over the Python objects collecting plain lists (comprehensions: this loop is the host-side cost
    # of a solve at J = 256), the filtering and the arithmetic are vectorised below
    counts = [len(task.strategies) for task in task_list]
    if 0 in counts:
        j = counts.index(0)
        raise SolverError("task %r has no strategies; run the trial runner first" % getattr(task_list[j], "name", j))
    keys = [g for task in task_list for g in task.strategies]
    strats = [st for task in task_list for st in task.strategies.values()]
    rts = [st.runtime for st in strats]
    jj_all = np.repeat(np.arange(J), counts)
    oo_all = np.concatenate([np.arange(c) for c in counts]) if J else np.zeros(0, dtype=np.int64)
    uu_all = np.fromiter((getattr(st, "executor", True) is not None for st in strats), dtype=bool, count=len(strats))
    ok_key = np.fromiter((isinstance(g, (int, np.integer)) and 1 <= g <= NSLOT for g in keys), dtype=bool, count=len(keys))
    r_all = np.array([np.nan if r is None else r for r in rts], dtype=np.float64)
    r_all = np.where((r_all < 0) & (r_all >= -1e-6), 0.0, r_all)   # forecast's in-place decrements (executor.py:166-168) can undershoot by an ulp
    ok = ok_key & np.isfinite(r_all) & (r_all >= 0)
    jj, oo, rr, uu = jj_all[ok], oo_all[ok], r_all[ok], uu_all[ok]
    kk = np.array([int(g) - 1 for g, k in zip(keys, ok) if k], dtype=np.int64)
    T = np.full((J, 1, NSLOT), np.inf, dtype=np.float32)
    optindex = np.full((J, NSLOT), -1, dtype=np.int64)
    usable = np.zeros((J, NSLOT), dtype=bool)
    if len(jj):
        r64 = np.asarray(rr, dtype=np.float64)
        v = r64.astype(np.float32)                                   # smallest fp32 >= rt: the device's start + ceil(rt)
        low = v.astype(np.float64) < r64
        v[low] = np.nextafter(v[low], np.float32(np.inf))
        # dict keys are unique, so a (task, gpu_count) cell is written at most once; keep the first of the
        # smallest anyway (e.g. the keys 2 and numpy.int64(2) of a hand-built dict)
        order = np.lexsort((oo, v, kk, jj))
        first = np.ones(len(order), dtype=bool)
        first[1:] = (jj[order][1:] != jj[order][:-1]) | (kk[order][1:] != kk[order][:-1])
        sel = order[first]
        T[jj[sel], 0, kk[sel]] = v[sel]
        optindex[jj[sel], kk[sel]] = oo[sel]
        usable[jj[sel], kk[sel]] = uu[sel]
    none = ~np.isfinite(T[:, 0, :]).any(axis=1)
    if none.any():
        j = int(np.argmax(none))
        raise SolverError("task %r has no option that fits a node of %d GPUs" % (getattr(task_list[j], "name", j), NSLOT))
    return T, usable, optindex


# ------------------------------------------------------------------------------------------ outputs
def plan_to_arrays(n_options: Sequence[int], opt_index: Sequence[int], start: Sequence[float],
                   slotmask: Sequence[int], position: Sequence[int], nodes: int = 1,
                   node_of: Optional[Sequence[int]] = None):
    """(start, GPU mask, chosen option, schedule position) per task -> the reference's arrays.

    Layout and meaning follow milp.py:330-352: sta[N][G][J] start times (0 where the task does
    not run), tga[J][N][G] occupancy, bss[J][S_t] one-hot option, bna[J][N] one-hot node,
    boa[a][b] == 1 iff task a is ordered before task b (milp.py:292-319,510); the diagonal is
    None exactly as the reference leaves it (those variables never enter a constraint).
    All entries are plain Python floats.
    """
    J = len(n_options)
    start_a = np.asarray(start, dtype=np.float64)
    mask_a = np.asarray(slotmask, dtype=np.int64)
    node_a = np.zeros(J, dtype=np.int64) if node_of is None else np.asarray(node_of, dtype=np.int64)
    occ = ((mask_a[:, None] >> np.arange(NSLOT)[None, :]) & 1).astype(bool)        # [J][8]
    tga_a = np.zeros((J, nodes, NSLOT))
    sta_a = np.zeros((nodes, NSLOT, J))
    jj, gg = np.nonzero(occ)
    tga_a[jj, node_a[jj], gg] = 1.0
    sta_a[node_a[jj], gg, jj] = start_a[jj]
    bna_a = np.zeros((J, nodes))
    bna_a[np.arange(J), node_a] = 1.0
    sta, tga, bna = sta_a.tolist(), tga_a.tolist(), bna_a.tolist()
    bss = [[0.0] * int(n_options[t]) for t in range(J)]
    for t in range(J):
        bss[t][int(opt_index[t])] = 1.0
    pos = np.asarray(position)
    boa = (pos[:, None] < pos[None, :]).astype(np.float64).tolist()
    for t in range(J):
        boa[t][t] = None
    return sta, tga, bss, bna, boa


def candidate_from_arrays(task_list, presolved, nodes: int = 1):
    """Warm start: turn a previous plan (the `presolved` tuple) back into a candidate
    (reduced opt bytes, priority order) — the role of setInitialValue at milp.py:103-104,151-155,197-202."""
    if presolved is None:
        return None
    try:
        sta, tga, bss, bna, boa, _mk = presolved
        J = len(task_list)
        if sta is None or len(tga) != J or len(bss) != J:
            return None
        opt = np.zeros(J, dtype=np.uint8)
        starts = np.zeros(J)
        for t, task in enumerate(task_list):
            keys = list(task.strategies.keys())
            if len(bss[t]) != len(keys):
                return None
            k = int(keys[int(np.argmax(bss[t]))])
            if not 1 <= k <= NSLOT:
                return None
            n = int(np.argmax(bna[t]))
            if n >= nodes:
                return None
            opt[t] = (k - 1) | ((n << 3) if nodes > 1 else 0)
            gl = [g for g, v in enumerate(tga[t][n]) if v is not None and round(v) == 1]
            starts[t] = sta[n][gl[0]][t] if gl else 0.0
        order = np.argsort(starts, kind="stable")
        return opt, order
    except Exception:
        return None


# ------------------------------------------------------------------------------------------ solve
_ENGINE = None
_MULTI: dict = {}
last_stats: dict = {}
FP32_EXACT_HORIZON = float(1 << 24)   # integer seconds are exact in the kernels' fp32 state below this
FP32_MAX = float(np.finfo(np.float32).max)
SQUARE_BOUND = float(1 << 50)   # a squared tardiness inside the horizon, (2^25)^2, with |d| < 2^24
_SQUARED = ("squared_tardiness", "squared_flow")   # the solve() objectives that run as the squared tardiness
_SCENARIO = ("worst_makespan", "mean_makespan")    # the solve() objectives over runtime scenarios (scenarios=...)
# the worst and mean (weighted) total tardiness and completion time over the same scenarios: the completion forms run
# as the tardiness forms with every due date +0
_SCENARIO_TARDINESS = ("worst_tardiness", "mean_tardiness")
_SCENARIO_COMPLETION = ("worst_completion", "mean_completion")
_SCENARIO_ALL = _SCENARIO + _SCENARIO_TARDINESS + _SCENARIO_COMPLETION


def _engine(devices=None):
    """The process-wide engine: one device (default), or — `devices` = N or a list of ordinals, else
    SATURN_B200_DEVICES — one handle per device of this process (engine.MultiEngine)."""
    global _ENGINE
    if devices is None:
        env = os.environ.get("SATURN_B200_DEVICES", "")
        if env:
            devices = [int(x) for x in env.split(",")] if "," in env else int(env)
    if devices is not None and not isinstance(devices, int):
        devices = tuple(int(d) for d in devices)
        if len(devices) == 1:
            devices = None if devices[0] == 0 else devices
    if devices is None or devices == 1:
        if _ENGINE is None:
            from .engine import Engine
            _ENGINE = Engine()
        return _ENGINE
    if devices not in _MULTI:
        from .engine import MultiEngine
        _MULTI[devices] = MultiEngine(devices)
    return _MULTI[devices]


def _check_horizon(T, found_makespan=None, release=None, tails=None):
    """The kernels keep schedule times in fp32: `start + ceil(rt)` is exact only below 2^24 s (194 days).
    Before the search: a table whose lower bound of the makespan — the area bound sum_j min_k k * rt_jk / 8, and
    with `release` (per-task release dates) also max_j (r_j + min_k rt_jk) — already reaches that bound cannot
    have an exactly representable plan and is refused.  With `tails` (objective="max_lateness": the delivery tails
    q_t = max d - d_t) the device's score is the tail makespan max_t (C_t + q_t), bounded below by
    max_t (min_k rt_tk + q_t), plus r_t with `release`.  After the search (`found_makespan`, the
    device's value): every time inside the winning schedule is <= its makespan, and fp32 addition rounds
    monotonically, so a makespan below 2^24 proves that all of its starts were computed exactly; anything
    else is refused instead of returned with silently rounded starts (rescale to coarser time units)."""
    if found_makespan is not None:
        if not float(found_makespan) < FP32_EXACT_HORIZON:
            raise SolverError("best plan found has makespan %.6g s >= 2^24 s: its start times are not exact in "
                              "fp32; express runtimes in coarser units (e.g. minutes)" % float(found_makespan))
        return
    k = np.arange(1, T.shape[-1] + 1, dtype=np.float64)
    area = np.where(np.isfinite(T), T.astype(np.float64) * k, np.inf).reshape(T.shape[0], -1).min(axis=1)
    lower = float(area.sum()) / NSLOT
    if release is not None:
        shortest = np.where(np.isfinite(T), T.astype(np.float64), np.inf).reshape(T.shape[0], -1).min(axis=1)
        lower = max(lower, float(np.max(np.asarray(release, dtype=np.float64) + shortest)))
    if tails is not None:
        shortest = np.where(np.isfinite(T), T.astype(np.float64), np.inf).reshape(T.shape[0], -1).min(axis=1)
        rel = np.asarray(release, dtype=np.float64) if release is not None else 0.0
        lower = max(lower, float(np.max(rel + shortest + np.asarray(tails, dtype=np.float64))))
    if lower >= FP32_EXACT_HORIZON:
        raise SolverError("area lower bound of the makespan is %.3g s >= 2^24 s: schedule times are not exact in "
                          "fp32 at that horizon; express runtimes in coarser units (e.g. minutes) or drop sentinel "
                          "options" % lower)

def _check_objective(objective, hysteresis=False, release=None):
    if objective not in ("makespan", "completion", "tardiness", "max_lateness", "late_tasks", "max_stretch",
                         "squared_tardiness", "squared_flow", "late_penalty", "completion_penalty") + _SCENARIO_ALL:
        raise SolverError("objective must be 'makespan', 'completion', 'tardiness', 'max_lateness', 'late_tasks', "
                          "'max_stretch', 'squared_tardiness', 'squared_flow', 'late_penalty', "
                          "'completion_penalty', 'worst_makespan', 'mean_makespan', 'worst_tardiness', "
                          "'mean_tardiness', 'worst_completion' or 'mean_completion', not %r" % (objective,))
    if objective != "makespan" and hysteresis:
        raise SolverError("hysteresis=True compares plans by makespan (milp.py:363-442); it is not defined for "
                          "objective=%r" % (objective,))
    if release is not None and hysteresis:
        raise SolverError("hysteresis=True compares plans by a makespan that knows nothing of release dates "
                          "(milp.py:363-442); it cannot be combined with release")


def _per_task(values, what, task_list):
    """A per-task argument as a list in task order: a sequence aligned with the tasks (or T's rows), or, with
    `task_list`, a mapping keyed by Task — what an orchestrate() loop needs, since its task list shrinks every
    interval."""
    if isinstance(values, Mapping):
        if task_list is None:
            raise SolverError("%s must be a sequence aligned with T's rows" % what)
        missing = [getattr(t, "name", repr(t)) for t in task_list if t not in values]
        if missing:
            raise SolverError("%s has no entry for task(s) %s" % (what, ", ".join(map(str, missing[:5]))))
        return [values[t] for t in task_list]
    if isinstance(values, (str, bytes)) or not hasattr(values, "__len__"):
        raise SolverError("%s must be a sequence of J numbers or a mapping Task -> number" % what)
    return values


def _resolve_weights(weights, objective, J, task_list=None):
    """The caller's per-task weights as (float64 values in task order, fp32 array for the device), or (None, None).
    Raises SolverError before any device call."""
    if weights is None:
        return None, None
    if objective == "max_stretch":
        raise SolverError("objective='max_stretch' weighs every task by 1 / its fastest runtime: it takes no weights "
                          "(for a weighted mean stretch use objective='completion' with weights)")
    if objective not in ("completion", "tardiness", "late_tasks", "squared_tardiness", "squared_flow", "late_penalty",
                         "completion_penalty") + _SCENARIO_TARDINESS + _SCENARIO_COMPLETION:
        raise SolverError("weights apply to objective='completion', 'tardiness', 'late_tasks', 'squared_tardiness', "
                          "'squared_flow', 'late_penalty', 'completion_penalty', 'worst_tardiness', "
                          "'mean_tardiness', 'worst_completion' or 'mean_completion' only, not to %r" % (objective,))
    weights = _per_task(weights, "weights", task_list)
    from .engine import weights_f32
    w32 = weights_f32(weights, J)
    if objective in _SQUARED and not J * float(w32.max()) * SQUARE_BOUND < FP32_MAX:
        # a plan inside the 2^24 horizon with |d| < 2^24 has every tardiness below 2^25, so every square below 2^50:
        # below this bound the device's fp32 sum of squares stays finite (sb_set_weights makes the same test)
        raise SolverError("objective=%r needs J * max(weights) * 2^50 < FLT_MAX (%d tasks, largest weight %g): beyond "
                          "it the fp32 sum of squares can overflow; scale the weights down" % (objective, J,
                                                                                                float(w32.max())))
    return [float(x) for x in weights], w32


def _resolve_due(due, objective, J, task_list=None):
    """The caller's per-task due dates as (float64 values in task order, fp32 array for the device), or (None, None)
    without objective="tardiness", "max_lateness", "late_tasks", "squared_tardiness", "late_penalty" or
    "completion_penalty", which require them.  Raises SolverError before any device call."""
    if objective in ("max_stretch", "squared_flow") and due is not None:
        raise SolverError("objective=%r measures every task from its release date: it takes no due dates "
                          "(pass release=...)" % (objective,))
    if objective in _SCENARIO_COMPLETION:
        if due is not None:
            raise SolverError("objective=%r scores completion times: it takes no due dates (for the tardiness over "
                              "scenarios use objective='worst_tardiness' or 'mean_tardiness')" % (objective,))
        # the tardiness forms with every due date +0 (C >= +0, so max(C - 0, 0) is C bit for bit)
        return [0.0] * J, np.zeros(J, dtype=np.float32)
    if objective not in ("tardiness", "max_lateness", "late_tasks", "squared_tardiness", "late_penalty",
                         "completion_penalty") + _SCENARIO_TARDINESS:
        if due is not None:
            raise SolverError("due dates apply to objective='tardiness', 'max_lateness', 'late_tasks', "
                              "'squared_tardiness', 'late_penalty', 'completion_penalty', 'worst_tardiness' or "
                              "'mean_tardiness' only, not to %r" % (objective,))
        return None, None
    if due is None:
        raise SolverError("objective=%r needs due dates (due=...)" % (objective,))
    due = _per_task(due, "due", task_list)
    from .engine import due_f32
    d32 = due_f32(due, J)
    if objective == "max_lateness" and J > 0 and not float(d32.max()) - float(d32.min()) < FP32_EXACT_HORIZON:
        # the device scores the tails max d - d_t in fp32: beyond 2^24 they round even for integer due dates
        raise SolverError("objective='max_lateness' needs max(due) - min(due) < 2^24")
    return [float(x) for x in due], d32


def _resolve_penalty(penalty, objective, J, task_list=None):
    """The caller's per-task late penalties as (float64 values in task order, fp32 array for the device), or
    (None, None) without objective="late_penalty" or "completion_penalty", which require them.  Raises SolverError
    before any device call."""
    if objective not in ("late_penalty", "completion_penalty"):
        if penalty is not None:
            raise SolverError("penalties apply to objective='completion_penalty' or 'late_penalty' only, not to %r"
                              % (objective,))
        return None, None
    if penalty is None:
        raise SolverError("objective=%r needs the penalty of each missed due date (penalty=...)" % (objective,))
    penalty = _per_task(penalty, "penalty", task_list)
    from .engine import penalty_f32
    p32 = penalty_f32(penalty, J)
    return [float(x) for x in penalty], p32


def _resolve_scenarios(scenarios, objective, J, task_list=None):
    """The caller's runtime scenarios, J rows of K factors each (a sequence aligned with the tasks or T's rows, or with
    `task_list` a mapping Task -> K factors), as (float64 [K][J], fp32 [K][J] for the device), or (None, None) without
    a scenario objective ("worst_makespan", "mean_makespan", "worst_tardiness", "mean_tardiness", "worst_completion"
    or "mean_completion"), which require them.  Raises SolverError before any device call."""
    if objective not in _SCENARIO_ALL:
        if scenarios is not None:
            raise SolverError("scenarios apply to objective='worst_makespan', 'mean_makespan', 'worst_tardiness', "
                              "'mean_tardiness', 'worst_completion' or 'mean_completion' only, not to %r"
                              % (objective,))
        return None, None
    if scenarios is None:
        raise SolverError("objective=%r needs runtime scenarios (scenarios=...)" % (objective,))
    rows = _per_task(scenarios, "scenarios", task_list)
    if len(rows) != J:
        raise SolverError("scenarios must have one row per task (%d), got %d" % (J, len(rows)))
    try:
        lens = {len(r) for r in rows}
    except TypeError:
        raise SolverError("each task's scenarios must be a sequence of K factors")
    if len(lens) > 1:
        raise SolverError("every task must have the same number of scenario factors, got %s" % sorted(lens))
    try:
        f64 = np.asarray([list(r) for r in rows], dtype=np.float64).reshape(J, -1).T.copy()
    except (TypeError, ValueError) as e:
        raise SolverError("scenario factors must be numbers: %s" % e)
    from .engine import scenarios_f32
    return f64, scenarios_f32(f64, J)


def _check_scenario_horizon(Tdev, f32, release=None):
    """_check_horizon on every scenario table T_k, formed in fp32 as the device forms it (one rounded product)."""
    with np.errstate(over="ignore"):
        for k in range(f32.shape[0]):
            _check_horizon((f32[k][:, None, None] * Tdev).astype(np.float32), release=release)


def _scenario_stats(rts, gpus, node, prio, f64, integer_starts, r64=None, w64=None, d64=None, objective=None):
    """scenario_makespans (each scenario's makespan, K values), worst_makespan and mean_makespan of a plan's options and
    order, in float64: the list rule re-run on every scenario's runtimes f[k][t] * rt_t (the tasks' own runtimes), with
    integer starts rounding each hold up as the device does.  With objective="worst_tardiness" / "mean_tardiness" also
    scenario_tardiness (each scenario's total tardiness sum_t w_t max(C_tk - d_t, 0), unit weights without w64),
    worst_tardiness and mean_tardiness; with "worst_completion" / "mean_completion" scenario_completion (each scenario's
    sum_t w_t C_tk), worst_completion and mean_completion."""
    J = len(rts)
    w = [1.0] * J if w64 is None else [float(x) for x in w64]
    d = [0.0] * J if d64 is None else [float(x) for x in d64]
    mks, sums = [], []
    for k in range(f64.shape[0]):
        ready = {}
        mk = 0.0
        total = 0.0
        for j in (int(x) for x in prio):
            rt = float(f64[k, j]) * float(rts[j])
            rd = ready.setdefault(int(node[j]), [0.0] * NSLOT)
            sel = sorted(range(NSLOT), key=lambda g: (rd[g], g))[:int(gpus[j])]
            st = rd[sel[-1]]
            if r64 is not None:
                rel = float(r64[j])
                st = max(st, math.ceil(rel) if integer_starts else rel)
            nxt = st + (math.ceil(rt) if integer_starts and math.isfinite(rt) else rt)
            for g in sel:
                rd[g] = nxt
            mk = max(mk, st + rt)
            total += w[j] * max(st + rt - d[j], 0.0)
        mks.append(mk)
        sums.append(total)
    out = {"scenario_makespans": mks, "worst_makespan": max(mks), "mean_makespan": sum(mks) / len(mks)}
    if objective in _SCENARIO_TARDINESS + _SCENARIO_COMPLETION:
        what = "tardiness" if objective in _SCENARIO_TARDINESS else "completion"
        out.update({"scenario_" + what: sums, "worst_" + what: max(sums), "mean_" + what: sum(sums) / len(sums)})
    return out


def _resolve_release(release, J, task_list=None):
    """The caller's per-task release dates as (float64 values in task order, fp32 array for the device, rounded up),
    or (None, None).  Valid under every objective.  Raises SolverError before any device call."""
    if release is None:
        return None, None
    release = _per_task(release, "release", task_list)
    from .engine import release_f32
    r32 = release_f32(release, J)
    return [float(x) for x in release], r32


def _set_objective(eng, objective, w32, d32, r32=None, p32=None):
    """Hand the weights, due dates, release dates and late penalties to the engine; returns the engine objective the
    search runs."""
    if r32 is not None:
        eng.set_release(r32)
    if p32 is not None:
        eng.set_penalty(p32)
    if w32 is not None:
        eng.set_weights(w32)
    if d32 is not None:
        eng.set_due(d32)
        if objective == "max_lateness":
            return objective
        if objective == "late_tasks":
            return "weighted_late_tasks" if w32 is not None else "late_tasks"
        if objective == "max_stretch":
            return "weighted_max_tardiness"
        if objective in _SQUARED:
            return "weighted_squared_tardiness" if w32 is not None else "squared_tardiness"
        if objective in ("late_penalty", "completion_penalty"):
            return "weighted_" + objective if w32 is not None else objective
        if objective in _SCENARIO_TARDINESS + _SCENARIO_COMPLETION:
            form = objective.split("_")[0] + "_tardiness"   # the completion forms: every due date 0
            return "weighted_" + form if w32 is not None else form
        return "weighted_tardiness" if w32 is not None else "tardiness"
    return "weighted_completion" if w32 is not None else objective


def _tardiness_stats(start, rts, w64, d64):
    """weighted_tardiness (unit weights without w64) and late_tasks of a plan, in float64."""
    late = [float(s) + float(r) - d for s, r, d in zip(start, rts, d64)]
    w = w64 if w64 is not None else [1.0] * len(late)
    return {"weighted_tardiness": sum(wi * max(0.0, x) for wi, x in zip(w, late)),
            "late_tasks": sum(1 for x in late if x > 0)}


def _late_count_stats(start, rts, w64, d64):
    """_tardiness_stats, and with w64 weighted_late_tasks, the weight of the tasks with C_t > d_t, in float64."""
    stats = _tardiness_stats(start, rts, w64, d64)
    if w64 is not None:
        stats["weighted_late_tasks"] = sum(w for s, r, d, w in zip(start, rts, d64, w64) if float(s) + float(r) - d > 0)
    return stats


def _lateness_stats(start, rts, d64):
    """max_lateness, max_t (C_t - d_t), and late_tasks of a plan, in float64."""
    late = [float(s) + float(r) - d for s, r, d in zip(start, rts, d64)]
    return {"max_lateness": max(late), "late_tasks": sum(1 for x in late if x > 0)}


def _stretch_form(Tdev, r32):
    """objective="max_stretch" as the weighted maximum tardiness: per task its fastest runtime p*_t, the smallest
    finite cell of the device table Tdev (the cells the search may propose; a task whose only cells are sentinels
    keeps the sentinel's value, the cell the search uses for it), the fp32 weights fp32(1 / p*_t) (the reciprocal
    in float64) and the fp32 due dates max(r32_t, +0) (+0 without release dates).  Raises SolverError, before any
    device call, when a p*_t is 0 (its stretch is undefined) or fp32(1 / p*_t) * 2^24 overflows fp32."""
    J = Tdev.shape[0]
    pstar = np.where(np.isfinite(Tdev), Tdev, np.inf).reshape(J, -1).min(axis=1).astype(np.float64)
    if not np.isfinite(pstar).all():
        raise SolverError("objective='max_stretch' needs a finite runtime for every task")
    if (pstar == 0).any():
        raise SolverError("objective='max_stretch' is undefined for a task whose fastest runtime is 0 (task %d)"
                          % int(np.argmax(pstar == 0)))
    with np.errstate(over="ignore"):
        w32 = (1.0 / pstar).astype(np.float32)
        scaled = w32 * np.float32(FP32_EXACT_HORIZON)
    if not np.isfinite(scaled).all():
        raise SolverError("objective='max_stretch': 1 / the fastest runtime of task %d overflows fp32 over a 2^24 "
                          "horizon; express runtimes in finer units" % int(np.argmax(~np.isfinite(scaled))))
    return pstar, w32, _release_due(r32, J)


def _release_due(r32, J):
    """The fp32 due dates max(r32_t, +0) (+0 without release dates) that measure every task from its release:
    objective="max_stretch" and "squared_flow" run against them."""
    return np.zeros(J, dtype=np.float32) if r32 is None else np.where(r32 > 0, r32, np.float32(0)).astype(np.float32)


def _stretch_stats(start, rts, pstar, r64):
    """max_stretch and mean_stretch of a plan, (C_t - max(r_t, 0)) / p*_t in float64 (r_t = 0 without r64)."""
    r = r64 if r64 is not None else [0.0] * len(rts)
    st = [(float(s) + float(rt) - max(x, 0.0)) / float(p) for s, rt, x, p in zip(start, rts, r, pstar)]
    return {"max_stretch": max(st), "mean_stretch": sum(st) / len(st)}


def _squared_stats(start, rts, w64, d64):
    """squared_tardiness, sum_t w_t max(0, C_t - d_t)^2 (unit weights without w64), with weighted_tardiness and
    late_tasks (_tardiness_stats), of a plan in float64."""
    w = w64 if w64 is not None else [1.0] * len(rts)
    stats = _tardiness_stats(start, rts, w64, d64)
    stats["squared_tardiness"] = sum(wi * max(0.0, float(s) + float(r) - d) ** 2
                                     for s, r, d, wi in zip(start, rts, d64, w))
    return stats


def _late_penalty_stats(start, rts, w64, d64, p64):
    """late_penalty, sum_t [C_t > d_t] (p_t + w_t (C_t - d_t)) (unit rate without w64), with weighted_tardiness and
    late_tasks (_tardiness_stats), of a plan in float64."""
    w = w64 if w64 is not None else [1.0] * len(rts)
    stats = _tardiness_stats(start, rts, w64, d64)
    late = [float(s) + float(r) - d for s, r, d in zip(start, rts, d64)]
    stats["late_penalty"] = sum(p + wi * x for x, p, wi in zip(late, p64, w) if x > 0)
    return stats


def _completion_penalty_stats(start, rts, w64, d64, p64):
    """completion_penalty, sum_t (w_t C_t + [C_t > d_t] p_t) (unit weights without w64), with weighted_completion,
    late_tasks and penalty_paid, sum_t [C_t > d_t] p_t, of a plan in float64."""
    w = w64 if w64 is not None else [1.0] * len(rts)
    comp = [float(s) + float(r) for s, r in zip(start, rts)]
    late = [c > d for c, d in zip(comp, d64)]
    wc = sum(wi * c for wi, c in zip(w, comp))
    paid = sum(p for p, x in zip(p64, late) if x)
    return {"completion_penalty": wc + paid, "weighted_completion": wc, "late_tasks": sum(late), "penalty_paid": paid}


def _squared_flow_stats(start, rts, w64, r64):
    """squared_flow, sum_t w_t (C_t - max(r_t, 0))^2 (unit weights without w64, r_t = 0 without r64), and
    total_flow_time, sum_t (C_t - max(r_t, 0)), of a plan in float64."""
    r = r64 if r64 is not None else [0.0] * len(rts)
    w = w64 if w64 is not None else [1.0] * len(rts)
    flow = [float(s) + float(rt) - max(x, 0.0) for s, rt, x in zip(start, rts, r)]
    return {"squared_flow": sum(wi * f * f for wi, f in zip(w, flow)), "total_flow_time": sum(flow)}


def _tails(d32):
    """The delivery tails max d - d_t of objective="max_lateness", as the device forms them (fp32)."""
    return d32.max() - d32 if d32 is not None else None


def _flow_stats(start, rts, r64):
    """total_flow_time of a plan, sum_t (C_t - max(r_t, 0)): the time from release to result, in float64."""
    return {"total_flow_time": sum(float(s) + float(r) - max(x, 0.0) for s, r, x in zip(start, rts, r64))}


def _plan_horizon(start, rt):
    """max(start + rt) of a decoded plan: the latest time the device's fp32 schedule holds.  With the
    sum-of-completion-times objective the device's score is a sum that may exceed 2^24 while every start is
    exact, so the horizon guard checks the plan itself."""
    return max((float(s) + float(r) for s, r in zip(start, rt)), default=0.0)


def _default_nodes() -> int:
    env = os.environ.get("SATURN_B200_NODES")
    if env:
        return max(1, int(env))
    ray = __import__("sys").modules.get("ray")      # never import Ray just to ask
    try:
        if ray is not None and ray.is_initialized():
            return max(1, len(ray.nodes()))
    except Exception:
        pass
    return 1


def solve(task_list, presolved=None, gurobi=True, threads=max(1, (os.cpu_count() or 4) // 4), interval=1000,
          timeout=500, *, chains: Optional[int] = None, rounds: Optional[int] = None, seed: int = 0,
          integer_starts: bool = True, engine=None, hysteresis: Optional[bool] = None,
          nodes: Optional[int] = None, devices=None, objective: str = "makespan", weights=None, due=None,
          release=None, penalty=None, scenarios=None, _warm=None):
    """Drop-in for saturn.solver.solve (milp.py:23).

    Objective.  "makespan" (the default, the reference's) or "completion": minimise the sum of the tasks'
    completion times sum_t (start_t + runtime_t) — equivalently the mean time a job waits for its result —
    which a makespan-optimal plan can leave poor (long jobs first, every short job finishes late).  The
    6th element returned is the plan's makespan under both objectives; last_stats["objective"] names the
    objective and last_stats["total_completion"] holds the plan's sum of completion times, recomputed in
    float64 from the emitted plan and the tasks' own runtimes; last_stats["device_makespan"] is the device's
    fp32 score of the plan (the sum, under "completion").  Anything else raises SolverError.

    Weights.  With objective="completion", `weights` (a sequence aligned with task_list, or a mapping keyed by
    Task, which survives orchestrate()'s shrinking task list) makes the objective the weighted sum
    sum_t w_t (start_t + runtime_t): a job's priority.  Every weight must be finite and > 0, and stay so in fp32;
    anything else, weights under objective="makespan", a wrong length or a task missing from the mapping raises
    SolverError before any device call.  last_stats["weighted_completion"] then holds the plan's weighted sum in
    float64 (the caller's weights, the tasks' own runtimes) and last_stats["device_makespan"] the device's fp32
    weighted sum; "total_completion" and the 6th element keep their meaning.

    Due dates.  objective="tardiness" with `due` (a sequence aligned with task_list, or a mapping keyed by Task,
    in the runtimes' units from the plan's t = 0) minimises the total tardiness sum_t max(0, C_t - d_t), with
    C_t = start_t + runtime_t; with `weights` as well, the weighted tardiness sum_t w_t max(0, C_t - d_t).  Every
    due date must be finite with |d| < 2^24 (negative: already overdue).  A missing `due`, `due` under another
    objective, a wrong length, a task missing from the mapping or a bad value raises SolverError before any device
    call, as does hysteresis=True.  The search stops as soon as it finds a plan with no tardiness.
    last_stats["weighted_tardiness"] (unit weights without `weights`) and last_stats["late_tasks"] (tasks with
    C_t > d_t) are computed in float64 from the emitted plan, the tasks' own runtimes and the caller's d and w;
    last_stats["device_makespan"] holds the device's fp32 tardiness.

    Maximum lateness.  objective="max_lateness" with `due` (as above) minimises L_max = max_t (C_t - d_t), which can be
    negative: it maximises the smallest margin any task keeps against its due date, where "tardiness" stops at the
    first plan that is not late.  L_max <= 0 means every due date is met; L_max > 0 is the smallest uniform delay of
    the due dates that makes them all feasible.  With `release` and due = release (+ a target), it is the longest
    any task waits from its release to its result.  `weights`, hysteresis=True and due dates spread over 2^24 or more
    raise SolverError before any device call, as do the `due` errors above.  The device scores L_max + max_t d_t
    (>= 0); last_stats["max_lateness"] and last_stats["late_tasks"] are recomputed in float64 from the emitted plan,
    the tasks' own runtimes and the caller's due dates, and last_stats["device_makespan"] holds the device's fp32
    score minus max_t d_t.  Shifting every due date by one constant gives the same plan.  The 6th element stays the
    plan's makespan.

    Late tasks.  objective="late_tasks" with `due` (as above) minimises the number of tasks that finish after their
    due date, C_t > d_t: the question of how many jobs miss a deadline, which any delay misses alike.  A task that
    finishes exactly at its due date is on time.  With `weights` as well it minimises sum_t w_t [C_t > d_t].  The
    `due` and `weights` rules and errors are those above, as is the refusal of hysteresis=True; `release` is valid.
    The search stops as soon as it finds a plan with no late task.  The device decides C_t > d_t in fp32 on the fp32
    due date, like the tardiness: with fractional data a completion within rounding of its due date may count either
    way.  last_stats["late_tasks"] and last_stats["weighted_tardiness"] are recomputed in float64 from the emitted
    plan, the tasks' own runtimes and the caller's d (and w), with `weights` also last_stats["weighted_late_tasks"],
    the weight of the late tasks; last_stats["device_makespan"] holds the device's fp32 score.  The 6th element
    stays the plan's makespan.

    Maximum stretch.  objective="max_stretch" minimises max_t S_t, the stretch (slowdown) of each task: its time from
    release to result divided by the time it would take with the cluster to itself, S_t = (C_t - max(r_t, 0)) /
    p*_t, where p*_t is the task's fastest runtime over the options the search may propose (its sentinel options
    only when it has nothing else, and then the sentinel's value).  It keeps every task's wait in proportion to its
    size, where "completion" favours short tasks and "makespan" lets a short task wait behind a long one.  It runs
    as the weighted maximum tardiness with w_t = fp32(1 / p*_t) (the reciprocal taken in float64) and due dates
    max(r_t, 0) in fp32 (0 without `release`); `release` is valid, `weights`, `due` and hysteresis=True raise
    SolverError, as does a task whose p*_t is 0 or whose fp32(1 / p*_t) * 2^24 overflows fp32, all before any device
    call.  last_stats["max_stretch"] and last_stats["mean_stretch"] are recomputed in float64 from the emitted plan, the
    tasks' own runtimes (p*_t over the same options) and the caller's r; last_stats["device_makespan"] holds the
    device's fp32 max stretch.  The 6th element stays the plan's makespan.  The mean stretch needs no objective of
    its own: objective="completion" with weights={t: 1 / p*_t} minimises sum_t (C_t - r_t) / p*_t up to a constant.

    Squared tardiness.  objective="squared_tardiness" with `due` (as above) minimises sum_t w_t max(0, C_t - d_t)^2
    (unit weights without `weights`): the l2 norm of the delays, between the total tardiness, which is indifferent
    between one task late by 10 h and ten late by 1 h each, and a maximum, which ignores every task but the worst.
    The `due` and `weights` rules and errors are those of "tardiness", as is the refusal of hysteresis=True;
    `release` is valid.  The search stops as soon as it finds a plan with no late task.  objective="squared_flow"
    minimises sum_t w_t (C_t - max(r_t, 0))^2, the l2 norm of each task's time from release to result (sum_t w_t C_t^2
    without `release`): it runs as the squared tardiness against the due dates max(r_t, 0) in fp32, as
    "max_stretch" does; `release` and `weights` are valid, `due` and hysteresis=True raise SolverError.  Under both,
    weights with J * max(weights) * 2^50 >= FLT_MAX raise SolverError before any device call (past it the device's
    fp32 sum of squares can overflow; unit weights never do).  last_stats["squared_tardiness"],
    ["weighted_tardiness"] and ["late_tasks"] (squared_tardiness), or last_stats["squared_flow"] and
    ["total_flow_time"] (squared_flow), are recomputed in float64 from the emitted plan, the tasks' own runtimes and
    the caller's d, r and w; last_stats["device_makespan"] holds the device's fp32 score.  The 6th element stays the
    plan's makespan.

    Late penalty.  objective="late_penalty" with `due` (as above) and `penalty` (a sequence aligned with task_list,
    or a mapping keyed by Task, every value finite and >= 0) minimises sum_t [C_t > d_t] (p_t + w_t (C_t - d_t)):
    each missed due date costs its fixed penalty p_t (a missed submission, an SLA credit) plus w_t per unit of time
    late (unit rate without `weights`).  With every p = 0 it is "tardiness"; with penalties above any total
    tardiness a plan can have it minimises the late count first and breaks ties by the tardiness.  The `due` and
    `weights` rules and errors are those of "tardiness", as is the refusal of hysteresis=True; `release` is valid.
    A missing `penalty`, `penalty` under any other objective, a wrong length, a task missing from the mapping, a
    negative, NaN or inf value, or penalties that overflow fp32 (J * max(penalty) >= 2^126) raise SolverError before
    any device call.  The search stops as soon as it finds a plan with no late task.  The device decides C_t > d_t
    in fp32, so with fractional runtimes or due dates a task that completes within rounding of its due date may be
    counted either way (integer data is exact).  last_stats["late_penalty"], ["weighted_tardiness"] and
    ["late_tasks"] are recomputed in float64 from the emitted plan, the tasks' own runtimes and the caller's d, w and
    p; last_stats["device_makespan"] holds the device's fp32 score.  The 6th element stays the plan's makespan.

    Completion penalty.  objective="completion_penalty" with `due` and `penalty` (as for "late_penalty") minimises
    sum_t (w_t C_t + [C_t > d_t] p_t): the (weighted) completion time, as "completion" minimises it, plus a fixed
    penalty for each missed due date (an SLA credit) that the late penalty's rate does not stand in for, since every
    task's completion time already counts.  With every p = 0 it is "completion", plan for plan.  A task that
    finishes exactly at its due date is on time, decided in fp32 as "late_penalty" decides it.  One due date H for
    every task with every penalty above any sum_t w_t C_t makes it "minimise the mean completion time subject to a
    makespan <= H" (solve_front runs it so).  The `due`, `weights`, `penalty` and `release` rules and errors are
    those of "late_penalty", as is the refusal of hysteresis=True; there is no stop at zero.
    last_stats["completion_penalty"], ["weighted_completion"] (unit weights without `weights`), ["late_tasks"] and
    ["penalty_paid"] are recomputed in float64 from the emitted plan, the tasks' own runtimes and the caller's d, w
    and p; last_stats["device_makespan"] holds the device's fp32 score.  The 6th element stays the plan's makespan.

    Runtime scenarios.  objective="worst_makespan" or "mean_makespan" with `scenarios` (a sequence aligned with
    task_list of K factors each, or a mapping Task -> K factors, 1 <= K <= 8, every factor finite and > 0) plans for
    runtimes that are estimates: scenario k runs every option of task t f[t][k] times as long (fp32(f * rt), one
    rounding), and the plan — its options and list order — minimises the largest makespan over the K scenarios, or
    their mean, the list rule re-run on each scenario's runtimes (not the same gangs replayed).  `release` is valid.
    A missing `scenarios`, `scenarios` under any other objective, ragged or out-of-range K, a bad factor,
    hysteresis=True, or a scenario whose table breaks the 2^24 s integer-start horizon raises SolverError before any
    device call.  The 6-tuple is the plan on the nominal runtimes (what the executor runs) and its 6th element the
    nominal makespan; last_stats["scenario_makespans"] (K values), ["worst_makespan"] and ["mean_makespan"] are
    re-run in float64 from the plan's options and order on f * the tasks' own runtimes; last_stats["device_makespan"]
    holds the device's fp32 score (the worst makespan, or the sum of the K makespans).

    The same scenarios serve the completion-time and tardiness users.  objective="worst_tardiness" or
    "mean_tardiness" (with `due`, `weights` optional) minimises the largest, or the mean, over the K scenarios of the
    TOTAL (weighted) tardiness sum_t w_t max(C_tk - d_t, 0) — the worst or mean of objective="tardiness", not the
    per-task maximum tardiness of the engine's "max_tardiness".  objective="worst_completion" or "mean_completion"
    (`weights` optional, `due` refused) does the same for the (weighted) completion time sum_t w_t C_tk, the classical
    stochastic objective sum w E[C] for "mean_completion"; the device runs them as the tardiness forms with every due
    date 0.  All four take `scenarios` (required), `release`, `nodes` and `devices`, and refuse `penalty` and
    hysteresis=True, with SolverError before any device call.  last_stats then also holds ["scenario_tardiness"] (K
    values), ["worst_tardiness"] and ["mean_tardiness"], or ["scenario_completion"], ["worst_completion"] and
    ["mean_completion"], re-run in float64 as the makespans are; last_stats["device_makespan"] holds the device's
    fp32 score (the worst total, or the sum of the K totals).

    Release dates.  `release` (a sequence aligned with task_list, or a mapping keyed by Task, in the runtimes' units
    from the plan's t = 0) keeps every task from starting before its release date, under every objective: a
    dataset or a parent checkpoint that is only ready later, a job that arrives tomorrow.  r <= 0 means already
    released.  Every value must be finite with |r| < 2^24; it is rounded up to fp32, and with integer_starts a task
    starts no earlier than ceil(r), so every emitted start is >= the caller's r.  A wrong length, a task missing
    from the mapping, a bad value, or hysteresis=True together with `release` raises SolverError before any device
    call.  The 6th element and last_stats["makespan"] then count from t = 0, releases included;
    last_stats["total_flow_time"] holds sum_t (C_t - max(r_t, 0)), the time from release to result, in float64
    (for fixed release dates, minimising it is minimising the sum of completion times).

    Returns (sta, tga, bss, bna, boa, makespan) — milp.py:445 — with a real float makespan
    (the reference returns None on a cold start, milp.py:394-399; callers only thread it back in
    as `presolved`).  Keyword-only extras tune the GPU search; environment overrides:
    SATURN_B200_CHAINS, SATURN_B200_ROUNDS, SATURN_B200_BUDGET_S, SATURN_B200_HYSTERESIS.

    Devices.  `devices=N` (or a list of CUDA ordinals, or SATURN_B200_DEVICES) shards the search population
    over N GPUs of this process — one handle per device, one MIN of a uint64 per group of rounds over NVLink
    peer memory (sb_search_run_multi); `chains` is per device.  The reference calls solve() from a single
    process (orchestrator.py:21-23,55,69), so this is how that call site uses the whole node.

    Nodes.  The reference plans over len(ray.nodes()) nodes of 8 GPUs each (milp.py:58-62); here the
    node count is the `nodes` keyword, else SATURN_B200_NODES, else an initialised Ray's node count,
    else 1.  A task runs on exactly one node (milp.py:117-137).

    Re-planning policy.  As shipped, the reference ALWAYS adopts the fresh plan: its comparator
    (milp.py:383-442) keys on `saved_makespan`, which stays None from the cold start on
    (milp.py:394-399 never assigns it), so the swap / keep branches are unreachable (SURVEY §3.2).
    That observable behaviour is the default here.  `hysteresis=True` (or SATURN_B200_HYSTERESIS=1)
    enables the documented intent instead: keep the current plan, shifted by one interval, unless
    the new one is better by more than interval + 500 s (milp.py:363,377,429-442).  The rule is stated
    in makespans: hysteresis=True with another objective raises SolverError, and
    SATURN_B200_HYSTERESIS applies to the makespan objective only.
    """
    from .search import run_search
    _check_objective(objective, bool(hysteresis), release)
    t_wall = time.perf_counter()
    task_list = list(task_list)
    J = len(task_list)
    w64, w32 = _resolve_weights(weights, objective, J, task_list)
    d64, d32 = _resolve_due(due, objective, J, task_list)
    p64, p32 = _resolve_penalty(penalty, objective, J, task_list)
    f64, f32 = _resolve_scenarios(scenarios, objective, J, task_list)
    r64, r32 = _resolve_release(release, J, task_list)
    if J == 0:
        return [[[] for _ in range(NSLOT)]], [], [], [], [], 0.0
    eng = engine if engine is not None else _engine(devices)
    T, usable, optindex = build_table(task_list)
    # sentinel cells (executor None) must never be proposed: they are removed from the device table
    # unless the task has nothing else; every remaining finite cell is usable (sentinel = +inf)
    Tdev = T.copy()
    for j in range(J):
        if usable[j].any():
            Tdev[j, 0, ~usable[j]] = np.inf
    _check_horizon(Tdev, release=r64, tails=_tails(d32) if objective == "max_lateness" else None)
    if f32 is not None:
        _check_scenario_horizon(Tdev, f32, r64)
    if objective == "max_stretch":
        _, w32, d32 = _stretch_form(Tdev, r32)
        # p*_t in the tasks' own runtimes: the fastest option among the cells the device table keeps
        pstar = [min(float(list(t.strategies.values())[int(optindex[j, g])].runtime)
                     for g in range(NSLOT) if np.isfinite(Tdev[j, 0, g])) for j, t in enumerate(task_list)]
    elif objective == "squared_flow":
        d32 = _release_due(r32, J)
    if nodes is None:
        nodes = _default_nodes()
    nodes = int(nodes)
    eng.set_table(Tdev, list(range(1, NSLOT + 1)), sentinel=float("inf"), nodes=nodes)
    search_objective = _set_objective(eng, objective, w32, d32, r32, p32)
    if f32 is not None:
        eng.set_scenarios(f32)
    if chains is None:
        chains = int(os.environ.get("SATURN_B200_CHAINS", 0))
        if chains <= 0:
            # about 131072 chains, rounded to whole waves of the round kernel (no partially filled last wave)
            wave = (eng.search_wave(reduced=True, **({"objective": search_objective} if objective in _SCENARIO_ALL
                                                     else {}))
                    if hasattr(eng, "search_wave") else 0)
            chains = max(1, round((1 << 17) / wave)) * wave if wave > 0 else 1 << 17
    if rounds is None:
        rounds = int(os.environ.get("SATURN_B200_ROUNDS", 400))
    budget = float(os.environ.get("SATURN_B200_BUDGET_S", 20.0))
    try:
        budget = min(budget, float(timeout))
    except (TypeError, ValueError):
        pass
    warm = _warm if _warm is not None else candidate_from_arrays(task_list, presolved, nodes)
    res = run_search(eng, chains=chains, rounds=rounds, seed=seed, integer_starts=integer_starts, reduced=True,
                     time_budget_s=budget, patience=max(40, rounds // 4), warm=warm,
                     **({"objective": search_objective} if search_objective != "makespan" else {}))
    if objective in ("makespan", "max_lateness"):
        _check_horizon(Tdev, res.makespan)
    dec = eng.decode(res.opt, res.prio, integer_starts=integer_starts, reduced=True)
    gpus = dec["gpus"].astype(np.int64)
    if objective != "makespan":
        _check_horizon(Tdev, _plan_horizon(dec["start"], Tdev[np.arange(J), 0, gpus - 1]))
    chosen = optindex[np.arange(J), gpus - 1]
    if (chosen < 0).any():
        raise SolverError("search returned an option a task does not have")
    position = np.empty(J, dtype=np.int64)
    position[res.prio.astype(np.int64)] = np.arange(J)
    n_options = [len(t.strategies) for t in task_list]
    prop = plan_to_arrays(n_options, chosen, dec["start"], dec["slotmask"], position, nodes=nodes,
                          node_of=dec["node"])
    # the makespan the caller sees is recomputed in float64 from the emitted plan and the tasks'
    # own (un-rounded) runtimes: max_t start_t + runtime_t  (milp.py:170-177)
    rts = [list(t.strategies.values())[int(chosen[i])].runtime for i, t in enumerate(task_list)]
    prop_makespan = max(float(dec["start"][i]) + float(rts[i]) for i in range(J))

    global last_stats
    last_stats = {"candidates": res.evaluated, "rounds": res.rounds, "search_wall_s": res.wall_s,
                  "device_makespan": res.makespan, "makespan": prop_makespan, "J": J, "chains": chains,
                  "nodes": nodes, "devices": len(getattr(eng, "engines", [eng])),
                  "total_wall_s": None, "adopted": True, "objective": objective,
                  "total_completion": sum(float(dec["start"][i]) + float(rts[i]) for i in range(J))}
    if w64 is not None:
        last_stats["weighted_completion"] = sum(w64[i] * (float(dec["start"][i]) + float(rts[i])) for i in range(J))
    if objective == "max_lateness":
        last_stats.update(_lateness_stats(dec["start"], rts, d64))
        last_stats["device_makespan"] = res.makespan - eng.due_shift
    elif objective == "late_tasks":
        last_stats.update(_late_count_stats(dec["start"], rts, w64, d64))
    elif objective == "max_stretch":
        last_stats.update(_stretch_stats(dec["start"], rts, pstar, r64))
    elif objective == "squared_tardiness":
        last_stats.update(_squared_stats(dec["start"], rts, w64, d64))
    elif objective == "squared_flow":
        last_stats.update(_squared_flow_stats(dec["start"], rts, w64, r64))
    elif objective == "late_penalty":
        last_stats.update(_late_penalty_stats(dec["start"], rts, w64, d64, p64))
    elif objective == "completion_penalty":
        last_stats.update(_completion_penalty_stats(dec["start"], rts, w64, d64, p64))
    elif objective in _SCENARIO_ALL:
        last_stats.update(_scenario_stats(rts, gpus, dec["node"], res.prio, f64, integer_starts, r64, w64, d64,
                                          objective))
        _check_horizon(Tdev, max(last_stats["scenario_makespans"]))
    elif d64 is not None:
        last_stats.update(_tardiness_stats(dec["start"], rts, w64, d64))
    if r64 is not None:
        last_stats.update(_flow_stats(dec["start"], rts, r64))

    # ---- introspection hysteresis (opt-in): the documented intent of milp.py:363-442
    out = prop + (prop_makespan,)
    if hysteresis is None:
        hysteresis = objective == "makespan" and release is None and os.environ.get("SATURN_B200_HYSTERESIS", "0") not in (
            "", "0", "false", "False")
    if presolved is not None and hysteresis:
        p_sta, p_tga, p_bss, p_bna, p_boa, saved = presolved
        same_tasks = p_tga is not None and len(p_tga) == J
        if saved is not None and same_tasks:
            try:
                itv = float(interval)
            except (TypeError, ValueError):
                itv = 1000.0
            if not (prop_makespan < float(saved) - itv - REPLAN_THRESHOLD):
                # keep the current plan, shifted by one interval (milp.py:429-442)
                kept_sta = [[[max(float(v) - itv, 0.0) for v in g] for g in n] for n in p_sta]
                out = (kept_sta, p_tga, p_bss, p_bna, p_boa, float(saved) - itv)
                last_stats["adopted"] = False
    last_stats["total_wall_s"] = time.perf_counter() - t_wall
    return out


# ------------------------------------------------------------------------------------------ dense T
NOT_PROFILED = 1.0e6   # PerformanceEvaluator.py:99  (gpu count outside the task's gpu_range)
FAILED = 1.0e8         # PerformanceEvaluator.py:106 (every executor failed at this gpu count)


def table_from_trials(n_tasks: int, n_executors: int, gpu_ranges, flat_results, max_gpus: int = NSLOT):
    """The trial runner's raw results as the dense tensor the GPU path ingests (SURVEY §8f-3).

    `flat_results` is the list PerformanceEvaluator.search collects (PerformanceEvaluator.py:78-93): one
    `(params, runtime)` per (task, g in the task's gpu_range, executor) in that nesting order, runtime
    already scaled to the whole job (`:24-26`), `params is None` for a failed trial.  `gpu_ranges[t]` is
    the task's gpu_range (None = 1..max_gpus).  Returns
        T[J][S][G] fp32  runtime of task j under executor s on g+1 GPUs; the reference's sentinels where
                         there is no measurement: 1e6 not profiled (`:99`), 1e8 failed (`:106`)
        mask[J][S][G]    True where a trial succeeded
        params[J][S][G]  the executor's tuned parameters (object array, None elsewhere)
    Instead of collapsing the executor axis into task.strategies on the host (`:101-115`) the solver is
    given all of it: `solve_table(T, mask)`; `strategies_from_table` gives the dict view."""
    G = int(max_gpus)
    T = np.full((n_tasks, n_executors, G), NOT_PROFILED, dtype=np.float32)
    mask = np.zeros((n_tasks, n_executors, G), dtype=bool)
    params = np.empty((n_tasks, n_executors, G), dtype=object)
    it = iter(flat_results)
    for t in range(n_tasks):
        rng_t = gpu_ranges[t] if gpu_ranges is not None and gpu_ranges[t] is not None else range(1, G + 1)
        for g in rng_t:
            for e in range(n_executors):
                prm, runtime = next(it)
                if not 1 <= int(g) <= G:
                    continue
                if prm is not None and runtime is not None:
                    v = np.float32(runtime)
                    if float(v) < float(runtime):                     # round up, as build_table does
                        v = np.nextafter(v, np.float32(np.inf))
                    T[t, e, int(g) - 1] = v
                    mask[t, e, int(g) - 1] = True
                    params[t, e, int(g) - 1] = prm
                else:
                    T[t, e, int(g) - 1] = FAILED
    return T, mask, params


def strategies_from_table(T, mask, executors=None, params=None, gcount=None):
    """The compatibility view: what PerformanceEvaluator.py:96-115 would have attached to each task —
    per task an ordered dict {g: Strategy(executor, g, params, runtime)} over ALL gpu counts, the fastest
    executor per g (first minimum wins, strict `<` at `:110`), Strategy(None, g, None, 1e6) where nothing was
    profiled and Strategy(None, g, None, 1e8) where every executor failed."""
    from .representations import Strategy
    T = np.asarray(T)
    mask = np.asarray(mask, dtype=bool)
    J, S, G = T.shape
    gcount = list(range(1, G + 1)) if gcount is None else [int(g) for g in gcount]
    out = []
    for j in range(J):
        d = {}
        for gi, g in enumerate(gcount):
            ok = mask[j, :, gi]
            if ok.any():
                col = np.where(ok, T[j, :, gi], np.inf)
                e = int(np.argmin(col))                                   # first minimum
                ex = executors[e] if executors is not None else e
                d[g] = Strategy(ex, g, params[j, e, gi] if params is not None else None, float(T[j, e, gi]))
            else:
                failed = bool((T[j, :, gi] >= FAILED).any())
                d[g] = Strategy(None, g, None, FAILED if failed else NOT_PROFILED)
        out.append(d)
    return out


def solve_table(T, mask=None, gcount=None, presolved=None, interval=1000, timeout=500, *,
                chains: Optional[int] = None, rounds: Optional[int] = None, seed: int = 0,
                integer_starts: bool = True, engine=None, nodes: Optional[int] = None, devices=None,
                objective: str = "makespan", weights=None, due=None, release=None, penalty=None, scenarios=None):
    """solve() on the dense profiler tensor T[J][S][G] (+ mask of usable cells, + gcount[G] GPU counts).
    `objective` as for solve(): "makespan" or "completion" (sum of completion times); `weights` as for solve(),
    a sequence aligned with T's rows (the weighted sum of completion times, last_stats["weighted_completion"]);
    `due` as for solve() with objective="tardiness", "max_lateness" or "late_tasks" (last_stats as there), a sequence
    aligned with T's rows; `release` as for solve(), under every objective, a sequence aligned with T's rows
    (last_stats["total_flow_time"]).  objective="max_stretch" as for solve(), with p*_t the smallest cell of row t
    the search may propose, over every strategy (last_stats["max_stretch"] and ["mean_stretch"] from T's values).
    objective="squared_tardiness" (with `due`) and "squared_flow" as for solve(), with their last_stats from T's values.
    objective="late_penalty" and "completion_penalty" (with `due` and `penalty`, sequences aligned with T's rows) as
    for solve(), with their last_stats from T's values.  objective="worst_makespan" and "mean_makespan" with
    `scenarios`, an array [J][K] of factors aligned with T's rows, as for solve(), with their last_stats from T's
    values; likewise "worst_tardiness" and "mean_tardiness" (with `due`) and "worst_completion" and
    "mean_completion" (no `due`), each with `weights` optional.
    Every cell of T must be
    >= 0 (-0.0 counts as zero), +inf or a sentinel: a negative or NaN cell raises SolverError, with or without `mask`.

    The table goes to the device un-reduced (sb_set_table: min over strategies with the first-minimum rule
    and its arg-min on the device, PerformanceEvaluator.py:101-115); the search runs on the reduced view
    (a slower strategy at the same GPU count is dominated).  Returns the reference's 6-tuple
    (sta, tga, bss, bna, boa, makespan) — bss[t] is one-hot over the G gpu-count columns, the option order
    task.strategies has after profiling — plus strategy[J], the index of the winning strategy (executor) of
    each task's chosen cell.  For the same seed and population the plan equals solve() on the
    `strategies_from_table` view."""
    from .search import run_search
    _check_objective(objective)
    T = np.ascontiguousarray(T, dtype=np.float32)
    if T.ndim != 3:
        raise SolverError("T must be [J][S][G]")
    if np.isnan(T).any() or (T < 0).any():
        # the device refuses them too (sb_set_table): a negative hold cannot be list-scheduled, a NaN is no runtime
        raise SolverError("T holds a negative or NaN runtime: every cell must be >= 0, +inf or a sentinel")
    J, S, G = T.shape
    w64, w32 = _resolve_weights(weights, objective, J)
    d64, d32 = _resolve_due(due, objective, J)
    p64, p32 = _resolve_penalty(penalty, objective, J)
    f64, f32 = _resolve_scenarios(scenarios, objective, J)
    r64, r32 = _resolve_release(release, J)
    if J == 0:
        return [[[] for _ in range(NSLOT)]], [], [], [], [], 0.0, np.zeros(0, dtype=np.int64)
    gcount = list(range(1, G + 1)) if gcount is None else [int(g) for g in gcount]
    if len(gcount) != G or len(set(gcount)) != G or not all(1 <= g <= NSLOT for g in gcount):
        raise SolverError("gcount must hold %d distinct GPU counts in 1..%d" % (G, NSLOT))
    usable = np.isfinite(T) & (T >= 0) if mask is None else (np.asarray(mask, dtype=bool) & np.isfinite(T))
    if mask is None:
        usable &= T < NOT_PROFILED
    Tdev = np.where(usable, T, np.inf).astype(np.float32)
    for j in np.nonzero(~usable.reshape(J, -1).any(axis=1))[0]:
        Tdev[j] = np.where(np.isfinite(T[j]), T[j], np.inf)      # nothing usable: the sentinels are all it has
    if not np.isfinite(Tdev.reshape(J, -1)).any(axis=1).all():
        raise SolverError("a task has no finite cell in T")
    _check_horizon(Tdev, release=r64, tails=_tails(d32) if objective == "max_lateness" else None)
    if f32 is not None:
        _check_scenario_horizon(Tdev, f32, r64)
    if objective == "max_stretch":
        pstar, w32, d32 = _stretch_form(Tdev, r32)
    elif objective == "squared_flow":
        d32 = _release_due(r32, J)
    eng = engine if engine is not None else _engine(devices)
    nodes = int(_default_nodes() if nodes is None else nodes)
    eng.set_table(Tdev, gcount, sentinel=float("inf"), nodes=nodes)
    search_objective = _set_objective(eng, objective, w32, d32, r32, p32)
    if f32 is not None:
        eng.set_scenarios(f32)
    if chains is None:
        chains = int(os.environ.get("SATURN_B200_CHAINS", 0))
        if chains <= 0:
            wave = eng.search_wave(reduced=True, **({"objective": search_objective} if objective in _SCENARIO_ALL
                                                    else {}))
            chains = max(1, round((1 << 17) / wave)) * wave if wave > 0 else 1 << 17
    if rounds is None:
        rounds = int(os.environ.get("SATURN_B200_ROUNDS", 400))
    budget = min(float(os.environ.get("SATURN_B200_BUDGET_S", 20.0)), float(timeout))
    col_of_k = {g: gi for gi, g in enumerate(gcount)}
    warm = None
    if presolved is not None:
        class _Opt:                      # the option list a task has in this view: every gpu-count column
            strategies = {g: None for g in gcount}
        warm = candidate_from_arrays([_Opt] * J, presolved, nodes)
    res = run_search(eng, chains=chains, rounds=rounds, seed=seed, integer_starts=integer_starts, reduced=True,
                     time_budget_s=budget, patience=max(40, rounds // 4), warm=warm,
                     **({"objective": search_objective} if search_objective != "makespan" else {}))
    if objective in ("makespan", "max_lateness"):
        _check_horizon(Tdev, res.makespan)
    dec = eng.decode(res.opt, res.prio, integer_starts=integer_starts, reduced=True)
    gpus = dec["gpus"].astype(np.int64)
    chosen = np.array([col_of_k[int(k)] for k in gpus], dtype=np.int64)
    position = np.empty(J, dtype=np.int64)
    position[res.prio.astype(np.int64)] = np.arange(J)
    arrays = plan_to_arrays([G] * J, chosen, dec["start"], dec["slotmask"], position, nodes=nodes, node_of=dec["node"])
    strategy = dec["strategy"].astype(np.int64)
    rts = [float(T[j, strategy[j], chosen[j]]) for j in range(J)]
    if objective != "makespan":
        _check_horizon(Tdev, _plan_horizon(dec["start"], rts))
    makespan = max(float(dec["start"][j]) + rts[j] for j in range(J))
    global last_stats
    last_stats = {"candidates": res.evaluated, "rounds": res.rounds, "search_wall_s": res.wall_s,
                  "device_makespan": res.makespan, "makespan": makespan, "J": J, "chains": chains, "nodes": nodes,
                  "devices": len(getattr(eng, "engines", [eng])), "total_wall_s": None, "adopted": True,
                  "objective": objective, "total_completion": sum(float(dec["start"][j]) + rts[j] for j in range(J))}
    if w64 is not None:
        last_stats["weighted_completion"] = sum(w64[j] * (float(dec["start"][j]) + rts[j]) for j in range(J))
    if objective == "max_lateness":
        last_stats.update(_lateness_stats(dec["start"], rts, d64))
        last_stats["device_makespan"] = res.makespan - eng.due_shift
    elif objective == "late_tasks":
        last_stats.update(_late_count_stats(dec["start"], rts, w64, d64))
    elif objective == "max_stretch":
        last_stats.update(_stretch_stats(dec["start"], rts, pstar, r64))
    elif objective == "squared_tardiness":
        last_stats.update(_squared_stats(dec["start"], rts, w64, d64))
    elif objective == "squared_flow":
        last_stats.update(_squared_flow_stats(dec["start"], rts, w64, r64))
    elif objective == "late_penalty":
        last_stats.update(_late_penalty_stats(dec["start"], rts, w64, d64, p64))
    elif objective == "completion_penalty":
        last_stats.update(_completion_penalty_stats(dec["start"], rts, w64, d64, p64))
    elif objective in _SCENARIO_ALL:
        last_stats.update(_scenario_stats(rts, gpus, dec["node"], res.prio, f64, integer_starts, r64, w64, d64,
                                          objective))
        _check_horizon(Tdev, max(last_stats["scenario_makespans"]))
    elif d64 is not None:
        last_stats.update(_tardiness_stats(dec["start"], rts, w64, d64))
    if r64 is not None:
        last_stats.update(_flow_stats(dec["start"], rts, r64))
    return arrays + (makespan, strategy)


# ------------------------------------------------------------------------------------------ front
class FrontPoint(NamedTuple):
    """One plan of solve_front: the makespan cap it was solved under (an fp32 value), its makespan and its (weighted)
    sum of completion times (float64, the tasks' own runtimes), solve()'s 6-tuple and that solve's last_stats."""
    cap: float
    makespan: float
    completion: float
    plan: tuple
    stats: dict


def _plan_schedule(task_list, plan, T):
    """The chosen option index, start (float64) and slot runtime (fp32, the device table T's cell) of every task of
    a solve() plan."""
    sta, tga, bss, bna, _boa, _mk = plan
    opt = np.array([int(np.argmax(b)) for b in bss], dtype=np.int64)
    node = np.array([int(np.argmax(b)) for b in bna], dtype=np.int64)
    start = np.empty(len(task_list))
    rt32 = np.empty(len(task_list), dtype=np.float32)
    for t, task in enumerate(task_list):
        k = int(list(task.strategies.keys())[opt[t]])
        g = [i for i, v in enumerate(tga[t][node[t]]) if v == 1.0][0]
        start[t] = sta[node[t]][g][t]
        rt32[t] = T[t, 0, k - 1]
    return opt, start, rt32


def _device_makespan(task_list, plan, T):
    """A plan's makespan in the device's arithmetic: max_t fp32(start_t + rt_t) over the fp32 starts and table cells,
    the value the kernels' makespan and due-date comparisons see."""
    _opt, start, rt32 = _plan_schedule(task_list, plan, T)
    return float(np.max(start.astype(np.float32) + rt32))


def _plan_candidate(task_list, plan, nodes):
    """A solve() plan as the exact search candidate it was decoded from: reduced opt bytes and the list order that
    boa records (candidate_from_arrays orders by start time instead, which need not list-schedule to the same
    plan)."""
    _sta, _tga, bss, bna, boa, _mk = plan
    J = len(task_list)
    opt = np.zeros(J, dtype=np.uint8)
    for t, task in enumerate(task_list):
        k = int(list(task.strategies.keys())[int(np.argmax(bss[t]))])
        opt[t] = (k - 1) | ((int(np.argmax(bna[t])) << 3) if nodes > 1 else 0)
    before = np.array([[v == 1.0 for v in row] for row in boa], dtype=bool)   # before[a][b]: a precedes b
    return opt, np.argsort(before.sum(axis=0), kind="stable")


def solve_front(task_list, points=8, weights=None, release=None, nodes=None, devices=None, seed=0,
                integer_starts=True, timeout=500, engine=None, *, chains: Optional[int] = None,
                rounds: Optional[int] = None, **refused):
    """The trade-off between the makespan and the (weighted) sum of completion times: up to `points` plans, each the
    best sum_t w_t C_t found under a makespan cap, sorted by makespan ascending with the sum strictly descending.

    1. solve(objective="makespan"); its makespan in the device's fp32 arithmetic, M0, is the first cap.
    2. solve(objective="completion") (with `weights`, the weighted sum); its fp32 makespan is M1.
    3. For `points` - 2 caps evenly spaced strictly between M0 and M1 (fp32, ascending), solve(objective=
       "completion_penalty") with every due date at the cap and every penalty P, the smallest power of two
       >= sum_t w_t * 2^24 (the horizon every plan's times stay below): a plan over the cap then scores above every
       plan that meets it, so this minimises the sum subject to makespan <= cap (the epsilon-constraint method).
       Each search starts from the previous point's plan, which meets the larger cap.
    4. Every plan is rescored in float64 and the dominated ones are dropped.
    If M1 <= M0 the front is the completion plan alone.  Each point is a FrontPoint(cap, makespan, completion, plan,
    stats): `plan` is solve()'s 6-tuple (convert_into_comprehensible takes it unchanged), `stats` that solve's
    last_stats, `completion` the float64 sum_t w_t C_t (unit weights without `weights`).  A plan's float64 makespan
    can exceed its fp32 cap by the rounding of the device's fp32 start + runtime (half an fp32 ulp of the cap).

    `weights` and `release` as for solve(); `seed`, `integer_starts`, `timeout`, `engine`, `nodes`, `devices`,
    `chains` and `rounds` go to every solve.  points < 2, `due`, `penalty`, `hysteresis` or `presolved`, weights
    whose P breaks the penalty bound (J * P >= 2^126), and a plan whose fp32 makespan exceeds its cap raise
    SolverError."""
    if not isinstance(points, (int, np.integer)) or isinstance(points, bool) or points < 2:
        raise SolverError("solve_front needs points >= 2, not %r" % (points,))
    for name in ("due", "penalty", "hysteresis", "presolved"):
        if name in refused:
            raise SolverError("solve_front sets every due date and penalty itself and starts from its own plans: it "
                              "takes no %s" % name)
    if refused:
        raise TypeError("solve_front() got unexpected keyword argument(s) %s" % ", ".join(sorted(refused)))
    task_list = list(task_list)
    J = len(task_list)
    w64, w32 = _resolve_weights(weights, "completion", J, task_list)
    _resolve_release(release, J, task_list)
    if J == 0:
        return []
    wsum = float(np.sum(w32, dtype=np.float64)) if w32 is not None else float(J)
    m, e = math.frexp(wsum * FP32_EXACT_HORIZON)
    P = math.ldexp(1.0, e - 1 if m == 0.5 else e)
    if not J * P < 2.0 ** 126:
        raise SolverError("solve_front's penalty P = %g (the smallest power of two >= sum(weights) * 2^24) gives "
                          "J * P >= 2^126; scale the weights down" % P)
    nodes = int(_default_nodes() if nodes is None else nodes)
    T, _usable, _optindex = build_table(task_list)
    common = dict(seed=seed, integer_starts=integer_starts, timeout=timeout, engine=engine, nodes=nodes,
                  devices=devices, chains=chains, rounds=rounds, release=release)

    def run(objective, cap=None, **extra):
        plan = solve(task_list, None, objective=objective, **common, **extra)
        return (cap if cap is not None else _device_makespan(task_list, plan, T)), plan, dict(last_stats)

    mk = run("makespan")
    cp = run("completion", weights=weights)
    if not cp[0] > mk[0]:
        runs = [cp]
    else:
        caps = []
        for i in range(1, points - 1):
            c = float(np.float32(mk[0] + (cp[0] - mk[0]) * i / (points - 1)))
            if mk[0] < c < cp[0] and (not caps or c > caps[-1]):
                caps.append(c)
        runs = [mk]
        for c in caps:
            runs.append(run("completion_penalty", cap=c, weights=weights, due=[c] * J, penalty=[P] * J,
                            _warm=_plan_candidate(task_list, runs[-1][1], nodes)))
            if _device_makespan(task_list, runs[-1][1], T) > c:
                raise SolverError("solve_front: the plan for the makespan cap %r has fp32 makespan %r over its cap"
                                  % (c, _device_makespan(task_list, runs[-1][1], T)))
        runs.append(cp)
    w = w64 if w64 is not None else [1.0] * J
    found = []
    for cap, plan, stats in runs:
        opt, start, _rt32 = _plan_schedule(task_list, plan, T)
        comp = [start[t] + float(list(task.strategies.values())[opt[t]].runtime) for t, task in enumerate(task_list)]
        found.append(FrontPoint(cap, max(comp), sum(wi * c for wi, c in zip(w, comp)), plan, stats))
    front = []
    for p in sorted(found, key=lambda p: (p.makespan, p.completion)):
        if not front or p.completion < front[-1].completion:
            front.append(p)
    return front


# ------------------------------------------------------------------------------------------ decode
def convert_into_comprehensible(task_list, bss, boa, tga, bna, sta):
    """Drop-in for saturn.solver.convert_into_comprehensible (milp.py:448-513).

    Returns (node_per_task: dict Task -> int, task_dependency_dict: defaultdict Task -> [Task],
    start_time_per_task: list[float]) and, as the reference does, records the chosen option on
    each task via task.select_strategy (milp.py:475-486).  The O(J^2 * G) Python triple loop of
    milp.py:492-511 is replaced by bit-mask arithmetic; results are identical.
    """
    task_list = list(task_list)
    J = len(task_list)
    node_per_task = {}
    nodes = np.zeros(J, dtype=np.int64)
    for idx, task in enumerate(task_list):
        n = np.argmax(bna[idx])
        node_per_task[task] = n
        nodes[idx] = int(n)
    for idx, task in enumerate(task_list):
        want = int(np.argmax(bss[idx]))
        for ctr, strat in enumerate(task.strategies.values()):
            if ctr == want:
                task.select_strategy(strat)
                break
    # occupancy of each task on its node: round(tga[t][n][g]) == 1  (milp.py:490-497), as one array operation
    tga_a = np.asarray(tga, dtype=np.float64).reshape(J, -1, NSLOT)
    occ = np.rint(tga_a[np.arange(J), nodes, :]) == 1                                # [J][8]
    if not occ.any(axis=1).all():
        raise SolverError("task %d occupies no GPU in tga" % int(np.argmin(occ.any(axis=1))))
    first = np.argmax(occ, axis=1)
    masks = (occ.astype(np.int64) << np.arange(NSLOT)[None, :]).sum(axis=1)
    start_time_per_task = [sta[int(nodes[idx])][int(first[idx])][idx] for idx in range(J)]
    task_dependency_dict = defaultdict(list)
    if J > 1:
        # before[p][t]: round(boa[p][t]) == 1; the diagonal (None in the reference, milp.py:263-270) never counts
        b = np.array(boa, dtype=object)
        b[np.equal(b, None)] = 0.0
        before = np.rint(b.astype(np.float64)) == 1
        np.fill_diagonal(before, False)
        share = ((masks[:, None] & masks[None, :]) != 0) & (nodes[:, None] == nodes[None, :])
        dep = before & share                       # dep[p][t]: p must finish before t launches
        for idx in np.nonzero(dep.any(axis=0))[0]:
            task_dependency_dict[task_list[int(idx)]] = [task_list[int(p)] for p in np.nonzero(dep[:, idx])[0]]
    return node_per_task, task_dependency_dict, start_time_per_task
