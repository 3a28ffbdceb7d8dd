"""`saturn.orchestrate` drop-in: the interval loop that calls the solver.

Mirrors the call structure of the reference (saturn/orchestrator.py:32-75): an initial blocking
solve, then per interval  forecast -> re-solve (overlapped with execution in the reference)
-> execute -> adopt the new plan, until every task has finished.  The solver is this
repository's GPU path; `forecast` restates saturn/executor/executor.py:132-178.  Executing the
training slices themselves (Ray actors + user-defined parallelisms, executor.py:88-129) is out
of scope for this hot-path build: pass `execute_fn`, or have the reference's Ray executor
importable as `saturn_reference_executor.execute`; without either, the loop runs the plan in
simulated time (useful for what-if planning and for the tests).
"""
from __future__ import annotations

import logging
from collections.abc import Mapping
from typing import Callable, Optional

from .solver import SolverError, convert_into_comprehensible, solve


def forecast(task_list, interval, interval_sta):
    """Which tasks run in the coming interval, for how many batches, and which finish.

    Restatement of executor.py:132-178, including its side effects: every strategy's runtime of a
    running task is reduced by the share of work forecast to complete, and total_batches is
    decremented (the solver sees the shrunken table at the next solve).
    Returns (relevant_tasks, batches_to_run, completed_tasks).
    """
    relevant, budget = [], []
    for task, st in zip(task_list, interval_sta):
        if st < interval:
            relevant.append(task)
            budget.append(interval - st)
    batches_to_run = []
    for task, window in zip(relevant, budget):
        per_batch = task.selected_strategy.runtime / task.total_batches
        batches_to_run.append(min(task.total_batches, window // per_batch))
    completed = set()
    for task, nb in zip(relevant, batches_to_run):
        for g_count, strat in task.strategies.items():
            task.strategies[g_count].runtime -= max(0, (strat.runtime / task.total_batches) * nb)
        task.total_batches = max(0, task.total_batches - nb)
        if task.total_batches <= 0:
            completed.add(task)
            logging.info("Task %s will finish entirely in the current interval.", task.name)
    return relevant, batches_to_run, completed


def orchestrate(task_list, log=False, interval=1000, gurobi=True, *,
                execute_fn: Optional[Callable] = None, max_intervals: Optional[int] = None, solver_kwargs=None):
    """Plan and run `task_list` to completion in intervals of `interval` seconds.

    Same positional signature as the reference (orchestrator.py:32).  `execute_fn(relevant_tasks,
    batches_to_run, interval, node_per_task, task_dependency_dict)` stands in for
    saturn.executor.execute; returns the list of per-interval records (plan makespan, tasks run).

    A `due` mapping Task -> due date in `solver_kwargs` (objective="tardiness", "max_lateness", "late_tasks",
    "squared_tardiness", "late_penalty", "completion_penalty", "worst_tardiness" or "mean_tardiness") is
    measured from the first plan's t = 0: the solve for interval n plans from n * interval on, so it receives
    {t: d - n * interval}, and the lateness each solve reports is against the original due dates (both sides shift
    alike).  A sequence `due` raises SolverError, since the task list shrinks from interval to interval.  A `release`
    mapping Task -> release date is shifted the same way, {t: r - n * interval}; a sequence `release` raises
    SolverError.  Under objective="max_stretch" the shifted release dates are what each solve measures stretch
    from, and each interval's fastest runtime p*_t comes from the runtimes `forecast` has shrunk: each solve
    minimises the stretch of the work that remains, not of the whole task.  Under objective="squared_tardiness" the
    shifted due dates leave every tardiness unchanged (C and d move alike).  Under objective="squared_flow" each solve
    measures flow from the shifted release dates, clamped at the interval's t = 0: a task released before the
    interval counts its flow from the interval's start, so each solve minimises the squares of the waits that
    remain, not of the whole flow time.  Under objective="late_penalty" and "completion_penalty" a `penalty` mapping
    Task -> penalty is passed to every solve unchanged: a penalty is what missing the due date costs, whenever the
    plan is made; a sequence `penalty` raises SolverError, as a sequence `due` does.  Under
    objective="worst_makespan", "mean_makespan", "worst_tardiness", "mean_tardiness", "worst_completion" and
    "mean_completion" a `scenarios` mapping Task -> K runtime factors is passed to every solve unchanged: a factor
    scales a task's remaining work as it scales the whole task; a sequence `scenarios` raises SolverError, as a
    sequence `due` does.  Under "worst_tardiness" and "mean_tardiness" the due dates shift as above, so every
    scenario's tardiness is against the original due dates; "worst_completion" and "mean_completion" take no due
    dates and, like "completion", count each interval's completion times from its start.
    """
    logging.basicConfig(level=logging.INFO if log else logging.WARNING,
                        format="%(asctime)s %(levelname)-8s %(message)s", datefmt="%Y-%m-%d %H:%M:%S")
    kw = dict(solver_kwargs or {})
    due = kw.pop("due", None)
    if due is not None and not isinstance(due, Mapping):
        raise SolverError("orchestrate() needs due as a mapping Task -> due date: its task list shrinks every interval")
    if kw.get("penalty") is not None and not isinstance(kw["penalty"], Mapping):
        raise SolverError("orchestrate() needs penalty as a mapping Task -> penalty: its task list shrinks every "
                          "interval")
    if kw.get("scenarios") is not None and not isinstance(kw["scenarios"], Mapping):
        raise SolverError("orchestrate() needs scenarios as a mapping Task -> runtime factors: its task list shrinks "
                          "every interval")
    release = kw.pop("release", None)
    if release is not None and not isinstance(release, Mapping):
        raise SolverError("orchestrate() needs release as a mapping Task -> release date: its task list shrinks "
                          "every interval")

    def kw_at(n):  # the solver arguments of the plan for interval n (whose t = 0 is n * interval)
        out = dict(kw)
        if due is not None:
            out["due"] = {t: d - n * interval for t, d in due.items()}
        if release is not None:
            out["release"] = {t: r - n * interval for t, r in release.items()}
        return out

    task_list = list(task_list)
    records = []
    presolved = solve(task_list, None, gurobi=gurobi, interval=interval, timeout=max(1, interval // 2), **kw_at(0))
    sta, tga, bss, bna, boa, makespan = presolved
    npt, tdd, sta_comp = convert_into_comprehensible(task_list, bss, boa, tga, bna, sta)
    n = 0
    while len(task_list) > 0:
        rtt, btr, done = forecast(task_list, interval, sta_comp)
        logging.info("Launching %s in this interval.", [t.name for t in rtt])
        records.append({"interval": n, "makespan": makespan, "launched": [t.name for t in rtt],
                        "batches": list(btr), "finishing": sorted(t.name for t in done)})
        task_list = [t for t in task_list if t not in done]
        if execute_fn is not None:
            execute_fn(rtt, btr, interval, npt, tdd)
        if len(task_list) == 0:
            break
        presolved = solve(task_list, presolved, gurobi=gurobi, interval=interval,
                          timeout=max(1, interval // 2), **kw_at(n + 1))
        sta, tga, bss, bna, boa, makespan = presolved
        npt, tdd, sta_comp = convert_into_comprehensible(task_list, bss, boa, tga, bna, sta)
        n += 1
        if max_intervals is not None and n >= max_intervals:
            break
    return records
