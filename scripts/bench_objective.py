"""Cost and effect of the sum-of-completion-times objectives (plain and weighted), of the weighted tardiness, of the
maximum lateness, of the (weighted) number of late tasks, of the maximum stretch and of release dates on one GPU;
prints one JSON line.

    python scripts/bench_objective.py [--steps 200] [--warmup 20] [--solve-chains 0] [--solve-rounds 400]
                                      [--only max_stretch | squared | late_penalty | completion_penalty | scenarios]

kernel: sb_eval on bench.py's C4 batch (J = 256, S = 8, 946,176 candidates, the same seeded inputs, integer
        starts), scored for the makespan, the sum of completion times, the weighted sum (seeded weights) and the
        weighted tardiness (the same weights, seeded due dates), and the release twins of the makespan and the
        weighted tardiness (seeded integer release dates in [0, 20000) s, SB_FLAG_RELEASE, a second handle on the
        same device), the maximum lateness (the tail makespan over the same due dates) and the weighted late count
        (the same weights and due dates) and the weighted maximum tardiness (the same weights and due dates), the
        nine launches alternated in one process (the order rotates every step) and timed with CUDA events; median
        of --steps launches each.
solve:  solve() wall time on a 256-task set (synthetic table, seed 3, 4 strategies) for the makespan, the sum of
        completion times and the weighted sum (seeded weights: 32 tasks of weight 8, the rest 1), each plan scored
        on all three measures (float64, the tasks' own runtimes); and the total tardiness (unit weights, seeded
        integer due dates in [0, 200000) s): its tardiness and late tasks against those of the makespan and
        completion plans; the maximum lateness (the same due dates): its L_max and late tasks against those of
        the tardiness and makespan plans; and the number of late tasks, unweighted and weighted (the same due dates
        and weights), every plan scored on late tasks, weighted late tasks, tardiness and L_max.  late_unit compares
        the late-count search's temperature unit, sum w (shipped), with the mean weight sum w / J (the same solve with
        t_start and t_end divided by J).
release: the same 256-task set with seeded release dates in [0, 0.5 x the makespan plan's makespan): per objective
        (makespan, completion, tardiness) the release-aware plan (solve(release=...)) against the release-blind plan
        (solve() without them, its options and list order rescored under the release rule), on makespan, total flow
        time sum_t (C_t - max(r_t, 0)) and, for the tardiness objective, the tardiness; all in float64.
stretch: the same 256-task set and release dates: solve(objective="max_stretch") against the completion, makespan
        and completion-with-w = 1 / p* plans (all release-aware), each rescored in float64 on max stretch, mean
        stretch and makespan (stretch (C_t - max(r_t, 0)) / p*_t, p*_t the task's fastest proposable runtime).
--only max_stretch times only the weighted tardiness and the weighted maximum tardiness and runs only the stretch
comparison.
--only squared times only the weighted tardiness and the weighted squared tardiness (the same weights and due dates),
alternated as above, and runs only the squared-flow comparison: on the same 256-task set and release dates,
solve(objective="squared_flow") against the completion, max_stretch and makespan plans (all release-aware), each
rescored in float64 on sum_t F_t^2, mean F_t and max F_t, the flow time F_t = C_t - max(r_t, 0).
--only late_penalty times only the weighted tardiness and the weighted late penalty (the same weights and due dates,
seeded integer penalties in [0, 100000) s), alternated as above, and runs only the late-penalty comparison: on the
256-task set with the seeded integer due dates of the late-count row and seeded integer penalties in [0, 100000),
solve(objective="late_penalty") against the tardiness, late_tasks and completion plans, each rescored in float64 on
the cost sum_t [C_t > d_t] (p_t + C_t - d_t), the late tasks and the tardiness.
--only completion_penalty times only the weighted completion and the weighted completion penalty (the same weights,
the due dates of the kernel rows, seeded integer penalties in [0, 100000) s), alternated as above, and runs only
solve_front(points=8) on the 256-task set with the release dates of the stretch comparison: per point its cap, its
makespan and its mean flow time (C_t - max(r_t, 0)) in float64, and the front's total wall time.
--only scenarios times, on the same C4 batch read through the reduced table (opt bytes k - 1), the makespan and the
worst makespan over K = 1, 4 and 8 seeded log-normal scenarios (sigma 0.3, median 1) on the two routes that score the
scenario forms: the generic kernel on job-indexed rows and the position-major kernel on rows by position, the eight
launches alternated as above.  Then solve() on the 256-task set with K = 8 seeded log-normal factors per task (sigma
0.3, median 1): the worst- and mean-makespan plans against the nominal makespan plan, each rescored in float64 under
the same 8 scenarios and under 64 held-out scenarios drawn from the same distribution (another seed): the worst and
mean makespan over each set, and the nominal makespan.
--only scenario_tardiness times, on the same C4 batch read through the reduced table, the weighted tardiness on its
normal route (the tile kernel on job-indexed rows, and the position-major kernel on rows by position) and the weighted
mean tardiness over K = 1, 4 and 8 seeded log-normal scenarios on the two scenario routes (the generic kernel on
job-indexed rows, the position-major kernel on rows by position), with the weights and due dates of the kernel rows,
the eight launches alternated as above.  Then solve() on the 256-task set with the seeded integer due dates of the
tardiness row and K = 8 seeded log-normal factors per task (sigma 0.3, median 1): the mean-tardiness plan against the
nominal tardiness plan, and the mean-completion plan against the nominal completion plan, each rescored in float64
under the same 8 scenarios and under 64 held-out scenarios drawn from the same distribution (another seed): the mean
and worst total tardiness (or completion time) over each set, and the nominal value.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi, read-only queries), and with
--only scenario_tardiness also the SM clock at the end of the kernel timing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card(index):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:  # noqa: BLE001 - the measurement still stands, the card is then named by torch only
        import torch
        return {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--solve-chains", type=int, default=0, help="0 = solve()'s default population")
    ap.add_argument("--solve-rounds", type=int, default=400)
    ap.add_argument("--only", choices=("all", "max_stretch", "squared", "late_penalty", "completion_penalty",
                                       "scenarios", "scenario_tardiness"), default="all")
    args = ap.parse_args()
    if args.only == "scenarios":
        scenarios_main(args)
        return
    if args.only == "scenario_tardiness":
        scenario_tardiness_main(args)
        return
    import numpy as np
    import torch
    from oracle import ref_eval as R
    from saturn_b200 import solver as S
    from saturn_b200.engine import Engine, random_candidates
    from saturn_b200.synth import synth_table
    torch.cuda.set_device(0)
    eng = Engine(0)
    J, Sx, G = 256, 8, 8
    B = 132 * 8 * 32 * 28                                   # bench.py's B_PER_GPU
    T, valid = synth_table(J, Sx, G, seed=0)
    eng.set_table(T)
    opt, prio = random_candidates(eng, B, valid, seed=1)
    eng.set_weights(np.random.default_rng(2).choice([1.0, 2.0, 3.0, 5.0, 8.0, 0.25, 0.5, 1.5], size=J))
    eng.set_due(np.random.default_rng(3).integers(0, 20000, size=J))
    eng_r = Engine(0)                                       # the same inputs, plus release dates
    eng_r.set_table(T)
    eng_r.set_weights(eng.weights)
    eng_r.set_due(eng.due)
    eng_r.set_release(np.random.default_rng(5).integers(0, 20000, size=J))
    out = torch.empty(B, dtype=torch.float32, device=eng.device)
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=eng.device)
    objs = ("makespan", "completion", "weighted_completion", "weighted_tardiness", "release_makespan",
            "release_weighted_tardiness", "max_lateness", "weighted_late_tasks", "weighted_max_tardiness")
    if args.only == "max_stretch":
        objs = ("weighted_tardiness", "weighted_max_tardiness")
    if args.only == "squared":
        objs = ("weighted_tardiness", "weighted_squared_tardiness")
    if args.only == "late_penalty":
        objs = ("weighted_tardiness", "weighted_late_penalty")
        eng.set_penalty(np.random.default_rng(7).integers(0, 100000, size=J))
    if args.only == "completion_penalty":
        objs = ("weighted_completion", "weighted_completion_penalty")
        eng.set_penalty(np.random.default_rng(7).integers(0, 100000, size=J))
    times = {o: [] for o in objs}
    for i in range(args.warmup + args.steps):
        for obj in objs[i % len(objs):] + objs[:i % len(objs)]:
            e = eng_r if obj.startswith("release_") else eng
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            e.eval(opt, prio, out=out, best_key=key, objective=obj.replace("release_", ""))
            b.record()
            b.synchronize()
            if i >= args.warmup:
                times[obj].append(a.elapsed_time(b))
    path = eng.last_eval_path()
    assert args.only != "all" or eng_r.last_eval_path() == path
    kernel = {o: {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
                  "p90_ms": float(np.percentile(t, 90)), "candidates_per_s": B / (float(np.median(t)) * 1e-3)}
              for o, t in times.items()}
    if args.only == "completion_penalty":
        kernel["completion_penalty_over_weighted_completion"] = (kernel["weighted_completion_penalty"]["median_ms"] /
                                                                 kernel["weighted_completion"]["median_ms"])
        kernel.update(B=B, J=J, S=Sx, path=path, steps=args.steps)
        del opt, prio, out
        eng_r.close()
        torch.cuda.empty_cache()
        tasks = _tasks256()
        kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                                   if args.solve_chains else {}))
        makespan = S.solve(tasks, None, **kw)[5]
        print(json.dumps({"card": card(0), "kernel": kernel, "front": front_effect(S, tasks, makespan, kw)}))
        eng.close()
        return
    if args.only == "late_penalty":
        kernel["late_penalty_over_weighted_tardiness"] = (kernel["weighted_late_penalty"]["median_ms"] /
                                                          kernel["weighted_tardiness"]["median_ms"])
        kernel.update(B=B, J=J, S=Sx, path=path, steps=args.steps)
        del opt, prio, out
        eng_r.close()
        torch.cuda.empty_cache()
        kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                                   if args.solve_chains else {}))
        print(json.dumps({"card": card(0), "kernel": kernel, "late_penalty": late_penalty_effect(S, R, _tasks256(),
                                                                                                   kw)}))
        eng.close()
        return
    if args.only == "squared":
        kernel["squared_over_weighted_tardiness"] = (kernel["weighted_squared_tardiness"]["median_ms"] /
                                                     kernel["weighted_tardiness"]["median_ms"])
        kernel.update(B=B, J=J, S=Sx, path=path, steps=args.steps)
        del opt, prio, out
        eng_r.close()
        torch.cuda.empty_cache()
        tasks = _tasks256()
        kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                                   if args.solve_chains else {}))
        makespan = S.solve(tasks, None, **kw)[5]
        print(json.dumps({"card": card(0), "kernel": kernel, "squared_flow": squared_effect(S, R, tasks, makespan, kw)}))
        eng.close()
        return
    kernel["max_tardiness_over_weighted_tardiness"] = (kernel["weighted_max_tardiness"]["median_ms"] /
                                                       kernel["weighted_tardiness"]["median_ms"])
    if args.only == "max_stretch":
        kernel.update(B=B, J=J, S=Sx, path=path, steps=args.steps)
        del opt, prio, out
        eng_r.close()
        torch.cuda.empty_cache()
        tasks = _tasks256()
        kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                                   if args.solve_chains else {}))
        makespan = S.solve(tasks, None, **kw)[5]
        print(json.dumps({"card": card(0), "kernel": kernel, "stretch": stretch_effect(S, R, tasks, makespan, kw)}))
        eng.close()
        return
    kernel["completion_over_makespan"] = kernel["completion"]["median_ms"] / kernel["makespan"]["median_ms"]
    kernel["weighted_over_completion"] = kernel["weighted_completion"]["median_ms"] / kernel["completion"]["median_ms"]
    kernel["tardiness_over_weighted"] = kernel["weighted_tardiness"]["median_ms"] / kernel["weighted_completion"]["median_ms"]
    kernel["release_over_makespan"] = kernel["release_makespan"]["median_ms"] / kernel["makespan"]["median_ms"]
    kernel["release_over_tardiness"] = (kernel["release_weighted_tardiness"]["median_ms"] /
                                        kernel["weighted_tardiness"]["median_ms"])
    kernel["max_lateness_over_makespan"] = kernel["max_lateness"]["median_ms"] / kernel["makespan"]["median_ms"]
    kernel["late_tasks_over_weighted_tardiness"] = (kernel["weighted_late_tasks"]["median_ms"] /
                                                    kernel["weighted_tardiness"]["median_ms"])
    kernel.update(B=B, J=J, S=Sx, path=path, steps=args.steps)
    del opt, prio, out
    eng_r.close()
    torch.cuda.empty_cache()

    tasks = _tasks256()
    kw = dict(rounds=args.solve_rounds, seed=1, engine=eng)
    if args.solve_chains:
        kw["chains"] = args.solve_chains
    S.solve(tasks, None, rounds=4, engine=eng)               # first launches load the kernels
    S.solve(tasks, None, rounds=4, engine=eng, objective="completion")
    w = [8.0 if j % 8 == 0 else 1.0 for j in range(len(tasks))]
    S.solve(tasks, None, rounds=4, engine=eng, objective="completion", weights=w)
    due = [float(x) for x in np.random.default_rng(4).integers(0, 200000, size=len(tasks))]
    S.solve(tasks, None, rounds=4, engine=eng, objective="tardiness", due=due)
    S.solve(tasks, None, rounds=4, engine=eng, objective="max_lateness", due=due)
    S.solve(tasks, None, rounds=4, engine=eng, objective="late_tasks", due=due)
    S.solve(tasks, None, rounds=4, engine=eng, objective="late_tasks", due=due, weights=w)
    solve = {}
    for name, obj, weights in (("makespan", "makespan", None), ("completion", "completion", None),
                               ("weighted_completion", "completion", w), ("tardiness", "tardiness", None),
                               ("max_lateness", "max_lateness", None), ("late_tasks", "late_tasks", None),
                               ("weighted_late_tasks", "late_tasks", w)):
        t0 = time.perf_counter()
        res = S.solve(tasks, None, objective=obj, weights=weights,
                      **({"due": due} if obj in ("tardiness", "max_lateness", "late_tasks") else {}), **kw)
        wall = time.perf_counter() - t0
        st = S.last_stats
        # the plan scored on all three measures, in float64 from its starts and the tasks' own runtimes
        tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
        comp = [p[0] + p[2] for p in R.plan_from_arrays(tuples, res[0], res[1], res[2], res[3])]
        solve[name] = {"wall_s": wall, "makespan": res[5], "total_completion": st["total_completion"],
                       "mean_completion": st["total_completion"] / len(tasks),
                       "weighted_completion": sum(wi * c for wi, c in zip(w, comp)),
                       "heavy_mean_completion": float(np.mean([c for wi, c in zip(w, comp) if wi > 1])),
                       "tardiness": sum(max(0.0, c - d) for c, d in zip(comp, due)),
                       "late_tasks": sum(1 for c, d in zip(comp, due) if c > d),
                       "max_lateness": max(c - d for c, d in zip(comp, due)),
                       "weighted_late_tasks": sum(wi for wi, c, d in zip(w, comp, due) if c > d),
                       "rounds": st["rounds"], "candidates": st["candidates"]}
    late_unit = late_unit_effect(S, R, tasks, due, w, kw)
    print(json.dumps({"card": card(0), "kernel": kernel, "solve": solve, "late_unit": late_unit,
                      "release": release_effect(S, R, tasks, due, solve["makespan"]["makespan"], kw),
                      "stretch": stretch_effect(S, R, tasks, solve["makespan"]["makespan"], kw)}))
    eng.close()


def _median(t):
    import numpy as np
    return {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
            "p90_ms": float(np.percentile(t, 90))}


def scenarios_main(args):
    import numpy as np
    import torch
    from saturn_b200 import solver as S
    from saturn_b200.engine import Engine, opt_by_position, random_candidates
    from saturn_b200.synth import synth_table
    torch.cuda.set_device(0)
    J, Sx, G = 256, 8, 8
    B = 132 * 8 * 32 * 28                                   # bench.py's B_PER_GPU
    T, valid = synth_table(J, Sx, G, seed=0)
    opt, prio = random_candidates(Engine(0).set_table(T), B, valid, seed=1)
    opt &= 7                                                # the reduced table's opt bytes: k - 1
    obp = opt_by_position(opt, prio)
    out = torch.empty(B, dtype=torch.float32, device=opt.device)
    engines = {}
    for K in (1, 4, 8):                                     # one handle per scenario count, the same table
        e = Engine(0)
        e.set_table(T)
        e.set_scenarios(np.random.default_rng(40 + K).lognormal(0.0, 0.3, size=(K, J)))
        engines[K] = e
    runs = []
    for route, o, kw in (("generic", opt, {}), ("position_major", obp, {"by_position": True})):
        runs.append((route + "/makespan", engines[1], o,
                     dict(kw, objective="makespan", **({"_force_generic": True} if route == "generic" else {}))))
        for K in (1, 4, 8):
            runs.append((route + "/worst_K%d" % K, engines[K], o, dict(kw, objective="worst_makespan")))
    times = {name: [] for name, _, _, _ in runs}
    paths = {}
    for i in range(args.warmup + args.steps):
        for name, e, o, kw in runs[i % len(runs):] + runs[:i % len(runs)]:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            e.eval(o, prio, out=out, reduced=True, **kw)
            b.record()
            b.synchronize()
            paths[name] = e.last_eval_path()
            if i >= args.warmup:
                times[name].append(a.elapsed_time(b))
    kernel = {name: dict(_median(t), path=paths[name]) for name, t in times.items()}
    for route in ("generic", "position_major"):
        base = kernel[route + "/makespan"]["median_ms"]
        for K in (1, 4, 8):
            kernel[route + "/worst_K%d" % K]["over_makespan"] = kernel[route + "/worst_K%d" % K]["median_ms"] / base
    kernel.update(B=B, J=J, S=Sx, steps=args.steps)
    del opt, prio, obp, out
    for e in engines.values():
        e.close()
    torch.cuda.empty_cache()

    eng = Engine(0)
    tasks = _tasks256()
    J = len(tasks)
    f8 = np.random.default_rng(50).lognormal(0.0, 0.3, size=(J, 8))
    held = np.random.default_rng(51).lognormal(0.0, 0.3, size=(64, J))
    kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                               if args.solve_chains else {}))

    def rescore(plan):
        opt, order = S._plan_candidate(tasks, plan, 1)
        gpus = (opt & 7).astype(np.int64) + 1
        rts = [float(t.strategies[int(g)].runtime) for t, g in zip(tasks, gpus)]
        node = np.zeros(J, dtype=np.int64)
        same = S._scenario_stats(rts, gpus, node, order, f8.T, True)
        other = S._scenario_stats(rts, gpus, node, order, held, True)
        return {"nominal_makespan": plan[5], "worst_8": same["worst_makespan"], "mean_8": same["mean_makespan"],
                "worst_64_held_out": other["worst_makespan"], "mean_64_held_out": other["mean_makespan"]}
    solve = {}
    for name, obj in (("makespan", "makespan"), ("worst_makespan", "worst_makespan"), ("mean_makespan", "mean_makespan")):
        t0 = time.perf_counter()
        plan = S.solve(tasks, None, objective=obj, **({"scenarios": f8} if obj != "makespan" else {}), **kw)
        wall = time.perf_counter() - t0
        solve[name] = dict(rescore(plan), wall_s=wall, rounds=S.last_stats["rounds"],
                           candidates=S.last_stats["candidates"])
    print(json.dumps({"card": card(0), "kernel": kernel, "scenarios": solve}))
    eng.close()


def _sm_clock(index):
    """The SM clock now, in MHz (a read-only nvidia-smi query), or None."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out)
    except Exception:  # noqa: BLE001
        return None


def scenario_tardiness_main(args):
    import numpy as np
    import torch
    from saturn_b200 import solver as S
    from saturn_b200.engine import Engine, opt_by_position, random_candidates
    from saturn_b200.synth import synth_table
    torch.cuda.set_device(0)
    J, Sx, G = 256, 8, 8
    B = 132 * 8 * 32 * 28                                   # bench.py's B_PER_GPU
    T, valid = synth_table(J, Sx, G, seed=0)
    opt, prio = random_candidates(Engine(0).set_table(T), B, valid, seed=1)
    opt &= 7                                                # the reduced table's opt bytes: k - 1
    obp = opt_by_position(opt, prio)
    out = torch.empty(B, dtype=torch.float32, device=opt.device)
    w = np.random.default_rng(2).choice([1.0, 2.0, 3.0, 5.0, 8.0, 0.25, 0.5, 1.5], size=J)
    d = np.random.default_rng(3).integers(0, 20000, size=J)
    engines = {}
    for K in (1, 4, 8):                                     # one handle per scenario count, the same inputs
        e = Engine(0)
        e.set_table(T)
        e.set_weights(w)
        e.set_due(d)
        e.set_scenarios(np.random.default_rng(40 + K).lognormal(0.0, 0.3, size=(K, J)))
        engines[K] = e
    runs = []
    for route, o, kw in (("generic", opt, {}), ("position_major", obp, {"by_position": True})):
        runs.append((route + "/weighted_tardiness", engines[1], o, dict(kw, objective="weighted_tardiness")))
        for K in (1, 4, 8):
            runs.append((route + "/weighted_mean_K%d" % K, engines[K], o, dict(kw, objective="weighted_mean_tardiness")))
    times = {name: [] for name, _, _, _ in runs}
    paths = {}
    for i in range(args.warmup + args.steps):
        for name, e, o, kw in runs[i % len(runs):] + runs[:i % len(runs)]:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            e.eval(o, prio, out=out, reduced=True, **kw)
            b.record()
            b.synchronize()
            paths[name] = e.last_eval_path()
            if i >= args.warmup:
                times[name].append(a.elapsed_time(b))
    sm_clock = _sm_clock(0)
    kernel = {name: dict(_median(t), path=paths[name]) for name, t in times.items()}
    for route in ("generic", "position_major"):
        base = kernel[route + "/weighted_tardiness"]["median_ms"]
        for K in (1, 4, 8):
            kernel[route + "/weighted_mean_K%d" % K]["over_tardiness"] = \
                kernel[route + "/weighted_mean_K%d" % K]["median_ms"] / base
    kernel.update(B=B, J=J, S=Sx, steps=args.steps, sm_clock_mhz_after=sm_clock)
    del opt, prio, obp, out
    for e in engines.values():
        e.close()
    torch.cuda.empty_cache()

    eng = Engine(0)
    tasks = _tasks256()
    J = len(tasks)
    due = [float(x) for x in np.random.default_rng(4).integers(0, 200000, size=J)]
    f8 = np.random.default_rng(50).lognormal(0.0, 0.3, size=(J, 8))
    held = np.random.default_rng(51).lognormal(0.0, 0.3, size=(64, J))
    kw = dict(rounds=args.solve_rounds, seed=1, engine=eng, **({"chains": args.solve_chains}
                                                               if args.solve_chains else {}))

    def rescore(plan, what):
        opt, order = S._plan_candidate(tasks, plan, 1)
        gpus = (opt & 7).astype(np.int64) + 1
        rts = [float(t.strategies[int(g)].runtime) for t, g in zip(tasks, gpus)]
        node = np.zeros(J, dtype=np.int64)
        dd = due if what == "tardiness" else None
        obj = "mean_" + what
        same = S._scenario_stats(rts, gpus, node, order, f8.T, True, None, None, dd, obj)
        other = S._scenario_stats(rts, gpus, node, order, held, True, None, None, dd, obj)
        nominal = S._scenario_stats(rts, gpus, node, order, np.ones((1, J)), True, None, None, dd, obj)
        return {"nominal": nominal["mean_" + what], "mean_8": same["mean_" + what], "worst_8": same["worst_" + what],
                "mean_64_held_out": other["mean_" + what], "worst_64_held_out": other["worst_" + what],
                "nominal_makespan": plan[5]}
    solve = {}
    for name, obj, what in (("tardiness", "tardiness", "tardiness"), ("mean_tardiness", "mean_tardiness", "tardiness"),
                            ("completion", "completion", "completion"),
                            ("mean_completion", "mean_completion", "completion")):
        okw = dict(kw)
        if what == "tardiness":
            okw["due"] = due
        if obj.startswith("mean_"):
            okw["scenarios"] = f8
        t0 = time.perf_counter()
        plan = S.solve(tasks, None, objective=obj, **okw)
        wall = time.perf_counter() - t0
        solve[name] = dict(rescore(plan, what), wall_s=wall, rounds=S.last_stats["rounds"],
                           candidates=S.last_stats["candidates"])
    print(json.dumps({"card": card(0), "kernel": kernel, "scenario_tardiness": solve}))
    eng.close()


class _Task:
    def __init__(self, name, strategies):
        self.name, self.strategies, self.selected_strategy = name, strategies, None

    def select_strategy(self, s):
        self.selected_strategy = s


def _tasks256():
    """The 256-task set of the solve measurements: synthetic table, seed 3, 4 strategies."""
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    T2, valid2 = synth_table(256, 4, 8, seed=3)
    strategies = strategies_from_table(T2, valid2)
    return [_Task("t%d" % j, strategies[j]) for j in range(256)]


def stretch_effect(S, R, tasks, makespan, kw):
    """The max-stretch plan against the completion, makespan and completion-with-w = 1 / p* plans on the 256-task set
    with the release dates of release_effect, every plan rescored in float64 (see the module doc)."""
    import numpy as np
    J = len(tasks)
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    r = [float(x) for x in np.random.default_rng(6).integers(0, int(0.5 * makespan), size=J)]
    # p*_t: the fastest of the task's own runtimes over the options solve() lets the search propose
    T, usable, optindex = S.build_table(tasks)
    pstar = []
    for j, t in enumerate(tasks):
        cells = [g for g in range(8) if np.isfinite(T[j, 0, g]) and (usable[j, g] or not usable[j].any())]
        pstar.append(min(float(list(t.strategies.values())[int(optindex[j, g])].runtime) for g in cells))
    out = {}
    for name, obj, weights in (("max_stretch", "max_stretch", None), ("completion", "completion", None),
                               ("makespan", "makespan", None),
                               ("completion_w_inv_pstar", "completion", [1.0 / p for p in pstar])):
        t0 = time.perf_counter()
        res = S.solve(tasks, None, objective=obj, weights=weights, release=r, **kw)
        wall = time.perf_counter() - t0
        comp = [p[0] + p[2] for p in R.plan_from_arrays(tuples, res[0], res[1], res[2], res[3])]
        st = [(c - max(x, 0.0)) / p for c, x, p in zip(comp, r, pstar)]
        out[name] = {"max_stretch": max(st), "mean_stretch": sum(st) / J, "makespan": max(comp), "wall_s": wall,
                     "rounds": S.last_stats["rounds"]}
    return out


def squared_effect(S, R, tasks, makespan, kw):
    """The squared-flow plan against the completion, max_stretch and makespan plans on the 256-task set with the
    release dates of release_effect, every plan rescored in float64 on the flow times F_t = C_t - max(r_t, 0) (see the
    module doc)."""
    import numpy as np
    J = len(tasks)
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    r = [float(x) for x in np.random.default_rng(6).integers(0, int(0.5 * makespan), size=J)]
    out = {}
    for obj in ("squared_flow", "completion", "max_stretch", "makespan"):
        t0 = time.perf_counter()
        res = S.solve(tasks, None, objective=obj, release=r, **kw)
        wall = time.perf_counter() - t0
        comp = [p[0] + p[2] for p in R.plan_from_arrays(tuples, res[0], res[1], res[2], res[3])]
        flow = [c - max(x, 0.0) for c, x in zip(comp, r)]
        out[obj] = {"sum_flow_squared": sum(f * f for f in flow), "mean_flow": sum(flow) / J, "max_flow": max(flow),
                    "makespan": max(comp), "wall_s": wall, "rounds": S.last_stats["rounds"]}
    return out


def late_penalty_effect(S, R, tasks, kw):
    """The late-penalty plan against the tardiness, late_tasks and completion plans on the 256-task set with the due
    dates of the late-count row and seeded penalties, every plan rescored in float64 (see the module doc)."""
    import numpy as np
    J = len(tasks)
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    due = [float(x) for x in np.random.default_rng(4).integers(0, 200000, size=J)]
    pen = [float(x) for x in np.random.default_rng(8).integers(0, 100000, size=J)]
    for obj in ("late_penalty", "tardiness", "late_tasks"):   # first launches load the kernels
        S.solve(tasks, None, rounds=4, engine=kw["engine"], objective=obj, due=due,
                **({"penalty": pen} if obj == "late_penalty" else {}))
    out = {}
    for obj in ("late_penalty", "tardiness", "late_tasks", "completion"):
        extra = {"due": due} if obj != "completion" else {}
        if obj == "late_penalty":
            extra["penalty"] = pen
        t0 = time.perf_counter()
        res = S.solve(tasks, None, objective=obj, **extra, **kw)
        wall = time.perf_counter() - t0
        comp = [p[0] + p[2] for p in R.plan_from_arrays(tuples, res[0], res[1], res[2], res[3])]
        late = [(c - d, p) for c, d, p in zip(comp, due, pen) if c > d]
        out[obj] = {"cost": sum(p + x for x, p in late), "late_tasks": len(late),
                    "tardiness": sum(x for x, _p in late), "penalties_paid": sum(p for _x, p in late),
                    "makespan": max(comp), "wall_s": wall, "rounds": S.last_stats["rounds"]}
    return out


def front_effect(S, tasks, makespan, kw):
    """solve_front(points=8) on the 256-task set with the release dates of release_effect: per point the cap, the
    makespan and the mean flow time in float64, and the front's wall time (see the module doc)."""
    import numpy as np
    J = len(tasks)
    r = [float(x) for x in np.random.default_rng(6).integers(0, int(0.5 * makespan), size=J)]
    S.solve_front(tasks, points=3, release=r, **dict(kw, rounds=4))   # first launches load the kernels
    t0 = time.perf_counter()
    front = S.solve_front(tasks, points=8, release=r, **kw)
    wall = time.perf_counter() - t0
    shift = sum(max(x, 0.0) for x in r)
    return {"wall_s": wall, "points": [{"cap": p.cap, "makespan": p.makespan, "mean_flow": (p.completion - shift) / J,
                                        "objective": p.stats["objective"], "rounds": p.stats["rounds"],
                                        "solve_wall_s": p.stats["total_wall_s"]} for p in front]}


def late_unit_effect(S, R, tasks, due, w, kw):
    """The late-count plans (unweighted and weighted) under the shipped temperature unit, sum w, and under the mean
    weight, sum w / J: the same solve with t_start and t_end divided by J (run_search's defaults)."""
    import inspect
    from saturn_b200 import search as SE
    J = len(tasks)
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    dflt = inspect.signature(SE.run_search).parameters
    t_start, t_end = dflt["t_start"].default, dflt["t_end"].default
    base = SE.run_search
    out = {}
    for unit, scale in (("sum_w", 1.0), ("mean_w", 1.0 / J)):
        def run(*a, **k):
            return base(*a, t_start=t_start * scale, t_end=t_end * scale, **k)
        SE.run_search = run
        try:
            for name, weights in (("late_tasks", None), ("weighted_late_tasks", w)):
                res = S.solve(tasks, None, objective="late_tasks", due=due, weights=weights, **kw)
                comp = [p[0] + p[2] for p in R.plan_from_arrays(tuples, res[0], res[1], res[2], res[3])]
                out["%s_%s" % (name, unit)] = {
                    "late_tasks": sum(1 for c, d in zip(comp, due) if c > d),
                    "weighted_late_tasks": sum(wi for wi, c, d in zip(w, comp, due) if c > d),
                    "rounds": S.last_stats["rounds"]}
        finally:
            SE.run_search = base
    return out


def release_effect(S, R, tasks, due, makespan, kw):
    """Release-aware against release-blind plans on the 256-task set (see the module doc)."""
    import numpy as np
    from oracle import ref_release as RR
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    tab, optmap = R.table_from_tuples(tuples)
    r = [float(x) for x in np.random.default_rng(6).integers(0, int(0.5 * makespan), size=len(tasks))]
    J = len(tasks)

    def measures(start, comp):
        return {"makespan": max(comp), "total_flow_time": sum(c - max(x, 0.0) for c, x in zip(comp, r)),
                "tardiness": sum(max(0.0, c - d) for c, d in zip(comp, due)),
                "earliest_slack": min(s - x for s, x in zip(start, r))}
    out = {}
    for obj in ("makespan", "completion", "tardiness"):
        extra = {"due": due} if obj == "tardiness" else {}
        t0 = time.perf_counter()
        aware = S.solve(tasks, None, objective=obj, release=r, **extra, **kw)
        wall = time.perf_counter() - t0
        plan = R.plan_from_arrays(tuples, *aware[:4])
        aware_m = measures([p[0] for p in plan], [p[0] + p[2] for p in plan])
        blind = S.solve(tasks, None, objective=obj, **extra, **kw)
        plan = R.plan_from_arrays(tuples, *blind[:4])
        opt = [optmap[t][plan[t][4]] for t in range(J)]
        order = sorted(range(J), key=lambda t: (plan[t][0], t))
        _score, start, _m, _rd = RR.list_schedule(tab, opt, order, r, True, np.float64)
        rt = [plan[t][2] for t in range(J)]
        out[obj] = {"aware": aware_m, "blind_rescored": measures(list(start), [start[t] + rt[t] for t in range(J)]),
                    "aware_wall_s": wall}
    return out


if __name__ == "__main__":
    main()
