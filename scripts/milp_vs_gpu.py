"""GPU search vs the reference's CPU MILP on the same T, same box (SURVEY §8d metric 2).

    python scripts/milp_vs_gpu.py [--limit 30]

For each instance: the reference MILP restated for scipy/HiGHS (oracle/ref_milp.py — the reference
tree and PuLP/Gurobi/CBC are not on the GPU box) runs with a wall-clock limit and its incumbent is
feasibility-checked; the GPU search (saturn.solver.solve's engine) runs until it reaches a makespan
<= the MILP's, and to its own convergence.  Oracle code is used here only as the baseline being
timed and as the checker.
"""
import argparse
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from oracle import ref_eval as R, ref_milp  # noqa: E402
from saturn_b200 import Strategy, convert_into_comprehensible, solve  # noqa: E402
from saturn_b200 import solver as S  # noqa: E402


class DuckTask:
    def __init__(self, name, strategies):
        self.name, self.strategies, self.selected_strategy = name, strategies, None

    def select_strategy(self, s):
        self.selected_strategy = s


def probe_tuples(J, options, seed):
    rnd = random.Random(seed)
    return [[(g, b / g ** 0.8) for g in options] for b in (rnd.uniform(500, 4000) for _ in range(J))]


def tasks_of(tuples):
    return [DuckTask("t%d" % t, {g: Strategy("x", g, {}, rt) for g, rt in tup}) for t, tup in enumerate(tuples)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--limit", type=float, default=30.0)
    ap.add_argument("--sizes", default="4,5,6,8,10,12,16,24")
    args = ap.parse_args()
    print("# GPU search vs reference MILP (HiGHS, sound big-M), same box; cores=%d\n" % (os.cpu_count() or 0))
    print("| J | options | MILP vars / rows | MILP build s | MILP result after %.0f s limit | MILP makespan | "
          "GPU makespan | GPU time to match MILP | GPU solve() total s | candidates |" % args.limit)
    print("|---|---|---|---|---|---|---|---|---|---|")
    # warm up the library (context creation, first launch) so that it is not billed to the first row
    solve(tasks_of(probe_tuples(4, [1, 2], 0)), None, chains=4096, rounds=5)
    for J in [int(x) for x in args.sizes.split(",")]:
        tuples = probe_tuples(J, [1, 2, 4, 8], 0)
        m = ref_milp.solve(tuples, time_limit=args.limit)
        if m["makespan"] is not None:
            rts = [tuples[t][o][1] for t, o in enumerate(m["opt_idx"])]
            ks = [tuples[t][o][0] for t, o in enumerate(m["opt_idx"])]
            ok = R.check_plan(m["start"], m["mask"], rts, ks)[0]
            mres = ("optimal in %.1f s" % m["wall_s"]) if m["proven_optimal"] else "incumbent at limit"
            if not ok:
                mres += " (INFEASIBLE plan)"
            mmk = "%.3f" % m["makespan"]
        else:
            mres, mmk = "no incumbent", "—"
        # time to match: solve() with a makespan target
        tasks = tasks_of(tuples)
        match = "—"
        if m["makespan"] is not None:
            from saturn_b200.search import run_search
            eng = S._engine()
            T, usable, optindex = S.build_table(tasks)
            Td = T.copy()
            for j in range(J):
                if usable[j].any():
                    Td[j, 0, ~usable[j]] = np.inf
            t0 = time.perf_counter()
            eng.set_table(Td, list(range(1, 9)), sentinel=float("inf"))
            res = run_search(eng, chains=1 << 16, rounds=400, seed=0, reduced=True, time_budget_s=20.0,
                             target_makespan=m["makespan"] * (1 + 1e-7), use_dist=False)
            dt = time.perf_counter() - t0
            match = ("%.4f s (%d rounds)" % (dt, res.rounds)) if res.makespan <= m["makespan"] * (1 + 1e-6) else \
                ("not reached in %.1f s (%.3f)" % (dt, res.makespan))
        t0 = time.perf_counter()
        out = solve(tasks, None, gurobi=False, timeout=60)
        dt = time.perf_counter() - t0
        viol = R.milp_constraints_hold(tuples, *out[:5], out[5])
        convert_into_comprehensible(tasks, out[2], out[4], out[1], out[3], out[0])
        print("| %d | {1,2,4,8} | %d / %d | %.2f | %s | %s | %.3f%s | %s | %.3f | %.2e |" % (
            J, m["n_vars"], m["n_cons"], m["build_s"], mres, mmk, out[5], "" if not viol else " (VIOLATIONS)",
            match, dt, S.last_stats["candidates"]))
        sys.stdout.flush()
    nv, nc = ref_milp.model_size(256, 8)
    from saturn_b200.synth import synth_table
    Tt, valid = synth_table(256, 8, 8, seed=0)
    tmin = np.where(valid, Tt, np.inf).min(axis=1)
    tuples = [[(g + 1, float(tmin[j, g])) for g in range(8) if np.isfinite(tmin[j, g])] for j in range(256)]
    tasks = tasks_of(tuples)
    t0 = time.perf_counter()
    out = solve(tasks, None, gurobi=False, timeout=60, chains=1 << 17, rounds=400)
    dt = time.perf_counter() - t0
    lb = sum(min(k * rt for k, rt in tup) for tup in tuples) / 8
    print("| 256 (C4 table, min over strategies) | 1..8 | %d / %d | — | not built: 8.4 M rows of Python objects / "
          "HiGHS has no incumbent at J=24 already | — | %.1f (area bound %.1f, gap %.2f %%) | — | %.3f | %.2e |" % (
              nv, nc, out[5], lb, 100 * (out[5] / lb - 1), dt, S.last_stats["candidates"]))


if __name__ == "__main__":
    main()
