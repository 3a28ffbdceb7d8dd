"""Fixtures for the late penalty (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_late_penalty.py     # writes tests/golden/late_penalty_cases.json

The 24 due-date instances of tests/golden/squared_tardiness_cases.json (flow = false: integer runtimes and due dates,
every other one weighted, four with release dates), each with seeded integer penalties p_t in [0, PMAX] drawn so that
some are 0 and, on every third instance, one dominates (DOMINANT, above any total tardiness these horizons allow).
Per instance:
  * the MILP of oracle/ref_late_penalty.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_LATE_PENALTY_LIMIT_S (default 120 s), several instances side by side — status, objective, plan, wall time;
  * the exhaustive list-schedule optimum of the late penalty in fp64 and fp32 (`brute_force`);
  * the exhaustive optima of the (weighted) tardiness and of the weighted late count (weights = the penalties, +1 so
    that none is 0) rescored as late penalties, and whether each differs from the optimum.
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 20261018
PMAX = 40
DOMINANT = 10000


def penalties(i, J):
    """Seeded integer penalties of instance i: uniform in [0, PMAX], about one in four set to 0, and on every third
    instance one job's penalty set to DOMINANT."""
    rng = np.random.default_rng(SEED + i)
    p = rng.integers(0, PMAX + 1, size=J).astype(float)
    p[rng.random(J) < 0.25] = 0.0
    if i % 3 == 0:
        p[int(rng.integers(0, J))] = float(DOMINANT)
    return [float(x) for x in p]


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, weights, due, penalty, limit = arg
    from oracle import ref_eval as R, ref_late_penalty as LP, ref_late_tasks as LT, ref_release as RR
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    r = [0.0] * J if release is None else [float(x) for x in release]
    best = LP.brute_force(tab, optmap, due, penalty, release, True, dtype=np.float64, weights=weights)
    best32 = LP.brute_force(tab, optmap, due, penalty, release, True, dtype=np.float32, weights=weights)

    def rescore(opt, prio):
        return float(LP.evaluate(tab, np.array([opt], np.uint8), np.array([prio], np.uint8), due, penalty, release,
                                 True, np.float64, weights=weights)[0])

    td = RR.brute_force(tab, optmap, r, "weighted_tardiness" if weights is not None else "tardiness",
                        integer_starts=True, dtype=np.float64, due=due, weights=weights)
    td_s = rescore(td[1], td[2])
    lw = [x + 1.0 for x in penalty]
    lc = LT.brute_force(tab, optmap, due, release, True, dtype=np.float64, weights=lw)
    lc_s = rescore(lc[1], lc[2])
    t0 = time.time()
    m = LP.milp_solve(tuples, due, penalty, release, weights, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    print(name, "status", m["status"], "milp", m["score"], "bf", best[0], "td", td_s, "lc", lc_s,
          "%.1fs" % mr["wall_s"], flush=True)
    return {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "weights": weights,
            "due": [float(x) for x in due], "penalty": penalty, "release": release, "milp": mr,
            "bruteforce_f64": {"score": best[0], "opt": list(best[1]), "prio": list(best[2])},
            "bruteforce_f32": {"score": best32[0], "opt": list(best32[1]), "prio": list(best32[2])},
            "tardiness_optimum": {"score": td_s, "opt": list(td[1]), "prio": list(td[2]),
                                  "differs": bool(td_s > best[0])},
            "late_count_optimum": {"score": lc_s, "weights": lw, "opt": list(lc[1]), "prio": list(lc[2]),
                                   "differs": bool(lc_s > best[0])}}


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "7"))
    limit = float(os.environ.get("GEN_LATE_PENALTY_LIMIT_S", "120"))
    with open(os.path.join(ROOT, "tests", "golden", "squared_tardiness_cases.json")) as f:
        base = [c for c in json.load(f)["cases"] if not c["flow"]]
    args = []
    for i, c in enumerate(base):
        tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
        args.append((c["name"], tuples, c["release"], c["weights"], c["due"], penalties(i, len(tuples)), limit))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_late_penalty.py",
           "about": "Late penalty sum_t [C_t > d_t] (p_t + w_t (C_t - d_t)) of list schedules, integer starts, one node "
                    "of 8 GPUs; the %d due-date instances of squared_tardiness_cases.json (integer runtimes and due "
                    "dates, their rates and release dates) with seeded integer penalties (seed %d + instance index, "
                    "0..%d, some 0, a dominant %d on every third instance).  milp = oracle/ref_late_penalty.py "
                    "milp_solve under HiGHS with mip_rel_gap = 0 and a time limit of %.0f s (score: the decoded plan's "
                    "late penalty in float64); bruteforce_f64 / _f32 = exhaustive list-schedule optimum; "
                    "tardiness_optimum / late_count_optimum = the exhaustive optima of the (weighted) tardiness and of "
                    "the late count weighted by p + 1, rescored as late penalties, and whether each is worse than the "
                    "optimum." % (len(recs), SEED, PMAX, DOMINANT, limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "late_penalty_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "differ from both:", sum(r["tardiness_optimum"]["differs"] and r["late_count_optimum"]["differs"]
                                   for r in recs))


if __name__ == "__main__":
    main()
