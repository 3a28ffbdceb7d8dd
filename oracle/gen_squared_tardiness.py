"""Fixtures for the (weighted) squared tardiness and the squared flow time (ORACLE INFRASTRUCTURE; runs on a CPU, needs
no reference).

    python oracle/gen_squared_tardiness.py     # writes tests/golden/squared_tardiness_cases.json

The instances of tests/golden/late_tasks_cases.json (oracle/gen_late_tasks.py: the 20 completion instances at J = 3..5,
every other one weighted with gen_weighted.WEIGHT_VALUES, and four with release dates) with their integer due dates and
every runtime rounded UP to an integer, plus N_FLOW squared-flow instances on the same runtimes with d_t = max(r_t, 0)
(0 without release dates), so that the score is sum_t w_t (C_t - max(r_t, 0))^2.  Integer runtimes, due dates and
starts give integer tardiness, where the tangent cuts of the MILP are exact (ref_squared_tardiness.milp_solve).  Per
instance:
  * the MILP of oracle/ref_squared_tardiness.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_SQUARED_TARDINESS_LIMIT_S (default 240 s), several instances side by side — status, objective, plan, wall time;
  * the exhaustive list-schedule optimum of the squared tardiness in fp64 and fp32 (`brute_force`);
  * the exhaustive optimum of the (weighted) tardiness rescored, and whether it is optimal for the squares.
"""
import json
import math
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_FLOW = 6  # the last three instances without release dates and three with them, as squared-flow instances


def flow_due(n, release):
    """max(r_t, 0) (0 without release dates), the due dates solve(objective="squared_flow") forms."""
    return [0.0] * n if release is None else [max(float(np.float32(r)), 0.0) for r in release]


def integer_runtimes(tuples):
    """Every runtime rounded up to an integer."""
    return [[(k, float(math.ceil(rt))) for k, rt in tup] for tup in tuples]


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, weights, due, flow, limit = arg
    from oracle import ref_eval as R, ref_release as RR, ref_squared_tardiness as SQ
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    r = [0.0] * J if release is None else [float(x) for x in release]
    best = SQ.brute_force(tab, optmap, due, release, True, dtype=np.float64, weights=weights)
    best32 = SQ.brute_force(tab, optmap, due, release, True, dtype=np.float32, weights=weights)
    td = RR.brute_force(tab, optmap, r, "weighted_tardiness" if weights is not None else "tardiness",
                        integer_starts=True, dtype=np.float64, due=due, weights=weights)
    td_s = float(SQ.evaluate(tab, np.array([td[1]], np.uint8), np.array([td[2]], np.uint8), due, release, True,
                             np.float64, weights=weights)[0])
    t0 = time.time()
    m = SQ.milp_solve(tuples, due, release, weights, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    print(name, "status", m["status"], "milp", m["score"], "bf", best[0], "%.1fs" % mr["wall_s"], flush=True)
    return {"name": name, "flow": flow, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples],
            "weights": weights, "due": [float(x) for x in due], "release": release, "milp": mr,
            "bruteforce_f64": {"score": best[0], "opt": list(best[1]), "prio": list(best[2])},
            "bruteforce_f32": {"score": best32[0], "opt": list(best32[1]), "prio": list(best32[2])},
            "tardiness_optimum": {"score": td_s, "is_optimal": bool(td_s <= best[0] * (1 + 1e-9) + 1e-12)}}


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "7"))
    limit = float(os.environ.get("GEN_SQUARED_TARDINESS_LIMIT_S", "240"))
    with open(os.path.join(ROOT, "tests", "golden", "late_tasks_cases.json")) as f:
        late = json.load(f)["cases"]
    args = []
    for c in late:
        tuples = integer_runtimes(c["gpu_time_tuples"])
        args.append((c["name"], tuples, c["release"], c["weights"], c["due"], False, limit))
    plain = [c for c in late if c["release"] is None][-(N_FLOW // 2):]
    released = [c for c in late if c["release"] is not None][: N_FLOW - len(plain)]
    for c in plain + released:
        tuples = integer_runtimes(c["gpu_time_tuples"])
        args.append((c["name"] + "_flow", tuples, c["release"], c["weights"], flow_due(len(tuples), c["release"]),
                     True, limit))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_squared_tardiness.py",
           "about": "(Weighted) squared tardiness sum_t w_t max(0, C_t - d_t)^2 of list schedules, integer starts, one "
                    "node of 8 GPUs; the instances of late_tasks_cases.json with their weights, due dates and release "
                    "dates and every runtime rounded up to an integer, plus %d squared-flow instances (flow = true) on "
                    "the same runtimes with d_t = max(r_t, 0), where the score is sum_t w_t (C_t - max(r_t, 0))^2.  "
                    "milp = oracle/ref_squared_tardiness.py milp_solve under HiGHS with mip_rel_gap = 0 and a time "
                    "limit of %.0f s (score: the decoded plan's squared tardiness in float64); bruteforce_f64 / _f32 = "
                    "exhaustive list-schedule optimum; tardiness_optimum = the exhaustive optimum of the (weighted) "
                    "tardiness rescored, and whether it is optimal for the squares." % (N_FLOW, limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "squared_tardiness_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "tardiness optimum optimal:", sum(r["tardiness_optimum"]["is_optimal"] for r in recs))


if __name__ == "__main__":
    main()
