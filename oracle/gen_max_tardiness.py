"""Fixtures for the maximum (weighted) tardiness and the maximum stretch (ORACLE INFRASTRUCTURE; runs on a CPU, needs
no reference).

    python oracle/gen_max_tardiness.py     # writes tests/golden/max_tardiness_cases.json

The instances of tests/golden/late_tasks_cases.json (oracle/gen_late_tasks.py: the 20 completion instances at J = 3..5,
every other one weighted with gen_weighted.WEIGHT_VALUES, and four with release dates) with their integer due dates,
plus N_STRETCH stretch instances on the same runtimes: w_t = fp32(1 / p*_t), p*_t the task's fastest runtime, and
d_t = max(r_t, 0) (0 without release dates), so that the score is the maximum stretch.  Per instance:
  * the MILP of oracle/ref_max_tardiness.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_MAX_TARDINESS_LIMIT_S (default 240 s), several instances side by side — status, objective, plan, wall time;
  * the exhaustive list-schedule optimum of the maximum tardiness in fp64 and fp32 (`brute_force`);
  * whether the plans that are optimal for the (weighted) tardiness and the makespan (exhaustive, the first minimum)
    are optimal for the maximum when rescored.
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

N_STRETCH = 8  # the last four instances without release dates and the four with them, as stretch instances


def stretch_form(tuples, release):
    """(weights, due): fp32(1 / p*_t) with p*_t the smallest runtime of task t (reciprocal in float64), and
    max(r_t, 0) (0 without release dates), as solve(objective="max_stretch") forms them."""
    pstar = [min(float(rt) for _k, rt in tup) for tup in tuples]
    w = [float(np.float32(1.0 / p)) for p in pstar]
    d = [0.0] * len(tuples) if release is None else [max(float(np.float32(r)), 0.0) for r in release]
    return w, d


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, weights, due, stretch, limit = arg
    from oracle import ref_eval as R, ref_max_tardiness as MT, ref_release as RR
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    r = [0.0] * J if release is None else [float(x) for x in release]
    best = MT.brute_force(tab, optmap, due, release, True, dtype=np.float64, weights=weights)
    best32 = MT.brute_force(tab, optmap, due, release, True, dtype=np.float32, weights=weights)

    def score_of(opt, prio):
        return float(MT.evaluate(tab, np.array([opt], np.uint8), np.array([prio], np.uint8), due, release, True,
                                 np.float64, weights=weights)[0])
    td = RR.brute_force(tab, optmap, r, "weighted_tardiness" if weights is not None else "tardiness",
                        integer_starts=True, dtype=np.float64, due=due, weights=weights)
    mk = RR.brute_force(tab, optmap, r, "makespan", integer_starts=True, dtype=np.float64)
    td_s, mk_s = score_of(td[1], td[2]), score_of(mk[1], mk[2])
    t0 = time.time()
    m = MT.milp_solve(tuples, due, release, weights, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    print(name, "status", m["status"], "milp", m["score"], "bf", best[0], "%.1fs" % mr["wall_s"], flush=True)
    return {"name": name, "stretch": stretch, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples],
            "weights": weights, "due": [float(x) for x in due], "release": release, "milp": mr,
            "bruteforce_f64": {"score": best[0], "opt": list(best[1]), "prio": list(best[2])},
            "bruteforce_f32": {"score": best32[0], "opt": list(best32[1]), "prio": list(best32[2])},
            "tardiness_optimum": {"score": td_s, "is_optimal": bool(td_s <= best[0] * (1 + 1e-9) + 1e-12)},
            "makespan_optimum": {"score": mk_s, "is_optimal": bool(mk_s <= best[0] * (1 + 1e-9) + 1e-12)}}


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "7"))
    limit = float(os.environ.get("GEN_MAX_TARDINESS_LIMIT_S", "240"))
    with open(os.path.join(ROOT, "tests", "golden", "late_tasks_cases.json")) as f:
        late = json.load(f)["cases"]
    args = []
    for c in late:
        tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
        args.append((c["name"], tuples, c["release"], c["weights"], c["due"], False, limit))
    plain = [c for c in late if c["release"] is None][-(N_STRETCH // 2):]
    released = [c for c in late if c["release"] is not None][: N_STRETCH - len(plain)]
    for c in plain + released:
        tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
        w, d = stretch_form(tuples, c["release"])
        args.append((c["name"] + "_stretch", tuples, c["release"], w, d, True, limit))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_max_tardiness.py",
           "about": "Maximum (weighted) tardiness max_t w_t max(0, C_t - d_t) of list schedules, integer starts, one "
                    "node of 8 GPUs; the instances of late_tasks_cases.json with their weights, due dates and release "
                    "dates, plus %d stretch instances (stretch = true) on the same runtimes with w_t = fp32(1 / p*_t), "
                    "p*_t the task's fastest runtime, and d_t = max(r_t, 0), where the score is the maximum stretch.  "
                    "milp = oracle/ref_max_tardiness.py milp_solve under HiGHS with mip_rel_gap = 0 and a time limit "
                    "of %.0f s (score: the decoded plan's maximum in float64); bruteforce_f64 / _f32 = exhaustive "
                    "list-schedule optimum; tardiness_optimum / makespan_optimum = the exhaustive optimum of that "
                    "objective rescored, and whether it is optimal for the maximum." % (N_STRETCH, limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "max_tardiness_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "tardiness optimum optimal:", sum(r["tardiness_optimum"]["is_optimal"] for r in recs),
          "makespan optimum optimal:", sum(r["makespan_optimum"]["is_optimal"] for r in recs))


if __name__ == "__main__":
    main()
