"""Fixtures for the maximum lateness (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_max_lateness.py        # writes tests/golden/max_lateness_cases.json

The instances of oracle/gen_completion.py (20 single-node instances at J = 3..5) with seeded integer due dates, and
the first four instances of tests/golden/release_cases.json with their release dates and seeded integer due dates.
Due dates are drawn in [lo, hi] x the makespan optimum (no release dates: of the instance; with them: under them),
alternating a generous range (lo, hi) = (0.9, 1.8), where every due date can be met and L_max* < 0 — the instances
where total tardiness is flat at zero — and a tight one, (0.2, 1.1).  Per instance:
  * the MILP of oracle/ref_max_lateness.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_MAX_LATENESS_LIMIT_S (default 240 s), several instances side by side — status, objective, plan, wall time;
  * the exhaustive list-schedule optimum of L_max in fp64 (`brute_force`);
  * whether the plan that is optimal for the total tardiness, and the one optimal for the makespan (exhaustive, the
    first minimum), are L_max-optimal when rescored.
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

from oracle.gen_completion import jobs  # noqa: E402

N_RELEASE = 4


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, generous, limit = arg
    from oracle import ref_eval as R, ref_max_lateness as ML, ref_release as RR
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    r = [0.0] * J if release is None else [float(x) for x in release]
    mk = RR.brute_force(tab, optmap, r, "makespan", integer_starts=True, dtype=np.float64)
    lo, hi = (0.9, 1.8) if generous else (0.2, 1.1)
    seed = sum(map(ord, name)) * 10 + (1 if generous else 0)
    d = [float(x) for x in np.round(np.random.default_rng(seed).uniform(lo, hi, size=J) * mk[0])]
    best = ML.brute_force(tab, optmap, d, release, True, dtype=np.float64)
    D = ML.tails(d, np.float64)[1]

    def lmax_of(opt, prio):
        return float(ML.evaluate(tab, np.array([opt], np.uint8), np.array([prio], np.uint8), d, release, True,
                                 np.float64)[0]) - D
    td = RR.brute_force(tab, optmap, r, "tardiness", integer_starts=True, dtype=np.float64, due=d)
    td_l, mk_l = lmax_of(td[1], td[2]), lmax_of(mk[1], mk[2])
    t0 = time.time()
    m = ML.milp_solve(tuples, d, release, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    print(name, "status", m["status"], "milp", m["score"], "bf", best[0], "%.1fs" % mr["wall_s"], flush=True)
    return {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "due": d,
            "due_seed": seed, "release": release, "milp": mr,
            "bruteforce_f64": {"score": best[0], "opt": list(best[1]), "prio": list(best[2])},
            "tardiness_optimum": {"max_lateness": td_l, "is_lmax_optimal": bool(td_l <= best[0] + 1e-9)},
            "makespan_optimum": {"max_lateness": mk_l, "is_lmax_optimal": bool(mk_l <= best[0] + 1e-9)}}


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "7"))
    limit = float(os.environ.get("GEN_MAX_LATENESS_LIMIT_S", "240"))
    args = [(name, tuples, None, i % 2 == 0, limit) for i, (name, tuples, _t) in enumerate(jobs())]
    with open(os.path.join(ROOT, "tests", "golden", "release_cases.json")) as f:
        rel = json.load(f)["cases"][:N_RELEASE]
    args += [(c["name"] + "_release", [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]], c["release"],
              i % 2 == 0, limit) for i, c in enumerate(rel)]
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_max_lateness.py",
           "about": "Maximum lateness L_max = max_t (C_t - d_t) of list schedules, integer starts, one node of 8 GPUs; "
                    "the instances of completion_cases.json and the first %d of release_cases.json (with their "
                    "release dates), each with seeded integer due dates.  milp = oracle/ref_max_lateness.py "
                    "milp_solve under HiGHS with mip_rel_gap = 0 and a time limit of %.0f s (score: the decoded "
                    "plan's L_max in float64); bruteforce_f64 = exhaustive list-schedule optimum of L_max; "
                    "tardiness_optimum / makespan_optimum = the exhaustive optimum of that objective rescored as "
                    "L_max, and whether it is L_max-optimal." % (N_RELEASE, limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "max_lateness_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "L_max* < 0:", sum(r["bruteforce_f64"]["score"] < 0 for r in recs),
          "tardiness optimum L_max-optimal:", sum(r["tardiness_optimum"]["is_lmax_optimal"] for r in recs),
          "makespan optimum L_max-optimal:", sum(r["makespan_optimum"]["is_lmax_optimal"] for r in recs))


if __name__ == "__main__":
    main()
