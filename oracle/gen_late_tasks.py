"""Fixtures for the number of late tasks (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_late_tasks.py        # writes tests/golden/late_tasks_cases.json

The instances of oracle/gen_completion.py (20 single-node instances at J = 3..5), every other one with seeded weights
from gen_weighted.WEIGHT_VALUES (exact in fp32) and the rest with unit weights, and the first four instances of
tests/golden/release_cases.json with their release dates (weighted likewise).  Due dates are integers drawn in
[0.2, 1.1] x the makespan optimum (no release dates: of the instance; with them: under them).  Per instance the due
dates of the first seed (of at most MAX_SEEDS) under which the optimum is > 0 and the plan that is optimal for the
(weighted) tardiness is not optimal for the (weighted) late count are kept; `due_qualifies` records whether a seed
did (else the first seed is kept).  Per instance:
  * the MILP of oracle/ref_late_tasks.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_LATE_TASKS_LIMIT_S (default 240 s), several instances side by side — status, objective, plan, wall time;
  * the exhaustive list-schedule optimum of the late count in fp64 and fp32 (`brute_force`);
  * whether the plans that are optimal for the tardiness, the maximum lateness and the makespan (exhaustive, the
    first minimum) are count-optimal when rescored.
"""
import itertools
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
from oracle.gen_weighted import WEIGHT_VALUES  # noqa: E402

N_RELEASE = 4
MAX_SEEDS = 200


def _candidates(optmap, J):
    opts = np.array(list(itertools.product(*optmap)), dtype=np.uint8).reshape(-1, J)
    perms = np.array(list(itertools.permutations(range(J))), dtype=np.uint8).reshape(-1, J)
    return np.repeat(opts, len(perms), axis=0), np.tile(perms, (len(opts), 1))


def pick_due(name, tab, optmap, release, weights, mk):
    """(due, seed, qualifies): the first seeded integer due dates in [0.2, 1.1] x mk under which the late-count
    optimum is > 0 and the first tardiness-optimal candidate is not count-optimal (all in float64)."""
    from oracle import ref_release as RR
    J = len(optmap)
    opt, prio = _candidates(optmap, J)
    r = np.zeros(J) if release is None else np.asarray(release, dtype=np.float64)
    _, start, _ = RR.c_evaluate(tab, opt, prio, r, True, np.float64, want_plan=True, threads=os.cpu_count() or 1)
    rt = np.asarray(tab, dtype=np.float64)[np.arange(J)[None, :], opt >> 3, opt & 7]
    C = start + rt
    w = np.ones(J) if weights is None else np.asarray(weights, dtype=np.float64)
    first = None
    for s in range(MAX_SEEDS):
        seed = sum(map(ord, name)) * 1000 + s
        d = np.round(np.random.default_rng(seed).uniform(0.2, 1.1, size=J) * mk)
        count = ((C > d[None, :]) * w[None, :]).sum(axis=1)
        tard = (np.maximum(C - d[None, :], 0.0) * w[None, :]).sum(axis=1)
        if first is None:
            first = (d, seed)
        if count.min() > 0 and count[int(np.argmin(tard))] > count.min():
            return [float(x) for x in d], seed, True
    return [float(x) for x in first[0]], first[1], False


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, weights, limit = arg
    from oracle import ref_eval as R, ref_late_tasks as LT, ref_max_lateness as ML, ref_release as RR
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    r = [0.0] * J if release is None else [float(x) for x in release]
    mk = RR.brute_force(tab, optmap, r, "makespan", integer_starts=True, dtype=np.float64)
    d, seed, qualifies = pick_due(name, tab, optmap, release, weights, mk[0])
    best = LT.brute_force(tab, optmap, d, release, True, dtype=np.float64, weights=weights)
    best32 = LT.brute_force(tab, optmap, d, release, True, dtype=np.float32, weights=weights)

    def count_of(opt, prio):
        return float(LT.evaluate(tab, np.array([opt], np.uint8), np.array([prio], np.uint8), d, release, True,
                                 np.float64, weights=weights)[0])
    td = RR.brute_force(tab, optmap, r, "weighted_tardiness" if weights is not None else "tardiness",
                        integer_starts=True, dtype=np.float64, due=d, weights=weights)
    lm = ML.brute_force(tab, optmap, d, release, True, dtype=np.float64)
    td_c, lm_c, mk_c = count_of(td[1], td[2]), count_of(lm[1], lm[2]), count_of(mk[1], mk[2])
    t0 = time.time()
    m = LT.milp_solve(tuples, d, release, weights, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    print(name, "status", m["status"], "milp", m["score"], "bf", best[0], "%.1fs" % mr["wall_s"], flush=True)
    return {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "weights": weights,
            "due": d, "due_seed": seed, "due_qualifies": qualifies, "release": release, "milp": mr,
            "bruteforce_f64": {"score": best[0], "opt": list(best[1]), "prio": list(best[2])},
            "bruteforce_f32": {"score": best32[0], "opt": list(best32[1]), "prio": list(best32[2])},
            "tardiness_optimum": {"late": td_c, "is_count_optimal": bool(td_c <= best[0] + 1e-9)},
            "max_lateness_optimum": {"late": lm_c, "is_count_optimal": bool(lm_c <= best[0] + 1e-9)},
            "makespan_optimum": {"late": mk_c, "is_count_optimal": bool(mk_c <= best[0] + 1e-9)}}


def _weights(i, J, seed):
    if i % 2 == 0:
        return None
    return [float(x) for x in np.random.default_rng(seed).choice(WEIGHT_VALUES, size=J)]


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "7"))
    limit = float(os.environ.get("GEN_LATE_TASKS_LIMIT_S", "240"))
    args = [(name, tuples, None, _weights(i, len(tuples), 700 + i), limit)
            for i, (name, tuples, _t) in enumerate(jobs())]
    with open(os.path.join(ROOT, "tests", "golden", "release_cases.json")) as f:
        rel = json.load(f)["cases"][:N_RELEASE]
    args += [(c["name"] + "_release", [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]], c["release"],
              _weights(i, len(c["gpu_time_tuples"]), 800 + i), limit) for i, c in enumerate(rel)]
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_late_tasks.py",
           "about": "(Weighted) number of late tasks sum_t w_t [C_t > d_t] of list schedules, integer starts, one node "
                    "of 8 GPUs; the instances of completion_cases.json (every other one weighted) and the first %d of "
                    "release_cases.json (with their release dates), each with seeded integer due dates under which "
                    "the optimum is > 0 and the tardiness-optimal plan is not count-optimal where a seed of at most "
                    "%d gives that (due_qualifies).  milp = oracle/ref_late_tasks.py milp_solve under HiGHS with "
                    "mip_rel_gap = 0 and a time limit of %.0f s (score: the decoded plan's count in float64); "
                    "bruteforce_f64 / _f32 = exhaustive list-schedule optimum of the count; tardiness_optimum / "
                    "max_lateness_optimum / makespan_optimum = the exhaustive optimum of that objective rescored as "
                    "the count, and whether it is count-optimal." % (N_RELEASE, MAX_SEEDS, limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "late_tasks_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "due dates qualify:", sum(r["due_qualifies"] for r in recs),
          "tardiness optimum count-optimal:", sum(r["tardiness_optimum"]["is_count_optimal"] for r in recs),
          "L_max optimum count-optimal:", sum(r["max_lateness_optimum"]["is_count_optimal"] for r in recs),
          "makespan optimum count-optimal:", sum(r["makespan_optimum"]["is_count_optimal"] for r in recs))


if __name__ == "__main__":
    main()
