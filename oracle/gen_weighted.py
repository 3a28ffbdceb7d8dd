"""Fixtures for the WEIGHTED sum of completion times (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_weighted.py              # writes tests/golden/weighted_completion_cases.json

The instances of oracle/gen_completion.py (20 single-node instances at J = 3..5), each with seeded per-task weights
and the objective sum_t w_t C_t.  The weights are exactly representable in fp32 (integers from {1, 2, 3, 5, 8} and
the dyadic fractions 0.25, 0.5, 1.5), so that the fp32 arg-min and the float64 MILP optimum cannot part on a
near-tie through the weights' rounding.  Per instance the first weight seed (of up to 16) under which the
unweighted optimum is no longer optimal is kept, so that the fixtures pin plans the unweighted ones do not;
`differs` records whether one was found.  For each: the MILP of oracle/ref_weighted.py (`milp_solve`) under HiGHS
with mip_rel_gap = 0 and a 20-minute limit (several instances side by side) — status, objective, plan, wall
time — and the exhaustive list-schedule optima in fp64 and fp32.
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

WEIGHT_VALUES = (1.0, 2.0, 3.0, 5.0, 8.0, 0.25, 0.5, 1.5)


def worker(job):
    """One instance under the weighted objective (its own process: HiGHS is single-threaded)."""
    name, tuples, timeout = job
    from oracle import ref_completion as RC, ref_eval as R, ref_weighted as RW
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    plain = RC.brute_force(tab, optmap, integer_starts=True, dtype=np.float64)
    seed0 = sum(map(ord, name))
    for attempt in range(16):
        rng = np.random.default_rng(seed0 * 100 + attempt)
        w = [float(x) for x in rng.choice(WEIGHT_VALUES, size=J)]
        bf = RW.brute_force(tab, optmap, integer_starts=True, dtype=np.float64, weights=w)
        # the unweighted optimum's plan, scored under the weights
        plain_w = RW.list_schedule(tab, plain[1], plain[2], True, np.float64, weights=w)[0]
        differs = plain_w > bf[0] * (1 + 1e-12)
        if differs:
            break
    t0 = time.time()
    m = RW.milp_solve(tuples, w, time_limit=timeout, mip_rel_gap=0.0)
    rec = {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "weights": w,
           "weight_seed": seed0 * 100 + attempt, "differs": bool(differs),
           "unweighted_optimum_weighted": plain_w,
           "milp": {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]),
                    "objective_value": m["objective_value"], "weighted_completion": m["weighted_completion"],
                    "total_completion": m["total_completion"], "start": m["start"], "mask": m["mask"],
                    "opt_idx": m["opt_idx"], "wall_s": time.time() - t0}}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        rec["milp"]["feasible"], rec["milp"]["overlaps"] = bool(ok), ov
    rec["bruteforce_f64"] = {"weighted_completion": bf[0], "opt": list(bf[1]), "prio": list(bf[2])}
    bf32 = RW.brute_force(tab, optmap, integer_starts=True, dtype=np.float32, weights=w)
    rec["bruteforce_f32"] = {"weighted_completion": bf32[0], "opt": list(bf32[1]), "prio": list(bf32[2])}
    print(name, "status", m["status"], "milp", m["weighted_completion"], "bf", bf[0], "differs", differs,
          "%.1fs" % rec["milp"]["wall_s"], flush=True)
    return rec


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "6"))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, jobs(), chunksize=1)
    out = {"generator": "oracle/gen_weighted.py",
           "about": "Weighted sum of completion times sum_t w_t (start_t + rt_t), integer starts, one node of 8 GPUs; "
                    "the instances of completion_cases.json with seeded weights exactly representable in fp32.  "
                    "milp = oracle/ref_weighted.py milp_solve under HiGHS with mip_rel_gap = 0; "
                    "bruteforce_* = exhaustive list-schedule optimum (ref_weighted.brute_force); differs = the "
                    "unweighted optimum's plan is not optimal under the weights (its weighted score is "
                    "unweighted_optimum_weighted).",
           "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "weighted_completion_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "differ:", sum(r["differs"] for r in recs))


if __name__ == "__main__":
    main()
