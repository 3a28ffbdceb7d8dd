"""Fixtures for the total weighted tardiness (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_tardiness.py             # writes tests/golden/tardiness_cases.json

The instances of oracle/gen_completion.py (20 single-node instances at J = 3..5), every other one with unit weights
and the rest with seeded weights from gen_weighted.WEIGHT_VALUES (exact in fp32), each with seeded integer due dates
(exact in fp32) in [0, the makespan of the plan that is optimal for d = 0].  Per instance the first due-date seed
(of up to 16) is kept under which the exhaustive tardiness optimum is > 0 and the plan that is optimal for d = 0
(the weighted, or unweighted, completion optimum) is not tardiness-optimal; `positive` and `differs` record both
facts.  For each: the MILP of oracle/ref_tardiness.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a
20-minute limit (several instances side by side) — status, objective, plan, wall time — and the exhaustive
list-schedule optima in fp64 and fp32.
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
from oracle.gen_weighted import WEIGHT_VALUES  # noqa: E402


def worker(arg):
    """One instance under the tardiness objective (its own process: HiGHS is single-threaded)."""
    i, (name, tuples, timeout) = arg
    from oracle import ref_eval as R, ref_tardiness as RT
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    seed0 = sum(map(ord, name))
    w = None
    if i % 2 == 1:
        w = [float(x) for x in np.random.default_rng(seed0 * 100 + 99).choice(WEIGHT_VALUES, size=J)]
    # the plan that is optimal for d = 0 (the weighted sum of completion times) and its makespan
    zero = RT.brute_force(tab, optmap, [0.0] * J, integer_starts=True, dtype=np.float64, weights=w)
    horizon = R.list_schedule(tab, zero[1], zero[2], True, np.float64)[0]
    for attempt in range(16):
        rng = np.random.default_rng(seed0 * 100 + attempt)
        d = [float(x) for x in rng.integers(0, int(horizon) + 1, size=J)]
        bf = RT.brute_force(tab, optmap, d, integer_starts=True, dtype=np.float64, weights=w)
        zero_t = RT.list_schedule(tab, zero[1], zero[2], d, True, np.float64, weights=w)[0]
        positive = bf[0] > 0
        differs = zero_t > bf[0] * (1 + 1e-12)
        if positive and differs:
            break
    t0 = time.time()
    m = RT.milp_solve(tuples, d, w, time_limit=timeout, mip_rel_gap=0.0)
    rec = {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "weights": w, "due": d,
           "due_seed": seed0 * 100 + attempt, "positive": bool(positive), "differs": bool(differs),
           "completion_optimum_tardiness": zero_t,
           "milp": {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]),
                    "objective_value": m["objective_value"], "weighted_tardiness": m["weighted_tardiness"],
                    "late_tasks": m["late_tasks"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
                    "wall_s": time.time() - t0}}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        rec["milp"]["feasible"], rec["milp"]["overlaps"] = bool(ok), ov
    rec["bruteforce_f64"] = {"weighted_tardiness": bf[0], "opt": list(bf[1]), "prio": list(bf[2])}
    bf32 = RT.brute_force(tab, optmap, d, integer_starts=True, dtype=np.float32, weights=w)
    rec["bruteforce_f32"] = {"weighted_tardiness": bf32[0], "opt": list(bf32[1]), "prio": list(bf32[2])}
    print(name, "status", m["status"], "milp", m["weighted_tardiness"], "bf", bf[0], "positive", positive,
          "differs", differs, "%.1fs" % rec["milp"]["wall_s"], flush=True)
    return rec


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "6"))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, list(enumerate(jobs())), chunksize=1)
    out = {"generator": "oracle/gen_tardiness.py",
           "about": "Weighted tardiness sum_t w_t max(0, start_t + rt_t - d_t), integer starts, one node of 8 GPUs; "
                    "the instances of completion_cases.json, every other one with seeded weights exactly "
                    "representable in fp32 (weights = null: unit weights), with seeded integer due dates.  "
                    "milp = oracle/ref_tardiness.py milp_solve under HiGHS with mip_rel_gap = 0; "
                    "bruteforce_* = exhaustive list-schedule optimum (ref_tardiness.brute_force); positive = that "
                    "optimum is > 0; differs = the plan optimal for d = 0 is not tardiness-optimal (its tardiness is "
                    "completion_optimum_tardiness).",
           "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "tardiness_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs),
          "positive:", sum(r["positive"] for r in recs), "differ:", sum(r["differs"] for r in recs))


if __name__ == "__main__":
    main()
