"""Fixtures for the completion penalty (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_completion_penalty.py     # writes tests/golden/completion_penalty_cases.json

The 24 due-date instances of tests/golden/late_penalty_cases.json (integer runtimes and due dates, every other one
weighted, four with release dates) with their penalties, plus a cap variant of each: every due date at one makespan
cap and every penalty P, the smallest power of two >= sum_t w_t * H with H = max_t r_t + sum_t max_s rt_ts, a bound on
every completion of a list schedule.  The cap lies halfway (rounded down to an integer) between the exhaustive
minimum makespan and the makespan of the exhaustive minimum of sum_t w_t C_t.  Per instance:
  * the MILP of oracle/ref_completion_penalty.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and a time limit of
    GEN_COMPLETION_PENALTY_LIMIT_S (default 60 s), for both variants, several instances side by side — status,
    objective, plan, wall time;
  * the exhaustive list-schedule optimum of both variants in fp64 and fp32 (`brute_force`);
  * the exhaustive (makespan, sum_t w_t C_t) front (`front_brute_force`) and its minimum at the cap.
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


def horizon_penalty(tuples, release, weights):
    """P, the smallest power of two >= sum_t w_t * H, H = max_t r_t + sum_t max_s rt_ts."""
    J = len(tuples)
    H = max([0.0] + [float(x) for x in (release or [])]) + sum(max(rt for _k, rt in tup) for tup in tuples)
    m, e = math.frexp((sum(weights) if weights is not None else J) * H)
    return math.ldexp(1.0, e - 1 if m == 0.5 else e)


def milp_record(tuples, due, penalty, release, weights, limit):
    from oracle import ref_completion_penalty as CP, ref_eval as R
    J = len(tuples)
    t0 = time.time()
    m = CP.milp_solve(tuples, due, penalty, release, weights, time_limit=limit, mip_rel_gap=0.0)
    mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]), "objective_value": m["objective_value"],
          "score": m["score"], "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"],
          "wall_s": time.time() - t0}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        mr["feasible"], mr["overlaps"] = bool(ok), ov
    return mr


def worker(arg):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, release, weights, due, penalty, limit = arg
    from oracle import ref_completion_penalty as CP, ref_eval as R
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)

    def bf(d, p):
        b64 = CP.brute_force(tab, optmap, d, p, release, True, dtype=np.float64, weights=weights)
        b32 = CP.brute_force(tab, optmap, d, p, release, True, dtype=np.float32, weights=weights)
        return ({"score": b64[0], "opt": list(b64[1]), "prio": list(b64[2])},
                {"score": b32[0], "opt": list(b32[1]), "prio": list(b32[2])})

    fr = CP.front_brute_force(tab, optmap, [], release, True, weights=weights)["front"]
    cap = float(math.floor((fr[0][0] + fr[-1][0]) / 2))
    P = horizon_penalty(tuples, release, weights)
    at_cap = CP.front_brute_force(tab, optmap, [cap], release, True, weights=weights)["at_cap"][0]
    b64, b32 = bf(due, penalty)
    c64, c32 = bf([cap] * J, [P] * J)
    m = milp_record(tuples, due, penalty, release, weights, limit)
    mc = milp_record(tuples, [cap] * J, [P] * J, release, weights, limit)
    print(name, "status", m["status"], mc["status"], "milp", m["score"], mc["score"], "bf", b64["score"],
          c64["score"], "front", len(fr), "cap", cap, at_cap, flush=True)
    return {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "weights": weights,
            "due": [float(x) for x in due], "penalty": penalty, "release": release, "milp": m,
            "bruteforce_f64": b64, "bruteforce_f32": b32,
            "cap": {"cap": cap, "P": P, "milp": mc, "bruteforce_f64": c64, "bruteforce_f32": c32,
                    "front_at_cap": at_cap},
            "front": fr}


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "8"))
    limit = float(os.environ.get("GEN_COMPLETION_PENALTY_LIMIT_S", "60"))
    with open(os.path.join(ROOT, "tests", "golden", "late_penalty_cases.json")) as f:
        base = json.load(f)["cases"]
    args = []
    for c in base:
        tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
        args.append((c["name"], tuples, c["release"], c["weights"], c["due"], c["penalty"], limit))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_completion_penalty.py",
           "about": "Completion penalty sum_t (w_t C_t + [C_t > d_t] p_t) of list schedules, integer starts, one node "
                    "of 8 GPUs; the %d instances of late_penalty_cases.json (integer runtimes and due dates, their "
                    "weights, penalties and release dates), and per instance a cap variant: every due date at `cap` "
                    "(halfway between the exhaustive minimum makespan and the makespan of the exhaustive minimum of "
                    "sum w C, rounded down) and every penalty P (the smallest power of two >= sum w * (max r + sum "
                    "of the largest runtimes)).  milp = oracle/ref_completion_penalty.py milp_solve under HiGHS with "
                    "mip_rel_gap = 0 and a time limit of %.0f s (status as HiGHS reports it; score: the decoded "
                    "plan's completion penalty in float64); bruteforce_f64 / _f32 = exhaustive list-schedule "
                    "optimum; front = the exhaustive non-dominated (fp32 makespan, fp64 sum w C) pairs; "
                    "cap.front_at_cap = the exhaustive minimum of sum w C with makespan <= cap."
                    % (len(recs), limit),
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "completion_penalty_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "and",
          sum(r["cap"]["milp"]["proven_optimal"] for r in recs), "(cap) of", len(recs))


if __name__ == "__main__":
    main()
