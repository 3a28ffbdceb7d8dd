"""Fixtures for release dates (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_release.py             # writes tests/golden/release_cases.json

The instances of oracle/gen_completion.py (20 single-node instances at J = 3..5), each with seeded integer release
dates in [0, the makespan of the plan that is optimal for r = 0 under the makespan objective].  Per instance the
first release seed (of up to 16) is kept under which the plan that is optimal for r = 0, rescored with r, is not
optimal, under the makespan objective and under the completion objective (`differs` records it per objective;
when no seed makes both differ, the last one is kept).  Four more instances (the first of each J = 3, 4, 5 group
and the first heterogeneous one) get release dates with a fractional part, which integer starts round up.  For each
instance and both objectives: the MILP of oracle/ref_release.py (`milp_solve`) under HiGHS with mip_rel_gap = 0 and
a time limit of at most 20 minutes (GEN_RELEASE_LIMIT_S, several instances side by side) — status, objective,
plan, wall time — and the exhaustive list-schedule optima in fp64 and fp32.
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

OBJECTIVES = ("makespan", "completion")
FRACTIONAL = ("J3_g8_seed200", "J4_g8_seed210", "J5_g8_seed220", "H4_hetero_seed230")


def worker(arg):
    """One instance under both objectives (its own process: HiGHS is single-threaded)."""
    name, tuples, limit, fractional = arg
    from oracle import ref_eval as R, ref_release as RR
    tab, optmap = R.table_from_tuples(tuples)
    J = len(tuples)
    seed0 = sum(map(ord, name)) + (7 if fractional else 0)
    zero_r = [0.0] * J
    zero = {o: RR.brute_force(tab, optmap, zero_r, o, integer_starts=True, dtype=np.float64) for o in OBJECTIVES}
    horizon = zero["makespan"][0]
    for attempt in range(16):
        rng = np.random.default_rng(seed0 * 100 + attempt)
        r = [float(x) for x in rng.integers(0, int(horizon) + 1, size=J)]
        if fractional:
            r = [x + float(f) for x, f in zip(r, rng.choice([0.25, 0.5, 0.75], size=J))]
        bf = {o: RR.brute_force(tab, optmap, r, o, integer_starts=True, dtype=np.float64) for o in OBJECTIVES}
        rescored = {o: RR.list_schedule(tab, zero[o][1], zero[o][2], r, True, np.float64, objective=o)[0]
                    for o in OBJECTIVES}
        differs = {o: rescored[o] > bf[o][0] * (1 + 1e-12) for o in OBJECTIVES}
        if all(differs.values()):
            break
    rec = {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples], "release": r,
           "release_seed": seed0 * 100 + attempt, "fractional": bool(fractional),
           "differs": {o: bool(differs[o]) for o in OBJECTIVES},
           "zero_optimum_rescored": {o: rescored[o] for o in OBJECTIVES}}
    for o in OBJECTIVES:
        t0 = time.time()
        m = RR.milp_solve(tuples, r, o, time_limit=limit, mip_rel_gap=0.0)
        mr = {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]),
              "objective_value": m["objective_value"], "score": m["score"], "start": m["start"], "mask": m["mask"],
              "opt_idx": m["opt_idx"], "wall_s": time.time() - t0}
        if m["start"] is not None:
            k = [tuples[t][m["opt_idx"][t]][0] for t in range(J)]
            rt = [tuples[t][m["opt_idx"][t]][1] for t in range(J)]
            ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
            mr["feasible"], mr["overlaps"] = bool(ok), ov
        bf32 = RR.brute_force(tab, optmap, r, o, integer_starts=True, dtype=np.float32)
        rec[o] = {"milp": mr,
                  "bruteforce_f64": {"score": bf[o][0], "opt": list(bf[o][1]), "prio": list(bf[o][2])},
                  "bruteforce_f32": {"score": bf32[0], "opt": list(bf32[1]), "prio": list(bf32[2])}}
        print(name, o, "status", m["status"], "milp", m["score"], "bf", bf[o][0], "differs", differs[o],
              "%.1fs" % mr["wall_s"], flush=True)
    return rec


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "6"))
    limit = min(1200.0, float(os.environ.get("GEN_RELEASE_LIMIT_S", "1200")))
    args = [(name, tuples, limit, False) for name, tuples, _t in jobs()]
    args += [(name + "_frac", tuples, limit, True) for name, tuples, _t in jobs() if name in FRACTIONAL]
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, args, chunksize=1)
    out = {"generator": "oracle/gen_release.py",
           "about": "List schedules with release dates (start = max(max ready, r), ceil(r) under integer starts), "
                    "integer starts, one node of 8 GPUs; the instances of completion_cases.json with seeded integer "
                    "release dates, plus *_frac instances whose release dates have a fractional part.  Per "
                    "objective (makespan, completion): milp = oracle/ref_release.py milp_solve under HiGHS with "
                    "mip_rel_gap = 0 and a time limit of %.0f s; bruteforce_* = exhaustive list-schedule optimum "
                    "(ref_release.brute_force); differs = the plan optimal for r = 0, rescored with r "
                    "(zero_optimum_rescored), is not optimal." % limit,
           "time_limit_s": limit, "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "release_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    for o in OBJECTIVES:
        print("wrote", dst, o, "proven optimal:", sum(r[o]["milp"]["proven_optimal"] for r in recs), "of", len(recs),
              "differ:", sum(r["differs"][o] for r in recs))


if __name__ == "__main__":
    main()
