"""Fixtures for the sum-of-completion-times objective (ORACLE INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_completion.py            # writes tests/golden/completion_cases.json

About 20 single-node instances at J = 3..5 over the option sets of the makespan fixtures (instance makers of
oracle/gen_golden.py).  For each: the MILP of oracle/ref_completion.py (`milp_solve`) under HiGHS with
mip_rel_gap = 0 and a 20-minute limit (several instances side by side, as `gen_golden.py --extra` runs them) —
status, objective, plan, wall time — and the exhaustive list-schedule optima in fp64 and fp32.

The reference cannot pin this objective: its completion-time branch (saturn/solver/milp.py:89,174-182,
makespan_opt=False) is unreachable from solve() (milp.py:372) and bounds each completion by the start alone.
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

from oracle.gen_golden import hetero_tuples, probe_tuples  # noqa: E402


def worker(job):
    """One instance (its own process: HiGHS is single-threaded)."""
    name, tuples, timeout = job
    from oracle import ref_completion as RC, ref_eval as R
    t0 = time.time()
    m = RC.milp_solve(tuples, time_limit=timeout, mip_rel_gap=0.0)
    rec = {"name": name, "gpu_time_tuples": [[list(x) for x in tup] for tup in tuples],
           "milp": {"status": m["status"], "proven_optimal": bool(m["proven_optimal"]),
                    "objective_value": m["objective_value"], "total_completion": m["total_completion"],
                    "start": m["start"], "mask": m["mask"], "opt_idx": m["opt_idx"], "wall_s": time.time() - t0}}
    if m["start"] is not None:
        k = [tuples[t][m["opt_idx"][t]][0] for t in range(len(tuples))]
        rt = [tuples[t][m["opt_idx"][t]][1] for t in range(len(tuples))]
        ok, ov, _mk = R.check_plan(m["start"], m["mask"], rt, k)
        rec["milp"]["feasible"], rec["milp"]["overlaps"] = bool(ok), ov
    tab, optmap = R.table_from_tuples(tuples)
    for key, dt in (("bruteforce_f64", np.float64), ("bruteforce_f32", np.float32)):
        bf = RC.brute_force(tab, optmap, integer_starts=True, dtype=dt)
        rec[key] = {"total_completion": bf[0], "opt": list(bf[1]), "prio": list(bf[2])}
    print(name, "status", m["status"], "milp", m["total_completion"], "bf", rec["bruteforce_f64"]["total_completion"],
          "%.1fs" % rec["milp"]["wall_s"], flush=True)
    return rec


def jobs():
    out = []
    for i, opts in enumerate(([8], [1, 2], [1, 2, 4, 8], [4, 8], [2, 4, 8])):
        out.append(("J3_g%s_seed%d" % ("".join(map(str, opts)), 200 + i), probe_tuples(3, opts, 200 + i), 1200))
    for i, opts in enumerate(([8], [1, 2], [1, 2, 4, 8], [4, 8], [2, 8], [1, 8])):
        out.append(("J4_g%s_seed%d" % ("".join(map(str, opts)), 210 + i), probe_tuples(4, opts, 210 + i), 1200))
    for i, opts in enumerate(([8], [4, 8], [2, 4, 8])):
        out.append(("J5_g%s_seed%d" % ("".join(map(str, opts)), 220 + i), probe_tuples(5, opts, 220 + i), 1200))
    for seed in range(230, 233):
        out.append(("H4_hetero_seed%d" % seed, hetero_tuples(4, seed), 1200))
    for seed in range(240, 243):
        out.append(("H5_hetero_seed%d" % seed, hetero_tuples(5, seed), 1200))
    return out


def main():
    import multiprocessing as mp
    workers = int(os.environ.get("GEN_GOLDEN_WORKERS", "6"))
    with mp.get_context("spawn").Pool(workers) as pool:
        recs = pool.map(worker, jobs(), chunksize=1)
    out = {"generator": "oracle/gen_completion.py",
           "about": "Sum of completion times sum_t (start_t + rt_t), integer starts, one node of 8 GPUs.  Not pinned "
                    "against the reference: its completion-time branch (saturn/solver/milp.py:89,174-182, "
                    "makespan_opt=False) is unreachable from solve() (milp.py:372) and bounds each completion by "
                    "the start alone.  milp = oracle/ref_completion.py milp_solve under HiGHS with mip_rel_gap = 0; "
                    "bruteforce_* = exhaustive list-schedule optimum (oracle/ref_completion.py brute_force).",
           "scipy": __import__("scipy").__version__, "cases": recs}
    dst = os.path.join(ROOT, "tests", "golden", "completion_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, "proven optimal:", sum(r["milp"]["proven_optimal"] for r in recs), "of", len(recs))


if __name__ == "__main__":
    main()
