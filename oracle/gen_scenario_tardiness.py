"""Fixtures for the worst and mean (weighted) total tardiness and completion time over runtime scenarios (ORACLE
INFRASTRUCTURE; runs on a CPU, needs no reference).

    python oracle/gen_scenario_tardiness.py     # writes tests/golden/scenario_tardiness_cases.json

The 20 instances of tests/golden/scenario_cases.json (oracle/gen_scenarios.py: tasks, nodes, factors, release dates),
each with seeded integer due dates and, on every even-numbered instance, seeded integer weights 1 to 4 (unit weights on
the others).  Per instance and per objective of `oracle/ref_scenario_tardiness.py` (worst_tardiness, mean_tardiness,
worst_completion, mean_completion), the exhaustive list-schedule optimum (`brute_force`) under integer starts, in fp32
(the device's rule) and in fp64, and the per-scenario totals S_k of each fp32 optimum.  There is no MILP leg: re-running
the list rule per scenario is not a natural MILP.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gen_scenarios  # noqa: E402


def instance(i):
    c = gen_scenarios.instance(i)
    J = len(c["gpu_time_tuples"])
    rng = np.random.default_rng(5000 + i)
    c["due"] = [float(x) for x in rng.integers(100, 1200, size=J)]
    c["weights"] = [float(x) for x in rng.integers(1, 5, size=J)] if i % 2 == 0 else None
    return c


def solve_case(c):
    from oracle import ref_eval as R, ref_scenario_tardiness as ST
    tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
    tab, optmap = R.table_from_tuples(tuples)
    out = dict(c)
    for obj in ST.OBJECTIVES:
        due = c["due"] if obj.endswith("tardiness") else None
        for name, dtype in (("f32", np.float32), ("f64", np.float64)):
            score, opt, prio, S = ST.brute_force(tab, optmap, c["factors"], obj, due, c["weights"], c["release"],
                                                 True, dtype, c["nodes"])
            rec = {"score": score, "opt": list(opt), "prio": list(prio)}
            if name == "f32":
                rec["totals"] = S
            out["%s_%s" % (obj, name)] = rec
    print(c["name"], {o: out[o + "_f32"]["score"] for o in ST.OBJECTIVES}, flush=True)
    return out


def main():
    cases = [solve_case(instance(i)) for i in range(20)]
    out = {"generator": "oracle/gen_scenario_tardiness.py",
           "about": "Worst total tardiness max_k S_k and summed total sum_k S_k (the mean times K) of list schedules "
                    "over K runtime scenarios, T_k[j] = fl(f[k][j] * T[j]), S_k = sum_j w_j max(C_jk - d_j, 0) folded "
                    "in schedule order (weights where given, else unit weights), integer starts, one or two nodes of "
                    "8 GPUs, release dates where given; the completion forms are the same with every d = 0.  "
                    "<objective>_f32 / _f64: the exhaustive list-schedule optimum (oracle/ref_scenario_tardiness.py "
                    "brute_force, first minimum in enumeration order) in fp32 (the device's rule, with the "
                    "per-scenario totals of the optimum) and in fp64.",
           "cases": cases}
    dst = os.path.join(ROOT, "tests", "golden", "scenario_tardiness_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, len(cases), "cases")


if __name__ == "__main__":
    main()
