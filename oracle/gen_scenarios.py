"""Fixtures for the worst and mean makespan over runtime scenarios (ORACLE INFRASTRUCTURE; runs on a CPU, needs no
reference).

    python oracle/gen_scenarios.py     # writes tests/golden/scenario_cases.json

20 seeded instances: J = 4 to 6 tasks with one to three (gpu count, integer runtime) options each, K in {2, 4, 8}
runtime scenarios with seeded log-normal factors (sigma 0.3, median 1) rounded to multiples of 1/64, one node of 8
GPUs or (J <= 5) two, every third one with integer release dates.  Per instance, the exhaustive list-schedule optimum
of both scores (`oracle/ref_scenarios.py`, `brute_force`) under integer starts, in fp32 (the device's rule) and in
fp64, and the scenario makespans of each fp32 optimum.  There is no MILP leg: re-running the list rule per scenario
is not a natural MILP.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KS = (2, 4, 8)


def instance(i):
    rng = np.random.default_rng(1000 + i)
    J = 4 + i % 3
    nodes = 2 if (i % 4 == 3 and J <= 5) else 1
    K = KS[i % 3] if not (i % 4 == 3 and J == 5) else 2
    nopt = 2 if nodes > 1 else 3
    tuples = []
    for _ in range(J):
        base = float(rng.integers(200, 2000))
        ks = sorted(rng.choice([1, 2, 4, 8], size=int(rng.integers(1, nopt + 1)), replace=False).tolist())
        tuples.append([[int(k), float(int(base / k ** 0.8))] for k in ks])
    factors = np.round(rng.lognormal(0.0, 0.3, size=(K, J)) * 64) / 64
    factors = np.maximum(factors, 1 / 64)
    release = [float(x) for x in rng.integers(0, 800, size=J)] if i % 3 == 2 else None
    return {"name": "J%d_K%d_n%d_seed%d" % (J, K, nodes, 1000 + i), "gpu_time_tuples": tuples, "nodes": nodes,
            "factors": factors.tolist(), "release": release}


def solve_case(c):
    from oracle import ref_eval as R, ref_scenarios as S
    tuples = [[tuple(x) for x in tup] for tup in c["gpu_time_tuples"]]
    tab, optmap = R.table_from_tuples(tuples)
    out = dict(c)
    for obj in S.OBJECTIVES:
        for name, dtype in (("f32", np.float32), ("f64", np.float64)):
            score, opt, prio = S.brute_force(tab, optmap, c["factors"], obj, c["release"], True, dtype, c["nodes"])
            rec = {"score": score, "opt": list(opt), "prio": list(prio)}
            if name == "f32":
                M = S.makespans(tab, np.array([opt], np.uint8), np.array([prio], np.uint8), c["factors"],
                                c["release"], True, np.float32, c["nodes"])
                rec["makespans"] = [float(x) for x in M[0]]
            out["%s_%s" % (obj, name)] = rec
    print(c["name"], {o: out[o + "_f32"]["score"] for o in S.OBJECTIVES}, flush=True)
    return out


def main():
    cases = [solve_case(instance(i)) for i in range(20)]
    out = {"generator": "oracle/gen_scenarios.py",
           "about": "Worst makespan max_k M_k and summed makespan sum_k M_k (the mean times K) of list schedules over K "
                    "runtime scenarios, T_k[j] = fl(f[k][j] * T[j]), integer starts, one or two nodes of 8 GPUs, "
                    "release dates where given.  <objective>_f32 / _f64: the exhaustive list-schedule optimum "
                    "(oracle/ref_scenarios.py brute_force, first minimum in enumeration order) in fp32 (the device's "
                    "rule, with the scenario makespans of the optimum) and in fp64.",
           "cases": cases}
    dst = os.path.join(ROOT, "tests", "golden", "scenario_cases.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", dst, len(cases), "cases")


if __name__ == "__main__":
    main()
