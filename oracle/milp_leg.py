"""The reference's CPU MILP, timed (ORACLE — measurement infrastructure; bench.py's cpu_baseline leg runs it).

    python oracle/milp_leg.py --sizes 8,16 --limit 12

BASELINE.json's metric has a second half — "wall-clock to match MILP makespan" — and its north_star asks
for "the reference's CPU MILP solver timed on the same box's host cores in the same run".  The reference's
solver path (saturn/solver/milp.py:89-327: PuLP model -> Gurobi/CBC) cannot run on the GPU box (no PuLP,
no MILP binary, no /root/reference there), so this runs oracle/ref_milp.py — the same model restated for
scipy's HiGHS with a sound big-M, validated against the fixtures recorded from the unmodified reference
(tests/test_oracle.py::test_milp_port_matches_reference_runs) — with the reference's own time-limit
mechanism (milp.py:23,323-325 `timeLimit`), and checks every incumbent for overlaps.  One JSON object on
stdout; bench.py then times saturn.solver.solve() on the same instances.
"""
import argparse
import json
import os
import random
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def probe_tuples(J, options, seed):
    """SURVEY §8c known-answer generator: base ~ U(500, 4000) s, T = base / g**0.8."""
    rnd = random.Random(seed)
    return [[(g, b / g ** 0.8) for g in options] for b in (rnd.uniform(500, 4000) for _ in range(J))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8,16")
    ap.add_argument("--limit", type=float, default=12.0)
    ap.add_argument("--options", default="1,2,4,8")
    args = ap.parse_args()
    os.environ.setdefault("OMP_NUM_THREADS", "1")     # HiGHS' MIP search is single-threaded
    import scipy
    from oracle import ref_eval as R, ref_milp
    options = [int(x) for x in args.options.split(",")]
    out = {"solver": "scipy %s HiGHS via oracle/ref_milp.py (reference model milp.py:89-321, sound big-M)" % scipy.__version__,
           "cores": 1, "limit_s": args.limit, "options": options, "instances": []}
    for J in [int(x) for x in args.sizes.split(",")]:
        tuples = probe_tuples(J, options, 0)
        t0 = time.perf_counter()
        m = ref_milp.solve(tuples, time_limit=args.limit)
        rec = {"J": J, "seed": 0, "n_vars": m["n_vars"], "n_cons": m["n_cons"], "build_s": m["build_s"],
               "solve_s": m["wall_s"], "wall_s": time.perf_counter() - t0, "makespan": m["makespan"],
               "result": "optimal" if m["proven_optimal"] else ("incumbent at limit" if m["makespan"] is not None
                                                                 else "no incumbent at limit")}
        if m["makespan"] is not None:
            rts = [tuples[t][o][1] for t, o in enumerate(m["opt_idx"])]
            ks = [tuples[t][o][0] for t, o in enumerate(m["opt_idx"])]
            ok, overlaps, _mk = R.check_plan(m["start"], m["mask"], rts, ks)
            rec["feasible"] = bool(ok)
            rec["overlaps"] = int(overlaps)
        out["instances"].append(rec)
    nv, nc = ref_milp.model_size(256, 8)
    out["c4_model"] = {"J": 256, "options_per_task": 8, "n_vars": nv, "n_cons": nc,
                       "formula": "vars = J*S + J*N + 2*N*G*J + J*(J-1) + 1; rows = 2J + N*G*J*S + 4*J*N*S + 2*J*N*S*G + "
                                  "2*S*N*G*J*(J-1), N=1, G=8 (SURVEY §8a A2/A3)",
                       "result": "not built: 8.4 M rows of Python/PuLP expression objects (milp.py:277-319 is an "
                                 "O(G*J^2*S) Python loop); HiGHS has no incumbent at J=24 within 30 s already"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
