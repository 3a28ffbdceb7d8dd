"""Plan a synthetic multi-model workload with the H100 solver through Saturn's own API.

    python examples/plan_synthetic.py [--jobs 32] [--nodes 1] [--devices 1] [--dense]

Stands in for the reference's examples/wikitext103/WikiText103.py after the trial runner has
filled `task.strategies` (saturn/trial_runner/PerformanceEvaluator.py:96-115): here the runtimes are
synthetic.  Everything below the `--- Saturn API ---` line is what a Saturn user already writes.
"""
import argparse
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from saturn.core.representations import HParams, Strategy, Task  # noqa: E402
from saturn.solver import convert_into_comprehensible, solve      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=32)
    ap.add_argument("--nodes", type=int, default=1)
    ap.add_argument("--devices", type=int, default=1, help="GPUs of this process the search is sharded over")
    ap.add_argument("--dense", action="store_true", help="also plan from the dense T[J][S][G] tensor (solve_table)")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    save_dir = tempfile.mkdtemp(prefix="saturn_b200_")
    tasks = []
    for j in range(args.jobs):
        t = Task(get_model=lambda: None, get_dataloader=lambda: range(100), loss_function=None,
                 hparams=HParams(lr=1e-4, epochs=1), name="model-%02d" % j, save_dir=save_dir)
        base = float(np.exp(rng.uniform(np.log(600), np.log(36000))))
        for g in range(1, 9):                       # what trial_runner.search() leaves behind
            if g == 1:
                t.strategies[g] = Strategy("spilled", g, {}, base * 1.3)
            elif rng.uniform() < 0.1:
                t.strategies[g] = Strategy(None, g, None, 1e8)       # every executor failed at this size
            else:
                t.strategies[g] = Strategy(rng.choice(["fsdp", "pipeline"]), g, {}, base / g ** rng.uniform(0.6, 0.95))
        tasks.append(t)

    # --- Saturn API -------------------------------------------------------------------------
    sta, tga, bss, bna, boa, makespan = solve(tasks, nodes=args.nodes, devices=args.devices)
    node_per_task, deps, starts = convert_into_comprehensible(tasks, bss, boa, tga, bna, sta)

    print("planned %d tasks on %d node(s): makespan %.0f s" % (len(tasks), args.nodes, makespan))
    for t, s in sorted(zip(tasks, starts), key=lambda x: x[1])[:12]:
        st = t.selected_strategy
        print("  %-9s node %d  start %8.0f  %d GPU(s)  %-8s  %8.0f s  after %s" % (
            t.name, node_per_task[t], s, st.gpu_apportionment, st.executor, st.runtime,
            [d.name for d in deps[t]][:3] if t in deps else []))

    if args.dense:
        # the same plan from the un-reduced profiler tensor: what the trial runner measured, before it is
        # collapsed into task.strategies (saturn_b200.solver.table_from_trials / solve_table)
        from saturn_b200 import solve_table
        execs = ["spilled", "fsdp", "pipeline"]
        T = np.full((len(tasks), len(execs), 8), 1e6, dtype=np.float32)
        mask = np.zeros(T.shape, dtype=bool)
        for j, t in enumerate(tasks):
            for g, st in t.strategies.items():
                if st.executor is not None:
                    T[j, execs.index(st.executor), g - 1] = st.runtime
                    mask[j, execs.index(st.executor), g - 1] = True
        out = solve_table(T, mask, nodes=args.nodes, devices=args.devices)
        print("dense entry: makespan %.0f s; executor per task %s ..." % (out[5], [execs[i] for i in out[6][:6]]))


if __name__ == "__main__":
    main()
