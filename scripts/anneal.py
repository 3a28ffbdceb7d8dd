"""Large-population anneal on a synthetic config (BASELINE configs C4 / C5), 1..8 GPUs.

    python scripts/anneal.py --config C5 --chains 262144 --candidates 1e9
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 scripts/anneal.py ...
    python scripts/anneal.py --config C5 --devices 8 ...      # ONE process driving 8 devices (sb_search_run_multi)

Prints the best-makespan-vs-time curve (rank 0) as a markdown table: the "1e9-candidate anneal on
8xH100; makespan vs reference MILP wall-clock" item of BASELINE.json (the MILP column is "no
incumbent": HiGHS finds none at J = 24 in 30 s and the J = 1024 model has 134 M rows).
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from saturn_b200.engine import Engine  # noqa: E402
from saturn_b200.search import run_search  # noqa: E402
from saturn_b200.synth import CONFIGS, synth_table  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--chains", type=int, default=1 << 18, help="per GPU")
    ap.add_argument("--candidates", type=float, default=1e9, help="total over all GPUs")
    ap.add_argument("--exchange-every", type=int, default=16)
    ap.add_argument("--devices", type=int, default=0, help="one process, this many devices (no torchrun)")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        warm = torch.zeros(1, dtype=torch.int64, device="cuda")
        dist.all_reduce(warm, op=dist.ReduceOp.MIN)          # communicator set-up is not part of the anneal
    J, S, G, seed = CONFIGS[args.config]
    T, valid = synth_table(J, S, G, seed=seed)
    if args.devices > 1:
        from saturn_b200.engine import MultiEngine
        eng = MultiEngine(args.devices)
        world = args.devices                     # for the candidate budget below; `rank` stays 0
    else:
        eng = Engine(local)
    eng.set_table(T)
    tmin, _ = eng.reduced_table()
    usable = np.where(tmin < 1e6, tmin, np.inf)
    lb = max(float((usable * np.arange(1, 9)[None, :]).min(axis=1).sum() / 8), float(usable.min(axis=1).max()))
    rounds = max(1, int(args.candidates / (args.chains * world)) - 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = run_search(eng, chains=args.chains, rounds=rounds, seed=0, reduced=True, record_history=True,
                     exchange_every=args.exchange_every, use_dist=args.devices <= 1)
    wall = time.perf_counter() - t0
    if rank == 0:
        print("# %s anneal: J=%d, S=%d (min over strategies), G=1..%d; %d GPU(s) x %d chains x %d rounds%s\n" % (
            args.config, J, S, G, world, args.chains, res.rounds,
            " (one process, sb_search_run_multi)" if args.devices > 1 else ""))
        print("candidates evaluated: %.3e in %.3f s  (%.3e candidates/s whole job); area lower bound %.1f\n" % (
            res.evaluated, wall, res.evaluated / wall, lb))
        print("| wall s | candidates | best makespan | gap to lower bound |\n|---|---|---|---|")
        h = res.history
        picks = sorted(set([0, 1, 2, 4, 8, 16, 32, 64] + list(range(0, len(h), max(1, len(h) // 12))) + [len(h) - 1]))
        for i in picks:
            if i < len(h):
                t, n, mk = h[i]
                print("| %.3f | %.2e | %.1f | %.2f %% |" % (t, n, mk, 100 * (mk / lb - 1)))
        print("\nreference MILP on the same T: model of %d x %d tasks/options cannot be built (SURVEY §8a: 134 M rows "
              "at J=1024; HiGHS has no incumbent at J=24 after 30 s)" % (J, 8))
    if world > 1 and args.devices <= 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
