"""A/B of the headline kernel's tile-boundary measures (k_eval_tiles, path 3) on bench.py's C4 batch.

    python scripts/exp_tile_fetch.py [--rounds 300]

Variants (the kernel's debug options, sb_debug_tile_options): the per-lane row copies with every warp starting at once (the earlier
kernel), each measure alone, and both.  Every variant is timed with CUDA events, one launch at a time, the
variants alternated in one process; then each runs once more under TILE_DEBUG_TIMING (a separate run: the
timing perturbs the kernel), which gives the share of the warps' tile-loop time spent waiting for a tile's rows.  Prints one
JSON line with the card's name, power limit and max SM clock (read-only nvidia-smi queries)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from saturn_b200 import _lib  # noqa: E402
from saturn_b200.engine import Engine, random_candidates  # noqa: E402
from saturn_b200.synth import synth_table  # noqa: E402

J, S, G = 256, 8, 8
B = 132 * 8 * 32 * 28  # bench.py's B_PER_GPU: 14 tiles for every resident warp of the H100's persistent grid
R, N = _lib.TILE_DEBUG_ROW_COPIES, _lib.TILE_DEBUG_NO_STAGGER
VARIANTS = [("row copies, no stagger", R | N), ("one copy per tile", N), ("stagger", R), ("both", 0)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=300)
    args = ap.parse_args()
    eng = Engine(0)
    T, valid = synth_table(J, S, G, seed=0)
    eng.set_table(T)
    opt, prio = random_candidates(eng, B, valid, seed=1)
    out = torch.empty(B, dtype=torch.float32, device=eng.device)
    ref = None
    for name, fl in VARIANTS:  # warm-up, and every variant gives the same bytes
        for _ in range(3):
            eng.eval(opt, prio, out=out, _tile_debug=fl)
        assert eng.last_eval_path() == 3
        got = out.clone()
        ref = got if ref is None else ref
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), name
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.rounds * len(VARIANTS))]
    k = 0
    for _ in range(args.rounds):
        for name, fl in VARIANTS:
            ev[k][0].record()
            eng.eval(opt, prio, out=out, _tile_debug=fl)
            ev[k][1].record()
            k += 1
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev]).reshape(args.rounds, len(VARIANTS))
    eng.debug_tile_wait()
    res = {}
    for i, (name, fl) in enumerate(VARIANTS):
        for _ in range(20):
            eng.eval(opt, prio, out=out, _tile_debug=fl | _lib.TILE_DEBUG_TIMING)
        wait, loop = eng.debug_tile_wait()
        med = float(np.median(ms[:, i]))
        res[name] = {"median_ms": round(med, 4), "p10_ms": round(float(np.percentile(ms[:, i], 10)), 4),
                     "p90_ms": round(float(np.percentile(ms[:, i], 90)), 4), "cand_per_s": B / (med * 1e-3),
                     "wait_fraction": round(wait / loop, 4) if loop else None}
    print(json.dumps({"card": card(), "candidates": B, "launches_per_variant": args.rounds, "variants": res}), flush=True)


if __name__ == "__main__":
    main()
