"""Round 2: fused search rounds — round-1 move generator vs windowed moves scored from position 0 vs
incremental (snapshots).  Prints a markdown table: ms per round at ~1 M chains (C4, reduced table) and the
plan quality / wall time of whole searches at the solve() population.

    python scripts/exp_incremental.py
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from saturn_b200 import _lib  # noqa: E402
from saturn_b200.engine import Engine  # noqa: E402
from saturn_b200.search import run_search  # noqa: E402
from saturn_b200.synth import synth_table  # noqa: E402

MODES = [("round-1 moves, scored from position 0", _lib.HOOK_ROUND1_MOVES),
         ("windowed moves, scored from position 0", _lib.HOOK_NO_INCREMENTAL),
         ("windowed moves, incremental (shipped)", 0),
         ("windowed moves, incremental, windows drawn with P(w) ~ w + 1 (experiment)", _lib.HOOK_WINDOW_BIAS)]


def main():
    torch.cuda.set_device(0)
    eng = Engine(0)
    print("# Fused search rounds: incremental re-evaluation (C4 table, min over strategies, integer starts)\n")
    for J, S in ((256, 8), (128, 4), (400, 8)):
        T, valid = synth_table(J, S, 8, seed=0)
        eng.set_table(T)
        wave = eng.search_wave(reduced=True)
        chains = wave * max(1, round((1 << 20) / wave))
        print("\n## J = %d: %d chains (%d per wave), CUDA events over 32 rounds after 8 warm-up rounds\n" % (J, chains, wave))
        print("| mode | ms / round | chain-rounds / s |\n|---|---|---|")
        for name, fl in MODES:
            eng.search_init(chains, seed=1, integer_starts=True, reduced=True, t_start=5e-4, t_end=1e-6, total_rounds=64,
                            resample_every=-1, _extra_flags=fl)
            eng.search_round(8)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.search_round(32)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 32
            print("| %s | %.4f | %.3e |" % (name, ms, chains / ms * 1e3))
        sys.stdout.flush()
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    wave = eng.search_wave(reduced=True)
    chains = 2 * wave
    print("\n## Whole searches on C4 (%d chains, sb_search_run, 5 seeds): mean best makespan, median wall\n" % chains)
    print("| mode | 400 rounds | 1600 rounds | equal wall: rounds that fit in the round-1 mode's 400-round time |\n|---|---|---|---|")
    base_wall = None
    for name, fl in MODES:
        cells = []
        for rounds in (400, 1600):
            mks, walls = [], []
            for seed in range(5):
                r = run_search(eng, chains=chains, rounds=rounds, seed=seed, reduced=True, use_dist=False, _extra_flags=fl)
                mks.append(r.makespan)
                walls.append(r.wall_s)
            cells.append("%.1f, %.1f ms" % (np.mean(mks), np.median(walls) * 1e3))
            if rounds == 400:
                w400 = float(np.median(walls))
        if base_wall is None:
            base_wall = w400
        rr = int(400 * base_wall / w400) // 16 * 16
        mks = [run_search(eng, chains=chains, rounds=rr, seed=seed, reduced=True, use_dist=False, _extra_flags=fl).makespan
               for seed in range(5)]
        print("| %s | %s | %s | %d rounds: %.1f |" % (name, cells[0], cells[1], rr, np.mean(mks)))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
