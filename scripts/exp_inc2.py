"""Diagnosis of the incremental search rounds: ms per round vs population size and tournament cadence."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from saturn_b200 import _lib  # noqa: E402
from saturn_b200.engine import Engine  # noqa: E402
from saturn_b200.synth import synth_table  # noqa: E402

eng = Engine(0)
print("| J | chains | resample | mode | ms / round | chain-rounds / s |\n|---|---|---|---|---|---|")
for J in (256, 1024):
    T, valid = synth_table(J, 8, 8, seed=0)
    eng.set_table(T)
    wave = eng.search_wave(reduced=True)
    for chains in (2 * wave, wave * round((1 << 20) / wave) if J == 256 else 4 * wave):
        for rs in ((0, 2) if J == 256 else (0, 8)):
            for name, fl in (("full", _lib.HOOK_NO_INCREMENTAL), ("incremental", 0)):
                eng.search_init(chains, seed=1, reduced=True, t_start=5e-4, t_end=1e-6, total_rounds=64, resample_every=rs,
                                _extra_flags=fl)
                eng.search_round(8)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                eng.search_round(32)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 32
                print("| %d | %d | %d | %s | %.4f | %.3e |" % (J, chains, rs, name, ms, chains / ms * 1e3), flush=True)
