"""Round 2: launch each kernel of interest a few times (for ncu captures).

    python scripts/profile_r02.py eval|search|search_full|pos|init
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from saturn_b200 import _lib  # noqa: E402
from saturn_b200.engine import Engine, random_candidates  # noqa: E402
from saturn_b200.synth import synth_table  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "eval"
eng = Engine(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
WAVE = SMS * 8 * 32
if which in ("eval", "eval_plain"):
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    opt, prio = random_candidates(eng, WAVE * 28, valid, seed=1)    # the bench batch
    out = torch.empty(WAVE * 28, dtype=torch.float32, device="cuda")
    for _ in range(5):
        eng.eval(opt, prio, out=out, _plain_addr=(which == "eval_plain"))
    torch.cuda.synchronize()
if which in ("search", "search_full"):
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    wave = eng.search_wave(reduced=True)
    eng.search_init(wave * round((1 << 20) / wave), seed=0, reduced=True, t_start=5e-4, t_end=1e-6, total_rounds=64,
                    resample_every=-1, _extra_flags=(_lib.HOOK_NO_INCREMENTAL if which == "search_full" else 0))
    eng.search_round(24)
    torch.cuda.synchronize()
if which == "pos":
    T, valid = synth_table(1024, 8, 8, seed=0)
    eng.set_table(T)
    eng.search_init(131072, seed=0, reduced=True, t_start=5e-4, t_end=1e-6, total_rounds=64, resample_every=-1)
    eng.search_round(24)
    torch.cuda.synchronize()
if which == "init":
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    for s in range(3):
        eng.search_init(1 << 20, seed=s, reduced=True)
    torch.cuda.synchronize()
print("ok", which)
