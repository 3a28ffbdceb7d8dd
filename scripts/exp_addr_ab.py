"""A/B of the headline kernel's look-up form (CUDA events, 3 x 50 launches each, alternating):
shipped (ADDR = 1: IMAD addresses, dot-product byte extraction) vs the round-1 form (IADD3 + LEA, PRMT)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from saturn_b200.engine import Engine, random_candidates  # noqa: E402
from saturn_b200.synth import synth_table  # noqa: E402

eng = Engine(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
T, valid = synth_table(256, 8, 8, seed=0)
eng.set_table(T)
B = SMS * 8 * 32 * 28
opt, prio = random_candidates(eng, B, valid, seed=1)
out = torch.empty(B, dtype=torch.float32, device="cuda")
ref = eng.eval(opt, prio, _plain_addr=True).clone()
assert torch.equal(ref, eng.eval(opt, prio))
res = {}
for rep in range(3):
    for name, plain in (("shipped (FMA-pipe look-ups)", False), ("round-1 form (IADD3 + LEA + PRMT)", True)):
        for _ in range(3):
            eng.eval(opt, prio, out=out, _plain_addr=plain)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            eng.eval(opt, prio, out=out, _plain_addr=plain)
        e1.record()
        torch.cuda.synchronize()
        res.setdefault(name, []).append(e0.elapsed_time(e1) / 50)
print("| look-up form | ms / launch (3 x 50 launches, 1,060,864 candidates) | candidates / s |\n|---|---|---|")
for k, v in res.items():
    print("| %s | %s | %.3e |" % (k, ", ".join("%.4f" % x for x in v), B / (min(v) * 1e-3)))
