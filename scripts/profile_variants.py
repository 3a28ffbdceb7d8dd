"""Launch the non-headline kernel variants once each (for ncu captures): fused search round, multi-node
evaluation, J = 1024 (u16 priorities) evaluation, real-valued starts."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from saturn_b200.engine import Engine, random_candidates
from saturn_b200.synth import synth_table

which = sys.argv[1] if len(sys.argv) > 1 else "all"
eng = Engine(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
WAVE = SMS * 16 * 32
if which in ("all", "search"):
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    eng.search_init(1 << 20, seed=0, reduced=True, t_start=5e-4, t_end=1e-6, total_rounds=20)
    eng.search_round(6)
    torch.cuda.synchronize()
if which in ("all", "multi"):
    T, valid = synth_table(256, 1, 8, seed=0, masked=False)
    eng.set_table(T, nodes=2)
    opt, prio = random_candidates(eng, WAVE * 8, valid, seed=1, nodes=2)
    for _ in range(4):
        eng.eval(opt, prio, reduced=True)
    torch.cuda.synchronize()
if which in ("all", "c5"):
    T, valid = synth_table(1024, 8, 8, seed=0)
    Tr = np.where(valid, T, np.inf).min(axis=1, keepdims=True)
    vr = np.isfinite(Tr)
    eng.set_table(np.where(vr, Tr, 1e8).astype(np.float32))
    opt, prio = random_candidates(eng, SMS * 6 * 32 * 8, vr, seed=1)
    for _ in range(4):
        eng.eval(opt, prio)
    torch.cuda.synchronize()
if which in ("all", "real"):
    T, valid = synth_table(256, 8, 8, seed=0)
    eng.set_table(T)
    opt, prio = random_candidates(eng, WAVE * 13, valid, seed=1)
    for _ in range(4):
        eng.eval(opt, prio, integer_starts=False)
    torch.cuda.synchronize()
print("ok")
