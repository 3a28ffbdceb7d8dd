import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np, torch
from saturn_b200.engine import Engine, random_candidates
from saturn_b200.synth import synth_table
eng = Engine(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
for nodes in (2, 4):
    T, valid = synth_table(256, 1, 8, seed=0, masked=False)
    eng.set_table(T, nodes=nodes)
    B = SMS * 16 * 32 * 8
    opt, prio = random_candidates(eng, B, valid, seed=1, nodes=nodes)
    for _ in range(3): eng.eval(opt, prio, reduced=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): eng.eval(opt, prio, reduced=True)
    e1.record(); torch.cuda.synchronize()
    print("nodes", nodes, "cand/s %.3e" % (B * 20 / (e0.elapsed_time(e1) * 1e-3)), "path", eng.last_eval_path())
