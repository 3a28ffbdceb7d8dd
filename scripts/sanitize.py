"""Small run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from saturn_b200 import _lib
from saturn_b200.engine import Engine, random_candidates, opt_by_position
from saturn_b200.search import run_search
from saturn_b200.synth import synth_table

eng = Engine(0)
for (J, S, G, B) in [(64, 6, 8, 2000), (100, 3, 8, 777), (300, 2, 8, 500)]:
    T, valid = synth_table(J, S, G, seed=1)
    eng.set_table(T)
    opt, prio = random_candidates(eng, B, valid, seed=2)
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=eng.device)
    a = eng.eval(opt, prio, best_key=key)
    b = eng.eval(opt, prio, _no_stream=True)
    c = eng.eval(opt.contiguous(), prio.contiguous())
    d = eng.eval(opt, prio, _force_generic=True)
    e, st, mk = eng.eval_full(opt, prio)
    f = eng.eval(opt, prio, alt_shape=True)                  # round 2: the warp-shuffle shape
    g = eng.eval(opt, prio, _plain_addr=True)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, d) and torch.equal(a, e)
    assert torch.equal(a, f) and torch.equal(a, g)
    # round 2: position-major scoring with the table in shared memory / global memory / a CTA pair, and the
    # device-side re-ordering of job-indexed rows in front of it
    obp = opt_by_position(opt, prio)
    for kw in ({}, {"_table_home": 1}, {"_table_home": 2}):
        assert torch.equal(a, eng.eval(obp, prio, by_position=True, **kw))
    assert torch.equal(a, eng.eval(opt, prio, _reorder=True)) and eng.last_eval_path() == 9
    assert eng.validate(opt, prio) == 0
    r = run_search(eng, chains=2048, rounds=6, use_dist=False)
    eng.decode(r.opt, r.prio)
    # round 2: incremental rounds with the verify hook (snapshots, windowed moves, in-kernel tournament)
    r = run_search(eng, chains=2048, rounds=20, reduced=True, use_dist=False, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL)
    assert eng.search_verify_count() == 0 and eng.search_validate() == 0
# large J: position-major search populations (k_search_pos), ragged tails, one and two nodes
for (J, nodes, chains) in [(1030, 1, 300), (777, 2, 130), (513, 1, 64)]:
    T, valid = synth_table(J, 1, 8, seed=3)
    eng.set_table(T, nodes=nodes)
    r = run_search(eng, chains=chains, rounds=6, reduced=True, use_dist=False)
    r = run_search(eng, chains=chains, rounds=18, reduced=True, use_dist=False, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, resample_every=4)
    assert eng.search_verify_count() == 0 and eng.search_validate() == 0
    eng.search_inject(r.opt, r.prio, copies=3)
    eng.search_resample()
    eng.search_round(2)
    eng.search_best()
# a table beyond one SM's shared memory (J = 1024, S = 8): default routes 9 and 8, and the round-1 route 4
T, valid = synth_table(1024, 8, 8, seed=4)
eng.set_table(T)
opt, prio = random_candidates(eng, 600, valid, seed=5)
a = eng.eval(opt, prio)
assert eng.last_eval_path() == 9
b = eng.eval(opt_by_position(opt, prio), prio, by_position=True)
assert eng.last_eval_path() == 8
c = eng.eval(opt, prio, _reorder=False)
assert eng.last_eval_path() == 4
d = eng.eval(opt_by_position(opt, prio), prio, by_position=True, _table_home=2)
torch.cuda.synchronize()
assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, d)
print("sanitize run ok")
