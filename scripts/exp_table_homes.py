"""C5 with the full 8-strategy table (256 KB): where the position-major kernel keeps the table.
CUDA-event timings of sb_eval on the same candidates, by route.  Writes profiles-style markdown to stdout."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from saturn_b200.engine import Engine, random_candidates, opt_by_position
from saturn_b200.synth import synth_table

eng = Engine(0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
J, S, G = 1024, 8, 8
B = SMS * 16 * 32 * 3          # 3 tiles per resident warp of the position-major kernel
T, valid = synth_table(J, S, G, seed=0)
eng.set_table(T)
stream = torch.cuda.current_stream()


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
    return ts[len(ts) // 2]


rows = []
opt, prio = random_candidates(eng, B, valid, seed=3)
obp = opt_by_position(opt, prio)
out = torch.empty(B, dtype=torch.float32, device=eng.device)
ref = eng.eval(opt, prio, _reorder=False).clone()
assert eng.last_eval_path() == 4
for name, fn, path in [
    ("job-indexed rows, tile kernel, table in global memory (round 1 route)", lambda: eng.eval(opt, prio, out=out, _reorder=False), 4),
    ("job-indexed rows re-ordered on the device + position-major kernel, table through L1 (default)", lambda: eng.eval(opt, prio, out=out), 9),
    ("job-indexed rows re-ordered on the device + position-major kernel, table over CTA pairs", lambda: eng.eval(opt, prio, out=out, _table_home=2), 9),
    ("rows by position, table in global memory, read through L1 / L2 (default)", lambda: eng.eval(obp, prio, out=out, by_position=True), 8),
    ("rows by position, table split over CTA pairs (ld.shared::cluster)", lambda: eng.eval(obp, prio, out=out, by_position=True, _table_home=2), 7),
]:
    ms = timed(fn)
    assert eng.last_eval_path() == path, (name, eng.last_eval_path())
    assert torch.equal(out, ref), name
    rows.append((name, path, ms, B / ms * 1e3))
# the reduced table (32 KB) for scale: the same kernel with the table in its own shared memory
vr = valid.any(axis=1, keepdims=True)
o1, p1 = random_candidates(eng, B, vr, seed=4)
ob1 = opt_by_position(o1, p1)
ref1 = eng.eval(o1, p1, reduced=True, _reorder=False).clone()
p_tile = eng.last_eval_path()
for name, fn, path in [
    ("reduced table: job-indexed rows, tile kernel", lambda: eng.eval(o1, p1, out=out, reduced=True, _reorder=False), p_tile),
    ("reduced table: job-indexed rows re-ordered + position-major kernel (default at J >= 1024)", lambda: eng.eval(o1, p1, out=out, reduced=True), 9),
    ("reduced table: rows by position, table in shared memory", lambda: eng.eval(ob1, p1, out=out, reduced=True, by_position=True), 5),
    ("reduced table: rows by position, table over CTA pairs (forced)", lambda: eng.eval(ob1, p1, out=out, reduced=True, by_position=True, _table_home=2), 7),
    ("reduced table: rows by position, table in global memory (forced)", lambda: eng.eval(ob1, p1, out=out, reduced=True, by_position=True, _table_home=1), 8),
]:
    ms = timed(fn)
    assert eng.last_eval_path() == path, (name, eng.last_eval_path())
    assert torch.equal(out, ref1), name
    rows.append((name, path, ms, B / ms * 1e3))
print("| route | kernel path | ms per %d candidates | candidates/s |" % B)
print("|---|---|---|---|")
for name, path, ms, rate in rows:
    print("| %s | %d | %.4f | %.3e |" % (name, path, ms, rate))
