"""GPU: the CUDA path (through the C ABI) against the oracle — bit-exact for slot indices, integer
starts and fp32 makespans; within 1e-6 relative of the float64 oracle for integer-start plans."""
import numpy as np
import pytest
import torch

from oracle import c_oracle, ref_eval as R
from saturn_b200.engine import padded_rows, random_candidates

pytestmark = pytest.mark.gpu

SHAPES = [  # (J, S, G, B)   BASELINE configs C1..C4 shapes + ragged sizes
    (4, 2, 2, 1000),       # C1
    (8, 3, 8, 5000),       # C2 (wikitext103 shape)
    (64, 6, 8, 20000),     # C3
    (256, 8, 8, 20000),    # C4 (the headline shape)
    (5, 1, 4, 333),
    (17, 2, 8, 1234),
    (100, 4, 7, 4097),
    (255, 3, 8, 2049),
]


def _setup(engine, J, S, G, B, seed=0):
    T, valid = R.synth_table(J, S, G, seed=seed)
    engine.set_table(T)
    opt, prio = random_candidates(engine, B, valid, seed=seed + 1)
    tab = R.canon_table(T, range(1, G + 1))
    return T, valid, tab, opt, prio


@pytest.mark.parametrize("J,S,G,B", SHAPES)
@pytest.mark.parametrize("ints", [True, False])
def test_makespan_bit_exact_vs_oracle_fp32(engine, J, S, G, B, ints):
    T, valid, tab, opt, prio = _setup(engine, J, S, G, B)
    assert engine.validate(opt, prio) == 0
    mk = engine.eval(opt, prio, integer_starts=ints)
    torch.cuda.synchronize()
    assert engine.last_eval_path() == 3          # tile kernel: TMA opt rows + streamed prio rows
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32, threads=8)
    assert np.array_equal(mk.cpu().numpy(), ref)
    ref64 = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float64, threads=8)
    rel = np.max(np.abs(mk.cpu().numpy().astype(np.float64) - ref64) / ref64)
    assert rel <= (1e-6 if ints else 2e-6)       # tolerance: 1e-6 rel (integer starts: <= 2^-24)


@pytest.mark.parametrize("J,S,G,B", SHAPES[:5])
@pytest.mark.parametrize("ints", [True, False])
def test_slot_indices_and_starts_bit_exact(engine, J, S, G, B, ints):
    T, valid, tab, opt, prio = _setup(engine, J, S, G, min(B, 4000), seed=3)
    mk, start, mask = engine.eval_full(opt, prio, integer_starts=ints)
    torch.cuda.synchronize()
    ref, rstart, rmask = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32,
                                           want_plan=True, threads=8)
    assert np.array_equal(mask.cpu().numpy().astype(np.uint32), rmask)      # integer slot indices: bit-exact
    assert np.array_equal(start.cpu().numpy(), rstart)
    assert np.array_equal(mk.cpu().numpy(), ref)
    assert np.array_equal(engine.eval(opt, prio, integer_starts=ints).cpu().numpy(), ref)   # fast == full


def test_all_kernel_paths_agree(engine):
    """Streaming tile kernel, TMA-only tile kernel, plain-load tile kernel (unaligned rows) and the
    generic kernel are four independent data paths over the same step function."""
    J, S, G, B = 100, 4, 8, 3001
    T, valid, tab, opt, prio = _setup(engine, J, S, G, B, seed=5)
    a = engine.eval(opt, prio)
    assert engine.last_eval_path() == 3
    a2 = engine.eval(opt, prio, _no_stream=True)
    assert engine.last_eval_path() == 2
    assert torch.equal(a, a2)
    for ints in (True, False):            # the streaming kernel with and without the FMA-pipe address form
        x = engine.eval(opt, prio, integer_starts=ints)
        y = engine.eval(opt, prio, integer_starts=ints, _plain_addr=True)
        assert engine.last_eval_path() == 3 and torch.equal(x, y)
    for ints in (True, False):            # the alternate warp-shuffle shape (4 candidates per warp, 8 lanes each)
        x = engine.eval(opt, prio, integer_starts=ints)
        key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
        y = engine.eval(opt, prio, integer_starts=ints, alt_shape=True, best_key=key, id_base=7)
        assert engine.last_eval_path() == 6 and torch.equal(x, y)
        k = int(key.item())
        assert (k & 0xffffffff) == 7 + int(torch.argmin(x).item()) and (k >> 32) == int(x.min().view(torch.int32).item())
    opt_u = opt.contiguous()              # row stride J = 100 bytes: not 16-byte aligned
    prio_u = prio.contiguous()
    b = engine.eval(opt_u, prio_u)
    assert engine.last_eval_path() == 1
    c = engine.eval(opt, prio, _force_generic=True)
    assert engine.last_eval_path() == 0
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("J,S", [(300, 2), (1024, 1)])
def test_u16_priorities(engine, J, S):
    B = 1500
    T, valid, tab, opt, prio = _setup(engine, J, S, 8, B, seed=7)
    assert prio.dtype == torch.uint16
    mk = engine.eval(opt, prio)
    torch.cuda.synchronize()
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy().astype(np.uint16), True, np.float32, threads=8)
    assert np.array_equal(mk.cpu().numpy(), ref)
    g = engine.eval(opt, prio, _force_generic=True)
    assert torch.equal(mk, g)
    assert torch.equal(mk, engine.eval(opt, prio, _no_stream=True))
    assert torch.equal(mk, engine.eval(opt, prio, alt_shape=True)) and engine.last_eval_path() == 6


def test_reduced_table_matches_profiler_reduction(engine):
    J, S, G = 64, 6, 8
    T, valid = R.synth_table(J, S, G, seed=11)
    T[5, 2, 3] = T[5, 1, 3]                     # a tie: the first (lowest s) minimum must win
    engine.set_table(T)
    tmin, args = engine.reduced_table()
    tab = R.canon_table(T, range(1, G + 1))
    rmin, rarg = R.reduce_table(tab)
    assert np.array_equal(tmin, rmin) and np.array_equal(args, rarg)
    # reduced-mode evaluation == full-mode evaluation of the arg-min strategies
    rng = np.random.default_rng(0)
    B = 2000
    col = rng.integers(0, 8, size=(B, J)).astype(np.uint8)
    opt_r = padded_rows(B, J, torch.uint8, engine.device)
    opt_f = padded_rows(B, J, torch.uint8, engine.device)
    opt_r.copy_(torch.from_numpy(col))
    opt_f.copy_(torch.from_numpy((rarg[np.arange(J)[None, :], col] << 3) | col))
    _, prio = random_candidates(engine, B, valid, seed=2)
    a = engine.eval(opt_r, prio, reduced=True)
    b = engine.eval(opt_f, prio, reduced=False)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_gcount_mapping_and_absent_options(engine):
    """Columns are scattered by GPU count; a candidate that selects an option a job does not have
    gets an infinite makespan (legal but terrible), exactly as the oracle says."""
    J, S, G = 12, 2, 4
    rng = np.random.default_rng(4)
    T = rng.uniform(10, 500, size=(J, S, G)).astype(np.float32)
    gcount = [8, 1, 4, 2]
    engine.set_table(T, gcount)
    tab = R.canon_table(T, gcount)
    valid = np.ones((J, S, G), dtype=bool)
    opt, prio = random_candidates(engine, 500, valid, seed=1)
    assert set(np.unique(opt.cpu().numpy() & 7)) <= {0, 1, 3, 7}
    mk = engine.eval(opt, prio)
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), True, np.float32)
    assert np.array_equal(mk.cpu().numpy(), ref)
    opt2 = padded_rows(500, J, torch.uint8, engine.device)
    opt2.copy_(opt)
    opt2[:, 3] = 2                      # 3 GPUs: no such column
    mk2 = engine.eval(opt2, prio)
    assert torch.isinf(mk2).all()
    assert engine.validate(opt2, prio) == 500
    prio2 = padded_rows(500, J, torch.uint8, engine.device)
    prio2.copy_(prio)
    prio2[7, 0] = prio2[7, 1]           # not a permutation
    assert engine.validate(opt, prio2) == 1


def test_sentinel_cells_are_legal_but_terrible(engine):
    J, S, G = 16, 3, 8
    T, valid = R.synth_table(J, S, G, seed=2)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    allv = np.ones_like(valid)
    opt, prio = random_candidates(engine, 2000, allv, seed=3)     # selects masked (1e8) cells too
    mk = engine.eval(opt, prio).cpu().numpy()
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), True, np.float32)
    assert np.array_equal(mk, ref) and (mk >= 1e8).any()


def test_empty_single_and_ragged_batches(engine):
    J, S, G = 64, 6, 8
    T, valid, tab, opt, prio = _setup(engine, J, S, G, 100, seed=9)
    out = engine.eval(opt[:0], prio[:0])
    assert out.numel() == 0
    for B in (1, 31, 32, 33, 100):
        mk = engine.eval(opt[:B], prio[:B]).cpu().numpy()
        ref = c_oracle.evaluate(tab, opt[:B].cpu().numpy(), prio[:B].cpu().numpy(), True, np.float32)
        assert np.array_equal(mk, ref)


def test_best_key_is_argmin(engine):
    J, S, G, B = 64, 6, 8, 50000
    T, valid, tab, opt, prio = _setup(engine, J, S, G, B, seed=13)
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
    mk = engine.eval(opt, prio, best_key=key, id_base=1000)
    torch.cuda.synchronize()
    k = int(key.item())
    m = mk.cpu().numpy()
    best = int(np.flatnonzero(m == m.min())[0])
    assert (k & 0xffffffff) == 1000 + best
    assert np.array([(k >> 32)], dtype=np.uint32).view(np.float32)[0] == m.min()


def test_golden_candidates(engine, golden):
    """The brute-force optimal candidates recorded next to the reference MILP runs evaluate, on the
    GPU, to the recorded optimum (= the MILP's proven optimum)."""
    for rec in golden["cases"]:
        if rec["variant"] != "tight_m":
            continue
        tuples = [[tuple(x) for x in t] for t in rec["gpu_time_tuples"]]
        tab, om = R.table_from_tuples(tuples)
        J, S = tab.shape[0], tab.shape[1]
        engine.set_table(tab.astype(np.float32), list(range(1, 9)))
        for key, ints in (("bruteforce_int", True), ("bruteforce_real", False)):
            bf = rec[key]
            opt = padded_rows(1, J, torch.uint8, engine.device)
            prio = padded_rows(1, J, torch.uint8, engine.device)
            opt.copy_(torch.tensor([bf["opt"]], dtype=torch.uint8))
            prio.copy_(torch.tensor([bf["prio"]], dtype=torch.uint8))
            mk = float(engine.eval(opt, prio, integer_starts=ints).item())
            assert mk == pytest.approx(bf["makespan"], rel=1e-6)
            if ints and rec["proven_optimal"]:
                assert mk == pytest.approx(rec["makespan"], rel=1e-6)


def test_host_buffer_path_equals_device_path(engine):
    J, S, G, B = 256, 8, 8, 200000
    T, valid = R.synth_table(J, S, G, seed=0)
    engine.set_table(T)
    opt_h, prio_h = random_candidates(engine, B, valid, seed=21, device="cpu", pinned=True)
    out_h = engine.eval_host(opt_h, prio_h)
    opt_d = padded_rows(B, J, torch.uint8, engine.device)
    prio_d = padded_rows(B, J, torch.uint8, engine.device)
    opt_d.copy_(opt_h)
    prio_d.copy_(prio_h)
    out_d = engine.eval(opt_d, prio_d)
    torch.cuda.synchronize()
    assert torch.equal(out_h, out_d.cpu())


def test_full_size_properties(engine):
    """BASELINE C4 at full batch size (1e6 candidates of J=256,S=8,G=8) through size-independent
    properties: (a) exact homogeneity — scaling T by 2 scales every real-valued makespan by exactly
    2; (b) bounds — makespan >= max job runtime and >= total GPU-seconds / 8; (c) the generic
    kernel reproduces the tile kernel bit for bit; (d) a 20000-candidate slice equals the oracle."""
    J, S, G, B = 256, 8, 8, 1_000_000
    T, valid = R.synth_table(J, S, G, seed=0)
    engine.set_table(T)
    opt, prio = random_candidates(engine, B, valid, seed=1)
    a_int = engine.eval(opt, prio, integer_starts=True)
    a_real = engine.eval(opt, prio, integer_starts=False)
    g_int = engine.eval(opt, prio, integer_starts=True, _force_generic=True)
    # bounds, on the device with torch as plumbing
    tabt = torch.from_numpy(R.canon_table(T, range(1, 9))).to(engine.device).reshape(J, S * 8)
    o = opt.long()
    rt = tabt[torch.arange(J, device=engine.device)[None, :], o]
    k = (o & 7) + 1
    lower = torch.maximum(rt.max(dim=1).values, (rt * k).sum(dim=1) / 8 * (1 - 1e-6))
    torch.cuda.synchronize()
    assert torch.equal(a_int, g_int)
    assert bool((a_real >= lower).all()) and bool((a_int >= a_real).all())
    engine.set_table(T * 2)
    b_real = engine.eval(opt, prio, integer_starts=False)
    torch.cuda.synchronize()
    assert torch.equal(b_real, a_real * 2)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    sl = slice(500_000, 520_000)
    ref = c_oracle.evaluate(tab, opt[sl].cpu().numpy(), prio[sl].cpu().numpy(), True, np.float32, threads=8)
    assert np.array_equal(a_int[sl].cpu().numpy(), ref)


@pytest.mark.parametrize("J,nodes,B", [(64, 2, 6000), (100, 3, 3001), (256, 2, 4000), (300, 4, 700)])
@pytest.mark.parametrize("ints", [True, False])
def test_multi_node_parity(engine, J, nodes, B, ints):
    """Several nodes (gangs confined to one node, milp.py:117-137): every kernel path == the oracle,
    bit for bit, including start times and (node, GPU-mask) per job."""
    T, valid = R.synth_table(J, 1, 8, seed=J, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=4, nodes=nodes)
    assert int((opt >> 3).max()) == nodes - 1 and engine.validate(opt, prio, reduced=True) == 0
    with pytest.raises(Exception):
        engine.eval(opt, prio, reduced=False)                   # multi-node needs the reduced table
    a = engine.eval(opt, prio, integer_starts=ints, reduced=True)
    assert engine.last_eval_path() == 3
    pnp = prio.cpu().numpy()
    ref, rstart, rmask = c_oracle.evaluate(tab, opt.cpu().numpy(), pnp, ints, np.float32, want_plan=True, threads=8,
                                           nodes=nodes)
    assert np.array_equal(a.cpu().numpy(), ref)
    assert torch.equal(a, engine.eval(opt, prio, integer_starts=ints, reduced=True, _no_stream=True))
    assert torch.equal(a, engine.eval(opt, prio, integer_starts=ints, reduced=True, _force_generic=True))
    assert torch.equal(a, engine.eval(opt.contiguous(), prio.contiguous(), integer_starts=ints, reduced=True))
    mk, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=True)
    assert np.array_equal(mk.cpu().numpy(), ref) and np.array_equal(start.cpu().numpy(), rstart)
    assert np.array_equal(mask.cpu().numpy().astype(np.uint32), rmask)
    bad = padded_rows(B, J, torch.uint8, engine.device)
    bad.copy_(opt)
    bad[5, 2] = (nodes << 3) | 1                                  # a node that does not exist
    assert engine.validate(bad, prio, reduced=True) == 1


def test_fuzz_small_and_odd_shapes(engine):
    """Seeded sweep over small / odd shapes (J from 1, ragged GPU-count sets, 1-3 nodes, both start
    modes, aligned and unaligned rows): every kernel path must equal the Python oracle exactly."""
    rng = np.random.default_rng(2024)
    for trial in range(40):
        J = int(rng.integers(1, 41))
        nodes = int(rng.choice([1, 1, 2, 3]))
        S = 1 if nodes > 1 else int(rng.integers(1, 5))
        G = int(rng.integers(1, 9))
        gcount = sorted(rng.choice(np.arange(1, 9), size=G, replace=False).tolist())
        ints = bool(rng.integers(0, 2))
        B = int(rng.integers(1, 90))
        T = rng.uniform(1.0, 900.0, size=(J, S, G)).astype(np.float32)
        if trial % 3 == 0:
            T = np.ceil(T)                                  # integer runtimes: lots of exact ties
        engine.set_table(T, gcount, nodes=nodes)
        tab = R.canon_table(T, gcount)
        valid = np.ones((J, S, G), dtype=bool)
        opt, prio = random_candidates(engine, B, valid, seed=trial, nodes=nodes)
        red = nodes > 1
        o_np, p_np = opt.cpu().numpy(), prio.cpu().numpy()
        ref = np.array([R.list_schedule(tab, o_np[b], p_np[b], ints, np.float32, nodes=nodes)[0] for b in range(B)],
                       dtype=np.float32)
        for kw in ({}, {"_no_stream": True}, {"_force_generic": True}):
            got = engine.eval(opt, prio, integer_starts=ints, reduced=red, **kw).cpu().numpy()
            assert np.array_equal(got, ref), (trial, J, S, gcount, nodes, ints, kw)
        got = engine.eval(opt.contiguous(), prio.contiguous(), integer_starts=ints, reduced=red).cpu().numpy()
        assert np.array_equal(got, ref), (trial, "unaligned")
        mk, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=red)
        b = int(rng.integers(0, B))
        m1, s1, k1, _ = R.list_schedule(tab, o_np[b], p_np[b], ints, np.float32, nodes=nodes)
        assert float(mk[b]) == m1 and mask[b].cpu().numpy().astype(np.uint32).tolist() == k1
        assert [float(x) for x in start[b].cpu().numpy()] == [float(x) for x in s1]


def test_large_batch_64bit_indexing(engine):
    """9.5 M candidates of J = 256: each encoding array is 2.4 GB, so row offsets exceed 2^31 bytes."""
    J, S, G = 256, 8, 8
    B = 132 * 16 * 32 * 140                                  # 9,461,760
    T, valid = R.synth_table(J, S, G, seed=0)
    engine.set_table(T)
    opt, prio = random_candidates(engine, B, valid, seed=77)
    assert opt.stride(0) * (B - 1) > 2 ** 31
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
    out = engine.eval(opt, prio, best_key=key)
    torch.cuda.synchronize()
    tab = R.canon_table(T, range(1, 9))
    for lo in (0, B // 2 + 12345, B - 4000):
        sl = slice(lo, lo + 4000)
        ref = c_oracle.evaluate(tab, opt[sl].cpu().numpy(), prio[sl].cpu().numpy(), True, np.float32, threads=8)
        assert np.array_equal(out[sl].cpu().numpy(), ref)
    k = int(key.item())
    assert np.array([(k >> 32)], dtype=np.uint32).view(np.float32)[0] == float(out.min())
    assert int(out.argmin()) == (k & 0xffffffff)
    del opt, prio, out
    torch.cuda.empty_cache()


def test_large_table_in_global_memory(engine):
    """J = 1024 with the full 8-strategy table (256 KB) does not fit in one SM's shared memory.  Default route
    (path 9): the opt rows are re-ordered into schedule order on the device and scored by the position-major
    kernel, which reads the table through L1.  With that route switched off the tile kernel keeps the table in
    global memory beside its tiles (path 4).  Both equal the oracle and the generic kernel."""
    J, S, G, B = 1024, 8, 8, 3000
    T, valid = R.synth_table(J, S, G, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy().astype(np.uint16), True, np.float32, threads=8)
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
    a = engine.eval(opt, prio, best_key=key, id_base=7)
    assert engine.last_eval_path() == 9
    assert np.array_equal(a.cpu().numpy(), ref)
    i = int(np.argmin(ref))
    assert int(key.item()) == (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (7 + i)
    b = engine.eval(opt, prio, _reorder=False)
    assert engine.last_eval_path() == 4
    assert torch.equal(a, b)
    assert torch.equal(a, engine.eval(opt, prio, _force_generic=True))
    assert np.array_equal(engine.eval(opt, prio, integer_starts=False).cpu().numpy(),
                          c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy().astype(np.uint16), False,
                                            np.float32, threads=8))
    # 512 KB of table: same route
    T2, valid2 = R.synth_table(2048, 8, G, seed=5)
    engine.set_table(T2)
    o2, p2 = random_candidates(engine, 300, valid2, seed=6)
    c = engine.eval(o2, p2)
    assert engine.last_eval_path() == 9
    assert np.array_equal(c.cpu().numpy(), c_oracle.evaluate(R.canon_table(T2, range(1, 9)), o2.cpu().numpy(),
                                                             p2.cpu().numpy().astype(np.uint16), True, np.float32,
                                                             threads=8))


@pytest.mark.parametrize("J,S,B", [(256, 8, 3000), (64, 6, 1500), (1024, 1, 700), (33, 2, 77), (1500, 1, 200),
                                   (520, 3, 1111), (1024, 8, 40000)])
@pytest.mark.parametrize("ints", [True, False])
def test_position_major_table_homes(engine, J, S, B, ints):
    """The position-major scoring kernel with its table (a) in global memory, read through L1 / L2 (path 8: the
    home of tables beyond one SM's shared memory), (b) split over the shared memory of a CTA pair and read with
    ld.shared::cluster (path 7: the measured alternative), and the job-indexed route that re-orders the opt rows
    on the device first (path 9): all bit-exact against the oracle, same arg-min key."""
    from saturn_b200.engine import opt_by_position
    T, valid = R.synth_table(J, S, 8, seed=J + S, masked=(S > 1 and J < 1000))
    engine.set_table(T)
    reduced = S == 1
    opt, prio = random_candidates(engine, B, valid, seed=15)
    ref = c_oracle.evaluate(R.canon_table(T, range(1, 9)), opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32,
                            threads=8)
    i = int(np.argmin(ref))
    want_key = (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (1000 + i)
    obp = opt_by_position(opt, prio)
    for home, path in ((2, 7), (1, 8)):
        key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
        got = engine.eval(obp, prio, integer_starts=ints, reduced=reduced, by_position=True, best_key=key,
                          id_base=1000, _table_home=home)
        assert engine.last_eval_path() == path
        assert np.array_equal(got.cpu().numpy(), ref)
        assert int(key.item()) == want_key
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, integer_starts=ints, reduced=reduced, best_key=key, id_base=1000, _reorder=True)
    assert engine.last_eval_path() == 9
    assert np.array_equal(got.cpu().numpy(), ref)
    assert int(key.item()) == want_key
    if J * S * 32 + 16 > 227 * 1024:                               # the full C5 table: global memory is the default home
        got = engine.eval(obp, prio, integer_starts=ints, by_position=True)
        assert engine.last_eval_path() == 8
        assert np.array_equal(got.cpu().numpy(), ref)


def test_error_paths_and_unpadded_host_buffers(engine):
    from saturn_b200._lib import SaturnB200Error
    from saturn_b200.engine import Engine
    fresh = Engine(0)
    o = torch.zeros((4, 8), dtype=torch.uint8, device=fresh.device)
    with pytest.raises((SaturnB200Error, ValueError)):
        fresh.eval(o, o)                                            # no table yet
    with pytest.raises(SaturnB200Error):
        fresh.set_table(np.ones((4, 1, 9), dtype=np.float32))        # G > 8
    with pytest.raises(SaturnB200Error):
        fresh.set_table(np.ones((4, 1, 2), dtype=np.float32), [1, 9])  # gpu count 9
    with pytest.raises(SaturnB200Error):
        fresh.set_table(np.ones((4, 1, 2), dtype=np.float32), nodes=9)
    fresh.close()
    J, S, G, B = 100, 3, 8, 5000
    T, valid = R.synth_table(J, S, G, seed=8)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt_h, prio_h = random_candidates(engine, B, valid, seed=9, device="cpu")
    opt_c, prio_c = opt_h.contiguous(), prio_h.contiguous()        # row stride 100 bytes, pageable memory
    out = engine.eval_host(opt_c, prio_c, out=torch.empty(B, dtype=torch.float32))
    assert engine.last_eval_path() == 1
    ref = c_oracle.evaluate(tab, opt_c.numpy(), prio_c.numpy(), True, np.float32, threads=8)
    assert np.array_equal(out.numpy(), ref)
    with pytest.raises(TypeError):
        engine.eval(opt_h.to(engine.device).to(torch.int32), prio_h.to(engine.device))
    with pytest.raises(ValueError):
        engine.eval(opt_h.to(engine.device)[:, :50], prio_h.to(engine.device)[:, :50])


@pytest.mark.parametrize("J,S,nodes,B", [(256, 8, 1, 3000), (64, 6, 1, 1500), (1024, 1, 1, 700), (700, 1, 2, 500),
                                         (33, 2, 1, 77), (1500, 1, 1, 200)])
@pytest.mark.parametrize("ints", [True, False])
def test_opt_by_position_encoding(engine, J, S, nodes, B, ints):
    """SB_FLAG_OPT_BY_POSITION: the same candidates with opt re-encoded in schedule order (kernel path 5:
    both rows streamed through registers, no shared-memory tile) score bit-exactly like the oracle and like
    the job-indexed rows, and fold the same arg-min key."""
    from saturn_b200.engine import opt_by_position
    T, valid = R.synth_table(J, S, 8, seed=J + S, masked=(S > 1))
    engine.set_table(T, nodes=nodes)
    reduced = S == 1
    opt, prio = random_candidates(engine, B, valid, seed=5, nodes=nodes)
    ref = c_oracle.evaluate(R.canon_table(T, range(1, 9)), opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32,
                            threads=8, nodes=nodes)
    key = torch.full((1,), 2 ** 63 - 1, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt_by_position(opt, prio), prio, integer_starts=ints, reduced=reduced, by_position=True,
                      best_key=key, id_base=1000)
    assert engine.last_eval_path() == 5
    assert np.array_equal(got.cpu().numpy(), ref)
    assert torch.equal(got, engine.eval(opt, prio, integer_starts=ints, reduced=reduced))
    i = int(np.argmin(ref))                                       # first index of the minimum
    assert int(key.item()) == (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (1000 + i)


def test_opt_by_position_is_refused_where_it_cannot_run(engine):
    from saturn_b200.engine import opt_by_position
    T, valid = R.synth_table(40, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    with pytest.raises(RuntimeError, match="32-byte"):             # 40-byte rows
        engine.eval(opt_by_position(opt, prio).contiguous(), prio.contiguous(), by_position=True)
    with pytest.raises(RuntimeError, match="sb_eval only"):
        from saturn_b200 import _lib
        import ctypes as C
        bad = C.c_int64(0)
        _lib.check(engine._lib.sb_validate(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64,
                                           opt.stride(0), _lib.FLAG_OPT_BY_POSITION, C.byref(bad)))
    T2, valid2 = R.synth_table(8000, 1, 8, seed=1)                 # two nodes: 250 KB of reduced table + node states
    engine.set_table(T2, nodes=2)
    o2, p2 = random_candidates(engine, 32, valid2, seed=1, nodes=2)
    with pytest.raises(RuntimeError, match="shared memory"):
        engine.eval(opt_by_position(o2, p2), p2, reduced=True, by_position=True)


def test_c5_route_parity(engine):
    """The route bench.py's `configs.C5` measures and the J > 512 search uses: the FULL C5 table (J = 1024,
    S = 8: 256 KB, does not fit in shared memory) is reduced over strategies on the device, candidates carry
    (k - 1) per schedule position, kernel path 5 scores them on the 32 KB reduced table — bit-exact against the
    oracle run on the host-side reduction of the same table, integer and real-valued starts."""
    from saturn_b200.engine import opt_by_position
    from saturn_b200.synth import synth_table
    J, S, G, B = 1024, 8, 8, 1200
    T, valid = synth_table(J, S, G, seed=0)
    engine.set_table(T)
    vr = valid.any(axis=1, keepdims=True)
    opt, prio = random_candidates(engine, B, vr, seed=9)
    tab = R.canon_table(T, range(1, G + 1))
    tmin, args = R.reduce_table(tab)
    dev_tmin, dev_args = engine.reduced_table()
    assert np.array_equal(dev_tmin, tmin) and np.array_equal(dev_args[np.isfinite(tmin)], args[np.isfinite(tmin)])
    for ints in (True, False):
        ref = c_oracle.evaluate(tmin[:, None, :], opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32, threads=8)
        got = engine.eval(opt_by_position(opt, prio), prio, integer_starts=ints, reduced=True, by_position=True)
        assert engine.last_eval_path() == 5
        assert np.array_equal(got.cpu().numpy(), ref)
        assert torch.equal(got, engine.eval(opt, prio, integer_starts=ints, reduced=True))   # job-indexed tile kernel
