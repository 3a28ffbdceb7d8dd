"""GPU: the tile-boundary measures of the streamed tile kernel (path 3) — one bulk copy per tile of packed rows and
staggered warp phases — change no score and no arg-min key.  Every
combination of their debug options (and the timing option) equals the fp32 oracle bit for bit, at batch sizes that leave
warps with 0, 1 or 2+ tiles (where the stagger gate must switch off or on), with padded rows (per-lane copies),
J = 200 (a partial last chunk), both address forms, every objective and release twin, and the fused key post."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from oracle import c_oracle, ref_eval as R, ref_release as RR
from saturn_b200 import _lib
from saturn_b200.engine import Engine, random_candidates

pytestmark = pytest.mark.gpu

KEY_MAX = 2 ** 63 - 1
OPTIONS = (_lib.TILE_DEBUG_ROW_COPIES, _lib.TILE_DEBUG_NO_STAGGER)
# every subset of the two measures switched off, and the timing option over the default and the earlier kernel
COMBOS = [sum(c) for n in range(len(OPTIONS) + 1) for c in itertools.combinations(OPTIONS, n)] + [
    _lib.TILE_DEBUG_TIMING, _lib.TILE_DEBUG_TIMING | sum(OPTIONS)]


def _wave():
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 32


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _cands(engine, J, B, valid, seed, row):
    """opt / prio of B candidates with a row stride of `row` bytes (row > J: padded rows)."""
    opt, prio = random_candidates(engine, B, valid, seed=seed)
    if row == J:
        return opt, prio
    po = torch.zeros((B, row), dtype=opt.dtype, device=opt.device)
    pp = torch.zeros((B, row), dtype=prio.dtype, device=prio.device)
    po[:, :J] = opt
    pp[:, :J] = prio
    return po[:, :J], pp[:, :J]


def _check_combos(engine, opt, prio, ref, combos=COMBOS, **kw):
    for fl in combos:
        key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
        got = engine.eval(opt, prio, best_key=key, id_base=7, _tile_debug=fl, **kw)
        torch.cuda.synchronize()
        assert engine.last_eval_path() == 3, (fl, kw)
        assert got.cpu().numpy().tobytes() == ref.tobytes(), (hex(fl), kw)
        assert int(key.item()) == _key_of(ref, 7), (hex(fl), kw)
    engine.debug_tile_wait()


@pytest.mark.parametrize("size", ["1", "31", "33", "wave-1", "wave", "wave+1", "2waves+17"])
def test_tile_fetch_hooks_at_every_batch_shape(engine, size):
    J, S = 256, 8
    w = _wave()
    B = {"1": 1, "31": 31, "33": 33, "wave-1": w - 1, "wave": w, "wave+1": w + 1, "2waves+17": 2 * w + 17}[size]
    T, valid = R.synth_table(J, S, 8, seed=J + B)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = _cands(engine, J, B, valid, B, J)
    for ints in (True, False):
        ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), ints, np.float32)
        _check_combos(engine, opt, prio, ref, integer_starts=ints)
        _check_combos(engine, opt, prio, ref, combos=[0, sum(OPTIONS)], integer_starts=ints, _plain_addr=True)


@pytest.mark.parametrize("J,row", [(256, 288), (200, 224), (224, 224), (64, 64)])
def test_tile_fetch_hooks_on_padded_rows_and_partial_chunks(engine, J, row):
    """row > J: the per-lane copies; J = 200: a partial last chunk; J = 64: too few chunks to stagger."""
    S, B = 4, 2 * _wave() + 17
    T, valid = R.synth_table(J, S, 8, seed=J)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = _cands(engine, J, B, valid, J, row)
    assert opt.stride(0) == row
    ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), True, np.float32)
    _check_combos(engine, opt, prio, ref)
    _check_combos(engine, opt, prio, ref, combos=[0, sum(OPTIONS)], _plain_addr=True)


@pytest.mark.parametrize("release", [False, True])
@pytest.mark.parametrize("fold", RR.OBJECTIVES)
def test_tile_fetch_hooks_under_every_objective(engine, fold, release):
    J, S, B = 256, 8, _wave() + 4111
    T, valid = R.synth_table(J, S, 8, seed=3)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = _cands(engine, J, B, valid, 3, J)
    span = float(RR.c_evaluate(tab, opt[:1].cpu().numpy(), prio[:1].cpu().numpy(), np.zeros(J), True, np.float64)[0])
    rng = np.random.default_rng(3)
    r = (rng.uniform(-0.1, 0.8, size=J) * span).astype(np.float32) if release else np.zeros(J, np.float32)
    w = rng.uniform(0.1, 12.0, size=J).astype(np.float32) if fold.startswith("weighted") else None
    d = (rng.uniform(0.0, 1.5, size=J) * span).astype(np.float32) if fold.endswith("tardiness") else None
    try:
        if release:
            engine.set_release(r)
        if w is not None:
            engine.set_weights(w)
        if d is not None:
            engine.set_due(d)
        for ints in (True, False):
            ref = RR.c_evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), r, ints, np.float32, threads=8,
                                objective=fold, weights=w, due=d)
            _check_combos(engine, opt, prio, ref, combos=[0, _lib.TILE_DEBUG_ROW_COPIES, _lib.TILE_DEBUG_NO_STAGGER, sum(OPTIONS)],
                          integer_starts=ints, objective=fold)
            _check_combos(engine, opt, prio, ref, combos=[0, sum(OPTIONS)], integer_starts=ints, objective=fold,
                          _plain_addr=True)
    finally:
        engine.set_release(None)


def test_tile_fetch_hooks_with_the_fused_key_post():
    """post_key / fold_prev on one rank: the kernel's tail posts the key and the next launch's warp 0 of CTA 0 (never
    gated) folds it; every hook combination ends on the same key."""
    J, S, B = 256, 8, 2 * _wave() + 17
    eng = Engine(0)
    try:
        T, valid = R.synth_table(J, S, 8, seed=11)
        eng.set_table(T)
        tab = R.canon_table(T, range(1, 9))
        arr = (C.c_void_p * 1)(eng._h.value)
        assert eng._lib.sb_xchg_connect_local(arr, 1) == 0
        keys = []
        for fl in COMBOS:
            key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=eng.device)
            refs = []
            for rnd in range(3):
                opt, prio = _cands(eng, J, B, valid, 100 + rnd, J)
                got = eng.eval(opt, prio, best_key=key, id_base=rnd * B, post_key=True, fold_prev=True, _tile_debug=fl)
                ref = c_oracle.evaluate(tab, opt.cpu().numpy(), prio.cpu().numpy(), True, np.float32)
                assert got.cpu().numpy().tobytes() == ref.tobytes(), hex(fl)
                refs.append(_key_of(ref, rnd * B))
            gmin = torch.zeros(1, dtype=torch.int64, device=eng.device)
            eng.xchg_reduce(gmin, fold=key)
            torch.cuda.synchronize()
            eng.xchg_check()
            assert int(key.item()) == int(gmin.item()) == min(refs), hex(fl)
            keys.append(int(key.item()))
        assert len(set(keys)) == 1
    finally:
        eng.close()


def test_tile_wait_counters(engine):
    """TILE_DEBUG_TIMING fills both counters (the wait is part of the loop); a call resets them."""
    J, S, B = 256, 8, 2 * _wave()
    T, valid = R.synth_table(J, S, 8, seed=5)
    engine.set_table(T)
    opt, prio = _cands(engine, J, B, valid, 5, J)
    engine.debug_tile_wait()
    engine.eval(opt, prio, _tile_debug=_lib.TILE_DEBUG_TIMING)
    wait, loop = engine.debug_tile_wait()
    assert 0 < wait < loop
    assert engine.debug_tile_wait() == (0, 0)
    engine.eval(opt, prio)
    assert engine.debug_tile_wait() == (0, 0)
