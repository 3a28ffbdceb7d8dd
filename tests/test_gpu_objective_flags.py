"""GPU: the return code of every combination of the objective flags and SB_FLAG_RELEASE against every state of the
per-job arrays on the handle, through sb_eval (B = 0: every check, no launch) and sb_search_init, and of every
combination through sb_search_wave, which refuses only the combinations that can never run.  The expected code comes
from the rules stated once below, so that a change in how the library decodes its flags cannot move a code."""
import ctypes as C
import itertools

import numpy as np
import pytest

from oracle import ref_eval as R

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_STATE = 0, -1, -3


def _refused(flags, lib):
    """The combinations of objective flags the ABI refuses (SB_ERR_ARG) whatever the handle holds."""
    SUM, W, DUE = flags & lib.FLAG_SUM_COMPLETION, flags & lib.FLAG_WEIGHTED, flags & lib.FLAG_DUE
    ML, LC, MT = flags & lib.FLAG_MAX_LATENESS, flags & lib.FLAG_LATE_COUNT, flags & lib.FLAG_MAX_TARDINESS
    if (LC or MT) and not (SUM and DUE):
        return True                                     # the late count and the maximum tardiness modify the tardiness
    if MT and (LC or ML):
        return True
    if ML and (SUM or W or DUE):
        return True                                     # the maximum lateness is an objective of its own
    return bool((W or DUE) and not SUM)                 # weights and due dates score the sum form


def _expected(flags, lib, has_w, has_d, has_r, q_exact):
    """The ABI's rules (include/saturn_b200.h): every refusal of a flag combination (SB_ERR_ARG) comes first, then
    the arrays the flags read (SB_ERR_STATE), where the maximum lateness also needs a due-date spread below 2^24
    (SB_ERR_ARG) once it has due dates."""
    W, DUE = flags & lib.FLAG_WEIGHTED, flags & lib.FLAG_DUE
    ML, REL = flags & lib.FLAG_MAX_LATENESS, flags & lib.FLAG_RELEASE
    if _refused(flags, lib):
        return ERR_ARG
    if (ML or DUE) and not has_d:
        return ERR_STATE
    if ML and not q_exact:
        return ERR_ARG
    if W and not has_w:
        return ERR_STATE
    if REL and not has_r:
        return ERR_STATE
    return OK


def test_flag_combinations_against_handle_states(engine):
    from saturn_b200 import _lib
    J = 24
    T, valid = R.synth_table(J, 2, 8, seed=3)
    bits = (_lib.FLAG_SUM_COMPLETION, _lib.FLAG_WEIGHTED, _lib.FLAG_DUE, _lib.FLAG_MAX_LATENESS, _lib.FLAG_LATE_COUNT,
            _lib.FLAG_MAX_TARDINESS, _lib.FLAG_RELEASE)
    narrow = np.arange(J, dtype=np.float32) * 3.0 - 20.0
    wide = np.zeros(J, np.float32)
    wide[0], wide[1] = -9.0e6, 9.0e6                   # spread 1.8e7 >= 2^24: the tails would round
    weights = np.linspace(0.5, 4.0, J).astype(np.float32)
    release = np.linspace(-1.0, 30.0, J).astype(np.float32)
    # state: (weights, due dates, release dates)
    states = {
        "nothing": (None, None, None),
        "weights": (weights, None, None),
        "due": (None, narrow, None),
        "release": (None, None, release),
        "wide_due": (None, wide, None),
        "all_wide_due": (weights, wide, release),
        "all": (weights, narrow, release),
    }
    seen = set()
    try:
        for name, (w, d, r) in states.items():
            engine.set_table(T)
            engine.set_weights(w)
            engine.set_due(d)
            engine.set_release(r)
            q_exact = d is None or float(d.max()) - float(d.min()) < 2.0 ** 24
            for pick in itertools.product((0, 1), repeat=len(bits)):
                flags = sum(b for b, on in zip(bits, pick) if on)
                want = _expected(flags, _lib, w is not None, d is not None, r is not None, q_exact)
                seen.add(want)
                got = engine._lib.sb_eval(engine._h, None, None, 0, J, flags, None, None, 0)
                assert got == want, (name, hex(flags), "sb_eval", got, want)
                p = _lib.SearchParams(seed=1, chains=64, flags=_lib.FLAG_REDUCED | flags, t_start=0.01, t_end=1e-4,
                                      total_rounds=2)
                got = engine._lib.sb_search_init(engine._h, C.byref(p), None, None)
                assert got == want, (name, hex(flags), "sb_search_init", got, want)
                # the wave sizes a population before any array is set: it refuses only what can never run
                n = C.c_int64(0)
                got = engine._lib.sb_search_wave(engine._h, _lib.FLAG_REDUCED | flags, C.byref(n))
                assert got == (ERR_ARG if _refused(flags, _lib) else OK), (name, hex(flags), "sb_search_wave", got)
                assert (n.value > 0) == (got == OK)
    finally:
        engine.set_table(T)                            # clears every per-job array of the shared engine
    assert seen == {OK, ERR_ARG, ERR_STATE}
