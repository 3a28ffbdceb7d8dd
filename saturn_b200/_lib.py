"""ctypes binding of include/saturn_b200.h.  There is no Python / CPU fallback: if the shared
library is missing or a CUDA device is absent, calls raise."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("SATURN_B200_LIB") or os.path.join(_HERE, "libsaturn_b200.so")

FLAG_INTEGER_STARTS = 1
FLAG_REDUCED = 2
FLAG_OPT_BY_POSITION = 4
FLAG_POST_KEY = 8
FLAG_FOLD_PREV = 16
FLAG_ALT_WARPSCAN = 32
FLAG_SUM_COMPLETION = 64
FLAG_WEIGHTED = 128
FLAG_DUE = 256
FLAG_RELEASE = 512
FLAG_MAX_LATENESS = 1024
FLAG_LATE_COUNT = 2048
FLAG_MAX_TARDINESS = 4096
FLAG_SQUARED = 8192
FLAG_LATE_PENALTY = 16384
FLAG_COMPLETION_PENALTY = 32768
FLAG_WORST_MAKESPAN = 65536
FLAG_MEAN_MAKESPAN = 131072
FLAG_WORST_TARDINESS = 262144
FLAG_MEAN_TARDINESS = 524288
IPC_HANDLE_BYTES = 64
# test hooks in the top bits of the same flags word: the enum in csrc/sb_internal.h says what each one forces
HOOK_FORCE_GENERIC = 0x80000000
HOOK_NO_STREAM = 0x40000000
HOOK_NO_FUSED = 0x20000000
HOOK_NO_INCREMENTAL = 0x10000000
HOOK_VERIFY_INCREMENTAL = 0x08000000
HOOK_ROUND1_MOVES = 0x04000000
HOOK_PLAIN_ADDR = 0x02000000
HOOK_WINDOW_BIAS = 0x01000000
HOOK_TABLE_GLOBAL = 0x00800000
HOOK_TABLE_PAIR = 0x00400000
HOOK_REORDER = 0x00200000
HOOK_NO_REORDER = 0x00100000
# debug options of the streamed tile kernel, set on the handle (sb_debug_tile_options; TileDebug in csrc/sb_internal.h)
TILE_DEBUG_TIMING = 1
TILE_DEBUG_ROW_COPIES = 2
TILE_DEBUG_NO_STAGGER = 4

# every symbol include/saturn_b200.h declares (tests check that the library exports them all)
SYMBOLS = [
    "sb_abi_version", "sb_last_error", "sb_create", "sb_destroy", "sb_sync", "sb_set_table",
    "sb_set_sentinel", "sb_set_weights", "sb_set_due", "sb_set_release", "sb_set_penalty", "sb_set_scenarios", "sb_get_reduced", "sb_eval", "sb_last_eval_path", "sb_validate", "sb_eval_host", "sb_eval_full", "sb_eval_scenarios",
    "sb_decode", "sb_xchg_create", "sb_xchg_connect", "sb_xchg_connect_local", "sb_xchg_post", "sb_xchg_reduce", "sb_xchg_check",
    "sb_search_init", "sb_search_round", "sb_search_best_key_ptr", "sb_search_best",
    "sb_search_inject", "sb_search_resample", "sb_search_seed_lpt", "sb_search_run", "sb_search_run_multi", "sb_search_wave", "sb_search_is_fused", "sb_search_stats", "sb_search_validate", "sb_search_verify_count",
    "sb_debug_tile_options", "sb_debug_tile_wait", "sb_debug_search_population",
]


class SearchParams(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("chains", C.c_int64), ("chain_base", C.c_uint64),
                ("flags", C.c_uint), ("t_start", C.c_float), ("t_end", C.c_float),
                ("total_rounds", C.c_int), ("resample_every", C.c_int)]


class SearchControl(C.Structure):
    _fields_ = [("rounds", C.c_int), ("resample_every", C.c_int), ("sync_every", C.c_int), ("patience", C.c_int),
                ("heuristic_seeds", C.c_int), ("target_makespan", C.c_float), ("time_budget_s", C.c_double),
                ("history_cap", C.c_int), ("history_len", C.POINTER(C.c_int)),
                ("history_wall_s", C.POINTER(C.c_double)), ("history_evaluated", C.POINTER(C.c_int64)),
                ("history_makespan", C.POINTER(C.c_float))]


class SearchResultC(C.Structure):
    _fields_ = [("makespan", C.c_float), ("key", C.c_uint64), ("evaluated", C.c_int64), ("rounds", C.c_int),
                ("stop_reason", C.c_int), ("wall_s", C.c_double)]


class SaturnB200Error(RuntimeError):
    pass


_lib = None


def load():
    """Load libsaturn_b200.so (building nothing: run `python -m saturn_b200.build` first)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise SaturnB200Error(
            "%s is missing — build it with `python -m saturn_b200.build` (nvcc, sm_90a). "
            "saturn_b200 has no CPU fallback." % SO_PATH)
    lib = C.CDLL(SO_PATH)
    vp, i64, u32, ci = C.c_void_p, C.c_int64, C.c_uint, C.c_int
    lib.sb_abi_version.restype = ci
    lib.sb_last_error.restype = C.c_char_p
    sigs = {
        "sb_create": [ci, vp, C.POINTER(vp)],
        "sb_destroy": [vp],
        "sb_sync": [vp],
        "sb_set_table": [vp, vp, vp, ci, ci, ci, ci],
        "sb_set_sentinel": [vp, C.c_float],
        "sb_set_weights": [vp, vp, ci],
        "sb_set_due": [vp, vp, ci],
        "sb_set_release": [vp, vp, ci],
        "sb_set_penalty": [vp, vp, ci],
        "sb_set_scenarios": [vp, vp, ci, ci],
        "sb_get_reduced": [vp, vp, vp],
        "sb_eval": [vp, vp, vp, i64, i64, u32, vp, vp, C.c_uint32],
        "sb_last_eval_path": [vp],
        "sb_validate": [vp, vp, vp, i64, i64, u32, C.POINTER(i64)],
        "sb_eval_host": [vp, vp, vp, i64, i64, u32, vp],
        "sb_eval_full": [vp, vp, vp, i64, i64, u32, vp, vp, vp],
        "sb_eval_scenarios": [vp, vp, vp, i64, i64, u32, vp, vp],
        "sb_decode": [vp, vp, vp, u32, vp, vp, vp, vp, vp, vp],
        "sb_xchg_create": [vp, ci, ci, vp],
        "sb_xchg_connect": [vp, vp],
        "sb_xchg_connect_local": [C.POINTER(vp), ci],
        "sb_xchg_post": [vp, vp],
        "sb_xchg_reduce": [vp, vp, vp],
        "sb_xchg_check": [vp],
        "sb_search_init": [vp, C.POINTER(SearchParams), vp, vp],
        "sb_search_round": [vp, ci],
        "sb_search_best_key_ptr": [vp, C.POINTER(vp)],
        "sb_search_best": [vp, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_uint64)],
        "sb_search_inject": [vp, vp, vp, i64, ci],
        "sb_search_resample": [vp],
        "sb_search_seed_lpt": [vp],
        "sb_search_run": [vp, C.POINTER(SearchParams), C.POINTER(SearchControl), vp, vp, vp, vp,
                          C.POINTER(SearchResultC)],
        "sb_search_run_multi": [C.POINTER(vp), ci, C.POINTER(SearchParams), C.POINTER(SearchControl), vp, vp, vp, vp,
                                C.POINTER(SearchResultC)],
        "sb_search_wave": [vp, C.c_uint, C.POINTER(i64)],
        "sb_search_is_fused": [vp],
        "sb_search_stats": [vp, C.POINTER(i64), C.POINTER(i64)],
        "sb_search_validate": [vp, C.POINTER(i64)],
        "sb_search_verify_count": [vp, C.POINTER(C.c_uint64)],
        "sb_debug_tile_options": [vp, C.c_uint],
        "sb_debug_tile_wait": [vp, C.POINTER(C.c_uint64)],
        "sb_debug_search_population": [vp, i64, i64, vp, vp, vp, C.POINTER(ci)],
    }
    for name, args in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = ci
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().sb_last_error()
        raise SaturnB200Error("saturn_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))
