"""Host-side wrapper of the C ABI (include/saturn_b200.h) over torch tensors.

PyTorch is used only as plumbing here: device memory (`torch.Tensor.data_ptr()`), the current
CUDA stream, and `torch.distributed` for the per-round MIN all-reduce.  All arithmetic runs in
the hand-written kernels of saturn_b200/csrc.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import FLAG_INTEGER_STARTS, FLAG_REDUCED, SaturnB200Error, SearchParams, check

NSLOT = 8


class Objective(NamedTuple):
    flags: int      # the SB_FLAG_* bits that select it
    weighted: bool  # scores with the weights of set_weights
    due: bool       # scores against the due dates of set_due


# Every objective of the engine.  "tardiness" is the total tardiness against set_due, "max_lateness" the maximum
# lateness scored as L_max + Engine.due_shift, "late_tasks" the number of tasks that complete after their due date,
# "max_tardiness" the largest tardiness, "squared_tardiness" the sum of squared tardiness; each "weighted_" form weighs
# the jobs by set_weights ("weighted_max_tardiness" with weights 1 / p* and due dates at the release dates is the
# maximum stretch; "squared_tardiness" with due dates at the release dates the squared flow time), "late_penalty" the
# fixed penalty of set_penalty plus the (weighted) tardiness of every late task.
_SUM, _W, _DUE = _lib.FLAG_SUM_COMPLETION, _lib.FLAG_WEIGHTED, _lib.FLAG_DUE
_OBJECTIVES = {
    "makespan": Objective(0, False, False),
    "completion": Objective(_SUM, False, False),
    "weighted_completion": Objective(_SUM | _W, True, False),
    "tardiness": Objective(_SUM | _DUE, False, True),
    "weighted_tardiness": Objective(_SUM | _DUE | _W, True, True),
    "max_lateness": Objective(_lib.FLAG_MAX_LATENESS, False, True),
    "late_tasks": Objective(_SUM | _DUE | _lib.FLAG_LATE_COUNT, False, True),
    "weighted_late_tasks": Objective(_SUM | _DUE | _lib.FLAG_LATE_COUNT | _W, True, True),
    "max_tardiness": Objective(_SUM | _DUE | _lib.FLAG_MAX_TARDINESS, False, True),
    "weighted_max_tardiness": Objective(_SUM | _DUE | _lib.FLAG_MAX_TARDINESS | _W, True, True),
    "squared_tardiness": Objective(_SUM | _DUE | _lib.FLAG_SQUARED, False, True),
    "weighted_squared_tardiness": Objective(_SUM | _DUE | _lib.FLAG_SQUARED | _W, True, True),
    "late_penalty": Objective(_SUM | _DUE | _lib.FLAG_LATE_PENALTY, False, True),
    "weighted_late_penalty": Objective(_SUM | _DUE | _lib.FLAG_LATE_PENALTY | _W, True, True),
}
# The squared forms, which the exact reference (oracle/ref_exact.py) and the cross-cutting sweeps of the test suite
# do not fold yet; they are held to their own oracle, oracle/ref_squared_tardiness.py.
SQUARED_OBJECTIVES = ("squared_tardiness", "weighted_squared_tardiness")
# The late-penalty forms, which also read the penalties of set_penalty (objective_reads_penalty); like the squared
# forms they are held to their own oracle, oracle/ref_late_penalty.py, until the cross-cutting sweeps fold them.
PENALTY_OBJECTIVES = ("late_penalty", "weighted_late_penalty")
# The objectives every cross-cutting check of the test suite covers: all of them but the squared and late-penalty forms.
OBJECTIVES = tuple(o for o in _OBJECTIVES if o not in SQUARED_OBJECTIVES + PENALTY_OBJECTIVES)
# The completion-penalty forms: the (weighted) completion time plus the set_penalty penalty of every task that completes
# after its due date (solver.solve_front runs them with one due date, a makespan cap, for every task).  A table of their
# own, held to oracle/ref_completion_penalty.py; objective_spec and objective_flag look names up in both tables.
COMPLETION_PENALTY_OBJECTIVES = {
    "completion_penalty": Objective(_SUM | _DUE | _lib.FLAG_COMPLETION_PENALTY, False, True),
    "weighted_completion_penalty": Objective(_SUM | _DUE | _lib.FLAG_COMPLETION_PENALTY | _W, True, True),
}
# The scenario forms: the worst makespan, max_k M_k, and the mean makespan, scored as sum_k M_k, over the K runtime
# scenarios of set_scenarios (M_k: the same options and order, the list schedule re-run on scenario table k).  A table
# of their own, held to oracle/ref_scenarios.py; objective_spec and objective_flag look names up here as well.
SCENARIO_OBJECTIVES = {
    "worst_makespan": Objective(_lib.FLAG_WORST_MAKESPAN, False, False),
    "mean_makespan": Objective(_lib.FLAG_MEAN_MAKESPAN, False, False),
}
# The tardiness forms over the same scenarios: the worst total (weighted) tardiness, max_k S_k, and the mean, scored as
# sum_k S_k, where S_k is the "tardiness" / "weighted_tardiness" score of the same options and order on scenario table
# k.  Not the per-task maximum tardiness ("max_tardiness").  With every due date 0 they score the worst and the mean
# (weighted) completion time (solver.solve's "worst_completion" and "mean_completion").  A table of their own, held to
# oracle/ref_scenario_tardiness.py; objective_spec and objective_flag look names up here as well.
SCENARIO_TARDINESS_OBJECTIVES = {
    "worst_tardiness": Objective(_SUM | _DUE | _lib.FLAG_WORST_TARDINESS, False, True),
    "weighted_worst_tardiness": Objective(_SUM | _DUE | _lib.FLAG_WORST_TARDINESS | _W, True, True),
    "mean_tardiness": Objective(_SUM | _DUE | _lib.FLAG_MEAN_TARDINESS, False, True),
    "weighted_mean_tardiness": Objective(_SUM | _DUE | _lib.FLAG_MEAN_TARDINESS | _W, True, True),
}


def objective_spec(objective: str) -> Objective:
    """The table entry of an objective name; raises SolverError for a name that is not one."""
    spec = _OBJECTIVES.get(objective) or COMPLETION_PENALTY_OBJECTIVES.get(objective) or \
        SCENARIO_OBJECTIVES.get(objective) or SCENARIO_TARDINESS_OBJECTIVES.get(objective)
    if spec is None:
        from .solver import SolverError
        names = list(_OBJECTIVES) + list(COMPLETION_PENALTY_OBJECTIVES) + list(SCENARIO_OBJECTIVES) + \
            list(SCENARIO_TARDINESS_OBJECTIVES)
        raise SolverError("objective must be one of %s, not %r" % (", ".join(map(repr, names)), objective))
    return spec


def objective_flag(objective: str) -> int:
    """The SB_FLAG_* bits of an objective name (see _OBJECTIVES)."""
    return objective_spec(objective).flags


def objective_reads_penalty(objective: str) -> bool:
    """Whether an objective scores with the late penalties of set_penalty (SB_FLAG_LATE_PENALTY or
    SB_FLAG_COMPLETION_PENALTY)."""
    return bool(objective_spec(objective).flags & (_lib.FLAG_LATE_PENALTY | _lib.FLAG_COMPLETION_PENALTY))


def weights_f32(w, J: int) -> np.ndarray:
    """J job weights as fp32 (round to nearest).  Every weight must be finite and > 0, and stay so in fp32 (a
    value that rounds to 0 or to inf is refused); raises SolverError otherwise."""
    from .solver import SolverError
    try:
        w64 = np.asarray(w, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise SolverError("weights must be numbers: %s" % e)
    if w64.shape != (J,):
        raise SolverError("weights must have one value per task (%d), got shape %s" % (J, w64.shape))
    if not (np.isfinite(w64).all() and (w64 > 0).all()):
        raise SolverError("every weight must be finite and > 0")
    with np.errstate(over="ignore", under="ignore"):
        w32 = w64.astype(np.float32)
    if not (np.isfinite(w32).all() and (w32 > 0).all()):
        raise SolverError("every weight must stay finite and > 0 in fp32 (a weight rounds to 0 or to inf)")
    return w32


def due_f32(d, J: int) -> np.ndarray:
    """J due dates as fp32 (round to nearest: integers are exact).  Every due date must be finite with |d| < 2^24
    (negative values are allowed: the job is already overdue); raises SolverError otherwise."""
    from .solver import SolverError
    try:
        d64 = np.asarray(d, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise SolverError("due dates must be numbers: %s" % e)
    if d64.shape != (J,):
        raise SolverError("due dates must have one value per task (%d), got shape %s" % (J, d64.shape))
    if not (np.isfinite(d64).all() and (np.abs(d64) < 2.0 ** 24).all()):
        raise SolverError("every due date must be finite with |d| < 2^24")
    return d64.astype(np.float32)


def penalty_f32(p, J: int) -> np.ndarray:
    """J late penalties as fp32 (round to nearest: integers below 2^24 are exact), -0 as +0.  Every penalty must be
    finite and >= 0, and J * max p < 2^126 once in fp32 (the fp32 sum of the penalties stays finite); raises
    SolverError otherwise."""
    from .solver import SolverError
    try:
        p64 = np.asarray(p, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise SolverError("penalties must be numbers: %s" % e)
    if p64.shape != (J,):
        raise SolverError("penalties must have one value per task (%d), got shape %s" % (J, p64.shape))
    if not (np.isfinite(p64).all() and (p64 >= 0).all()):
        raise SolverError("every penalty must be finite and >= 0")
    with np.errstate(over="ignore"):
        p32 = p64.astype(np.float32) + np.float32(0)
    if not (np.isfinite(p32).all() and J * float(p32.max(initial=0.0)) < 2.0 ** 126):
        raise SolverError("penalties must keep J * max(penalty) below 2^126 in fp32 (%d tasks, largest penalty %g): "
                          "beyond it the fp32 sum can overflow" % (J, float(p64.max(initial=0.0))))
    return p32


def release_f32(r, J: int) -> np.ndarray:
    """J release dates as fp32, rounded UP (like build_table's runtimes), so that a start >= the fp32 value is
    >= the caller's value in float64 too.  Every release date must be finite with |r| < 2^24, in fp32 as well
    (r <= 0: the job is already released); raises SolverError otherwise."""
    from .solver import SolverError
    try:
        r64 = np.asarray(r, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise SolverError("release dates must be numbers: %s" % e)
    if r64.shape != (J,):
        raise SolverError("release dates must have one value per task (%d), got shape %s" % (J, r64.shape))
    if not (np.isfinite(r64).all() and (np.abs(r64) < 2.0 ** 24).all()):
        raise SolverError("every release date must be finite with |r| < 2^24")
    r32 = r64.astype(np.float32)
    low = r32.astype(np.float64) < r64
    r32[low] = np.nextafter(r32[low], np.float32(np.inf))
    if not (np.abs(r32) < np.float32(2.0 ** 24)).all():
        raise SolverError("every release date must stay below 2^24 in magnitude once rounded up to fp32")
    return r32


def scenarios_f32(f, J: int) -> np.ndarray:
    """K runtime scenarios [K][J] as fp32 (round to nearest), 1 <= K <= 8.  Every factor must be finite and > 0, and
    stay so in fp32; raises SolverError otherwise."""
    from .solver import SolverError
    try:
        f64 = np.asarray(f, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise SolverError("scenario factors must be numbers: %s" % e)
    if f64.ndim != 2 or f64.shape[1] != J or not 1 <= f64.shape[0] <= 8:
        raise SolverError("scenarios must be K x %d factors with 1 <= K <= 8, got shape %s" % (J, f64.shape))
    if not (np.isfinite(f64).all() and (f64 > 0).all()):
        raise SolverError("every scenario factor must be finite and > 0")
    with np.errstate(over="ignore", under="ignore"):
        f32 = f64.astype(np.float32)
    if not (np.isfinite(f32).all() and (f32 > 0).all()):
        raise SolverError("every scenario factor must stay finite and > 0 in fp32 (a factor rounds to 0 or to inf)")
    return f32


def _flags(integer_starts: bool, reduced: bool, objective: str = "makespan") -> int:
    return (FLAG_INTEGER_STARTS if integer_starts else 0) | (FLAG_REDUCED if reduced else 0) | objective_flag(objective)


def _require_due(due, objective: str):
    """The tardiness objectives (the maximum tardiness among them), the late counts and the maximum lateness score
    against the due dates of set_due: refuse them, before any device call, on an engine that has none (set_table
    clears them)."""
    spec = _OBJECTIVES.get(objective) or COMPLETION_PENALTY_OBJECTIVES.get(objective) or \
        SCENARIO_TARDINESS_OBJECTIVES.get(objective)
    if spec is not None and spec.due and due is None:
        from .solver import SolverError
        raise SolverError("objective=%r needs due dates: call set_due after set_table" % (objective,))


def _require_penalty(penalty, objective: str):
    """The late-penalty objectives score with the penalties of set_penalty: refuse them, before any device call, on
    an engine that has none (set_table clears them)."""
    if (objective in _OBJECTIVES or objective in COMPLETION_PENALTY_OBJECTIVES) and objective_reads_penalty(objective) \
            and penalty is None:
        from .solver import SolverError
        raise SolverError("objective=%r needs late penalties: call set_penalty after set_table" % (objective,))


class Engine:
    """One solver handle bound to one CUDA device."""

    def __init__(self, device: int | torch.device | None = None, stream: Optional[torch.cuda.Stream] = None):
        self._h = C.c_void_p()
        lib = _lib.load()
        if not torch.cuda.is_available():
            raise SaturnB200Error("no CUDA device is visible; saturn_b200 has no CPU path")
        if device is None:
            device = torch.cuda.current_device()
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.device = dev
        self._lib = lib
        if stream is None:
            stream = torch.cuda.current_stream(dev)
        self._stream = stream
        sptr = C.c_void_p(stream.cuda_stream) if stream.cuda_stream else None
        check(lib.sb_create(dev.index or 0, sptr, C.byref(self._h)))
        self.J = 0
        self.S = 0
        self.G = 0
        self.gcount = None
        self.nodes = 1
        self.weights = None  # fp32 job weights of objective="weighted_completion" (set_weights)
        self.penalty = None  # fp32 job late penalties of the late-penalty objectives (set_penalty)
        self.due = None  # fp32 job due dates of the tardiness, late-count and max-lateness objectives (set_due)
        self.due_shift = None  # max of self.due: objective="max_lateness" scores L_max + due_shift (>= 0)
        self.release = None  # fp32 job release dates, under every objective (set_release)
        self.scenarios = None  # fp32 runtime factors [K][J] of the scenario objectives (set_scenarios)

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if self._h:
            self._lib.sb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        check(self._lib.sb_sync(self._h))

    # ------------------------------------------------------------------ table
    def set_table(self, T, gcount: Optional[Sequence[int]] = None, sentinel: Optional[float] = None, nodes: int = 1):
        """T[J][S][G] fp32 (numpy array or torch tensor, host or device); gcount[G] GPU counts.
        `sentinel`: cells at/above it are never proposed by the search (default 1e6).
        `nodes` > 1: candidates are evaluated with reduced=True and opt = (node << 3) | (k - 1)."""
        if sentinel is not None:
            check(self._lib.sb_set_sentinel(self._h, C.c_float(sentinel)))
        if isinstance(T, torch.Tensor):
            Tt = T.detach().to(torch.float32).contiguous()
            J, S, G = Tt.shape
            ptr = Tt.data_ptr()
            keep = Tt
        else:
            Ta = np.ascontiguousarray(T, dtype=np.float32)
            J, S, G = Ta.shape
            ptr = Ta.ctypes.data
            keep = Ta
        if gcount is None:
            gcount = list(range(1, G + 1))
        gc = np.ascontiguousarray(gcount, dtype=np.uint8)
        if gc.shape != (G,):
            raise ValueError("gcount must have %d entries" % G)
        check(self._lib.sb_set_table(self._h, C.c_void_p(ptr), C.c_void_p(gc.ctypes.data), J, S, G, int(nodes)))
        del keep
        self.J, self.S, self.G = int(J), int(S), int(G)
        self.gcount = [int(x) for x in gc]
        self.nodes = int(nodes)
        self.weights = None  # sb_set_table clears them
        self.due = None
        self.due_shift = None
        self.release = None
        self.penalty = None
        self.scenarios = None
        return self

    def set_weights(self, w) -> "Engine":
        """Per-job weights (J values, finite and > 0, converted to fp32) for objective="weighted_completion", which
        scores sum_j w_j (start_j + rt_j).  None clears them; set_table clears them too."""
        if w is None:
            check(self._lib.sb_set_weights(self._h, None, 0))
            self.weights = None
            return self
        w32 = np.ascontiguousarray(weights_f32(w, self.J))
        check(self._lib.sb_set_weights(self._h, C.c_void_p(w32.ctypes.data), int(self.J)))
        self.weights = w32
        return self

    def set_due(self, d) -> "Engine":
        """Per-job due dates (J values, finite with |d| < 2^24, converted to fp32) for objective="tardiness", which
        scores sum_j max(0, start_j + rt_j - d_j), and "weighted_tardiness" (each term times the set_weights
        weight), and "max_lateness", which scores max_j (start_j + rt_j + q_j) with the tails q_j = D - d_j (fp32),
        D = due_shift = max_j d_j: that is L_max + D >= 0, and subtracting D gives L_max, and "late_tasks" /
        "weighted_late_tasks", which count (or weigh) the jobs with start_j + rt_j > d_j, and "max_tardiness" /
        "weighted_max_tardiness", which score max_j w_j max(0, start_j + rt_j - d_j), and "squared_tardiness" /
        "weighted_squared_tardiness", which score sum_j w_j max(0, start_j + rt_j - d_j)^2.  None clears them;
        set_table clears them too."""
        if d is None:
            check(self._lib.sb_set_due(self._h, None, 0))
            self.due = None
            self.due_shift = None
            return self
        d32 = np.ascontiguousarray(due_f32(d, self.J))
        check(self._lib.sb_set_due(self._h, C.c_void_p(d32.ctypes.data), int(self.J)))
        self.due = d32
        self.due_shift = float(d32.max())
        return self

    def set_release(self, r) -> "Engine":
        """Per-job release dates (J values, finite with |r| < 2^24, rounded up to fp32) in the runtimes' units from
        the plan's t = 0: no job starts before its release date, under every objective (ceil(r) with integer
        starts).  While they are set, every evaluation and search call of this engine passes SB_FLAG_RELEASE.
        None clears them; set_table clears them too."""
        if r is None:
            check(self._lib.sb_set_release(self._h, None, 0))
            self.release = None
            return self
        r32 = np.ascontiguousarray(release_f32(r, self.J))
        check(self._lib.sb_set_release(self._h, C.c_void_p(r32.ctypes.data), int(self.J)))
        self.release = r32
        return self

    def set_penalty(self, p) -> "Engine":
        """Per-job late penalties (J values, finite and >= 0, converted to fp32) for objective="late_penalty", which
        scores sum_j [C_j > d_j] (p_j + (C_j - d_j)) with C_j = start_j + rt_j against the due dates of set_due, and
        "weighted_late_penalty", which multiplies each tardiness by the set_weights weight, and for
        objective="completion_penalty" / "weighted_completion_penalty", which score sum_j (w_j C_j + [C_j > d_j] p_j).
        None clears them; set_table clears them too."""
        if p is None:
            check(self._lib.sb_set_penalty(self._h, None, 0))
            self.penalty = None
            return self
        p32 = np.ascontiguousarray(penalty_f32(p, self.J))
        check(self._lib.sb_set_penalty(self._h, C.c_void_p(p32.ctypes.data), int(self.J)))
        self.penalty = p32
        return self

    def set_scenarios(self, f) -> "Engine":
        """K runtime scenarios, f[K][J] factors (1 <= K <= 8, each finite and > 0, converted to fp32), for
        objective="worst_makespan", which scores max_k M_k, and "mean_makespan", which scores sum_k M_k: M_k is the
        makespan of the same options and order on the table whose row j is fp32(f[k][j] * T[j]).  The same scenarios
        serve SCENARIO_TARDINESS_OBJECTIVES, which score max_k S_k or sum_k S_k with S_k the (weighted) tardiness total
        on that table.  None clears them; set_table clears them too."""
        if f is None:
            check(self._lib.sb_set_scenarios(self._h, None, 0, 0))
            self.scenarios = None
            return self
        f32 = np.ascontiguousarray(scenarios_f32(f, self.J))
        check(self._lib.sb_set_scenarios(self._h, C.c_void_p(f32.ctypes.data), int(f32.shape[0]), int(self.J)))
        self.scenarios = f32
        return self

    def _release_flag(self) -> int:
        return _lib.FLAG_RELEASE if self.release is not None else 0

    def _flags(self, integer_starts: bool, reduced: bool, objective: str) -> int:
        _require_due(self.due, objective)
        _require_penalty(self.penalty, objective)
        if (objective in SCENARIO_OBJECTIVES or objective in SCENARIO_TARDINESS_OBJECTIVES) and self.scenarios is None:
            from .solver import SolverError
            raise SolverError("objective=%r needs runtime scenarios: call set_scenarios after set_table" % (objective,))
        return _flags(integer_starts, reduced, objective) | self._release_flag()

    def reduced_table(self) -> Tuple[np.ndarray, np.ndarray]:
        tmin = np.empty((self.J, NSLOT), dtype=np.float32)
        args = np.empty((self.J, NSLOT), dtype=np.uint8)
        check(self._lib.sb_get_reduced(self._h, C.c_void_p(tmin.ctypes.data), C.c_void_p(args.ctypes.data)))
        return tmin, args

    @property
    def prio_dtype(self):
        return torch.uint8 if self.J <= 256 else torch.uint16

    # ------------------------------------------------------------------ evaluation
    def _check_cands(self, opt: torch.Tensor, prio: torch.Tensor, on_device: bool):
        if opt.dtype != torch.uint8:
            raise TypeError("opt must be uint8")
        if prio.dtype != self.prio_dtype:
            raise TypeError("prio must be %s for J=%d" % (self.prio_dtype, self.J))
        if opt.dim() != 2 or prio.dim() != 2 or opt.shape != prio.shape:
            raise ValueError("opt / prio must both be [B][J]")
        if opt.shape[1] != self.J:
            raise ValueError("candidates have %d jobs, table has %d" % (opt.shape[1], self.J))
        if opt.stride(1) != 1 or prio.stride(1) != 1 or (opt.shape[0] > 1 and opt.stride(0) != prio.stride(0)):
            raise ValueError("opt / prio rows must be contiguous with the same row stride")
        if on_device and (opt.device != self.device or prio.device != self.device):
            raise ValueError("candidates must live on %s" % self.device)
        if not on_device and (opt.is_cuda or prio.is_cuda):
            raise ValueError("host evaluation takes CPU tensors")
        B = opt.shape[0]
        stride = opt.stride(0) if B > 1 else max(opt.stride(0), self.J)
        return B, stride

    def eval(self, opt: torch.Tensor, prio: torch.Tensor, integer_starts: bool = True, reduced: bool = False,
             out: Optional[torch.Tensor] = None, best_key: Optional[torch.Tensor] = None, id_base: int = 0,
             _force_generic: bool = False, _no_stream: bool = False, post_key: bool = False, fold_prev: bool = False,
             by_position: bool = False, _plain_addr: bool = False, alt_shape: bool = False,
             _table_home: int = 0, _reorder: Optional[bool] = None, objective: str = "makespan",
             _tile_debug: int = 0) -> torch.Tensor:
        """Makespan of every candidate (device tensors).  Asynchronous on the handle's stream.
        objective="completion": the sum of completion times instead (SB_FLAG_SUM_COMPLETION), in `out` and `best_key`.
        by_position: opt[b][i] is the option of the job scheduled i-th (see `opt_by_position`).
        alt_shape: the alternate warp-shuffle kernel (SB_FLAG_ALT_WARPSCAN; a measurement, not a fast path).
        Test hooks: _table_home 2 / 1 puts the position-major kernel's table in a CTA pair's shared memory / in
        global memory whatever its size; _reorder True / False forces / forbids the route that re-orders
        job-indexed opt rows on the device (path 9); _tile_debug: the streamed tile kernel's debug options
        (_lib.TILE_DEBUG_*, sb_debug_tile_options), for this call only."""
        B, stride = self._check_cands(opt, prio, True)
        if out is None:
            out = torch.empty(B, dtype=torch.float32, device=self.device)
        fl = self._flags(integer_starts, reduced, objective) | (_lib.HOOK_FORCE_GENERIC if _force_generic else 0) | (
            _lib.HOOK_NO_STREAM if _no_stream else 0) | (_lib.HOOK_PLAIN_ADDR if _plain_addr else 0) | (
            _lib.FLAG_POST_KEY if post_key else 0) | (
            _lib.FLAG_FOLD_PREV if (post_key and fold_prev) else 0) | (
            _lib.FLAG_OPT_BY_POSITION if by_position else 0) | (_lib.FLAG_ALT_WARPSCAN if alt_shape else 0) | (
            {0: 0, 1: _lib.HOOK_TABLE_GLOBAL, 2: _lib.HOOK_TABLE_PAIR}[_table_home]) | (
            0 if _reorder is None else (_lib.HOOK_REORDER if _reorder else _lib.HOOK_NO_REORDER))
        kp = C.c_void_p(best_key.data_ptr()) if best_key is not None else None
        if _tile_debug:
            check(self._lib.sb_debug_tile_options(self._h, int(_tile_debug)))
        try:
            check(self._lib.sb_eval(self._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), B, stride, fl,
                                    C.c_void_p(out.data_ptr()), kp, id_base & 0xffffffff))
        finally:
            if _tile_debug:
                check(self._lib.sb_debug_tile_options(self._h, 0))
        return out

    def debug_tile_wait(self):
        """(fetch-wait ns, tile-loop ns) summed over the warps of every streamed tile launch since the last call that
        ran with _tile_debug=_lib.TILE_DEBUG_TIMING; resets both (sb_debug_tile_wait)."""
        v = (C.c_uint64 * 2)()
        check(self._lib.sb_debug_tile_wait(self._h, v))
        return int(v[0]), int(v[1])

    def last_eval_path(self) -> int:
        return int(self._lib.sb_last_eval_path(self._h))

    def validate(self, opt: torch.Tensor, prio: torch.Tensor, reduced: bool = False) -> int:
        B, stride = self._check_cands(opt, prio, True)
        bad = C.c_int64(0)
        check(self._lib.sb_validate(self._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), B, stride,
                                    _flags(False, reduced), C.byref(bad)))
        return int(bad.value)

    def eval_host(self, opt: torch.Tensor, prio: torch.Tensor, integer_starts: bool = True, reduced: bool = False,
                  out: Optional[torch.Tensor] = None, objective: str = "makespan") -> torch.Tensor:
        """Same through HOST tensors (pinned for full PCIe speed): H2D + kernel + D2H, synchronous."""
        B, stride = self._check_cands(opt, prio, False)
        if out is None:
            out = torch.empty(B, dtype=torch.float32, pin_memory=True)
        check(self._lib.sb_eval_host(self._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), B, stride,
                                     self._flags(integer_starts, reduced, objective), C.c_void_p(out.data_ptr())))
        return out

    def eval_full(self, opt: torch.Tensor, prio: torch.Tensor, integer_starts: bool = True, reduced: bool = False,
                  objective: str = "makespan"):
        """(makespan[B], start[B][J], slotmask[B][J]) — slot-exact plan of every candidate (the first element is the
        sum of completion times with objective="completion"; starts and masks do not depend on the objective)."""
        B, stride = self._check_cands(opt, prio, True)
        mk = torch.empty(B, dtype=torch.float32, device=self.device)
        start = torch.empty((B, self.J), dtype=torch.float32, device=self.device)
        mask = torch.empty((B, self.J), dtype=torch.int32, device=self.device)
        check(self._lib.sb_eval_full(self._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), B, stride,
                                     self._flags(integer_starts, reduced, objective), C.c_void_p(mk.data_ptr()),
                                     C.c_void_p(start.data_ptr()), C.c_void_p(mask.data_ptr())))
        return mk, start, mask

    def eval_scenarios(self, opt: torch.Tensor, prio: torch.Tensor, integer_starts: bool = True, reduced: bool = False,
                       objective: str = "worst_makespan"):
        """(score[B], per_scenario[B][K]) of every candidate under a scenario objective, slot-exact
        (sb_eval_scenarios): per_scenario holds each scenario's makespan M_k, or under the tardiness forms its total
        (weighted) tardiness S_k."""
        B, stride = self._check_cands(opt, prio, True)
        K = 0 if self.scenarios is None else self.scenarios.shape[0]
        score = torch.empty(B, dtype=torch.float32, device=self.device)
        mks = torch.empty((B, max(K, 1)), dtype=torch.float32, device=self.device)
        check(self._lib.sb_eval_scenarios(self._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), B, stride,
                                          self._flags(integer_starts, reduced, objective),
                                          C.c_void_p(score.data_ptr()), C.c_void_p(mks.data_ptr())))
        return score, mks

    def decode(self, opt: np.ndarray, prio: np.ndarray, integer_starts: bool = True, reduced: bool = False,
               objective: str = "makespan"):
        """One candidate (host arrays) -> dict(start, slotmask, strategy, gpus, makespan); with
        objective="completion" the "makespan" entry holds the sum of completion times."""
        J = self.J
        opt = np.ascontiguousarray(opt, dtype=np.uint8)
        prio = np.ascontiguousarray(prio, dtype=np.uint8 if J <= 256 else np.uint16)
        if opt.shape != (J,) or prio.shape != (J,):
            raise ValueError("opt / prio must have J=%d entries" % J)
        start = np.empty(J, dtype=np.float32)
        mask = np.empty(J, dtype=np.uint32)
        strat = np.empty(J, dtype=np.uint8)
        gpus = np.empty(J, dtype=np.uint8)
        node = np.empty(J, dtype=np.uint8)
        mk = C.c_float(0)
        check(self._lib.sb_decode(self._h, C.c_void_p(opt.ctypes.data), C.c_void_p(prio.ctypes.data),
                                  self._flags(integer_starts, reduced, objective), C.c_void_p(start.ctypes.data),
                                  C.c_void_p(mask.ctypes.data), C.c_void_p(strat.ctypes.data),
                                  C.c_void_p(gpus.ctypes.data), C.c_void_p(node.ctypes.data), C.byref(mk)))
        return {"start": start, "slotmask": mask, "strategy": strat, "gpus": gpus, "node": node,
                "makespan": float(mk.value)}

    # ------------------------------------------------------------------ multi-GPU exchange (NVLink peer memory)
    def xchg_init(self, dist) -> bool:
        """Set up the peer-memory MIN exchange over the ranks of an initialised torch.distributed
        group (one process per GPU of one node).  The 64-byte CUDA IPC handles are all-gathered with
        the group itself; returns False (and leaves the engine on the NCCL path) if a peer mapping
        cannot be opened."""
        rank, world = dist.get_rank(), dist.get_world_size()
        hdl = np.zeros(_lib.IPC_HANDLE_BYTES, dtype=np.uint8)
        # success or failure is decided COLLECTIVELY: a rank whose local step fails still takes part in the
        # all_gather / all_reduce below, so no rank is left waiting in a collective and all ranks end up
        # with the same answer (some posting to mailboxes while others call NCCL would deadlock)
        ok_local = self._lib.sb_xchg_create(self._h, rank, world, C.c_void_p(hdl.ctypes.data)) == 0
        mine = torch.from_numpy(hdl).to(self.device)
        allh = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allh, mine)
        okt = torch.tensor([1 if ok_local else 0], dtype=torch.int32, device=self.device)
        dist.all_reduce(okt, op=dist.ReduceOp.MIN)           # every rank created its mailbox?
        if bool(okt.item()):
            flat = torch.stack(allh).cpu().numpy().copy()
            ok_local = self._lib.sb_xchg_connect(self._h, C.c_void_p(flat.ctypes.data)) == 0
            okt.fill_(1 if ok_local else 0)
            dist.all_reduce(okt, op=dist.ReduceOp.MIN)       # every rank mapped every peer?
        self._xchg = bool(okt.item())
        return self._xchg

    @property
    def has_xchg(self) -> bool:
        return getattr(self, "_xchg", False)

    def xchg_post(self, key: torch.Tensor):
        check(self._lib.sb_xchg_post(self._h, C.c_void_p(key.data_ptr())))

    def xchg_reduce(self, out: torch.Tensor, fold: Optional[torch.Tensor] = None):
        """out[0] = MIN over all ranks of the keys posted this round; `fold` is MIN-ed in place."""
        check(self._lib.sb_xchg_reduce(self._h, C.c_void_p(out.data_ptr()),
                                       C.c_void_p(fold.data_ptr()) if fold is not None else None))

    def xchg_check(self):
        check(self._lib.sb_xchg_check(self._h))

    # ------------------------------------------------------------------ search
    def search_init(self, chains: int, seed: int = 0, chain_base: int = 0, integer_starts: bool = True,
                    reduced: bool = False, t_start: float = 0.02, t_end: float = 1e-4, total_rounds: int = 200,
                    warm: Optional[Tuple[np.ndarray, np.ndarray]] = None, resample_every: int = 0,
                    _no_fused: bool = False, _extra_flags: int = 0, objective: str = "makespan"):
        """resample_every > 0: search_round resamples the population by tournament on that cadence itself.
        objective="completion": minimise the sum of completion times (every score and key holds that sum).
        _extra_flags: test hooks of sb_search_params.flags (_lib.HOOK_*)."""
        p = SearchParams(seed=seed, chains=chains, chain_base=chain_base, resample_every=int(resample_every or 0),
                         flags=self._flags(integer_starts, reduced, objective) | (_lib.HOOK_NO_FUSED if _no_fused else 0) |
                         int(_extra_flags),
                         t_start=t_start, t_end=t_end, total_rounds=total_rounds)
        wo = wp = None
        keep = None
        if warm is not None:
            o = np.ascontiguousarray(warm[0], dtype=np.uint8)
            pr = np.ascontiguousarray(warm[1], dtype=np.uint8 if self.J <= 256 else np.uint16)
            keep = (o, pr)
            wo, wp = C.c_void_p(o.ctypes.data), C.c_void_p(pr.ctypes.data)
        check(self._lib.sb_search_init(self._h, C.byref(p), wo, wp))
        del keep
        self._search_chains = chains
        self._search_base = chain_base

    def search_seed_lpt(self):
        """Plant the three longest-processing-time seeds into an eighth of the population each (shortest-processing-time
        orders when the search minimises the sum of completion times)."""
        check(self._lib.sb_search_seed_lpt(self._h))

    def search_run(self, chains: int, rounds: int, seed: int = 0, chain_base: int = 0, integer_starts: bool = True,
                   reduced: bool = False, t_start: float = 5e-4, t_end: float = 1e-6,
                   warm: Optional[Tuple[np.ndarray, np.ndarray]] = None, resample_every: int = -1, sync_every: int = 16,
                   patience: int = 0, time_budget_s: float = 0.0, target_makespan: float = 0.0,
                   heuristic_seeds: bool = True, record_history: bool = False, _no_fused: bool = False,
                   _extra_flags: int = 0, objective: str = "makespan"):
        """The whole single-GPU search in one C call (sb_search_run).  Returns a dict: opt, prio, makespan, key,
        evaluated, rounds, stop_reason, wall_s, history [(wall s, evaluated, makespan)].  With
        objective="completion" every "makespan" there is the sum of completion times, and target_makespan targets it."""
        _require_due(self.due, objective)
        _require_penalty(self.penalty, objective)
        return _search_run(self._lib, [self._h], self.J, chains, rounds, seed, chain_base, integer_starts, reduced,
                           t_start, t_end, warm, resample_every, sync_every, patience, time_budget_s, target_makespan,
                           heuristic_seeds, record_history, _no_fused, int(_extra_flags) | self._release_flag(),
                           objective)

    def search_wave(self, reduced: bool = False, objective: str = "makespan") -> int:
        """Chains that fill the device exactly once with the round kernel of the current table; populations
        that are whole multiples of it leave no partially filled last wave.  The objective's per-job arrays (weights,
        due dates) and the release dates sit beside the table and can change the round kernel's shape."""
        n = C.c_int64(0)
        check(self._lib.sb_search_wave(self._h, _flags(False, reduced, objective) | self._release_flag(), C.byref(n)))
        return int(n.value)

    def search_is_fused(self) -> bool:
        return bool(self._lib.sb_search_is_fused(self._h))

    def search_round(self, rounds: int = 1):
        check(self._lib.sb_search_round(self._h, rounds))

    def search_best_key(self) -> torch.Tensor:
        """A 1-element int64 tensor aliasing the device-resident best key (makespan bits << 32 | id)."""
        ptr = C.c_void_p()
        check(self._lib.sb_search_best_key_ptr(self._h, C.byref(ptr)))
        return _alias_int64(ptr.value, self.device)

    def search_best(self):
        J = self.J
        opt = np.empty(J, dtype=np.uint8)
        prio = np.empty(J, dtype=np.uint8 if J <= 256 else np.uint16)
        mk = C.c_float(0)
        key = C.c_uint64(0)
        check(self._lib.sb_search_best(self._h, C.c_void_p(opt.ctypes.data), C.c_void_p(prio.ctypes.data),
                                       C.byref(mk), C.byref(key)))
        return opt, prio, float(mk.value), int(key.value)

    def search_inject(self, opt: np.ndarray, prio: np.ndarray, copies: int = 1, first: int = -1):
        o = np.ascontiguousarray(opt, dtype=np.uint8)
        p = np.ascontiguousarray(prio, dtype=np.uint8 if self.J <= 256 else np.uint16)
        check(self._lib.sb_search_inject(self._h, C.c_void_p(o.ctypes.data), C.c_void_p(p.ctypes.data), first,
                                         copies))

    def search_resample(self):
        check(self._lib.sb_search_resample(self._h))

    def search_verify_count(self) -> int:
        """Incremental scores that differed from a from-scratch score (test hook: needs
        _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL)."""
        n = C.c_uint64(0)
        check(self._lib.sb_search_verify_count(self._h, C.byref(n)))
        return int(n.value)

    def search_validate(self) -> int:
        """Chains of the current population whose rows are not a permutation + existing table cells."""
        bad = C.c_int64(0)
        check(self._lib.sb_search_validate(self._h, C.byref(bad)))
        return int(bad.value)

    def debug_search_population(self, first: int = 0, count: Optional[int] = None):
        """Chains [first, first + count) of the search population (all from `first` when count is None):
        (opt [count][J] u8 job-indexed, prio [count][J] u8/u16, score [count] fp32, layout), layout 0 for
        propose / evaluate / accept rounds, 1 for the fused tile round, 2 for the position-major round."""
        if count is None:
            count = self._search_chains - first
        J = self.J
        opt = np.empty((count, J), dtype=np.uint8)
        prio = np.empty((count, J), dtype=np.uint8 if J <= 256 else np.uint16)
        score = np.empty(count, dtype=np.float32)
        layout = C.c_int(-1)
        check(self._lib.sb_debug_search_population(self._h, int(first), int(count), C.c_void_p(opt.ctypes.data),
                                                   C.c_void_p(prio.ctypes.data), C.c_void_p(score.ctypes.data),
                                                   C.byref(layout)))
        return opt, prio, score, int(layout.value)

    def search_stats(self):
        ev, rd = C.c_int64(0), C.c_int64(0)
        check(self._lib.sb_search_stats(self._h, C.byref(ev), C.byref(rd)))
        return int(ev.value), int(rd.value)


def _search_run(lib, handles, J, chains, rounds, seed, chain_base, integer_starts, reduced, t_start, t_end, warm,
                resample_every, sync_every, patience, time_budget_s, target_makespan, heuristic_seeds,
                record_history, _no_fused, _extra_flags=0, objective="makespan"):
    """sb_search_run (one handle) / sb_search_run_multi (one handle per device of this process)."""
    pdt = np.uint8 if J <= 256 else np.uint16
    p = SearchParams(seed=seed, chains=chains, chain_base=chain_base,
                     flags=_flags(integer_starts, reduced, objective) | (_lib.HOOK_NO_FUSED if _no_fused else 0) |
                     int(_extra_flags),
                     t_start=t_start, t_end=t_end, total_rounds=max(rounds, 1))
    cap = (max(rounds, 1) // max(1, sync_every) + 3) if record_history else 0
    hw, he, hm = np.zeros(cap, np.float64), np.zeros(cap, np.int64), np.zeros(cap, np.float32)
    hl = C.c_int(0)
    ctl = _lib.SearchControl(rounds=max(rounds, 1), resample_every=int(resample_every), sync_every=max(1, int(sync_every)),
                             patience=int(patience or 0), heuristic_seeds=1 if heuristic_seeds else 0,
                             target_makespan=float(target_makespan or 0.0), time_budget_s=float(time_budget_s or 0.0),
                             history_cap=cap, history_len=C.pointer(hl),
                             history_wall_s=hw.ctypes.data_as(C.POINTER(C.c_double)),
                             history_evaluated=he.ctypes.data_as(C.POINTER(C.c_int64)),
                             history_makespan=hm.ctypes.data_as(C.POINTER(C.c_float)))
    wo = wp = None
    keep = None
    if warm is not None:
        keep = (np.ascontiguousarray(warm[0], dtype=np.uint8), np.ascontiguousarray(warm[1], dtype=pdt))
        wo, wp = C.c_void_p(keep[0].ctypes.data), C.c_void_p(keep[1].ctypes.data)
    opt, prio = np.empty(J, dtype=np.uint8), np.empty(J, dtype=pdt)
    res = _lib.SearchResultC()
    if len(handles) == 1:
        check(lib.sb_search_run(handles[0], C.byref(p), C.byref(ctl), wo, wp, C.c_void_p(opt.ctypes.data),
                                C.c_void_p(prio.ctypes.data), C.byref(res)))
    else:
        arr = (C.c_void_p * len(handles))(*[h.value for h in handles])
        check(lib.sb_search_run_multi(arr, len(handles), C.byref(p), C.byref(ctl), wo, wp,
                                      C.c_void_p(opt.ctypes.data), C.c_void_p(prio.ctypes.data), C.byref(res)))
    del keep
    n = int(hl.value)
    return {"opt": opt, "prio": prio, "makespan": float(res.makespan), "key": int(res.key),
            "evaluated": int(res.evaluated), "rounds": int(res.rounds), "stop_reason": int(res.stop_reason),
            "wall_s": float(res.wall_s), "history": [(float(hw[i]), int(he[i]), float(hm[i])) for i in range(n)]}


class MultiEngine:
    """N handles on N devices of THIS process behind the interface `saturn.solver.solve` uses: the table is
    replicated, the search population is sharded by global chain id (sb_search_run_multi: one MIN of a uint64
    per group of rounds over NVLink peer memory, no torchrun, no NCCL), the winner is decoded on the first
    device.  The reference calls its solver from one process (saturn/orchestrator.py:21-23,55,69); this is how
    that call site reaches every GPU of the node."""

    def __init__(self, devices):
        if isinstance(devices, int):
            devices = list(range(devices))
        devices = [int(d) for d in devices]
        if len(devices) < 1:
            raise ValueError("need at least one device")
        if len(set(devices)) != len(devices):
            raise ValueError("devices must be distinct")
        self.engines = [Engine(d, stream=torch.cuda.current_stream(torch.device("cuda", d))) for d in devices]
        self._lib = self.engines[0]._lib
        self.device = self.engines[0].device
        self.devices = devices
        self._pool = None

    def close(self):
        if self._pool is not None:
            self._pool.shutdown()
            self._pool = None
        for e in self.engines:
            e.close()

    def set_table(self, T, gcount=None, sentinel=None, nodes: int = 1):
        # one host thread per device: sb_set_table synchronises its stream (ctypes releases the GIL in the call)
        if self._pool is None:
            from concurrent.futures import ThreadPoolExecutor
            self._pool = ThreadPoolExecutor(max_workers=len(self.engines))
        list(self._pool.map(lambda e: e.set_table(T, gcount, sentinel=sentinel, nodes=nodes), self.engines))
        return self

    J = property(lambda self: self.engines[0].J)
    S = property(lambda self: self.engines[0].S)
    G = property(lambda self: self.engines[0].G)
    gcount = property(lambda self: self.engines[0].gcount)
    nodes = property(lambda self: self.engines[0].nodes)
    prio_dtype = property(lambda self: self.engines[0].prio_dtype)

    def reduced_table(self):
        return self.engines[0].reduced_table()

    def set_weights(self, w):
        """Engine.set_weights on every device."""
        for e in self.engines:
            e.set_weights(w)
        return self

    weights = property(lambda self: self.engines[0].weights)

    def set_due(self, d):
        """Engine.set_due on every device."""
        for e in self.engines:
            e.set_due(d)
        return self

    due = property(lambda self: self.engines[0].due)
    due_shift = property(lambda self: self.engines[0].due_shift)

    def set_release(self, r):
        """Engine.set_release on every device."""
        for e in self.engines:
            e.set_release(r)
        return self

    release = property(lambda self: self.engines[0].release)

    def set_scenarios(self, f):
        """Engine.set_scenarios on every device."""
        for e in self.engines:
            e.set_scenarios(f)
        return self

    scenarios = property(lambda self: self.engines[0].scenarios)

    def set_penalty(self, p):
        """Engine.set_penalty on every device."""
        for e in self.engines:
            e.set_penalty(p)
        return self

    penalty = property(lambda self: self.engines[0].penalty)

    def decode(self, *a, **kw):
        return self.engines[0].decode(*a, **kw)

    def search_wave(self, reduced: bool = False, objective: str = "makespan") -> int:
        """chains PER DEVICE that fill one device exactly once."""
        return self.engines[0].search_wave(reduced, objective)

    def search_run(self, chains: int, rounds: int, seed: int = 0, chain_base: int = 0, integer_starts: bool = True,
                   reduced: bool = False, t_start: float = 5e-4, t_end: float = 1e-6, warm=None,
                   resample_every: int = -1, sync_every: int = 16, patience: int = 0, time_budget_s: float = 0.0,
                   target_makespan: float = 0.0, heuristic_seeds: bool = True, record_history: bool = False,
                   _no_fused: bool = False, _extra_flags: int = 0, objective: str = "makespan"):
        """`chains` is per device; the result's `evaluated` counts every device."""
        _require_due(self.due, objective)
        _require_penalty(self.penalty, objective)
        return _search_run(self._lib, [e._h for e in self.engines], self.J, chains, rounds, seed, chain_base,
                           integer_starts, reduced, t_start, t_end, warm, resample_every, sync_every, patience,
                           time_budget_s, target_makespan, heuristic_seeds, record_history, _no_fused,
                           int(_extra_flags) | self.engines[0]._release_flag(), objective)


class _CudaArrayView:
    """Minimal __cuda_array_interface__ carrier so torch can alias library-owned device memory."""

    def __init__(self, ptr, nbytes, typestr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2,
                                         "strides": None}
        self._nbytes = nbytes


def _alias_int64(ptr: int, device: torch.device) -> torch.Tensor:
    with torch.cuda.device(device):
        return torch.as_tensor(_CudaArrayView(ptr, 8, "<i8", (1,)), device=device)


# ---------------------------------------------------------------------- candidate helpers
def opt_by_position(opt: torch.Tensor, prio: torch.Tensor) -> torch.Tensor:
    """Re-encode job-indexed opt rows in schedule order (opt'[b][i] = opt[b][prio[b][i]]), keeping the row
    stride of `opt` — the encoding SB_FLAG_OPT_BY_POSITION evaluates."""
    B, J = opt.shape
    out = padded_rows(B, J, torch.uint8, opt.device)
    out.copy_(torch.gather(opt, 1, prio.to(torch.int32).to(torch.int64)))
    return out


def padded_rows(B: int, J: int, dtype: torch.dtype, device, pinned: bool = False) -> torch.Tensor:
    """A [B][J] view into storage whose rows are a multiple of 32 ELEMENTS apart, so that the byte
    stride of both opt (u8) and prio (u8/u16) rows is 32-byte aligned (the kernel's fast path)."""
    stride = (J + 31) // 32 * 32
    if pinned:
        buf = torch.zeros((B, stride), dtype=dtype, pin_memory=True)
    else:
        buf = torch.zeros((B, stride), dtype=dtype, device=device)
    return buf[:, :J]


def random_candidates(engine: Engine, B: int, valid: np.ndarray, seed: int = 0, gcount=None, device=None,
                      pinned: bool = False, nodes: int = 1):
    """opt ~ U{valid cells of each job}, prio = random permutations (torch RNG on `device`).
    nodes > 1: `valid` must describe the reduced table (S = 1); a uniform node index is OR-ed into
    bits 3.. of every opt byte."""
    J = engine.J
    device = engine.device if device is None else torch.device(device)
    gen_dev = device if device.type == "cuda" else torch.device("cpu")
    g = torch.Generator(device=gen_dev)
    g.manual_seed(seed)
    _, S, G = valid.shape
    gcount = engine.gcount if gcount is None else list(gcount)
    opt = padded_rows(B, J, torch.uint8, device, pinned)
    prio = padded_rows(B, J, engine.prio_dtype, device, pinned)
    nmax = int(valid.reshape(J, -1).sum(axis=1).max())
    cells = np.zeros((J, nmax), dtype=np.uint8)
    ncell = np.zeros(J, dtype=np.int64)
    for j in range(J):
        c = [(s << 3) | (gcount[gi] - 1) for s in range(S) for gi in range(G) if valid[j, s, gi]]
        cells[j, :len(c)] = c
        ncell[j] = len(c)
    cells_t = torch.from_numpy(cells).to(gen_dev)
    ncell_t = torch.from_numpy(ncell).to(gen_dev)
    chunk = max(1, min(B, (1 << 24) // max(J, 1)))
    for b0 in range(0, B, chunk):
        nb = min(chunk, B - b0)
        u = torch.rand((nb, J), generator=g, device=gen_dev)
        pick = torch.minimum((u * ncell_t[None, :]).long(), ncell_t[None, :] - 1)
        o = torch.gather(cells_t[None, :, :].expand(nb, -1, -1), 2, pick[:, :, None])[:, :, 0]
        keys = torch.rand((nb, J), generator=g, device=gen_dev)
        p = torch.argsort(keys, dim=1)
        if nodes > 1:
            nd = torch.randint(0, nodes, (nb, J), generator=g, device=gen_dev, dtype=torch.uint8)
            o = o | (nd << 3)
        opt[b0:b0 + nb].copy_(o)
        if engine.prio_dtype == torch.uint8:
            prio[b0:b0 + nb].copy_(p.to(torch.uint8))
        else:
            prio[b0:b0 + nb].copy_(p.to(torch.int32).to(torch.uint16))
    return opt, prio
