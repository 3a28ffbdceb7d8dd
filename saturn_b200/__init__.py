"""saturn_b200 — Hopper-native (H100, sm_90a) SPASE solver hot path behind Saturn's own solver API.

Public surface (mirrors the reference's module layout, see the `saturn/` alias package):
    saturn_b200.solver.solve / convert_into_comprehensible     <- saturn.solver
    saturn_b200.orchestrator.orchestrate / forecast            <- saturn.orchestrate, saturn.executor.forecast
    saturn_b200.representations.Task / HParams / Strategy / Techniques
    saturn_b200.solver.solve_table / table_from_trials         <- the dense T[J][S][G] entry (SURVEY §8f-3)
    saturn_b200.solver.solve_front                             <- makespan against mean completion time
    saturn_b200.engine.Engine / MultiEngine                    <- ctypes wrapper of include/saturn_b200.h
"""
from .representations import HParams, Strategy, Task, Techniques  # noqa: F401
from .solver import (FrontPoint, convert_into_comprehensible, solve, solve_front, solve_table,  # noqa: F401
                     strategies_from_table, table_from_trials)
from .orchestrator import forecast, orchestrate  # noqa: F401

__all__ = ["HParams", "Strategy", "Task", "Techniques", "solve", "solve_table", "solve_front", "FrontPoint",
           "table_from_trials",
           "strategies_from_table", "convert_into_comprehensible", "orchestrate", "forecast"]
