"""Import-path alias: `import saturn` resolves to the H100-native implementation in saturn_b200.

Keeps the reference's entry points (saturn/__init__.py:1, saturn/solver/__init__.py:1-2,
saturn/core/representations/__init__.py:1-2) importable without PuLP, Ray or Gurobi.  Submodules
this repository does not implement (saturn.library, saturn.trial_runner, saturn.core.executors,
saturn.utilities) fall through to an installed reference distribution, see saturn_b200/_alias.py.
"""
from saturn_b200._alias import fall_through as _fall_through

__path__ = _fall_through(__name__, __path__)

from saturn_b200.orchestrator import orchestrate  # noqa: E402,F401
