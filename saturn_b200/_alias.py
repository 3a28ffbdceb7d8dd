"""Fall-through for the `saturn` import-path alias.

The alias package `saturn/` of this repository implements ONE path of the reference — the solver and the
interval loop that calls it (`saturn.orchestrate`, `saturn.solver`, `saturn.core.representations`,
`saturn.executor.forecast`).  Everything else of the reference's package (`saturn.library`,
`saturn.trial_runner`, `saturn.core.executors`, `saturn.executor.execute`, `saturn.utilities`) is out of
scope here (SURVEY.md §8).  So that shadowing the name `saturn` does not break those imports where the
reference distribution IS installed, every alias package appends the same-named directories of any other
`saturn` distribution on sys.path to its `__path__` (submodules this repository does not provide resolve
there), and names it does not define are looked up lazily in the reference's module of the same role.
Without an installed reference they raise ImportError naming what is missing.
"""
import importlib.util
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def other_package_dirs(pkg_name):
    """Directories of packages named `pkg_name` that belong to another distribution on sys.path."""
    rel = pkg_name.split(".")
    out = []
    for p in sys.path:
        base = os.path.abspath(p or ".")
        if base == _ROOT:
            continue
        d = os.path.join(base, *rel)
        if os.path.isfile(os.path.join(d, "__init__.py")) and d not in out:
            out.append(d)
    return out


def fall_through(pkg_name, pkg_path):
    """The alias package's own __path__ followed by the reference's, if one is installed."""
    path = list(pkg_path)
    for d in other_package_dirs(pkg_name):
        if d not in path:
            path.append(d)
    return path


def reference_attr(pkg_name, module_file, attr):
    """Load `<reference>/<pkg dir>/<module_file>` under a private name and return `attr` from it."""
    for d in other_package_dirs(pkg_name):
        f = os.path.join(d, module_file)
        if os.path.isfile(f):
            name = "_saturn_reference_." + pkg_name + "." + module_file[:-3]
            mod = sys.modules.get(name)
            if mod is None:
                spec = importlib.util.spec_from_file_location(name, f)
                mod = importlib.util.module_from_spec(spec)
                sys.modules[name] = mod
                try:
                    spec.loader.exec_module(mod)
                except Exception:
                    del sys.modules[name]
                    raise
            return getattr(mod, attr)
    raise ImportError(
        "%s.%s is not part of the saturn_b200 solver drop-in (it implements saturn.solver, saturn.orchestrate, "
        "saturn.core.representations and saturn.executor.forecast only) and no reference `saturn` "
        "distribution was found on sys.path to fall through to" % (pkg_name, attr))
