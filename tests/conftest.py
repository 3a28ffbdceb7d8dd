import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import json
    p = os.path.join(ROOT, "tests", "golden", "milp_cases.json")
    with open(p) as f:
        d = json.load(f)
    # round 2: more instances recorded from the unmodified reference (oracle/gen_golden.py --extra, HiGHS run
    # to a zero gap): heterogeneous J = 4..5 and J = 6 — same record layout, so every golden test covers them
    import glob
    for extra in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "milp_cases_extra*.json"))):
        with open(extra) as f:
            d = dict(d, cases=d["cases"] + json.load(f)["cases"])
    return d


@pytest.fixture(scope="session")
def golden_n2():
    import json
    p = os.path.join(ROOT, "tests", "golden", "milp_cases_n2.json")
    with open(p) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def engine():
    import torch
    from saturn_b200.engine import Engine
    torch.cuda.set_device(0)
    e = Engine(0)
    yield e
    e.close()


class DuckTask:
    """The slice of Task the solver path touches (milp.py:77-81, 481-486)."""

    def __init__(self, name, strategies, total_batches=100):
        self.name = name
        self.strategies = strategies
        self.selected_strategy = None
        self.total_batches = total_batches

    def select_strategy(self, s):
        self.selected_strategy = s


def tasks_from_tuples(tuples, executor="exec"):
    from saturn_b200 import Strategy
    out = []
    for t, tup in enumerate(tuples):
        out.append(DuckTask("t%d" % t, {int(g): Strategy(executor, int(g), {}, float(rt)) for g, rt in tup}))
    return out


def build_c_host(out_dir):
    """Compile examples/c_host.c (plain C, -Wall -Werror) against include/saturn_b200.h and link it with the
    in-tree library; returns the binary's path."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    from saturn_b200 import _lib
    libdir = os.path.dirname(_lib.SO_PATH)
    exe = os.path.join(str(out_dir), "c_host")
    subprocess.run(["gcc", "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"),
                    os.path.join(root, "examples", "c_host.c"), "-L", libdir, "-lsaturn_b200",
                    "-Wl,-rpath," + libdir, "-lm", "-o", exe], check=True, capture_output=True)
    return exe
