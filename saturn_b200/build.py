"""In-tree build of libsaturn_b200.so (nvcc, sm_90a only).

    python -m saturn_b200.build [--force] [-v]

The shared library is kept next to this file so that it travels with the repository
snapshot to the GPU box; it is git-ignored.

Every source is a translation unit of its own (no relocatable device code), so the sources are compiled to objects
side by side, one nvcc per source, and then linked: the same kernels, instruction for instruction, as one nvcc
command over all of them, in the time of the slowest source instead of the sum of them all.  The objects go to a
temporary directory.
"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libsaturn_b200.so")
SOURCES = ["sb_api.cu", "sb_eval.cu", "sb_eval_alt.cu", "sb_table.cu", "sb_search.cu", "sb_xchg.cu"]
HEADERS = ["sb_common.cuh", "sb_lane.cuh", "sb_internal.h", "sb_search.h", os.path.join("..", "..", "include", "saturn_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _run(cmd):
    """Run one compiler command; returns (returncode, its combined output)."""
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return p.returncode, p.stdout


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    nvcc = _nvcc()
    tmp = SO + ".%d.tmp" % os.getpid()      # never leave a half-written library where a snapshot could pick it up
    try:
        with tempfile.TemporaryDirectory(prefix="saturn_b200_build_") as objdir:
            objs = [os.path.join(objdir, os.path.splitext(s)[0] + ".o") for s in SOURCES]
            cmds = [[nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", o, os.path.join(CSRC, s)]
                    for s, o in zip(SOURCES, objs)]
            with ThreadPoolExecutor(max_workers=len(cmds)) as pool:
                results = list(pool.map(_run, cmds))
            for cmd, (rc, out) in zip(cmds, results):
                if out:
                    sys.stdout.write(out)
                if rc:
                    raise subprocess.CalledProcessError(rc, cmd, out)
            subprocess.check_call([nvcc] + ARCH + ["-shared", "-Xcompiler", "-fPIC", "-o", tmp] + objs)
        os.replace(tmp, SO)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
