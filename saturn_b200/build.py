"""In-tree build of libsaturn_b200.so (nvcc, sm_90a only).

    python -m saturn_b200.build [--force]

The shared library is kept next to this file so that it travels with the repository
snapshot to the GPU box; it is git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libsaturn_b200.so")
SOURCES = ["sb_api.cu", "sb_eval.cu", "sb_eval_alt.cu", "sb_table.cu", "sb_search.cu", "sb_xchg.cu"]
HEADERS = ["sb_common.cuh", "sb_lane.cuh", "sb_internal.h", "sb_search.h", os.path.join("..", "..", "include", "saturn_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


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


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    tmp = SO + ".%d.tmp" % os.getpid()      # never leave a half-written library where a snapshot could pick it up
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    try:
        subprocess.check_call(cmd)
        os.replace(tmp, SO)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
