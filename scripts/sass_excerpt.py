"""SASS evidence for the hot kernels (runs on the build box: cuobjdump only, no GPU).

    python scripts/sass_excerpt.py

For each kernel of interest: instruction count of the fully unrolled 32-step block of the hot loop, the
opcode histogram per scheduling step, and an excerpt of one step; plus the whole-library counts of the
Hopper opcodes the path relies on (UBLKCP = TMA bulk copy, SYNCS = mbarrier, LDG.E.*.128 = 128-bit loads)
and the absence of tensor-core opcodes (the path has no contraction).
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "saturn_b200", "libsaturn_b200.so")


def functions(sass):
    cur, out = None, collections.OrderedDict()
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", line)
        if m and cur:
            out[cur].append(m.group(2).strip())
    return out


def opcode(ins):
    t = ins.split()
    op = t[1] if t[0].startswith("@") else t[0]
    return op.split(".")[0]


def demangle(name):
    try:
        return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
    except OSError:
        return name


def hot_block(ins):
    """The longest run between two branch instructions = the unrolled block of 32 (or 16) scheduling steps."""
    cuts = [i for i, x in enumerate(ins) if opcode(x) in ("BRA", "EXIT", "BSYNC", "BSSY", "WARPSYNC")]
    best = (0, 0)
    prev = -1
    for c in cuts + [len(ins)]:
        if c - prev > best[1] - best[0]:
            best = (prev + 1, c)
        prev = c
    return ins[best[0]:best[1]]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    archs = sorted(set(re.findall(r"arch = (sm_\w+)", sass)))
    fns = functions(sass)
    print("# SASS of saturn_b200/libsaturn_b200.so (cuobjdump -sass; architectures in the fatbin: %s)\n" % ", ".join(archs))
    allins = [x for v in fns.values() for x in v]
    hist = collections.Counter(opcode(x) for x in allins)
    full = collections.Counter()
    for x in allins:
        t = x.split()
        op = t[1] if t[0].startswith("@") else t[0]
        if op.startswith("LDG") and ".128" in op:
            full["LDG.*.128"] += 1
    print("Whole library: %d kernels, %d instructions.  UBLKCP (TMA bulk copy) %d, SYNCS (mbarrier) %d, %s %d, "
          "R2P %d; tensor-core opcodes (HMMA / IMMA / UTCHMMA / UTCQMMA / QGMMA): %d.\n" % (
              len(fns), len(allins), hist["UBLKCP"], hist["SYNCS"], "LDG.*.128", full["LDG.*.128"], hist["R2P"],
              sum(hist[k] for k in hist if k in ("HMMA", "IMMA", "UTCHMMA", "UTCQMMA", "QGMMA", "UTCIMMA", "BMMA"))))
    want = [("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb0ELb0ELi0ELb0EEEvNS_8TileArgsE", "the measured kernel (bench `value`): C4, integer starts, prio streamed, look-up addresses on the FMA pipe", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb0ELi0ELb0EEEvNS_8TileArgsE", "the same kernel scoring the sum of completion times (SB_FLAG_SUM_COMPLETION): one FADD per step instead of half a VIMNMX3", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb1ELi0ELb0EEEvNS_8TileArgsE", "the same kernel scoring the weighted sum of completion times (SB_FLAG_WEIGHTED): one more gather (IMAD + LDS) and one FMUL per step", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb1ELi1ELb0EEEvNS_8TileArgsE", "the same kernel scoring the weighted tardiness (SB_FLAG_DUE): one more gather (IMAD + LDS), one FADD and one FMNMX per step", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb1ELi2ELb0EEEvNS_8TileArgsE", "the same kernel scoring the weighted number of late tasks (SB_FLAG_DUE | SB_FLAG_LATE_COUNT): w * [e > d] as FSET + FMUL, then the FADD, in place of the tardiness' FADD + FMNMX + FMUL + FADD", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb1ELi3ELb0EEEvNS_8TileArgsE", "the same kernel scoring the weighted maximum tardiness (SB_FLAG_DUE | SB_FLAG_MAX_TARDINESS): the product w * (e - d) folded by one VIMNMX, in place of the tardiness' FMNMX + FADD", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb0ELb0ELi0ELb1EEEvNS_8TileArgsE", "the measured kernel with release dates (SB_FLAG_RELEASE): one more gather (IMAD + LDS) and one FMNMX per step", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi1ELb1ELb1ELi1ELb1EEEvNS_8TileArgsE", "the weighted-tardiness kernel with release dates (SB_FLAG_DUE | SB_FLAG_RELEASE)", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb1ELb0ELb0ELb0ELi0ELb0ELb0ELi0ELb0EEEvNS_8TileArgsE", "the same kernel with plain C++ addressing (test hook HOOK_PLAIN_ADDR; the round-1 form)", 32),
            ("_ZN2sb12k_eval_tilesILi1ELb1ELb0ELb0ELb1ELb0ELi0ELb0ELb0ELi0ELb0EEEvNS_8TileArgsE", "fused search round (solve()): rows in shared memory, incremental scoring", 16),
            ("_ZN2sb12k_search_posILi2ELb1ELb0ELb0ELi0ELb0ELb0ELi0ELb0EEEvNS_7PosArgsE", "position-major search round (J > ~450, u16 priorities)", 32),
            ("_ZN2sb13k_eval_groupsILi1ELb1EEEvNS_7AltArgsE", "the alternate shape (SB_FLAG_ALT_WARPSCAN): 8 lanes per candidate, shuffles; the block is the 8 steps of one look-up batch for 4 candidates", 8)]
    for name, what, steps in want:
        if name not in fns:
            print("## %s\n\nnot found in this build\n" % name)
            continue
        ins = fns[name]
        blk = hot_block(ins)
        h = collections.Counter(opcode(x) for x in blk)
        print("## `%s`\n\n%s.  %d instructions in the kernel; the longest branch-free block (the unrolled %d-step body) has "
              "%d instructions = **%.1f per scheduling step**.\n" % (demangle(name), what, len(ins), steps, len(blk), len(blk) / steps))
        print("| opcode | count in the block | per step |\n|---|---|---|")
        for op, n in h.most_common(14):
            print("| %s | %d | %.2f |" % (op, n, n / steps))
        # one step: from a PRMT (byte extraction of the next job id) to the next one, taken mid-block
        prmts = [i for i, x in enumerate(blk) if opcode(x) == "PRMT"]
        if len(prmts) > 6:
            a, b = prmts[len(prmts) // 2], prmts[len(prmts) // 2 + 1]
            print("\nOne step as scheduled by ptxas (instructions of neighbouring steps are interleaved):\n\n```")
            for x in blk[a:b]:
                print("    " + x)
            print("```\n")
    mem = [x for x in fns.get(want[0][0], []) if re.search(r"UBLKCP|SYNCS|LDG\.E\.\S*128|ATOMG|STG|ld\.acquire|LDG\.E\.64\.STRONG\.SYS|ST\.E\S*STRONG\.SYS|STG\.E\S*STRONG\.SYS", x)]
    print("## Memory / synchronisation instructions of the measured kernel (deduplicated)\n\n```")
    seen = set()
    for x in mem:
        k = re.sub(r"R\d+|UR\d+|0x[0-9a-f]+", "_", x)
        if k not in seen:
            seen.add(k)
            print("    " + x)
    print("```")


if __name__ == "__main__":
    main()
