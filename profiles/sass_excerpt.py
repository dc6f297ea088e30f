#!/usr/bin/env python
"""Static SASS summary of the hot kernels (no GPU needed): `python profiles/sass_excerpt.py [LIB]`.
Counts the memory / synchronisation / FP64 mnemonics per kernel from `cuobjdump -sass glomap_b200/libb200sfm.so`, and
for the per-observation kernels of LOOP_KERNELS the instructions of their inner loop (the span between the largest
backward branch and its target): all, FP64 + MUFU, and loads.  For the one-warp-per-segment kernels of SEG_KERNELS it counts the
SHFL and global reduction instructions, all of which sit in the per-segment epilogue."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ["ba3_linearize_points", "ba2_linearize_cams", "ba3_pass_a", "ba2_pass_b", "ba2_schur_diag", "ba3_cost",
           "ba2_pcg_direction_pack", "pcg_update", "pcg_apply_diag", "bax_pass_b", "ba2k_cross", "gp_schur_pass", "ra_laplacian_csr",
           "ra2_laplacian_dot", "ra2_coarse", "p2p_allreduce_sum", "proc_undistort", "trk_hook"]
KEEP = re.compile(r"^(LDG|STG|LDS|STS|RED|ATOM|BAR|SHFL|DFMA|DMUL|DADD|MUFU|CCTL|UBLKCP|SYNCS|MEMBAR|ERRBAR|LDGSTS)")
LOOP_KERNELS = ["ba2_pass_b", "ba2_schur_diag", "ba2_linearize_cams", "ba3_pass_a"]
# one warp per camera-order segment: every SHFL and global reduction of these kernels is in the per-segment epilogue
SEG_KERNELS = ["ba2_pass_b", "ba2_schur_diag", "ba2_linearize_cams", "bax_pass_b", "bax_linearize_blocks"]
SHFL = re.compile(r"^SHFL\b")
RED = re.compile(r"^(RED|REDG|ATOMG?)\.")
FP64 = re.compile(r"^(DFMA|DMUL|DADD|DSETP|DMNMX|MUFU)")
LOADS = re.compile(r"^(LDG|LD|LDS|LDL|LDC)\b")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)([^;]*);")


def inner_loop(insns):
    """(instructions, FP64 + MUFU, loads) between the backward branch spanning the most instructions and its target."""
    best = None
    for addr, op, args in insns:
        m = re.search(r"0x([0-9a-f]+)\s*$", args.strip())
        if op.startswith("BRA") and m and int(m.group(1), 16) < addr:
            body = [(a, o) for a, o, _ in insns if int(m.group(1), 16) <= a <= addr]
            if best is None or len(body) > len(best):
                best = body
    if not best:
        return None
    ops = [o for _, o in best]
    return len(ops), sum(bool(FP64.match(o)) for o in ops), sum(bool(LOADS.match(o)) for o in ops)


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "glomap_b200", "libb200sfm.so")
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", txt)), capture_output=True, text=True).stdout.split("\n")
    mangled = re.findall(r"Function : (\S+)", txt)
    demangle = dict(zip(mangled, names))
    cur, counts, totals = None, collections.defaultdict(collections.Counter), collections.Counter()
    insns = collections.defaultdict(list)
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = demangle.get(m.group(1), m.group(1))
            continue
        m = INSN.search(line)
        if m and cur:
            totals[cur] += 1
            op = m.group(2)
            insns[cur].append((int(m.group(1), 16), op, m.group(3)))
            if KEEP.match(op):
                counts[cur][op] += 1
    print("# SASS mnemonics of the hot kernels (cuobjdump -sass glomap_b200/libb200sfm.so, sm_90a)")
    print("# per kernel: total instructions, then the memory / synchronisation / FP64 mnemonics with their static counts")
    print("# (profiles/sass_excerpt.py regenerates this file; no tensor-core or TMA mnemonics are expected: FP64 streaming kernels)\n")
    for k in sorted(counts):
        if not any(re.search(r"\b" + re.escape(n) + r"\b", k) for n in KERNELS + SEG_KERNELS):
            continue
        ops = ", ".join(f"{o} x{c}" for o, c in counts[k].most_common(14))
        print(k[:200])
        print(f"    total {totals[k]} instructions: {ops}")
        if any(re.search(r"\b" + n + r"\b", k) for n in LOOP_KERNELS):
            loop = inner_loop(insns[k])
            if loop:
                print(f"    inner loop: {loop[0]} instructions, {loop[1]} FP64 + MUFU, {loop[2]} loads")
        if any(re.search(r"\b" + n + r"\b", k) for n in SEG_KERNELS):
            ops = [o for _, o, _ in insns[k]]
            red = collections.Counter(o for o in ops if RED.match(o))
            print(f"    segment epilogue: SHFL x{sum(bool(SHFL.match(o)) for o in ops)}, global reductions "
                  + (", ".join(f"{o} x{c}" for o, c in red.most_common()) or "none"))


if __name__ == "__main__":
    main()
