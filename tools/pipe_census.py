#!/usr/bin/env python3
"""Static pipe census of the warp kernel's loops (no GPU needed).

    python tools/pipe_census.py [lib.so] [--kernel SUBSTR] [--ins 512] [--marks 489]

For every loop of one instantiation of merge_logs_warp_kernel (default <8, packed3>) whose back edge is a conditional branch on
a line of warp_kernel.cuh, prints the SASS instructions of the loop body by the pipe they issue to.  An H100 SM sub-partition
has 16 lanes of the INT32 pipe and 16 of the FMA-heavy pipe that runs IMAD, so a warp instruction on either takes 2 cycles of
its pipe; a scheduler issues one instruction per cycle.  One trip of a loop body therefore costs at least
max(issue, 2 x INT, 2 x IMAD) cycles, and with 32 warps per SM each scheduler serves 8 warps.  For the two streaming passes
(A+B over the ins/del records, G over the mark records, 32 records per trip) the model's cycles per log are

    records / 32 / unroll x max(issue, 2 x INT, 2 x IMAD) x 8

with the defaults at the c4 shape (512 ins/del and 489 mark records per log, from a 900-log sample of workload.generate("c4")).
A pass whose last partial trip is peeled off the loop is charged that trip at the loop's rate.  The counts are static: every
instruction of the body counts once per trip, taken branches or not."""
from __future__ import annotations

import argparse
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sass_dump import sass  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "peritext_b200", "csrc", "warp_kernel.cuh")

INT = {"ISETP", "LOP3", "SHF", "SEL", "IADD3", "LEA", "VIADD", "VIADDMNMX", "VIMNMX", "IMNMX", "POPC", "FLO", "BREV", "PRMT",
       "PLOP3", "IABS", "BMSK", "SGXT", "P2R", "R2P", "ISCADD", "MOV"}
MEM = {"LDS", "STS", "ATOMS", "LDG", "STG", "ATOMG", "RED", "CCTL", "LD", "ST", "LDSM", "LDGSTS"}
CTRL = {"BRA", "BSSY", "BSYNC", "WARPSYNC", "BAR", "YIELD", "EXIT", "CALL", "RET", "BMOV", "BREAK", "JMP"}
SHFL = {"SHFL", "VOTE", "MATCH", "REDUX"}
CLASSES = ["INT", "IMAD", "mem", "ctrl", "shfl/vote", "other"]
# streaming passes: the loop header's source text -> (name, record count option)
PASSES = [(re.compile(r"for \(uint32_t base = .*; base < (n|nFull); base \+= 32\)"), "A+B", "ins"),
          (re.compile(r"for \(uint32_t kb = .*; kb < (m|mFull); kb \+= 32\)"), "G", "marks")]


def pipe_class(text: str) -> str:
    op = re.sub(r"^@!?U?P\w+\s+", "", text).split()[0].split(".")[0]
    if op == "IMAD":
        return "IMAD"
    for name, ops in (("INT", INT), ("mem", MEM), ("ctrl", CTRL), ("shfl/vote", SHFL)):
        if op in ops:
            return name
    return "other"


def loops(lib: str, kernel: str):
    """[(first, last, back-edge source line), ...] over the instruction list, and the list: (address, file:line, text)."""
    ins, labels = [], {}
    for a, line, text in sass(lib, kernel):
        if a is None:
            labels[text.rstrip(":")] = len(ins)
        else:
            ins.append((a, line, text))
    if not ins:
        raise SystemExit(f"no kernel matching {kernel!r} in {lib}")
    out = []
    for i, (_, line, text) in enumerate(ins):
        m = re.match(r"@!?P\w+\s+BRA\s.*?(\.L_x_\d+)", text)
        if m and labels.get(m.group(1), i + 1) <= i and line.startswith("warp_kernel.cu:"):
            out.append((labels[m.group(1)], i, int(line.split(":")[1])))
    return out, ins


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("lib", nargs="?", default=os.path.join(ROOT, "peritext_b200", "libperitext_b200.so"))
    ap.add_argument("--kernel", default="merge_logs_warp_kernelILi8ELi2EE", help="kernel name substring (default <8, packed3>)")
    ap.add_argument("--ins", type=float, default=512, help="ins/del records per log (c4: 512)")
    ap.add_argument("--marks", type=float, default=489, help="mark records per log (c4: 489)")
    ap.add_argument("--warps", type=int, default=8, help="warps per scheduler (32 per SM: 8)")
    ap.add_argument("--src", default=SRC, help="the warp_kernel.cuh the library was built from (default: this tree's)")
    args = ap.parse_args()

    src = open(args.src).read().split("\n")
    found, ins = loops(args.lib, args.kernel)
    print(f"{os.path.basename(args.lib)}  {args.kernel}: {len(ins)} SASS instructions")
    print(f"{'line':>5} {'unroll':>6} {'SASS':>5} " + " ".join(f"{c:>9}" for c in CLASSES) + f" {'cyc/body':>8} {'cyc/log':>8}  header")
    best = {}
    for first, last, line in found:
        counts = dict.fromkeys(CLASSES, 0)
        for _, _, text in ins[first:last + 1]:
            counts[pipe_class(text)] += 1
        total = last - first + 1
        cyc = max(total, 2 * counts["INT"], 2 * counts["IMAD"])
        header = src[line - 1].strip() if 0 < line <= len(src) else ""
        prev = src[line - 2].strip() if 1 < line <= len(src) else ""
        m = re.match(r"#pragma unroll (\d+)", prev)
        unroll = int(m.group(1)) if m else 1
        per_log = ""
        for rx, name, opt in PASSES:
            if rx.search(header):
                v = getattr(args, opt) / 32.0 / unroll * cyc * args.warps
                per_log = f"{v:8.0f}"
                if name not in best or total < best[name][0]:       # the innermost loop of the pass
                    best[name] = (total, v, counts, cyc)
        print(f"{line:>5} {unroll:>6} {total:>5} " + " ".join(f"{counts[c]:>9}" for c in CLASSES) + f" {cyc:>8} {per_log:>8}  {header[:70]}")
    print()
    for name in ("A+B", "G"):
        if name in best:
            total, v, counts, cyc = best[name]
            print(f"{name}: {total} SASS per body ({counts['INT']} INT, {counts['IMAD']} IMAD), {cyc} cycles per body, "
                  f"{v:.0f} cycles per c4 log")


if __name__ == "__main__":
    main()
