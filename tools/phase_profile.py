#!/usr/bin/env python3
"""Per-phase cycle profile of the warp kernel (the c4 path); needs a GPU.

    python tools/phase_profile.py [--docs 100000] [--warmup 3] [--steps 5] [--lib PATH]

Builds the engine with `make PHASE_CLOCKS=1` into a temporary directory (the tree is not written), merges the c4 batch
`--warmup` times, then `--steps` more times with the counters reset, and prints the mean cycles per log of each phase,
summed over the warps that merged the logs.  The instrumented build is slower than the default one (a clock64 read and an
add per phase boundary); read the table for where the time of a log goes, and time the default build with bench.py."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["log start", "A+B records", "C runs", "D run tree", "E ranking", "F text", "G marks", "I spans", "round wait"]


def build_instrumented(out_dir: str) -> str:
    lib = os.path.join(out_dir, "libperitext_b200.so")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "peritext_b200", "csrc"), "-s", "PHASE_CLOCKS=1", f"OUT={lib}", lib])
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=0, help="c4 documents (default: the config's 100 000)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--lib", help="an already instrumented library (default: build one)")
    args = ap.parse_args()

    from peritext_b200 import engine, workload
    tmp = tempfile.mkdtemp(prefix="pt_phase_")
    engine.LIB_PATH = args.lib or build_instrumented(tmp)
    L = engine.load_library()
    if not hasattr(L, "pt_phase_clocks"):
        raise SystemExit(f"{engine.LIB_PATH} was not built with PHASE_CLOCKS=1")
    out = (ctypes.c_uint64 * (len(PHASES) + 1))()
    L.pt_phase_clocks.argtypes = [ctypes.c_void_p, ctypes.c_int]

    batch = workload.generate("c4", n_docs=args.docs or None, threads=os.cpu_count() or 8)
    eng = engine.BatchEngine(0)
    eng.upload(batch)
    for _ in range(args.warmup):
        eng.merge(); eng.sync()
    engine._check(L.pt_phase_clocks(out, 1), "pt_phase_clocks")
    for _ in range(args.steps):
        eng.merge(); eng.sync()
    engine._check(L.pt_phase_clocks(out, 0), "pt_phase_clocks")
    eng.close()

    logs = out[len(PHASES)]
    if not logs:
        raise SystemExit("no log went through the warp kernel")
    per_log = [out[k] / logs for k in range(len(PHASES))]
    total = sum(per_log)
    print(f"c4, {batch.n_logs} logs x {args.steps} merges: {logs} warp-kernel logs, cycles per log (per warp)")
    for name, c in zip(PHASES, per_log):
        print(f"  {name:<12} {c:10.0f}  {100 * c / total:5.1f} %")
    print(f"  {'total':<12} {total:10.0f}")
    print(json.dumps({"logs": logs, "cycles_per_log": dict(zip(PHASES, [round(c, 1) for c in per_log]))}))


if __name__ == "__main__":
    main()
