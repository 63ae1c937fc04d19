"""pt_batch_change at the benchmark shapes: the call time, the time of its kernels, and the merge that follows under a patch window
of the new ops.

  python tools/change_probe.py [--c4-docs N] [--c5-inputs K]

Cases: the c4 shape (default full size, 100 000 documents) with 1 and with 16 InputOperations per document, and one c5 document
with K (default 10 000) InputOperations.  The InputOperations are inserts of one value, deletes of one element and strong /
link marks at spread-out indices, each with its own counter.  Per case: the wall time of the call (it synchronises), the
device time of each kernel it launched (torch.profiler, in a run of its own), and the device time of the merge that follows
with the patch window set to the new ops.  Prints one JSON line per case, with the GPU's name and power limit; needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from peritext_b200 import workload  # noqa: E402
from peritext_b200.engine import BatchEngine  # noqa: E402
from peritext_b200.packing import INPUT_OP_DT  # noqa: E402


def inputs_for(batch, res, per_log, seed=7):
    """per_log InputOperations for every log that merged: one-value inserts, one-element deletes, strong / link marks."""
    rng = np.random.default_rng(seed)
    n = batch.n_logs
    ok = res["status"] == 0
    cnt = np.where(ok, per_log, 0).astype(np.int64)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(cnt)
    total = int(off[-1])
    log = np.repeat(np.arange(n), cnt)
    k = np.arange(total) - np.repeat(off[:-1].astype(np.int64), cnt)
    vis = res["n_visible"].astype(np.int64)[log]
    ops = np.zeros(total, INPUT_OP_DT)
    kind = rng.integers(0, 4, total)
    kind[vis < 4] = 0                                    # an (almost) empty document only gets inserts
    span = np.maximum(vis - 2, 1)
    idx = rng.integers(0, 1 << 30, total) % span
    ops["action"] = np.where(kind < 2, kind, 2)
    ops["mark_type"] = np.where(kind == 3, 3, 0)
    ops["index"] = idx
    ops["arg"] = np.where(kind == 0, 1, np.where(kind == 1, 1, np.minimum(idx + 1 + rng.integers(0, 64, total), vis)))
    ops["attr"] = np.where(kind == 3, 0, 0xFFFFFFFF)
    ops["first_ctr"] = batch.desc["max_ctr"].astype(np.int64)[log] + 1 + k
    ops["tok_off"] = np.arange(total)
    actor = np.where(ok, 0, 0xFFFFFFFF).astype(np.uint32)
    return actor, off, ops, np.full(total, 97, np.uint32)


def call(e, batch, actor, off, ops, tokens):
    t0 = time.perf_counter()
    st, desc, _, _ = e.change_packed(actor, off, ops, tokens, 0, len(batch.link_attrs), 0)
    return time.perf_counter() - t0, desc, st


def case(name, batch, per_log):
    e = BatchEngine(0, emit_patches=True)
    try:
        e.upload(batch); e.merge()
        res = e.results()
        args = inputs_for(batch, res, per_log)
        dt, desc, st = call(e, batch, *args)
        first = (batch.desc["n_insdel"].astype(np.int64) + batch.desc["n_mark"]).astype(np.uint32)
        e.set_patch_window(first)
        e.merge()
        merge_ms = e.last_merge_ms
        # the kernels of the call, in a run of their own under the profiler
        import torch
        from torch.profiler import ProfilerActivity, profile
        e.upload(batch); e.merge(); e.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(e, batch, *args)
        kern = {}
        for ev in prof.key_averages():                    # kernels and copies with their device time
            if getattr(ev, "device_time_total", 0):
                kern[ev.key.split("(")[0][:80]] = round(ev.device_time_total / 1000.0, 3)
        torch.cuda.synchronize()
        return {"case": name, "logs": batch.n_logs, "inputs": int(args[1][-1]), "failed_logs": int((st["status"] != 0).sum()),
                "new_records": int(desc["n_insdel"].sum() + desc["n_mark"].sum()), "call_ms": round(dt * 1000, 3),
                "kernel_ms": kern, "window_merge_ms": round(float(merge_ms), 3)}
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c4-docs", type=int, default=100000)
    ap.add_argument("--c5-inputs", type=int, default=10000)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    c4 = workload.generate("c4", n_docs=a.c4_docs)
    rows = [case("c4 x1", c4, 1), case("c4 x16", c4, 16)]
    del c4
    rows.append(case(f"c5 x{a.c5_inputs}", workload.generate("c5", n_docs=1), a.c5_inputs))
    for r in rows:
        r["gpu"] = gpu
        print(json.dumps(r))


if __name__ == "__main__":
    main()
