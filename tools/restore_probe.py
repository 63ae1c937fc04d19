"""Cost of pt_batch_restore: full-size c4 with 1 % of its logs checked out at half their change table and each source restored to
its checkout, and a c5 sample (--c5-docs documents) restored the same way.

Every log gets a two-change table (its first half of list ops, then the rest, by actor rank 0), so the version is the first
change and the restore deletes or restores what the second change did.  Per workload it reports:
  - per mode (TEXT, then MARKS after a merge) the call's wall time (host clock around the call, which synchronises): median,
    min and max of --reps, each on a fresh upload, checkout and merge;
  - the count and write kernels' and the splice kernels' device time from a torch.profiler run of its own;
  - the generated ops, and whether after a merge every restored log's visible text equals its version's;
  - the card's name and power limit.
Needs a GPU.

    python tools/restore_probe.py [--reps 3] [--c5-docs 8] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

KERNELS = ("restore_kernel<false>", "restore_kernel<true>", "splice_records_kernel", "splice_changes_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def prepared(e, full, lg):
    """Upload, checkout of logs lg at their first change, merge; returns the restore requests."""
    n0 = full.n_logs
    e.upload(full); e.upload_changes(full.changes)
    assert (e.checkout(lg, n_changes=[1] * len(lg)) == 0).all()
    e.merge(); e.sync()
    return [(s, n0 + k, 0, int(full.desc[s]["max_ctr"]) + 1) for k, s in enumerate(lg)]


def probe(full, lg, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0, emit_sequence=True)
    out = {"n_logs": full.n_logs, "requests": len(lg)}
    try:
        times = {1: [], 2: []}
        n_ops = {}
        for _ in range(reps):
            reqs = prepared(e, full, lg)
            for mode in (1, 2):                                       # TEXT, merge, MARKS (first_ctr above TEXT's ops)
                if mode == 2:
                    e.merge(); e.sync()
                    reqs = [(s, v, a, f + int(k)) for (s, v, a, f), k in zip(reqs, n_ops[1])]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                st, n_ops[mode], _ = e.restore(reqs, mode)
                times[mode].append((time.perf_counter() - t0) * 1e3)
                assert (st == 0).all()
        for mode, name in ((1, "text"), (2, "marks")):
            t = times[mode]
            out[name] = {"call_ms": {"median": float(np.median(t)), "min": min(t), "max": max(t)}, "ops": int(n_ops[mode].sum())}
        e.merge()
        got = e.download()
        n0 = full.n_logs
        out["text_equal"] = bool(all(np.array_equal(got.tokens(s), got.tokens(n0 + k)) for k, s in enumerate(lg)))
        reqs = prepared(e, full, lg)
        for mode, name in ((1, "text"), (2, "marks")):
            if mode == 2:
                e.merge(); e.sync()
                reqs = [(s, v, a, f + int(k)) for (s, v, a, f), k in zip(reqs, n_ops[1])]
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                st, n_ops[mode], _ = e.restore(reqs, mode)
                torch.cuda.synchronize()
            ms = dict.fromkeys(KERNELS, 0.0)
            for ev in prof.events():
                for k in KERNELS:
                    if k in ev.name:
                        ms[k] += (getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)) / 1e3
            out[name]["kernel_ms"] = ms
    finally:
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c5-docs", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from checkout_probe import halves_table
    from peritext_b200 import workload

    out = {"card": card()}
    full = workload.generate("c4")
    full.changes = halves_table(full)
    out["c4"] = probe(full, list(range(0, full.n_logs, 100)), a.reps)
    c5 = workload.generate("c5", n_docs=a.c5_docs)
    c5.changes = halves_table(c5)
    out["c5"] = probe(c5, list(range(c5.n_logs)), a.reps)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
