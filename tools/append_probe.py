"""Cost of pt_batch_append against a full re-upload, on full-size c4 and the c5 sample.

Per workload:
  (a) upload of the whole batch from pinned host memory + merge + result headers back (the path every re-merge takes
      without append);
  (b) after an untimed upload of each log's first 99 % of ins/del records (and the marks that arrived before them), append
      of the last 1 % from pinned memory + merge + result headers back.
Both report the wall time of one call sequence (host clock around work that ends in a synchronise), median / min / max of
--reps, and the bytes each copies host -> device.  A separate torch.profiler pass gives the splice kernels' device time.
(b) is also split into the append call alone (it synchronises) and the merge + result headers after it.  The result headers
(status, counts, 128-bit digest) of (a) and (b) must be equal.  Prints the card name and power limit.
Needs a GPU.

    python tools/append_probe.py [--docs 100000] [--c5-docs 296] [--reps 5] [--json OUT]
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


def pinned(a):
    import torch
    t = torch.empty(max(1, a.nbytes), dtype=torch.uint8).pin_memory()
    out = t.numpy()[: a.nbytes].view(a.dtype)
    out[...] = a
    return out, t


def pinned_batch(b):
    from peritext_b200.packing import PackedBatch
    ins, k1 = pinned(b.insdel)
    mk, k2 = pinned(b.marks)
    return PackedBatch(b.desc, ins, mk), (k1, k2)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        ts.append(fn())
    return dict(ms=round(float(np.median(ts)), 3), ms_min=round(min(ts), 3), ms_max=round(max(ts), 3))


def splice_kernel_ms(e, prefix, delta):
    import torch
    from torch.profiler import ProfilerActivity, profile
    e.upload(prefix)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        e.append(delta)
        torch.cuda.synchronize()
    ms = 0.0
    for ev in prof.events():
        if "splice_records_kernel" in ev.name or "splice_changes_kernel" in ev.name:
            ms += (getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)) / 1e3
    return round(ms, 3)


def case(name, full, reps):
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import split_records
    n_ins = full.desc["n_insdel"].astype(np.int64)
    prefix, delta = split_records(full, (n_ins * 99) // 100)
    pf, k0 = pinned_batch(full)
    pp, k1 = pinned_batch(prefix)
    pd, k2 = pinned_batch(delta)
    e = BatchEngine(0)

    def upload_merge():
        t0 = time.perf_counter()
        e.upload(pf); e.merge(); e.results()
        return (time.perf_counter() - t0) * 1e3

    parts = []

    def append_merge():
        e.upload(pp); e.sync()
        t0 = time.perf_counter()
        e.append(pd)                                    # synchronises
        t1 = time.perf_counter()
        e.merge(); e.results()
        t2 = time.perf_counter()
        parts.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3))
        return (t2 - t0) * 1e3

    upload_merge(); want = e.results()                  # warm-up of every shape
    append_merge(); got = e.results()
    assert got.tobytes() == want.tobytes(), name
    row = dict(case=name, logs=full.n_logs, records=int(len(full.insdel) + len(full.marks)),
               delta_records=int(len(delta.insdel) + len(delta.marks)),
               upload_h2d_bytes=int(full.desc.nbytes + full.insdel.nbytes + full.marks.nbytes),
               append_h2d_bytes=int(2 * delta.desc.nbytes + delta.insdel.nbytes + delta.marks.nbytes),
               upload_merge=timed(upload_merge, reps), append_merge=timed(append_merge, reps),
               splice_kernel_ms=splice_kernel_ms(e, pp, pd), digests_equal=True)
    row["append_call_ms"] = round(float(np.median([a for a, _ in parts[1:]])), 3)     # the timed reps only
    row["merge_after_append_ms"] = round(float(np.median([m for _, m in parts[1:]])), 3)
    e.close()
    del k0, k1, k2
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=100000, help="c4 documents (3 logs each)")
    ap.add_argument("--c5-docs", type=int, default=296, help="c5 documents (2 logs each)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="also write the rows to this file")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    rows = []
    for name, make in (("c4", lambda: workload.generate("c4", n_docs=a.docs)), ("c5", lambda: workload.generate("c5", n_docs=a.c5_docs))):
        full = make()
        rows.append(case(name, full, a.reps))
        del full
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
