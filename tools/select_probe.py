"""Cost of pt_batch_select_logs against a re-upload, on full-size c4 and the c5 sample.

Per workload the resident batch is --docs documents (every replica of each); the select retires 1 % of the documents (all
their replicas) and admits as many new ones:
  (a) upload of the resulting batch from pinned host memory + merge + result headers back (the path without select);
  (b) after an untimed upload of the resident batch, select_logs with the admitted logs from pinned memory + merge + result
      headers back.
Both report the wall time of one call sequence (host clock around work that ends in a synchronise), median / min / max of
--reps, and the bytes each copies host -> device.  (b) is also split into the select call alone (it synchronises) and the
merge + result headers after it.  A separate torch.profiler pass, with actor tables attached so that the gather runs too,
gives the device time of the splice and gather kernels; the select call's time outside them is host checks, allocation and
copies.  The result headers (status, counts, 128-bit digest) of (a) and (b) must be equal.  Prints the card name and power
limit.  Needs a GPU.

    python tools/select_probe.py [--docs 100000] [--c5-docs 296] [--reps 5] [--json OUT]
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

from append_probe import pinned_batch, timed  # noqa: E402

KERNELS = ("splice_records_kernel", "splice_changes_kernel", "actor_gather_kernel")


def actor_tables(desc):
    """Made-up actor ids for generated logs (which carry none): log i's ids are a00, a01, ... (n_actors of them, JS order)."""
    from peritext_b200.packing import _ranges
    na = desc["n_actors"].astype(np.int64)
    rank = _ranges(np.zeros(len(na)), na)
    ids = np.frombuffer("".join(f"a{k:02d}" for k in range(100)).encode("utf-16-le"), np.uint8).reshape(100, 6)
    first = np.zeros(len(na) + 1, np.uint64); first[1:] = np.cumsum(na)
    return {"actors": ids[rank].reshape(-1), "actors_off": np.arange(len(rank) + 1, dtype=np.uint64) * 6, "actors_first": first}


def kernel_ms(e, resident, from_, fresh):
    import torch
    from torch.profiler import ProfilerActivity, profile
    e.upload(resident)
    e.upload_actors(actor_tables(resident.desc))
    fresh.log_actors = [[f"a{k:02d}" for k in range(int(n))] for n in fresh.desc["n_actors"]]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        e.select_logs(from_, fresh)
        torch.cuda.synchronize()
    ms = dict.fromkeys(KERNELS, 0.0)
    for ev in prof.events():
        for k in KERNELS:
            if k in ev.name:
                ms[k] += (getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)) / 1e3
    fresh.log_actors = []
    return {k: round(v, 3) for k, v in ms.items()}


def case(name, full, n_docs, reps):
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import SELECT_ADDED, apply_select
    R = int(full.meta["replicas"])
    n_new = max(1, n_docs // 100)
    resident, fresh = full.slice_logs(0, n_docs * R), full.slice_logs(n_docs * R, (n_docs + n_new) * R)
    retired = set(range(0, n_docs, max(1, n_docs // n_new))[:n_new])
    from_ = np.array([d * R + r for d in range(n_docs) if d not in retired for r in range(R)] + [SELECT_ADDED] * fresh.n_logs, np.uint32)
    want = apply_select(resident, from_, fresh)
    pw, k0 = pinned_batch(want)
    pr, k1 = pinned_batch(resident)
    pf, k2 = pinned_batch(fresh)
    e = BatchEngine(0)

    def upload_merge():
        t0 = time.perf_counter()
        e.upload(pw); e.merge(); e.results()
        return (time.perf_counter() - t0) * 1e3

    parts = []

    def select_merge():
        e.upload(pr); e.sync()
        t0 = time.perf_counter()
        e.select_logs(from_, pf)                        # synchronises
        t1 = time.perf_counter()
        e.merge(); e.results()
        t2 = time.perf_counter()
        parts.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3))
        return (t2 - t0) * 1e3

    upload_merge(); ref = e.results()                   # warm-up of every shape
    select_merge(); got = e.results()
    assert got.tobytes() == ref.tobytes(), name
    row = dict(case=name, logs=resident.n_logs, new_logs=want.n_logs, retired_logs=len(retired) * R, added_logs=fresh.n_logs,
               records=int(len(want.insdel) + len(want.marks)),
               upload_h2d_bytes=int(want.desc.nbytes + want.insdel.nbytes + want.marks.nbytes),
               select_h2d_bytes=int(from_.nbytes + 2 * want.desc.nbytes + fresh.insdel.nbytes + fresh.marks.nbytes),
               upload_merge=timed(upload_merge, reps), select_merge=timed(select_merge, reps), digests_equal=True)
    row["select_call_ms"] = round(float(np.median([a for a, _ in parts[1:]])), 3)     # the timed reps only
    row["merge_after_select_ms"] = round(float(np.median([m for _, m in parts[1:]])), 3)
    row["kernel_ms"] = kernel_ms(e, resident, from_, fresh)
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
    for name, cfg, docs in (("c4", "c4", a.docs), ("c5", "c5", a.c5_docs)):
        full = workload.generate(cfg, n_docs=docs + max(1, docs // 100))
        rows.append(case(name, full, docs, a.reps))
        del full
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
