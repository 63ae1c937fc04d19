"""Cost of pt_batch_find_elements (batched findListElement / resolveCursor) on merged documents.

Merges full-size c4 (100 000 documents x 3 replicas) with the element sequence enabled, then times the call for 1 and for 16
random existing elements per log (300 K and 4.8 M queries), and one c5 log (~111 K records) with 10 K queries.  Per case it
prints the wall time of one call (host clock around a call that synchronises: H2D copy of the refs, the kernel, D2H copy of
the answers) as the median of --reps calls, the queries per second that gives, and the kernel's own device time from a
separate torch.profiler pass.  Needs a GPU.

    python tools/find_elements_probe.py [--docs 100000] [--reps 10] [--json OUT]
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


def random_refs(batch, merged, logs, per_log, rng):
    """`per_log` random elements (tombstones included) of each log in `logs`, as packed (log, ctr, actor)."""
    logs = np.repeat(np.asarray(logs, np.int64), per_log)
    n_el = merged.results["n_elems"][logs].astype(np.int64)
    pos = (rng.random(len(logs)) * n_el).astype(np.int64)
    rec = merged.seq[merged.seq_off[logs].astype(np.int64) + pos].astype(np.int64) & 0x3FFFFFFF
    ins = batch.insdel[batch.desc["insdel_off"][logs].astype(np.int64) + rec]
    return logs.astype(np.uint32), np.ascontiguousarray(ins["ctr"]), np.ascontiguousarray(ins["actor"])


def kernel_ms(engine, q):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine.find_elements(*q)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "find_elements_kernel" in ev.key:
            return getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3
    return float("nan")


def time_case(engine, name, q, reps):
    got = engine.find_elements(*q)                   # warm-up (module load, first allocation)
    assert (got["index"] != 0xFFFFFFFF).all(), name   # every query names an existing element
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        engine.find_elements(*q)
        ts.append((time.perf_counter() - t0) * 1e3)
    ms = float(np.median(ts))
    kms = kernel_ms(engine, q)
    row = dict(case=name, queries=len(q[0]), call_ms=round(ms, 3), call_ms_min=round(min(ts), 3), call_ms_max=round(max(ts), 3),
               queries_per_s=float("%.3g" % (len(q[0]) / (ms / 1e3))), kernel_ms=round(kms, 3),
               kernel_queries_per_s=float("%.3g" % (len(q[0]) / (kms / 1e3))))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=100000, help="c4 documents (3 logs each)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", help="also write the rows to this file")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    from peritext_b200.engine import BatchEngine
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    rng = np.random.default_rng(1)
    rows = []
    eng = BatchEngine(0, emit_sequence=True)
    batch = workload.generate("c4", n_docs=a.docs)
    merged = eng.run(batch)
    assert (merged.results["status"] == 0).all()
    print(json.dumps(dict(c4_logs=batch.n_logs, c4_records=int(len(batch.insdel)), mean_elems=float(merged.results["n_elems"].mean()))), flush=True)
    for per in (1, 16):
        rows.append(time_case(eng, f"c4 x{per} per log", random_refs(batch, merged, np.arange(batch.n_logs), per, rng), a.reps))
    del batch, merged
    batch = workload.generate("c5", n_docs=1)
    merged = eng.run(batch)
    assert int(merged.results["status"][0]) == 0
    rows.append(time_case(eng, "c5 one log x10000", random_refs(batch, merged, [0], 10000, rng), a.reps))
    eng.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
