"""Cost of pt_batch_render_json (every merged document's FormatSpanWithText[] as JSON text, rendered on the device).

Merges full-size c4 (100 000 documents x 3 replicas; comment ranks densified, not timed) and renders it.  Per case it prints
the wall time of one call (host clock around a call that synchronises: pool upload, size pass, scan, total read-back, write
pass, copy of the offsets and bytes) as the median of --reps calls, the kernel time of the size and write kernels from a
separate torch.profiler pass, the output bytes and the bytes/s written, and beside it the rate of the pure-Python
specification (tests/test_gpu_render_json.py render_spans_json) on a 3 000-log sample on this host's CPU.  The same for the
c5 sample (--c5-docs documents x 2 replicas), and for a single c5 log: if one log alone takes about as long as the whole c5
batch, the one-warp-per-log tail dominates.  Needs a GPU.

    python tools/render_probe.py [--docs 100000] [--c5-docs 296] [--reps 10] [--json OUT]
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


def kernel_ms(engine, batch, pools):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        engine.render_json(batch, pools)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for k in ("json_size_kernel", "json_write_kernel"):
            if k in ev.name:
                t = getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)
                out[k] = out.get(k, 0.0) + t / 1e3
    return out


def cpu_spec_rate(batch, merged, pools, n=3000):
    from tests.test_gpu_render_json import render_spans_json
    idx = np.linspace(0, batch.n_logs - 1, min(n, batch.n_logs)).astype(np.int64)
    t0 = time.perf_counter()
    nbytes = sum(len(render_spans_json(batch, merged, int(i), pools)) for i in idx)
    dt = time.perf_counter() - t0
    return dict(cpu_spec_logs=len(idx), cpu_spec_s=round(dt, 3), cpu_spec_logs_per_s=float("%.3g" % (len(idx) / dt)),
                cpu_spec_bytes_per_s=float("%.3g" % (nbytes / dt)))


def time_case(engine, name, batch, merged, pools, reps, cpu=True):
    data, off = engine.render_json(batch, pools)            # warm-up (module load, first allocations)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        engine.render_json(batch, pools)
        ts.append((time.perf_counter() - t0) * 1e3)
    ms = float(np.median(ts))
    k = kernel_ms(engine, batch, pools)
    ks, kw = k.get("json_size_kernel", float("nan")), k.get("json_write_kernel", float("nan"))
    row = dict(case=name, logs=batch.n_logs, out_bytes=int(off[-1]), call_ms=round(ms, 3), call_ms_min=round(min(ts), 3),
               call_ms_max=round(max(ts), 3), call_bytes_per_s=float("%.3g" % (int(off[-1]) / (ms / 1e3))),
               size_kernel_ms=round(ks, 3), write_kernel_ms=round(kw, 3),
               write_kernel_bytes_per_s=float("%.3g" % (int(off[-1]) / (kw / 1e3))))
    if cpu:
        row.update(cpu_spec_rate(batch, merged, pools))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=100000, help="c4 documents (3 logs each)")
    ap.add_argument("--c5-docs", type=int, default=296, help="c5 documents (2 logs each)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", help="also write the rows to this file")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import json_pools
    from tests.test_gpu_render_json import dense_comments
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    rows = []
    eng = BatchEngine(0)
    for name, make in (("c4", lambda: workload.generate("c4", n_docs=a.docs)),
                       ("c5", lambda: workload.generate("c5", n_docs=a.c5_docs))):
        batch = dense_comments(make())
        pools = json_pools(batch)
        merged = eng.run(batch)
        assert (merged.results["status"] == 0).all(), name
        rows.append(time_case(eng, f"{name} {batch.n_logs} logs", batch, merged, pools, a.reps))
        if name == "c5":
            one = batch.select([0])
            eng.run(one)
            rows.append(time_case(eng, "c5 one log", one, None, pools, a.reps, cpu=False))
        del batch, merged
    eng.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
