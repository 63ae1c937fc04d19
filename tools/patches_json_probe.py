"""Cost of pt_batch_render_patches_json (every log's Patch stream as JSON text, rendered on the device).

Merges a c4 slice (--c4-docs documents x 3 replicas; comment ranks densified, not timed) and a c3 sample with the device
Patch stream, and renders it.  Per case it prints the wall time of one call (host clock around a call that synchronises:
demand check, pool upload, item ordering, size pass, scan, total read-back, write pass, copy of the offsets and bytes) as the
median of --reps calls, the kernel times of the item-ordering, size and write kernels from a separate torch.profiler pass,
the output bytes and the bytes/s written by the write kernel, and beside it the rate of the Python path this replaces
(`packing.patch_stream` + `json.dumps`) on a sample of logs on this host's CPU.  Prints the card's name and power limit first.
Needs a GPU.

    python tools/patches_json_probe.py [--c4-docs 3000] [--c3-docs 4] [--reps 10] [--json OUT]
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

KERNELS = ("pitem_count_kernel", "pitem_scatter_kernel", "pitem_rank_kernel", "patches_json_size_kernel", "patches_json_write_kernel")


def kernel_ms(engine, batch, pools):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        engine.render_patches_json(batch, pools)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for k in KERNELS:
            if k in ev.name:
                t = getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)
                out[k] = out.get(k, 0.0) + t / 1e3
    return out


def python_rate(batch, dp, n=300):
    """patch_stream + json.dumps per log, with op dicts rebuilt from the records (the caller's ops, in the Python path)."""
    from peritext_b200.packing import patch_stream
    idx = np.linspace(0, batch.n_logs - 1, min(n, batch.n_logs)).astype(np.int64)
    names = ("strong", "em", "comment", "link")
    opss = []
    for i in idx:
        ins, mk = batch.log_slice(int(i))
        ops, j = [], 0
        for r in mk:
            while j < min(int(r["arrival"]), len(ins)):
                ops.append({"action": "set" if int(ins[j]["payload"]) >> 30 == 0 else "del", "value": "x"}); j += 1
            k = int(r["kind"])
            ops.append({"action": "removeMark" if k & 1 else "addMark", "markType": names[(k >> 1) & 3], "attrs": {"id": "a"}})
        ops += [{"action": "set" if int(ins[x]["payload"]) >> 30 == 0 else "del", "value": "x"} for x in range(j, len(ins))]
        opss.append(ops)
    dp._index()                                                # the per-log grouping of the pool, built once
    t0 = time.perf_counter()
    nbytes = sum(len(json.dumps(patch_stream(batch, dp, int(i), ops), separators=(",", ":"))) for i, ops in zip(idx, opss))
    dt = time.perf_counter() - t0
    return dict(py_logs=len(idx), py_s=round(dt, 3), py_logs_per_s=float("%.3g" % (len(idx) / dt)), py_bytes_per_s=float("%.3g" % (nbytes / dt)))


def time_case(engine, name, batch, dp, pools, reps):
    data, off = engine.render_patches_json(batch, pools)     # warm-up (module load, first allocations)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        engine.render_patches_json(batch, pools)
        ts.append((time.perf_counter() - t0) * 1e3)
    ms = float(np.median(ts))
    k = kernel_ms(engine, batch, pools)
    kw = k.get("patches_json_write_kernel", float("nan"))
    row = dict(case=name, logs=batch.n_logs, computed=int((dp.status == 0).sum()), items=len(dp.items), out_bytes=int(off[-1]),
               bytes_per_log=round(int(off[-1]) / max(1, int((dp.status == 0).sum()))), call_ms=round(ms, 3), call_ms_min=round(min(ts), 3),
               call_ms_max=round(max(ts), 3), order_kernels_ms=round(sum(k.get(x, 0.0) for x in KERNELS[:3]), 3),
               size_kernel_ms=round(k.get("patches_json_size_kernel", float("nan")), 3), write_kernel_ms=round(kw, 3),
               write_kernel_bytes_per_s=float("%.3g" % (int(off[-1]) / (kw / 1e3))))
    row.update(python_rate(batch, dp))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c4-docs", type=int, default=3000, help="c4 documents (3 logs each)")
    ap.add_argument("--c3-docs", type=int, default=4, help="c3 documents of 10 000 records")
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
    eng = BatchEngine(0, emit_patches=True)
    for name, make in (("c4", lambda: workload.generate("c4", n_docs=a.c4_docs)),
                       ("c3", lambda: workload.generate("c3", n_docs=a.c3_docs, ops_per_doc=10000))):
        batch = dense_comments(make())
        pools = json_pools(batch)
        merged, dp = eng.run_with_patches(batch)
        assert (merged.results["status"] == 0).all(), name
        rows.append(time_case(eng, f"{name} {batch.n_logs} logs", batch, dp, pools, a.reps))
        del batch, merged, dp
    eng.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
