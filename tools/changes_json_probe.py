"""Call and kernel times of pt_batch_render_changes_json on the benchmark shapes.

  python tools/changes_json_probe.py [--c4-docs N] [--c5-docs M] [--reps R]

Three measurements, each the median of R calls after a warm-up call (every call synchronises):
  range    whole-log RANGE over every log of a c4 batch with workload.history_table (one change per log holding all its list
           ops); full-size c4 would render about 40 GB of text, so the default is 4 000 documents (12 000 logs, 12 M records)
  missing  MISSING for the pairs of one workload.sync_round on that batch, after its change: each pair's target clock is the
           other replica's, so a request selects the changer's new change
  c5       whole-log RANGE over a c5 sample (one ~111 K-op change per log: the item slicing's case)
Reported per measurement: the call's wall time, the summed device time of the render's kernels (torch.profiler, one extra
call), the output bytes and the kernel launches.  Generated batches carry no extras, so this is the list-op projection, which
is the whole device cost (an extra is one pool copy).  Prints one JSON line with the GPU's name and power limit; needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from peritext_b200 import workload  # noqa: E402
from peritext_b200.engine import BatchEngine  # noqa: E402
from peritext_b200.packing import _pool, canon, clock_requests, range_requests  # noqa: E402


def named(batch):
    """A generated batch with the string tables the render needs: actor rank r is "doc{r+1}", the list is "1@doc1"."""
    batch.log_actors = [["doc%d" % (r + 1) for r in range(int(a))] for a in batch.desc["n_actors"]]
    batch.log_lists = ["1@doc1"] * batch.n_logs
    batch.log_counters = [None] * batch.n_logs
    n_com = int(batch.marks["attr"][(batch.marks["kind"] >> 1 & 3) == 2].max()) + 1 if len(batch.marks) and ((batch.marks["kind"] >> 1 & 3) == 2).any() else 0
    pools = _pool([]) + _pool([canon(a).encode() for a in batch.link_attrs]) + _pool([canon({"id": "c%d" % k}).encode() for k in range(n_com)])
    return batch, pools


def measure(e, batch, req, pools, reps):
    e.render_changes_json(batch, req, None, pools)                 # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        data, off, status = e.render_changes_json(batch, req, None, pools)
        ts.append((time.perf_counter() - t0) * 1000)
    assert (status == 0).all()
    import torch
    from torch.profiler import ProfilerActivity, profile
    l0 = e.launch_count
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.render_changes_json(batch, req, None, pools)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("changes_" in ev.name or "out_" in ev.name):
            k = ev.name.split("(")[0].split("::")[-1]
            kernels[k] = kernels.get(k, 0.0) + ev.device_time / 1000.0
    return {"requests": int(len(req[0] if isinstance(req, tuple) else req)), "bytes": int(len(data)), "call_ms_median": round(statistics.median(ts), 3),
            "call_ms_min": round(min(ts), 3), "kernel_ms_total": round(sum(kernels.values()), 3),
            "kernel_ms": {k: round(v, 3) for k, v in sorted(kernels.items())}, "launches": int(e.launch_count - l0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c4-docs", type=int, default=4000)
    ap.add_argument("--c5-docs", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"probe": "changes_json", "gpu": gpu, "reps": a.reps}
    base, pools = named(workload.generate("c4", n_docs=a.c4_docs))
    base.changes = workload.history_table(base)
    e = BatchEngine(0, emit_sequence=True)
    try:
        e.upload(base); e.upload_changes(base.changes)
        print("range c4", file=sys.stderr, flush=True)
        out["range_c4"] = {"logs": base.n_logs, "records": int(len(base.insdel) + len(base.marks)), **measure(e, base, range_requests(range(base.n_logs)), pools, a.reps)}
        # one sync step: after the changers' new changes, each pair asks for what its target's clock lacks
        from tools.exchange_probe import change
        actor, off, ops, tokens, table, pairs, maps = workload.sync_round(base)
        e.merge(); e.sync()
        change(e, base, actor, off, ops, tokens, table)
        clocks = []
        for d in pairs[:, 1]:
            c = {"doc1": 1}
            if actor[d] != 0xFFFFFFFF:
                c["doc%d" % (int(actor[d]) + 1)] = 2 if actor[d] == 0 else 1
            clocks.append(c)
        print("missing c4", file=sys.stderr, flush=True)
        out["missing_c4"] = {"pairs": int(len(pairs)), **measure(e, base, clock_requests(base, pairs[:, 0], clocks), pools, a.reps)}
    finally:
        e.close()
    c5, pools5 = named(workload.generate("c5", n_docs=a.c5_docs))
    c5.changes = workload.history_table(c5)
    e = BatchEngine(0)
    try:
        e.upload(c5); e.upload_changes(c5.changes)
        print("range c5", file=sys.stderr, flush=True)
        out["range_c5"] = {"logs": c5.n_logs, "ops_per_change": int(c5.changes.changes["n_ops"].mean()), **measure(e, c5, range_requests(range(c5.n_logs)), pools5, a.reps)}
    finally:
        e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
