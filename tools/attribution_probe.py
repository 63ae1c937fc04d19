"""Cost of pt_batch_attribute on full-size c4 and on the c5 sample, merged with the element sequence.

Every log gets a table of many changes (its list ops in changes of --ops-per-change, by actor rank 0), so the runs follow the
changes; a one-change table would give one run per log and measure nothing.  Cases: all logs and 1 % of the logs, each without a
clock and at a clock covering half of each log's changes.  Reports per case:
  - the call's wall time (host clock around the call, which synchronises): median, min and max of --reps, after a warm-up;
  - the resolve, count and write kernels' device time from a torch.profiler run of its own;
  - runs and run bytes per requested log, and the peak scratch from the header's cost model (28 B per ins/del record, 8 B per
    change of the requested logs, 32 B per run), with the device memory free before the call;
  - whether the call ran at all (an all-logs request on full c4 may not fit beside the resident batch; the error is recorded);
  - the card's name and power limit.
Needs a GPU.

    python tools/attribution_probe.py [--reps 5] [--json OUT]
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

KERNELS = ("attribute_resolve_kernel", "attribute_runs_kernel<false>", "attribute_runs_kernel<true>")


def split_table(batch, per):
    """Every log's list ops as changes of `per` ops (the last one shorter) by actor rank 0, seq 1 .. n."""
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, ChangeTable
    ops = (batch.desc["n_insdel"] + batch.desc["n_mark"]).astype(np.int64)
    cnt = np.maximum(1, (ops + per - 1) // per)
    cd = np.zeros(batch.n_logs, CDESC_DT)
    cd["n_changes"] = cnt
    cd["change_off"][1:] = np.cumsum(cnt)[:-1]
    ch = np.zeros(int(cnt.sum()), CHANGE_DT)
    first = np.repeat(cd["change_off"].astype(np.int64), cnt)
    ch["seq"] = np.arange(len(ch)) - first + 1
    ch["n_ops"] = per
    last = cd["change_off"].astype(np.int64) + cnt - 1
    ch["n_ops"][last] = ops - per * (cnt - 1)
    return ChangeTable(cd, ch, np.zeros(0, DEP_DT))


def half_clocks(batch, logs):
    from peritext_b200.packing import CLOCK_DT
    off = np.arange(len(logs) + 1, dtype=np.uint64)
    ent = np.zeros(len(logs), CLOCK_DT)
    ent["seq"] = batch.changes.desc["n_changes"][logs] // 2
    return off, ent


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def kernel_ms(prof):
    ms = dict.fromkeys(KERNELS, 0.0)
    for ev in prof.events():
        for k in KERNELS:
            if ev.name.startswith("void pta::" + k) or ev.name.startswith(k) or ("pta::" + k) in ev.name:
                ms[k] += (getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)) / 1e3
    return ms


def measure(e, batch, logs, clock, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from peritext_b200.engine import EngineError
    lg = np.asarray(logs, np.int64)
    out = {"requests": len(lg), "records": int(batch.desc["n_insdel"][lg].sum()), "changes": int(batch.changes.desc["n_changes"][lg].sum()),
           "free_bytes_before": int(torch.cuda.mem_get_info()[0])}
    try:
        st, off, runs = e.attribute(logs, clock)                       # warm-up
    except EngineError as x:
        out["error"] = str(x)
        return out
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        st, off, runs = e.attribute(logs, clock)
        times.append((time.perf_counter() - t0) * 1e3)
    out["ok"] = bool((st == 0).all())
    out["call_ms"] = {"median": float(np.median(times)), "min": min(times), "max": max(times)}
    out["runs"] = len(runs)
    out["runs_per_log"] = len(runs) / len(lg)
    out["run_bytes_per_log"] = 32 * len(runs) / len(lg)
    out["flagged_runs"] = int((runs["flags"] != 0).sum())
    out["peak_scratch_bytes"] = 28 * out["records"] + 8 * out["changes"] + 32 * len(runs) + 40 * len(lg)
    out["scratch_bytes_per_record"] = out["peak_scratch_bytes"] / max(1, out["records"])
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.attribute(logs, clock)
        torch.cuda.synchronize()
    out["kernel_ms"] = kernel_ms(prof)
    return out


def workload_cases(name, batch, per, reps):
    from peritext_b200.engine import BatchEngine
    batch.changes = split_table(batch, per)
    e = BatchEngine(0, emit_sequence=True)
    res = {"n_logs": batch.n_logs, "records": int(batch.desc["n_insdel"].sum()), "changes": int(batch.changes.desc["n_changes"].sum())}
    try:
        e.upload(batch); e.upload_changes(batch.changes); e.merge(); e.sync()
        assert (e.results()["status"] == 0).all()
        every = list(range(batch.n_logs))
        some = every[::100] if batch.n_logs >= 100 else every[:1]
        for tag, lg in (("all", every), ("1pct", some)):
            res[tag] = measure(e, batch, lg, None, reps)
            res[tag + "_clock"] = measure(e, batch, lg, half_clocks(batch, lg), reps)
    finally:
        e.close()
    return name, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ops-per-change", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    out = {"card": card(), "ops_per_change": a.ops_per_change}
    for name, b in (("c4", lambda: workload.generate("c4")), ("c5_sample", lambda: workload.generate("c5", n_docs=8))):
        k, v = workload_cases(name, b(), a.ops_per_change, a.reps)
        out[k] = v
        print(json.dumps({k: v}), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
