"""Cost of pt_batch_checkout on full-size c4: 1 % of the logs checked out at half their change table.

Every c4 log gets a two-change table (its first half of list ops, then the rest, by actor rank 0), so half the table is the first
change and the checkout gathers half of each source's records.  Reports:
  - the call's wall time (host clock around the call, which synchronises): median, min and max of --reps, each after an
    untimed pt_batch_select_logs that retires the previous checkouts;
  - the select, gather and splice kernels' device time from a torch.profiler run of its own;
  - the bytes the call copies host -> device and device -> host, counted from its copies (requests, layout, per-log
    descriptors of the re-planned batch) for this shape;
  - whether the checkouts' result headers (status, counts, 128-bit digest) equal those of an upload of apply_checkout's batch
    (built on the host from the sources alone, since a checkout does not depend on the other logs);
  - the card's name and power limit.
Needs a GPU.

    python tools/checkout_probe.py [--reps 5] [--json OUT]
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

KERNELS = ("checkout_select_kernel", "exchange_gather_kernel", "splice_records_kernel", "splice_changes_kernel")


def halves_table(batch):
    """Every log's list ops as two changes by actor rank 0: the first half, then the rest."""
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, ChangeTable
    n = batch.n_logs
    ops = (batch.desc["n_insdel"] + batch.desc["n_mark"]).astype(np.int64)
    cd = np.zeros(n, CDESC_DT)
    cd["change_off"] = 2 * np.arange(n); cd["n_changes"] = 2
    ch = np.zeros(2 * n, CHANGE_DT)
    ch["seq"] = np.tile([1, 2], n)
    ch["n_ops"][0::2] = ops // 2; ch["n_ops"][1::2] = ops - ops // 2
    return ChangeTable(cd, ch, np.zeros(0, DEP_DT))


def pcie_bytes(n0, n):
    """The call's copies for n requests on n0 resident logs (engine.cu pt_batch_checkout, splice, install_plan)."""
    nn = n0 + n
    h2d = 4 * n + 4 * n + 8 * (n + 1)            # logs, n_changes, scratch slots
    h2d += 8 * n + 8 * (n + 1) + 32 * n           # gather pairs, delivered offsets, delta bases
    h2d += 2 * 32 * nn + 4 * nn + 2 * 24 * nn     # splice: delta and new descriptors, from, delta and new change descriptors
    h2d += 32 * nn + 4 * nn + 8 * nn + 8 * nn     # the re-planned batch: descriptors, order, text and span offsets
    d2h = 32 * n + 4                              # per-request totals, the splice's refusal flag
    return h2d, d2h


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from peritext_b200 import workload
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import apply_checkout

    full = workload.generate("c4")
    full.changes = halves_table(full)
    n0 = full.n_logs
    lg = list(range(0, n0, 100))
    n = len(lg)
    half = [1] * n
    e = BatchEngine(0)
    out = {"card": card(), "n_logs": n0, "requests": n}
    try:
        e.upload(full); e.upload_changes(full.changes)
        e.checkout(lg, n_changes=half)                                   # warm-up
        times = []
        for _ in range(a.reps):
            e.select_logs(list(range(n0)))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = e.checkout(lg, n_changes=half)
            times.append((time.perf_counter() - t0) * 1e3)
            assert (st == 0).all()
        out["call_ms"] = {"median": float(np.median(times)), "min": min(times), "max": max(times)}
        e.merge()
        res = e.results()
        # the checkouts against an upload of apply_checkout's batch
        src = full.select(lg)
        want, status = apply_checkout(src, list(range(n)), n_changes=half)
        assert (status == 0).all()
        u = BatchEngine(0)
        try:
            u.upload(want); u.upload_changes(want.changes); u.merge()
            ref = u.results()
        finally:
            u.close()
        out["digest_equal"] = bool(res[n0:].tobytes() == ref[n:].tobytes() and (res["status"][n0:] == 0).all())
        out["records_gathered"] = int(want.desc["n_insdel"][n:].sum() + want.desc["n_mark"][n:].sum())
        # kernel times, a run of its own
        e.select_logs(list(range(n0)))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.checkout(lg, n_changes=half)
            torch.cuda.synchronize()
        ms = dict.fromkeys(KERNELS, 0.0)
        for ev in prof.events():
            for k in KERNELS:
                if k in ev.name:
                    ms[k] += (getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)) / 1e3
        out["kernel_ms"] = ms
        h2d, d2h = pcie_bytes(n0, n)
        out["h2d_bytes"], out["d2h_bytes"] = h2d, d2h
    finally:
        e.close()
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
