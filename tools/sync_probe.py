"""pt_batch_sync_pairs against the host maps on the c4 shape: one change and one two-way sync per document.

  python tools/sync_probe.py [--slice-docs N] [--c4-docs N] [--ops-per-doc K] [--reps R] [--out DIR]

Every document has three replicas (logs of one resident batch) with the actor ids a0, a1, ...  A step: one replica of every
document inserts a character (pt_batch_change, outside the timed window), then syncs both ways with another replica.  Timed,
as medians of R repetitions after a warm-up, each from a fresh upload, merge and change:
  sync_pairs   pt_batch_sync_pairs of the pairs (the maps derived on the device from the actor tables)
  host_maps    on the slice only: the host copy of the batch brought up to date (apply_append of the change), packing.exchange_maps
               over it, then pt_batch_exchange
Both must leave the same batch (the merges' digests are compared).  A separate torch.profiler pass over one pt_batch_sync_pairs
gives the device time of the derive, merge and map kernels, written under --out; whether a pre-append splice ran is read from
the view.  Prints one JSON line with the GPU's name, power limit and SM clock; needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from peritext_b200 import workload  # noqa: E402
from peritext_b200.engine import BatchEngine  # noqa: E402
from peritext_b200.packing import PackedBatch, apply_append, exchange_maps  # noqa: E402
from tools.exchange_probe import change  # noqa: E402


def batch_of(docs, ops):
    base = workload.generate("c4", n_docs=docs, ops_per_doc=ops)
    base.changes = workload.history_table(base)
    base.log_actors = [[f"a{k}" for k in range(int(x))] for x in base.desc["n_actors"]]
    return base


def fresh(e, base, rnd):
    """Upload, tables, merge and the round's change (untimed); returns the host's copy of the changed batch."""
    actor, off, ops, tokens, table = rnd
    e.upload(base); e.upload_changes(base.changes); e.upload_actors(base)
    e.merge(); e.sync()
    desc, recs = change(e, base, actor, off, ops, tokens, table)
    return PackedBatch(desc, recs, base.marks[:0], log_actors=base.log_actors, changes=table)


def run(base, reps, host, prof_dir=None):
    actor, off, ops, tokens, table, pairs, _ = workload.sync_round(base)
    rnd = (actor, off, ops, tokens, table)
    e = BatchEngine(0, emit_sequence=True)
    rows = {"sync_pairs": [], "host_maps": []}
    dig, pre_ran = {}, None
    try:
        for rep in range(reps + 1):
            for path in ("sync_pairs", "host_maps") if host else ("sync_pairs",):
                delta = fresh(e, base, rnd)
                t0 = time.perf_counter()
                if path == "sync_pairs":
                    st, _, desc, (aoff, _) = e.sync_pairs(pairs)
                    pre_ran = bool(int(aoff[-1]) or (desc["n_actors"] != base.desc["n_actors"]).any())
                else:
                    cur = apply_append(base, delta)
                    maps, pre = exchange_maps(cur, [tuple(p) for p in pairs.tolist()])
                    assert pre is None
                    st, _, _ = e.exchange(pairs, maps)
                dt = time.perf_counter() - t0
                assert (st == 0).all()
                if rep:
                    rows[path].append(dt * 1000)
                e.merge()
                dig[path] = e.results()["digest"].tobytes()
        if host:
            assert dig["sync_pairs"] == dig["host_maps"]
        kernels = None
        if prof_dir:
            import torch
            from torch.profiler import ProfilerActivity, profile
            fresh(e, base, rnd)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.sync_pairs(pairs)
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(prof_dir, f"sync_pairs_{base.n_logs}.json"))
            kernels = {}
            for ev in prof.key_averages():
                if any(k in ev.key for k in ("sync_derive_kernel", "actor_merge_kernel", "sync_maps_kernel", "exchange_select_kernel", "exchange_gather_kernel",
                                             "splice_records_kernel", "splice_changes_kernel")):
                    name = next(k for k in ("sync_derive", "actor_merge", "sync_maps", "exchange_select", "exchange_gather", "splice_records", "splice_changes") if k in ev.key)
                    kernels[name + "_us"] = round(ev.device_time_total, 1)
        out = {"logs": base.n_logs, "pairs": int(len(pairs)), "records": int(len(base.insdel) + len(base.marks)), "pre_append_ran": pre_ran,
               "kernels_device_us": kernels}
        for path, r in rows.items():
            if r:
                out[path] = {"ms_median": round(statistics.median(r), 3), "ms_min": round(min(r), 3), "ms_max": round(max(r), 3)}
        return out
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slice-docs", type=int, default=3000)
    ap.add_argument("--c4-docs", type=int, default=100000)
    ap.add_argument("--ops-per-doc", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    res = {"probe": "sync", "gpu": gpu, "reps": a.reps,
           "slice": run(batch_of(a.slice_docs, a.ops_per_doc), a.reps, True, a.out),
           "full": run(batch_of(a.c4_docs, a.ops_per_doc), a.reps, False, a.out)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
