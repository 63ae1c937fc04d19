"""One fuzz step per document on the c4 shape, with the sync on the device and with the sync through the host.

  python tools/exchange_probe.py [--c4-docs N] [--ops-per-doc K] [--reps R]

Every document has three replicas (logs of one resident batch).  A step (reference test/fuzz.ts:167-199): one replica of
every document inserts a character (pt_batch_change), then syncs both ways with another replica.  Two ways to sync:
  (a) device   pt_batch_exchange of the pairs {changer -> other, other -> changer}
  (b) host     the path without it: the generated records come back in pt_batch_change's view, the host re-addresses them to
               the other replica's log (vectorised numpy here; the packing helpers change_dicts + pack_append do the same per
               document in Python, far slower) and pt_batch_append uploads them again
Per path: the wall time of change + sync (each call synchronises), medians of R repetitions after a warm-up, each repetition
from a fresh upload and merge outside the timed window; the bytes each way over PCIe, counted from the arrays the change and the
sync move (each splice's re-plan also uploads per-log descriptors and plan arrays, the same on both paths and left out); and
the kernel launches (pt_batch_launch_count).  Both paths must leave the same batch: the merges' digests are compared.
Prints one JSON line with the GPU's name and power limit; needs a GPU.
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
from peritext_b200.packing import CDESC_DT, DESC_DT, MARK_DT, ChangeTable, PackedBatch, _ranges  # noqa: E402


def change(e, batch, actor, off, ops, tokens, table):
    """``change_packed`` of the round; returns the delta's descriptors and ins/del records (the probe's change has no marks)."""
    _, desc, recs, _ = e.change_packed(actor, off, ops, tokens, 0, len(batch.link_attrs), 0, table)
    return desc, recs


def readdress(batch, desc, recs, table, src, dst):
    """Path (b)'s host step: the delta of pt_batch_append that gives every dst its src's generated records and change."""
    n = batch.n_logs
    order = np.argsort(dst)
    s = src[order]
    d2 = np.zeros(n, DESC_DT)
    d2["n_actors"] = batch.desc["n_actors"]
    d2["max_ctr"] = desc["max_ctr"]; d2["max_ctr"][dst] = np.maximum(desc["max_ctr"][dst], desc["max_ctr"][src])
    d2["n_insdel"][dst] = desc["n_insdel"][src]
    d2["insdel_off"] = np.cumsum(d2["n_insdel"].astype(np.uint64)) - d2["n_insdel"]
    out = recs[_ranges(desc["insdel_off"][s], desc["n_insdel"][s])]
    cd = np.zeros(n, CDESC_DT)
    cd["n_changes"][dst] = 1; cd["n_deps"][dst] = table.desc["n_deps"][src]
    cd["change_off"] = np.cumsum(cd["n_changes"]) - cd["n_changes"]; cd["dep_off"] = np.cumsum(cd["n_deps"]) - cd["n_deps"]
    chs = table.changes[table.desc["change_off"][s].astype(np.int64)]
    dps = table.deps[_ranges(table.desc["dep_off"][s], table.desc["n_deps"][s])]
    return PackedBatch(d2, out, np.zeros(0, MARK_DT), changes=ChangeTable(cd, chs, dps))


def nbytes(*arrays):
    return int(sum(a.nbytes for a in arrays if a is not None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c4-docs", type=int, default=100000)
    ap.add_argument("--ops-per-doc", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    base = workload.generate("c4", n_docs=a.c4_docs, ops_per_doc=a.ops_per_doc)
    base.changes = workload.history_table(base)
    actor, off, ops, tokens, table, pairs, maps = workload.sync_round(base)
    src, dst = pairs[0::2, 0], pairs[0::2, 1]
    n = base.n_logs
    e = BatchEngine(0, emit_sequence=True)
    rows = {"device": [], "host": []}
    digests, launches, pcie = {}, {}, {}
    try:
        for rep in range(a.reps + 1):                     # the first repetition warms up both paths
            for path in ("device", "host"):
                e.upload(base); e.upload_changes(base.changes)
                e.merge(); e.sync()
                l0 = e.launch_count
                t0 = time.perf_counter()
                desc, recs = change(e, base, actor, off, ops, tokens, table)
                if path == "device":
                    status, (doff, flat), xdesc = e.exchange(pairs, maps)
                else:
                    delta = readdress(base, desc, recs, table, src, dst)
                    e.append(delta)
                dt = time.perf_counter() - t0
                launches[path] = e.launch_count - l0
                np_ = pairs.shape[0]
                if path == "device":              # pairs, maps, slot offsets, delivered offsets and bases up; totals (twice) and indices down
                    assert (status == 0).all()
                    up = np_ * 8 + nbytes(maps.actor_off, maps.actor_map) + 2 * (np_ + 1) * 8 + np_ * 32
                    down = 2 * np_ * 32 + flat.nbytes
                else:                             # the re-addressed records, change records and their descriptors up
                    up = nbytes(delta.desc, delta.insdel, delta.changes.desc, delta.changes.changes, delta.changes.deps)
                    down = 0
                pcie[path] = {"change_h2d_bytes": nbytes(actor, off, ops, tokens, table.desc, table.changes, table.deps),
                              "change_d2h_bytes": n * 8 + nbytes(recs), "sync_h2d_bytes": up, "sync_d2h_bytes": down}
                if rep:
                    rows[path].append(dt * 1000)
                e.merge()
                digests[path] = e.results()["digest"].copy()
        assert digests["device"].tobytes() == digests["host"].tobytes()
        out = {"probe": "exchange", "logs": n, "documents": n // 3, "records": int(len(base.insdel) + len(base.marks)), "reps": a.reps,
               "gpu": gpu, "same_digests": True}
        for path in ("device", "host"):
            out[path] = {"step_ms_median": round(statistics.median(rows[path]), 3), "step_ms_min": round(min(rows[path]), 3),
                         "step_ms_max": round(max(rows[path]), 3), "launches": int(launches[path]), **pcie[path]}
        print(json.dumps(out))
    finally:
        e.close()


if __name__ == "__main__":
    main()
