"""Cost of the device Patch stream of large logs (PT_FLAG_EMIT_LARGE_PATCHES, patch_large_kernel).

Cases, in one session:
* the c5 sample (--docs documents x 2 replicas, dense comments; every log is above the warp patch kernel's limits): the merge without
  patches, then with the flag on whole logs and on the 1 % window after pt_batch_append (each log's first 99 % of ins/del
  records uploaded, the last 1 % appended, first_op = the old n_insdel + n_mark), alternated;
* the c4 slice (--slice-docs documents x 3 replicas, dense comments, as tools/patch_window_probe.py) with whole logs, the
  warp kernel (PT_FLAG_EMIT_PATCHES) alternated with the sweep on every log (the flag and PT_PATCH_WARP=0).
Per row: the merge time (pt_batch_last_merge_ms: CUDA events around the merge, patch kernels included; median / min / max of
--reps after one warm-up), the patch kernels' device time from a separate torch.profiler pass, the logs computed, the item
demand (n_items_needed), and for the c5 window the wall time of one pt_batch_render_patches_json call (median of --reps) and
its output bytes.  The whole-log render of the c5 sample is not attempted.  Prints the card's name and power limit first.
Needs a GPU.

    python tools/large_patches_probe.py [--docs 296] [--slice-docs 3000] [--reps 5] [--json OUT]
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

from patch_window_probe import kernel_ms, stats  # noqa: E402

KERNELS = ("patch_logs_kernel", "patch_large_kernel")


def env(value):
    if value is None:
        os.environ.pop("PT_PATCH_WARP", None)
    else:
        os.environ["PT_PATCH_WARP"] = value


def timed_merges(engines, reps):
    """Alternate the merges of `engines` (name -> (engine, setup)); the first round is a warm-up."""
    ms = {k: [] for k in engines}
    for r in range(reps + 1):
        for k, (e, setup) in engines.items():
            setup()
            e.merge()
            t = e.last_merge_ms
            e.sync()
            if r:
                ms[k].append(t)
    return ms


def row_of(name, e, full, ms, setup, window_ops):
    setup()
    pk = kernel_ms(lambda: (e.merge(), e.sync()), KERNELS)
    _, items, status, nd = e.download_patches()
    return dict(case=name, logs=full.n_logs, records=int(len(full.insdel) + len(full.marks)), window_ops=int(window_ops),
                patch_status_computed=int((status == 0).sum()), n_items_needed=int(nd), merge=stats(ms),
                **{k + "_ms": pk.get(k, float("nan")) for k in KERNELS}), items, nd


def c5_rows(full, reps):
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import json_pools, split_records
    rows = []
    plain = BatchEngine(0)
    plain.upload(full)
    whole = BatchEngine(0, large_patches=True)
    whole.upload(full)
    n_ins = full.desc["n_insdel"].astype(np.int64)
    prefix, delta = split_records(full, (n_ins * 99) // 100)
    old = (prefix.desc["n_insdel"].astype(np.int64) + prefix.desc["n_mark"].astype(np.int64)).astype(np.uint32)
    win = BatchEngine(0, large_patches=True)
    win.upload(prefix)
    win.append(delta)
    win.set_patch_window(old)
    nop = lambda: None
    ms = timed_merges({"merge only": (plain, nop), "whole": (whole, nop), "1%": (win, nop)}, reps)
    res = plain.download()
    assert (res.results["status"] == 0).all()
    rows.append(dict(case="c5 merge without patches", logs=full.n_logs, merge=stats(ms["merge only"])))
    total_ops = int((full.desc["n_insdel"].astype(np.int64) + full.desc["n_mark"].astype(np.int64)).sum())
    r, _, _ = row_of("c5 whole logs", whole, full, ms["whole"], nop, total_ops)
    r["render"] = "not attempted"
    rows.append(r)
    r, items, nd = row_of("c5 1 % window after append", win, full, ms["1%"], nop, total_ops - int(old.astype(np.int64).sum()))
    if nd <= len(items):
        pools = json_pools(full)
        win.render_patches_json(full, pools)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            data, off = win.render_patches_json(full, pools)
            ts.append((time.perf_counter() - t0) * 1e3)
        r.update(render_call=stats(ts), render_bytes=int(off[-1]))
    rows.append(r)
    for e in (plain, whole, win):
        e.close()
    return rows


def c4_rows(full, reps):
    from peritext_b200.engine import BatchEngine
    warp = BatchEngine(0, emit_patches=True)
    warp.upload(full)
    sweep = BatchEngine(0, large_patches=True)
    env("0")
    try:
        sweep.upload(full)                                   # PT_PATCH_WARP is read at upload
    finally:
        env(None)
    ms = timed_merges({"warp": (warp, lambda: None), "sweep": (sweep, lambda: None)}, reps)
    total_ops = int((full.desc["n_insdel"].astype(np.int64) + full.desc["n_mark"].astype(np.int64)).sum())
    rows = []
    for k, e in (("warp", warp), ("sweep", sweep)):
        r, _, _ = row_of(f"c4 slice, {k} kernel", e, full, ms[k], lambda: None, total_ops)
        rows.append(r)
        e.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=296, help="c5 documents (2 logs each)")
    ap.add_argument("--slice-docs", type=int, default=3000, help="c4 slice documents (3 logs each); 0 skips it")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="also write the rows to this file")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    from tests.test_gpu_render_json import dense_comments
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    rows = []
    for r in c5_rows(dense_comments(workload.generate("c5", n_docs=a.docs)), a.reps):
        print(json.dumps(r), flush=True); rows.append(r)
    if a.slice_docs:
        for r in c4_rows(dense_comments(workload.generate("c4", n_docs=a.slice_docs)), a.reps):
            print(json.dumps(r), flush=True); rows.append(r)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
