"""Cost of the device Patch stream under a patch window (pt_batch_set_patch_window) against whole logs.

Per case: each log's first 99 % of ins/del records (and the marks that arrived before them) are uploaded (not timed), the
last 1 % is appended with pt_batch_append, and the merge runs with PT_FLAG_EMIT_PATCHES alternately under
window 0 (whole logs) and under the 1 % window (first_op = the old n_insdel + n_mark: exactly the appended ops), in one
session.  Per window it prints the merge time (pt_batch_last_merge_ms: CUDA events around the merge, patch kernel
included; median / min / max of --reps), patch_logs_kernel's device time from a separate torch.profiler pass, the item
demand (n_items_needed), and for the render (pt_batch_render_patches_json) the call's wall time (median of --reps), its
kernel times and its output bytes.  The whole-log render of the full-size case (about 24 GB of JSON) is not attempted.
Cases: a c4 slice (--slice-docs documents x 3 replicas) and full-size c4 (--docs).  If the full-size batch does not fit at
the default patch pool, the pool is sized to 1.25 x the whole-log demand extrapolated from the slice, and the row says so.
Prints the card's name and power limit first.  Needs a GPU.

    python tools/patch_window_probe.py [--slice-docs 3000] [--docs 100000] [--reps 5] [--json OUT]
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

RENDER_KERNELS = ("pitem_count_kernel", "pitem_scatter_kernel", "pitem_rank_kernel", "patches_json_size_kernel", "patches_json_write_kernel")


def kernel_ms(fn, names):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for k in names:
            if k in ev.name:
                t = getattr(ev, "device_time_total", 0.0) or getattr(ev, "cuda_time_total", 0.0) or getattr(ev, "device_time", 0.0)
                out[k] = out.get(k, 0.0) + t / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def stats(ts):
    return dict(ms=round(float(np.median(ts)), 3), ms_min=round(min(ts), 3), ms_max=round(max(ts), 3))


def case(name, full, reps, pool=None, whole_render=True):
    from peritext_b200.engine import BatchEngine, EngineError
    from peritext_b200.packing import json_pools, split_records
    n_ins = full.desc["n_insdel"].astype(np.int64)
    prefix, delta = split_records(full, (n_ins * 99) // 100)
    old = (prefix.desc["n_insdel"].astype(np.int64) + prefix.desc["n_mark"].astype(np.int64)).astype(np.uint32)
    pools = json_pools(full)
    e = BatchEngine(0, emit_patches=True)
    note = "default patch pool"
    if pool is not None:
        e.set_patch_pool(pool)
        note = f"patch pool sized to {int(pool)} items"
    try:
        e.upload(prefix)
    except EngineError:
        e.close()
        raise
    e.append(delta)                                          # untimed: the resident history, then the new 1 %
    windows = {"whole": None, "1%": old}
    merge_ms = {k: [] for k in windows}
    needed = {}
    for r in range(reps + 1):                                # alternate the two windows; the first round is warm-up
        for k, w in windows.items():
            e.set_patch_window(w)
            e.merge()
            ms = e.last_merge_ms
            _, _, status, nd = e.download_patches()
            needed[k] = nd
            if r:
                merge_ms[k].append(ms)
    res = e.results()
    assert (res["status"] == 0).all(), name
    rows = []
    for k, w in windows.items():
        e.set_patch_window(w)
        pk = kernel_ms(lambda: (e.merge(), e.sync()), ("patch_logs_kernel",))
        _, items, status, nd = e.download_patches()
        row = dict(case=name, window=k, logs=full.n_logs, records=int(len(full.insdel) + len(full.marks)),
                   window_ops=int(sum(int(x) for x in (full.desc["n_insdel"].astype(np.int64) + full.desc["n_mark"].astype(np.int64))
                                      - (0 if w is None else w.astype(np.int64)))),
                   patch_status_computed=int((status == 0).sum()), pool=note, n_items_needed=int(nd),
                   merge=stats(merge_ms[k]), patch_logs_kernel_ms=pk.get("patch_logs_kernel", float("nan")))
        if (k != "whole" or whole_render) and nd <= len(items):
            data, off = e.render_patches_json(full, pools)       # warm-up
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                data, off = e.render_patches_json(full, pools)
                ts.append((time.perf_counter() - t0) * 1e3)
            row.update(render_call=stats(ts), render_kernels_ms=kernel_ms(lambda: e.render_patches_json(full, pools), RENDER_KERNELS),
                       render_bytes=int(off[-1]))
            del data, off
        elif k == "whole":
            row["render"] = "not attempted" if not whole_render else "pool below the whole-log demand"
        print(json.dumps(row), flush=True)
        rows.append(row)
    e.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slice-docs", type=int, default=3000, help="c4 slice documents (3 logs each)")
    ap.add_argument("--docs", type=int, default=100000, help="full-size c4 documents (3 logs each); 0 skips it")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="also write the rows to this file")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from peritext_b200 import workload
    from peritext_b200.engine import EngineError
    from tests.test_gpu_render_json import dense_comments
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    rows = case(f"c4 slice {a.slice_docs} docs", dense_comments(workload.generate("c4", n_docs=a.slice_docs)), a.reps)
    if a.docs:
        full = dense_comments(workload.generate("c4", n_docs=a.docs))
        try:
            rows += case(f"c4 {a.docs} docs", full, a.reps, whole_render=False)
        except EngineError as ex:
            print(json.dumps(dict(note=f"default patch pool does not fit: {ex}")), flush=True)
            per_log = rows[0]["n_items_needed"] / rows[0]["logs"]
            rows += case(f"c4 {a.docs} docs", full, a.reps, pool=int(per_log * full.n_logs * 1.25), whole_render=False)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
