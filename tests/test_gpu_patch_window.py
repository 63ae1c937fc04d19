"""pt_batch_set_patch_window on the device: a merge under a window computes the Patches of each log's newest ops only, and
they are exactly the tail of the whole-log Patch stream.

One handle merges with whole logs, another the same batch under a window; the windowed records, items, demand and rendered
bytes are compared with the whole-log ones cut at the window, and with the oracle's applyChange results.  Then the append
flow (upload a prefix, append the rest, window at the old op count), a pool sized to the window's demand on a c4-shaped
batch, and the entry point's state rules."""
import json

import numpy as np
import pytest

from peritext_b200.packing import _root_text_list, apply_append, json_pools, pack_append, pack_logs
from tests.harness import fuzz_session
from tests.test_gpu_patch_bounds import list_ops
from tests.test_gpu_render_json import dense_comments, kat_logs
from tests.test_gpu_render_patches_json import O, oracle_per_change
from tests.test_patch_window import cut_json, in_window, inner_spans, n_ops, window_split

PT_ERR_INVALID, PT_ERR_STATE = 1, 4
ZERO_REC = (0, 0, 0xFFFFFFFF, 0)


def engine(patches=True):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_patches=patches)


def merge_all(e, batch):
    """merge -> (results, recs, items, status, needed, per-log patch JSON), merged once more with a pool of the reported
    demand if the item pool was too small."""
    e.merge()
    out = e._download_with_pool_retry()
    recs, items, status, needed = e.download_patches()
    if needed > len(items):
        e.set_patch_pool(needed)
        e.merge(); out = e.download()
        recs, items, status, needed = e.download_patches()
    assert needed == len(items)
    return out.results, recs, items, status, needed, e.render_patches_json_list(batch)


def item_rows(items):
    return sorted(map(tuple, items.tolist())) if len(items) else []


def per_change_tail(log, c, got):
    """The per-op patch lists `got` of changes c.. of `log`, concatenated per change."""
    lid = _root_text_list(log)
    out, k = [], 0
    for ch in log[c:]:
        cnt = sum(1 for op in ch["ops"] if op.get("obj") == lid)
        out.append([p for ps in got[k:k + cnt] for p in ps]); k += cnt
    assert k == len(got)
    return out


def check_window(batch, whole, win, w, spans=None):
    """The windowed merge `win` against the whole-log merge `whole` cut at the windows `w`."""
    res, recs, items, status, needed, text = win
    wres, wrecs, witems, wstatus, _, wtext = whole
    assert res["status"].tolist() == wres["status"].tolist() and status.tobytes() == wstatus.tobytes()
    for i in range(batch.n_logs):
        o, n = int(batch.desc[i]["insdel_off"]), int(batch.desc[i]["n_insdel"])
        k0, j0 = window_split(batch, i, int(w[i]))
        if int(status[i]) == 0:
            assert recs[o:o + j0].tolist() == [ZERO_REC] * j0, (i, int(w[i]))
            assert recs[o + j0:o + n].tobytes() == wrecs[o + j0:o + n].tobytes(), (i, int(w[i]))
        want = cut_json(wtext[i], int(w[i]), None if spans is None else spans[i])
        assert text[i] == want, (i, int(w[i]), text[i][:200], want[:200])
    keep = witems[in_window(batch, witems, w)] if len(witems) else witems
    assert item_rows(items) == item_rows(keep)
    assert needed == len(keep)


def small_corpus():
    logs = kat_logs()
    for seed, steps in ((41, 60), (42, 60), (43, 120)):
        _, lg, _ = fuzz_session(O, seed, steps, sync_prob=0.6, zero_width_prob=0.2, remove_comments=True)
        logs += lg
    return logs


# ------------------------------------------------------------------------------------------------------------------
# 1. Every cut of small logs, different windows per log in one batch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_every_cut_of_small_logs():
    logs = small_corpus()
    batch = pack_logs(logs)
    e = engine()
    try:
        e.upload(batch)
        whole = merge_all(e, batch)
        assert (whole[0]["status"] == 0).all() and (whole[3] == 0).all()
        spans = [inner_spans(t) for t in whole[5]]
        parsed = [json.loads(t) for t in whole[5]]
        top = max(n_ops(batch, i) for i in range(batch.n_logs))
        assert top >= 100
        for t in range(top + 1):
            w = np.array([(t + 7 * i) % (n_ops(batch, i) + 1) for i in range(batch.n_logs)], np.uint32)
            e.set_patch_window(w)
            win = merge_all(e, batch)
            check_window(batch, whole, win, w, spans)
            for i in range(0, batch.n_logs, 5):
                assert json.loads(win[5][i]) == parsed[i][int(w[i]):]
        # the whole-log stream itself is the oracle's
        for i, log in enumerate(logs):
            want = oracle_per_change(log)
            if want is not None:
                assert per_change_tail(log, 0, parsed[i]) == want, i
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. Windows at change boundaries: applyChange's results for changes c..
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_windows_at_change_boundaries_give_apply_change_results():
    logs = small_corpus()
    batch = pack_logs(logs, with_changes=True)
    ch = batch.changes
    starts = []
    for i in range(batch.n_logs):
        c0, nc = int(ch.desc[i]["change_off"]), int(ch.desc[i]["n_changes"])
        starts.append(np.concatenate([[0], np.cumsum(ch.changes["n_ops"][c0:c0 + nc].astype(np.int64))]))
    wants = [oracle_per_change(lg) for lg in logs]
    e = engine()
    checked = 0
    try:
        e.upload(batch); e.upload_changes(ch)
        whole = merge_all(e, batch)
        for c in range(max(len(lg) for lg in logs) + 1):
            cs = [min(c, len(lg)) for lg in logs]
            w = np.array([int(starts[i][cs[i]]) for i in range(batch.n_logs)], np.uint32)
            e.set_patch_window(w)
            win = merge_all(e, batch)
            check_window(batch, whole, win, w)
            for i, log in enumerate(logs):
                if wants[i] is not None:
                    assert per_change_tail(log, cs[i], json.loads(win[5][i])) == wants[i][cs[i]:], (i, cs[i])
                    checked += 1
    finally:
        e.close()
    assert checked >= len(logs) * 10


# ------------------------------------------------------------------------------------------------------------------
# 3. The append flow
# ------------------------------------------------------------------------------------------------------------------
def shared_arrival_log():
    """A mark ends the prefix and another mark starts the delta, both with arrival == the prefix's n_insdel."""
    lid, u = "1@u", "u"

    def chg(seq, ctr, ops):
        return {"actor": u, "seq": seq, "deps": {}, "startOp": ctr, "ops": ops}

    def ins(ctr, after, v):
        return {"opId": "%d@u" % ctr, "action": "set", "obj": lid, "elemId": after, "insert": True, "value": v}

    def mark(ctr, action, mt, a, b, attrs=None):
        op = {"opId": "%d@u" % ctr, "action": action, "obj": lid, "markType": mt, "start": {"type": "before", "elemId": a},
              "end": {"type": "after", "elemId": b}}
        if attrs is not None:
            op["attrs"] = attrs
        return op
    return [chg(1, 1, [{"opId": lid, "action": "makeList", "obj": "_root", "key": "text"}, ins(2, "_head", "a"), ins(3, "2@u", "b"),
                       ins(4, "3@u", "c")]),
            chg(2, 5, [mark(5, "addMark", "strong", "2@u", "3@u")]),
            chg(3, 6, [mark(6, "addMark", "comment", "3@u", "4@u", {"id": "x"})]),
            chg(4, 7, [ins(7, "2@u", "d")]),
            chg(5, 8, [mark(8, "removeMark", "strong", "7@u", "7@u")])]


def append_corpora():
    from tests.test_gpu_append import corpora
    out = dict(corpora())
    out["shared-arrival"] = ([shared_arrival_log(), shared_arrival_log()], [2, 3])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "compact", "runs"])
@pytest.mark.parametrize("name", ["kats", "fuzz", "quirks", "early-actor", "comments-links", "sparse", "shared-arrival"])
def test_append_then_window_gives_the_new_changes_patches(name, form):
    from tests.test_append_packing import fraction_splits, split
    from tests.test_gpu_wire_forms import upload_as
    logs, ks = append_corpora()[name]
    splits = [ks] if ks is not None else [fraction_splits(logs, (0.5,))[0], fraction_splits(logs)[-1]]
    wants = [oracle_per_change(lg) for lg in logs]
    e, u = engine(), engine()
    try:
        for cut in splits:
            prefix, suffix = split(logs, cut)
            prev = pack_logs(prefix)
            delta, remap = pack_append(prev, suffix)
            full = apply_append(prev, delta, remap)
            keep = upload_as(e, prev, form)
            merge_all(e, prev)
            e.append(delta, remap)
            del keep
            old = (prev.desc["n_insdel"].astype(np.int64) + prev.desc["n_mark"].astype(np.int64)).astype(np.uint32)
            if name == "shared-arrival":
                i0 = int(full.desc[0]["mark_off"])
                assert int(full.marks[i0]["arrival"]) == int(full.marks[i0 + 1]["arrival"]) == int(prev.desc[0]["n_insdel"])
                assert int(old[0]) == 4 and int(prev.desc[0]["n_mark"]) == 1
            e.set_patch_window(old)
            win = merge_all(e, full)
            u.upload(full)
            whole = merge_all(u, full)
            check_window(full, whole, win, old)
            for i, log in enumerate(logs):
                if int(win[3][i]) != 0 or int(win[0][i]["status"]) != 0:
                    continue
                if wants[i] is not None:
                    assert per_change_tail(log, cut[i], json.loads(win[5][i])) == wants[i][cut[i]:], (name, form, i)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. A pool sized to the window's demand, below the whole-log demand
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c4_tail_window_fits_a_pool_of_its_demand():
    from peritext_b200 import workload
    batch = dense_comments(workload.generate("c4", n_docs=1000))
    tot = batch.desc["n_insdel"].astype(np.int64) + batch.desc["n_mark"].astype(np.int64)
    w = (tot - -(-tot // 100)).astype(np.uint32)                      # each log's last 1 % of list ops
    u, e = engine(), engine()
    try:
        u.upload(batch)
        whole = merge_all(u, batch)
        assert (whole[0]["status"] == 0).all() and (whole[3] == 0).all()
        e.upload(batch)
        e.set_patch_window(w)
        e.set_patch_pool(16)
        e.merge(); e.download()
        _, items, _, needed = e.download_patches()
        assert len(items) == min(16, needed) and 16 < needed < whole[4] // 10, (needed, whole[4])
        e.set_patch_pool(needed)
        win = merge_all(e, batch)
        assert win[4] == needed
        check_window(batch, whole, win, w)
    finally:
        u.close(); e.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. State rules
# ------------------------------------------------------------------------------------------------------------------
def raw_set(e, first_op, n):
    arr = None if first_op is None else np.ascontiguousarray(first_op, dtype=np.uint32)
    return e._L.pt_batch_set_patch_window(e._h, None if arr is None or not len(arr) else arr.ctypes.data, n)


@pytest.mark.gpu
def test_state_rules():
    from peritext_b200.engine import EngineError
    logs = small_corpus()[:30]
    batch = pack_logs(logs)
    tot = np.array([n_ops(batch, i) for i in range(batch.n_logs)], np.int64)
    w1 = (tot // 2).astype(np.uint32)
    e = engine()
    try:
        # no batch yet
        assert raw_set(e, w1, batch.n_logs) == PT_ERR_STATE
        e.upload(batch)
        whole = merge_all(e, batch)
        e.set_patch_window(w1)
        # set after a merge: that merge's patches are stale until the next merge
        with pytest.raises(EngineError, match="out of order.*patch window was set after the last merge"):
            e.download_patches()
        with pytest.raises(EngineError, match="out of order.*patch window was set after the last merge"):
            e.render_patches_json(batch)
        win = merge_all(e, batch)
        check_window(batch, whole, win, w1)
        # two merges under one window: identical bytes
        again = merge_all(e, batch)
        assert again[5] == win[5] and item_rows(again[2]) == item_rows(win[2]) and again[1].tobytes() == win[1].tobytes()
        # refusals change nothing (and do not make the last merge stale)
        bad = w1.copy(); bad[3] = tot[3] + 1
        assert raw_set(e, bad, batch.n_logs) == PT_ERR_INVALID
        assert b"log 3" in e._L.pt_last_error()
        assert raw_set(e, w1, batch.n_logs - 1) == PT_ERR_INVALID
        assert raw_set(e, w1, batch.n_logs + 1) == PT_ERR_INVALID
        assert e.render_patches_json_list(batch) == win[5]
        assert merge_all(e, batch)[5] == win[5]
        # the exact edge n_insdel + n_mark is the empty window
        e.set_patch_window(tot.astype(np.uint32))
        empty = merge_all(e, batch)
        assert empty[5] == [b"[]"] * batch.n_logs and empty[4] == 0 and len(empty[2]) == 0
        check_window(batch, whole, empty, tot)
        # NULL resets to whole logs
        e.set_patch_window(w1)
        e.set_patch_window(None)
        back = merge_all(e, batch)
        assert back[5] == whole[5] and back[1].tobytes() == whole[1].tobytes()
        # an upload resets the window; so does an append (an empty delta)
        e.set_patch_window(w1)
        e.upload(batch)
        assert e.patch_window is None
        assert merge_all(e, batch)[5] == whole[5]
        e.set_patch_window(w1)
        delta, remap = pack_append(batch, [[] for _ in logs])
        e.append(delta, remap)
        assert e.patch_window is None
        assert merge_all(e, batch)[5] == whole[5]
        # run_with_patches carries the window into the DevicePatches
        from peritext_b200.packing import patch_stream
        merged, dp = e.run_with_patches(batch, first_ops=w1)
        assert dp.first_op.tolist() == w1.tolist()
        for i in range(0, batch.n_logs, 3):
            assert patch_stream(batch, dp, i, list_ops(logs[i])) == json.loads(whole[5][i])[int(w1[i]):]
        # a batch of zero logs
        e.upload(batch.select([]))
        assert raw_set(e, None, 0) == 0 and raw_set(e, [], 0) == 0
        assert raw_set(e, w1, 1) == PT_ERR_INVALID
    finally:
        e.close()
    # a handle without PT_FLAG_EMIT_PATCHES
    p = engine(patches=False)
    try:
        p.upload(batch)
        assert raw_set(p, w1, batch.n_logs) == PT_ERR_STATE
        assert b"PT_FLAG_EMIT_PATCHES" in p._L.pt_last_error()
        assert p._L.pt_batch_set_patch_window(None, None, 0) == PT_ERR_INVALID
    finally:
        p.close()


@pytest.mark.gpu
def test_failed_and_not_computed_logs_stay_empty_under_a_window():
    from peritext_b200 import workload
    from tests.test_gpu_routes import FAULTS, batch_of, route_base, with_fault
    logs = []
    for k, f in enumerate(f for f in FAULTS if f != "clean"):
        logs += [route_base("compact"), with_fault(route_base("direct" if k % 2 else "packed3"), f)]
    batch = batch_of(logs)
    tot = np.array([n_ops(batch, i) for i in range(batch.n_logs)], np.int64)
    w = (tot // 3).astype(np.uint32)
    u, e = engine(), engine()
    try:
        u.upload(batch); whole = merge_all(u, batch)
        e.upload(batch); e.set_patch_window(w); win = merge_all(e, batch)
        st = win[0]["status"]
        assert (st[0::2] == 0).all() and (st[1::2] != 0).all()
        assert all(win[5][i] == b"" for i in range(1, batch.n_logs, 2))
        assert (win[3][1::2] == 1).all()
        check_window(batch, whole, win, w)
        # a log too large for the device patch kernel: status 1, zero bytes, whatever the window
        big = dense_comments(workload.generate("c2", n_docs=1, ops_per_doc=40000))
        e.upload(big)
        e.set_patch_window([n_ops(big, i) - 5 for i in range(big.n_logs)])
        res, recs, items, status, needed, text = merge_all(e, big)
        assert (res["status"] == 0).all() and (status == 1).all() and text == [b""] * big.n_logs and needed == 0
    finally:
        u.close(); e.close()
