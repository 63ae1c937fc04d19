"""The patch window (pt_batch_set_patch_window) on the host: `packing.patch_stream` of DevicePatches cut to a window equals the
whole-log decode from the window's first op on, for every cut of the KAT and fuzz logs.  The patches are the oracle's own,
encoded on the CPU.  Also pins the list-op order the window's positions use, the change-table rule for change boundaries,
and the JSON-aware cut the GPU tests compare the rendered bytes with."""
import json

import numpy as np

from peritext_b200.packing import DevicePatches, pack_logs, patch_stream
from tests.harness import fuzz_session
from tests.test_gpu_patch_bounds import list_ops, oracle_per_op
from tests.test_gpu_render_json import kat_logs
from tests.test_gpu_render_patches_json import O, encoded_patches, render_patches_json
from peritext_b200.packing import json_pools


# ------------------------------------------------------------------------------------------------------------------
# Helpers (the GPU tests use them too)
# ------------------------------------------------------------------------------------------------------------------
def window_split(batch, i, first_op):
    """(k0, j0): the mark records and ins/del records of log i before list-op position first_op (mark k sits at
    min(arrival_k, n) + k)."""
    d = batch.desc[i]
    n, mo, m = int(d["n_insdel"]), int(d["mark_off"]), int(d["n_mark"])
    arr = np.minimum(batch.marks["arrival"][mo:mo + m].astype(np.int64), n)
    k0 = int(((arr + np.arange(m)) < first_op).sum())
    return k0, first_op - k0


def n_ops(batch, i):
    return int(batch.desc[i]["n_insdel"]) + int(batch.desc[i]["n_mark"])


def in_window(batch, items, first_ops):
    """Mask of the pool items owned by an op inside its log's window."""
    keep = np.zeros(len(items), bool)
    cut = {i: window_split(batch, i, int(first_ops[i])) for i in set(items["log"].tolist())}
    for q, (log, tag) in enumerate(zip(items["log"].tolist(), items["tag"].tolist())):
        k0, j0 = cut[log]
        keep[q] = (tag & 0x7FFFFFFF) >= (k0 if tag & 0x80000000 else j0)
    return keep


def cut_patches(batch, dp, first_ops):
    """What a merge under the window `first_ops` leaves, from the whole-log `dp`: the records before each window
    {0, 0, PT_ATTR_NONE, 0}, the items of ops before it dropped."""
    recs = dp.recs.copy()
    for i in range(batch.n_logs):
        _, j0 = window_split(batch, i, int(first_ops[i]))
        o = int(batch.desc[i]["insdel_off"])
        recs[o:o + j0] = (0, 0, 0xFFFFFFFF, 0)
    items = dp.items[in_window(batch, dp.items, first_ops)] if len(dp.items) else dp.items
    return DevicePatches(recs, items, dp.status, np.asarray(first_ops, np.uint32))


def inner_spans(text: bytes):
    """(start, end) byte offsets of the inner arrays of one log's patch JSON, split by a JSON-aware walk (strings may hold
    brackets and commas)."""
    s = text.decode("utf-8")
    assert s[0] == "[" and s[-1] == "]"
    dec, out, p = json.JSONDecoder(), [], 1
    while s[p] != "]":
        _, e = dec.raw_decode(s, p)
        out.append((len(s[:p].encode("utf-8")), len(s[:e].encode("utf-8"))))
        p = e + 1 if s[e] == "," else e
    return out


def cut_json(text: bytes, first_op: int, spans=None) -> bytes:
    """The whole-log patch JSON with its first `first_op` inner arrays removed."""
    if not text:
        return b""
    sp = inner_spans(text) if spans is None else spans
    if first_op >= len(sp):
        return b"[]"
    return b"[" + text[sp[first_op][0]: sp[-1][1]] + b"]"


def small_logs():
    logs = kat_logs()
    for seed in (31, 32, 33):
        _, lg, _ = fuzz_session(O, seed, 60, zero_width_prob=0.2, remove_comments=True)
        logs += lg
    return logs


def encodable(logs):
    """The logs whose oracle patches `encode` can attribute to single ops (it refuses a change with two consecutive mark ops
    of one type and action)."""
    out = []
    for lg in logs:
        try:
            oracle_per_op(lg)
        except AssertionError:
            continue
        out.append(lg)
    return out


# ------------------------------------------------------------------------------------------------------------------
# Tests
# ------------------------------------------------------------------------------------------------------------------
def test_patch_stream_under_every_window_is_the_whole_log_tail():
    logs = encodable(small_logs())
    assert len(logs) >= 60
    batch = pack_logs(logs)
    dp = encoded_patches(batch, logs, seed=3)
    opss = [list_ops(lg) for lg in logs]
    whole = [patch_stream(batch, dp, i, ops) for i, ops in enumerate(opss)]
    assert patch_stream(batch, DevicePatches(dp.recs, dp.items, dp.status, np.zeros(batch.n_logs, np.uint32)), 0, opss[0]) == whole[0]
    top = max(n_ops(batch, i) for i in range(batch.n_logs))
    checked = 0
    for t in range(top + 1):
        w = np.array([(t + 7 * i) % (n_ops(batch, i) + 1) for i in range(batch.n_logs)], np.uint32)
        cp = cut_patches(batch, dp, w)
        for i, ops in enumerate(opss):
            assert patch_stream(batch, cp, i, ops) == whole[i][int(w[i]):], (i, int(w[i]))
            checked += 1
    assert checked == (top + 1) * batch.n_logs and top >= 60


def test_window_positions_are_the_list_op_order():
    """Mark record k is list op min(arrival_k, n) + k, and a change table's n_ops counts the change's list ops, so change c
    starts at the sum of the earlier changes' n_ops."""
    logs = small_logs()
    batch = pack_logs(logs, with_changes=True)
    ch = batch.changes
    for i, lg in enumerate(logs):
        ops = list_ops(lg)
        assert len(ops) == n_ops(batch, i)
        d = batch.desc[i]
        arr = batch.marks["arrival"][int(d["mark_off"]):int(d["mark_off"]) + int(d["n_mark"])].astype(np.int64)
        pos = np.minimum(arr, int(d["n_insdel"])) + np.arange(len(arr))
        assert [k for k, op in enumerate(ops) if op["action"] in ("addMark", "removeMark")] == pos.tolist()
        c0, nc = int(ch.desc[i]["change_off"]), int(ch.desc[i]["n_changes"])
        starts = np.concatenate([[0], np.cumsum(ch.changes["n_ops"][c0:c0 + nc].astype(np.int64))])
        assert starts.tolist() == [len(list_ops(lg[:c])) if c else 0 for c in range(len(lg) + 1)]
        for c in range(len(lg) + 1):
            k0, j0 = window_split(batch, i, int(starts[c]))
            assert k0 == sum(1 for op in ops[:starts[c]] if op["action"] in ("addMark", "removeMark")) and k0 + j0 == starts[c]


def test_json_cut_is_the_parsed_tail():
    logs = encodable(small_logs())[:40]
    batch = pack_logs(logs)
    dp = encoded_patches(batch, logs, seed=4)
    pools = json_pools(batch)
    for i in range(batch.n_logs):
        text = render_patches_json(batch, dp, i, pools)
        full = json.loads(text)
        sp = inner_spans(text)
        assert len(sp) == len(full) == n_ops(batch, i)
        for w in range(len(full) + 1):
            got = cut_json(text, w, sp)
            assert json.loads(got) == full[w:]
            assert got[1:] == text[len(text) - len(got) + 1:]            # a byte-exact tail of the whole-log text
        assert cut_json(text, 0, sp) == text
