"""Restoring an earlier version (``pt_batch_restore``, include/peritext_b200.h): the local change that makes a resident log's
visible text equal to a version's, generated against the log's last merge.

``restore_inputs`` and ``restore_change_record`` are the readable host specification of the device call: the change is by
definition ``Micromerge.change`` of the InputOperations ``restore_inputs`` returns, under the header
``restore_change_record`` returns.  ``BatchEngine.restore`` runs it on the device.
"""
from __future__ import annotations

import ctypes

import numpy as np

from .packing import (ATTR_NONE, CDESC_DT, CHANGE_DT, DEP_DT, MARK_DT, MARK_TYPES, SPAN_COMMENT, SPAN_EM, SPAN_LINK, SPAN_STRONG, ChangeTable,
                      MergedBatch, PackedBatch, _checkout_table_ok, canon, js_key, token_str)

RESTORE_REQUEST_DT = np.dtype([("log", "<u4"), ("version", "<u4"), ("actor", "<u4"), ("first_ctr", "<u4")])
RESTORE_TEXT, RESTORE_MARKS = 1, 2
RESTORE_OK, RESTORE_LOG_FAILED, RESTORE_BAD_TABLE, RESTORE_FOREIGN, RESTORE_TEXT_DIFFERS = 0, 1, 2, 3, 4
KEEP, DELETE, RESTORE, NOTHING = "keep", "delete", "restore", "nothing"


class _RestoreView(ctypes.Structure):
    _fields_ = [("n", ctypes.c_uint32), ("status", ctypes.c_void_p), ("n_ops", ctypes.c_void_p), ("seq", ctypes.c_void_p)]


def _elements(batch: PackedBatch, merged: MergedBatch, i: int):
    """Log i's element sequence as [(packed opId, deleted, after slot defined, value token)]."""
    ins, _ = batch.log_slice(i)
    out = []
    for w in merged.sequence(i):
        r = ins[int(w) & 0x3FFFFFFF]
        out.append(((int(r["ctr"]), int(r["actor"])), bool(int(w) >> 31), bool((int(w) >> 30) & 1), int(r["payload"]) & 0x3FFFFFFF))
    return out


def classify(batch: PackedBatch, merged: MergedBatch, log: int, version: int):
    """The merge-join of log's element sequence with version's by packed opId: per element of log its class (KEEP, DELETE,
    RESTORE, NOTHING) and value token, or None when the version is no ordered subsequence of the log (FOREIGN).  A log
    element matches when its opId is that of the next unmatched version element."""
    have = _elements(batch, merged, log)
    want = _elements(batch, merged, version)
    j, out = 0, []
    for oid, deleted, _, tok in have:
        in_vis = False
        if j < len(want) and want[j][0] == oid:
            in_vis = not want[j][1]
            j += 1
        out.append(((KEEP if in_vis else DELETE) if not deleted else (RESTORE if in_vis else NOTHING), tok))
    return out if j == len(want) else None


def restore_runs(classes) -> list[tuple]:
    """The runs of a classification: [(DELETE or RESTORE, visible index v, [value tokens] or count)], v counted in the document
    as changed by the earlier runs.  A run is a maximal sequence of one action; "nothing" does not break it, a kept element does."""
    runs, v, cur = [], 0, None
    for cls, tok in classes:
        if cls == NOTHING:
            continue
        if cls == KEEP:
            cur = None
            v += 1
            continue
        if cur is None or cur[0] != cls:
            cur = [cls, v, []]
            runs.append(cur)
        cur[2].append(tok)
        if cls == RESTORE:
            v += 1
    return [(a, idx, toks if a == RESTORE else len(toks)) for a, idx, toks in runs]


def position_formats(batch: PackedBatch, merged: MergedBatch, i: int) -> list[tuple]:
    """Log i's formatting per visible position: (strong, em, link attrs or None, {comment id: attrs}).  The `comment` key with no
    ids (quirk Q3) reads as no comments."""
    out = []
    sp = merged.span_records(i)
    nv = int(merged.results[i]["n_visible"])
    for j, s in enumerate(sp):
        a, e = int(s["start"]), int(sp[j + 1]["start"]) if j + 1 < len(sp) else nv
        f = int(s["flags"])
        co = int(s["comment_off"])
        cm = {batch.comment_ids[int(x)]["id"]: batch.comment_ids[int(x)] for x in merged.comment_pool[co: co + (f >> 8)]} if f & SPAN_COMMENT else {}
        fmt = (bool(f & SPAN_STRONG), bool(f & SPAN_EM), batch.link_attrs[int(s["link_attr"])] if f & SPAN_LINK else None, cm)
        out += [fmt] * (e - a)
    return out


def marks_inputs(have: list[tuple], want: list[tuple]) -> list[dict]:
    """The MARKS InputOperations that turn formatting `have` into `want` (position_formats' tuples, equal lengths): one op per
    maximal range of positions that differ the same way, per mark type and comment id, ordered by startIndex, then ALL_MARKS
    order, then comment id in JS string order (the comment rank)."""
    def diffs(p):
        (s0, e0, l0, c0), (s1, e1, l1, c1) = have[p], want[p]
        d = {}
        for t, x, y in (("strong", s0, s1), ("em", e0, e1)):
            if x != y:
                d[(t, None)] = ("addMark" if y else "removeMark", None)
        for cid in set(c0) ^ set(c1):
            d[("comment", cid)] = ("addMark", c1[cid]) if cid in c1 else ("removeMark", c0[cid])
        if l1 is not None and (l0 is None or canon(l0) != canon(l1)):
            d[("link", None)] = ("addMark", l1)
        elif l1 is None and l0 is not None:
            d[("link", None)] = ("removeMark", None)
        return d
    open_: dict = {}
    ops = []
    for p in range(len(have) + 1):
        d = diffs(p) if p < len(have) else {}
        for key in list(open_):
            kind, attrs, start = open_[key]
            if key not in d or (d[key][0], canon(d[key][1])) != (kind, canon(attrs)):
                ops.append((start, key, kind, attrs, p))
                del open_[key]
        for key, (kind, attrs) in d.items():
            if key not in open_:
                open_[key] = (kind, attrs, p)
    ops.sort(key=lambda o: (o[0], MARK_TYPES.index(o[1][0]), js_key(o[1][1]) if o[1][1] is not None else b""))
    out = []
    for start, (t, _), kind, attrs, end in ops:
        op = {"path": ["text"], "action": kind, "startIndex": start, "endIndex": end, "markType": t}
        if attrs is not None:
            op["attrs"] = attrs
        out.append(op)
    return out


def restore_inputs(batch: PackedBatch, merged: MergedBatch, log: int, version: int, mode: int = RESTORE_TEXT):
    """The host specification of one ``pt_batch_restore`` request: (status RESTORE_*, the InputOperations of the change, in the
    reference's form).  MARKS: ``marks_inputs`` of the two logs' formatting, TEXT_DIFFERS where their visible tokens differ.
    LOG_FAILED: log's or version's merge status is not OK; BAD_TABLE: log's change table fails
    pt_batch_exchange's BAD_TABLE rules for a src; FOREIGN: the version is no ordered subsequence of the log.  A delete run is
    {delete, index v, count k}, a restore run {insert, index v, values}: the restored elements' values as NEW elements."""
    if mode not in (RESTORE_TEXT, RESTORE_MARKS):
        raise ValueError(f"restore_inputs: mode {mode} is not exactly one of RESTORE_TEXT, RESTORE_MARKS")
    if batch.changes is None:
        raise ValueError("restore_inputs: the batch has no change table")
    if int(merged.results[log]["status"]) != 0 or int(merged.results[version]["status"]) != 0:
        return RESTORE_LOG_FAILED, []
    if not _checkout_table_ok(batch, log):
        return RESTORE_BAD_TABLE, []
    if mode == RESTORE_MARKS:
        if not np.array_equal(merged.tokens(log), merged.tokens(version)):
            return RESTORE_TEXT_DIFFERS, []
        return RESTORE_OK, marks_inputs(position_formats(batch, merged, log), position_formats(batch, merged, version))
    classes = classify(batch, merged, log, version)
    if classes is None:
        return RESTORE_FOREIGN, []
    ops = []
    for action, v, arg in restore_runs(classes):
        if action == DELETE:
            ops.append({"path": ["text"], "action": "delete", "index": v, "count": arg})
        else:
            ops.append({"path": ["text"], "action": "insert", "index": v, "values": [token_str(t, batch.values) for t in arg]})
    return RESTORE_OK, ops


def restore_tokens(batch: PackedBatch, merged: MergedBatch, log: int, version: int) -> list[tuple]:
    """The runs of an OK request with their value tokens (what the device writes into the records)."""
    return restore_runs(classify(batch, merged, log, version))


def restore_change_record(batch: PackedBatch, log: int, actor: int, n_ops: int) -> tuple[int, list[tuple[int, int]]]:
    """(seq, deps) of the change actor rank `actor` appends to `log` with n_ops list ops: seq = the log's changes by the actor
    + 1; deps = (actor rank, count) of every actor with changes in the log, in the order the table first shows them (the key
    order of the reference's ``Object.assign({}, this.clock)``)."""
    cd = batch.changes.desc[log]
    ch = batch.changes.changes[int(cd["change_off"]): int(cd["change_off"]) + int(cd["n_changes"])]
    count: dict[int, int] = {}
    for c in ch:
        a = int(c["actor"])
        count[a] = count.get(a, 0) + 1
    return count.get(actor, 0) + 1, list(count.items())


def restore_change_table(batch: PackedBatch, requests, n_ops) -> ChangeTable:
    """The change table of the changes the requests append (one per request with ops), as pt_batch_append takes it."""
    cd = np.zeros(batch.n_logs, CDESC_DT)
    rows, deps = {}, {}
    for q, k in zip(np.asarray(requests, RESTORE_REQUEST_DT), n_ops):
        if int(k):
            seq, dp = restore_change_record(batch, int(q["log"]), int(q["actor"]), int(k))
            rows[int(q["log"])] = (seq, int(q["actor"]), len(dp), 0, int(k))
            deps[int(q["log"])] = [(s, a, 0) for a, s in dp]
    ch, dp = [], []
    for i in range(batch.n_logs):
        cd[i] = (len(ch), len(dp), int(i in rows), len(deps.get(i, [])))
        if i in rows:
            ch.append(rows[i]); dp += deps[i]
    return ChangeTable(cd, np.array(ch, CHANGE_DT) if ch else np.zeros(0, CHANGE_DT), np.array(dp, DEP_DT) if dp else np.zeros(0, DEP_DT))



def restore_mark_records(batch: PackedBatch, merged: MergedBatch, log: int, ops: list[dict], actor: int, first_ctr: int) -> np.ndarray:
    """The MARK_DT records of a MARKS request's InputOperations `ops` on `log` (pt_batch_change's boundaries; a removeMark link
    has attr ATTR_NONE; every mark arrives after the log's ins/del records)."""
    ins, _ = batch.log_slice(log)
    vis = [int(w) & 0x3FFFFFFF for w in merged.sequence(log) if not int(w) >> 31]
    nv = len(vis)
    oid = lambda p: (int(ins[vis[p]]["ctr"]), int(ins[vis[p]]["actor"]))
    comment_rank = {c["id"]: r for r, c in enumerate(batch.comment_ids)}
    link_index = {canon(a): i for i, a in enumerate(batch.link_attrs)}
    out = np.zeros(len(ops), MARK_DT)
    for j, op in enumerate(ops):
        t = MARK_TYPES.index(op["markType"])
        s, e = op["startIndex"], op["endIndex"]
        if t < 2:
            eb, ec = (3, (0, 0)) if e >= nv else (0, oid(e))
        else:
            eb, ec = 1, oid(e - 1)
        attr = ATTR_NONE
        if t == 2:
            attr = comment_rank[op["attrs"]["id"]]
        elif t == 3 and op["action"] == "addMark":
            attr = link_index[canon(op["attrs"])]
        sc = oid(s)
        out[j] = (first_ctr + j, actor, (1 if op["action"] == "removeMark" else 0) | (t << 1), 0 | (eb << 2), sc[0], ec[0], sc[1], ec[1], attr,
                  int(batch.desc[log]["n_insdel"]), 0)
    return out
