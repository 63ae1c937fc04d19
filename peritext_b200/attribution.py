"""Attribution of merged documents (``pt_batch_attribute``, include/peritext_b200.h): which change inserted and which change
deleted every element, as runs over the element sequence, and what changed since a version named by a vector clock.

``attribution_runs`` is the readable host specification of the device call; ``BatchEngine.attribute`` returns the same arrays.
"""
from __future__ import annotations

import ctypes
from typing import Sequence

import numpy as np

from .packing import (KIND_DELETE, KIND_INSERT, MergedBatch, PackedBatch, _checkout_table_ok, _request_clocks, change_record_ranges)

ATTR_RUN_DT = np.dtype([("elem", "<u4"), ("visible", "<u4"), ("n", "<u4"), ("flags", "<u4"), ("ins_seq", "<u4"), ("del_seq", "<u4"),
                        ("ins_actor", "<u2"), ("del_actor", "<u2"), ("reserved", "<u4")])
ATTR_INSERTED_SINCE, ATTR_DELETED_SINCE = 1, 2
ATTR_OK, ATTR_LOG_FAILED, ATTR_BAD_TABLE = 0, 1, 2


class _AttrView(ctypes.Structure):
    _fields_ = [("n", ctypes.c_uint32), ("status", ctypes.c_void_p), ("off", ctypes.c_void_p), ("runs", ctypes.c_void_p),
                ("n_runs", ctypes.c_uint64)]


def _log_runs(batch: PackedBatch, merged: MergedBatch, s: int, clk: dict | None) -> list[tuple]:
    """The runs of log s (an OK merge and a table that passes), as ATTR_RUN_DT rows."""
    cd = batch.changes.desc[s]
    ch = batch.changes.changes[int(cd["change_off"]): int(cd["change_off"]) + int(cd["n_changes"])]
    rng = change_record_ranges(batch, s)
    ins, _ = batch.log_slice(s)
    change_of = np.zeros(len(ins), np.int64)                 # the change whose list-op range holds each ins/del record
    for c in range(len(ch)):
        change_of[int(rng[c, 0]): int(rng[c, 1])] = c
    covered = [clk is None or int(c["seq"]) <= clk.get(int(c["actor"]), 0) for c in ch]
    kind = ins["payload"] >> 30
    insert_at = {(int(r["ctr"]), int(r["actor"])): j for j, r in enumerate(ins) if kind[j] == KIND_INSERT}
    first_del: dict[int, tuple] = {}                         # insert record -> (smallest delete opId, its change)
    del_covered: set[int] = set()
    for j in np.flatnonzero(kind == KIND_DELETE):
        t = insert_at[(int(ins[j]["ref_ctr"]), int(ins[j]["ref_actor"]))]
        key = (int(ins[j]["ctr"]), int(ins[j]["actor"]))     # compareOpIds order on packed ids
        if t not in first_del or key < first_del[t][0]:
            first_del[t] = (key, int(change_of[j]))
        if covered[change_of[j]]:
            del_covered.add(t)
    rows, prev = [], None
    visible = 0
    for e, w in enumerate(merged.sequence(s)):
        r = int(w) & 0x3FFFFFFF
        ci = int(change_of[r])
        dc = first_del[r][1] if r in first_del else None
        flags = (0 if covered[ci] else ATTR_INSERTED_SINCE) | (ATTR_DELETED_SINCE if dc is not None and r not in del_covered else 0)
        tup = (ci, dc, flags)
        if tup != prev:
            rows.append([e, visible, 0, flags, int(ch[ci]["seq"]), 0 if dc is None else int(ch[dc]["seq"]), int(ch[ci]["actor"]),
                         0 if dc is None else int(ch[dc]["actor"]), 0])
            prev = tup
        rows[-1][2] += 1
        visible += dc is None
    return [tuple(x) for x in rows]


def attribution_runs(batch: PackedBatch, merged: MergedBatch, logs: Sequence[int], clock=None) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The host specification of ``pt_batch_attribute``: (u32 status [n] ATTR_*, u64 offsets [n + 1], ATTR_RUN_DT runs) for
    request k on log ``logs[k]`` of `batch`, whose merge (with its element sequence) is `merged`.
      insert  an element's insert record lies in the list-op range [P_c, P_c + n_ops_c) of change c (``change_record_ranges``);
              ins_actor / ins_seq are c's.
      delete  of the deletes that target it, the one with the smallest packed opId (ctr, actor rank) is attributed; del_actor /
              del_seq are its change's, and del_seq 0 means not deleted.
      clock   ``clock`` = (u64 offsets [n + 1], CLOCK_DT entries by actor rank), ``packing.checkout_clocks``: a change is covered
              iff seq <= clock[actor] (absent: 0).  INSERTED_SINCE: the inserting change is not covered; DELETED_SINCE: deleted
              and no delete of the element is covered.  Without a clock the flags are 0.
    A run is a maximal stretch of consecutive elements (tombstones included) with equal (ins, del, flags); ``elem`` is its first
    element's index and ``visible`` the visible elements before it.  LOG_FAILED: the log's merge status is not OK;
    BAD_TABLE: its table fails pt_batch_exchange's BAD_TABLE rules for a src.  Raises ValueError where the device refuses
    (a log outside the batch; a bad clock)."""
    logs = [int(x) for x in logs]
    if batch.changes is None:
        raise ValueError("attribution_runs: the batch has no change table")
    if any(not 0 <= s < batch.n_logs for s in logs):
        raise ValueError("attribution_runs: a request names no log of the batch")
    clocks = _request_clocks(batch, logs, None, clock) if clock is not None else [None] * len(logs)
    status = np.zeros(len(logs), np.uint32)
    off = np.zeros(len(logs) + 1, np.uint64)
    rows: list[tuple] = []
    for k, (s, clk) in enumerate(zip(logs, clocks)):
        if int(merged.results[s]["status"]) != 0:
            status[k] = ATTR_LOG_FAILED
        elif not _checkout_table_ok(batch, s):
            status[k] = ATTR_BAD_TABLE
        else:
            rows += _log_runs(batch, merged, s, clk)
        off[k + 1] = len(rows)
    return status, off, np.array(rows, ATTR_RUN_DT) if rows else np.zeros(0, ATTR_RUN_DT)
