"""ctypes binding of the engine's C-ABI (include/peritext_b200.h, built as peritext_b200/libperitext_b200.so).

There is no CPU fallback: if the shared library is missing or no CUDA device is usable, every entry point raises
``EngineError``.  torch is not needed here; pass ``torch.cuda.current_stream().cuda_stream`` as ``stream`` to enqueue
on a torch stream.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from .packing import (CDESC_DT, CHANGE_DT, CLOCK_DT, CHANGES_REQUEST_DT, EXTRA_DT, ChangeExtras, CHANGE_OK, CHANGE_STATUS_DT, DEP_DT, DESC_DT, ELEM_NOT_FOUND, ELEM_POS_DT, ELEM_REF_DT, INSDEL_DT, MARK_DT,
                      RESULT_DT, SPAN_DT, AppendRemap, ChangeTable, ExchangeMaps, MergedBatch, PackedBatch, apply_append, change_dicts, change_inputs, elem_refs,
                      string_pools)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libperitext_b200.so")
_lib = None

EXPORTS = ["pt_batch_create", "pt_batch_upload", "pt_batch_upload_runs", "pt_compress_runs", "pt_compact_ops", "pt_batch_upload_compact", "pt_batch_adopt_device", "pt_batch_upload_changes",
           "pt_batch_append", "pt_batch_change", "pt_batch_exchange", "pt_batch_upload_actors", "pt_batch_download_actors", "pt_batch_add_actors", "pt_batch_sync_pairs", "pt_ingest_create", "pt_ingest_parse", "pt_ingest_packed", "pt_ingest_pool", "pt_ingest_error", "pt_ingest_destroy", "pt_batch_merge", "pt_batch_sync",
           "pt_batch_download", "pt_batch_download_begin", "pt_batch_download_results", "pt_batch_device_results", "pt_batch_launch_count", "pt_batch_stats",
           "pt_batch_last_merge_ms", "pt_batch_set_comment_pool", "pt_batch_download_patches", "pt_batch_set_patch_pool", "pt_batch_set_patch_window", "pt_batch_query_elements", "pt_batch_find_elements",
           "pt_batch_render_json", "pt_batch_render_patches_json", "pt_batch_render_changes_json", "pt_ingest_change_extras", "pt_batch_destroy", "pt_strerror", "pt_last_error", "pt_version"]


class EngineError(RuntimeError):
    pass


class _PackedOps(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("logs", ctypes.c_void_p), ("insdel", ctypes.c_void_p),
                ("n_insdel_total", ctypes.c_uint64), ("marks", ctypes.c_void_p), ("n_mark_total", ctypes.c_uint64)]


class _PackedRuns(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("logs", ctypes.c_void_p), ("run_off", ctypes.c_void_p), ("tok_off", ctypes.c_void_p),
                ("runs", ctypes.c_void_p), ("tokens", ctypes.c_void_p), ("marks", ctypes.c_void_p),
                ("n_insdel_total", ctypes.c_uint64), ("n_mark_total", ctypes.c_uint64)]


INSDEL_C8_DT = np.dtype([("ctr", "<u2"), ("ref_ctr", "<u2"), ("w", "<u4")])
MARK_C16_DT = np.dtype([("ctr", "<u2"), ("start_ctr", "<u2"), ("end_ctr", "<u2"), ("arrival", "<u2"), ("attr", "<u4"), ("w", "<u4")])
RUN_DT = np.dtype([("ctr0", "<u4"), ("ref_ctr", "<u4"), ("actor", "<u2"), ("ref_actor", "<u2"), ("kind_count", "<u4")])


class PackedRuns:
    """Run-compressed wire form of a PackedBatch (include/peritext_b200.h pt_packed_runs): typing runs and consecutive
    deletes collapse to one 16-byte run record (+ 4 bytes per inserted value)."""

    def __init__(self, desc, run_off, tok_off, runs, tokens, marks, n_insdel_total, changes: ChangeTable | None = None):
        self.desc, self.run_off, self.tok_off, self.runs, self.tokens, self.marks = desc, run_off, tok_off, runs, tokens, marks
        self.n_insdel_total = int(n_insdel_total)
        self.changes = changes        # the batch's change table (admission pre-pass), if it has one

    @property
    def n_logs(self) -> int:
        return int(self.desc.shape[0])

    @property
    def nbytes(self) -> int:
        return int(self.desc.nbytes + self.run_off.nbytes + self.tok_off.nbytes + self.runs.nbytes + self.tokens.nbytes + self.marks.nbytes)

    def slice_logs(self, a: int, b: int) -> "PackedRuns":
        """Logs [a, b) as views (pinned memory stays pinned); offsets re-based (small copies of the offset arrays)."""
        d = self.desc[a:b].copy()
        ro = self.run_off[a:b + 1].copy(); to = self.tok_off[a:b + 1].copy()
        r0, r1, t0, t1 = int(ro[0]), int(ro[-1]), int(to[0]), int(to[-1])
        if len(d):
            i0, m0 = int(d[0]["insdel_off"]), int(d[0]["mark_off"])
            m1 = int(d[-1]["mark_off"]) + int(d[-1]["n_mark"]); i1 = int(d[-1]["insdel_off"]) + int(d[-1]["n_insdel"])
            d["insdel_off"] -= i0; d["mark_off"] -= m0
        else:
            i0 = i1 = m0 = m1 = 0
        return PackedRuns(d, ro - ro[0], to - to[0], self.runs[r0:r1], self.tokens[t0:t1], self.marks[m0:m1], i1 - i0,
                          self.changes.slice_logs(a, b) if self.changes is not None else None)


def compress_runs(batch: PackedBatch, pin=None) -> PackedRuns:
    """Host-side run compression (pt_compress_runs).  `pin(nbytes_array) -> array` may place the big arrays in pinned memory."""
    L = load_library()
    desc = np.ascontiguousarray(batch.desc)
    insdel = np.ascontiguousarray(batch.insdel)
    marks = np.ascontiguousarray(batch.marks)
    ops = _PackedOps(len(desc), desc.ctypes.data, insdel.ctypes.data, len(insdel), marks.ctypes.data, len(marks))
    n = len(desc)
    run_off = np.zeros(n + 1, np.uint64); tok_off = np.zeros(n + 1, np.uint64)
    nr, nt = ctypes.c_uint64(0), ctypes.c_uint64(0)
    _check(L.pt_compress_runs(ctypes.byref(ops), run_off.ctypes.data, tok_off.ctypes.data, None, None, ctypes.byref(nr), ctypes.byref(nt)), "pt_compress_runs")
    alloc = pin or (lambda a: a)
    runs = alloc(np.zeros(max(1, nr.value), RUN_DT)); tokens = alloc(np.zeros(max(1, nt.value), np.uint32))
    _check(L.pt_compress_runs(ctypes.byref(ops), run_off.ctypes.data, tok_off.ctypes.data, runs.ctypes.data, tokens.ctypes.data, ctypes.byref(nr), ctypes.byref(nt)), "pt_compress_runs")
    return PackedRuns(desc, alloc(run_off), alloc(tok_off), runs[: nr.value], tokens[: nt.value], alloc(marks) if pin else marks, len(insdel),
                      batch.changes)


class _ChangeTable(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("logs", ctypes.c_void_p), ("changes", ctypes.c_void_p), ("n_changes_total", ctypes.c_uint64),
                ("deps", ctypes.c_void_p), ("n_deps_total", ctypes.c_uint64)]


class _AppendRemap(ctypes.Structure):
    _fields_ = [("actor_off", ctypes.c_void_p), ("actor_map", ctypes.c_void_p), ("ctr_off", ctypes.c_void_p), ("ctr_map", ctypes.c_void_p),
                ("comment_map", ctypes.c_void_p), ("n_comment_map", ctypes.c_uint64)]


def _change_struct(table: ChangeTable):
    """(pt_change_table, the contiguous arrays it points into)."""
    d, c, p = np.ascontiguousarray(table.desc), np.ascontiguousarray(table.changes), np.ascontiguousarray(table.deps)
    return _ChangeTable(len(d), d.ctypes.data, c.ctypes.data if len(c) else 0, len(c), p.ctypes.data if len(p) else 0, len(p)), (d, c, p)


class _ChangeInput(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("actor", ctypes.c_void_p), ("input_off", ctypes.c_void_p), ("ops", ctypes.c_void_p),
                ("tokens", ctypes.c_void_p), ("n_tokens", ctypes.c_uint64), ("n_values", ctypes.c_uint32), ("n_links", ctypes.c_uint32),
                ("n_comments", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class _ChangeView(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("status", ctypes.c_void_p), ("delta", _PackedOps)]


class _ExchangeInput(ctypes.Structure):
    _fields_ = [("n_pairs", ctypes.c_uint32), ("pairs", ctypes.c_void_p), ("actor_off", ctypes.c_void_p), ("actor_map", ctypes.c_void_p),
                ("ctr_off", ctypes.c_void_p), ("ctr_map", ctypes.c_void_p)]


class _ExchangeView(ctypes.Structure):
    _fields_ = [("n_pairs", ctypes.c_uint32), ("status", ctypes.c_void_p), ("delivered_off", ctypes.c_void_p), ("delivered", ctypes.c_void_p),
                ("delta", ctypes.c_void_p)]


PAIR_DT = np.dtype([("src", "<u4"), ("dst", "<u4")])


class _ActorTables(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("data", ctypes.c_void_p), ("off", ctypes.c_void_p), ("count", ctypes.c_uint64),
                ("per_log_first", ctypes.c_void_p), ("counters_first", ctypes.c_void_p)]


class _ActorInput(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("data", ctypes.c_void_p), ("off", ctypes.c_void_p), ("count", ctypes.c_uint64),
                ("per_log_first", ctypes.c_void_p)]


class _ActorView(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("count", ctypes.c_uint64), ("rank", ctypes.c_void_p), ("actor_off", ctypes.c_void_p),
                ("actor_map", ctypes.c_void_p), ("spliced", ctypes.c_uint32)]


class _SyncView(ctypes.Structure):
    _fields_ = [("n_pairs", ctypes.c_uint32), ("status", ctypes.c_void_p), ("delivered_off", ctypes.c_void_p), ("delivered", ctypes.c_void_p),
                ("delta", ctypes.c_void_p), ("actor_off", ctypes.c_void_p), ("actor_map", ctypes.c_void_p)]


def _view_array(p, count, dt):
    """A copy of `count` elements of dtype `dt` at address p (engine-owned view memory)."""
    if not count or not p:
        return np.zeros(0, dt)
    return np.frombuffer((ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(p), dtype=dt, count=count).copy()


class _SpansView(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("results", ctypes.c_void_p), ("text_off", ctypes.c_void_p),
                ("span_off", ctypes.c_void_p), ("text", ctypes.c_void_p), ("spans", ctypes.c_void_p),
                ("comment_pool", ctypes.c_void_p), ("comment_pool_used", ctypes.c_uint64), ("seq", ctypes.c_void_p),
                ("seq_off", ctypes.c_void_p), ("comment_pool_needed", ctypes.c_uint64)]


class _Limits(ctypes.Structure):
    _fields_ = [("comment_pool_entries", ctypes.c_uint64), ("flags", ctypes.c_uint32), ("patch_pool_items", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32 * 4)]


class _PatchView(ctypes.Structure):
    _fields_ = [("recs", ctypes.c_void_p), ("items", ctypes.c_void_p), ("n_items", ctypes.c_uint64), ("n_items_needed", ctypes.c_uint64),
                ("status", ctypes.c_void_p)]


class _JsonPools(ctypes.Structure):
    _fields_ = [("values", ctypes.c_void_p), ("values_off", ctypes.c_void_p), ("n_values", ctypes.c_uint64),
                ("links", ctypes.c_void_p), ("links_off", ctypes.c_void_p), ("n_links", ctypes.c_uint64),
                ("comments", ctypes.c_void_p), ("comments_off", ctypes.c_void_p), ("n_comments", ctypes.c_uint64)]


class _JsonView(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("off", ctypes.c_void_p), ("bytes", ctypes.c_void_p), ("n_bytes", ctypes.c_uint64)]


class _ChangesJsonInput(ctypes.Structure):
    _fields_ = [("n_requests", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("requests", ctypes.c_void_p), ("clock", ctypes.c_void_p),
                ("n_clock", ctypes.c_uint64), ("pools", _JsonPools), ("actors", ctypes.c_void_p), ("actors_off", ctypes.c_void_p),
                ("actors_first", ctypes.c_void_p), ("counters", ctypes.c_void_p), ("counters_first", ctypes.c_void_p),
                ("list_ids", ctypes.c_void_p), ("list_ids_off", ctypes.c_void_p), ("extras", ctypes.c_void_p), ("n_extras", ctypes.c_uint64),
                ("extra_ops", ctypes.c_void_p), ("extra_ops_off", ctypes.c_void_p), ("n_extra_ops", ctypes.c_uint64)]


class _ChangesJsonView(ctypes.Structure):
    _fields_ = [("n_requests", ctypes.c_uint32), ("off", ctypes.c_void_p), ("bytes", ctypes.c_void_p), ("n_bytes", ctypes.c_uint64),
                ("status", ctypes.c_void_p)]


QUERY_DT = np.dtype([("log", "<u4"), ("index", "<u4"), ("flags", "<u4"), ("reserved", "<u4")])
PATCH_REC_DT = np.dtype([("index", "<u4"), ("flags", "<u4"), ("link_attr", "<u4"), ("reserved", "<u4")])
PATCH_ITEM_DT = np.dtype([("log", "<u4"), ("tag", "<u4"), ("a", "<u4"), ("b", "<u4")])
FLAG_EMIT_SEQUENCE = 1
FLAG_EMIT_PATCHES = 2
FLAG_EMIT_LARGE_PATCHES = 4


def load_library() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          f"(make -C peritext_b200/csrc). There is no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH)
    vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
    L.pt_batch_create.argtypes = [ctypes.c_int, vp, vp, ctypes.POINTER(vp)]
    L.pt_batch_upload.argtypes = [vp, vp]
    L.pt_batch_adopt_device.argtypes = [vp, vp]
    L.pt_batch_upload_runs.argtypes = [vp, vp]
    L.pt_compress_runs.argtypes = [vp, vp, vp, vp, vp, ctypes.POINTER(u64), ctypes.POINTER(u64)]
    L.pt_batch_upload_changes.argtypes = [vp, vp]
    L.pt_batch_append.argtypes = [vp, vp, vp, vp]
    L.pt_batch_change.argtypes = [vp, vp, vp, vp]
    L.pt_batch_exchange.argtypes = [vp, vp, vp]
    L.pt_batch_upload_actors.argtypes = [vp, vp]
    L.pt_batch_download_actors.argtypes = [vp, vp]
    L.pt_batch_sync_pairs.argtypes = [vp, vp, u32, vp]
    L.pt_batch_add_actors.argtypes = [vp, vp, vp]
    L.pt_compact_ops.argtypes = [vp, vp, vp, ctypes.c_int]
    L.pt_batch_upload_compact.argtypes = [vp, vp]
    L.pt_ingest_create.argtypes = [ctypes.POINTER(vp)]
    L.pt_ingest_parse.argtypes = [vp, vp, vp, u32, ctypes.c_int]
    L.pt_ingest_packed.argtypes = [vp, vp, vp]
    L.pt_ingest_pool.argtypes = [vp, ctypes.c_int, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.POINTER(vp)]
    L.pt_ingest_error.argtypes = [vp]; L.pt_ingest_error.restype = ctypes.c_char_p
    L.pt_ingest_destroy.argtypes = [vp]; L.pt_ingest_destroy.restype = None
    L.pt_batch_merge.argtypes = [vp]
    L.pt_batch_sync.argtypes = [vp]
    L.pt_batch_download.argtypes = [vp, vp]
    L.pt_batch_download_begin.argtypes = [vp]
    L.pt_batch_download_results.argtypes = [vp, vp, u32]
    L.pt_batch_device_results.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(u32)]
    L.pt_batch_launch_count.argtypes = [vp]; L.pt_batch_launch_count.restype = u64
    L.pt_batch_stats.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64 * 4)]
    L.pt_batch_last_merge_ms.argtypes = [vp]; L.pt_batch_last_merge_ms.restype = ctypes.c_float
    L.pt_batch_set_comment_pool.argtypes = [vp, u64]
    L.pt_batch_download_patches.argtypes = [vp, vp]
    L.pt_batch_set_patch_pool.argtypes = [vp, u64]
    L.pt_batch_set_patch_window.argtypes = [vp, vp, u32]
    L.pt_batch_query_elements.argtypes = [vp, vp, u32, vp]
    L.pt_batch_find_elements.argtypes = [vp, vp, u32, vp]
    L.pt_batch_render_json.argtypes = [vp, vp, vp]
    L.pt_batch_render_patches_json.argtypes = [vp, vp, vp]
    L.pt_batch_render_changes_json.argtypes = [vp, vp, vp]
    L.pt_ingest_change_extras.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(u64)]
    L.pt_batch_destroy.argtypes = [vp]; L.pt_batch_destroy.restype = None
    L.pt_strerror.argtypes = [ctypes.c_int]; L.pt_strerror.restype = ctypes.c_char_p
    L.pt_last_error.restype = ctypes.c_char_p
    L.pt_version.restype = ctypes.c_char_p
    _lib = L
    return L


def _check(rc: int, what: str):
    if rc != 0:
        L = load_library()
        raise EngineError(f"{what}: {L.pt_strerror(rc).decode()} ({L.pt_last_error().decode()})")


class BatchEngine:
    """One handle per (GPU, batch).  ``upload`` -> ``merge`` -> ``download``."""

    def __init__(self, device: int = 0, stream: int | None = None, comment_pool_entries: int = 0, emit_sequence: bool = False,
                 emit_patches: bool = False, large_patches: bool = False):
        """``large_patches`` (PT_FLAG_EMIT_LARGE_PATCHES, implies ``emit_patches``): the device also derives the Patch stream of
        the logs too large for the warp patch kernel, so a log's patch status is 1 only if its merge failed."""
        L = load_library()
        self._L = L
        self._h = ctypes.c_void_p()
        emit_patches = emit_patches or large_patches
        self.emit_patches = emit_patches
        self.large_patches = large_patches
        flags = (FLAG_EMIT_SEQUENCE if (emit_sequence or emit_patches) else 0) | (FLAG_EMIT_PATCHES if emit_patches else 0) | \
            (FLAG_EMIT_LARGE_PATCHES if large_patches else 0)
        lim = _Limits(comment_pool_entries, flags, 0, (ctypes.c_uint32 * 4)())
        _check(L.pt_batch_create(device, ctypes.byref(lim), ctypes.c_void_p(stream or 0), ctypes.byref(self._h)), "pt_batch_create")
        self._keep = None
        self._uploaded(np.zeros(0, DESC_DT), 0)

    def _uploaded(self, desc, n_insdel_total):
        """Record the shape of the batch just uploaded, in whichever form: what the downloads size their views by."""
        self.n_logs = len(desc)
        self.patch_window = None                                             # every upload resets the window to whole logs
        self._n_insdel = int(n_insdel_total)                                 # patch records: one per ins/del record
        self._n_seq = int(desc["n_insdel"].astype(np.uint64).sum())          # element sequences: the capacity layout

    def _ops_struct(self, desc, insdel_ptr, n_insdel, marks_ptr, n_mark):
        return _PackedOps(len(desc), desc.ctypes.data, insdel_ptr, n_insdel, marks_ptr, n_mark)

    def upload(self, batch: PackedBatch):
        desc = np.ascontiguousarray(batch.desc)
        insdel = np.ascontiguousarray(batch.insdel)
        marks = np.ascontiguousarray(batch.marks)
        ops = self._ops_struct(desc, insdel.ctypes.data, len(insdel), marks.ctypes.data, len(marks))
        _check(self._L.pt_batch_upload(self._h, ctypes.byref(ops)), "pt_batch_upload")
        self._uploaded(desc, len(insdel))

    def upload_changes(self, table: ChangeTable):
        """Attach the batch's change table: the next merge runs the admission pre-pass (seq / deps checks of
        Micromerge.applyChange, reference src/micromerge.ts:501-509) and rejected logs report status 6 / 7."""
        t, _keep = _change_struct(table)
        _check(self._L.pt_batch_upload_changes(self._h, ctypes.byref(t)), "pt_batch_upload_changes")

    def append(self, delta: PackedBatch, remap: AppendRemap | None = None, changes: ChangeTable | None = None):
        """Extend every log of the resident batch with the delta's records on the device (pt_batch_append): afterwards the
        handle holds what an upload of ``packing.apply_append(batch, delta, remap)`` would hold, and needs a merge.  `delta`
        and `remap` come from ``packing.pack_append``; `changes` is the delta's change table (default ``delta.changes``),
        required exactly when the resident batch has one.  Works after every upload form and after an earlier append."""
        r = remap or AppendRemap()
        desc = np.ascontiguousarray(delta.desc)
        insdel = np.ascontiguousarray(delta.insdel); marks = np.ascontiguousarray(delta.marks)
        ops = self._ops_struct(desc, insdel.ctypes.data if len(insdel) else 0, len(insdel), marks.ctypes.data if len(marks) else 0, len(marks))
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=dt)
                for a, dt in ((r.actor_off, np.uint64), (r.actor_map, np.uint16), (r.ctr_off, np.uint64), (r.ctr_map, np.uint32), (r.comment_map, np.uint32))]
        ptr = lambda a: None if a is None else a.ctypes.data
        st = _AppendRemap(*[ptr(a) for a in arrs], 0 if arrs[4] is None else len(arrs[4]))
        table = delta.changes if changes is None else changes
        ct = _change_struct(table) if table is not None else None
        _check(self._L.pt_batch_append(self._h, ctypes.byref(ops), ctypes.byref(st), ctypes.byref(ct[0]) if ct else None), "pt_batch_append")
        self._n_insdel += len(insdel)
        self._n_seq += int(desc["n_insdel"].astype(np.uint64).sum())
        self.patch_window = None                                             # so does an append

    def change(self, batch: PackedBatch, inputs, actor_ranks, changes: ChangeTable | None = None):
        """Micromerge.change for many documents on the device (pt_batch_change): ``inputs[i]`` is None (no change) or
        {"seq", "deps", "startOp", "ops": [InputOperation...]} of the change that actor ``batch.log_actors[i][actor_ranks[i]]``
        makes on log i, resolved against the last merge (``batch`` = the batch that merge merged, with its pools and tables).
        ``changes`` is the change table of the new changes, required exactly when the resident batch has one.  Returns
        (the batch the handle now holds = ``apply_append`` of the generated records, the Change objects (None where there is no
        change or it failed), the per-log CHANGE_STATUS_DT rows); a failed log ("List index out of bounds") appends nothing
        and its row names the failing InputOperation.  Needs emit_sequence; the handle needs a merge afterwards."""
        n = batch.n_logs
        actor, off, ops, tokens, values, links, counters = change_inputs(batch, inputs, actor_ranks)
        ptr = lambda a: a.ctypes.data if len(a) else None
        inp = _ChangeInput(n, ptr(actor), ptr(off), ptr(ops), ptr(tokens), len(tokens), len(values), len(links), len(batch.comment_ids), 0)
        ct = _change_struct(changes) if changes is not None else None
        v = _ChangeView()
        _check(self._L.pt_batch_change(self._h, ctypes.byref(inp), ctypes.byref(ct[0]) if ct else None, ctypes.byref(v)), "pt_batch_change")

        def arr(p, count, dt):
            if not count or not p:
                return np.zeros(0, dt)
            return np.frombuffer((ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(p), dtype=dt, count=count).copy()
        status = arr(v.status, n, CHANGE_STATUS_DT)
        desc = arr(v.delta.logs, n, DESC_DT)
        failed = [i for i in range(n) if int(status[i]["status"]) != CHANGE_OK]
        for i in failed:                                 # no records: the counter table stays as it was
            counters[i] = batch.log_counters[i] if batch.log_counters else None
        dch = None
        if changes is not None:
            cd = changes.desc.copy()
            cd["n_changes"][failed] = 0; cd["n_deps"][failed] = 0
            dch = ChangeTable(cd, changes.changes, changes.deps)
        delta = PackedBatch(desc, arr(v.delta.insdel, int(v.delta.n_insdel_total), INSDEL_DT), arr(v.delta.marks, int(v.delta.n_mark_total), MARK_DT),
                            values, links, batch.comment_ids, batch.other_attrs, dict(batch.meta), list(batch.log_actors), counters, dch,
                            list(batch.log_lists))
        self._n_insdel += int(desc["n_insdel"].astype(np.uint64).sum())
        self._n_seq += int(desc["n_insdel"].astype(np.uint64).sum())
        self.patch_window = None                                             # the append resets the window
        return apply_append(batch, delta), change_dicts(batch, inputs, actor_ranks, status, delta), status

    def exchange(self, pairs, maps: ExchangeMaps):
        """Sync between logs of the resident batch on the device (pt_batch_exchange): for every (src, dst) of `pairs` (a list of
        tuples or an (n, 2) array), log dst receives the changes it is missing from log src, in the reference's
        getMissingChanges / applyChanges order, all pairs reading the batch as it is before the call.  `maps` comes from
        ``packing.exchange_maps``, after its pre-append if it returned one.  Returns (per-pair status EXCHANGE_*, the delivered
        indices into each src's change table in delivery order as (u64 offsets [n_pairs + 1], u32 indices), the DESC_DT delta:
        per log the records it received, its n_actors and new max_ctr).  The handle then holds ``packing.apply_exchange`` of
        the batch and needs a merge; a log's old n_insdel + n_mark as its patch window gives the Patches applyChanges
        returned.  Needs a change table."""
        a = np.asarray(pairs, np.int64).reshape(-1, 2)
        pr = np.zeros(len(a), PAIR_DT)
        pr["src"], pr["dst"] = a[:, 0], a[:, 1]
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=dt)
                for a, dt in ((maps.actor_off, np.uint64), (maps.actor_map, np.uint16), (maps.ctr_off, np.uint64), (maps.ctr_map, np.uint32))]
        ptr = lambda a: None if a is None or not len(a) else a.ctypes.data
        inp = _ExchangeInput(len(pr), ptr(pr), *[ptr(a) for a in arrs])
        v = _ExchangeView()
        _check(self._L.pt_batch_exchange(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_exchange")

        def arr(p, count, dt):
            if not count or not p:
                return np.zeros(0, dt)
            return np.frombuffer((ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(p), dtype=dt, count=count).copy()
        status = arr(v.status, v.n_pairs, np.uint32)
        off = arr(v.delivered_off, v.n_pairs + 1, np.uint64)
        flat = arr(v.delivered, int(off[-1]) if len(off) else 0, np.uint32)
        desc = arr(v.delta, self.n_logs, DESC_DT)
        got = int(desc["n_insdel"].astype(np.uint64).sum())
        self._n_insdel += got
        self._n_seq += got
        self.patch_window = None                                             # the splice resets the window
        return status, (off, flat), desc

    def upload_actors(self, batch_or_pools):
        """Attach the per-log actor ids (pt_batch_upload_actors): a PackedBatch (its ``string_pools``) or a dict with the keys
        actors / actors_off / actors_first and optionally counters_first (``packing.string_pools``, or pt_ingest_pool kinds 4
        and 5).  Every upload and any append that can change a log's actors drop them."""
        p = string_pools(batch_or_pools) if isinstance(batch_or_pools, PackedBatch) else batch_or_pools
        data = np.ascontiguousarray(p["actors"], np.uint8)
        off = np.ascontiguousarray(p["actors_off"], np.uint64)
        first = np.ascontiguousarray(p["actors_first"], np.uint64)
        cf = p.get("counters_first")
        cf = None if cf is None else np.ascontiguousarray(cf, np.uint64)
        t = _ActorTables(len(first) - 1 if len(first) else 0, data.ctypes.data if len(data) else None, off.ctypes.data if len(off) else None,
                         max(0, len(off) - 1), first.ctypes.data if len(first) else None, None if cf is None else cf.ctypes.data)
        _check(self._L.pt_batch_upload_actors(self._h, ctypes.byref(t)), "pt_batch_upload_actors")

    def actors(self) -> list[list[str]]:
        """The handle's actor tables (pt_batch_download_actors), per log its ids in rank order."""
        t = _ActorTables()
        _check(self._L.pt_batch_download_actors(self._h, ctypes.byref(t)), "pt_batch_download_actors")
        off = _view_array(t.off, int(t.count) + 1, np.uint64)
        first = _view_array(t.per_log_first, t.n_logs + 1, np.uint64)
        data = _view_array(t.data, int(off[-1]) if len(off) else 0, np.uint8).tobytes()
        ids = [data[int(off[k]): int(off[k + 1])].decode("utf-16-le", "surrogatepass") for k in range(int(t.count))]
        return [ids[int(first[i]): int(first[i + 1])] for i in range(t.n_logs)]

    def add_actors(self, names):
        """Introduce actor ids per log on the device (pt_batch_add_actors): ``names[i]`` = ids for log i, in any order.  Returns
        (per log the rank of each given id afterwards, the per-log old -> new actor maps as (u64 offsets [n_logs + 1], u16
        maps)).  The handle then holds what ``packing.add_actors`` specifies; where a rank moved or an n_actors grew, the
        records were spliced and the batch needs a merge."""
        enc = [x.encode("utf-16-le", "surrogatepass") for ids in names for x in ids]
        data = np.frombuffer(b"".join(enc), np.uint8) if enc else np.zeros(0, np.uint8)
        off = np.zeros(len(enc) + 1, np.uint64)
        off[1:] = np.cumsum([len(x) for x in enc])
        first = np.zeros(len(names) + 1, np.uint64)
        first[1:] = np.cumsum([len(ids) for ids in names])
        inp = _ActorInput(len(names), data.ctypes.data if len(data) else None, off.ctypes.data, len(enc), first.ctypes.data)
        v = _ActorView()
        _check(self._L.pt_batch_add_actors(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_add_actors")
        rank = _view_array(v.rank, int(v.count), np.uint16)
        aoff = _view_array(v.actor_off, self.n_logs + 1, np.uint64)
        amap = _view_array(v.actor_map, int(aoff[-1]) if len(aoff) else 0, np.uint16)
        if v.spliced:
            self.patch_window = None                                         # the splice resets the window
        return [rank[int(first[i]): int(first[i + 1])].tolist() for i in range(len(names))], (aoff, amap)

    def sync_pairs(self, pairs):
        """``exchange`` with the maps and the pre-append derived on the device from the actor tables (pt_batch_sync_pairs):
        only the pairs cross PCIe.  Returns (per-pair status, EXCHANGE_DENSE included, the delivered indices as (offsets,
        indices), the DESC_DT delta, the pre-append's per-log actor maps as (u64 offsets [n_logs + 1], u16 maps)).  The
        handle then holds what ``packing.sync_maps`` specifies and needs a merge."""
        a = np.asarray(pairs, np.int64).reshape(-1, 2)
        pr = np.zeros(len(a), PAIR_DT)
        pr["src"], pr["dst"] = a[:, 0], a[:, 1]
        v = _SyncView()
        _check(self._L.pt_batch_sync_pairs(self._h, pr.ctypes.data if len(pr) else None, len(pr), ctypes.byref(v)), "pt_batch_sync_pairs")
        status = _view_array(v.status, v.n_pairs, np.uint32)
        off = _view_array(v.delivered_off, v.n_pairs + 1, np.uint64)
        flat = _view_array(v.delivered, int(off[-1]) if len(off) else 0, np.uint32)
        desc = _view_array(v.delta, self.n_logs, DESC_DT)
        aoff = _view_array(v.actor_off, self.n_logs + 1, np.uint64)
        amap = _view_array(v.actor_map, int(aoff[-1]) if len(aoff) else 0, np.uint16)
        got = int(desc["n_insdel"].astype(np.uint64).sum())
        self._n_insdel += got
        self._n_seq += got
        self.patch_window = None                                             # the splices reset the window
        return status, (off, flat), desc, (aoff, amap)

    def upload_compact(self, batch: PackedBatch, cins: np.ndarray | None = None, cmarks: np.ndarray | None = None, threads: int = 0):
        """Upload in the compact wire format (8-byte ins/del, 16-byte mark records; expanded on the device): the conversion
        (pt_compact_ops, multithreaded) writes into `cins` / `cmarks` (INSDEL_C8_DT / MARK_C16_DT arrays, ideally pinned)."""
        desc = np.ascontiguousarray(batch.desc)
        insdel = np.ascontiguousarray(batch.insdel); marks = np.ascontiguousarray(batch.marks)
        if cins is None:
            cins = np.zeros(max(1, len(insdel)), INSDEL_C8_DT)
        if cmarks is None:
            cmarks = np.zeros(max(1, len(marks)), MARK_C16_DT)
        ops = self._ops_struct(desc, insdel.ctypes.data, len(insdel), marks.ctypes.data, len(marks))
        _check(self._L.pt_compact_ops(ctypes.byref(ops), cins.ctypes.data, cmarks.ctypes.data, threads), "pt_compact_ops")
        cc = _PackedOps(len(desc), desc.ctypes.data, cins.ctypes.data, len(insdel), cmarks.ctypes.data, len(marks))     # same field layout as pt_packed_compact
        self._keep = (desc, cins, cmarks)
        _check(self._L.pt_batch_upload_compact(self._h, ctypes.byref(cc)), "pt_batch_upload_compact")
        self._uploaded(desc, len(insdel))

    def upload_runs(self, r: PackedRuns):
        desc = np.ascontiguousarray(r.desc)
        st = _PackedRuns(len(desc), desc.ctypes.data, r.run_off.ctypes.data, r.tok_off.ctypes.data, r.runs.ctypes.data if len(r.runs) else 0,
                         r.tokens.ctypes.data if len(r.tokens) else 0, r.marks.ctypes.data if len(r.marks) else 0, r.n_insdel_total, len(r.marks))
        self._keep = (desc, r)
        _check(self._L.pt_batch_upload_runs(self._h, ctypes.byref(st)), "pt_batch_upload_runs")
        self._uploaded(desc, r.n_insdel_total)

    def adopt_device(self, desc: np.ndarray, insdel_dev_ptr: int, n_insdel: int, marks_dev_ptr: int, n_mark: int):
        """Use op arrays already resident in device memory (e.g. ``tensor.data_ptr()``); caller keeps them alive."""
        desc = np.ascontiguousarray(desc)
        ops = self._ops_struct(desc, insdel_dev_ptr, n_insdel, marks_dev_ptr, n_mark)
        _check(self._L.pt_batch_adopt_device(self._h, ctypes.byref(ops)), "pt_batch_adopt_device")
        self._uploaded(desc, n_insdel)

    def merge(self):
        _check(self._L.pt_batch_merge(self._h), "pt_batch_merge")

    def sync(self):
        _check(self._L.pt_batch_sync(self._h), "pt_batch_sync")

    @property
    def last_merge_ms(self) -> float:
        return float(self._L.pt_batch_last_merge_ms(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._L.pt_batch_launch_count(self._h))

    def stats(self) -> dict:
        out = (ctypes.c_uint64 * 4)()
        _check(self._L.pt_batch_stats(self._h, ctypes.byref(out)), "pt_batch_stats")
        return {"logs_shared_only": int(out[0]), "logs_spill_path": int(out[1]), "logs_deferred_to_big_bin": int(out[2]),
                "comment_pool_needed": int(out[3])}

    def device_results_ptr(self) -> int:
        p = ctypes.c_void_p(); n = ctypes.c_uint32()
        _check(self._L.pt_batch_device_results(self._h, ctypes.byref(p), ctypes.byref(n)), "pt_batch_device_results")
        return int(p.value or 0)

    def results(self) -> np.ndarray:
        out = np.zeros(self.n_logs, RESULT_DT)
        _check(self._L.pt_batch_download_results(self._h, out.ctypes.data, self.n_logs), "pt_batch_download_results")
        return out

    def download_begin(self):
        _check(self._L.pt_batch_download_begin(self._h), "pt_batch_download_begin")

    def download(self, copy: bool = True) -> MergedBatch:
        v = _SpansView()
        _check(self._L.pt_batch_download(self._h, ctypes.byref(v)), "pt_batch_download")
        n = v.n_logs

        def arr(ptr, count, dt):
            if not count:
                return np.zeros(0, dt)
            buf = (ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(ptr)
            a = np.frombuffer(buf, dtype=dt, count=count)
            return a.copy() if copy else a

        results = arr(v.results, n, RESULT_DT)
        text_off = arr(v.text_off, n + 1, np.uint64)      # packed on the device: offsets are the scan of the counts
        span_off = arr(v.span_off, n + 1, np.uint64)
        n_text, n_span = int(text_off[-1]), int(span_off[-1])
        seq_off = arr(v.seq_off, n, np.uint64) if (n and v.seq) else None
        n_seq = self._n_seq if seq_off is not None else 0      # (a failed log's n_elems is no element count)
        self.comment_pool_needed = int(v.comment_pool_needed)
        self.comment_pool_used = int(v.comment_pool_used)
        return MergedBatch(results, text_off, span_off, arr(v.text, n_text, np.uint32), arr(v.spans, n_span, SPAN_DT),
                           arr(v.comment_pool, int(v.comment_pool_used), np.uint32),
                           arr(v.seq, n_seq, np.uint32) if v.seq else None, seq_off)

    def download_patches(self):
        """PT_FLAG_EMIT_PATCHES: (patch records per ins/del record, pool items, per-log status, items needed) of the last merge."""
        v = _PatchView()
        _check(self._L.pt_batch_download_patches(self._h, ctypes.byref(v)), "pt_batch_download_patches")

        def arr(ptr, count, dt):
            if not count or not ptr:
                return np.zeros(0, dt)
            buf = (ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(ptr)
            return np.frombuffer(buf, dtype=dt, count=count).copy()
        return arr(v.recs, self._n_insdel, PATCH_REC_DT), arr(v.items, int(v.n_items), PATCH_ITEM_DT), arr(v.status, self.n_logs, np.uint32), int(v.n_items_needed)

    def set_patch_window(self, first_ops=None):
        """Restrict the Patch stream of the following merges to a suffix of every log's list ops (pt_batch_set_patch_window):
        `first_ops[i]` is the position of log i's first op inside the window, in arrival order of the log's list ops (the
        order of ``packing.list_ops`` / the patch JSON); None = whole logs.  After ``append``, the old n_insdel + n_mark of
        each log gives exactly the new changes' ops.  Uploads and appends reset it; setting it after a merge makes that merge's
        patches unavailable until the next merge."""
        if first_ops is None:
            _check(self._L.pt_batch_set_patch_window(self._h, None, self.n_logs), "pt_batch_set_patch_window")
            self.patch_window = None
            return
        w = np.ascontiguousarray(first_ops, dtype=np.uint32)
        _check(self._L.pt_batch_set_patch_window(self._h, w.ctypes.data if len(w) else None, len(w)), "pt_batch_set_patch_window")
        self.patch_window = w.copy()

    def run_with_patches(self, batch: PackedBatch, first_ops=None):
        """upload -> merge (+ device Patch stream) -> download; returns (MergedBatch, DevicePatches).  `first_ops`: the
        patch window of the merge (see ``set_patch_window``), carried into the DevicePatches."""
        if first_ops is None:
            out = self.run(batch)
        else:
            self.upload(batch)
            if getattr(batch, "changes", None) is not None:
                self.upload_changes(batch.changes)
            self.set_patch_window(first_ops)
            self.merge()
            out = self._download_with_pool_retry()
        recs, items, status, needed = self.download_patches()
        if needed > len(items):
            _check(self._L.pt_batch_set_patch_pool(self._h, needed + 16), "pt_batch_set_patch_pool")
            self.merge(); out = self.download()
            recs, items, status, needed = self.download_patches()
        from .packing import DevicePatches
        return out, DevicePatches(recs, items, status, self.patch_window)

    def query_elements(self, logs, indices, look_after_tombstones=False) -> np.ndarray:
        """Batched getListElementId on the device (reference src/micromerge.ts:762-805): for query k the index of the insert
        record of log `logs[k]`'s `indices[k]`-th visible element (with `look_after_tombstones`: moved to the last following
        tombstone whose after-slot is defined, the rule `change()` uses for insert positions); 0xFFFFFFFF = out of bounds.
        Needs emit_sequence and a completed merge."""
        q = np.zeros(len(logs), QUERY_DT)
        q["log"], q["index"] = logs, indices
        q["flags"] = np.asarray(look_after_tombstones, dtype=np.uint32) if not np.isscalar(look_after_tombstones) else (1 if look_after_tombstones else 0)
        out = np.zeros(len(q), np.uint32)
        _check(self._L.pt_batch_query_elements(self._h, q.ctypes.data, len(q), out.ctypes.data), "pt_batch_query_elements")
        return out

    def find_elements(self, logs, ctrs, actors) -> np.ndarray:
        """Batched findListElement on the device (reference src/micromerge.ts:731-755): for query k the element of log
        `logs[k]` whose insert has the packed opId (`ctrs[k]`, `actors[k]`) (see ``packing.elem_refs``).  Returns ELEM_POS_DT
        rows: `index` in the element sequence incl. tombstones, `visible` = non-deleted elements before it (resolveCursor),
        `record` = its insert record in the log, `flags` = ELEM_DELETED | ELEM_AFTER_DEFINED | ELEM_LOG_FAILED;
        index = record = ELEM_NOT_FOUND where no insert of the log has that opId.  Needs emit_sequence and a completed merge."""
        q = np.zeros(len(logs), ELEM_REF_DT)
        q["log"], q["ctr"], q["actor"] = logs, ctrs, actors
        out = np.zeros(len(q), ELEM_POS_DT)
        _check(self._L.pt_batch_find_elements(self._h, q.ctypes.data, len(q), out.ctypes.data), "pt_batch_find_elements")
        return out

    def resolve_cursors(self, batch: PackedBatch, logs, elem_ids) -> np.ndarray:
        """resolveCursor (reference src/micromerge.ts:475-477) for many documents in one device pass: the number of visible
        elements before the element `elem_ids[k]` ("ctr@actor") of the merged log `logs[k]` of `batch` (the batch of the
        last merge), or -1 where the reference throws "List element not found"."""
        refs, ok = elem_refs(batch, logs, elem_ids)
        out = np.full(len(refs), -1, np.int64)
        if ok.any():
            pos = self.find_elements(refs["log"][ok], refs["ctr"][ok], refs["actor"][ok])
            out[ok] = np.where(pos["index"] != ELEM_NOT_FOUND, pos["visible"].astype(np.int64), -1)
        return out

    def _render(self, entry: str, batch: PackedBatch, pools) -> tuple[np.ndarray, np.ndarray]:
        from .packing import json_pools
        p = json_pools(batch) if pools is None else pools
        arrs = [np.ascontiguousarray(a, dtype=np.uint8 if k % 2 == 0 else np.uint64) for k, a in enumerate(p)]
        ptr = lambda a: a.ctypes.data if a.size else None
        st = _JsonPools(ptr(arrs[0]), ptr(arrs[1]), max(0, len(arrs[1]) - 1), ptr(arrs[2]), ptr(arrs[3]), max(0, len(arrs[3]) - 1),
                        ptr(arrs[4]), ptr(arrs[5]), max(0, len(arrs[5]) - 1))
        v = _JsonView()
        _check(getattr(self._L, entry)(self._h, ctypes.byref(st), ctypes.byref(v)), entry)
        off = np.frombuffer((ctypes.c_char * ((v.n_logs + 1) * 8)).from_address(v.off), np.uint64).copy()
        data = np.frombuffer((ctypes.c_char * v.n_bytes).from_address(v.bytes), np.uint8).copy() if v.n_bytes else np.zeros(0, np.uint8)
        return data, off

    @staticmethod
    def _split(data: np.ndarray, off: np.ndarray) -> list[bytes]:
        raw = data.tobytes()
        return [raw[int(off[i]): int(off[i + 1])] for i in range(len(off) - 1)]

    def render_json(self, batch: PackedBatch, pools=None) -> tuple[np.ndarray, np.ndarray]:
        """getTextWithFormatting's return value of every log of the last merge as UTF-8 JSON text, rendered on the device
        (pt_batch_render_json): (uint8 bytes, uint64 offsets [n_logs + 1]); log i is bytes[off[i]:off[i+1]], empty for a log
        that did not merge.  `pools` = (values, values_off, links, links_off, comments, comments_off), default
        ``packing.json_pools(batch)`` of the merged batch."""
        return self._render("pt_batch_render_json", batch, pools)

    def render_json_list(self, batch: PackedBatch, pools=None) -> list[bytes]:
        """``render_json`` as one bytes object per log."""
        return self._split(*self.render_json(batch, pools))

    def render_patches_json(self, batch: PackedBatch, pools=None) -> tuple[np.ndarray, np.ndarray]:
        """The Patch[] that applyChange returned for every list op of every log of the last merge, as UTF-8 JSON text rendered
        on the device (pt_batch_render_patches_json; needs emit_patches): (uint8 bytes, uint64 offsets [n_logs + 1]); log i is
        bytes[off[i]:off[i+1]], one inner array per list op in arrival order, empty for a log that did not merge or whose
        patches were not computed on the device.  `pools` as for ``render_json``."""
        return self._render("pt_batch_render_patches_json", batch, pools)

    def render_patches_json_list(self, batch: PackedBatch, pools=None) -> list[bytes]:
        """``render_patches_json`` as one bytes object per log."""
        return self._split(*self.render_patches_json(batch, pools))

    def render_changes_json(self, batch: PackedBatch, requests, extras: ChangeExtras | None = None, pools=None):
        """Change objects of resident logs as UTF-8 JSON text rendered on the device (pt_batch_render_changes_json; needs a change
        table, no merge).  ``requests``: a CHANGES_REQUEST_DT array of RANGE requests (``packing.range_requests``), or the
        (requests, CLOCK_DT clock) pair of ``packing.clock_requests``.  ``batch`` = the batch the handle holds (its actor, counter
        and list-id tables); ``extras`` = the ``ChangeExtras`` of its changes (None: the list-op projection); ``pools`` as for
        ``render_json``.  Returns (uint8 bytes, uint64 offsets [n_requests + 1], uint32 status per request): request r is
        bytes[off[r]:off[r+1]], a Change[] array, empty for a request whose status is not CHANGES_OK."""
        from .packing import json_pools, string_pools
        req, clock = requests if isinstance(requests, tuple) else (requests, np.zeros(0, CLOCK_DT))
        req = np.ascontiguousarray(req, CHANGES_REQUEST_DT); clock = np.ascontiguousarray(clock, CLOCK_DT)
        p = json_pools(batch) if pools is None else pools
        jp = [np.ascontiguousarray(a, dtype=np.uint8 if k % 2 == 0 else np.uint64) for k, a in enumerate(p)]
        sp = string_pools(batch)
        ex = extras if extras is not None else ChangeExtras(np.zeros(0, EXTRA_DT), [])
        rows = np.ascontiguousarray(ex.rows, EXTRA_DT)
        xdata, xoff = ex.pools()
        keep = [req, clock, jp, sp, rows, xdata, xoff]
        ptr = lambda a: a.ctypes.data if a.size else None
        st = _JsonPools(ptr(jp[0]), ptr(jp[1]), max(0, len(jp[1]) - 1), ptr(jp[2]), ptr(jp[3]), max(0, len(jp[3]) - 1),
                        ptr(jp[4]), ptr(jp[5]), max(0, len(jp[5]) - 1))
        inp = _ChangesJsonInput(len(req), 0, ptr(req), ptr(clock), len(clock), st, ptr(sp["actors"]), ptr(sp["actors_off"]), ptr(sp["actors_first"]),
                                ptr(sp["counters"]), ptr(sp["counters_first"]), ptr(sp["list_ids"]), ptr(sp["list_ids_off"]),
                                ptr(rows), len(rows), ptr(xdata), ptr(xoff), len(ex.ops))
        v = _ChangesJsonView()
        _check(self._L.pt_batch_render_changes_json(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_render_changes_json")
        del keep
        nr = len(req)
        off = np.frombuffer((ctypes.c_char * ((nr + 1) * 8)).from_address(v.off), np.uint64).copy()
        data = np.frombuffer((ctypes.c_char * v.n_bytes).from_address(v.bytes), np.uint8).copy() if v.n_bytes else np.zeros(0, np.uint8)
        status = np.frombuffer((ctypes.c_char * (nr * 4)).from_address(v.status), np.uint32).copy() if nr else np.zeros(0, np.uint32)
        return data, off, status

    def render_changes_json_list(self, batch: PackedBatch, requests, extras: ChangeExtras | None = None, pools=None) -> list[bytes]:
        """``render_changes_json`` as one bytes object per request."""
        data, off, _ = self.render_changes_json(batch, requests, extras, pools)
        return self._split(data, off)

    def set_comment_pool(self, entries: int):
        _check(self._L.pt_batch_set_comment_pool(self._h, int(entries)), "pt_batch_set_comment_pool")

    def run(self, batch: PackedBatch) -> MergedBatch:
        """upload -> merge -> download.  The comment pool has a default capacity; a log whose comment lists do not fit
        reports status 4 without consuming pool space and the engine reports the batch's exact demand, so one re-merge
        with a pool of that size always succeeds (documents with many overlapping comments are valid input)."""
        self.upload(batch)
        if getattr(batch, "changes", None) is not None:
            self.upload_changes(batch.changes)
        self.merge()
        return self._download_with_pool_retry()

    def _download_with_pool_retry(self, copy: bool = True) -> MergedBatch:
        """download, and if some log overflowed the comment pool (status 4), one re-merge with a pool of the reported demand."""
        out = self.download(copy=copy)
        if len(out.results) and (out.results["status"] == 4).any() and self.comment_pool_needed > self.comment_pool_used:
            self.set_comment_pool(self.comment_pool_needed + 16)
            self.merge(); out = self.download(copy=copy)
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.pt_batch_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PipelinedEngine:
    """Host <-> device pipelining for one big batch: the batch is cut into `chunks` runs of logs, each with its own
    engine handle and CUDA stream, so chunk k+1's upload overlaps chunk k's merge and chunk k-1's download (separate
    copy engines).  Inputs should live in pinned host memory (otherwise the uploads synchronise)."""

    def __init__(self, device: int = 0, chunks: int = 4, streams=None):
        self.chunks = chunks
        self._streams = streams
        if streams is None:
            import torch
            self._streams = [torch.cuda.Stream(device=device) for _ in range(chunks)]
        self.engines = [BatchEngine(device, stream=s.cuda_stream) for s in self._streams]

    def _compact_buffers(self, k: int, n_ins: int, n_mk: int):
        """Pinned conversion targets of chunk k (allocated once, grown on demand)."""
        import torch
        if not hasattr(self, "_cbuf"):
            self._cbuf = {}
        cur = self._cbuf.get(k)
        if cur is None or cur[0].numel() < n_ins * 8 or cur[1].numel() < n_mk * 16:
            cur = (torch.empty(max(16, n_ins * 8 + n_ins), dtype=torch.uint8).pin_memory(), torch.empty(max(16, n_mk * 16 + n_mk), dtype=torch.uint8).pin_memory())
            self._cbuf[k] = cur
        return cur[0].numpy()[: n_ins * 8].view(INSDEL_C8_DT), cur[1].numpy()[: n_mk * 16].view(MARK_C16_DT)

    def run(self, batch, copy: bool = False, compact: bool = False, threads: int = 0) -> list[MergedBatch]:
        """`batch`: a PackedBatch, or a PackedRuns (run-compressed upload).  `compact`: convert every chunk to the compact wire
        format on the host (multithreaded, inside this call) and upload half the bytes; chunk k+1's conversion overlaps
        chunk k's transfer.  Like ``BatchEngine.run``, each chunk's change table is attached (admission) and a chunk whose
        comments overflow the default pool is merged once more with a pool of its reported demand."""
        n = batch.n_logs
        # cut by records, not by log count, so the chunks carry similar work
        w = np.cumsum(batch.desc["n_insdel"].astype(np.int64) + 2 * batch.desc["n_mark"].astype(np.int64))
        cuts = [0] + [int(np.searchsorted(w, w[-1] * (k + 1) / self.chunks, side="left")) + 1 for k in range(self.chunks - 1)] + [n] if n else [0, 0]
        cuts = sorted(set(min(max(c, 0), n) for c in cuts))
        subs = [batch.slice_logs(a, b) for a, b in zip(cuts, cuts[1:]) if b > a]
        used = self.engines[: len(subs)]
        for e, sb in zip(used, subs):
            if isinstance(sb, PackedRuns):
                e.upload_runs(sb)
            elif compact:
                ci, cm = self._compact_buffers(used.index(e), len(sb.insdel), len(sb.marks))
                e.upload_compact(sb, ci, cm, threads)
            else:
                e.upload(sb)
            if sb.changes is not None:
                e.upload_changes(sb.changes)
            e.merge(); e.download_begin()
        return [e._download_with_pool_retry(copy=copy) for e in used]

    def close(self):
        for e in self.engines:
            e.close()


def pack_logs_native(logs_json, threads: int = 0) -> PackedBatch:
    """Native (C++, multithreaded) wire-format ingest: ``logs_json[i]`` = JSON text (str or bytes) of the Change objects
    replica i applied, in arrival order -> PackedBatch with its change table (csrc/ingest.cpp, pt_ingest_*).  Packs exactly
    like ``packing.pack_logs(..., with_changes=True)``."""
    return _ingest(logs_json, threads)[0]


def ingest_native(logs_json, threads: int = 0):
    """``pack_logs_native`` plus what ``render_changes_json`` needs to give the logs back exactly: returns (PackedBatch with
    ``log_lists`` set from the list-id pool, its ``ChangeExtras`` (pt_ingest_change_extras and the extra-ops pool), the raw
    pools {kind: (bytes, u64 offsets, u64 per-log first or None)} of every PT_POOL_* kind 0-7)."""
    return _ingest(logs_json, threads, with_extras=True)


def _ingest(logs_json, threads: int = 0, with_extras: bool = False):
    import json
    L = load_library()
    blobs = [s.encode("utf-8", "surrogatepass") if isinstance(s, str) else bytes(s) for s in logs_json]
    n = len(blobs)
    ptrs = (ctypes.c_char_p * max(1, n))(*blobs) if n else (ctypes.c_char_p * 1)()
    lens = (ctypes.c_uint64 * max(1, n))(*[len(b) for b in blobs]) if n else (ctypes.c_uint64 * 1)()
    h = ctypes.c_void_p()
    _check(L.pt_ingest_create(ctypes.byref(h)), "pt_ingest_create")
    try:
        rc = L.pt_ingest_parse(h, ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(lens, ctypes.c_void_p), n, threads)
        if rc != 0:
            raise ValueError(L.pt_ingest_error(h).decode("utf-8", "replace"))
        ops, tab = _PackedOps(), _ChangeTable()
        _check(L.pt_ingest_packed(h, ctypes.byref(ops), ctypes.byref(tab)), "pt_ingest_packed")

        def arr(ptr, count, dt):
            if not count or not ptr:
                return np.zeros(0, dt)
            buf = (ctypes.c_char * (count * np.dtype(dt).itemsize)).from_address(ptr)
            return np.frombuffer(buf, dtype=dt, count=count).copy()

        def pool(kind):
            data, off, cnt, first = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_void_p()
            _check(L.pt_ingest_pool(h, kind, ctypes.byref(data), ctypes.byref(off), ctypes.byref(cnt), ctypes.byref(first)), "pt_ingest_pool")
            o = arr(off.value, cnt.value + 1, np.uint64)
            raw = bytes(arr(data.value, int(o[-1]), np.uint8)) if cnt.value else b""
            items = [raw[int(o[k]): int(o[k + 1])] for k in range(cnt.value)]
            f = arr(first.value, n + 1, np.uint64) if first.value else None
            return items, f

        u16 = lambda b: b.decode("utf-16-le", "surrogatepass")
        values = [u16(b) for b in pool(0)[0]]
        link_attrs = [json.loads(b.decode("utf-8", "surrogatepass")) for b in pool(1)[0]]
        comment_attrs = [json.loads(b.decode("utf-8", "surrogatepass")) for b in pool(3)[0]]
        actors, afirst = pool(4)
        counters, cfirst = pool(5)
        log_actors = [[u16(x) for x in actors[int(afirst[i]): int(afirst[i + 1])]] for i in range(n)]
        log_counters = []
        for i in range(n):
            c = counters[int(cfirst[i]): int(cfirst[i + 1])]
            log_counters.append(np.array([int.from_bytes(x, "little") for x in c], dtype=np.uint64) if c else None)
        table = ChangeTable(arr(tab.logs, tab.n_logs, CDESC_DT), arr(tab.changes, tab.n_changes_total, CHANGE_DT), arr(tab.deps, tab.n_deps_total, DEP_DT))
        batch = PackedBatch(arr(ops.logs, ops.n_logs, DESC_DT), arr(ops.insdel, ops.n_insdel_total, INSDEL_DT), arr(ops.marks, ops.n_mark_total, MARK_DT),
                            values, link_attrs, comment_attrs, [], log_actors=log_actors, log_counters=log_counters, changes=table)
        if not with_extras:
            return batch, None, None
        raw = {}
        for kind in range(8):
            data, off, cnt, first = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_void_p()
            _check(L.pt_ingest_pool(h, kind, ctypes.byref(data), ctypes.byref(off), ctypes.byref(cnt), ctypes.byref(first)), "pt_ingest_pool")
            o = arr(off.value, cnt.value + 1, np.uint64)
            raw[kind] = (bytes(arr(data.value, int(o[-1]), np.uint8)) if cnt.value else b"", o, arr(first.value, n + 1, np.uint64) if first.value else None)
        batch.log_lists = [u16(x) or None for x in pool(6)[0]]
        xp, xn = ctypes.c_void_p(), ctypes.c_uint64()
        _check(L.pt_ingest_change_extras(h, ctypes.byref(xp), ctypes.byref(xn)), "pt_ingest_change_extras")
        extras = ChangeExtras(arr(xp.value, xn.value, EXTRA_DT), [b.decode("utf-8", "surrogatepass") for b in pool(7)[0]])
        return batch, extras, raw
    finally:
        L.pt_ingest_destroy(h)
