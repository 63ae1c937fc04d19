"""ctypes binding of the engine's C-ABI (include/peritext_b200.h, built as peritext_b200/libperitext_b200.so).

There is no CPU fallback: if the shared library is missing or no CUDA device is usable, every entry point raises
``EngineError``.  torch is not needed here; pass ``torch.cuda.current_stream().cuda_stream`` as ``stream`` to enqueue
on a torch stream.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from .packing import (CDESC_DT, CHANGE_DT, CLOCK_DT, CHANGES_REQUEST_DT, EXTRA_DT, ChangeExtras, CHANGE_OK, CHANGE_STATUS_DT, DEP_DT, DESC_DT, ELEM_NOT_FOUND, ELEM_POS_DT, ELEM_REF_DT,
                      INPUT_OP_DT, INSDEL_DT, MARK_DT, RESULT_DT, SELECT_ADDED, SPAN_DT, AppendRemap, ChangeTable, ExchangeMaps, MergedBatch, PackedBatch, apply_append, change_dicts,
                      change_inputs, elem_refs, json_pools, string_pools)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libperitext_b200.so")
_lib = None

_vp, _u32, _u64, _int, _str, _out = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int, ctypes.c_char_p, ctypes.POINTER
# every export of include/peritext_b200.h: name -> (argtypes, restype); an int restype is a pt_status
_ENTRY_POINTS = {
    "pt_batch_create": ([_int, _vp, _vp, _out(_vp)], _int),
    "pt_batch_upload": ([_vp, _vp], _int),
    "pt_batch_upload_runs": ([_vp, _vp], _int),
    "pt_compress_runs": ([_vp, _vp, _vp, _vp, _vp, _out(_u64), _out(_u64)], _int),
    "pt_compact_ops": ([_vp, _vp, _vp, _int], _int),
    "pt_batch_upload_compact": ([_vp, _vp], _int),
    "pt_batch_adopt_device": ([_vp, _vp], _int),
    "pt_batch_upload_changes": ([_vp, _vp], _int),
    "pt_batch_append": ([_vp, _vp, _vp, _vp], _int),
    "pt_batch_change": ([_vp, _vp, _vp, _vp], _int),
    "pt_batch_exchange": ([_vp, _vp, _vp], _int),
    "pt_batch_upload_actors": ([_vp, _vp], _int),
    "pt_batch_download_actors": ([_vp, _vp], _int),
    "pt_batch_add_actors": ([_vp, _vp, _vp], _int),
    "pt_batch_sync_pairs": ([_vp, _vp, _u32, _vp], _int),
    "pt_batch_select_logs": ([_vp, _vp, _u32, _vp, _vp, _vp, _vp, _u64], _int),
    "pt_batch_checkout": ([_vp, _vp, _u32, _vp, _vp, _vp, _vp], _int),
    "pt_batch_download_clocks": ([_vp, _out(_vp), _out(_vp), _out(_vp)], _int),
    "pt_batch_download_descs": ([_vp, _out(_vp)], _int),
    "pt_ingest_create": ([_out(_vp)], _int),
    "pt_ingest_parse": ([_vp, _vp, _vp, _u32, _int], _int),
    "pt_ingest_packed": ([_vp, _vp, _vp], _int),
    "pt_ingest_pool": ([_vp, _int, _out(_vp), _out(_vp), _out(_u64), _out(_vp)], _int),
    "pt_ingest_error": ([_vp], _str),
    "pt_ingest_destroy": ([_vp], None),
    "pt_batch_merge": ([_vp], _int),
    "pt_batch_sync": ([_vp], _int),
    "pt_batch_download": ([_vp, _vp], _int),
    "pt_batch_download_begin": ([_vp], _int),
    "pt_batch_download_results": ([_vp, _vp, _u32], _int),
    "pt_batch_device_results": ([_vp, _out(_vp), _out(_u32)], _int),
    "pt_batch_launch_count": ([_vp], _u64),
    "pt_batch_stats": ([_vp, _out(_u64 * 4)], _int),
    "pt_batch_last_merge_ms": ([_vp], ctypes.c_float),
    "pt_batch_set_comment_pool": ([_vp, _u64], _int),
    "pt_batch_download_patches": ([_vp, _vp], _int),
    "pt_batch_set_patch_pool": ([_vp, _u64], _int),
    "pt_batch_set_patch_window": ([_vp, _vp, _u32], _int),
    "pt_batch_query_elements": ([_vp, _vp, _u32, _vp], _int),
    "pt_batch_find_elements": ([_vp, _vp, _u32, _vp], _int),
    "pt_batch_attribute": ([_vp, _vp, _u32, _vp, _vp, _vp], _int),
    "pt_batch_restore": ([_vp, _vp, _u32, _u32, _vp], _int),
    "pt_batch_render_json": ([_vp, _vp, _vp], _int),
    "pt_batch_render_patches_json": ([_vp, _vp, _vp], _int),
    "pt_batch_render_changes_json": ([_vp, _vp, _vp], _int),
    "pt_ingest_change_extras": ([_vp, _out(_vp), _out(_u64)], _int),
    "pt_batch_destroy": ([_vp], None),
    "pt_strerror": ([_int], _str),
    "pt_last_error": ([], _str),
    "pt_version": ([], _str),
}
EXPORTS = list(_ENTRY_POINTS)


class EngineError(RuntimeError):
    """A failed engine call; ``status`` is the pt_status code it returned (None when no call was made)."""

    def __init__(self, message: str, status: int | None = None):
        super().__init__(message)
        self.status = status


def _ptr(a):
    """The data pointer of a numpy array, or NULL (None) for None or an empty array."""
    return None if a is None or not a.size else a.ctypes.data


def _view(p, count, dt, copy: bool = True) -> np.ndarray:
    """`count` elements of dtype `dt` at address `p` (memory a native library owns): a copy, or with ``copy=False`` a zero-copy
    array over that memory, valid until the library reuses it.  Empty when `count` is 0 or `p` is NULL."""
    dt, count = np.dtype(dt), int(count)
    if not count or not p:
        return np.zeros(0, dt)
    a = np.frombuffer((ctypes.c_char * (count * dt.itemsize)).from_address(p), dtype=dt, count=count)
    return a.copy() if copy else a


class _PackedOps(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("logs", ctypes.c_void_p), ("insdel", ctypes.c_void_p),
                ("n_insdel_total", ctypes.c_uint64), ("marks", ctypes.c_void_p), ("n_mark_total", ctypes.c_uint64)]


def _packed_ops(desc, insdel, n_insdel, marks, n_mark) -> _PackedOps:
    """pt_packed_ops, and pt_packed_compact (the same layout): `insdel` / `marks` are host arrays or device addresses."""
    p = lambda a: _ptr(a) if isinstance(a, np.ndarray) else a
    return _PackedOps(len(desc), _ptr(desc), p(insdel), n_insdel, p(marks), n_mark)


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
    ops = _packed_ops(desc, insdel, len(insdel), marks, len(marks))
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
    return _ChangeTable(len(d), _ptr(d), _ptr(c), len(c), _ptr(p), len(p)), (d, c, p)


# the map fields of pt_append_remap, in order; pt_exchange_input has the first four
_MAP_FIELDS = (("actor_off", np.uint64), ("actor_map", np.uint16), ("ctr_off", np.uint64), ("ctr_map", np.uint32), ("comment_map", np.uint32))


def _map_arrays(maps: AppendRemap | ExchangeMaps) -> list:
    """The maps of an AppendRemap or ExchangeMaps as typed contiguous arrays (None stays None), in the struct's field order."""
    return [None if getattr(maps, k) is None else np.ascontiguousarray(getattr(maps, k), dt) for k, dt in _MAP_FIELDS if hasattr(maps, k)]


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


def _pairs(pairs) -> np.ndarray:
    """(src, dst) pairs (a list of tuples or an (n, 2) array) as PAIR_DT rows."""
    a = np.asarray(pairs, np.int64).reshape(-1, 2)
    pr = np.zeros(len(a), PAIR_DT)
    pr["src"], pr["dst"] = a[:, 0], a[:, 1]
    return pr


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


def _json_pools(batch: PackedBatch, pools):
    """(pt_json_pools of `pools` (values, values_off, links, links_off, comments, comments_off; default
    ``packing.json_pools(batch)``), the contiguous arrays it points into)."""
    a = [np.ascontiguousarray(x, dtype=np.uint8 if k % 2 == 0 else np.uint64) for k, x in enumerate(json_pools(batch) if pools is None else pools)]
    n = lambda off: max(0, len(off) - 1)
    return _JsonPools(_ptr(a[0]), _ptr(a[1]), n(a[1]), _ptr(a[2]), _ptr(a[3]), n(a[3]), _ptr(a[4]), _ptr(a[5]), n(a[5])), a


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
    for name, (argtypes, restype) in _ENTRY_POINTS.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = argtypes, restype
    _lib = L
    return L


def _check(rc: int, what: str):
    if rc != 0:
        L = load_library()
        raise EngineError(f"{what}: {L.pt_strerror(rc).decode()} ({L.pt_last_error().decode()})", rc)


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
        self._log_insdel = desc["n_insdel"].astype(np.uint64)                # per log, and its n_actors: what a select moves
        self._log_n_actors = desc["n_actors"].astype(np.uint32)
        self._n_seq = int(self._log_insdel.sum())                            # element sequences: the capacity layout
        self._has_changes = self._has_actors = False                         # every upload drops both tables

    _ops_struct = staticmethod(_packed_ops)                                  # the builder under its earlier method name

    def _spliced(self, delta_desc):
        """Record a splice into the resident batch (append, change, exchange, sync, a re-ranking add_actors): the device rebuilds
        the records tightly from the new descriptors, so it then holds exactly their n_insdel sum; a splice also resets the
        patch window."""
        if len(delta_desc):
            self._log_insdel = self._log_insdel + delta_desc["n_insdel"].astype(np.uint64)
            self._log_n_actors = delta_desc["n_actors"].astype(np.uint32)
        self._n_seq = int(self._log_insdel.sum())
        self._n_insdel = self._n_seq
        self.patch_window = None

    def upload(self, batch: PackedBatch):
        desc = np.ascontiguousarray(batch.desc)
        insdel = np.ascontiguousarray(batch.insdel)
        marks = np.ascontiguousarray(batch.marks)
        ops = _packed_ops(desc, insdel, len(insdel), marks, len(marks))
        _check(self._L.pt_batch_upload(self._h, ctypes.byref(ops)), "pt_batch_upload")
        self._uploaded(desc, len(insdel))

    def _upload_with_changes(self, batch, upload=None, *args):
        """``upload(batch, *args)`` (default the plain form), then attach the batch's change table if it has one, so the next
        merge runs the admission pre-pass."""
        (upload or self.upload)(batch, *args)
        if getattr(batch, "changes", None) is not None:
            self.upload_changes(batch.changes)

    def upload_changes(self, table: ChangeTable):
        """Attach the batch's change table: the next merge runs the admission pre-pass (seq / deps checks of
        Micromerge.applyChange, reference src/micromerge.ts:501-509) and rejected logs report status 6 / 7."""
        t, _keep = _change_struct(table)
        _check(self._L.pt_batch_upload_changes(self._h, ctypes.byref(t)), "pt_batch_upload_changes")
        self._has_changes = True

    def append(self, delta: PackedBatch, remap: AppendRemap | None = None, changes: ChangeTable | None = None):
        """Extend every log of the resident batch with the delta's records on the device (pt_batch_append): afterwards the
        handle holds what an upload of ``packing.apply_append(batch, delta, remap)`` would hold, and needs a merge.  `delta`
        and `remap` come from ``packing.pack_append``; `changes` is the delta's change table (default ``delta.changes``),
        required exactly when the resident batch has one.  Works after every upload form and after an earlier append."""
        desc = np.ascontiguousarray(delta.desc)
        insdel = np.ascontiguousarray(delta.insdel); marks = np.ascontiguousarray(delta.marks)
        ops = _packed_ops(desc, insdel, len(insdel), marks, len(marks))
        arrs = _map_arrays(remap or AppendRemap())
        # not _ptr: an empty comment_map is no identity (NULL is), it maps no resident comment rank and the device refuses
        st = _AppendRemap(*[None if a is None else a.ctypes.data for a in arrs], 0 if arrs[4] is None else len(arrs[4]))
        table = delta.changes if changes is None else changes
        ct = _change_struct(table) if table is not None else None
        _check(self._L.pt_batch_append(self._h, ctypes.byref(ops), ctypes.byref(st), ctypes.byref(ct[0]) if ct else None), "pt_batch_append")
        # the engine drops the actor tables where a log's actor set can have changed (pt_batch_upload_actors' lifetime rule)
        if arrs[1] is not None and len(arrs[1]) or arrs[3] is not None and len(arrs[3]) or (desc["n_actors"] != self._log_n_actors).any():
            self._has_actors = False
        self._spliced(desc)

    def select_logs(self, from_, added: PackedBatch | None = None, comment_map=None):
        """Change which logs the resident batch holds, on the device (pt_batch_select_logs): new log i is resident log
        ``from_[i]``, or, where ``from_[i]`` is SELECT_ADDED, the next log of `added` (``packing.pack_select``).  Kept logs keep
        everything they hold on the device; `comment_map` (old comment rank -> new rank, SELECT_DROPPED for a rank no kept log
        names; None = identity) moves their comment ranks.  `added` brings its change table when the handle has one and its
        ``log_actors`` when the handle has actor tables.  The handle then holds what an upload of ``packing.apply_select``
        would hold, and needs a merge."""
        frm = np.ascontiguousarray(from_, np.uint32)
        ops = ct = at = None
        keep = []
        if added is not None:
            desc = np.ascontiguousarray(added.desc)
            insdel = np.ascontiguousarray(added.insdel); marks = np.ascontiguousarray(added.marks)
            ops = _packed_ops(desc, insdel, len(insdel), marks, len(marks))
            keep += [desc, insdel, marks]
            if self._has_changes and added.changes is not None:
                ct, arrs = _change_struct(added.changes)
                keep.append(arrs)
            if self._has_actors:
                p = string_pools(added)
                data, off, first = (np.ascontiguousarray(p[k], dt) for k, dt in (("actors", np.uint8), ("actors_off", np.uint64), ("actors_first", np.uint64)))
                cf = np.ascontiguousarray(p["counters_first"], np.uint64)
                at = _ActorTables(len(desc), _ptr(data), _ptr(off), max(0, len(off) - 1), _ptr(first), _ptr(cf))
                keep += [data, off, first, cf]
        cm = None if comment_map is None else np.ascontiguousarray(comment_map, np.uint32)
        ref = lambda st: ctypes.byref(st) if st is not None else None
        _check(self._L.pt_batch_select_logs(self._h, _ptr(frm), len(frm), ref(ops), ref(ct), ref(at),
                                            None if cm is None else cm.ctypes.data, 0 if cm is None else len(cm)), "pt_batch_select_logs")
        add = added.desc if added is not None else np.zeros(0, DESC_DT)
        kept = frm != SELECT_ADDED
        ins, act = np.zeros(len(frm), np.uint64), np.zeros(len(frm), np.uint32)
        ins[kept], act[kept] = self._log_insdel[frm[kept]], self._log_n_actors[frm[kept]]
        ins[~kept], act[~kept] = add["n_insdel"], add["n_actors"]
        self.n_logs = len(frm)
        self._log_insdel, self._log_n_actors = ins, act
        self._spliced(np.zeros(0, DESC_DT))

    def checkout(self, logs, n_changes=None, clock=None) -> np.ndarray:
        """Fork resident logs at an earlier version, on the device (pt_batch_checkout): request k appends a new log holding log
        ``logs[k]`` at the version of its first ``n_changes[k]`` changes (prefix mode) or of a vector clock (clock mode:
        ``clock`` = (u64 offsets [n + 1], CLOCK_DT entries by actor rank), ``packing.checkout_clocks``).  Exactly one of the two
        is given.  Returns the per-request status CHECKOUT_*; a request that is not OK adds an empty log.  The handle then
        holds what an upload of ``packing.apply_checkout`` would hold, and needs a merge.  Needs a change table."""
        lg = np.ascontiguousarray(logs, np.uint32)
        nch = None if n_changes is None else np.ascontiguousarray(n_changes, np.uint32)
        off = ent = None
        if clock is not None:
            off, ent = np.ascontiguousarray(clock[0], np.uint64), np.ascontiguousarray(clock[1], CLOCK_DT)
        status = np.zeros(len(lg), np.uint32)
        ptr = lambda a: None if a is None else a.ctypes.data                 # not _ptr: an empty array still names its mode
        _check(self._L.pt_batch_checkout(self._h, _ptr(lg), len(lg), ptr(nch), ptr(off), _ptr(ent), _ptr(status)), "pt_batch_checkout")
        if len(lg):
            d = ctypes.c_void_p()
            _check(self._L.pt_batch_download_descs(self._h, ctypes.byref(d)), "pt_batch_download_descs")
            desc = _view(d.value, self.n_logs + len(lg), DESC_DT)
            self.n_logs = len(desc)
            self._log_insdel = desc["n_insdel"].astype(np.uint64)
            self._log_n_actors = desc["n_actors"].astype(np.uint32)
            self._spliced(np.zeros(0, DESC_DT))
        return status

    def clocks(self):
        """Every log's clock (pt_batch_download_clocks): (u64 offsets [n_logs + 1], u32 seq, u32 status), log i's number of
        changes by actor rank a at seq[off[i] + a]; status CHECKOUT_BAD_TABLE (and zeros) where the table is not
        seq-contiguous.  ``packing.clocks`` is its host specification.  Needs a change table."""
        off, seq, st = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        _check(self._L.pt_batch_download_clocks(self._h, ctypes.byref(off), ctypes.byref(seq), ctypes.byref(st)), "pt_batch_download_clocks")
        o = _view(off.value, self.n_logs + 1, np.uint64)
        return o, _view(seq.value, int(o[-1]), np.uint32), _view(st.value, self.n_logs, np.uint32)

    def change_packed(self, actor, input_off, ops, tokens, n_values: int, n_links: int, n_comments: int, changes: ChangeTable | None = None):
        """pt_batch_change from its arrays (``packing.change_inputs``, ``workload.sync_round``): per log i the actor rank of its
        change (CHANGE_NO_ACTOR: none) and its InputOperations ops[input_off[i]:input_off[i + 1]] (INPUT_OP_DT), the value
        tokens they name, and the sizes of the value, link and comment pools their tokens and attrs index.  ``changes`` is the
        change table of the new changes, required exactly when the resident batch has one.  Returns (the per-log
        CHANGE_STATUS_DT rows, the DESC_DT delta, its ins/del records, its mark records); the handle needs a merge afterwards."""
        actor, off = np.ascontiguousarray(actor, np.uint32), np.ascontiguousarray(input_off, np.uint64)
        ops, tokens = np.ascontiguousarray(ops, INPUT_OP_DT), np.ascontiguousarray(tokens, np.uint32)
        n = len(actor)
        inp = _ChangeInput(n, _ptr(actor), _ptr(off), _ptr(ops), _ptr(tokens), len(tokens), n_values, n_links, n_comments, 0)
        ct = _change_struct(changes) if changes is not None else None
        v = _ChangeView()
        _check(self._L.pt_batch_change(self._h, ctypes.byref(inp), ctypes.byref(ct[0]) if ct else None, ctypes.byref(v)), "pt_batch_change")
        desc = _view(v.delta.logs, n, DESC_DT)
        self._spliced(desc)
        return (_view(v.status, n, CHANGE_STATUS_DT), desc, _view(v.delta.insdel, v.delta.n_insdel_total, INSDEL_DT),
                _view(v.delta.marks, v.delta.n_mark_total, MARK_DT))

    def change(self, batch: PackedBatch, inputs, actor_ranks, changes: ChangeTable | None = None):
        """Micromerge.change for many documents on the device (pt_batch_change): ``inputs[i]`` is None (no change) or
        {"seq", "deps", "startOp", "ops": [InputOperation...]} of the change that actor ``batch.log_actors[i][actor_ranks[i]]``
        makes on log i, resolved against the last merge (``batch`` = the batch that merge merged, with its pools and tables).
        ``changes`` is the change table of the new changes, required exactly when the resident batch has one.  Returns
        (the batch the handle now holds = ``apply_append`` of the generated records, the Change objects (None where there is no
        change or it failed), the per-log CHANGE_STATUS_DT rows); a failed log ("List index out of bounds") appends nothing
        and its row names the failing InputOperation.  Needs emit_sequence; the handle needs a merge afterwards."""
        actor, off, ops, tokens, values, links, counters = change_inputs(batch, inputs, actor_ranks)
        status, desc, insdel, marks = self.change_packed(actor, off, ops, tokens, len(values), len(links), len(batch.comment_ids), changes)
        failed = [i for i in range(batch.n_logs) if int(status[i]["status"]) != CHANGE_OK]
        for i in failed:                                 # no records: the counter table stays as it was
            counters[i] = batch.log_counters[i] if batch.log_counters else None
        dch = None
        if changes is not None:
            cd = changes.desc.copy()
            cd["n_changes"][failed] = 0; cd["n_deps"][failed] = 0
            dch = ChangeTable(cd, changes.changes, changes.deps)
        delta = PackedBatch(desc, insdel, marks, values, links, batch.comment_ids, batch.other_attrs, dict(batch.meta), list(batch.log_actors), counters, dch,
                            list(batch.log_lists))
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
        pr = _pairs(pairs)
        inp = _ExchangeInput(len(pr), _ptr(pr), *[_ptr(a) for a in _map_arrays(maps)])
        v = _ExchangeView()
        _check(self._L.pt_batch_exchange(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_exchange")
        return self._delivered(v)

    def _delivered(self, v):
        """(per-pair status, (delivered offsets, indices), DESC_DT delta) of an exchange or sync view; records the splice."""
        status = _view(v.status, v.n_pairs, np.uint32)
        off = _view(v.delivered_off, v.n_pairs + 1, np.uint64)
        flat = _view(v.delivered, off[-1] if len(off) else 0, np.uint32)
        desc = _view(v.delta, self.n_logs, DESC_DT)
        self._spliced(desc)
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
        t = _ActorTables(max(0, len(first) - 1), _ptr(data), _ptr(off), max(0, len(off) - 1), _ptr(first), _ptr(cf))
        _check(self._L.pt_batch_upload_actors(self._h, ctypes.byref(t)), "pt_batch_upload_actors")
        self._has_actors = True

    def actors(self) -> list[list[str]]:
        """The handle's actor tables (pt_batch_download_actors), per log its ids in rank order."""
        t = _ActorTables()
        _check(self._L.pt_batch_download_actors(self._h, ctypes.byref(t)), "pt_batch_download_actors")
        off = _view(t.off, t.count + 1, np.uint64)
        first = _view(t.per_log_first, t.n_logs + 1, np.uint64)
        data = _view(t.data, off[-1] if len(off) else 0, np.uint8).tobytes()
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
        inp = _ActorInput(len(names), _ptr(data), _ptr(off), len(enc), _ptr(first))
        v = _ActorView()
        _check(self._L.pt_batch_add_actors(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_add_actors")
        rank = _view(v.rank, v.count, np.uint16)
        aoff = _view(v.actor_off, self.n_logs + 1, np.uint64)
        amap = _view(v.actor_map, aoff[-1] if len(aoff) else 0, np.uint16)
        if v.spliced:                                                        # re-ranked records, none added
            self._spliced(np.zeros(0, DESC_DT))
        return [rank[int(first[i]): int(first[i + 1])].tolist() for i in range(len(names))], (aoff, amap)

    def sync_pairs(self, pairs):
        """``exchange`` with the maps and the pre-append derived on the device from the actor tables (pt_batch_sync_pairs):
        only the pairs cross PCIe.  Returns (per-pair status, EXCHANGE_DENSE included, the delivered indices as (offsets,
        indices), the DESC_DT delta, the pre-append's per-log actor maps as (u64 offsets [n_logs + 1], u16 maps)).  The
        handle then holds what ``packing.sync_maps`` specifies and needs a merge."""
        pr = _pairs(pairs)
        v = _SyncView()
        _check(self._L.pt_batch_sync_pairs(self._h, _ptr(pr), len(pr), ctypes.byref(v)), "pt_batch_sync_pairs")
        status, delivered, desc = self._delivered(v)
        aoff = _view(v.actor_off, self.n_logs + 1, np.uint64)
        return status, delivered, desc, (aoff, _view(v.actor_map, aoff[-1] if len(aoff) else 0, np.uint16))

    def upload_compact(self, batch: PackedBatch, cins: np.ndarray | None = None, cmarks: np.ndarray | None = None, threads: int = 0):
        """Upload in the compact wire format (8-byte ins/del, 16-byte mark records; expanded on the device): the conversion
        (pt_compact_ops, multithreaded) writes into `cins` / `cmarks` (INSDEL_C8_DT / MARK_C16_DT arrays, ideally pinned)."""
        desc = np.ascontiguousarray(batch.desc)
        insdel = np.ascontiguousarray(batch.insdel); marks = np.ascontiguousarray(batch.marks)
        if cins is None:
            cins = np.zeros(max(1, len(insdel)), INSDEL_C8_DT)
        if cmarks is None:
            cmarks = np.zeros(max(1, len(marks)), MARK_C16_DT)
        ops = _packed_ops(desc, insdel, len(insdel), marks, len(marks))
        _check(self._L.pt_compact_ops(ctypes.byref(ops), _ptr(cins), _ptr(cmarks), threads), "pt_compact_ops")
        cc = _packed_ops(desc, cins, len(insdel), cmarks, len(marks))
        self._keep = (desc, cins, cmarks)
        _check(self._L.pt_batch_upload_compact(self._h, ctypes.byref(cc)), "pt_batch_upload_compact")
        self._uploaded(desc, len(insdel))

    def upload_runs(self, r: PackedRuns):
        desc = np.ascontiguousarray(r.desc)
        st = _PackedRuns(len(desc), _ptr(desc), _ptr(r.run_off), _ptr(r.tok_off), _ptr(r.runs), _ptr(r.tokens), _ptr(r.marks), r.n_insdel_total, len(r.marks))
        self._keep = (desc, r)
        _check(self._L.pt_batch_upload_runs(self._h, ctypes.byref(st)), "pt_batch_upload_runs")
        self._uploaded(desc, r.n_insdel_total)

    def adopt_device(self, desc: np.ndarray, insdel_dev_ptr: int, n_insdel: int, marks_dev_ptr: int, n_mark: int):
        """Use op arrays already resident in device memory (e.g. ``tensor.data_ptr()``); caller keeps them alive."""
        desc = np.ascontiguousarray(desc)
        ops = _packed_ops(desc, insdel_dev_ptr, n_insdel, marks_dev_ptr, n_mark)
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
        _check(self._L.pt_batch_download_results(self._h, _ptr(out), self.n_logs), "pt_batch_download_results")
        return out

    def download_begin(self):
        _check(self._L.pt_batch_download_begin(self._h), "pt_batch_download_begin")

    def download(self, copy: bool = True) -> MergedBatch:
        v = _SpansView()
        _check(self._L.pt_batch_download(self._h, ctypes.byref(v)), "pt_batch_download")
        n = v.n_logs
        arr = lambda p, count, dt: _view(p, count, dt, copy)
        results = arr(v.results, n, RESULT_DT)
        text_off = arr(v.text_off, n + 1, np.uint64)      # packed on the device: offsets are the scan of the counts
        span_off = arr(v.span_off, n + 1, np.uint64)
        n_text, n_span = int(text_off[-1]), int(span_off[-1])
        seq_off = arr(v.seq_off, n, np.uint64) if (n and v.seq) else None
        n_seq = self._n_seq if seq_off is not None else 0      # (a failed log's n_elems is no element count)
        self.comment_pool_needed = int(v.comment_pool_needed)
        self.comment_pool_used = int(v.comment_pool_used)
        return MergedBatch(results, text_off, span_off, arr(v.text, n_text, np.uint32), arr(v.spans, n_span, SPAN_DT),
                           arr(v.comment_pool, v.comment_pool_used, np.uint32),
                           arr(v.seq, n_seq, np.uint32) if v.seq else None, seq_off)

    def download_patches(self):
        """PT_FLAG_EMIT_PATCHES: (patch records per ins/del record, pool items, per-log status, items needed) of the last merge."""
        v = _PatchView()
        _check(self._L.pt_batch_download_patches(self._h, ctypes.byref(v)), "pt_batch_download_patches")
        return _view(v.recs, self._n_insdel, PATCH_REC_DT), _view(v.items, v.n_items, PATCH_ITEM_DT), _view(v.status, self.n_logs, np.uint32), int(v.n_items_needed)

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
        _check(self._L.pt_batch_set_patch_window(self._h, _ptr(w), len(w)), "pt_batch_set_patch_window")
        self.patch_window = w.copy()

    def run_with_patches(self, batch: PackedBatch, first_ops=None):
        """upload -> merge (+ device Patch stream) -> download; returns (MergedBatch, DevicePatches).  `first_ops`: the
        patch window of the merge (see ``set_patch_window``), carried into the DevicePatches."""
        if first_ops is None:
            out = self.run(batch)
        else:
            self._upload_with_changes(batch)
            self.set_patch_window(first_ops)
            self.merge()
            out = self._download_with_pool_retry()
        recs, items, status, needed = self.download_patches()
        if needed > len(items):
            self.set_patch_pool(needed + 16)
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
        _check(self._L.pt_batch_query_elements(self._h, _ptr(q), len(q), _ptr(out)), "pt_batch_query_elements")
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
        _check(self._L.pt_batch_find_elements(self._h, _ptr(q), len(q), _ptr(out)), "pt_batch_find_elements")
        return out

    def attribute(self, logs, clock=None):
        """Attribute every element of the resident logs ``logs[k]`` to the changes that inserted and deleted it, on the device
        (pt_batch_attribute), after a merge with ``emit_sequence``: (u32 status [n], u64 offsets [n + 1], ATTR_RUN_DT runs),
        request k's runs at runs[off[k]:off[k + 1]].  ``clock`` (u64 offsets [n + 1], CLOCK_DT entries by actor rank;
        ``packing.checkout_clocks``) also flags what was inserted or deleted since that version.  ``attribution.attribution_runs``
        is its host specification.  Needs a change table."""
        from .attribution import ATTR_RUN_DT, _AttrView
        lg = np.ascontiguousarray(logs, np.uint32)
        off = ent = None
        if clock is not None:
            off, ent = np.ascontiguousarray(clock[0], np.uint64), np.ascontiguousarray(clock[1], CLOCK_DT)
        v = _AttrView()
        _check(self._L.pt_batch_attribute(self._h, _ptr(lg), len(lg), None if off is None else off.ctypes.data, _ptr(ent), ctypes.byref(v)),
               "pt_batch_attribute")
        o = _view(v.off, len(lg) + 1, np.uint64) if len(lg) else np.zeros(1, np.uint64)
        return _view(v.status, len(lg), np.uint32), o, _view(v.runs, v.n_runs, ATTR_RUN_DT)

    def restore(self, requests, mode: int = 1):
        """Restore resident logs to earlier versions as new local changes, on the device (pt_batch_restore), after a merge with
        ``emit_sequence``: request k (``restore.RESTORE_REQUEST_DT`` rows, or (log, version, actor, first_ctr) tuples) appends
        to log ``log`` the change by actor rank ``actor`` that makes its visible text (``mode`` RESTORE_TEXT = 1) or its formatting
        (RESTORE_MARKS = 2) equal to that of log ``version`` (a checkout of it), ops counted from ``first_ctr``.  Returns (u32 status RESTORE_*, u32 n_ops, u32 seq) per request; a
        request with no ops appends nothing.  ``restore.restore_inputs`` / ``restore_change_record`` are its host
        specification.  The handle then needs a merge.  Needs a change table."""
        from .restore import RESTORE_REQUEST_DT, _RestoreView
        req = np.ascontiguousarray(np.array([tuple(int(x) for x in q) for q in requests], RESTORE_REQUEST_DT) if len(requests) else np.zeros(0, RESTORE_REQUEST_DT))
        v = _RestoreView()
        _check(self._L.pt_batch_restore(self._h, _ptr(req), len(req), mode, ctypes.byref(v)), "pt_batch_restore")
        status, n_ops, seq = (_view(p, len(req), np.uint32) for p in (v.status, v.n_ops, v.seq))
        if len(req):
            desc = np.zeros(self.n_logs, DESC_DT)
            desc["n_actors"] = self._log_n_actors
            desc["n_insdel" if mode == 1 else "n_mark"][req["log"]] = n_ops
            self._spliced(desc)
        return status, n_ops, seq

    def restore_version(self, logs, versions, actors, first_ctrs=None):
        """The full restore of each ``logs[k]`` to ``versions[k]`` by actor rank ``actors[k]``: restore TEXT, merge, MARKS,
        merge (MARKS compares the formatting the restored text inherits, which only a merge computes).  ``first_ctrs`` default
        to each log's max_ctr + 1 at each step.  Returns ((status, n_ops, seq) of TEXT, the same of MARKS); the handle is
        merged afterwards.  Needs emit_sequence and a change table."""
        from .restore import RESTORE_MARKS, RESTORE_TEXT
        out = []
        for step, mode in enumerate((RESTORE_TEXT, RESTORE_MARKS)):
            if first_ctrs is not None and step == 0:
                ctrs = [int(c) for c in first_ctrs]
            else:
                d = ctypes.c_void_p()
                _check(self._L.pt_batch_download_descs(self._h, ctypes.byref(d)), "pt_batch_download_descs")
                desc = _view(d.value, self.n_logs, DESC_DT)
                ctrs = [int(desc[int(i)]["max_ctr"]) + 1 for i in logs]
            out.append(self.restore(list(zip(logs, versions, actors, ctrs)), mode))
            self.merge()
        self.sync()
        return tuple(out)

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
        st, _keep = _json_pools(batch, pools)
        v = _JsonView()
        _check(getattr(self._L, entry)(self._h, ctypes.byref(st), ctypes.byref(v)), entry)
        return _view(v.bytes, v.n_bytes, np.uint8), _view(v.off, v.n_logs + 1, np.uint64)

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
        req, clock = requests if isinstance(requests, tuple) else (requests, np.zeros(0, CLOCK_DT))
        req = np.ascontiguousarray(req, CHANGES_REQUEST_DT); clock = np.ascontiguousarray(clock, CLOCK_DT)
        st, jp = _json_pools(batch, pools)
        sp = string_pools(batch)
        ex = extras if extras is not None else ChangeExtras(np.zeros(0, EXTRA_DT), [])
        rows = np.ascontiguousarray(ex.rows, EXTRA_DT)
        xdata, xoff = ex.pools()
        keep = [req, clock, jp, sp, rows, xdata, xoff]
        inp = _ChangesJsonInput(len(req), 0, _ptr(req), _ptr(clock), len(clock), st, _ptr(sp["actors"]), _ptr(sp["actors_off"]), _ptr(sp["actors_first"]),
                                _ptr(sp["counters"]), _ptr(sp["counters_first"]), _ptr(sp["list_ids"]), _ptr(sp["list_ids_off"]),
                                _ptr(rows), len(rows), _ptr(xdata), _ptr(xoff), len(ex.ops))
        v = _ChangesJsonView()
        _check(self._L.pt_batch_render_changes_json(self._h, ctypes.byref(inp), ctypes.byref(v)), "pt_batch_render_changes_json")
        del keep
        nr = len(req)
        return _view(v.bytes, v.n_bytes, np.uint8), _view(v.off, nr + 1, np.uint64), _view(v.status, nr, np.uint32)

    def render_changes_json_list(self, batch: PackedBatch, requests, extras: ChangeExtras | None = None, pools=None) -> list[bytes]:
        """``render_changes_json`` as one bytes object per request."""
        data, off, _ = self.render_changes_json(batch, requests, extras, pools)
        return self._split(data, off)

    def set_comment_pool(self, entries: int):
        _check(self._L.pt_batch_set_comment_pool(self._h, int(entries)), "pt_batch_set_comment_pool")

    def set_patch_pool(self, items: int):
        """The capacity of the Patch item pool (pt_batch_set_patch_pool) from the next merge on: a merge whose patches do not
        fit reports the items it needed (``download_patches``), and one re-merge with a pool of that size fits them."""
        _check(self._L.pt_batch_set_patch_pool(self._h, int(items)), "pt_batch_set_patch_pool")

    def run(self, batch: PackedBatch) -> MergedBatch:
        """upload -> merge -> download.  The comment pool has a default capacity; a log whose comment lists do not fit
        reports status 4 without consuming pool space and the engine reports the batch's exact demand, so one re-merge
        with a pool of that size always succeeds (documents with many overlapping comments are valid input)."""
        self._upload_with_changes(batch)
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
        for k, (e, sb) in enumerate(zip(used, subs)):
            if isinstance(sb, PackedRuns):
                e._upload_with_changes(sb, e.upload_runs)
            elif compact:
                e._upload_with_changes(sb, e.upload_compact, *self._compact_buffers(k, len(sb.insdel), len(sb.marks)), threads)
            else:
                e._upload_with_changes(sb)
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

        def pool(kind):
            """pt_ingest_pool: (bytes, u64 offsets [count + 1], u64 per-log first [n + 1] or None)."""
            data, off, cnt, first = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_void_p()
            _check(L.pt_ingest_pool(h, kind, ctypes.byref(data), ctypes.byref(off), ctypes.byref(cnt), ctypes.byref(first)), "pt_ingest_pool")
            o = _view(off.value, cnt.value + 1, np.uint64)
            return (_view(data.value, o[-1], np.uint8).tobytes() if cnt.value else b""), o, (_view(first.value, n + 1, np.uint64) if first.value else None)

        pools = {kind: pool(kind) for kind in (range(8) if with_extras else (0, 1, 3, 4, 5))}
        items = lambda kind: [pools[kind][0][int(a): int(b)] for a, b in zip(pools[kind][1][:-1], pools[kind][1][1:])]
        u16 = lambda b: b.decode("utf-16-le", "surrogatepass")
        values = [u16(b) for b in items(0)]
        link_attrs = [json.loads(b.decode("utf-8", "surrogatepass")) for b in items(1)]
        comment_attrs = [json.loads(b.decode("utf-8", "surrogatepass")) for b in items(3)]
        actors, afirst = items(4), pools[4][2]
        counters, cfirst = items(5), pools[5][2]
        log_actors = [[u16(x) for x in actors[int(afirst[i]): int(afirst[i + 1])]] for i in range(n)]
        log_counters = []
        for i in range(n):
            c = counters[int(cfirst[i]): int(cfirst[i + 1])]
            log_counters.append(np.array([int.from_bytes(x, "little") for x in c], dtype=np.uint64) if c else None)
        table = ChangeTable(_view(tab.logs, tab.n_logs, CDESC_DT), _view(tab.changes, tab.n_changes_total, CHANGE_DT), _view(tab.deps, tab.n_deps_total, DEP_DT))
        batch = PackedBatch(_view(ops.logs, ops.n_logs, DESC_DT), _view(ops.insdel, ops.n_insdel_total, INSDEL_DT), _view(ops.marks, ops.n_mark_total, MARK_DT),
                            values, link_attrs, comment_attrs, [], log_actors=log_actors, log_counters=log_counters, changes=table)
        if not with_extras:
            return batch, None, None
        batch.log_lists = [u16(x) or None for x in items(6)]
        xp, xn = ctypes.c_void_p(), ctypes.c_uint64()
        _check(L.pt_ingest_change_extras(h, ctypes.byref(xp), ctypes.byref(xn)), "pt_ingest_change_extras")
        extras = ChangeExtras(_view(xp.value, xn.value, EXTRA_DT), [b.decode("utf-8", "surrogatepass") for b in items(7)])
        return batch, extras, pools
    finally:
        L.pt_ingest_destroy(h)
