"""Seeded synthetic workloads for the BASELINE.json configs (SURVEY.md §8d) — binding of csrc/workload.cpp.

``generate("c2", n_docs=...)`` returns a ``PackedBatch`` whose log ``d * R + r`` is what replica ``r`` of document ``d``
applied, in its own arrival order.  Comment attrs are synthetic integers (``doc * 4096 + k``), already in rank order;
link attrs are url ids 0..25 (``A.com``..``Z.com``, reference test/fuzz.ts:28).
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from .engine import _view
from .packing import CDESC_DT, CHANGE_DT, CHANGE_NO_ACTOR, DEP_DT, DESC_DT, INPUT_OP_DT, INSDEL_DT, MARK_DT, ChangeTable, ExchangeMaps, PackedBatch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpt_workload.so")
_lib = None

# name -> (kind, default docs, ops per doc, replicas, n_marks)   (BASELINE.json configs[1..4])
CONFIGS = {
    "c2": dict(kind=2, n_docs=1000, ops_per_doc=10000, replicas=2, n_marks=0,
               label="1K docs x 10K ops, insert/delete only, 2 replicas"),
    "c3": dict(kind=3, n_docs=1000, ops_per_doc=10000, replicas=2, n_marks=0,
               label="1K docs x 10K ops with bold/italic/link/comment marks, 2 replicas"),
    "c4": dict(kind=4, n_docs=100000, ops_per_doc=1000, replicas=3, n_marks=0,
               label="100K docs x 1K ops fuzz-generated, 3 concurrent replicas"),
    "c5": dict(kind=5, n_docs=10000, ops_per_doc=100000, replicas=2, n_marks=10000,
               label="10K docs x 100K-char long-form, dense overlapping marks"),
}


class _Config(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_uint32), ("n_docs", ctypes.c_uint32), ("doc_first", ctypes.c_uint32),
                ("ops_per_doc", ctypes.c_uint32), ("replicas", ctypes.c_uint32), ("n_marks", ctypes.c_uint32),
                ("seed", ctypes.c_uint64), ("threads", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class _Batch(ctypes.Structure):
    _fields_ = [("n_logs", ctypes.c_uint32), ("desc", ctypes.c_void_p), ("insdel", ctypes.c_void_p),
                ("n_insdel", ctypes.c_uint64), ("marks", ctypes.c_void_p), ("n_marks", ctypes.c_uint64),
                ("unique_ops", ctypes.c_uint64)]


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run __graft_entry__.build()")
        L = ctypes.CDLL(LIB_PATH)
        L.ptw_generate.argtypes = [ctypes.POINTER(_Config), ctypes.POINTER(ctypes.POINTER(_Batch))]
        L.ptw_generate.restype = ctypes.c_int
        L.ptw_free.argtypes = [ctypes.POINTER(_Batch)]
        _lib = L
    return _lib


class _SyntheticComments:
    def __getitem__(self, i):
        return {"id": "comment-%010d" % int(i)}


def generate(config: str, *, n_docs: int | None = None, ops_per_doc: int | None = None, replicas: int | None = None,
             n_marks: int | None = None, doc_first: int = 0, seed: int | None = None, threads: int = 0) -> PackedBatch:
    cfg = dict(CONFIGS[config])
    if n_docs is not None: cfg["n_docs"] = n_docs
    if ops_per_doc is not None: cfg["ops_per_doc"] = ops_per_doc
    if replicas is not None: cfg["replicas"] = replicas
    if n_marks is not None: cfg["n_marks"] = n_marks
    seed = (0x5EED0000 + cfg["kind"]) if seed is None else seed
    L = _load()
    c = _Config(cfg["kind"], cfg["n_docs"], doc_first, cfg["ops_per_doc"], cfg["replicas"], cfg["n_marks"], seed, threads, 0)
    out = ctypes.POINTER(_Batch)()
    rc = L.ptw_generate(ctypes.byref(c), ctypes.byref(out))
    if rc != 0:
        raise RuntimeError(f"ptw_generate failed: {rc}")
    b = out.contents
    batch = PackedBatch(_view(b.desc, b.n_logs, DESC_DT), _view(b.insdel, b.n_insdel, INSDEL_DT), _view(b.marks, b.n_marks, MARK_DT),
                        values=[], link_attrs=[{"url": f"{ch}.com"} for ch in "ABCDEFGHIJKLMNOPQRSTUVWXYZ"],
                        comment_ids=_SyntheticComments(), other_attrs=[],
                        meta=dict(config=config, label=cfg["label"], n_docs=cfg["n_docs"], replicas=cfg["replicas"],
                                  ops_per_doc=cfg["ops_per_doc"], unique_ops=int(b.unique_ops), seed=seed, doc_first=doc_first))
    L.ptw_free(out)
    return batch


def history_table(batch: PackedBatch) -> ChangeTable:
    """A change table for a generated batch: every log's records as ONE change (seq 1 by actor rank 0, no deps, n_ops = all the
    log's list ops), so all replicas of a document start with equal clocks.  Enough for the calls that need a table
    (admission, pt_batch_change, pt_batch_exchange); the generated records carry no change boundaries of their own."""
    n = batch.n_logs
    cd = np.zeros(n, CDESC_DT)
    cd["change_off"] = np.arange(n); cd["n_changes"] = 1
    ch = np.zeros(n, CHANGE_DT)
    ch["seq"] = 1
    ch["n_ops"] = batch.desc["n_insdel"].astype(np.uint64) + batch.desc["n_mark"]
    return ChangeTable(cd, ch, np.zeros(0, DEP_DT))


def sync_round(batch: PackedBatch, seed: int = 1):
    """One fuzz step (reference test/fuzz.ts:167-199) per document of a generated batch that carries ``history_table``: replica
    r (random) of every document inserts one character at index 0 as actor rank r, then syncs both ways with another random
    replica.  Returns (actor, input_off, ops, tokens: the arrays of pt_change_input; the change table of the new changes;
    the pairs as an (n, 2) array, document by document {changer -> other, other -> changer}; their ExchangeMaps, all identity).
    Vectorised: no per-document Python."""
    R = int(batch.meta["replicas"])
    n = batch.n_logs
    docs = n // R
    rng = np.random.default_rng(seed)
    r = rng.integers(0, R, docs)
    other = (r + 1 + rng.integers(0, R - 1, docs)) % R
    log = np.arange(docs) * R + r
    actor = np.full(n, CHANGE_NO_ACTOR, np.uint32)
    actor[log] = r
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(actor != CHANGE_NO_ACTOR)
    ops = np.zeros(docs, INPUT_OP_DT)
    ops["arg"] = 1; ops["attr"] = 0xFFFFFFFF
    ops["first_ctr"] = batch.desc["max_ctr"][log].astype(np.uint64) + 1
    ops["tok_off"] = np.arange(docs)
    tokens = np.full(docs, ord("x"), np.uint32)
    cd = np.zeros(n, CDESC_DT)
    cd["n_changes"][log] = 1; cd["n_deps"][log] = r != 0
    cd["change_off"] = np.cumsum(cd["n_changes"]) - cd["n_changes"]; cd["dep_off"] = np.cumsum(cd["n_deps"]) - cd["n_deps"]
    ch = np.zeros(docs, CHANGE_DT)                    # actor 0 made the history's change: its next is seq 2; the others depend on it
    ch["seq"] = np.where(r == 0, 2, 1); ch["actor"] = r; ch["n_deps"] = r != 0; ch["n_ops"] = 1
    dp = np.zeros(int((r != 0).sum()), DEP_DT)
    dp["seq"] = 1
    pairs = np.stack([np.stack([log, np.arange(docs) * R + other], 1), np.stack([np.arange(docs) * R + other, log], 1)], 1).reshape(-1, 2)
    na = batch.desc["n_actors"][pairs[:, 0]].astype(np.int64)
    aoff = np.zeros(len(pairs) + 1, np.uint64)
    aoff[1:] = np.cumsum(na)
    amap = (np.arange(int(aoff[-1])) - np.repeat(aoff[:-1].astype(np.int64), na)).astype(np.uint16)
    return actor, off, ops, tokens, ChangeTable(cd, ch, dp), pairs, ExchangeMaps(aoff, amap)


def to_change_json(batch: PackedBatch, i: int) -> str:
    """Log i of a generated batch as the reference's wire format (JSON text of Change objects, one op per change) — the
    input of the native ingest path (`engine.pack_logs_native`); used to measure ingest throughput and to test the ingest on
    the benchmark shapes.  Actor rank r becomes "doc{r+1}", the list is "1@doc1" (the generator's first insert has ctr 2)."""
    import json
    ins, mk = batch.log_slice(i)
    name = lambda r: "doc%d" % (int(r) + 1)
    oid = lambda c, a: "%d@%s" % (int(c), name(a))
    lid = "1@doc1"
    seqs: dict = {}
    out = [{"actor": "doc1", "seq": 1, "deps": {}, "startOp": 1, "ops": [{"opId": lid, "action": "makeList", "obj": "_root", "key": "text"}]}]
    seqs["doc1"] = 1
    btypes = ["before", "after", "startOfText", "endOfText"]
    mtypes = ["strong", "em", "comment", "link"]

    def emit(actor, ctr, op):
        a = name(actor)
        seqs[a] = seqs.get(a, 0) + 1
        out.append({"actor": a, "seq": seqs[a], "deps": {}, "startOp": int(ctr), "ops": [op]})
    k = 0
    for j in range(len(ins) + 1):
        while k < len(mk) and int(mk[k]["arrival"]) == j:
            r = mk[k]; k += 1
            kind, mt = int(r["kind"]) & 1, (int(r["kind"]) >> 1) & 3
            sb, eb = int(r["bounds"]) & 3, (int(r["bounds"]) >> 2) & 3
            op = {"opId": oid(r["ctr"], r["actor"]), "action": "removeMark" if kind else "addMark", "obj": lid, "markType": mtypes[mt],
                  "start": {"type": btypes[sb], **({"elemId": oid(r["start_ctr"], r["start_actor"])} if sb <= 1 else {})},
                  "end": {"type": btypes[eb], **({"elemId": oid(r["end_ctr"], r["end_actor"])} if eb <= 1 else {})}}
            if mt == 3 and not kind:
                op["attrs"] = batch.link_attrs[int(r["attr"])]
            elif mt == 2:
                op["attrs"] = batch.comment_ids[int(r["attr"])]
            emit(r["actor"], r["ctr"], op)
        if j == len(ins):
            break
        r = ins[j]
        if int(r["payload"]) >> 30 == 0:
            op = {"opId": oid(r["ctr"], r["actor"]), "action": "set", "obj": lid, "insert": True, "value": chr(int(r["payload"]) & 0x1FFFFFFF),
                  "elemId": oid(r["ref_ctr"], r["ref_actor"]) if int(r["ref_ctr"]) else "_head"}
        else:
            op = {"opId": oid(r["ctr"], r["actor"]), "action": "del", "obj": lid, "elemId": oid(r["ref_ctr"], r["ref_actor"])}
        emit(r["actor"], r["ctr"], op)
    return json.dumps(out, separators=(",", ":"))
