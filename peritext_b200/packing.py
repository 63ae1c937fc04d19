"""Wire-format ingest: reference ``Change`` objects -> packed op logs (include/peritext_b200.h), and the inverse
decode of the engine's binary results into the reference's ``FormatSpanWithText[]`` shape.

Reference shapes handled here:
  * ``Change`` / ``Operation``          reference src/micromerge.ts:60-71, 143-212
  * ``MarkOperation`` / boundaries      reference src/peritext.ts:11-65
  * ``FormatSpanWithText`` / ``MarkMap`` reference src/peritext.ts:35-38, 135-137
  * map LWW incl. ``makeList``          reference src/micromerge.ts:571-603  (host-side: a handful of ops per doc)

opIds ``"ctr@actor"`` become ``(ctr, actor_rank)`` with ranks in JS string order (UTF-16 code units), so that the
device compares them exactly like ``compareOpIds`` (src/micromerge.ts:812-827).  JSON-saved traces lost their Symbol
fields (SURVEY.md §9.3 Q6): a missing ``obj`` means ROOT and an insert without ``elemId`` means HEAD.
"""
from __future__ import annotations

import json
import re
from dataclasses import dataclass, field
from typing import Any, Iterable, Sequence

import numpy as np

INSDEL_DT = np.dtype([("ctr", "<u4"), ("ref_ctr", "<u4"), ("actor", "<u2"), ("ref_actor", "<u2"), ("payload", "<u4")])
MARK_DT = np.dtype([("ctr", "<u4"), ("actor", "<u2"), ("kind", "u1"), ("bounds", "u1"), ("start_ctr", "<u4"),
                    ("end_ctr", "<u4"), ("start_actor", "<u2"), ("end_actor", "<u2"), ("attr", "<u4"),
                    ("arrival", "<u4"), ("reserved", "<u4")])
DESC_DT = np.dtype([("insdel_off", "<u8"), ("mark_off", "<u8"), ("n_insdel", "<u4"), ("n_mark", "<u4"),
                    ("n_actors", "<u4"), ("max_ctr", "<u4")])
RESULT_DT = np.dtype([("status", "<u4"), ("n_elems", "<u4"), ("n_visible", "<u4"), ("n_spans", "<u4"),
                      ("digest", "<u8", (2,))])
SPAN_DT = np.dtype([("start", "<u4"), ("flags", "<u4"), ("link_attr", "<u4"), ("comment_off", "<u4")])
CHANGE_DT = np.dtype([("seq", "<u4"), ("actor", "<u2"), ("n_deps", "<u2"), ("dep_off", "<u4"), ("n_ops", "<u4")])
DEP_DT = np.dtype([("seq", "<u4"), ("actor", "<u2"), ("reserved", "<u2")])
CDESC_DT = np.dtype([("change_off", "<u8"), ("dep_off", "<u8"), ("n_changes", "<u4"), ("n_deps", "<u4")])
ELEM_REF_DT = np.dtype([("log", "<u4"), ("ctr", "<u4"), ("actor", "<u2"), ("reserved0", "<u2"), ("reserved1", "<u4")])
ELEM_POS_DT = np.dtype([("index", "<u4"), ("visible", "<u4"), ("record", "<u4"), ("flags", "<u4")])
assert CHANGE_DT.itemsize == 16 and DEP_DT.itemsize == 8 and CDESC_DT.itemsize == 24
assert ELEM_REF_DT.itemsize == 16 and ELEM_POS_DT.itemsize == 16
assert INSDEL_DT.itemsize == 16 and MARK_DT.itemsize == 32 and DESC_DT.itemsize == 32
assert RESULT_DT.itemsize == 32 and SPAN_DT.itemsize == 16

KIND_INSERT, KIND_DELETE = 0, 1
TOKEN_POOLED = 0x20000000
ATTR_NONE = 0xFFFFFFFF
ELEM_NOT_FOUND = 0xFFFFFFFF
ELEM_DELETED, ELEM_AFTER_DEFINED, ELEM_LOG_FAILED = 1, 2, 4      # pt_elem_pos.flags
MARK_TYPES = ["strong", "em", "comment", "link"]  # ALL_MARKS order, reference src/schema.ts:125
BOUND_TYPES = ["before", "after", "startOfText", "endOfText"]
SPAN_STRONG, SPAN_EM, SPAN_LINK, SPAN_COMMENT = 1, 2, 4, 8

LOG_STATUS = {0: "ok", 1: "List element not found", 2: "bad opId", 3: "bad record kind", 4: "capacity overflow",
              5: "reference element does not precede insert", 6: "Expected sequence number", 7: "Missing dependency"}

_OPID_RE = re.compile(r"^([0-9]+)@(.*)$", re.S)  # reference src/micromerge.ts:815


def js_key(s: str) -> bytes:
    """Sort key reproducing JS ``<`` on strings (UTF-16 code-unit order)."""
    return s.encode("utf-16-be", "surrogatepass")


def parse_op_id(s: str) -> tuple[int, str]:
    m = _OPID_RE.match(s)
    if not m:
        raise ValueError(f"Invalid operation ID: {s}")
    return int(m.group(1)), m.group(2)


def canon(obj: Any) -> str:
    return json.dumps(obj, sort_keys=True, separators=(",", ":"), ensure_ascii=False)


@dataclass
class PackedBatch:
    """A batch of packed logs plus the host-side pools needed to turn results back into strings."""
    desc: np.ndarray                      # DESC_DT [n_logs]
    insdel: np.ndarray                    # INSDEL_DT
    marks: np.ndarray                     # MARK_DT
    values: list[str] = field(default_factory=list)        # value pool: multi-code-point element values
    link_attrs: list[Any] = field(default_factory=list)    # link attr id -> attrs object
    comment_ids: list[Any] = field(default_factory=list)   # comment rank -> attrs object ({"id": ...}), JS id order
    other_attrs: list[Any] = field(default_factory=list)   # strong/em attrs (normally none)
    meta: dict = field(default_factory=dict)
    log_actors: list[list[str]] = field(default_factory=list)   # per log: actor rank -> actorId
    log_counters: list = field(default_factory=list)            # per log: None, or dense counter rank -> original counter
    changes: Any = None                                         # optional ChangeTable (admission pre-pass)

    @property
    def n_logs(self) -> int:
        return int(self.desc.shape[0])

    @property
    def n_ops(self) -> int:
        return int(self.insdel.shape[0] + self.marks.shape[0])

    def log_slice(self, i: int) -> tuple[np.ndarray, np.ndarray]:
        d = self.desc[i]
        return (self.insdel[int(d["insdel_off"]): int(d["insdel_off"]) + int(d["n_insdel"])],
                self.marks[int(d["mark_off"]): int(d["mark_off"]) + int(d["n_mark"])])

    def slice_logs(self, a: int, b: int) -> "PackedBatch":
        """Logs [a, b) as VIEWS of this batch's arrays (no copy: pinned host memory stays pinned); offsets re-based."""
        d = self.desc[a:b].copy()
        changes = self.changes.slice_logs(a, b) if self.changes is not None else None
        if len(d) == 0:
            return PackedBatch(d, self.insdel[:0], self.marks[:0], self.values, self.link_attrs, self.comment_ids, self.other_attrs, dict(self.meta),
                               changes=changes)
        i0, m0 = int(d[0]["insdel_off"]), int(d[0]["mark_off"])
        i1 = int(d[-1]["insdel_off"]) + int(d[-1]["n_insdel"]); m1 = int(d[-1]["mark_off"]) + int(d[-1]["n_mark"])
        d["insdel_off"] -= i0; d["mark_off"] -= m0
        return PackedBatch(d, self.insdel[i0:i1], self.marks[m0:m1], self.values, self.link_attrs, self.comment_ids, self.other_attrs,
                           dict(self.meta), self.log_actors[a:b] if self.log_actors else [],
                           self.log_counters[a:b] if self.log_counters else [], changes)

    def select(self, idx: Sequence[int]) -> "PackedBatch":
        """Sub-batch with the given logs (re-based offsets); pools are shared."""
        idx = list(idx)
        ins_parts, mk_parts = [], []
        desc = np.zeros(len(idx), DESC_DT)
        io = mo = 0
        for k, i in enumerate(idx):
            a, b = self.log_slice(i)
            ins_parts.append(a); mk_parts.append(b)
            desc[k] = self.desc[i]
            desc[k]["insdel_off"] = io; desc[k]["mark_off"] = mo
            io += len(a); mo += len(b)
        ins = np.concatenate(ins_parts) if ins_parts else np.zeros(0, INSDEL_DT)
        mk = np.concatenate(mk_parts) if mk_parts else np.zeros(0, MARK_DT)
        return PackedBatch(desc, ins, mk, self.values, self.link_attrs, self.comment_ids, self.other_attrs, dict(self.meta),
                           changes=self.changes.select(idx) if self.changes is not None else None)

    def algorithmic_bytes(self, results: np.ndarray | None = None) -> int:
        """SURVEY.md §8(d): 16 B per ins/del + 32 B per mark read; 4 B per visible element, 16 B per span and
        16 B per log written."""
        b = 16 * int(self.insdel.shape[0]) + 32 * int(self.marks.shape[0]) + 16 * self.n_logs
        if results is not None:
            b += 4 * int(results["n_visible"].sum()) + 16 * int(results["n_spans"].sum())
        return b


@dataclass
class ChangeTable:
    """Per-change admission records (include/peritext_b200.h pt_change_table): what Micromerge.applyChange checks before
    applying a change (reference src/micromerge.ts:499-511)."""
    desc: np.ndarray      # CDESC_DT [n_logs]
    changes: np.ndarray   # CHANGE_DT
    deps: np.ndarray      # DEP_DT

    def slice_logs(self, a: int, b: int) -> "ChangeTable":
        """Logs [a, b) as views of the change and dep arrays; offsets re-based (a change's dep_off is relative to its log)."""
        d = self.desc[a:b].copy()
        if len(d) == 0:
            return ChangeTable(d, self.changes[:0], self.deps[:0])
        c0, p0 = int(d[0]["change_off"]), int(d[0]["dep_off"])
        c1 = int(d[-1]["change_off"]) + int(d[-1]["n_changes"]); p1 = int(d[-1]["dep_off"]) + int(d[-1]["n_deps"])
        d["change_off"] -= c0; d["dep_off"] -= p0
        return ChangeTable(d, self.changes[c0:c1], self.deps[p0:p1])

    def select(self, idx: Sequence[int]) -> "ChangeTable":
        """The tables of the given logs, in that order (copies; offsets re-based)."""
        parts = [self.slice_logs(i, i + 1) for i in idx]
        desc = np.zeros(len(parts), CDESC_DT)
        co = do = 0
        for k, t in enumerate(parts):
            desc[k] = t.desc[0]
            desc[k]["change_off"] = co; desc[k]["dep_off"] = do
            co += len(t.changes); do += len(t.deps)
        return ChangeTable(desc, np.concatenate([t.changes for t in parts] + [self.changes[:0]]),
                           np.concatenate([t.deps for t in parts] + [self.deps[:0]]))


class _LogBuilder:
    """Collects one log's ops (arrival order) before ranks are known."""

    def __init__(self):
        self.insdel: list[tuple] = []   # (ctr, actor, ref_ctr|0, ref_actor|None, kind, value|None)
        self.marks: list[tuple] = []    # (ctr, actor, add, mtype, sb, (sctr, sactor), eb, (ectr, eactor), attrs, arrival)
        self.actors: set[str] = set()
        self.max_ctr = 0
        self.changes: list[tuple] = []  # (actor, seq, [(dep actor, dep seq)...], n list ops)


def _root_text_list(changes: Iterable[dict]) -> str | None:
    """Sequentially replays the ROOT-map ops to find which list `["text"]` resolves to
    (reference src/micromerge.ts:571-603, :446-463).  Returns the list's object id string or None."""
    key_meta: dict[str, tuple[int, bytes]] = {}
    children: dict[str, str] = {}
    for ch in changes:
        for op in ch["ops"]:
            obj = op.get("obj")
            if obj not in (None, "_root"):
                continue
            key = op.get("key")
            if key is None or op["action"] in ("addMark", "removeMark"):
                continue
            c, a = parse_op_id(op["opId"])
            me = (c, js_key(a))
            if key not in key_meta or key_meta[key] < me:       # :585
                key_meta[key] = me
                if op["action"] in ("makeList", "makeMap"):      # :589-596
                    children[key] = op["opId"]
    return children.get("text")


def pack_logs(logs: Sequence[Sequence[dict]], *, list_ids: Sequence[str | None] | None = None, with_changes: bool = False) -> PackedBatch:
    """Pack ``logs[i]`` = the Change objects one replica applied, in arrival order.

    Ops that do not target the log's text list (ROOT-map ops, other lists) are host-side bookkeeping and are not
    packed.  ``list_ids[i]`` overrides the list object id (default: what ``["text"]`` resolves to).  ``with_changes``
    also builds the per-change admission table (then the change / deps actors take part in the log's actor ranking).
    The native, multithreaded equivalent over JSON text is ``pack_logs_native`` (csrc/ingest.cpp)."""
    builders: list[_LogBuilder] = []
    values: list[str] = []
    value_index: dict[str, int] = {}
    link_attrs: list[Any] = []
    link_index: dict[str, int] = {}
    comment_objs: dict[str, Any] = {}
    other_attrs: list[Any] = []
    other_index: dict[str, int] = {}

    def token_of(v: Any) -> int:
        """Element value -> 30-bit token: the code point of a one-code-point string, else a value-pool reference
        (an element may hold a multi-character string, reference test/micromerge.ts:202)."""
        if not isinstance(v, str):
            raise TypeError("Expected value inserted into text to be a string")   # src/micromerge.ts:654-656
        if len(v) == 1:
            return ord(v)
        if v not in value_index:
            value_index[v] = len(values)
            values.append(v)
        return TOKEN_POOLED | value_index[v]

    for li, changes in enumerate(logs):
        b = _LogBuilder()
        lid = list_ids[li] if list_ids is not None and list_ids[li] is not None else _root_text_list(changes)
        for ch in changes:
            if with_changes:
                b.actors.add(ch["actor"])
                deps = list((ch.get("deps") or {}).items())
                for a, _ in deps:
                    b.actors.add(a)
                b.changes.append([ch["actor"], int(ch["seq"]), [(a, int(v)) for a, v in deps], 0])
            for op in ch["ops"]:
                if lid is None or op.get("obj") != lid:
                    continue
                if with_changes:
                    b.changes[-1][3] += 1
                ctr, actor = parse_op_id(op["opId"])
                b.actors.add(actor)
                b.max_ctr = max(b.max_ctr, ctr)
                act = op["action"]
                if act in ("addMark", "removeMark"):
                    mt = MARK_TYPES.index(op["markType"])
                    bounds = []
                    for side in ("start", "end"):
                        bd = op[side]
                        t = BOUND_TYPES.index(bd["type"])
                        if t <= 1:
                            ec, ea = parse_op_id(bd["elemId"])
                            b.actors.add(ea)
                        else:
                            ec, ea = 0, None
                        bounds.append((t, ec, ea))
                    attrs = op.get("attrs")
                    attr_ref = None
                    if attrs is not None:
                        if mt == 3:
                            k = canon(attrs)
                            if k not in link_index:
                                link_index[k] = len(link_attrs)
                                link_attrs.append(attrs)
                            attr_ref = ("link", link_index[k])
                        elif mt == 2:
                            cid = attrs["id"]
                            comment_objs.setdefault(cid, attrs)
                            attr_ref = ("comment", cid)
                        else:
                            k = canon(attrs)
                            if k != '{"active":true}':
                                if k not in other_index:
                                    other_index[k] = len(other_attrs)
                                    other_attrs.append(attrs)
                                attr_ref = ("other", other_index[k])
                    elif mt == 2:
                        raise ValueError("comment mark without attrs")
                    b.marks.append((ctr, actor, act == "addMark", mt, bounds[0], bounds[1], attr_ref, len(b.insdel)))
                elif act == "set" and op.get("insert"):
                    ref = op.get("elemId")
                    if ref in (None, "_head"):
                        rc, ra = 0, None
                    else:
                        rc, ra = parse_op_id(ref)
                        b.actors.add(ra)
                    b.insdel.append((ctr, actor, rc, ra, KIND_INSERT, token_of(op.get("value"))))
                elif act == "del" and op.get("key") is None:
                    ref = op.get("elemId")
                    if ref in (None, "_head"):
                        raise ValueError("List element not found: _head")
                    rc, ra = parse_op_id(ref)
                    b.actors.add(ra)
                    b.insdel.append((ctr, actor, rc, ra, KIND_DELETE, 0))
                else:
                    raise NotImplementedError(f"{act} on a list")                   # src/micromerge.ts:567
        builders.append(b)

    comment_sorted = sorted(comment_objs, key=js_key)       # sortBy(..., c => c.id), src/peritext.ts:318
    comment_rank = {cid: i for i, cid in enumerate(comment_sorted)}

    n_ins = sum(len(b.insdel) for b in builders)
    n_mk = sum(len(b.marks) for b in builders)
    desc = np.zeros(len(builders), DESC_DT)
    insdel = np.zeros(n_ins, INSDEL_DT)
    marks = np.zeros(n_mk, MARK_DT)
    io = mo = 0
    counters: list = []      # per log: None, or dense counter rank -> original counter
    for li, b in enumerate(builders):
        ranked = sorted(b.actors, key=js_key)
        rank = {a: i for i, a in enumerate(ranked)}
        if len(ranked) > 0xFFFF:
            raise ValueError("more than 65535 actors in one log")
        # Sparse counters (a peer may choose any startOp, reference src/micromerge.ts:511): the engine's id table is
        # direct-addressed by (ctr, actor), so counters far beyond the op count are re-ranked densely.  Only the ORDER
        # of counters matters to compareOpIds, and the dense rank preserves it.
        dense = None
        if b.max_ctr > 2 * (len(b.insdel) + len(b.marks)) + 16:
            used = {c for (c, _a, rc, _ra, _k, _t) in b.insdel for c in (c, rc)} | {c for mk_ in b.marks for c in (mk_[0], mk_[4][1], mk_[5][1])}
            used.discard(0)
            order = sorted(used)
            dense = {c: i + 1 for i, c in enumerate(order)}
            dense[0] = 0
            counters.append(np.array([0] + order, dtype=np.uint64))
        else:
            counters.append(None)
        dc = (lambda c: dense[c]) if dense is not None else (lambda c: c)
        desc[li] = (io, mo, len(b.insdel), len(b.marks), max(1, len(ranked)), dc(b.max_ctr) if dense is not None else b.max_ctr)
        for k, (ctr, actor, rc, ra, kind, tok) in enumerate(b.insdel):
            insdel[io + k] = (dc(ctr), dc(rc), rank[actor], rank[ra] if ra is not None else 0, (kind << 30) | tok)
        for k, (ctr, actor, add, mt, sb, eb, attr_ref, arrival) in enumerate(b.marks):
            if attr_ref is None:
                attr = ATTR_NONE
            elif attr_ref[0] == "comment":
                attr = comment_rank[attr_ref[1]]
            elif attr_ref[0] == "link":
                attr = attr_ref[1]
            else:
                attr = ATTR_NONE  # non-default strong/em attrs are not representable on the device path
                raise NotImplementedError("strong/em marks with custom attrs")
            marks[mo + k] = (dc(ctr), rank[actor], (0 if add else 1) | (mt << 1), sb[0] | (eb[0] << 2),
                             dc(sb[1]), dc(eb[1]), rank[sb[2]] if sb[2] is not None else 0,
                             rank[eb[2]] if eb[2] is not None else 0, attr, arrival, 0)
        io += len(b.insdel); mo += len(b.marks)
    table = None
    if with_changes:
        cdesc = np.zeros(len(builders), CDESC_DT)
        crecs = np.zeros(sum(len(b.changes) for b in builders), CHANGE_DT)
        cdeps = np.zeros(sum(len(c[2]) for b in builders for c in b.changes), DEP_DT)
        co = do = 0
        for li, b in enumerate(builders):
            rank = {a: i for i, a in enumerate(sorted(b.actors, key=js_key))}
            nd = 0
            cdesc[li]["change_off"] = co; cdesc[li]["dep_off"] = do; cdesc[li]["n_changes"] = len(b.changes)
            for (actor, seq, deps, n_ops) in b.changes:
                crecs[co] = (seq, rank[actor], len(deps), nd, n_ops); co += 1
                for a, v in deps:
                    cdeps[do] = (v, rank[a], 0); do += 1; nd += 1
            cdesc[li]["n_deps"] = nd
        table = ChangeTable(cdesc, crecs, cdeps)
    return PackedBatch(desc, insdel, marks, values, link_attrs, [comment_objs[c] for c in comment_sorted], other_attrs,
                       log_actors=[sorted(b.actors, key=js_key) for b in builders], log_counters=counters, changes=table)


def elem_refs(batch: PackedBatch, logs: Sequence[int], elem_ids: Sequence[str]) -> tuple[np.ndarray, np.ndarray]:
    """elemIds ``"ctr@actor"`` of the logs ``logs[k]`` -> packed ids for ``pt_batch_find_elements``: (ELEM_REF_DT array,
    bool mask of the ids that can exist in their log).  The actor becomes its rank in ``batch.log_actors[log]``; the counter
    its dense rank in ``batch.log_counters[log]`` where the packer re-ranked sparse counters.  Masked (and not to be sent to
    the device; their rows hold ctr 0): a log index outside the batch, ``"_head"`` or a malformed id, an actor the log never
    saw, a counter missing from the log's re-rank table or beyond 32 bits.  Batches from ``pack_logs`` and
    ``pack_logs_native`` carry the same tables, so both give the same refs."""
    n = len(elem_ids)
    refs = np.zeros(n, ELEM_REF_DT)
    ok = np.zeros(n, bool)
    logs = np.asarray(logs, dtype=np.int64)
    if logs.shape != (n,):
        raise ValueError("logs and elem_ids must have the same length")
    refs["log"] = np.clip(logs, 0, 0xFFFFFFFF)
    ranks: dict[int, dict[str, int]] = {}
    for k in range(n):
        i = int(logs[k])
        if i < 0 or i >= batch.n_logs or i >= len(batch.log_actors):
            continue
        m = _OPID_RE.match(elem_ids[k]) if isinstance(elem_ids[k], str) else None
        if m is None:
            continue
        ctr = int(m.group(1))
        rank = ranks.get(i)
        if rank is None:
            rank = ranks[i] = {a: r for r, a in enumerate(batch.log_actors[i])}
        a = rank.get(m.group(2))
        if a is None:
            continue
        cmap = batch.log_counters[i] if i < len(batch.log_counters) else None
        if cmap is not None:
            c = int(np.searchsorted(cmap, ctr)) if ctr < 2 ** 64 else len(cmap)
            if c >= len(cmap) or int(cmap[c]) != ctr:
                continue
            ctr = c
        if ctr > 0xFFFFFFFF:
            continue
        refs["ctr"][k] = ctr
        refs["actor"][k] = a
        ok[k] = True
    return refs, ok


# ------------------------------------------------------------------------------------------------------------------
# Decode
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class MergedBatch:
    """Engine output for a batch (host copies)."""
    results: np.ndarray        # RESULT_DT [n_logs]
    text_off: np.ndarray       # u64 [n_logs]
    span_off: np.ndarray       # u64 [n_logs]
    text: np.ndarray           # u32 tokens
    spans: np.ndarray          # SPAN_DT
    comment_pool: np.ndarray   # u32
    seq: np.ndarray | None = None   # u32 per element (record index | deleted << 31), only with emit_sequence
    seq_off: np.ndarray | None = None   # u64 [n_logs] offsets into seq (capacity layout); None: same as text_off

    def sequence(self, i: int) -> np.ndarray:
        o = int((self.seq_off if self.seq_off is not None else self.text_off)[i]); return self.seq[o: o + int(self.results[i]["n_elems"])]

    def tokens(self, i: int) -> np.ndarray:
        o = int(self.text_off[i]); return self.text[o: o + int(self.results[i]["n_visible"])]

    def span_records(self, i: int) -> np.ndarray:
        o = int(self.span_off[i]); return self.spans[o: o + int(self.results[i]["n_spans"])]

    def canonical(self, i: int) -> tuple:
        """Offset-free canonical form of log i's output, for exact comparison between implementations."""
        r = self.results[i]
        sp = self.span_records(i)
        spans = []
        for s in sp:
            nc = int(s["flags"]) >> 8
            co = int(s["comment_off"])
            spans.append((int(s["start"]), int(s["flags"]), int(s["link_attr"]),
                          tuple(int(x) for x in self.comment_pool[co: co + nc])))
        return (int(r["status"]), int(r["n_elems"]), int(r["n_visible"]), int(r["n_spans"]),
                tuple(int(x) for x in self.tokens(i)), tuple(spans), (int(r["digest"][0]), int(r["digest"][1])))


def token_str(tok: int, values: Sequence[str]) -> str:
    return values[tok & (TOKEN_POOLED - 1)] if tok & TOKEN_POOLED else chr(tok)


def decode_spans(batch: PackedBatch, merged: MergedBatch, i: int) -> list[dict]:
    """Log i's result as the reference's FormatSpanWithText[] (src/peritext.ts:35-38): ``[{marks, text}, ...]``.
    MarkMap key order is canonical (strong, em, comment, link); equality with the reference is deep equality
    (SURVEY.md §9.3 Q8)."""
    r = merged.results[i]
    if int(r["status"]) != 0:
        raise RangeError(LOG_STATUS.get(int(r["status"]), f"status {int(r['status'])}"))
    toks = merged.tokens(i)
    sp = merged.span_records(i)
    out = []
    for j, s in enumerate(sp):
        a = int(s["start"])
        b = int(sp[j + 1]["start"]) if j + 1 < len(sp) else int(r["n_visible"])
        flags = int(s["flags"])
        marks: dict[str, Any] = {}
        if flags & SPAN_STRONG:
            marks["strong"] = {"active": True}
        if flags & SPAN_EM:
            marks["em"] = {"active": True}
        if flags & SPAN_COMMENT:
            co = int(s["comment_off"])
            marks["comment"] = [batch.comment_ids[int(x)] for x in merged.comment_pool[co: co + (flags >> 8)]]
        if flags & SPAN_LINK:
            marks["link"] = batch.link_attrs[int(s["link_attr"])]
        out.append({"marks": marks, "text": "".join(token_str(int(t), batch.values) for t in toks[a:b])})
    return out


def _pool(items: Sequence[bytes]) -> tuple[np.ndarray, np.ndarray]:
    off = np.zeros(len(items) + 1, np.uint64)
    if items:
        off[1:] = np.cumsum([len(b) for b in items], dtype=np.uint64)
    return np.frombuffer(b"".join(items), np.uint8).copy(), off


def json_pools(batch: PackedBatch) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """The string pools ``pt_batch_render_json`` reads, built from a PackedBatch: (values, values_off, links, links_off,
    comments, comments_off), each data as uint8 plus uint64 byte offsets [count + 1].  Values are UTF-16LE; link attrs and
    comment attrs are their canonical JSON (``canon``) in UTF-8, the form ``pt_ingest_pool`` kinds 1 and 3 hold; lone
    surrogates pass through in their 3-byte encoding, which the render writes as ``\\udxxx``."""
    try:
        n_comments = len(batch.comment_ids)
    except TypeError:
        raise ValueError("json_pools: batch.comment_ids has no length (a generated workload's synthetic comment ids): "
                         "attach a list of the comment attrs objects in rank order first") from None
    vals = _pool([v.encode("utf-16-le", "surrogatepass") for v in batch.values])
    links = _pool([canon(a).encode("utf-8", "surrogatepass") for a in batch.link_attrs])
    comments = _pool([canon(batch.comment_ids[k]).encode("utf-8", "surrogatepass") for k in range(n_comments)])
    return vals + links + comments


class RangeError(Exception):
    """JS RangeError equivalents (reference src/micromerge.ts:503, 507, 539, 752)."""


def output_layout(desc: np.ndarray) -> tuple[np.ndarray, np.ndarray, int, int]:
    """Per-log output offsets (the engine and the oracle replay use the same capacities):
    text capacity = n_insdel tokens; span capacity = min(n_insdel, 2*n_mark + 1) (every mark op adds at most two
    boundaries, and a span needs at least one visible element)."""
    n_ins = desc["n_insdel"].astype(np.uint64)
    cap_sp = np.minimum(n_ins, 2 * desc["n_mark"].astype(np.uint64) + 1)
    text_off = np.zeros(len(desc), np.uint64)
    span_off = np.zeros(len(desc), np.uint64)
    if len(desc):
        text_off[1:] = np.cumsum(n_ins)[:-1]
        span_off[1:] = np.cumsum(cap_sp)[:-1]
    return text_off, span_off, int(n_ins.sum()), int(cap_sp.sum())


def comment_pool_capacity(batch: PackedBatch) -> int:
    mk = batch.marks
    n_comment = int((((mk["kind"] >> 1) & 3) == 2).sum()) if len(mk) else 0
    return 64 * n_comment + 1024


@dataclass
class DevicePatches:
    """The device Patch stream of a merged batch (include/peritext_b200.h pt_patch_view)."""
    recs: np.ndarray      # PATCH_REC_DT per ins/del record (batch offsets)
    items: np.ndarray     # PATCH_ITEM_DT pool entries, any order
    status: np.ndarray    # per log: 0 computed on the device, 1 not computed (derive on the host)

    def _index(self):
        if not hasattr(self, "_by_log"):
            by = {}
            for it in self.items:
                by.setdefault(int(it["log"]), []).append((int(it["tag"]), int(it["a"]), int(it["b"])))
            self._by_log = by
        return self._by_log


def patch_stream(batch: PackedBatch, dp: DevicePatches, i: int, ops: Sequence[dict]) -> list[list[dict]]:
    """Patches of log i as the reference's Patch objects (reference src/micromerge.ts:25-58), one list per list op of `ops`
    (= the log's list ops in arrival order, the same ops `pack_logs` packed).  insert: {path, action, index, values, marks};
    delete: {path, action, index, count: 1} (only the element's first delete emits); marks: {action, markType, path,
    startIndex, [attrs], endIndex}."""
    if int(dp.status[i]) != 0:
        raise RangeError("patches of this log were not computed on the device")
    d = batch.desc[i]
    io = int(d["insdel_off"])
    items = dp._index().get(i, [])
    comments: dict[int, list[int]] = {}
    mpatches: dict[int, list[tuple[int, int]]] = {}
    for tag, a, b in items:
        if tag & 0x80000000:
            mpatches.setdefault(tag & 0x7FFFFFFF, []).append((a, b))
        else:
            comments.setdefault(tag, []).append(a)
    out = []
    ri = mi = 0
    for op in ops:
        act = op["action"]
        if act in ("addMark", "removeMark"):
            ps = []
            for a, b in sorted(mpatches.get(mi, [])):
                patch = {"action": act, "markType": op["markType"], "path": ["text"], "startIndex": a}
                if act == "addMark" and op["markType"] in ("link", "comment"):
                    patch["attrs"] = op["attrs"]
                patch["endIndex"] = b
                ps.append(patch)
            out.append(ps); mi += 1
            continue
        r = dp.recs[io + ri]
        idx, emits = int(r["index"]) & 0x7FFFFFFF, bool(int(r["index"]) >> 31)
        if act == "set":
            flags = int(r["flags"])
            marks: dict[str, Any] = {}
            if flags & SPAN_STRONG:
                marks["strong"] = {"active": True}
            if flags & SPAN_EM:
                marks["em"] = {"active": True}
            if flags & SPAN_COMMENT:
                marks["comment"] = [batch.comment_ids[c] for c in sorted(comments.get(ri, []))]
            if flags & SPAN_LINK:
                marks["link"] = batch.link_attrs[int(r["link_attr"])]
            out.append([{"path": ["text"], "action": "insert", "index": idx, "values": [op["value"]], "marks": marks}])
        else:
            out.append([{"path": ["text"], "action": "delete", "index": idx, "count": 1}] if emits else [])
        ri += 1
    return out
