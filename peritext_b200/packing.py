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
    log_lists: list = field(default_factory=list)               # per log: the object id of the text list that was packed

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
                               changes=changes, log_lists=self.log_lists[a:b] if self.log_lists else [])
        i0, m0 = int(d[0]["insdel_off"]), int(d[0]["mark_off"])
        i1 = int(d[-1]["insdel_off"]) + int(d[-1]["n_insdel"]); m1 = int(d[-1]["mark_off"]) + int(d[-1]["n_mark"])
        d["insdel_off"] -= i0; d["mark_off"] -= m0
        return PackedBatch(d, self.insdel[i0:i1], self.marks[m0:m1], self.values, self.link_attrs, self.comment_ids, self.other_attrs,
                           dict(self.meta), self.log_actors[a:b] if self.log_actors else [],
                           self.log_counters[a:b] if self.log_counters else [], changes, self.log_lists[a:b] if self.log_lists else [])

    def select(self, idx: Sequence[int]) -> "PackedBatch":
        """Sub-batch with the given logs (re-based offsets); pools are shared, per-log tables follow their logs."""
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
        pick = lambda t: [t[i] for i in idx] if t else []
        return PackedBatch(desc, ins, mk, self.values, self.link_attrs, self.comment_ids, self.other_attrs, dict(self.meta),
                           pick(self.log_actors), pick(self.log_counters), self.changes.select(idx) if self.changes is not None else None,
                           pick(self.log_lists))

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


class _Pools:
    """A batch's interned strings: the value pool, link attrs, comment attrs (the first-seen attrs object per comment id)
    and other attrs.  Known entries keep their index; new ones get the next."""

    def __init__(self, values=(), link_attrs=(), comment_attrs=(), other_attrs=()):
        self.values = list(values)
        self.value_index = {v: i for i, v in enumerate(self.values)}
        self.link_attrs = list(link_attrs)
        self.link_index = {canon(a): i for i, a in enumerate(self.link_attrs)}
        self.comment_objs: dict[str, Any] = {a["id"]: a for a in comment_attrs}
        self.other_attrs = list(other_attrs)
        self.other_index = {canon(a): i for i, a in enumerate(self.other_attrs)}

    def token_of(self, v: Any) -> int:
        """Element value -> 30-bit token: the code point of a one-code-point string, else a value-pool reference
        (an element may hold a multi-character string, reference test/micromerge.ts:202)."""
        if not isinstance(v, str):
            raise TypeError("Expected value inserted into text to be a string")   # src/micromerge.ts:654-656
        if len(v) == 1:
            return ord(v)
        if v not in self.value_index:
            self.value_index[v] = len(self.values)
            self.values.append(v)
        return TOKEN_POOLED | self.value_index[v]


def _collect_log(changes: Iterable[dict], lid: str | None, with_changes: bool, pools: _Pools) -> _LogBuilder:
    """One log's ops that target list `lid` (arrival order), with their ids still as strings; see ``pack_logs``."""
    b = _LogBuilder()
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
                        if k not in pools.link_index:
                            pools.link_index[k] = len(pools.link_attrs)
                            pools.link_attrs.append(attrs)
                        attr_ref = ("link", pools.link_index[k])
                    elif mt == 2:
                        cid = attrs["id"]
                        pools.comment_objs.setdefault(cid, attrs)
                        attr_ref = ("comment", cid)
                    else:
                        k = canon(attrs)
                        if k != '{"active":true}':
                            if k not in pools.other_index:
                                pools.other_index[k] = len(pools.other_attrs)
                                pools.other_attrs.append(attrs)
                            attr_ref = ("other", pools.other_index[k])
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
                b.insdel.append((ctr, actor, rc, ra, KIND_INSERT, pools.token_of(op.get("value"))))
            elif act == "del" and op.get("key") is None:
                ref = op.get("elemId")
                if ref in (None, "_head"):
                    raise ValueError("List element not found: _head")
                rc, ra = parse_op_id(ref)
                b.actors.add(ra)
                b.insdel.append((ctr, actor, rc, ra, KIND_DELETE, 0))
            else:
                raise NotImplementedError(f"{act} on a list")                   # src/micromerge.ts:567
    return b


def _used_counters(b: _LogBuilder) -> set[int]:
    """Every counter a log's ops name (opIds, references, mark boundaries), HEAD excluded."""
    used = {c for (c, _a, rc, _ra, _k, _t) in b.insdel for c in (c, rc)} | {c for mk_ in b.marks for c in (mk_[0], mk_[4][1], mk_[5][1])}
    used.discard(0)
    return used


def _wants_dense(max_ctr: int, n_ops: int) -> bool:
    """Sparse counters (a peer may choose any startOp, reference src/micromerge.ts:511): the engine's id table is
    direct-addressed by (ctr, actor), so counters far beyond the op count are re-ranked densely.  Only the ORDER of
    counters matters to compareOpIds, and the dense rank preserves it."""
    return max_ctr > 2 * n_ops + 16


def _emit_log(b: _LogBuilder, rank: dict, dc, comment_rank: dict, insdel: np.ndarray, io: int, marks: np.ndarray, mo: int,
              arrival_base: int = 0) -> None:
    """Writes one log's records at insdel[io:] / marks[mo:] in the packed id space (`rank`: actor ranks, `dc`: counters)."""
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
                         rank[eb[2]] if eb[2] is not None else 0, attr, arrival_base + arrival, 0)


def _change_table(builders: Sequence[_LogBuilder], ranks: Sequence[dict]) -> ChangeTable:
    cdesc = np.zeros(len(builders), CDESC_DT)
    crecs = np.zeros(sum(len(b.changes) for b in builders), CHANGE_DT)
    cdeps = np.zeros(sum(len(c[2]) for b in builders for c in b.changes), DEP_DT)
    co = do = 0
    for li, b in enumerate(builders):
        rank = ranks[li]
        nd = 0
        cdesc[li]["change_off"] = co; cdesc[li]["dep_off"] = do; cdesc[li]["n_changes"] = len(b.changes)
        for (actor, seq, deps, n_ops) in b.changes:
            crecs[co] = (seq, rank[actor], len(deps), nd, n_ops); co += 1
            for a, v in deps:
                cdeps[do] = (v, rank[a], 0); do += 1; nd += 1
        cdesc[li]["n_deps"] = nd
    return ChangeTable(cdesc, crecs, cdeps)


def pack_logs(logs: Sequence[Sequence[dict]], *, list_ids: Sequence[str | None] | None = None, with_changes: bool = False) -> PackedBatch:
    """Pack ``logs[i]`` = the Change objects one replica applied, in arrival order.

    Ops that do not target the log's text list (ROOT-map ops, other lists) are host-side bookkeeping and are not
    packed.  ``list_ids[i]`` overrides the list object id (default: what ``["text"]`` resolves to).  ``with_changes``
    also builds the per-change admission table (then the change / deps actors take part in the log's actor ranking).
    The native, multithreaded equivalent over JSON text is ``pack_logs_native`` (csrc/ingest.cpp)."""
    pools = _Pools()
    builders: list[_LogBuilder] = []
    lids: list[str | None] = []
    for li, changes in enumerate(logs):
        lid = list_ids[li] if list_ids is not None and list_ids[li] is not None else _root_text_list(changes)
        lids.append(lid)
        builders.append(_collect_log(changes, lid, with_changes, pools))

    comment_sorted = sorted(pools.comment_objs, key=js_key)       # sortBy(..., c => c.id), src/peritext.ts:318
    comment_rank = {cid: i for i, cid in enumerate(comment_sorted)}
    desc, insdel, marks, counters, ranks = _emit_logs(builders, comment_rank)
    table = _change_table(builders, ranks) if with_changes else None
    return PackedBatch(desc, insdel, marks, pools.values, pools.link_attrs, [pools.comment_objs[c] for c in comment_sorted], pools.other_attrs,
                       log_actors=[sorted(b.actors, key=js_key) for b in builders], log_counters=counters, changes=table, log_lists=lids)


def _emit_logs(builders: Sequence[_LogBuilder], comment_rank: dict):
    """Whole logs in the packed id space (``pack_logs``' rules per log): (descriptors, ins/del records, mark records, per log
    None or the dense counter table, per log actor -> rank)."""
    n_ins = sum(len(b.insdel) for b in builders)
    n_mk = sum(len(b.marks) for b in builders)
    desc = np.zeros(len(builders), DESC_DT)
    insdel = np.zeros(n_ins, INSDEL_DT)
    marks = np.zeros(n_mk, MARK_DT)
    io = mo = 0
    counters: list = []      # per log: None, or dense counter rank -> original counter
    ranks: list[dict] = []
    for li, b in enumerate(builders):
        ranked = sorted(b.actors, key=js_key)
        rank = {a: i for i, a in enumerate(ranked)}
        ranks.append(rank)
        if len(ranked) > 0xFFFF:
            raise ValueError("more than 65535 actors in one log")
        dense = None
        if _wants_dense(b.max_ctr, len(b.insdel) + len(b.marks)):
            order = sorted(_used_counters(b))
            dense = {c: i + 1 for i, c in enumerate(order)}
            dense[0] = 0
            counters.append(np.array([0] + order, dtype=np.uint64))
        else:
            counters.append(None)
        dc = (lambda c: dense[c]) if dense is not None else (lambda c: c)
        desc[li] = (io, mo, len(b.insdel), len(b.marks), max(1, len(ranked)), dc(b.max_ctr) if dense is not None else b.max_ctr)
        _emit_log(b, rank, dc, comment_rank, insdel, io, marks, mo)
        io += len(b.insdel); mo += len(b.marks)
    return desc, insdel, marks, counters, ranks


# ------------------------------------------------------------------------------------------------------------------
# Append (include/peritext_b200.h pt_batch_append)
# ------------------------------------------------------------------------------------------------------------------
CTR_UNUSED = 0xFFFFFFFF      # a counter-map entry for an old counter that no record of the log names


@dataclass
class AppendRemap:
    """How the resident records' ids move when a batch grows (pt_append_remap); None = identity.  Log i's actor map is
    actor_map[actor_off[i]:actor_off[i+1]] (old rank -> new rank; empty = identity), its counter map likewise (old ctr ->
    new ctr, entry 0 = 0; CTR_UNUSED for an old counter no record names); comment_map: old comment rank -> new rank."""
    actor_off: np.ndarray | None = None      # u64 [n_logs + 1]
    actor_map: np.ndarray | None = None      # u16
    ctr_off: np.ndarray | None = None        # u64 [n_logs + 1]
    ctr_map: np.ndarray | None = None        # u32
    comment_map: np.ndarray | None = None    # u32


def _flat_maps(maps: Sequence[Sequence[int] | None], dtype) -> tuple[np.ndarray | None, np.ndarray | None]:
    """Per-log maps (None = identity) -> (offsets [n + 1], concatenated map), or (None, None) if every map is the identity."""
    if all(m is None for m in maps):
        return None, None
    off = np.zeros(len(maps) + 1, np.uint64)
    off[1:] = np.cumsum([0 if m is None else len(m) for m in maps])
    flat = [x for m in maps if m is not None for x in m]
    return off, np.array(flat, dtype)


def _grown_ids(prev: PackedBatch, i: int, new_actors, new_max_ctr: int, n_new_ops: int, new_used):
    """Log i's packed id space after it gains `n_new_ops` ops that name the actors `new_actors`, have opId counters up to
    `new_max_ctr` and name the counters `new_used()` (original counters; called only where the grown log is dense): ``pack_logs``'s
    rules on the full log.  Returns (actors in rank order, actor -> rank, old rank -> new rank or None for the identity, the
    dense counter table or None, original -> packed counter, the packed max_ctr, old packed -> new packed counter or None)."""
    d = prev.desc[i]
    old_actors = list(prev.log_actors[i])
    ranked = sorted(set(old_actors) | set(new_actors), key=js_key)
    if len(ranked) > 0xFFFF:
        raise ValueError("more than 65535 actors in one log")
    rank = {a: r for r, a in enumerate(ranked)}
    amap = [rank[a] for a in old_actors]
    old_dense = prev.log_counters[i] if i < len(prev.log_counters) else None
    old_max_ctr = int(d["max_ctr"])
    full_max = max(int(old_dense[old_max_ctr]) if old_dense is not None else old_max_ctr, new_max_ctr)
    full_ops = int(d["n_insdel"]) + int(d["n_mark"]) + n_new_ops
    if _wants_dense(full_max, full_ops):
        if old_dense is not None:
            old_used = set(int(c) for c in old_dense[1:])
        else:
            ins, mk = prev.log_slice(i)
            old_used = set(np.concatenate([ins["ctr"], ins["ref_ctr"], mk["ctr"], mk["start_ctr"], mk["end_ctr"]]).astype(np.int64).tolist())
            old_used.discard(0)
        order = sorted(old_used | new_used())
        dense = {c: k + 1 for k, c in enumerate(order)}
        dense[0] = 0
        table = np.array([0] + order, dtype=np.uint64)
        dc = dense.__getitem__
        new_max = dense[full_max]
        if old_dense is not None:
            cm = [dense[int(c)] for c in old_dense]
        else:
            # the domain: every counter the old records name (a mark boundary may name an element inserted later), up
            # to a bound that keeps a reference far past the log's opIds from sizing the map
            cap = 2 * (old_max_ctr + int(d["n_insdel"]) + int(d["n_mark"])) + 16
            hi = max([old_max_ctr] + [c for c in old_used if c <= cap])
            cm = [dense.get(c, CTR_UNUSED) for c in range(hi + 1)]
    else:
        table = None
        dc = (lambda c: c)
        new_max = full_max
        cm = [int(c) for c in old_dense] if old_dense is not None else None
    return (ranked, rank, amap if amap != list(range(len(amap))) else None, table, dc, new_max,
            cm if cm is not None and cm != list(range(len(cm))) else None)


def add_actors(batch: PackedBatch, names: Sequence[Sequence[str]]) -> tuple[PackedBatch, AppendRemap, list[list[int]]]:
    """The host specification of ``pt_batch_add_actors``: ``names[i]`` are ids for log i in any order (duplicates and known ids
    allowed).  Returns (the empty delta and the remap of ``pt_batch_append`` that make each log's actor table the sorted union,
    n_actors = max(1, count), counters untouched; per log the rank of every given id afterwards)."""
    n = batch.n_logs
    if len(names) != n:
        raise ValueError(f"add_actors: {len(names)} id lists for a batch of {n} logs")
    desc = np.zeros(n, DESC_DT)
    actor_maps, log_actors, ranks = [], [], []
    for i in range(n):
        ranked, rank, amap, _, _, _, _ = _grown_ids(batch, i, names[i], 0, 0, set)
        actor_maps.append(amap); log_actors.append(ranked)
        ranks.append([rank[a] for a in names[i]])
        desc[i]["n_actors"] = max(1, len(ranked)); desc[i]["max_ctr"] = batch.desc[i]["max_ctr"]
    aoff, amaps = _flat_maps(actor_maps, np.uint16)
    table = ChangeTable(np.zeros(n, CDESC_DT), np.zeros(0, CHANGE_DT), np.zeros(0, DEP_DT)) if batch.changes is not None else None
    delta = PackedBatch(desc, np.zeros(0, INSDEL_DT), np.zeros(0, MARK_DT), batch.values, batch.link_attrs, batch.comment_ids, batch.other_attrs,
                        dict(batch.meta), log_actors, list(batch.log_counters) if batch.log_counters else [None] * n, table, list(batch.log_lists))
    return delta, AppendRemap(aoff, amaps), ranks


def pack_append(prev: PackedBatch, new_logs: Sequence[Sequence[dict]], *, with_changes: bool = False,
                list_ids: Sequence[str | None] | None = None) -> tuple[PackedBatch, AppendRemap]:
    """The delta and remap of ``pt_batch_append`` that extend every log of ``prev`` (a ``pack_logs`` batch) with the Change
    objects ``new_logs[i]``, so that ``apply_append(prev, delta, remap)`` is ``pack_logs`` of the concatenated logs.

    Everything about the old logs comes from ``prev``: actors from ``log_actors``, used counters from ``log_counters`` (or
    from the records where a log was not re-ranked), comment ids from ``comment_ids``, pools from ``values`` /
    ``link_attrs``, the text list from ``log_lists`` (or ``list_ids``; a log with old records and neither raises ValueError,
    since the new changes alone rarely name the list).  ``pack_logs``'s rules apply to the FULL log: the actor set (with the
    change and dep actors when ``with_changes``, which must match how ``prev`` was packed), the dense-counter rule, the
    batch-wide comment order.  Known strings keep their pool index and new ones get the next, so the result names the same
    strings as ``pack_logs`` of the full logs, maybe at other indices; a known comment id keeps its first-seen attrs.  A log's
    counter map covers every counter its old records name, except, where a plain log turns dense, counters beyond
    2 x (old max_ctr + old records) + 16, which only a reference to an element far past the log's opIds can name: those become
    0xFFFFFFFF where ``pack_logs`` would rank them.
    The delta carries the new pools, ``log_actors``, ``log_counters`` and ``log_lists``, and the change table of the new
    changes."""
    n = prev.n_logs
    if len(new_logs) != n:
        raise ValueError(f"pack_append: {len(new_logs)} new logs for a batch of {n}")
    if with_changes != (prev.changes is not None):
        raise ValueError("pack_append: with_changes must match whether prev has a change table")
    if len(prev.log_actors) != n:
        raise ValueError("pack_append: prev carries no log_actors (pack it with pack_logs)")
    pools = _Pools(prev.values, prev.link_attrs, prev.comment_ids, prev.other_attrs)
    builders, lids = [], []
    for i, changes in enumerate(new_logs):
        old_recs = int(prev.desc[i]["n_insdel"]) + int(prev.desc[i]["n_mark"])
        if list_ids is not None and list_ids[i] is not None:
            lid = list_ids[i]
        elif i < len(prev.log_lists) and prev.log_lists[i] is not None:
            lid = prev.log_lists[i]
        elif old_recs and i >= len(prev.log_lists):
            raise ValueError(f"pack_append: log {i} has records but prev does not record its text list (a batch from "
                             "pack_logs_native or built by hand): pass list_ids")
        else:
            lid = _root_text_list(changes)       # the old log has no text list: the new changes may create it
        lids.append(lid)
        builders.append(_collect_log(changes, lid, with_changes, pools))
    old_cids = [a["id"] for a in prev.comment_ids]
    comment_sorted = sorted(pools.comment_objs, key=js_key)
    comment_rank = {cid: i for i, cid in enumerate(comment_sorted)}
    cmap = [comment_rank[c] for c in old_cids]

    desc = np.zeros(n, DESC_DT)
    insdel = np.zeros(sum(len(b.insdel) for b in builders), INSDEL_DT)
    marks = np.zeros(sum(len(b.marks) for b in builders), MARK_DT)
    io = mo = 0
    actor_maps, ctr_maps, log_actors, counters, ranks = [], [], [], [], []
    for i, b in enumerate(builders):
        d = prev.desc[i]
        ranked, rank, amap, table, dc, new_max, cm = _grown_ids(prev, i, b.actors, b.max_ctr, len(b.insdel) + len(b.marks), lambda b=b: _used_counters(b))
        ranks.append(rank); log_actors.append(ranked)
        actor_maps.append(amap); counters.append(table); ctr_maps.append(cm)
        desc[i] = (io, mo, len(b.insdel), len(b.marks), max(1, len(ranked)), new_max)
        _emit_log(b, rank, dc, comment_rank, insdel, io, marks, mo, arrival_base=int(d["n_insdel"]))
        io += len(b.insdel); mo += len(b.marks)
    aoff, amaps = _flat_maps(actor_maps, np.uint16)
    coff, cmaps = _flat_maps(ctr_maps, np.uint32)
    remap = AppendRemap(aoff, amaps, coff, cmaps, np.array(cmap, np.uint32) if cmap != list(range(len(cmap))) else None)
    delta = PackedBatch(desc, insdel, marks, pools.values, pools.link_attrs, [pools.comment_objs[c] for c in comment_sorted], pools.other_attrs,
                        dict(prev.meta), log_actors, counters, _change_table(builders, ranks) if with_changes else None, lids)
    return delta, remap


def split_records(batch: PackedBatch, cuts) -> tuple[PackedBatch, PackedBatch]:
    """(prefix, delta) of a record-level batch: log i keeps its first cuts[i] ins/del records and the marks that arrived
    before them (marks must be in arrival order), the rest is the delta of ``pt_batch_append`` with identity maps.  Both
    keep the log's n_actors / max_ctr.  For benchmarks and tests that grow generated workloads; vectorised."""
    d = batch.desc
    n_mk = d["n_mark"].astype(np.int64)
    cuts = np.minimum(np.asarray(cuts, np.int64), d["n_insdel"].astype(np.int64))
    li = np.repeat(np.arange(batch.n_logs), n_mk)
    keep = batch.marks["arrival"][_ranges(d["mark_off"], n_mk)].astype(np.int64) < cuts[li]
    m_pre = np.bincount(li[keep], minlength=batch.n_logs).astype(np.int64)
    first_mk = np.concatenate([[0], np.cumsum(n_mk)[:-1]]).astype(np.int64)
    if not (keep == (np.arange(len(li)) - first_mk[li] < m_pre[li])).all():
        raise ValueError("split_records: a log's marks are not in arrival order")

    def part(first_ins, cnt_ins, first_m, cnt_m):
        desc = np.zeros(batch.n_logs, DESC_DT)
        desc["n_insdel"], desc["n_mark"] = cnt_ins, cnt_m
        desc["insdel_off"], desc["mark_off"] = _excl_scan(cnt_ins), _excl_scan(cnt_m)
        desc["n_actors"], desc["max_ctr"] = d["n_actors"], d["max_ctr"]
        return PackedBatch(desc, batch.insdel[_ranges(d["insdel_off"].astype(np.int64) + first_ins, cnt_ins)],
                           batch.marks[_ranges(d["mark_off"].astype(np.int64) + first_m, cnt_m)], batch.values, batch.link_attrs,
                           batch.comment_ids, batch.other_attrs)
    return (part(np.zeros_like(cuts), cuts, np.zeros_like(m_pre), m_pre),
            part(cuts, d["n_insdel"].astype(np.int64) - cuts, m_pre, n_mk - m_pre))


def _ranges(off: np.ndarray, cnt: np.ndarray) -> np.ndarray:
    """Indices [off[i], off[i] + cnt[i]) of every i, concatenated."""
    cnt = np.asarray(cnt, np.int64)
    if int(cnt.sum()) == 0:
        return np.zeros(0, np.int64)
    first = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return np.repeat(np.asarray(off, np.int64) - first, cnt) + np.arange(int(cnt.sum()), dtype=np.int64)


def _excl_scan(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.uint64)
    out = np.zeros(len(x), np.uint64)
    if len(x):
        out[1:] = np.cumsum(x)[:-1]
    return out


def _through(vals: np.ndarray, log: np.ndarray, off: np.ndarray | None, m: np.ndarray | None, fill: int) -> np.ndarray:
    """vals[k] through the map of log log[k] (m[off[l]:off[l+1]], empty = identity); outside the map's domain -> fill."""
    vals = np.asarray(vals, np.int64)
    if off is None or len(vals) == 0:
        return vals
    off = np.asarray(off, np.int64)
    ln = (off[1:] - off[:-1])[log]
    out = vals.copy()
    mapped = ln > 0
    inside = mapped & (vals < ln)
    out[mapped & ~inside] = fill
    out[inside] = np.asarray(m, np.int64)[(off[:-1][log] + vals)[inside]]
    return out


def apply_append(prev: PackedBatch, delta: PackedBatch, remap: AppendRemap | None = None) -> PackedBatch:
    """The readable host specification of ``pt_batch_append``'s splice: the batch the handle holds after appending
    ``delta`` with ``remap`` to ``prev``.  Logs are contiguous and in order, each with its old records (ids through the
    log's maps) and then its delta records.  An id whose counter is 0 (HEAD, a text boundary) keeps its actor field; a value
    outside its map's domain, or mapped to CTR_UNUSED, becomes 0xFFFF / 0xFFFFFFFF.  A comment mark's rank goes through the
    comment map (PT_ATTR_NONE stays); a rank outside it raises ValueError, as the device refuses it.  The change table is
    concatenated per log with old actor ranks mapped and the delta's dep_off rebased.  Pools, ``log_actors``,
    ``log_counters`` and ``log_lists`` are the delta's."""
    r = remap or AppendRemap()
    n = prev.n_logs
    if delta.n_logs != n:
        raise ValueError(f"apply_append: the delta has {delta.n_logs} logs and the batch {n}")
    od, dd = prev.desc, delta.desc
    desc = np.zeros(n, DESC_DT)
    desc["n_insdel"] = od["n_insdel"].astype(np.uint64) + dd["n_insdel"]
    desc["n_mark"] = od["n_mark"].astype(np.uint64) + dd["n_mark"]
    desc["insdel_off"] = _excl_scan(desc["n_insdel"]); desc["mark_off"] = _excl_scan(desc["n_mark"])
    desc["n_actors"] = dd["n_actors"]; desc["max_ctr"] = dd["max_ctr"]
    logs = np.arange(n)

    def splice(recs, drecs, off_f, cnt_f, dt, remap_fn):
        out = np.zeros(int(desc[cnt_f].astype(np.int64).sum()), dt)
        o = recs[_ranges(od[off_f], od[cnt_f])].copy()
        remap_fn(o, np.repeat(logs, od[cnt_f].astype(np.int64)))
        out[_ranges(desc[off_f], od[cnt_f])] = o
        out[_ranges(desc[off_f].astype(np.int64) + od[cnt_f], dd[cnt_f])] = drecs[_ranges(dd[off_f], dd[cnt_f])]
        return out

    def ctr(v, lg):
        return _through(v, lg, r.ctr_off, r.ctr_map, 0xFFFFFFFF)

    def id_actor(c, a, lg):      # counter 0 names no actor
        return np.where(np.asarray(c) != 0, _through(a, lg, r.actor_off, r.actor_map, 0xFFFF), np.asarray(a, np.int64))

    def map_insdel(o, lg):
        c, rc = o["ctr"].copy(), o["ref_ctr"].copy()
        o["actor"] = id_actor(c, o["actor"], lg); o["ref_actor"] = id_actor(rc, o["ref_actor"], lg)
        o["ctr"] = ctr(c, lg); o["ref_ctr"] = ctr(rc, lg)

    def map_marks(o, lg):
        c, sc, ec = o["ctr"].copy(), o["start_ctr"].copy(), o["end_ctr"].copy()
        o["actor"] = id_actor(c, o["actor"], lg)
        o["start_actor"] = id_actor(sc, o["start_actor"], lg); o["end_actor"] = id_actor(ec, o["end_actor"], lg)
        o["ctr"] = ctr(c, lg); o["start_ctr"] = ctr(sc, lg); o["end_ctr"] = ctr(ec, lg)
        if r.comment_map is not None:
            com = (((o["kind"] >> 1) & 3) == 2) & (o["attr"] != ATTR_NONE)
            cm = np.asarray(r.comment_map, np.int64)
            if (o["attr"][com] >= len(cm)).any():
                raise ValueError("apply_append: a resident comment rank is outside comment_map")
            o["attr"][com] = cm[o["attr"][com].astype(np.int64)]

    insdel = splice(prev.insdel, delta.insdel, "insdel_off", "n_insdel", INSDEL_DT, map_insdel)
    marks = splice(prev.marks, delta.marks, "mark_off", "n_mark", MARK_DT, map_marks)
    changes = None
    if (prev.changes is None) != (delta.changes is None):
        raise ValueError("apply_append: a change table on one side only")
    if prev.changes is not None:
        oc, dcg = prev.changes, delta.changes
        ocd, dcd = oc.desc, dcg.desc
        cdesc = np.zeros(n, CDESC_DT)
        cdesc["n_changes"] = ocd["n_changes"].astype(np.uint64) + dcd["n_changes"]
        cdesc["n_deps"] = ocd["n_deps"].astype(np.uint64) + dcd["n_deps"]
        cdesc["change_off"] = _excl_scan(cdesc["n_changes"]); cdesc["dep_off"] = _excl_scan(cdesc["n_deps"])

        def cat(recs, drecs, off_f, cnt_f, dt, fix_old, fix_new):
            out = np.zeros(int(cdesc[cnt_f].astype(np.int64).sum()), dt)
            o = recs[_ranges(ocd[off_f], ocd[cnt_f])].copy()
            fix_old(o, np.repeat(logs, ocd[cnt_f].astype(np.int64)))
            d = drecs[_ranges(dcd[off_f], dcd[cnt_f])].copy()
            fix_new(d, np.repeat(logs, dcd[cnt_f].astype(np.int64)))
            out[_ranges(cdesc[off_f], ocd[cnt_f])] = o
            out[_ranges(cdesc[off_f].astype(np.int64) + ocd[cnt_f], dcd[cnt_f])] = d
            return out

        def map_actor(o, lg):
            o["actor"] = _through(o["actor"], lg, r.actor_off, r.actor_map, 0xFFFF)

        def rebase(d, lg):
            d["dep_off"] += ocd["n_deps"][lg]

        changes = ChangeTable(cdesc, cat(oc.changes, dcg.changes, "change_off", "n_changes", CHANGE_DT, map_actor, rebase),
                              cat(oc.deps, dcg.deps, "dep_off", "n_deps", DEP_DT, map_actor, lambda d, lg: None))
    return PackedBatch(desc, insdel, marks, delta.values, delta.link_attrs, delta.comment_ids, delta.other_attrs, dict(prev.meta),
                       delta.log_actors, delta.log_counters, changes, delta.log_lists)


# ------------------------------------------------------------------------------------------------------------------
# Select (include/peritext_b200.h pt_batch_select_logs)
# ------------------------------------------------------------------------------------------------------------------
SELECT_ADDED = 0xFFFFFFFF    # a `from_` entry: the next log of `added`
SELECT_DROPPED = 0xFFFFFFFF  # a comment-map entry: a rank that no kept log names


def pack_select(prev: PackedBatch, from_: Sequence[int], new_logs: Sequence[Sequence[dict]], *, with_changes: bool) -> tuple[PackedBatch, np.ndarray | None]:
    """The added logs and comment map of ``pt_batch_select_logs``: ``new_logs`` are the Change logs of the entries of ``from_``
    that are SELECT_ADDED, in order, packed as ``pack_logs`` would pack them against ``prev``'s pools.  Known strings keep their
    pool index and new ones take the next; the batch-wide comment order is ``prev``'s ids and the new ones in JS order, and the
    comment map says where each old rank moves (None when none moves).  Only ``prev``'s pools are read, so this also works when
    the kept logs' records live only on the device.  ``with_changes`` builds the added logs' change table."""
    n_add = sum(1 for f in from_ if int(f) == SELECT_ADDED)
    if len(new_logs) != n_add:
        raise ValueError(f"pack_select: {len(new_logs)} new logs for {n_add} SELECT_ADDED entries")
    pools = _Pools(prev.values, prev.link_attrs, prev.comment_ids, prev.other_attrs)
    lids = [_root_text_list(changes) for changes in new_logs]
    builders = [_collect_log(changes, lid, with_changes, pools) for changes, lid in zip(new_logs, lids)]
    comment_sorted = sorted(pools.comment_objs, key=js_key)
    comment_rank = {cid: i for i, cid in enumerate(comment_sorted)}
    cmap = [comment_rank[a["id"]] for a in prev.comment_ids]
    desc, insdel, marks, counters, ranks = _emit_logs(builders, comment_rank)
    added = PackedBatch(desc, insdel, marks, pools.values, pools.link_attrs, [pools.comment_objs[c] for c in comment_sorted], pools.other_attrs,
                        dict(prev.meta), [sorted(b.actors, key=js_key) for b in builders], counters,
                        _change_table(builders, ranks) if with_changes else None, lids)
    return added, (np.array(cmap, np.uint32) if cmap != list(range(len(cmap))) else None)


def apply_select(prev: PackedBatch, from_: Sequence[int], added: PackedBatch | None = None, comment_map=None) -> PackedBatch:
    """The readable host specification of ``pt_batch_select_logs``: new log i is ``prev``'s log ``from_[i]``, or, where it is
    SELECT_ADDED, the next log of ``added``.  Kept logs keep their records, change tables, ``log_actors``, ``log_counters`` and
    ``log_lists``; their comment marks' ranks go through ``comment_map`` (None = identity), and a kept rank outside it or mapped
    to SELECT_DROPPED raises ValueError, as the device refuses it.  Added logs are copied verbatim.  The pools are ``added``'s,
    or without added logs ``prev``'s with the comment ids moved through the map."""
    from_ = [int(f) for f in from_]
    n_prev, n_add = prev.n_logs, (added.n_logs if added is not None else 0)
    if sum(1 for f in from_ if f == SELECT_ADDED) != n_add:
        raise ValueError("apply_select: the SELECT_ADDED entries do not match the added logs")
    if any(f != SELECT_ADDED and not 0 <= f < n_prev for f in from_):
        raise ValueError("apply_select: an entry names no log of prev")
    if added is not None and n_add and (prev.changes is None) != (added.changes is None):
        raise ValueError("apply_select: a change table on one side only")
    marks = prev.marks.copy()
    if comment_map is not None:
        cm = np.asarray(comment_map, np.int64)
        li = np.repeat(np.arange(n_prev), prev.desc["n_mark"].astype(np.int64))
        at = _ranges(prev.desc["mark_off"], prev.desc["n_mark"])
        kept = np.isin(li, [f for f in from_ if f != SELECT_ADDED])
        m = marks[at]
        com = kept & (((m["kind"] >> 1) & 3) == 2) & (m["attr"] != ATTR_NONE)
        rank = m["attr"][com].astype(np.int64)
        new = np.full(len(rank), SELECT_DROPPED, np.int64)
        new[rank < len(cm)] = cm[rank[rank < len(cm)]]
        if (new == SELECT_DROPPED).any():
            raise ValueError("apply_select: a kept comment rank is outside comment_map or dropped")
        m["attr"][com] = new
        marks[at] = m
    both = PackedBatch(prev.desc.copy(), prev.insdel, marks)
    if added is not None:
        d = added.desc.copy()
        d["insdel_off"] += len(prev.insdel); d["mark_off"] += len(prev.marks)
        both = PackedBatch(np.concatenate([prev.desc, d]), np.concatenate([prev.insdel, added.insdel]), np.concatenate([marks, added.marks]))
    cat = lambda x, y: list(x or []) + list(y or []) if (x or not n_prev) and (not n_add or y) else []
    src = added if added is not None else prev
    both.log_actors = cat(prev.log_actors, added.log_actors if added is not None else [])
    both.log_counters = cat(prev.log_counters, added.log_counters if added is not None else [])
    both.log_lists = cat(prev.log_lists, added.log_lists if added is not None else [])
    if prev.changes is not None:
        ct = prev.changes
        if added is not None and added.changes is not None:
            cd = added.changes.desc.copy()
            cd["change_off"] += len(ct.changes); cd["dep_off"] += len(ct.deps)
            ct = ChangeTable(np.concatenate([ct.desc, cd]), np.concatenate([ct.changes, added.changes.changes]), np.concatenate([ct.deps, added.changes.deps]))
        both.changes = ct
    idx = [f if f != SELECT_ADDED else n_prev + k for k, f in zip(np.cumsum([f == SELECT_ADDED for f in from_]) - 1, from_)]
    out = both.select(idx)
    comment_ids = src.comment_ids
    if added is None and comment_map is not None:
        comment_ids = [None] * (max([int(c) for c in comment_map if int(c) != SELECT_DROPPED] + [-1]) + 1)
        for r, c in enumerate(comment_map):
            if int(c) != SELECT_DROPPED:
                comment_ids[int(c)] = prev.comment_ids[r]
    out.values, out.link_attrs, out.comment_ids, out.other_attrs, out.meta = src.values, src.link_attrs, comment_ids, src.other_attrs, dict(prev.meta)
    return out


# ------------------------------------------------------------------------------------------------------------------
# Exchange (include/peritext_b200.h pt_batch_exchange)
# ------------------------------------------------------------------------------------------------------------------
EXCHANGE_OK, EXCHANGE_BAD_TABLE, EXCHANGE_STUCK, EXCHANGE_UNMAPPED = 0, 1, 2, 3
EXCHANGE_DENSE = 4           # pt_batch_sync_pairs only: see sync_maps
ACTOR_UNMAPPED = 0xFFFF      # an actor-map entry for a src actor without a rank in dst


@dataclass
class ExchangeMaps:
    """The maps of ``pt_batch_exchange`` (pt_exchange_input), flat like ``AppendRemap``: pair p's actor map is
    actor_map[actor_off[p]:actor_off[p+1]] (src actor rank -> dst actor rank, ACTOR_UNMAPPED = none; exactly src's n_actors
    entries), its counter map ctr_map[ctr_off[p]:ctr_off[p+1]] (src packed counter -> dst packed counter, entry 0 = 0,
    CTR_UNUSED = none; an empty range, or ctr_off None, is the identity)."""
    actor_off: np.ndarray                    # u64 [n_pairs + 1]
    actor_map: np.ndarray                    # u16
    ctr_off: np.ndarray | None = None        # u64 [n_pairs + 1]
    ctr_map: np.ndarray | None = None        # u32

    @staticmethod
    def of(actor_maps: Sequence, ctr_maps: Sequence | None = None) -> "ExchangeMaps":
        """From one array per pair (a counter map may be None: identity)."""
        def flat(maps, dt):
            off = np.zeros(len(maps) + 1, np.uint64)
            off[1:] = np.cumsum([0 if m is None else len(m) for m in maps])
            return off, np.concatenate([np.asarray(m, dt) for m in maps if m is not None] + [np.zeros(0, dt)])
        aoff, amap = flat(actor_maps, np.uint16)
        if ctr_maps is None or all(m is None for m in ctr_maps):
            return ExchangeMaps(aoff, amap)
        return ExchangeMaps(aoff, amap, *flat(ctr_maps, np.uint32))

    def actor(self, p: int) -> np.ndarray:
        return self.actor_map[int(self.actor_off[p]): int(self.actor_off[p + 1])]

    def ctr(self, p: int) -> np.ndarray | None:
        if self.ctr_off is None or self.ctr_off[p + 1] == self.ctr_off[p]:
            return None
        return self.ctr_map[int(self.ctr_off[p]): int(self.ctr_off[p + 1])]


def change_record_ranges(batch: PackedBatch, i: int) -> np.ndarray | None:
    """Per change of log i (rows) the record ranges [ins_lo, ins_hi, mk_lo, mk_hi) of its list ops: change c holds the
    list-op positions [P_c, P_c + n_ops_c), P_c = the sum of the earlier n_ops; mark record k sits at position
    min(arrival_k, n_insdel) + k.  None if n_ops does not sum to the log's records or the arrivals do not fit."""
    cd = batch.changes.desc[i]
    ch = batch.changes.changes[int(cd["change_off"]): int(cd["change_off"]) + int(cd["n_changes"])]
    ins, mk = batch.log_slice(i)
    n, m = len(ins), len(mk)
    ends = np.cumsum(ch["n_ops"].astype(np.int64))
    if (int(ends[-1]) if len(ends) else 0) != n + m:
        return None
    x = np.stack([ends - ch["n_ops"], ends], 1)
    mpos = np.minimum(mk["arrival"].astype(np.int64), n) + np.arange(m)

    def before(pos):             # the first k with mpos[k] >= pos, by the bisection the device uses
        lo, hi = 0, m
        while lo < hi:
            k = (lo + hi) // 2
            if mpos[k] < pos:
                lo = k + 1
            else:
                hi = k
        return lo
    k = np.array([[before(int(a)), before(int(b))] for a, b in x], np.int64).reshape(len(ch), 2)
    r = np.stack([x[:, 0] - k[:, 0], x[:, 1] - k[:, 1], k[:, 0], k[:, 1]], 1)
    if len(r) and ((r < 0).any() or (r[:, 1] > n).any() or (r[:, 1] < r[:, 0]).any() or (r[:, 3] < r[:, 2]).any()):
        return None
    return r


def _log_changes(batch: PackedBatch, i: int):
    cd = batch.changes.desc[i]
    ch = batch.changes.changes[int(cd["change_off"]): int(cd["change_off"]) + int(cd["n_changes"])]
    dp = batch.changes.deps[int(cd["dep_off"]): int(cd["dep_off"]) + int(cd["n_deps"])]
    return ch, dp


def _missing_ids(batch: PackedBatch, src: int, dst: int):
    """What log src delivers to log dst, read from the change tables and src's records: (the actor ids the missing changes
    name, their top opId counter, their record count, a callable giving every counter they name), or None if nothing is
    missing or src's change table does not fit its records.  Counters are original ones."""
    sch, sdp = _log_changes(batch, src)
    dch, _ = _log_changes(batch, dst)
    have: dict[str, int] = {}
    for c in dch:
        a = batch.log_actors[dst][int(c["actor"])]
        have[a] = have.get(a, 0) + 1
    sn = batch.log_actors[src]
    miss = [k for k, c in enumerate(sch) if int(c["seq"]) > have.get(sn[int(c["actor"])], 0)]
    rng = change_record_ranges(batch, src)
    if not miss or rng is None:
        return None
    ins, mk = batch.log_slice(src)
    ins = np.concatenate([ins[rng[k, 0]: rng[k, 1]] for k in miss]); mk = np.concatenate([mk[rng[k, 2]: rng[k, 3]] for k in miss])
    st = batch.log_counters[src] if batch.log_counters else None      # src's records are in the batch's id space
    orig = (lambda c: int(c)) if st is None else (lambda c, st=st: int(st[int(c)]) if int(c) < len(st) else int(c))
    actors = {sn[int(sch[k]["actor"])] for k in miss}
    actors |= {sn[int(q["actor"])] for k in miss for q in sdp[int(sch[k]["dep_off"]): int(sch[k]["dep_off"]) + int(sch[k]["n_deps"])]}
    for recs, ids in ((ins, (("ctr", "actor"), ("ref_ctr", "ref_actor"))), (mk, (("ctr", "actor"), ("start_ctr", "start_actor"), ("end_ctr", "end_actor")))):
        for cf, af in ids:
            actors |= {sn[int(a)] for c, a in zip(recs[cf], recs[af]) if int(c)}
    used = lambda: {orig(c) for recs, fs in ((ins, ("ctr", "ref_ctr")), (mk, ("ctr", "start_ctr", "end_ctr"))) for f in fs for c in recs[f] if int(c)}
    top = max([0] + [orig(c) for c in ins["ctr"]] + [orig(c) for c in mk["ctr"]])
    return actors, top, len(ins) + len(mk), used


def exchange_maps(batch: PackedBatch, pairs, *, grow=None) -> tuple[ExchangeMaps, tuple[PackedBatch, AppendRemap] | None]:
    """The maps of ``pt_batch_exchange`` for `pairs` = [(src, dst), ...] on `batch` (a ``pack_logs(..., with_changes=True)``
    batch or one grown from it), and the empty pre-append that introduces what the deliveries bring to each dst: new actors
    (``log_actors``) and, where ``pack_logs`` would rank the grown log's counters densely (``log_counters``), its new counter
    ranks.  Returns (maps, (delta, remap)) or (maps, None) if no log's id space moves; the maps are in the id spaces AFTER
    ``apply_append(batch, delta, remap)`` / ``BatchEngine.append(delta, remap)``, so {A->B, B->A} sees both logs grown.
    What a dst will receive is read from the change tables alone: src's changes by an actor past dst's count of that actor.
    ``grow(src, dst)`` False leaves that pair's dst as it is (default: every pair may grow its dst)."""
    n = batch.n_logs
    names = [list(a) for a in batch.log_actors]
    tables = list(batch.log_counters) if batch.log_counters else [None] * n
    n_actors = batch.desc["n_actors"].astype(np.int64)
    max_ctr = batch.desc["max_ctr"].astype(np.int64)
    actor_maps_pre, ctr_maps_pre = [None] * n, [None] * n
    moved = False
    for src, dst in pairs:
        got = _missing_ids(batch, src, dst) if grow is None or grow(src, dst) else None
        if got is None:
            continue
        actors, top, n_ops, used = got
        ranked, _, amap, table, _, _, cm = _grown_ids(batch, dst, actors, top, n_ops, used)
        old_max = int(batch.desc[dst]["max_ctr"])
        moved = moved or ranked != names[dst] or amap is not None or cm is not None or (table is None) != (tables[dst] is None) or \
            (table is not None and len(table) != len(tables[dst]))
        names[dst], tables[dst] = ranked, table
        actor_maps_pre[dst], ctr_maps_pre[dst] = amap, cm
        n_actors[dst] = max(1, len(ranked))
        max_ctr[dst] = old_max if cm is None else cm[old_max]       # the image of the old max_ctr: nothing is delivered yet
    amaps, cmaps = [], []
    for src, dst in pairs:
        rank = {a: r for r, a in enumerate(names[dst])}
        amaps.append(np.array([rank.get(a, ACTOR_UNMAPPED) for a in names[src]] + [ACTOR_UNMAPPED] * (int(n_actors[src]) - len(names[src])), np.uint16))
        st, dt = tables[src], tables[dst]
        if st is None and dt is None:
            cmaps.append(None)
            continue
        orig = np.arange(int(max_ctr[src]) + 1, dtype=np.uint64) if st is None else np.asarray(st[: int(max_ctr[src]) + 1], np.uint64)
        if dt is None:
            cm = np.where(orig < CTR_UNUSED, orig, CTR_UNUSED).astype(np.uint32)
        else:
            at = np.minimum(np.searchsorted(dt, orig), len(dt) - 1)
            cm = np.where(dt[at] == orig, at, CTR_UNUSED).astype(np.uint32)
        cmaps.append(cm)
    maps = ExchangeMaps.of(amaps, cmaps)
    if not moved:
        return maps, None
    desc = np.zeros(n, DESC_DT)
    desc["n_actors"], desc["max_ctr"] = n_actors, max_ctr
    aoff, aflat = _flat_maps(actor_maps_pre, np.uint16)
    coff, cflat = _flat_maps(ctr_maps_pre, np.uint32)
    delta = PackedBatch(desc, np.zeros(0, INSDEL_DT), np.zeros(0, MARK_DT), batch.values, batch.link_attrs, batch.comment_ids, batch.other_attrs,
                        dict(batch.meta), names, tables, ChangeTable(np.zeros(n, CDESC_DT), np.zeros(0, CHANGE_DT), np.zeros(0, DEP_DT)), list(batch.log_lists))
    return maps, (delta, AppendRemap(aoff, aflat, coff, cflat))


def _clock_ok(batch: PackedBatch, i: int) -> bool:
    """Log i's change table passes pt_batch_exchange's clock checks: actors < n_actors, seq == count + 1, deps inside."""
    ch, dp = _log_changes(batch, i)
    cnt: dict[int, int] = {}
    for c in ch:
        a = int(c["actor"])
        if a >= int(batch.desc[i]["n_actors"]) or int(c["seq"]) != cnt.get(a, 0) + 1 or int(c["dep_off"]) + int(c["n_deps"]) > len(dp):
            return False
        cnt[a] = cnt.get(a, 0) + 1
    return True


def sync_maps(batch: PackedBatch, pairs) -> tuple[np.ndarray, list, ExchangeMaps, tuple[PackedBatch, AppendRemap] | None]:
    """The host specification of ``pt_batch_sync_pairs``: (per-pair status, EXCHANGE_DENSE or 0, the pairs that are not DENSE,
    and ``exchange_maps`` of those).  A pair is DENSE when src or dst has a dense counter table (``log_counters``) or when dst,
    grown by what it is missing from src, would get one (``_wants_dense``); exactly then ``exchange_maps`` would give it a
    counter table or a counter map.  A pair whose change tables fail the exchange's clock checks does not grow its dst (the
    exchange reports it as EXCHANGE_BAD_TABLE).  The handle afterwards holds ``apply_exchange(apply_append(batch, *pre), live,
    maps)``, with the DENSE pairs' statuses in their places."""
    dense = lambda i: bool(batch.log_counters) and batch.log_counters[i] is not None
    ok = lambda s, d: _clock_ok(batch, s) and _clock_ok(batch, d)
    status = np.zeros(len(pairs), np.uint32)
    live = []
    for p, (src, dst) in enumerate(pairs):
        got = None if dense(src) or dense(dst) or not ok(src, dst) else _missing_ids(batch, src, dst)
        d = batch.desc[dst]
        if dense(src) or dense(dst) or (got is not None and _wants_dense(max(int(d["max_ctr"]), got[1]), int(d["n_insdel"]) + int(d["n_mark"]) + got[2])):
            status[p] = EXCHANGE_DENSE
        else:
            live.append((int(src), int(dst)))
    maps, pre = exchange_maps(batch, live, grow=ok)
    return status, live, maps, pre


def _exchange_order(batch: PackedBatch, src: int, dst: int, amap: np.ndarray) -> tuple[int, list[int]]:
    """Steps 1-3 of ``pt_batch_exchange`` for one pair: (status, src change indices in delivery order)."""
    sch, sdp = _log_changes(batch, src)
    dch, ddp = _log_changes(batch, dst)

    def clock(ch, n_deps, n_actors):
        cnt: dict[int, int] = {}
        for c in ch:
            a = int(c["actor"])
            if a >= n_actors or int(c["seq"]) != cnt.get(a, 0) + 1 or int(c["dep_off"]) + int(c["n_deps"]) > n_deps:
                return None
            cnt[a] = cnt.get(a, 0) + 1
        return cnt
    rs, rd = int(batch.desc[src]["n_actors"]), int(batch.desc[dst]["n_actors"])
    clk = clock(dch, len(ddp), rd)
    cs = clock(sch, len(sdp), rs)
    if clk is None or cs is None or change_record_ranges(batch, src) is None:
        return EXCHANGE_BAD_TABLE, []
    image = lambda a: int(amap[a]) if a < len(amap) else ACTOR_UNMAPPED
    have = lambda a: clk.get(image(a), 0) if image(a) != ACTOR_UNMAPPED else 0
    deps = lambda c: sdp[int(c["dep_off"]): int(c["dep_off"]) + int(c["n_deps"])]
    # getMissingChanges (reference test/merge.ts:25-38): actors in the order src first saw them, ascending seq
    queue = [k for a in dict.fromkeys(int(c["actor"]) for c in sch) for k, c in enumerate(sch) if int(c["actor"]) == a and int(c["seq"]) > have(a)]
    if any(int(q["actor"]) >= rs for k in queue for q in deps(sch[k])):
        return EXCHANGE_BAD_TABLE, []
    if any(image(int(sch[k]["actor"])) == ACTOR_UNMAPPED or any(image(int(q["actor"])) == ACTOR_UNMAPPED for q in deps(sch[k])) for k in queue):
        return EXCHANGE_UNMAPPED, []
    # applyChanges (test/merge.ts:4-23): the front is applied or goes to the back
    order = []
    since = 0                        # requeues since the last delivery: a whole queue of them is a pass that admitted nothing
    while queue:
        k = queue.pop(0)
        c = sch[k]
        a = image(int(c["actor"]))
        if int(c["seq"]) == clk.get(a, 0) + 1 and all(0 < clk.get(image(int(q["actor"])), 0) >= int(q["seq"]) for q in deps(c)):
            clk[a] = int(c["seq"]); order.append(k); since = 0
        else:
            queue.append(k); since += 1
            if since >= len(queue):
                return EXCHANGE_STUCK, []
    return EXCHANGE_OK, order


def apply_exchange(batch: PackedBatch, pairs, maps: ExchangeMaps) -> tuple[PackedBatch, np.ndarray, list[list[int]], np.ndarray]:
    """The readable host specification of ``pt_batch_exchange``: every pair (src, dst) delivers to log dst the changes it is
    missing from log src, all pairs reading `batch` as it is.  Returns (the batch the handle holds afterwards, the per-pair
    status EXCHANGE_*, per pair the delivered indices into src's change table in delivery order, the DESC_DT delta: per log
    the records it received, its n_actors and new max_ctr).  Order: ``getMissingChanges`` then ``applyChanges`` (reference
    test/merge.ts:4-38).  Records: the delivered changes' ins/del records in delivery order, then likewise their marks, ids
    through the pair's maps (an id with counter 0 keeps its actor field), a mark's arrival = dst's old n_insdel + the delivered
    ins/del records before it; change and dep actors through the actor map, dep_off relative to the delivered deps.  A pair
    that is not EXCHANGE_OK delivers nothing.  Pools and per-log tables are `batch`'s."""
    n = batch.n_logs
    if batch.changes is None:
        raise ValueError("apply_exchange: the batch has no change table")
    seen = set()
    for src, dst in pairs:
        if not (0 <= src < n and 0 <= dst < n) or src == dst or dst in seen:
            raise ValueError(f"apply_exchange: bad pair ({src}, {dst})")
        seen.add(dst)
    status = np.zeros(len(pairs), np.uint32)
    delivered: list[list[int]] = []
    ddesc = np.zeros(n, DESC_DT)
    ddesc["n_actors"], ddesc["max_ctr"] = batch.desc["n_actors"], batch.desc["max_ctr"]
    cdesc = np.zeros(n, CDESC_DT)
    parts = {}
    for p, (src, dst) in enumerate(pairs):
        amap = maps.actor(p).astype(np.int64)
        cmap = maps.ctr(p)
        st, order = _exchange_order(batch, src, dst, amap)
        if st == EXCHANGE_OK and order:
            rng = change_record_ranges(batch, src)
            sins, smk = batch.log_slice(src)
            sch, sdp = _log_changes(batch, src)
            ins = np.concatenate([sins[rng[k, 0]: rng[k, 1]] for k in order]).copy()
            mk = np.concatenate([smk[rng[k, 2]: rng[k, 3]] for k in order]).copy()
            # arrivals: dst's old records, the delivered ins/del records of the earlier changes, the mark's place in its own
            before = np.cumsum([0] + [rng[k, 1] - rng[k, 0] for k in order])
            mk["arrival"] = np.concatenate([int(batch.desc[dst]["n_insdel"]) + before[j] + np.clip(smk["arrival"][rng[k, 2]: rng[k, 3]].astype(np.int64) - rng[k, 0], 0, rng[k, 1] - rng[k, 0])
                                            for j, k in enumerate(order)] + [np.zeros(0, np.int64)])
            ch = sch[order].copy()
            dp = np.concatenate([sdp[int(c["dep_off"]): int(c["dep_off"]) + int(c["n_deps"])] for c in ch] + [sdp[:0]]).copy()
            ch["dep_off"] = np.cumsum([0] + [int(c["n_deps"]) for c in ch])[:-1]
            ok = True

            def actor(c, a):             # counter 0 names no actor
                nonlocal ok
                img = np.where(a < len(amap), amap[np.minimum(a, len(amap) - 1)] if len(amap) else ACTOR_UNMAPPED, ACTOR_UNMAPPED)
                ok = ok and not ((c != 0) & (img == ACTOR_UNMAPPED)).any()
                return np.where(c != 0, img, a)

            def ctr(c):
                nonlocal ok
                if cmap is None or len(cmap) == 0:
                    return c
                img = np.where(c < len(cmap), np.asarray(cmap, np.int64)[np.minimum(c, len(cmap) - 1)], CTR_UNUSED)
                ok = ok and not (img == CTR_UNUSED).any()
                return img
            for recs, ids in ((ins, (("ctr", "actor"), ("ref_ctr", "ref_actor"))), (mk, (("ctr", "actor"), ("start_ctr", "start_actor"), ("end_ctr", "end_actor")))):
                for cf, af in ids:
                    c = recs[cf].astype(np.int64)
                    recs[af] = actor(c, recs[af].astype(np.int64)); recs[cf] = ctr(c)
            one = np.ones(1, np.int64)
            ch["actor"] = actor(np.repeat(one, len(ch)), ch["actor"].astype(np.int64)); dp["actor"] = actor(np.repeat(one, len(dp)), dp["actor"].astype(np.int64))
            if not ok:
                st, order = EXCHANGE_UNMAPPED, []
            else:
                parts[dst] = (ins, mk, ch, dp)
                ddesc[dst]["n_insdel"], ddesc[dst]["n_mark"] = len(ins), len(mk)
                ddesc[dst]["max_ctr"] = max([int(batch.desc[dst]["max_ctr"])] + [int(x) for x in ins["ctr"]] + [int(x) for x in mk["ctr"]])
                cdesc[dst]["n_changes"], cdesc[dst]["n_deps"] = len(ch), len(dp)
        status[p] = st
        delivered.append([int(k) for k in order] if st == EXCHANGE_OK else [])
    ddesc["insdel_off"], ddesc["mark_off"] = _excl_scan(ddesc["n_insdel"]), _excl_scan(ddesc["n_mark"])
    cdesc["change_off"], cdesc["dep_off"] = _excl_scan(cdesc["n_changes"]), _excl_scan(cdesc["n_deps"])
    got = [parts[i] for i in sorted(parts)]
    cat = lambda j, dt: np.concatenate([g[j] for g in got] + [np.zeros(0, dt)])
    delta = PackedBatch(ddesc, cat(0, INSDEL_DT), cat(1, MARK_DT), batch.values, batch.link_attrs, batch.comment_ids, batch.other_attrs, dict(batch.meta),
                        batch.log_actors, batch.log_counters, ChangeTable(cdesc, cat(2, CHANGE_DT), cat(3, DEP_DT)), batch.log_lists)
    return apply_append(batch, delta), status, delivered, ddesc


# ------------------------------------------------------------------------------------------------------------------
# Checkout (include/peritext_b200.h pt_batch_checkout, pt_batch_download_clocks)
# ------------------------------------------------------------------------------------------------------------------
CHECKOUT_OK, CHECKOUT_BAD_TABLE, CHECKOUT_UNKNOWN, CHECKOUT_NOT_CLOSED = 0, 1, 2, 3


def _checkout_table_ok(batch: PackedBatch, i: int) -> bool:
    """pt_batch_exchange's BAD_TABLE rules for log i as a src: the clock checks, every dep actor < n_actors, and record ranges
    that fit the log."""
    if not _clock_ok(batch, i):
        return False
    ch, dp = _log_changes(batch, i)
    deps = [q for c in ch for q in dp[int(c["dep_off"]): int(c["dep_off"]) + int(c["n_deps"])]]
    if any(int(q["actor"]) >= int(batch.desc[i]["n_actors"]) for q in deps):
        return False
    return change_record_ranges(batch, i) is not None


def _request_clocks(batch: PackedBatch, logs: Sequence[int], n_changes, clock) -> list[dict]:
    """Per request the clock {actor rank: seq} it names, after pt_batch_checkout's host checks (ValueError)."""
    if (n_changes is None) == (clock is None):
        raise ValueError("apply_checkout: exactly one of n_changes and clock must be given")
    if any(not 0 <= s < batch.n_logs for s in logs):
        raise ValueError("apply_checkout: a request names no log of the batch")
    out = []
    if n_changes is not None:
        n_changes = [int(x) for x in n_changes]
        if len(n_changes) != len(logs):
            raise ValueError("apply_checkout: one n_changes entry per request")
        for s, m in zip(logs, n_changes):
            ch, _ = _log_changes(batch, s)
            req: dict[int, int] = {}
            for c in ch[:m]:
                req[int(c["actor"])] = req.get(int(c["actor"]), 0) + 1
            out.append(req)
        return out
    off, ent = np.asarray(clock[0], np.int64), np.asarray(clock[1], CLOCK_DT)
    if len(off) != len(logs) + 1 or off[0] != 0 or (np.diff(off) < 0).any() or off[-1] > len(ent):
        raise ValueError("apply_checkout: clock offsets are not non-decreasing from 0 within the clock array")
    for k, s in enumerate(logs):
        req = {}
        for e in ent[int(off[k]): int(off[k + 1])]:
            a = int(e["actor"])
            if a >= int(batch.desc[s]["n_actors"]):
                raise ValueError(f"apply_checkout: request {k}: clock actor {a} >= the log's n_actors")
            if a in req:
                raise ValueError(f"apply_checkout: request {k}: actor {a} is named twice")
            req[a] = int(e["seq"])
        out.append(req)
    return out


def apply_checkout(batch: PackedBatch, logs: Sequence[int], n_changes=None, clock=None) -> tuple[PackedBatch, np.ndarray]:
    """The readable host specification of ``pt_batch_checkout``: request k appends a new log holding log ``logs[k]`` at a
    version, covering the first ``n_changes[k]`` changes of its table (prefix mode) or the changes with seq <= the clock's entry
    for their actor (clock mode, ``clock`` = (u64 offsets [n + 1], CLOCK_DT entries by actor rank); an absent actor counts as
    0).  The new log holds the covered changes' ins/del records in table order, then their mark records, a mark's arrival being
    the covered ins/del records before it; their change records with dep_off rebased, and their deps; the source's id space,
    ``log_actors``, ``log_counters`` and ``log_lists``.  Returns (``apply_select`` of the batch with the new logs added, the
    per-request status CHECKOUT_*); a request that is not OK adds a log without records or changes.  NOT_CLOSED is
    applyChange's dep check (reference src/micromerge.ts:505-509) against the covered changes before each one in table order."""
    logs = [int(x) for x in logs]
    if batch.changes is None:
        raise ValueError("apply_checkout: the batch has no change table")
    reqs = _request_clocks(batch, logs, n_changes, clock)
    n = len(logs)
    status = np.zeros(n, np.uint32)
    desc, cdesc = np.zeros(n, DESC_DT), np.zeros(n, CDESC_DT)
    parts = []
    for k, (s, req) in enumerate(zip(logs, reqs)):
        ch, dp = _log_changes(batch, s)
        desc[k]["n_actors"], desc[k]["max_ctr"] = batch.desc[s]["n_actors"], batch.desc[s]["max_ctr"]
        have: dict[int, int] = {}
        for c in ch:
            have[int(c["actor"])] = have.get(int(c["actor"]), 0) + 1
        covered = [int(c["seq"]) <= req.get(int(c["actor"]), 0) for c in ch]
        if not _checkout_table_ok(batch, s):
            status[k] = CHECKOUT_BAD_TABLE
        elif any(seq > have.get(a, 0) for a, seq in req.items()):
            status[k] = CHECKOUT_UNKNOWN
        else:
            run: dict[int, int] = {}
            for c, cov in zip(ch, covered):
                if not cov:
                    continue
                if any(run.get(int(q["actor"]), 0) < max(int(q["seq"]), 1) for q in dp[int(c["dep_off"]): int(c["dep_off"]) + int(c["n_deps"])]):
                    status[k] = CHECKOUT_NOT_CLOSED
                    break
                run[int(c["actor"])] = run.get(int(c["actor"]), 0) + 1
        order = [j for j, cov in enumerate(covered) if cov] if status[k] == CHECKOUT_OK else []
        rng = change_record_ranges(batch, s) if order else None
        sins, smk = batch.log_slice(s)
        ins = np.concatenate([sins[rng[j, 0]: rng[j, 1]] for j in order] + [sins[:0]]).copy()
        mk = np.concatenate([smk[rng[j, 2]: rng[j, 3]] for j in order] + [smk[:0]]).copy()
        before = np.cumsum([0] + [rng[j, 1] - rng[j, 0] for j in order])
        mk["arrival"] = np.concatenate([before[t] + np.clip(smk["arrival"][rng[j, 2]: rng[j, 3]].astype(np.int64) - rng[j, 0], 0, rng[j, 1] - rng[j, 0])
                                        for t, j in enumerate(order)] + [np.zeros(0, np.int64)])
        c2 = ch[order].copy()
        d2 = np.concatenate([dp[int(c["dep_off"]): int(c["dep_off"]) + int(c["n_deps"])] for c in c2] + [dp[:0]]).copy()
        c2["dep_off"] = _excl_scan(c2["n_deps"]) if len(c2) else c2["dep_off"]
        desc[k]["n_insdel"], desc[k]["n_mark"] = len(ins), len(mk)
        cdesc[k]["n_changes"], cdesc[k]["n_deps"] = len(c2), len(d2)
        parts.append((ins, mk, c2, d2))
    desc["insdel_off"], desc["mark_off"] = _excl_scan(desc["n_insdel"]), _excl_scan(desc["n_mark"])
    cdesc["change_off"], cdesc["dep_off"] = _excl_scan(cdesc["n_changes"]), _excl_scan(cdesc["n_deps"])
    cat = lambda j, dt: np.concatenate([p[j] for p in parts] + [np.zeros(0, dt)])
    pick = lambda t: [t[s] for s in logs] if t else []
    added = PackedBatch(desc, cat(0, INSDEL_DT), cat(1, MARK_DT), batch.values, batch.link_attrs, batch.comment_ids, batch.other_attrs, dict(batch.meta),
                        pick(batch.log_actors), pick(batch.log_counters), ChangeTable(cdesc, cat(2, CHANGE_DT), cat(3, DEP_DT)), pick(batch.log_lists))
    return apply_select(batch, list(range(batch.n_logs)) + [SELECT_ADDED] * n, added), status


def checkout_clocks(batch: PackedBatch, logs: Sequence[int], clocks_by_actor_id: Sequence[dict]) -> tuple[np.ndarray, np.ndarray]:
    """The clock-mode arrays of ``pt_batch_checkout``: request k's clock {actor id: seq} (``Micromerge.clock``) in log
    ``logs[k]``'s actor ranks, as (u64 offsets [n + 1], CLOCK_DT entries in rank order).  An id the log does not know is dropped
    when its seq is 0 and raises ValueError otherwise (the version would hold changes the log cannot name)."""
    off = np.zeros(len(logs) + 1, np.uint64)
    rows = []
    for k, (s, clk) in enumerate(zip(logs, clocks_by_actor_id)):
        rank = {a: r for r, a in enumerate(batch.log_actors[int(s)])}
        ent = []
        for a, seq in clk.items():
            if a not in rank:
                if int(seq):
                    raise ValueError(f"checkout_clocks: request {k}: log {int(s)} does not know actor {a!r}")
                continue
            ent.append((rank[a], int(seq)))
        rows += sorted(ent)
        off[k + 1] = len(rows)
    return off, np.array(rows, CLOCK_DT) if rows else np.zeros(0, CLOCK_DT)


def clocks(batch: PackedBatch) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The host specification of ``pt_batch_download_clocks``: (u64 offsets [n_logs + 1] = the exclusive scan of n_actors, u32
    seq, u32 status): log i's number of changes by actor rank a at seq[off[i] + a], and CHECKOUT_BAD_TABLE with zeros where its
    table fails pt_batch_exchange's clock checks."""
    n_act = batch.desc["n_actors"].astype(np.uint64)
    off = np.zeros(batch.n_logs + 1, np.uint64)
    off[1:] = np.cumsum(n_act)
    seq = np.zeros(int(off[-1]), np.uint32)
    status = np.zeros(batch.n_logs, np.uint32)
    for i in range(batch.n_logs):
        if not _clock_ok(batch, i):
            status[i] = CHECKOUT_BAD_TABLE
            continue
        ch, _ = _log_changes(batch, i)
        np.add.at(seq, int(off[i]) + ch["actor"].astype(np.int64), 1)
    return off, seq, status


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
    first_op: np.ndarray | None = None   # per log: the patch window's first list op (None: whole logs); recs and items
                                         # cover only the ops from there on

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
    startIndex, [attrs], endIndex}.  Under a patch window (``dp.first_op``) the lists are those of ``ops[first_op[i]:]``."""
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
    w0 = 0 if dp.first_op is None else int(dp.first_op[i])
    mi = sum(1 for op in ops[:w0] if op["action"] in ("addMark", "removeMark"))
    ri = w0 - mi
    for op in ops[w0:]:
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


# ------------------------------------------------------------------------------------------------------------------
# Local changes (include/peritext_b200.h pt_batch_change)
# ------------------------------------------------------------------------------------------------------------------
INPUT_OP_DT = np.dtype([("action", "u1"), ("mark_type", "u1"), ("reserved0", "<u2"), ("index", "<i4"), ("arg", "<i4"), ("attr", "<u4"),
                        ("first_ctr", "<u4"), ("reserved1", "<u4"), ("tok_off", "<u8")])
CHANGE_STATUS_DT = np.dtype([("status", "<u4"), ("input", "<u4")])
assert INPUT_OP_DT.itemsize == 32 and CHANGE_STATUS_DT.itemsize == 8
INPUT_ACTIONS = {"insert": 0, "delete": 1, "addMark": 2, "removeMark": 3}
CHANGE_OK, CHANGE_OUT_OF_BOUNDS = 0, 1
CHANGE_NO_ACTOR = 0xFFFFFFFF
INCLUSIVE_MARKS = ("strong", "em")          # markSpec.inclusive, reference src/schema.ts:45-96


class ChangeOutOfBounds(RangeError):
    """``List index out of bounds`` thrown while generating a change; ``input`` is the failing InputOperation's index."""

    def __init__(self, msg: str, input: int):
        super().__init__(msg)
        self.input = input


def _list_element_id(meta, index: int, look_after_tombstones: bool = False) -> int:
    """getListElementId (reference src/micromerge.ts:762-805) on a mirror `meta` = [[elemId, deleted, after_defined], ...]:
    the position of the element, or ChangeOutOfBounds (input -1, set by the caller)."""
    visible = -1
    for pos, e in enumerate(meta):
        if not e[1]:
            visible += 1
            if visible == index:
                if look_after_tombstones:
                    peek, latest = pos + 1, 0
                    while peek < len(meta) and meta[peek][1]:
                        if meta[peek][2]:
                            latest = peek
                        peek += 1
                    if latest:
                        return latest
                return pos
    raise ChangeOutOfBounds(f"List index out of bounds: {index}", -1)


def generate_change(meta, change: dict, list_id: str) -> dict:
    """The host specification of ``pt_batch_change`` for one document: the Change object that the reference's
    ``Micromerge.change`` (src/micromerge.ts:308-441; changeMark src/peritext.ts:458-501) returns, on a mirror of the text
    list's metadata as the facade keeps it (``meta`` = [[elemId, deleted, after_defined, ...], ...] in list order, e.g. the
    engine's element sequence or the oracle's ``elements()``; not modified).  ``change`` = {"actor", "seq", "deps",
    "startOp", "ops": [InputOperation...]}: the header is the replica's (seq / clock / maxOp + 1) and passes through.
    ROOT-map InputOperations (path []) take a counter each and touch no list.  Raises ``ChangeOutOfBounds`` naming the failing
    InputOperation (the whole change is dropped, the deviation of pt_batch_change)."""
    meta = [list(e[:3]) for e in meta]
    actor, ctr = change["actor"], int(change["startOp"])
    ops = []

    def make(body):
        nonlocal ctr
        op = {"opId": f"{ctr}@{actor}", **body}
        ctr += 1
        ops.append(op)
        return op

    def elem(k, index, look=False):
        try:
            return _list_element_id(meta, index, look)
        except ChangeOutOfBounds as e:
            raise ChangeOutOfBounds(str(e), k) from None

    for k, inp in enumerate(change["ops"]):
        path = list(inp.get("path") or [])
        action = inp["action"]
        if path == []:
            if action not in ("makeList", "makeMap", "del", "set") or inp.get("key") == "text":
                raise ValueError(f"InputOperation {k}: unsupported ROOT-map operation")
            body = {"action": action, "obj": "_root", "key": inp["key"]}
            if action == "set":
                body["value"] = inp.get("value")
            make(body)
            continue
        if path != ["text"]:
            raise ValueError(f"InputOperation {k}: no object at path {path!r}")
        visible_len = sum(1 for e in meta if not e[1])
        if action == "insert":
            pos = -1 if inp["index"] == 0 else elem(k, inp["index"] - 1, True)       # :347-350, before the values
            ref = "_head" if pos < 0 else meta[pos][0]
            for value in inp["values"]:
                if not isinstance(value, str):
                    raise TypeError("Expected value inserted into text to be a string")
                op = make({"action": "set", "obj": list_id, "elemId": ref, "insert": True, "value": value})
                pos += 1                                    # its opId exceeds every other: it lands right after its reference
                meta.insert(pos, [op["opId"], False, False])
                ref = op["opId"]
        elif action == "delete":
            for _ in range(inp["count"]):
                pos = elem(k, inp["index"])
                make({"action": "del", "obj": list_id, "elemId": meta[pos][0]})
                meta[pos][1] = True
        elif action in ("addMark", "removeMark"):
            mt = inp["markType"]
            start = {"type": "before", "elemId": meta[elem(k, inp["startIndex"])][0]}        # peritext.ts:488
            after = None
            if mt in INCLUSIVE_MARKS and inp["endIndex"] >= visible_len:
                end = {"type": "endOfText"}                                                 # :491-492
            elif mt in INCLUSIVE_MARKS:
                end = {"type": "before", "elemId": meta[elem(k, inp["endIndex"])][0]}      # :494
            else:
                after = elem(k, inp["endIndex"] - 1)
                end = {"type": "after", "elemId": meta[after][0]}                          # :496
            body = {"action": action, "obj": list_id, "start": start, "end": end, "markType": mt}
            if isinstance(inp.get("attrs"), dict):
                body["attrs"] = inp["attrs"]
            make(body)
            if after is not None:
                meta[after][2] = True
        else:
            raise ValueError(f"InputOperation {k}: unimplemented action {action!r}")
    return {"actor": actor, "seq": change["seq"], "deps": dict(change["deps"]), "startOp": change["startOp"], "ops": ops}


def change_inputs(batch: PackedBatch, changes: Sequence[dict | None], actor_ranks: Sequence[int | None]):
    """The device input of ``pt_batch_change`` for ``changes[i]`` (None: no change; else {"startOp", "ops", ...} as for
    ``generate_change``) made by actor ``batch.log_actors[i][actor_ranks[i]]``.  Returns (actor u32 [n], input_off u64
    [n + 1], INPUT_OP_DT ops, u32 tokens, values, link_attrs, counters): the value and link pools with the change's new strings
    appended (neither carries an order), and per log the counter table extended by the new counters of a dense log.  A comment
    id the batch does not know shifts ranks: ValueError (append it first)."""
    n = batch.n_logs
    actor = np.full(n, CHANGE_NO_ACTOR, np.uint32)
    off = np.zeros(n + 1, np.uint64)
    rows, tokens = [], []
    pools = _Pools(batch.values, batch.link_attrs)
    comment_rank = {c["id"]: r for r, c in enumerate(batch.comment_ids)}
    counters = list(batch.log_counters) if batch.log_counters else [None] * n
    for i in range(n):
        ch = changes[i]
        if ch is not None:
            actor[i] = actor_ranks[i]
            cmap = counters[i]
            ctr = int(ch["startOp"])                     # the original counter of the next op
            new = []                                     # original counters of a dense log's new list ops
            if cmap is not None and ctr <= int(cmap[-1]):
                raise ValueError(f"log {i}: startOp {ctr} does not exceed the log's counters")
            for inp in ch["ops"]:
                if list(inp.get("path") or []) == []:
                    ctr += 1
                    continue
                a = INPUT_ACTIONS[inp["action"]]
                first = ctr if cmap is None else len(cmap) + len(new)
                row = [a, 0, 0, 0, 0, ATTR_NONE, first, 0, len(tokens)]
                if a == 0:
                    row[3], row[4] = inp["index"], len(inp["values"])
                    tokens += [pools.token_of(v) for v in inp["values"]]
                    gen = len(inp["values"])
                elif a == 1:
                    row[3], row[4] = inp["index"], inp["count"]
                    gen = max(0, inp["count"])
                else:
                    mt = inp["markType"]
                    row[1], row[3], row[4] = MARK_TYPES.index(mt), inp["startIndex"], inp["endIndex"]
                    attrs = inp.get("attrs")
                    if mt == "link":
                        k = canon(attrs)
                        if k not in pools.link_index:
                            pools.link_index[k] = len(pools.link_attrs)
                            pools.link_attrs.append(attrs)
                        row[5] = pools.link_index[k]
                    elif mt == "comment":
                        if attrs["id"] not in comment_rank:
                            raise ValueError(f"log {i}: comment id {attrs['id']!r} is new to the batch: introduce it with an append first")
                        row[5] = comment_rank[attrs["id"]]
                    gen = 1
                rows.append(tuple(row))
                if cmap is not None:
                    new += range(ctr, ctr + gen)
                ctr += gen
            if cmap is not None:
                counters[i] = np.concatenate([cmap, np.array(new, np.uint64)])
        off[i + 1] = len(rows)
    ops = np.array(rows, INPUT_OP_DT) if rows else np.zeros(0, INPUT_OP_DT)
    return actor, off, ops, np.array(tokens, np.uint32), pools.values, pools.link_attrs, counters


def change_dicts(batch: PackedBatch, changes: Sequence[dict | None], actor_ranks, status: np.ndarray, delta: PackedBatch) -> list:
    """The Change objects of ``pt_batch_change``'s view: per log, None for no change or a failed one, else {"actor", "seq",
    "deps", "startOp", "ops"} with the generated records' packed ids turned back into strings through ``delta``'s actor and
    counter tables (the batch after the change) and the ROOT-map InputOperations in their places."""
    out = []
    for i, ch in enumerate(changes):
        if ch is None or int(status[i]["status"]) != CHANGE_OK:
            out.append(None)
            continue
        actors = delta.log_actors[i]
        cmap = delta.log_counters[i] if delta.log_counters else None
        oc = (lambda c: int(c)) if cmap is None else (lambda c: int(cmap[int(c)]))
        eid = lambda c, a: "_head" if int(c) == 0 else f"{oc(c)}@{actors[int(a)]}"
        ins, mk = delta.log_slice(i)
        lid = batch.log_lists[i]
        me, ri, mi, ops = actors[int(actor_ranks[i])], 0, 0, []
        for inp in ch["ops"]:
            if list(inp.get("path") or []) == []:        # the ops of a change have consecutive counters from startOp
                body = {"opId": f"{int(ch['startOp']) + len(ops)}@{me}", "action": inp["action"], "obj": "_root", "key": inp["key"]}
                if inp["action"] == "set":
                    body["value"] = inp.get("value")
                ops.append(body)
                continue
            a = inp["action"]
            if a == "insert":
                for v in inp["values"]:
                    r = ins[ri]; ri += 1
                    ops.append({"opId": eid(r["ctr"], r["actor"]), "action": "set", "obj": lid, "elemId": eid(r["ref_ctr"], r["ref_actor"]), "insert": True, "value": v})
            elif a == "delete":
                for _ in range(max(0, inp["count"])):
                    r = ins[ri]; ri += 1
                    ops.append({"opId": eid(r["ctr"], r["actor"]), "action": "del", "obj": lid, "elemId": eid(r["ref_ctr"], r["ref_actor"])})
            else:
                m = mk[mi]; mi += 1
                eb = BOUND_TYPES[(int(m["bounds"]) >> 2) & 3]
                end = {"type": eb} if eb == "endOfText" else {"type": eb, "elemId": eid(m["end_ctr"], m["end_actor"])}
                body = {"opId": eid(m["ctr"], m["actor"]), "action": a, "obj": lid, "start": {"type": "before", "elemId": eid(m["start_ctr"], m["start_actor"])},
                        "end": end, "markType": inp["markType"]}
                if isinstance(inp.get("attrs"), dict):
                    body["attrs"] = inp["attrs"]
                ops.append(body)
        out.append({"actor": me, "seq": ch["seq"], "deps": dict(ch["deps"]), "startOp": ch["startOp"], "ops": ops})
    return out


# ------------------------------------------------------------------------------------------------------------------
# Changes as JSON (include/peritext_b200.h pt_batch_render_changes_json)
# ------------------------------------------------------------------------------------------------------------------
EXTRA_DT = np.dtype([("log", "<u4"), ("change", "<u4"), ("pos", "<u4"), ("reserved", "<u4"), ("start_op", "<u8"), ("op", "<u8")])
CHANGES_REQUEST_DT = np.dtype([("log", "<u4"), ("mode", "<u4"), ("first", "<u4"), ("count", "<u4"), ("clock_off", "<u8"), ("n_clock", "<u4"),
                               ("reserved", "<u4")])
CLOCK_DT = np.dtype([("actor", "<u4"), ("seq", "<u4")])
assert EXTRA_DT.itemsize == 32 and CHANGES_REQUEST_DT.itemsize == 32
EXTRA_NONE = 0xFFFFFFFFFFFFFFFF
CHANGES_RANGE, CHANGES_MISSING = 0, 1
CHANGES_OK, CHANGES_BAD_TABLE = 0, 1


@dataclass
class ChangeExtras:
    """What the packed records lose of each change (pt_change_extra): one row per op that does not target the log's text list,
    at its index in ``change.ops``, with the change's startOp; a row with op == EXTRA_NONE carries only the startOp of a change
    that has no such op and either no list op or a startOp other than its first list op's counter.  ``ops[k]`` is the canonical
    JSON (``canon``) of the op of rows whose op is k."""
    rows: np.ndarray                                   # EXTRA_DT, sorted by (log, change, pos)
    ops: list[str] = field(default_factory=list)

    def pools(self) -> tuple[np.ndarray, np.ndarray]:
        """The extra-ops pool as pt_ingest_pool kind 7 holds it: UTF-8 bytes and u64 offsets [count + 1]."""
        return _pool([o.encode("utf-8", "surrogatepass") for o in self.ops])


def join_extras(*parts: ChangeExtras) -> ChangeExtras:
    """Several ChangeExtras as one (op indices re-based, rows sorted by (log, change, pos))."""
    rows, ops = [], []
    for p in parts:
        r = p.rows.copy()
        has = r["op"] != np.uint64(EXTRA_NONE)
        r["op"][has] += np.uint64(len(ops))
        rows.append(r); ops += p.ops
    r = np.concatenate(rows + [np.zeros(0, EXTRA_DT)])
    return ChangeExtras(r[np.lexsort((r["pos"], r["change"], r["log"]))], ops)


def _extra_rows(li: int, ci: int, ops: Sequence[dict], start, is_list, rows: list, out_ops: list) -> None:
    n0, first = len(rows), None
    for pos, op in enumerate(ops):
        if not is_list(op):
            rows.append((li, ci, pos, 0, int(start or 0), len(out_ops)))
            out_ops.append(canon(op))
        elif first is None:
            first = parse_op_id(op["opId"])[0]
    if len(rows) == n0 and start is not None and (first is None or first != int(start)):
        rows.append((li, ci, 0, 0, int(start), EXTRA_NONE))


def change_extras(logs: Sequence[Sequence[dict]], *, list_ids: Sequence[str | None] | None = None) -> tuple[ChangeExtras, list[str]]:
    """The host specification of the native ingest's extras (pt_ingest_change_extras, pool PT_POOL_EXTRA_OPS) and of its list-id
    pool (PT_POOL_LIST_IDS): (ChangeExtras of ``logs`` packed as ``pack_logs`` packs them, each log's text-list id or "")."""
    rows, ops, lids = [], [], []
    for li, changes in enumerate(logs):
        lid = list_ids[li] if list_ids is not None and list_ids[li] is not None else _root_text_list(changes)
        lids.append(lid or "")
        for ci, ch in enumerate(changes):
            _extra_rows(li, ci, ch["ops"], ch.get("startOp"), lambda op: lid is not None and op.get("obj") == lid, rows, ops)
    return ChangeExtras(np.array(rows, EXTRA_DT) if rows else np.zeros(0, EXTRA_DT), ops), lids


def input_extras(batch: PackedBatch, changes: Sequence[dict | None], actor_ranks, status: np.ndarray) -> ChangeExtras:
    """The extras of the changes ``pt_batch_change`` generated from ``changes`` (as for ``change_inputs``; ``batch`` = the batch
    before the call, with its change table; ``status`` = the call's rows): the ROOT-map InputOperations (path []) at their places
    in ``change.ops``, so that ``render_changes_json`` of a log's new change gives exactly the Change object ``change_dicts``
    returns.  A failed log, or one without a change, has no new change and no rows."""
    rows, ops = [], []
    for i, ch in enumerate(changes):
        if ch is None or int(status[i]["status"]) != CHANGE_OK:
            continue
        me, ctr, body = batch.log_actors[i][int(actor_ranks[i])], int(ch["startOp"]), []
        for inp in ch["ops"]:
            if list(inp.get("path") or []) == []:
                op = {"opId": f"{ctr}@{me}", "action": inp["action"], "obj": "_root", "key": inp["key"]}
                if inp["action"] == "set":
                    op["value"] = inp.get("value")
                body.append(op); ctr += 1
                continue
            a = inp["action"]
            gen = len(inp["values"]) if a == "insert" else max(0, inp["count"]) if a == "delete" else 1
            body += [{"opId": f"{ctr + k}@{me}", "obj": None} for k in range(gen)]
            ctr += gen
        ci = int(batch.changes.desc[i]["n_changes"])
        _extra_rows(i, ci, body, ch["startOp"], lambda op: "key" not in op, rows, ops)
    return ChangeExtras(np.array(rows, EXTRA_DT) if rows else np.zeros(0, EXTRA_DT), ops)


def range_requests(logs: Sequence[int], first: int = 0, count: int = 0xFFFFFFFF) -> np.ndarray:
    """RANGE requests: changes [first, first + count) of each log's table (default: the whole table)."""
    req = np.zeros(len(logs), CHANGES_REQUEST_DT)
    req["log"] = np.asarray(logs, np.uint32) if len(logs) else 0
    req["mode"] = CHANGES_RANGE; req["first"] = first; req["count"] = count
    return req


def clock_requests(batch: PackedBatch, logs: Sequence[int], clocks: Sequence[dict]) -> tuple[np.ndarray, np.ndarray]:
    """MISSING requests: what a peer whose clock is ``clocks[k]`` ({actorId: seq}) is missing from log ``logs[k]``.  Actor ids
    become the log's ranks; an actor the log does not know is dropped (it has no change there to send).  Returns (requests,
    CLOCK_DT entries)."""
    req = np.zeros(len(logs), CHANGES_REQUEST_DT)
    entries = []
    for k, (log, clock) in enumerate(zip(logs, clocks)):
        rank = {a: r for r, a in enumerate(batch.log_actors[int(log)])}
        e = [(rank[a], int(s)) for a, s in clock.items() if a in rank]
        req[k] = (int(log), CHANGES_MISSING, 0, 0, len(entries), len(e), 0)
        entries += e
    return req, np.array(entries, CLOCK_DT) if entries else np.zeros(0, CLOCK_DT)


def string_pools(batch: PackedBatch) -> dict:
    """The per-log string pools of ``pt_batch_render_changes_json`` from a PackedBatch (the layouts of pt_ingest_pool kinds 4, 5
    and 6): actors (UTF-16LE, byte offsets, u64 first [n_logs + 1]), counters (u64 entries, first [n_logs + 1]) and list ids."""
    n = batch.n_logs
    actors = [a.encode("utf-16-le", "surrogatepass") for acts in (batch.log_actors or [[]] * n) for a in acts]
    afirst = np.zeros(n + 1, np.uint64)
    afirst[1:] = np.cumsum([len(acts) for acts in (batch.log_actors or [[]] * n)], dtype=np.uint64)
    counters = [np.zeros(0, np.uint64) if c is None else np.asarray(c, np.uint64) for c in (batch.log_counters or [None] * n)]
    cfirst = np.zeros(n + 1, np.uint64)
    cfirst[1:] = np.cumsum([len(c) for c in counters], dtype=np.uint64)
    lids = _pool([(l or "").encode("utf-16-le", "surrogatepass") for l in (batch.log_lists or [""] * n)])
    a = _pool(actors)
    return {"actors": a[0], "actors_off": a[1], "actors_first": afirst, "counters": np.concatenate(counters + [np.zeros(0, np.uint64)]),
            "counters_first": cfirst, "list_ids": lids[0], "list_ids_off": lids[1]}
