"""pt_batch_render_changes_json on the device: the Change objects of resident logs as JSON text, a range of each log's table or
what a peer with a given clock is missing (getMissingChanges, reference test/merge.ts:25-38).

``render_log_spec`` below is the readable specification of the bytes.  The device output must equal it byte for byte, decode
to the Change objects the logs were made of, and re-ingest (pt_ingest_parse) to exactly the batch it came from."""
import json

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200 import workload
from peritext_b200.packing import (ATTR_NONE, BOUND_TYPES, CHANGES_BAD_TABLE, CHANGES_MISSING, CHANGES_OK, CHANGES_REQUEST_DT, CLOCK_DT, EXTRA_DT,
                                   EXTRA_NONE, KIND_INSERT, MARK_TYPES, ChangeExtras, ChangeTable, apply_exchange, canon, change_extras,
                                   clock_requests, exchange_maps, input_extras, join_extras, pack_logs, range_requests, token_str)
from tests.harness import fuzz_session, generateDocs, getMissingChanges

PT_ERR_INVALID, PT_ERR_STATE = 1, 4
S = 1024            # list ops per work item (changes_json_kernel.cuh kSlice)

_ESC = {0x22: '\\"', 0x5C: "\\\\", 8: "\\b", 9: "\\t", 10: "\\n", 12: "\\f", 13: "\\r"}


def js_str(s: str) -> str:
    """A string as JSON.stringify writes it (the span render's rules): the escapes above, \\u00xx below U+0020, a surrogate pair
    as one character, a lone surrogate as \\udxxx, everything else raw."""
    b = s.encode("utf-16-le", "surrogatepass")
    u = [b[i] | b[i + 1] << 8 for i in range(0, len(b), 2)]
    out, i = ['"'], 0
    while i < len(u):
        c = u[i]
        if 0xD800 <= c < 0xDC00 and i + 1 < len(u) and 0xDC00 <= u[i + 1] < 0xE000:
            out.append(chr(0x10000 + ((c - 0xD800) << 10) + u[i + 1] - 0xDC00)); i += 2
            continue
        out.append("\\u%04x" % c if 0xD800 <= c < 0xE000 or (c < 0x20 and c not in _ESC) else _ESC.get(c, chr(c)))
        i += 1
    return "".join(out) + '"'


def frag(text: str) -> str:
    """A pool fragment: verbatim, a lone surrogate (its 3-byte encoding in the pool) as \\udxxx."""
    return "".join("\\u%04x" % ord(ch) if 0xD800 <= ord(ch) < 0xE000 else ch for ch in text)


def render_log_spec(batch, extras: ChangeExtras, log: int, changes) -> bytes:
    """The Change[] JSON of changes `changes` (indices into the log's table, in output order) of log `log` of `batch`."""
    actors = batch.log_actors[log]
    cmap = batch.log_counters[log] if batch.log_counters else None
    oc = (lambda c: int(c)) if cmap is None or not len(cmap) else (lambda c: int(cmap[int(c)]))
    eid = lambda c, a: '"_head"' if int(c) == 0 else js_str(f"{oc(c)}@{actors[int(a)]}")
    lid = js_str(batch.log_lists[log] or "")
    ins, mk = batch.log_slice(log)
    n = len(ins)
    order, k = [], 0                           # list ops in arrival order: mark k right before ins/del record arrival_k
    for j in range(n + 1):
        while k < len(mk) and min(int(mk[k]["arrival"]), n) == j:
            order.append(("m", k)); k += 1
        if j < n:
            order.append(("i", j))

    def bound(t, c, a):
        return '{"type":"%s"}' % BOUND_TYPES[t] if t >= 2 else '{"elemId":%s,"type":"%s"}' % (eid(c, a), BOUND_TYPES[t])

    def op_text(kind, j):
        if kind == "i":
            r = ins[j]
            if int(r["payload"]) >> 30 == KIND_INSERT:
                return '{"action":"set","elemId":%s,"insert":true,"obj":%s,"opId":%s,"value":%s}' % (
                    eid(r["ref_ctr"], r["ref_actor"]), lid, eid(r["ctr"], r["actor"]), js_str(token_str(int(r["payload"]) & 0x3FFFFFFF, batch.values)))
            return '{"action":"del","elemId":%s,"obj":%s,"opId":%s}' % (eid(r["ref_ctr"], r["ref_actor"]), lid, eid(r["ctr"], r["actor"]))
        m = mk[j]
        t = (int(m["kind"]) >> 1) & 3
        attrs = ""
        if int(m["attr"]) != ATTR_NONE:
            a = batch.link_attrs[int(m["attr"])] if t == 3 else batch.comment_ids[int(m["attr"])]
            attrs = '"attrs":%s,' % frag(canon(a))
        return '{"action":"%s",%s"end":%s,"markType":"%s","obj":%s,"opId":%s,"start":%s}' % (
            "removeMark" if int(m["kind"]) & 1 else "addMark", attrs, bound((int(m["bounds"]) >> 2) & 3, m["end_ctr"], m["end_actor"]),
            MARK_TYPES[t], lid, eid(m["ctr"], m["actor"]), bound(int(m["bounds"]) & 3, m["start_ctr"], m["start_actor"]))

    t = batch.changes
    cd = t.desc[log]
    crec = t.changes[int(cd["change_off"]): int(cd["change_off"]) + int(cd["n_changes"])]
    deps = t.deps[int(cd["dep_off"]): int(cd["dep_off"]) + int(cd["n_deps"])]
    pos = np.concatenate([[0], np.cumsum(crec["n_ops"].astype(np.int64))])
    rows = extras.rows[extras.rows["log"] == log]
    out = []
    for c in changes:
        r = crec[c]
        lops = [op_text(*x) for x in order[int(pos[c]): int(pos[c]) + int(r["n_ops"])]]
        mine = rows[rows["change"] == c]
        ex = [(int(x["pos"]), frag(extras.ops[int(x["op"])])) for x in mine if int(x["op"]) != EXTRA_NONE]
        ops, it = [None] * (len(lops) + len(ex)), iter(lops)
        for p, txt in ex:
            ops[p] = txt
        ops = [o if o is not None else next(it) for o in ops]
        if len(mine):
            start = int(mine[0]["start_op"])
        else:
            kind, j = order[int(pos[c])]
            start = oc((ins if kind == "i" else mk)[j]["ctr"])
        dd = deps[int(r["dep_off"]): int(r["dep_off"]) + int(r["n_deps"])]
        out.append('{"actor":%s,"deps":{%s},"ops":[%s],"seq":%d,"startOp":%d}' % (
            js_str(actors[int(r["actor"])]), ",".join("%s:%d" % (js_str(actors[int(d["actor"])]), int(d["seq"])) for d in dd), ",".join(ops),
            int(r["seq"]), start))
    return ("[" + ",".join(out) + "]").encode("utf-8", "surrogatepass")


def engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, **kw)


def ingest(logs):
    from peritext_b200.engine import ingest_native
    return ingest_native([json.dumps(l, ensure_ascii=False).encode("utf-8", "surrogatepass") if not isinstance(l, (str, bytes)) else l for l in logs])


def resident(batch):
    e = engine(emit_patches=True)
    e.upload(batch)
    e.upload_changes(batch.changes)
    return e


def whole(batch):
    return range_requests(range(batch.n_logs))


def decode(b: bytes):
    return json.loads(b.decode("utf-8", "surrogatepass"))


def same_ingest(a, b):
    """Two native ingests are byte-identical: records, descriptors, change table, extras and pools 0-7."""
    (ba, xa, ra), (bb, xb, rb) = a, b
    for f in ("desc", "insdel", "marks"):
        assert getattr(ba, f).tobytes() == getattr(bb, f).tobytes(), f
    for f in ("desc", "changes", "deps"):
        assert getattr(ba.changes, f).tobytes() == getattr(bb.changes, f).tobytes(), f
    assert xa.rows.tobytes() == xb.rows.tobytes() and xa.ops == xb.ops
    for k in range(8):
        assert ra[k][0] == rb[k][0] and ra[k][1].tolist() == rb[k][1].tolist(), k
        assert (ra[k][2] is None) == (rb[k][2] is None) and (ra[k][2] is None or ra[k][2].tolist() == rb[k][2].tolist()), k


def with_head(lg):
    return [dict(ch, ops=[dict(op, elemId=op.get("elemId", "_head")) if op.get("insert") else op for op in ch["ops"]]) for ch in lg]


# ------------------------------------------------------------------------------------------------------------------
# 1. Exactness and the round trip
# ------------------------------------------------------------------------------------------------------------------
from tests.test_change_extras import CORPORA


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CORPORA))
def test_whole_logs_render_exactly_and_round_trip(name):
    logs = CORPORA[name]()
    first = ingest(logs)
    batch, extras, _ = first
    e = resident(batch)
    try:
        got = e.render_changes_json_list(batch, whole(batch), extras)
        _, _, status = e.render_changes_json(batch, whole(batch), extras)
        assert (status == CHANGES_OK).all()
        for i, lg in enumerate(logs):
            assert got[i] == render_log_spec(batch, extras, i, range(len(lg)))
            if name != "links_minimal":                          # that trace lost its Symbol fields: HEAD has no elemId there
                assert decode(got[i]) == with_head(lg)
        same_ingest(ingest(got), first)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["c2", "c3", "c4"])
def test_generated_batches_round_trip(config):
    g = workload.generate(config, n_docs=40, seed=5)
    logs = [workload.to_change_json(g, i) for i in range(g.n_logs)]
    first = ingest(logs)
    batch, extras, _ = first
    e = resident(batch)
    try:
        got = e.render_changes_json_list(batch, whole(batch), extras)
        for i in range(0, g.n_logs, 7):
            assert got[i] == render_log_spec(batch, extras, i, range(int(batch.changes.desc[i]["n_changes"])))
        assert [decode(b) for b in got] == [json.loads(s) for s in logs]
        same_ingest(ingest(got), first)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. Sync: MISSING against the harness's getMissingChanges
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed", [11, 12, 13])
def test_missing_is_get_missing_changes(seed):
    docs, logs, queues = fuzz_session(O, seed, 60, replicas=3, sync_prob=0.3, full_sync_at_end=False)
    batch, extras, _ = ingest(logs)
    e = resident(batch)
    try:
        pairs = [(s, d) for s in range(3) for d in range(3) if s != d]
        clocks = [dict(docs[d].clock) for _, d in pairs]
        extra = [{}, dict(docs[0].clock), {"nobody": 3, **{a: 10 ** 6 for a in docs[1].clock}}, {a: s + 1000 for a, s in docs[2].clock.items()}]
        logs_req = [s for s, _ in pairs] + [0, 0, 1, 2]
        req = clock_requests(batch, logs_req, clocks + extra)
        got = e.render_changes_json_list(batch, req, extras)
        def table_index(s, changes):       # the changes' indices in log s's table, which holds each (actor, seq) once
            at = {(ch["actor"], ch["seq"]): k for k, ch in enumerate(logs[s])}
            return [at[(ch["actor"], ch["seq"])] for ch in changes]

        for k, (s, d) in enumerate(pairs):
            want = getMissingChanges(docs[s], docs[d], queues)
            assert decode(got[k]) == with_head(want)
            assert got[k] == render_log_spec(batch, extras, s, table_index(s, want))          # the bytes, in sync order
        empty = type("Peer", (), {"clock": {}})()
        want = getMissingChanges(docs[0], empty, queues)
        assert decode(got[len(pairs)]) == with_head(want)                                    # an empty clock: all, in sync order
        assert got[len(pairs)] == render_log_spec(batch, extras, 0, table_index(0, want))
        assert got[len(pairs) + 1] == b"[]"                                      # a full clock
        assert got[len(pairs) + 2] == b"[]"                                      # unknown actors and seqs past the log
        assert got[len(pairs) + 3] == b"[]"
        _, off, status = e.render_changes_json(batch, req, extras)
        assert (status == CHANGES_OK).all()
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. Resident flows: change (with a ROOT InputOperation), exchange, append, failed merges
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_after_change_the_last_change_is_the_returned_change():
    docs, _, init = generateDocs(O, "hello", 2)
    logs = [[init], [init]]
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0, emit_sequence=True)
    try:
        e.upload(batch); e.upload_changes(batch.changes)
        e.merge(); e.download()
        inputs = [{"seq": 2, "deps": {"doc1": 1}, "startOp": 7, "ops": [{"path": [], "action": "makeMap", "key": "meta"},
                   {"path": ["text"], "action": "insert", "index": 2, "values": ["x", "y"]},
                   {"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 3, "markType": "link", "attrs": {"url": "u"}},
                   {"path": [], "action": "set", "key": "title", "value": "t"}]},
                  {"seq": 2, "deps": {"doc1": 1}, "startOp": 7, "ops": [{"path": ["text"], "action": "delete", "index": 0, "count": 0}]}]
        ranks = [0, 0]                                   # log 1's change generates no op: only its extra gives its startOp
        new = ChangeTable(*_new_table(batch, inputs, ranks))
        after, objs, status = e.change(batch, inputs, ranks, new)
        x = join_extras(extras, input_extras(batch, inputs, ranks, status))
        req = range_requests([0, 1], first=1, count=1)
        got = e.render_changes_json_list(after, req, x)
        for i in range(2):
            assert decode(got[i]) == [objs[i]]
            assert got[i] == render_log_spec(after, x, i, [1])
    finally:
        e.close()


def _new_table(batch, inputs, ranks):
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, INPUT_ACTIONS
    n = batch.n_logs
    cd = np.zeros(n, CDESC_DT); ch = np.zeros(n, CHANGE_DT); dp = []
    for i, inp in enumerate(inputs):
        cd[i]["change_off"] = i; cd[i]["n_changes"] = 1; cd[i]["dep_off"] = len(dp); cd[i]["n_deps"] = len(inp["deps"])
        n_ops = 0
        for o in inp["ops"]:
            if o.get("path") == []:
                continue
            n_ops += len(o["values"]) if o["action"] == "insert" else max(0, o["count"]) if o["action"] == "delete" else 1
        ch[i] = (inp["seq"], ranks[i], len(inp["deps"]), 0, n_ops)
        rank = {a: r for r, a in enumerate(batch.log_actors[i])}
        dp += [(s, rank[a], 0) for a, s in inp["deps"].items()]
    return cd, ch, np.array(dp, DEP_DT)


@pytest.mark.gpu
def test_after_exchange_and_append_and_before_any_merge():
    docs, logs, queues = fuzz_session(O, 21, 40, replicas=3, sync_prob=0.3, full_sync_at_end=False)
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    e = resident(batch)
    try:
        assert e.render_changes_json_list(batch, whole(batch), extras) == [render_log_spec(batch, extras, i, range(len(l))) for i, l in enumerate(logs)]
        pairs = [(0, 1), (1, 2)]
        maps, pre = exchange_maps(batch, pairs)
        cur = batch
        if pre is not None:
            from peritext_b200.packing import apply_append
            e.append(*pre); cur = apply_append(cur, *pre)
        want, st, delivered, _ = apply_exchange(cur, pairs, maps)
        e.exchange(pairs, maps)
        new_logs = list(logs)                                  # dst received src's changes, in delivery order
        for (src, dst), dl in zip(pairs, delivered):
            new_logs[dst] = logs[dst] + [logs[src][k] for k in dl]
        x2, _ = change_extras(new_logs)
        got = e.render_changes_json_list(want, whole(want), x2)
        for i, lg in enumerate(new_logs):
            assert got[i] == render_log_spec(want, x2, i, range(len(lg)))
            assert decode(got[i]) == with_head(lg)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Edges
# ------------------------------------------------------------------------------------------------------------------
def one_big_change(n_ops: int, actor="a"):
    lid = f"1@{actor}"
    ops = [{"opId": lid, "action": "makeList", "obj": "_root", "key": "text"}]
    prev = "_head"
    for k in range(n_ops):
        oid = f"{k + 2}@{actor}"
        ops.append({"opId": oid, "action": "set", "obj": lid, "elemId": prev, "insert": True, "value": "abcdefg"[k % 7]})
        prev = oid
    return [{"actor": actor, "seq": 1, "deps": {}, "startOp": 1, "ops": ops}]


@pytest.mark.gpu
def test_slices_at_the_item_boundary_and_a_c5_sized_change():
    logs = [one_big_change(n) for n in (S - 1, S, S + 1, 2 * S, 111_000)]
    logs.append([{"actor": "m", "seq": 1, "deps": {}, "startOp": 1, "ops": [{"opId": "1@m", "action": "makeList", "obj": "_root", "key": "text"}]},
                 {"actor": "m", "seq": 2, "deps": {"m": 1}, "startOp": 2, "ops": [
                     {"opId": "2@m", "action": "set", "obj": "1@m", "elemId": "_head", "insert": True, "value": "x"},
                     {"opId": "3@m", "action": "addMark", "obj": "1@m", "start": {"type": "startOfText"}, "end": {"type": "endOfText"}, "markType": "strong"},
                     {"opId": "4@m", "action": "makeMap", "obj": "_root", "key": "z"}]}])
    first = ingest(logs)
    batch, extras, _ = first
    e = resident(batch)
    try:
        got = e.render_changes_json_list(batch, whole(batch), extras)
        for i, lg in enumerate(logs):
            assert got[i] == render_log_spec(batch, extras, i, range(len(lg)))
            assert decode(got[i]) == lg
        same_ingest(ingest(got), first)
        assert e.render_changes_json_list(batch, whole(batch), extras) == got            # two calls: identical bytes
    finally:
        e.close()


@pytest.mark.gpu
def test_a_true_shape_c5_change():
    """A generated c5 document's history as one change (workload.history_table): about 111 K list ops with 10 K dense overlapping
    marks, so the slices' mark-slot masks and cuts run at every slice of a long change."""
    from peritext_b200.packing import _pool
    g = workload.generate("c5", n_docs=1)
    g.changes = workload.history_table(g)
    g.log_actors = [["doc%d" % (r + 1) for r in range(int(a))] for a in g.desc["n_actors"]]
    g.log_lists = ["1@doc1"] * g.n_logs
    g.log_counters = [None] * g.n_logs
    com = (g.marks["kind"] >> 1) & 3 == 2
    n_com = int(g.marks["attr"][com].max()) + 1 if com.any() else 0
    pools = _pool([]) + _pool([canon(a).encode() for a in g.link_attrs]) + _pool([canon(g.comment_ids[k]).encode() for k in range(n_com)])
    none = ChangeExtras(np.zeros(0, EXTRA_DT), [])
    assert int(g.changes.changes["n_ops"].min()) > 100 * S and len(g.marks) >= 10_000
    e = resident(g)
    try:
        data, off, status = e.render_changes_json(g, whole(g), None, pools)
        assert (status == CHANGES_OK).all()
        raw = data.tobytes()
        for i in range(g.n_logs):
            assert raw[int(off[i]): int(off[i + 1])] == render_log_spec(g, none, i, [0])
    finally:
        e.close()


@pytest.mark.gpu
def test_ranges_empty_logs_and_tampered_tables():
    docs, logs, _ = fuzz_session(O, 31, 30, replicas=2, sync_prob=0.5, full_sync_at_end=False)
    logs = logs + [[]]                                                                   # a log without changes
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    e = resident(batch)
    try:
        n0 = len(logs[0])
        req = np.concatenate([range_requests([0], 0, 0), range_requests([0], n0 + 5, 3), range_requests([0], n0 - 2, 10), range_requests([2]),
                              range_requests([1], 3, 4)])
        got = e.render_changes_json_list(batch, req, extras)
        assert got[:2] == [b"[]", b"[]"] and got[3] == b"[]"
        assert got[2] == render_log_spec(batch, extras, 0, [n0 - 2, n0 - 1])
        assert got[4] == render_log_spec(batch, extras, 1, range(3, 7))
        # a table that is not seq-contiguous: MISSING is BAD_TABLE with zero bytes, RANGE still renders
        t = batch.changes
        bad = ChangeTable(t.desc.copy(), t.changes.copy(), t.deps.copy())
        bad.changes[int(t.desc[0]["change_off"]) + 3]["seq"] += 7
        e.upload_changes(bad)
        req2, clk = clock_requests(batch, [0, 1], [{}, {}])
        data, off, status = e.render_changes_json(batch, (np.concatenate([req2, range_requests([0])]), clk), extras)
        assert status.tolist() == [CHANGES_BAD_TABLE, CHANGES_OK, CHANGES_OK] and int(off[1]) == int(off[0]) == 0
        # n_ops that do not sum to the log's records: BAD_TABLE in every mode
        bad2 = ChangeTable(t.desc.copy(), t.changes.copy(), t.deps.copy())
        bad2.changes[int(t.desc[1]["change_off"])]["n_ops"] += 1
        e.upload_changes(bad2)
        _, _, status = e.render_changes_json(batch, whole(batch), extras)
        assert status.tolist() == [CHANGES_OK, CHANGES_BAD_TABLE, CHANGES_OK]
        # a change whose deps leave the log's dep records: BAD_TABLE in every mode, nothing read past the deps
        bad3 = ChangeTable(t.desc.copy(), t.changes.copy(), t.deps.copy())
        c0 = int(t.desc[0]["change_off"])
        k = c0 + int(np.flatnonzero(t.changes[c0: c0 + n0]["n_deps"] > 0)[0])
        bad3.changes[k]["dep_off"] = 0xFFFFFF00
        e.upload_changes(bad3)
        req3, clk3 = clock_requests(batch, [0], [{}])
        data, off, status = e.render_changes_json(batch, (np.concatenate([range_requests([0, 1]), range_requests([0], k - c0, 1), req3]), clk3), extras)
        assert status.tolist() == [CHANGES_BAD_TABLE, CHANGES_OK, CHANGES_BAD_TABLE, CHANGES_BAD_TABLE]
        assert off.tolist() == [0, 0, int(off[2]), int(off[2]), int(off[2])] and off[2] > 0
    finally:
        e.close()


@pytest.mark.gpu
def test_logs_whose_merge_failed():
    """A log that admission rejects (a sequence gap) and one whose records fail the merge (an insert whose reference is moved to
    the log's largest counter) still render after the merge: RANGE needs neither causal order nor a merged document."""
    docs, logs, _ = fuzz_session(O, 61, 30, replicas=3, sync_prob=0.5, full_sync_at_end=False)
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    t = batch.changes
    gap = ChangeTable(t.desc.copy(), t.changes.copy(), t.deps.copy())
    gap.changes[int(t.desc[0]["change_off"]) + 2]["seq"] += 5                    # log 0: "Expected sequence number"
    batch.changes = gap
    i0 = int(batch.desc[1]["insdel_off"])
    ins = np.flatnonzero(batch.insdel[i0: i0 + int(batch.desc[1]["n_insdel"])]["ref_ctr"] > 0)
    batch.insdel[i0 + int(ins[-1])]["ref_ctr"] = batch.desc[1]["max_ctr"]        # log 1: the reference does not precede it
    e = resident(batch)
    try:
        e.merge()
        st = e.results()["status"].tolist()
        assert st[0] == 6 and st[1] != 0 and st[2] == 0
        got = e.render_changes_json_list(batch, whole(batch), extras)
        for i, lg in enumerate(logs):
            assert got[i] == render_log_spec(batch, extras, i, range(len(lg)))
        assert decode(got[2]) == with_head(logs[2])
    finally:
        e.close()


def missing_pool(e, batch, extras, match, **fields):
    from peritext_b200.engine import EngineError
    short = type(batch)(**{**batch.__dict__, **fields})
    with pytest.raises(EngineError, match=match):
        e.render_changes_json(short, whole(batch), extras)


@pytest.mark.gpu
def test_missing_pool_entries():
    """Every pool the output reads names the first entry it lacks: link and comment attrs, actors, and the counters of a log whose
    counters were re-ranked."""
    from tests.test_change_extras import sparse_logs, unicode_logs
    logs = unicode_logs()
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    mt = (batch.marks["kind"] >> 1) & 3
    assert (mt == 3).any() and (mt == 2).any()                                   # the corpus holds link and comment marks
    e = resident(batch)
    try:
        missing_pool(e, batch, extras, "names link pool entry 0", link_attrs=[])
        missing_pool(e, batch, extras, "names comment pool entry", comment_ids=batch.comment_ids[:1])
        missing_pool(e, batch, extras, "log 1 names actor 1, which the caller's actor pool does not hold",
                     log_actors=[batch.log_actors[0], batch.log_actors[1][:1]])
    finally:
        e.close()
    logs = sparse_logs()
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    assert batch.log_counters[0] is not None
    e = resident(batch)
    try:
        assert e.render_changes_json_list(batch, whole(batch), extras)[0] == render_log_spec(batch, extras, 0, range(len(logs[0])))
        missing_pool(e, batch, extras, "log 0 names counter 3, which the caller's counter pool does not hold", log_counters=[batch.log_counters[0][:3]])
    finally:
        e.close()


@pytest.mark.gpu
def test_refusals():
    from peritext_b200.engine import EngineError
    docs, logs, _ = fuzz_session(O, 41, 20, replicas=2, sync_prob=0.5, full_sync_at_end=False)
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    e = engine()
    try:
        e.upload(batch)
        with pytest.raises(EngineError, match="no change table"):
            e.render_changes_json(batch, whole(batch), extras)
        e.upload_changes(batch.changes)
        assert e.render_changes_json(batch, range_requests([]), extras)[1].tolist() == [0]
        req, clk = clock_requests(batch, [0], [{}])
        clk = np.array([(int(batch.desc[0]["n_actors"]), 1)], CLOCK_DT)
        req["n_clock"] = 1
        with pytest.raises(EngineError, match="clock entry 0 names actor"):
            e.render_changes_json(batch, (req, clk), extras)
        rev = ChangeExtras(extras.rows[::-1].copy(), extras.ops)
        with pytest.raises(EngineError, match="not sorted"):
            e.render_changes_json(batch, whole(batch), rev)
        none = ChangeExtras(np.zeros(0, EXTRA_DT), [])
        with pytest.raises(EngineError, match="neither list ops nor extras"):       # the first change's only op in a log without text ops
            lone = [[{"actor": "a", "seq": 1, "deps": {}, "startOp": 1, "ops": [{"opId": "1@a", "action": "makeList", "obj": "_root", "key": "text"}]}]]
            b2 = pack_logs(lone, with_changes=True)
            e2 = resident(b2)
            try:
                e2.render_changes_json(b2, whole(b2), none)
            finally:
                e2.close()
    finally:
        e.close()


@pytest.mark.gpu
def test_no_interference_with_the_other_outputs():
    from tests.test_gpu_append import canon as mcanon, merged
    docs, logs, _ = fuzz_session(O, 51, 40, replicas=3, sync_prob=0.5, full_sync_at_end=False)
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    e = resident(batch)
    try:
        m0 = merged(e)
        spans0 = e.render_json_list(batch); patches0 = e.render_patches_json_list(batch)
        p0 = e.download_patches()
        a = e.render_changes_json_list(batch, whole(batch), extras)
        assert mcanon(e.download()) == mcanon(m0)
        assert e.render_json_list(batch) == spans0 and e.render_patches_json_list(batch) == patches0
        p1 = e.download_patches()
        assert all(np.array_equal(x, y) for x, y in zip(p0[:3], p1[:3])) and p0[3] == p1[3]
        assert e.render_changes_json_list(batch, whole(batch), extras) == a
    finally:
        e.close()
