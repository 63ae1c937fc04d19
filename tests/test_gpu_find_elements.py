"""Batched elemId -> position resolution (pt_batch_find_elements): the device form of findListElement (reference
src/micromerge.ts:731-755), whose `.visible` is resolveCursor (:475-477).

CPU: `packing.elem_refs`, which turns "ctr@actor" strings into the packed ids the device query takes, and masks the ids that
cannot exist in their log.  GPU: every element of every replica of seeded fuzz sessions against the oracle's element sequence
and resolveCursor, the reference's cursor KATs, the round trip with pt_batch_query_elements on a c4-shaped batch, every
merge-kernel route case in every kernel configuration against the downloaded sequence, large c5 / c2 documents, and the edge
cases of the entry point."""
import json
import random

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.engine import pack_logs_native
from peritext_b200.packing import (ELEM_AFTER_DEFINED, ELEM_DELETED, ELEM_LOG_FAILED, ELEM_NOT_FOUND, ELEM_REF_DT, KIND_INSERT,
                                   elem_refs, pack_logs)
from tests.harness import fuzz_session, generateDocs, load_kats

NF = ELEM_NOT_FOUND


def list_ops(log):
    """(opId, action) of every op of the log that targets its text list (the ops pack_logs packs)."""
    lid = next(op["opId"] for op in log[0]["ops"] if op["action"] == "makeList")
    return [(op["opId"], op["action"]) for ch in log for op in ch["ops"] if op.get("obj") == lid]


def elem_id(batch, i, rec):
    ins, _ = batch.log_slice(i)
    r = ins[int(rec)]
    cmap = batch.log_counters[i] if batch.log_counters else None
    ctr = int(r["ctr"]) if cmap is None else int(cmap[int(r["ctr"])])
    return f"{ctr}@{batch.log_actors[i][int(r['actor'])]}"


def unpack_ref(batch, ref):
    """The elemId string a packed ref stands for (inverse of elem_refs)."""
    i = int(ref["log"])
    cmap = batch.log_counters[i] if batch.log_counters else None
    ctr = int(ref["ctr"]) if cmap is None else int(cmap[int(ref["ctr"])])
    return f"{ctr}@{batch.log_actors[i][int(ref['actor'])]}"


def sparse_counter_logs():
    """A log the packer re-ranks (a peer picked startOp 5 000 000, reference src/micromerge.ts:511 allows any)."""
    docs, _, init = generateDocs(O, "abc", 2)
    big = {"actor": "doc2", "seq": 1, "deps": {"doc1": 1}, "startOp": 5_000_000, "ops": [
        {"opId": "5000000@doc2", "action": "set", "obj": "1@doc1", "elemId": "2@doc1", "insert": True, "value": "X"},
        {"opId": "5000001@doc2", "action": "set", "obj": "1@doc1", "elemId": "5000000@doc2", "insert": True, "value": "Y"},
        {"opId": "5000003@doc2", "action": "del", "obj": "1@doc1", "elemId": "3@doc1"},
        {"opId": "5000007@doc2", "action": "addMark", "obj": "1@doc1", "start": {"type": "before", "elemId": "5000000@doc2"},
         "end": {"type": "after", "elemId": "4@doc1"}, "markType": "link", "attrs": {"url": "u"}}]}
    return [[init, big]]


def unicode_actor_logs():
    """Actor ids whose JS (UTF-16 code unit) order differs from code-point order, plus a non-ASCII BMP id."""
    return [[{"actor": "\U00010000", "seq": 1, "deps": {}, "startOp": 1, "ops": [
        {"opId": "1@\U00010000", "action": "makeList", "obj": "_root", "key": "text"},
        {"opId": "2@\U00010000", "action": "set", "obj": "1@\U00010000", "elemId": "_head", "insert": True, "value": "x"}]},
        {"actor": "￿", "seq": 1, "deps": {"\U00010000": 1}, "startOp": 3, "ops": [
            {"opId": "3@￿", "action": "set", "obj": "1@\U00010000", "elemId": "2@\U00010000", "insert": True, "value": "y"}]},
        {"actor": "é", "seq": 1, "deps": {"￿": 1}, "startOp": 4, "ops": [
            {"opId": "4@é", "action": "set", "obj": "1@\U00010000", "elemId": "3@￿", "insert": True, "value": "z"},
            {"opId": "5@é", "action": "del", "obj": "1@\U00010000", "elemId": "2@\U00010000"}]}]]


# ------------------------------------------------------------------------------------------------------------------
# CPU: elem_refs
# ------------------------------------------------------------------------------------------------------------------
def test_elem_refs_ranks_actors_in_utf16_order():
    logs = unicode_actor_logs()
    batch = pack_logs(logs)
    assert batch.log_actors[0] == ["é", "\U00010000", "￿"]     # surrogate pair D800.. sorts before FFFF
    refs, ok = elem_refs(batch, [0, 0, 0, 0], ["2@\U00010000", "3@￿", "4@é", "5@é"])
    assert ok.all()
    assert refs["actor"].tolist() == [1, 2, 0, 0] and refs["ctr"].tolist() == [2, 3, 4, 5] and refs["log"].tolist() == [0, 0, 0, 0]
    ins, _ = batch.log_slice(0)
    # every insert's packed opId is what elem_refs makes of its string
    for r in ins[(ins["payload"] >> 30) == KIND_INSERT]:
        k = np.flatnonzero((refs["ctr"] == r["ctr"]) & (refs["actor"] == r["actor"]))
        assert len(k) == 1


def test_elem_refs_maps_reranked_counters():
    logs = sparse_counter_logs()
    batch = pack_logs(logs)
    cmap = batch.log_counters[0]
    assert cmap is not None and int(batch.desc[0]["max_ctr"]) < 20
    ids = [op for op, _ in list_ops(logs[0])]
    refs, ok = elem_refs(batch, [0] * len(ids), ids)
    assert ok.all()
    ins, mk = batch.log_slice(0)
    packed = {(int(r["ctr"]), int(r["actor"])) for r in ins} | {(int(r["ctr"]), int(r["actor"])) for r in mk}
    assert {(int(r["ctr"]), int(r["actor"])) for r in refs} == packed
    big = ids.index("5000000@doc2")
    assert int(refs["ctr"][big]) == int(np.searchsorted(cmap, 5_000_000)) and int(refs["ctr"][big]) < 20
    for k, s in enumerate(ids):
        assert unpack_ref(batch, refs[k]) == s


def test_elem_refs_masks_ids_that_cannot_exist():
    logs = sparse_counter_logs() + unicode_actor_logs()
    batch = pack_logs(logs)
    assert batch.log_counters[0] is not None and batch.log_counters[1] is None
    cases = [
        (0, "5000002@doc2", "counter missing from the re-rank table"),
        (0, "4999999@doc2", "counter below the table's entries"),
        (0, "9000000@doc2", "counter beyond the table"),
        (0, "1@nobody", "unknown actor"),
        (1, "2@doc1", "actor of another log"),
        (1, "1@", "empty actor"),
        (0, "_head", "HEAD"),
        (1, "_head", "HEAD"),
        (1, "abc", "malformed"),
        (1, "@é", "no counter"),
        (1, "-1@é", "negative counter"),
        (1, " 4@é", "leading space"),
        (1, "4@é ", "trailing space on the actor"),
        (1, None, "not a string"),
        (1, "4294967296@é", "counter beyond 32 bits"),
        (2, "4@é", "log outside the batch"),
        (-1, "4@é", "negative log"),
    ]
    refs, ok = elem_refs(batch, [c[0] for c in cases], [c[1] for c in cases])
    for (log, s, why), good in zip(cases, ok):
        assert not good, why
    assert (refs["ctr"] == 0).all()
    # ... next to ids that do exist (the device answers not-found for ctr 0 / ctr > max_ctr itself)
    refs, ok = elem_refs(batch, [1, 1, 0, 0], ["4@é", "0@é", "2@doc1", "0@doc1"])
    assert ok.tolist() == [True, True, True, True] and refs["ctr"].tolist()[:2] == [4, 0]


@pytest.mark.parametrize("seed", range(3))
def test_elem_refs_same_for_python_and_native_packers(seed):
    _, logs, _ = fuzz_session(O, 9100 + seed, 120)
    logs = logs + sparse_counter_logs() + unicode_actor_logs()
    qlog, qid = [], []
    for i, log in enumerate(logs):
        for op, _ in list_ops(log):
            qlog.append(i); qid.append(op)
        qlog += [i, i, i]; qid += ["_head", "1@nobody", "x@doc2"]
    py = pack_logs(logs, with_changes=True)
    nat = pack_logs_native([json.dumps(l) for l in logs])
    a, oka = elem_refs(py, qlog, qid)
    b, okb = elem_refs(nat, qlog, qid)
    assert a.tobytes() == b.tobytes() and (oka == okb).all()
    plain = pack_logs(logs)
    c, okc = elem_refs(plain, qlog, qid)
    assert (okc == oka).all() and int(oka.sum()) == len(qid) - 3 * len(logs)
    for k in np.flatnonzero(okc):
        assert unpack_ref(plain, c[k]) == qid[k] and unpack_ref(nat, b[k]) == qid[k]


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sengine():
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0, emit_sequence=True)
    yield e
    e.close()


def expected_positions(batch, merged, i):
    """From the downloaded sequence of log i, per ins/del record of the log: (index, visible, flags), the inverse permutation
    and an exclusive prefix count of the non-deleted elements; records that are not elements get (NF, 0, 0)."""
    s = merged.sequence(i).astype(np.int64)
    n = int(batch.desc[i]["n_insdel"])
    rec, dead, after = s & 0x3FFFFFFF, (s >> 31) & 1, (s >> 30) & 1
    index = np.full(n, NF, np.int64); visible = np.zeros(n, np.int64); flags = np.zeros(n, np.int64)
    index[rec] = np.arange(len(s))
    visible[rec] = np.concatenate([[0], np.cumsum(1 - dead)[:-1]]) if len(s) else []
    flags[rec] = dead * ELEM_DELETED | after * ELEM_AFTER_DEFINED
    return index, visible, flags


def find_every_record(engine, batch, merged, logs=None):
    """Query the opId of every ins/del record of `logs`; check against expected_positions; return the answers."""
    logs = range(batch.n_logs) if logs is None else logs
    qlog, qctr, qact, want = [], [], [], []
    for i in logs:
        ins, _ = batch.log_slice(i)
        index, visible, flags = expected_positions(batch, merged, i)
        qlog.append(np.full(len(ins), i, np.uint32)); qctr.append(ins["ctr"]); qact.append(ins["actor"])
        is_ins = (ins["payload"] >> 30) == KIND_INSERT
        assert (index[is_ins] != NF).all() and (index[~is_ins] == NF).all()
        rec = np.where(is_ins, np.arange(len(ins)), NF)
        want.append(np.stack([index, visible, rec, flags], 1))
    got = engine.find_elements(np.concatenate(qlog), np.concatenate(qctr), np.concatenate(qact))
    want = np.concatenate(want)
    got2 = np.stack([got["index"], got["visible"], got["record"], got["flags"]], 1).astype(np.int64)
    bad = np.flatnonzero((got2 != want).any(1))
    assert len(bad) == 0, (len(bad), got2[bad[:4]].tolist(), want[bad[:4]].tolist())
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_find_matches_oracle_on_fuzz_sessions(sengine, seed):
    _, logs, _ = fuzz_session(O, 7100 + seed, 140, sync_prob=0.5, full_sync_at_end=bool(seed % 2), remove_comments=True)
    batch = pack_logs(logs)
    merged = sengine.run(batch)
    assert (merged.results["status"] == 0).all()
    fresh, qlog, qid, want = [], [], [], []
    for i, log in enumerate(logs):
        o = O("observer")
        for ch in log:
            o.applyChange(ch)
        fresh.append(o)
        vis = 0
        for p, e in enumerate(o.elements()):
            qlog.append(i); qid.append(e["elemId"])
            want.append((p, vis, bool(e["deleted"]), bool(e["after"])))
            vis += not e["deleted"]
    refs, ok = elem_refs(batch, qlog, qid)
    assert ok.all()
    got = sengine.find_elements(refs["log"], refs["ctr"], refs["actor"])
    assert any(w[2] for w in want) and any(w[3] for w in want)      # tombstones and defined after-slots are both exercised
    for k in range(len(want)):
        g = got[k]
        assert (int(g["index"]), int(g["visible"]), bool(g["flags"] & ELEM_DELETED), bool(g["flags"] & ELEM_AFTER_DEFINED)) == want[k], (qlog[k], qid[k])
        assert not g["flags"] & ELEM_LOG_FAILED and elem_id(batch, qlog[k], g["record"]) == qid[k]
    # resolveCursor of the oracle replica on a sample (tombstones included)
    sample = random.Random(seed).sample(range(len(qid)), min(80, len(qid)))
    res = sengine.resolve_cursors(batch, [qlog[k] for k in sample], [qid[k] for k in sample])
    for k, r in zip(sample, res):
        oid = next(op["opId"] for op in logs[qlog[k]][0]["ops"] if op["action"] == "makeList")
        assert fresh[qlog[k]].resolveCursor({"objectId": oid, "elemId": qid[k]}) == r
    # opIds of delete and mark ops are no list elements: the reference's scan never matches them
    other = [(i, op) for i, log in enumerate(logs) for op, act in list_ops(log) if act in ("del", "addMark", "removeMark")]
    assert {act for log in logs for _, act in list_ops(log)} >= {"del", "addMark"}
    refs, ok = elem_refs(batch, [i for i, _ in other], [op for _, op in other])
    assert ok.all()
    got = sengine.find_elements(refs["log"], refs["ctr"], refs["actor"])
    assert (got["index"] == NF).all() and (got["record"] == NF).all() and (got["visible"] == 0).all() and (got["flags"] == 0).all()
    assert (sengine.resolve_cursors(batch, [i for i, _ in other], [op for _, op in other]) == -1).all()


@pytest.mark.gpu
def test_resolve_cursor_kats(sengine):
    kats = [k for k in load_kats() if k["kind"] == "script" and any(st["do"] == "resolveCursor" for st in k["steps"])]
    assert len(kats) == 6
    for kat in kats:
        docs, _, init = generateDocs(O, kat["initialText"])
        logs = [[init], [init]]
        changes, cursors = {}, {}
        n_checked = 0
        for st in kat["steps"]:
            d = st["doc"] - 1
            if st["do"] == "change":
                ch = docs[d].change(st["ops"])["change"]; logs[d].append(ch)
                if "save" in st:
                    changes[st["save"]] = ch
            elif st["do"] == "applyChange":
                docs[d].applyChange(changes[st["change"]]); logs[d].append(changes[st["change"]])
            elif st["do"] == "getCursor":
                cursors[st["save"]] = docs[d].getCursor(["text"], st["index"])
            elif st["do"] == "resolveCursor":
                batch = pack_logs([logs[d]])
                sengine.run(batch)
                got = sengine.resolve_cursors(batch, [0], [cursors[st["cursor"]]["elemId"]])
                assert int(got[0]) == st["expect"], kat["name"]
                n_checked += 1
        assert n_checked, kat["name"]


@pytest.mark.gpu
def test_find_inverts_the_index_query_on_c4(sengine):
    from peritext_b200 import workload
    batch = workload.generate("c4", n_docs=1000)
    merged = sengine.run(batch)
    assert batch.n_logs == 3000 and (merged.results["status"] == 0).all()
    nv = merged.results["n_visible"].astype(np.int64)
    qlog = np.repeat(np.arange(batch.n_logs, dtype=np.uint32), nv)
    qidx = np.concatenate([np.arange(v, dtype=np.uint32) for v in nv])
    assert len(qlog) > 1000
    rec = sengine.query_elements(qlog, qidx)
    assert (rec != NF).all()
    ins = batch.insdel[batch.desc["insdel_off"][qlog].astype(np.int64) + rec.astype(np.int64)]
    got = sengine.find_elements(qlog, ins["ctr"], ins["actor"])
    assert (got["visible"] == qidx).all() and (got["record"] == rec).all() and (got["flags"] & (ELEM_DELETED | ELEM_LOG_FAILED) == 0).all()
    live = np.concatenate([np.flatnonzero((merged.sequence(i) >> 31) == 0) for i in range(batch.n_logs)])
    assert (got["index"] == live).all()


@pytest.mark.gpu
def test_find_every_record_of_every_route_case():
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_routes import CONFIGS, all_cases, joint_batch, kernel_config
    batch = joint_batch(all_cases())
    answers = {}
    for cfg in CONFIGS:
        with kernel_config(cfg):
            e = BatchEngine(0, emit_sequence=True)
            try:
                merged = e.run(batch)
                assert (merged.results["status"] == 0).all(), cfg
                answers[cfg] = find_every_record(e, batch, merged)
            finally:
                e.close()
    first = answers["default"]
    for cfg, got in answers.items():
        assert got.tobytes() == first.tobytes(), cfg


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["c5", "c2-40k"])
def test_find_in_large_documents(sengine, shape):
    from peritext_b200 import workload
    batch = workload.generate("c5", n_docs=1) if shape == "c5" else workload.generate("c2", n_docs=1, ops_per_doc=40000)
    merged = sengine.run(batch)
    assert (merged.results["status"] == 0).all()
    i = 0
    n = int(batch.desc[i]["n_insdel"])
    assert n > (100000 if shape == "c5" else 38000)
    ins, _ = batch.log_slice(i)
    s = merged.sequence(i)
    index, visible, flags = expected_positions(batch, merged, i)
    inserts = np.flatnonzero((ins["payload"] >> 30) == KIND_INSERT)
    recs = np.concatenate([np.random.default_rng(5).choice(inserts, 3000, replace=False), [s[0] & 0x3FFFFFFF, s[-1] & 0x3FFFFFFF]]).astype(np.int64)
    got = sengine.find_elements(np.full(len(recs), i, np.uint32), ins["ctr"][recs], ins["actor"][recs])
    assert (got["record"] == recs).all()
    assert (got["index"] == index[recs]).all() and (got["visible"] == visible[recs]).all() and (got["flags"] == flags[recs]).all()
    assert int(got["index"][-2]) == 0 and int(got["index"][-1]) == len(s) - 1


@pytest.mark.gpu
def test_find_edge_cases(sengine):
    from peritext_b200.engine import BatchEngine, EngineError
    from tests.test_gpu_routes import Log, batch_of, route_base, typing_forward, with_fault
    empty = Log(1)
    dead = Log(2)
    for k, e in enumerate(typing_forward(dead, 70, [0, 1])):
        dead.delete(k % 2, e)
    fault = with_fault(route_base("direct"), "missing-reference")
    clean = route_base("compact")
    batch = batch_of([empty, dead, fault, clean])
    merged = sengine.run(batch)
    assert merged.results["status"].tolist() == [0, 0, 1, 0] and int(merged.results["n_elems"][0]) == 0
    # n == 0: no launch, PT_OK, also with null pointers
    assert len(sengine.find_elements([], [], [])) == 0
    assert sengine._L.pt_batch_find_elements(sengine._h, None, 0, None) == 0
    assert sengine._L.pt_batch_find_elements(sengine._h, None, 1, None) == 1          # PT_ERR_INVALID
    # every element of the all-deleted log: found, deleted, nothing visible before it
    got = find_every_record(sengine, batch, merged, logs=[1])
    ins = (batch.log_slice(1)[0]["payload"] >> 30) == KIND_INSERT
    assert (got["visible"] == 0).all() and (got["flags"][ins] == ELEM_DELETED).all() and sorted(got["index"][ins].tolist()) == list(range(70))
    find_every_record(sengine, batch, merged, logs=[3])
    C = int(batch.desc[3]["max_ctr"]); R = int(batch.desc[3]["n_actors"])
    q = [(0, 1, 0, 0), (3, 0, 0, 0), (3, C + 1, 0, 0), (3, 1, R, 0), (3, 0xFFFFFFFF, 0xFFFF, 0),     # not found
         (2, int(batch.log_slice(2)[0]["ctr"][0]), int(batch.log_slice(2)[0]["actor"][0]), ELEM_LOG_FAILED),   # faulted log
         (4, 1, 0, ELEM_LOG_FAILED), (0xFFFFFFFF, 1, 0, ELEM_LOG_FAILED)]                             # log >= n_logs
    got = sengine.find_elements([x[0] for x in q], [x[1] for x in q], [x[2] for x in q])
    assert (got["index"] == NF).all() and (got["record"] == NF).all() and (got["visible"] == 0).all()
    assert got["flags"].tolist() == [x[3] for x in q]
    # the reserved fields of a ref are ignored
    r0 = batch.log_slice(3)[0][0]
    r = np.zeros(1, ELEM_REF_DT)
    r["log"], r["ctr"], r["actor"], r["reserved0"], r["reserved1"] = 3, r0["ctr"], r0["actor"], 7, 9
    out = np.zeros(1, got.dtype)
    assert sengine._L.pt_batch_find_elements(sengine._h, r.ctypes.data, 1, out.ctypes.data) == 0
    assert int(out["record"][0]) == 0 and int(out["index"][0]) != NF
    # PT_ERR_STATE: before any merge, after an upload without a merge, and on a handle without emit_sequence
    e = BatchEngine(0, emit_sequence=True)
    try:
        with pytest.raises(EngineError, match="out of order"):
            e.find_elements([0], [1], [0])
        e.upload(batch)
        with pytest.raises(EngineError, match="out of order"):
            e.find_elements([0], [1], [0])
        assert e._L.pt_batch_find_elements(e._h, None, 0, None) == 4
    finally:
        e.close()
    e = BatchEngine(0)
    try:
        e.run(batch)
        with pytest.raises(EngineError, match="EMIT_SEQUENCE"):
            e.find_elements([3], [1], [0])
    finally:
        e.close()
