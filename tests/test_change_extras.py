"""The extras of pt_batch_render_changes_json on the host: ``packing.change_extras`` (the readable specification) against the
native ingest's extras and its list-id / extra-ops pools (PT_POOL_LIST_IDS, PT_POOL_EXTRA_OPS), and the Python render
specification of tests/test_gpu_render_changes_json.py against the Change objects the logs were made of.  Host code only."""
import json
import os

import numpy as np
import pytest

from oracle.oracle import Micromerge
from peritext_b200.engine import ingest_native
from peritext_b200.packing import EXTRA_NONE, change_extras, pack_logs
from tests.harness import GOLDEN, fuzz_session, generateDocs, load_kats, run_concurrent


def kat_logs():
    logs = []
    for kat in [k for k in load_kats() if k["kind"] == "concurrent"]:
        rec = []
        run_concurrent(Micromerge, kat, record=rec)
        logs += rec
    return logs


def unicode_logs():
    docs, _, init = generateDocs(Micromerge, "ab", 1)
    d = docs[0]
    c1 = d.change([{"path": ["text"], "action": "insert", "index": 1, "values": [" is great!", "é", "\U0001F600", "", "中", "q\"\\\n\x01"]}])["change"]
    c2 = d.change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 3, "markType": "comment", "attrs": {"id": "zé"}},
                   {"path": ["text"], "action": "addMark", "startIndex": 1, "endIndex": 4, "markType": "comment", "attrs": {"id": "a\U0001F600"}},
                   {"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 2, "markType": "link", "attrs": {"url": "https://x.y/?q=\"1\"&r=\\\x02"}}])["change"]
    odd = [{"actor": "\U00010000\"\udbff", "seq": 1, "deps": {}, "startOp": 1, "ops": [
        {"opId": "1@\U00010000\"\udbff", "action": "makeList", "obj": "_root", "key": "text"},
        {"opId": "2@\U00010000\"\udbff", "action": "set", "obj": "1@\U00010000\"\udbff", "elemId": "_head", "insert": True, "value": "x"}]},
        {"actor": "￿\t", "seq": 1, "deps": {"\U00010000\"\udbff": 1}, "startOp": 3, "ops": [
            {"opId": "3@￿\t", "action": "set", "obj": "1@\U00010000\"\udbff", "elemId": "2@\U00010000\"\udbff", "insert": True, "value": "y"},
            {"opId": "4@\uffff\t", "action": "set", "obj": "_root", "key": "title", "value": "t\udc00 "},
            {"opId": "5@\uffff\t", "action": "set", "obj": "1@\U00010000\"\udbff", "elemId": "3@\uffff\t", "insert": True, "value": "\ud800"},
            {"opId": "6@\uffff\t", "action": "addMark", "obj": "1@\U00010000\"\udbff", "start": {"type": "before", "elemId": "2@\U00010000\"\udbff"},
             "end": {"type": "after", "elemId": "5@\uffff\t"}, "markType": "link", "attrs": {"url": "\udc01\u2028/"}}]},
        {"actor": "￿\t", "seq": 2, "deps": {"￿\t": 1}, "startOp": 7, "ops": []}]
    return [[init, c1, c2], odd]


def sparse_logs():
    docs, _, init = generateDocs(Micromerge, "abc", 2)
    big = {"actor": "doc2", "seq": 1, "deps": {"doc1": 1}, "startOp": 5_000_000, "ops": [
        {"opId": "5000000@doc2", "action": "set", "obj": "1@doc1", "elemId": "2@doc1", "insert": True, "value": "X"},
        {"opId": "5000002@doc2", "action": "addMark", "obj": "1@doc1", "start": {"type": "before", "elemId": "5000000@doc2"},
         "end": {"type": "after", "elemId": "3@doc1"}, "markType": "link", "attrs": {"url": "u"}}]}
    late = {"actor": "doc2", "seq": 2, "deps": {"doc2": 1}, "startOp": 7_000_000, "ops": [
        {"opId": "7000001@doc2", "action": "del", "obj": "1@doc1", "elemId": "5000000@doc2"}]}
    return [[init, big, late]]


def links_minimal_logs():
    q = json.load(open(os.path.join(GOLDEN, "links_minimal_queues.json")))["queues"]
    return [[q["doc0"][0], q["doc0"][1], q["doc1"][0], q["doc2"][0]], [q["doc0"][0], q["doc2"][0], q["doc1"][0], q["doc0"][1]]]


CORPORA = {
    "kat": kat_logs,
    "fuzz": lambda: [l for s in range(3) for l in fuzz_session(Micromerge, 700 + s, 120, sync_prob=0.5)[1]],
    "links_minimal": links_minimal_logs,
    "unicode": unicode_logs,
    "sparse": sparse_logs,
}


@pytest.mark.parametrize("name", sorted(CORPORA))
def test_extras_and_pools_match_the_ingest(name):
    logs = CORPORA[name]()
    spec, lids = change_extras(logs)
    batch, extras, raw = ingest_native([json.dumps(l, ensure_ascii=False).encode("utf-8", "surrogatepass") for l in logs])
    assert extras.rows.tobytes() == spec.rows.tobytes()
    assert extras.ops == spec.ops
    data, off = spec.pools()
    assert raw[7][0] == data.tobytes() and raw[7][1].tolist() == off.tolist()
    assert raw[6][0] == b"".join(l.encode("utf-16-le", "surrogatepass") for l in lids)
    assert len(raw[6][1]) == len(logs) + 1
    assert [l or "" for l in batch.log_lists] == lids
    # the extras are sorted, every change's entries share one start_op, a NONE entry stands alone
    r = extras.rows
    key = r["log"].astype(np.uint64) << np.uint64(32) | r["change"]
    assert (np.diff(key.astype(np.int64)) >= 0).all()
    for k in range(1, len(r)):
        if key[k] == key[k - 1]:
            assert r[k]["pos"] > r[k - 1]["pos"] and r[k]["start_op"] == r[k - 1]["start_op"]
            assert r[k]["op"] != EXTRA_NONE and r[k - 1]["op"] != EXTRA_NONE


@pytest.mark.parametrize("name", ["kat", "fuzz", "unicode", "sparse"])
def test_python_spec_gives_back_the_change_objects(name):
    from tests.test_gpu_render_changes_json import render_log_spec
    logs = CORPORA[name]()
    batch = pack_logs(logs, with_changes=True)
    extras, _ = change_extras(logs)
    for i, lg in enumerate(logs):
        got = json.loads(render_log_spec(batch, extras, i, range(len(lg))).decode("utf-8", "surrogatepass"))
        want = [dict(ch, ops=[dict(op, elemId=op.get("elemId", "_head")) if op.get("insert") else op for op in ch["ops"]]) for ch in lg]
        assert got == want


def test_projection_without_extras():
    from tests.test_gpu_render_changes_json import render_log_spec
    logs = kat_logs()[:2]
    batch = pack_logs(logs, with_changes=True)
    none, _ = change_extras([[] for _ in logs])
    for i, lg in enumerate(logs):
        got = json.loads(render_log_spec(batch, none, i, range(len(lg))))
        for g, ch in zip(got, lg):
            lops = [op for op in ch["ops"] if op.get("obj") == batch.log_lists[i]]
            assert g["ops"] == lops and g["startOp"] == int(lops[0]["opId"].split("@")[0])
