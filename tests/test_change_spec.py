"""The host specification of pt_batch_change, ``packing.generate_change``, against the oracle's ``Micromerge.change``.

Every case is (a Change log, the acting actor, InputOperations): the oracle replica that applied the log makes the change,
and the spec generates it from the replica's element sequence (``elements()``, the facade's mirror form).  The Change objects
must be equal (opIds, elemIds, boundary objects); where the oracle throws "List index out of bounds" the spec must name the
InputOperation the oracle fails on.  The corpora here are reused by tests/test_gpu_change.py."""
import random

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.oracle import RangeError
from peritext_b200.packing import (CHANGE_NO_ACTOR, INPUT_OP_DT, ChangeOutOfBounds, _root_text_list, change_inputs, generate_change,
                                   pack_logs)
from tests.harness import generateDocs, load_kats, with_path
from tests.test_append_packing import comment_and_link_logs, early_actor_logs, fuzz_logs, quirk_logs, sparse_logs


# ------------------------------------------------------------------------------------------------------------------
# Cases
# ------------------------------------------------------------------------------------------------------------------
def replica(log, actor):
    d = O(actor)
    for ch in log:
        d.applyChange(ch)
    return d


def next_op(log):
    return max([ch["startOp"] + len(ch["ops"]) - 1 for ch in log] + [0]) + 1


def oracle_change(log, actor, inputs):
    """(meta before the change, the oracle's Change or None, the failing InputOperation or None)."""
    d = replica(log, actor)
    meta = [[e["elemId"], e["deleted"], e["after"]] for e in d.elements()]
    try:
        return meta, d.change(inputs)["change"], None
    except RangeError:
        pass
    for k in range(len(inputs)):
        try:
            replica(log, actor).change(inputs[: k + 1])
        except RangeError:
            return meta, None, k
    raise AssertionError("the oracle threw only on the whole change")


def header(log, actor):
    """seq / deps / startOp of the change a fresh replica of `log` makes: its first own change, its clock, maxOp + 1."""
    d = replica(log, actor)
    clock = d.clock
    return {"actor": actor, "seq": 1, "deps": clock, "startOp": next_op(log)}


def kat_cases():
    out = []
    for kat in [k for k in load_kats() if k["kind"] == "concurrent"]:
        docs, _, init = generateDocs(O, kat["initialText"])
        log = [init]
        if kat.get("preOps"):
            r0 = docs[0].change(with_path(kat["preOps"]))
            log.append(r0["change"])
        out.append((f"L{kat['line']}-doc1", log, "doc1", with_path(kat["inputOps1"])))
        out.append((f"L{kat['line']}-doc2", log, "doc2", with_path(kat["inputOps2"])))
    return out


def random_inputs(rng, length, n_ops, comment_ids=(), links=("A.com", "B.com")):
    """Fuzz-shaped InputOperations whose indices follow the document as the change goes, a few of them out of bounds."""
    ops = []
    for _ in range(n_ops):
        kind = rng.choice(["insert", "insert", "delete", "mark"])
        off = 1 if rng.random() < 0.08 else 0                       # now and then one past the end
        if kind == "insert" or length == 0:
            vals = [rng.choice(["a", "b", "é", "\U0001F600", "xyz"]) for _ in range(rng.randrange(4))]
            ops.append({"path": ["text"], "action": "insert", "index": rng.randrange(length + 1) + off, "values": vals})
            length += len(vals)
        elif kind == "delete":
            i = rng.randrange(length) + off
            c = rng.randrange(1, 4)
            ops.append({"path": ["text"], "action": "delete", "index": i, "count": c})
            length = max(0, length - c)
        else:
            mt = rng.choice(["strong", "em", "link"] + (["comment"] if comment_ids else []))
            s = rng.randrange(length) + off
            e = s + rng.randrange(0, length - s + 2)
            op = {"path": ["text"], "action": rng.choice(["addMark", "addMark", "removeMark"]), "startIndex": s, "endIndex": e, "markType": mt}
            if mt == "link":
                op["attrs"] = {"url": rng.choice(links)}
            elif mt == "comment":
                op["attrs"] = {"id": rng.choice(list(comment_ids))}
            ops.append(op)
    return ops


def log_comment_ids(log):
    return sorted({op["attrs"]["id"] for ch in log for op in ch["ops"] if op.get("markType") == "comment" and op.get("attrs")})


def fuzz_cases(logs, seed, per_log=2, tag="fuzz"):
    rng = random.Random(seed)
    out = []
    for li, log in enumerate(logs):
        actors = sorted({ch["actor"] for ch in log})
        for t in range(per_log):
            actor = rng.choice(actors)
            length = len(replica(log, actor).root["text"])
            out.append((f"{tag}{li}.{t}", log, actor, random_inputs(rng, length, rng.randrange(1, 9), log_comment_ids(log))))
    return out


def corpus_cases():
    out = fuzz_cases(fuzz_logs()[:12], 1)
    out += fuzz_cases(quirk_logs() + early_actor_logs(), 2, 4, "quirk")
    out += fuzz_cases(comment_and_link_logs()[0], 3, 4, "comments")
    out += fuzz_cases(sparse_logs()[0], 4, 4, "sparse")
    return out


def corner_cases():
    """(name, log, actor, inputs) of the named corners of change()."""
    T = lambda **kw: {"path": ["text"], **kw}
    out = []
    _, _, empty = generateDocs(O, "", 1)
    out.append(("insert-at-0-empty", [empty], "doc1", [T(action="insert", index=0, values=["a", "b"])]))
    out.append(("insert-1-empty", [empty], "doc1", [T(action="insert", index=1, values=["a"])]))
    docs, _, init = generateDocs(O, "abcd", 1)
    d = docs[0]
    base = [init]
    out.append(("insert-at-length", base, "doc1", [T(action="insert", index=4, values=["z"])]))
    out.append(("insert-past-length", base, "doc1", [T(action="insert", index=5, values=["z"])]))
    out.append(("zero-value-insert-out-of-bounds", base, "doc1", [T(action="insert", index=9, values=[])]))
    out.append(("zero-value-insert", base, "doc1", [T(action="insert", index=2, values=[]), T(action="insert", index=1, values=["q"])]))
    out.append(("delete-off-the-end", base, "doc1", [T(action="delete", index=2, count=5)]))
    out.append(("delete-zero", base, "doc1", [T(action="delete", index=7, count=0), T(action="insert", index=0, values=["q"])]))
    for e in (3, 4, 6):
        out.append((f"inclusive-end-{e}", base, "doc1", [T(action="addMark", startIndex=1, endIndex=e, markType="strong")]))
    out.append(("non-inclusive-end-0", base, "doc1", [T(action="addMark", startIndex=0, endIndex=0, markType="link", attrs={"url": "u"})]))
    out.append(("start-out-of-bounds", base, "doc1", [T(action="addMark", startIndex=4, endIndex=4, markType="em")]))
    out.append(("zero-width", base, "doc1", [T(action="addMark", startIndex=2, endIndex=2, markType="strong"),
                                             T(action="addMark", startIndex=2, endIndex=2, markType="link", attrs={"url": "u"}),
                                             T(action="removeMark", startIndex=1, endIndex=1, markType="em")]))
    out.append(("dependent-indices", base, "doc1", [T(action="insert", index=0, values=["x", "y"]), T(action="delete", index=1, count=2),
                                                    T(action="addMark", startIndex=0, endIndex=3, markType="em"),
                                                    T(action="insert", index=3, values=["z"]), T(action="delete", index=0, count=1),
                                                    T(action="addMark", startIndex=1, endIndex=4, markType="link", attrs={"url": "v"})]))
    out.append(("root-ops-interleaved", base, "doc1", [{"path": [], "action": "set", "key": "title", "value": "t"},
                                                       T(action="insert", index=1, values=["m", "n"]),
                                                       {"path": [], "action": "makeMap", "key": "meta"},
                                                       T(action="addMark", startIndex=0, endIndex=2, markType="strong")]))
    # tombstones after the reference element, with and without a defined after slot
    c1 = d.change([T(action="addMark", startIndex=0, endIndex=2, markType="link", attrs={"url": "u"})])["change"]   # after(elem 1 = b)
    c2 = d.change([T(action="delete", index=1, count=2)])["change"]                                                  # b, c -> tombstones
    out.append(("after-tombstone-with-slot", base + [c1, c2], "doc1", [T(action="insert", index=1, values=["x"])]))
    docs2, _, init2 = generateDocs(O, "abcd", 1)
    c3 = docs2[0].change([T(action="delete", index=1, count=2)])["change"]
    out.append(("after-tombstones-without-slot", [init2, c3], "doc1", [T(action="insert", index=1, values=["x"])]))
    out.append(("slot-defined-earlier-in-the-change", base, "doc1", [T(action="addMark", startIndex=1, endIndex=3, markType="comment", attrs={"id": "k"}),
                                                                     T(action="delete", index=2, count=1),
                                                                     T(action="insert", index=2, values=["x"])]))
    return out


def all_cases():
    return kat_cases() + corpus_cases() + corner_cases()


def spec_change(log, actor, inputs):
    """generate_change on the oracle replica's elements: (Change or None, failing InputOperation or None)."""
    d = replica(log, actor)
    meta = [[e["elemId"], e["deleted"], e["after"]] for e in d.elements()]
    h = header(log, actor)
    try:
        return generate_change(meta, {**h, "ops": inputs}, _root_text_list(log)), None
    except ChangeOutOfBounds as e:
        return None, e.input


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def check_cases(cases):
    n_fail = 0
    for name, log, actor, inputs in cases:
        _, want, want_fail = oracle_change(log, actor, inputs)
        got, got_fail = spec_change(log, actor, inputs)
        assert got_fail == want_fail, name
        if want is not None:
            assert want["startOp"] == next_op(log), name
            assert got == want, name
        n_fail += want_fail is not None
    return n_fail


def test_kat_input_ops():
    cases = kat_cases()
    assert len(cases) == 62
    check_cases(cases)


def test_fuzz_shaped_and_append_corpora():
    cases = corpus_cases()
    assert check_cases(cases) > 0                  # some changes run out of bounds
    assert sum(len(c[3]) > 1 for c in cases) > len(cases) // 2


def test_named_corners():
    cases = corner_cases()
    fails = {name: oracle_change(log, actor, inputs)[2] for name, log, actor, inputs in cases}
    assert fails["zero-value-insert-out-of-bounds"] == 0 and fails["delete-off-the-end"] == 0 and fails["non-inclusive-end-0"] == 0
    assert fails["insert-past-length"] == 0 and fails["insert-1-empty"] == 0 and fails["start-out-of-bounds"] == 0
    assert fails["zero-width"] is None and fails["dependent-indices"] is None and fails["slot-defined-earlier-in-the-change"] is None
    check_cases(cases)


def test_the_after_slot_moves_the_insert():
    """The corners exercise what they are named for: the insert lands after the tombstone whose after slot is defined."""
    by = {c[0]: c for c in corner_cases()}
    got = {k: spec_change(*by[k][1:])[0]["ops"][-1]["elemId"] for k in ("after-tombstone-with-slot", "after-tombstones-without-slot",
                                                                         "slot-defined-earlier-in-the-change")}
    assert got == {"after-tombstone-with-slot": "3@doc1", "after-tombstones-without-slot": "2@doc1", "slot-defined-earlier-in-the-change": "4@doc1"}


def test_device_inputs_follow_the_counters():
    """change_inputs: one record per list InputOperation, first_ctr = startOp + the ops before it (ROOT-map ops included);
    a dense log counts in dense ranks past its counter table."""
    by = {c[0]: c for c in corner_cases()}
    _, log, actor, inputs = by["root-ops-interleaved"]
    batch = pack_logs([log])
    rank = batch.log_actors[0].index(actor)
    h = header(log, actor)
    act, off, ops, tokens, values, links, counters = change_inputs(batch, [{**h, "ops": inputs}], [rank])
    assert ops.dtype == INPUT_OP_DT and list(off) == [0, 2] and int(act[0]) == rank
    assert list(ops["first_ctr"]) == [h["startOp"] + 1, h["startOp"] + 4] and list(ops["arg"]) == [2, 2]
    assert [chr(t) for t in tokens] == ["m", "n"]
    act, off, *_ = change_inputs(batch, [None], [None])
    assert int(act[0]) == CHANGE_NO_ACTOR and list(off) == [0, 0]
    logs, _ = sparse_logs()
    sb = pack_logs(logs[:1])
    assert sb.log_counters[0] is not None
    h = header(logs[0], "doc1")
    _, _, ops, _, _, _, counters = change_inputs(sb, [{**h, "ops": [{"path": ["text"], "action": "insert", "index": 0, "values": ["a", "b"]}]}], [0])
    assert int(ops["first_ctr"][0]) == len(sb.log_counters[0])
    assert [int(c) for c in counters[0][-2:]] == [h["startOp"], h["startOp"] + 1]


def test_struct_layouts():
    from peritext_b200.packing import CHANGE_STATUS_DT
    assert INPUT_OP_DT.itemsize == 32 and CHANGE_STATUS_DT.itemsize == 8
    assert INPUT_OP_DT.fields["index"][1] == 4 and INPUT_OP_DT.fields["first_ctr"][1] == 16 and INPUT_OP_DT.fields["tok_off"][1] == 24
