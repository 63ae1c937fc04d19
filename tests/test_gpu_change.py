"""pt_batch_change on the device: the Change objects equal the oracle's ``Micromerge.change``, failing logs name the oracle's
failing InputOperation while the others proceed, and the batch the handle holds afterwards is exactly the batch
``apply_append`` of the generated records gives: every output of a merge equals a fresh upload of it, the spans equal the
oracle's after its change, and the Patch JSON of the new ops (patch window) equals the patches change() returned.

Cases come from tests/test_change_spec.py (KAT inputOps, fuzz-shaped multi-op changes on the append corpora, the named
corners); tests/test_change_spec.py pins the host specification ``packing.generate_change`` on the same cases."""
import json

import numpy as np
import pytest

from oracle.oracle import RangeError
from oracle.packed import replay_packed
from peritext_b200.packing import (CHANGE_OUT_OF_BOUNDS, DESC_DT, INPUT_OP_DT, INSDEL_DT, MARK_DT, AppendRemap, PackedBatch,
                                   apply_append, decode_spans, js_key, pack_append, pack_logs)
from tests.test_change_spec import corner_cases, corpus_cases, header, kat_cases, oracle_change, random_inputs, replica
from tests.test_gpu_append import canon, everything, merged
from tests.test_gpu_wire_forms import FORMS, upload_as

PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_patches=True, **kw)


def new_comments(batch, cs):
    """The attrs of the comment ids the cases' InputOperations name and the batch does not know, by id."""
    known = {c["id"] for c in batch.comment_ids}
    return {op["attrs"]["id"]: op["attrs"] for _, _, _, ops in cs for op in ops
            if op.get("markType") == "comment" and op.get("attrs") and op["attrs"]["id"] not in known}


def introduce(e, batch, cs, table=None):
    """The header's recipe for an actor a log has not seen and a comment id the batch has not seen: pt_batch_append of an empty
    delta whose remap ranks them among the old ones.  Returns the batch the handle holds."""
    n = batch.n_logs
    actors = [actor for _, _, actor, _ in cs]
    ranked = [sorted(set(batch.log_actors[i]) | {actors[i]}, key=js_key) for i in range(n)]
    maps = [[r.index(a) for a in batch.log_actors[i]] for i, r in enumerate(ranked)]
    aoff = np.zeros(n + 1, np.uint64)
    aoff[1:] = np.cumsum([len(m) for m in maps])
    comments = sorted(list(batch.comment_ids) + list(new_comments(batch, cs).values()), key=lambda c: js_key(c["id"]))
    cmap = np.array([comments.index(c) for c in batch.comment_ids], np.uint32)
    desc = np.zeros(n, DESC_DT)
    desc["n_actors"] = [max(1, len(r)) for r in ranked]
    desc["max_ctr"] = batch.desc["max_ctr"]
    delta = PackedBatch(desc, np.zeros(0, INSDEL_DT), np.zeros(0, MARK_DT), batch.values, batch.link_attrs, comments, batch.other_attrs,
                        dict(batch.meta), ranked, batch.log_counters, table, batch.log_lists)
    remap = AppendRemap(aoff, np.array([x for m in maps for x in m], np.uint16), comment_map=cmap)
    e.append(delta, remap, table)
    return apply_append(batch, delta, remap)


def oracle_result(log, actor, inputs):
    """(Change, patches, spans after the change) of the oracle, or (None, None, spans before it) where it throws."""
    d = replica(log, actor)
    try:
        r = d.change(inputs)
    except RangeError:
        return None, None, replica(log, actor).getTextWithFormatting()
    return r["change"], r["patches"], d.getTextWithFormatting()


def change_batch(e, batch, cases):
    """The cases' changes through the handle (merged over `batch`)."""
    inputs = [{**header(log, actor), "ops": ops} for _, log, actor, ops in cases]
    ranks = [batch.log_actors[i].index(actor) for i, (_, _, actor, _) in enumerate(cases)]
    return e.change(batch, inputs, ranks)


def check_cases(e, u, batch, cases, windows=True):
    """Change on handle `e` (merged over `batch`), then the checks of the module docstring; `u` uploads for comparison."""
    new, dicts, status = change_batch(e, batch, cases)
    n_fail = 0
    wants = [oracle_result(log, actor, ops) for _, log, actor, ops in cases]
    for i, (name, log, actor, ops) in enumerate(cases):
        want, _, _ = wants[i]
        if want is None:
            fail = oracle_change(log, actor, ops)[2]
            assert int(status[i]["status"]) == CHANGE_OUT_OF_BOUNDS and int(status[i]["input"]) == fail and dicts[i] is None, name
            n_fail += 1
        else:
            assert int(status[i]["status"]) == 0 and dicts[i] == want, name
    got = merged(e)
    u.upload(new)
    ref = merged(u)
    assert canon(got) == canon(ref)
    assert canon(got) == canon(replay_packed(new)[0])
    for i, (name, *_rest) in enumerate(cases):
        assert decode_spans(new, got, i) == wants[i][2], name
    assert everything(e, new, got) == everything(u, new, ref)
    if windows:
        first = (batch.desc["n_insdel"].astype(np.int64) + batch.desc["n_mark"]).astype(np.uint32)
        e.set_patch_window(first)
        e.merge()
        rendered = e.render_patches_json_list(new)
        for i, (name, *_rest) in enumerate(cases):
            pw = [p for p in (wants[i][1] or []) if p["action"] != "makeList"]
            assert [p for op in json.loads(rendered[i]) for p in op] == pw, name
    return new, n_fail


# ------------------------------------------------------------------------------------------------------------------
# 1-4. The corpora through every upload form, and after an append
# ------------------------------------------------------------------------------------------------------------------
_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = kat_cases() + corner_cases() + corpus_cases()
    return _CASES


def prepared(e, cs, form, after_append=False):
    """Upload the cases' logs in `form` (the last change of every log through pt_batch_append when `after_append`), introduce
    the acting actors a log has not seen, merge.  Returns (batch, what must stay alive)."""
    logs = [log for _, log, _, _ in cs]
    if after_append:
        prev = pack_logs([lg[:-1] for lg in logs])
        keep = upload_as(e, prev, form)
        delta, remap = pack_append(prev, [lg[-1:] for lg in logs])
        e.append(delta, remap)
        batch = apply_append(prev, delta, remap)
    else:
        batch = pack_logs(logs)
        keep = upload_as(e, batch, form)
    if any(actor not in batch.log_actors[i] for i, (_, _, actor, _) in enumerate(cs)) or new_comments(batch, cs):
        batch = introduce(e, batch, cs)
    merged(e)
    return batch, keep


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_change_matches_the_oracle(form):
    e, u = engine(), engine()
    try:
        batch, keep = prepared(e, cases(), form)
        _, n_fail = check_cases(e, u, batch, cases())
        assert 0 < n_fail < len(cases()) // 2
        del keep
    finally:
        e.close(); u.close()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "compact", "runs"])
def test_change_after_an_append(form):
    cs = [c for c in cases() if len(c[1]) > 1]
    e, u = engine(), engine()
    try:
        batch, keep = prepared(e, cs, form, after_append=True)
        check_cases(e, u, batch, cs)
        del keep
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_chained_changes_and_the_change_table():
    """Two changes in a row on a batch with a change table (merge between them), against the oracle replica making both."""
    cs = [c for c in kat_cases()[:10]]
    logs = [log for _, log, _, _ in cs]
    e, u = engine(), engine()
    try:
        batch = pack_logs(logs, with_changes=True)
        e.upload(batch); e.upload_changes(batch.changes)
        batch = introduce(e, batch, cs, empty_table(batch.n_logs))
        merged(e)
        clocks = [replica(log, actor).clock for _, log, actor, _ in cs]
        inputs = [{**header(log, actor), "seq": clocks[i].get(actor, 0) + 1, "ops": ops} for i, (_, log, actor, ops) in enumerate(cs)]
        ranks = [batch.log_actors[i].index(a) for i, (_, _, a, _) in enumerate(cs)]
        new, dicts, status = e.change(batch, inputs, ranks, change_table(batch, inputs, ranks))
        assert (status["status"] == 0).all()
        got = merged(e)
        assert (got.results["status"] == 0).all()               # the admission pre-pass accepts the appended change records
        assert int(new.changes.desc["n_changes"].sum()) == int(batch.changes.desc["n_changes"].sum()) + len(cs)
        follow = [[{"path": ["text"], "action": "insert", "index": 0, "values": ["w"]}] for _ in cs]
        inputs2 = [{"actor": d["actor"], "seq": d["seq"] + 1, "deps": {**d["deps"], d["actor"]: d["seq"]}, "startOp": d["startOp"] + len(d["ops"]), "ops": f}
                   for d, f in zip(dicts, follow)]
        new2, dicts2, status2 = e.change(new, inputs2, ranks, change_table(new, inputs2, ranks))
        got2 = merged(e)
        assert (got2.results["status"] == 0).all()
        for i, (_, log, actor, ops) in enumerate(cs):
            d = replica(log, actor)
            first, second = d.change(ops)["change"], d.change(follow[i])["change"]
            assert dicts[i]["ops"] == first["ops"] and dicts2[i]["ops"] == second["ops"]
            assert decode_spans(new2, got2, i) == d.getTextWithFormatting()
        u.upload(new2); u.upload_changes(new2.changes)
        assert canon(merged(u)) == canon(merged(e))
    finally:
        e.close(); u.close()


def change_table(batch, inputs, ranks):
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, ChangeTable
    n = batch.n_logs
    desc = np.zeros(n, CDESC_DT)
    recs, deps = [], []
    for i, ch in enumerate(inputs):
        desc[i] = (len(recs), len(deps), 1, len(ch["deps"]))
        rank = {a: r for r, a in enumerate(batch.log_actors[i])}
        recs.append((ch["seq"], ranks[i], len(ch["deps"]), 0, sum(1 for op in ch["ops"] if op.get("path") == ["text"])))
        deps += [(v, rank[a], 0) for a, v in ch["deps"].items()]
    return ChangeTable(desc, np.array(recs, CHANGE_DT), np.array(deps, DEP_DT) if deps else np.zeros(0, DEP_DT))


def empty_table(n):
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, ChangeTable
    return ChangeTable(np.zeros(n, CDESC_DT), np.zeros(0, CHANGE_DT), np.zeros(0, DEP_DT))


# ------------------------------------------------------------------------------------------------------------------
# 5. Benchmark shapes: a c4-shaped batch and one true-shape c5 document
# ------------------------------------------------------------------------------------------------------------------
def workload_logs(config, **kw):
    from peritext_b200 import workload
    b = workload.generate(config, **kw)
    return [json.loads(workload.to_change_json(b, i)) for i in range(b.n_logs)]


def shape_cases(logs, seed, n_ops):
    import random
    rng = random.Random(seed)
    out = []
    for li, log in enumerate(logs):
        actor = "doc1"
        length = len(replica(log, actor).root["text"])
        out.append((f"shape{li}", log, actor, random_inputs(rng, length, n_ops)))
    return out


@pytest.mark.gpu
def test_c4_shaped_batch():
    cs = shape_cases(workload_logs("c4", n_docs=48, ops_per_doc=1000), 5, 16)
    e, u = engine(), engine()
    try:
        batch, _ = prepared(e, cs, "plain")
        check_cases(e, u, batch, cs, windows=False)
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_true_shape_c5_document():
    logs = workload_logs("c5", n_docs=1)
    assert sum(len(ch["ops"]) for ch in logs[0]) > 100000
    n = len(replica(logs[0], "doc1").root["text"])
    T = lambda **kw: {"path": ["text"], **kw}
    ops = [T(action="insert", index=n // 2, values=list("hello")), T(action="delete", index=n // 3, count=40),
           T(action="addMark", startIndex=10, endIndex=n - 100, markType="strong"), T(action="addMark", startIndex=5, endIndex=n // 2, markType="link", attrs={"url": "A.com"}),
           T(action="insert", index=n // 2, values=["x"])]
    cs = [("c5", logs[0], "doc1", ops)]
    e, u = engine(), engine()
    try:
        batch, _ = prepared(e, cs, "plain")
        check_cases(e, u, batch, cs, windows=False)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 6. Refusals and state rules
# ------------------------------------------------------------------------------------------------------------------
def change(e, actor, off, ops, tokens=(), pools=(0, 0, 0), table=None):
    """``change_packed`` from lists: `ops` as op() tuples, `pools` the value, link and comment pool sizes."""
    return e.change_packed(actor, off, np.array(ops, INPUT_OP_DT), tokens, *pools, table)


def refusal(call):
    """The pt_status of a call the engine refuses."""
    from peritext_b200.engine import EngineError
    with pytest.raises(EngineError) as err:
        call()
    return err.value.status


def op(action, index=0, arg=0, first_ctr=0, mark_type=0, attr=0xFFFFFFFF, tok_off=0):
    return (action, mark_type, 0, index, arg, attr, first_ctr, 0, tok_off)


@pytest.mark.gpu
def test_refusals_leave_the_batch_unchanged_and_the_state_rules():
    from peritext_b200.engine import BatchEngine
    cs = kat_cases()[:4]
    logs = [log for _, log, _, _ in cs]
    batch = pack_logs(logs)
    e = engine()
    try:
        e.upload(batch)
        assert refusal(lambda: change(e, [0] * 4, [0] * 5, [])) == PT_ERR_STATE                  # no merge since the upload
        before = merged(e)
        snap = everything(e, batch, before)
        mc = [int(x) for x in batch.desc["max_ctr"]]
        na = [int(x) for x in batch.desc["n_actors"]]
        none = 0xFFFFFFFF
        bad = {
            "n_logs": lambda: change(e, [0] * 3, [0] * 4, []),
            "actor": lambda: change(e, [na[0], none, none, none], [0] * 5, []),
            "inputs-without-actor": lambda: change(e, [none] * 4, [0, 1, 1, 1, 1], [op(0, 0, 0, mc[0] + 1)]),
            "first_ctr": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(1, 0, 1, mc[0])]),
            "overlap": lambda: change(e, [0, none, none, none], [0, 2, 2, 2, 2], [op(1, 0, 2, mc[0] + 1), op(1, 0, 1, mc[0] + 2)]),
            "backwards": lambda: change(e, [0, none, none, none], [0, 2, 2, 2, 2], [op(1, 0, 1, mc[0] + 5), op(1, 0, 1, mc[0] + 3)]),
            "counter-past-32-bits": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(1, 0, 2, 0xFFFFFFFF)]),
            "action": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(7, 0, 1, mc[0] + 1)]),
            "mark-type": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(2, 0, 1, mc[0] + 1, mark_type=4)]),
            "attr-link": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(2, 0, 1, mc[0] + 1, mark_type=3, attr=2)], pools=(0, 2, 0)),
            "attr-strong": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(2, 0, 1, mc[0] + 1, mark_type=0, attr=0)]),
            "token-range": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(0, 0, 2, mc[0] + 1)], tokens=[97]),
            "token-pool": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(0, 0, 1, mc[0] + 1)], tokens=[0x20000000 | 3], pools=(3, 0, 0)),
            "token-code-point": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(0, 0, 1, mc[0] + 1)], tokens=[0x110000]),
            "negative-values": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(0, 0, -1, mc[0] + 1)]),
            "max_ctr-x-actors": lambda: change(e, [0, none, none, none], [0, 1, 1, 1, 1], [op(1, 0, 1, 0x7FFFFFFF // na[0] + 1)]),
            "table-on-one-side": lambda: change(e, [none] * 4, [0] * 5, [], table=change_table(batch, [], [])),
        }
        for name, call in bad.items():
            assert refusal(call) == PT_ERR_INVALID, name
        after = merged(e)
        assert canon(after) == canon(before) and everything(e, batch, after) == snap
        # a log whose merge failed: refused, the batch stays as it was
        broken = pack_logs(logs)
        j = int(broken.desc[1]["insdel_off"]) + int(broken.desc[1]["n_insdel"]) - 1
        broken.insdel[j]["ref_ctr"] = broken.insdel[j]["ctr"]          # references itself: not found when it arrives
        broken.insdel[j]["ref_actor"] = broken.insdel[j]["actor"]
        f = engine()
        try:
            f.upload(broken)
            fb = merged(f)
            assert int(fb.results[1]["status"]) != 0
            assert refusal(lambda: change(f, [none, 0, none, none], [0, 0, 1, 1, 1], [op(1, 0, 1, int(broken.desc[1]["max_ctr"]) + 1)])) == PT_ERR_INVALID
            assert refusal(lambda: change(f, [none, 0, none, none], [0] * 5, [])) == PT_ERR_INVALID      # with an empty change too
            assert canon(merged(f)) == canon(fb)
        finally:
            f.close()
        # the state rules: a change needs a merge after every upload, append and change
        inputs = [{**header(log, a), "ops": ops} for _, log, a, ops in cs]
        batch2 = introduce(e, batch, cs)
        assert refusal(lambda: change(e, [none] * 4, [0] * 5, [])) == PT_ERR_STATE             # no merge since the append
        merged(e)
        ranks = [batch2.log_actors[i].index(a) for i, (_, _, a, _) in enumerate(cs)]
        new, _, status = e.change(batch2, inputs, ranks)
        assert refusal(lambda: change(e, [none] * 4, [0] * 5, [])) == PT_ERR_STATE             # no merge since the change
        with pytest.raises(Exception):
            e.download()                                                              # views of the last merge are invalid
        merged(e)
        change(e, [none] * 4, [0] * 5, [])                                            # an empty change: nothing appended
        merged(e)
        g = BatchEngine(0)
        try:
            g.upload(batch); g.merge()
            assert refusal(lambda: change(g, [none] * 4, [0] * 5, [])) == PT_ERR_STATE         # no PT_FLAG_EMIT_SEQUENCE
        finally:
            g.close()
        with pytest.raises(ValueError, match="append it first|introduce it"):
            e.change(new, [{**header(cs[0][1], cs[0][2]), "startOp": 10_000, "ops": [{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 1,
                                                                                      "markType": "comment", "attrs": {"id": "brand-new"}}]}, None, None, None],
                     ranks)
    finally:
        e.close()
