"""pt_batch_render_patches_json: the Patch[] that Micromerge.applyChange returned for every list op of every log (reference
src/micromerge.ts:25-31, 659-703; src/peritext.ts:175-281) as UTF-8 JSON text, rendered on the device.

`render_patches_json` below is the readable specification of the output (include/peritext_b200.h, DESIGN.md §4.7), built from
the packed records and `DevicePatches` with the span render's string rules.  CPU: it emits hand-written bytes on a tiny log,
and on patch arrays encoded from the oracle's own patches it parses to what `packing.patch_stream` and the oracle return.
GPU: the device bytes equal the spec on KATs, the Patch KATs, fuzz sessions, a unicode corpus, c4 / c3 shapes and batches with
failed logs; JSON.parse of the bytes equals `patch_stream` and the oracle's applyChange results; plus the entry point's edges."""
import ctypes
import json
import random
from collections import Counter

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import (SPAN_COMMENT, SPAN_EM, SPAN_LINK, SPAN_STRONG, DevicePatches, _root_text_list, json_pools, pack_logs,
                                   patch_stream)
from tests.harness import fuzz_session, generateDocs, load_kats
from tests.test_gpu_patch_bounds import encode, list_ops, oracle_per_op
from tests.test_gpu_render_json import (HI, LO, dense_comments, fragment, fuzz_logs, ingest_pools, json_string, kat_logs, token_units,
                                        unicode_logs)

MARK_TYPES = (b"strong", b"em", b"comment", b"link")


# ------------------------------------------------------------------------------------------------------------------
# The specification
# ------------------------------------------------------------------------------------------------------------------
def _entry(data, off, k):
    return bytes(data[int(off[k]): int(off[k + 1])])


def _items_by_log(dp):
    if not hasattr(dp, "_spec_items"):
        by = {}
        for log, tag, a, b in dp.items.tolist():
            by.setdefault(log, []).append((tag, a, b))
        dp._spec_items = by
    return dp._spec_items


def render_patches_json(batch, dp, i, pools) -> bytes:
    """Log i's patches as the engine renders them: b"" unless the device computed them (patch status 0, which implies a
    merged log), else one inner array per list op in arrival order (mark record k right before ins/del record arrival_k)."""
    vals, voff, links, loff, coms, coff = pools
    if int(dp.status[i]) != 0:
        return b""
    d = batch.desc[i]
    io, mo, n, m = int(d["insdel_off"]), int(d["mark_off"]), int(d["n_insdel"]), int(d["n_mark"])
    comments, mpatches = {}, {}
    for tag, a, b in _items_by_log(dp).get(i, []):
        if tag & 0x80000000:
            mpatches.setdefault(tag & 0x7FFFFFFF, []).append((a, b))
        else:
            comments.setdefault(tag, []).append(a)

    def insdel(j):
        r = dp.recs[io + j]
        index, payload = int(r["index"]), int(batch.insdel[io + j]["payload"])
        idx = index & 0x7FFFFFFF
        if payload >> 30 == 1:
            return b'[{"action":"delete","count":1,"index":%d,"path":["text"]}]' % idx if index >> 31 else b"[]"
        f = int(r["flags"])
        marks = []
        if f & SPAN_COMMENT:
            marks.append(b'"comment":[' + b",".join(fragment(_entry(coms, coff, c)) for c in sorted(comments.get(j, []))) + b"]")
        if f & SPAN_EM:
            marks.append(b'"em":{"active":true}')
        if f & SPAN_LINK:
            marks.append(b'"link":' + fragment(_entry(links, loff, int(r["link_attr"]))))
        if f & SPAN_STRONG:
            marks.append(b'"strong":{"active":true}')
        value = json_string(token_units(payload & 0x3FFFFFFF, vals, voff))
        return b'[{"action":"insert","index":%d,"marks":{%s},"path":["text"],"values":[%s]}]' % (idx, b",".join(marks), value)

    def mark(k):
        rec = batch.marks[mo + k]
        kind, attr = int(rec["kind"]), int(rec["attr"])
        t, add = MARK_TYPES[(kind >> 1) & 3], not (kind & 1)
        ps = []
        for a, b in sorted(mpatches.get(k, [])):
            p = b'{"action":"%s",' % (b"addMark" if add else b"removeMark")
            if add and t == b"link":
                p += b'"attrs":' + fragment(_entry(links, loff, attr)) + b","
            elif add and t == b"comment":
                p += b'"attrs":' + fragment(_entry(coms, coff, attr)) + b","
            ps.append(p + b'"endIndex":%d,"markType":"%s","path":["text"],"startIndex":%d}' % (b, t, a))
        return b"[" + b",".join(ps) + b"]"

    parts, j = [], 0
    for k in range(m):
        while j < min(int(batch.marks[mo + k]["arrival"]), n):
            parts.append(insdel(j)); j += 1
        parts.append(mark(k))
    parts += [insdel(x) for x in range(j, n)]
    return b"[" + b",".join(parts) + b"]"


def per_change(log, per_op):
    """Per-op patch lists concatenated per change, as applyChange returns them."""
    lid = _root_text_list(log)
    out, k = [], 0
    for ch in log:
        c = sum(1 for op in ch["ops"] if op.get("obj") == lid)
        out.append([p for ps in per_op[k:k + c] for p in ps]); k += c
    return out


def oracle_per_change(log):
    """The oracle's applyChange results per change, makeList dropped; None where they hold a lone surrogate, which the
    oracle's UTF-8 boundary cannot carry."""
    fresh = O("observer")
    try:
        return [[p for p in fresh.applyChange(ch) if p["action"] != "makeList"] for ch in log]
    except UnicodeDecodeError:
        return None


def encoded_patches(batch, logs, seed=0):
    """DevicePatches of a batch encoded from the oracle's own patches (CPU), the item pool shuffled."""
    recs = np.zeros(len(batch.insdel), [("index", "<u4"), ("flags", "<u4"), ("link_attr", "<u4"), ("reserved", "<u4")])
    items = Counter()
    for i, log in enumerate(logs):
        per_op, elements = oracle_per_op(log)
        r, it = encode(batch, i, list_ops(log), per_op, elements)
        o = int(batch.desc[i]["insdel_off"])
        for k, row in enumerate(r):
            recs[o + k] = row
        items += it
    flat = [k for k, v in items.items() for _ in range(v)]
    random.Random(seed).shuffle(flat)
    arr = np.array(flat, dtype=[("log", "<u4"), ("tag", "<u4"), ("a", "<u4"), ("b", "<u4")]) if flat else \
        np.zeros(0, [("log", "<u4"), ("tag", "<u4"), ("a", "<u4"), ("b", "<u4")])
    return DevicePatches(recs, arr, np.zeros(batch.n_logs, np.uint32))


def tiny_log():
    """Three elements typed, a comment and a link, an element inserted inside the comment, a delete, a removeMark."""
    lid, u = "1@u", "u"

    def ch(seq, ctr, ops):
        return {"actor": u, "seq": seq, "deps": {}, "startOp": ctr, "ops": ops}

    def ins(ctr, after, v):
        return {"opId": "%d@u" % ctr, "action": "set", "obj": lid, "elemId": after, "insert": True, "value": v}

    def mark(ctr, action, mt, a, b, attrs=None):
        op = {"opId": "%d@u" % ctr, "action": action, "obj": lid, "markType": mt, "start": {"type": "before", "elemId": a},
              "end": {"type": "after", "elemId": b}}
        if attrs is not None:
            op["attrs"] = attrs
        return op
    return [ch(1, 1, [{"opId": lid, "action": "makeList", "obj": "_root", "key": "text"}, ins(2, "_head", "a"), ins(3, "2@u", HI),
                      ins(4, "3@u", '"')]),
            ch(2, 5, [mark(5, "addMark", "comment", "2@u", "3@u", {"id": "c\u00e9"}), mark(6, "addMark", "link", "3@u", "4@u", {"url": "u"})]),
            ch(3, 7, [ins(7, "2@u", LO)]),
            ch(4, 8, [{"opId": "8@u", "action": "del", "obj": lid, "elemId": "2@u"}]),
            ch(5, 9, [mark(9, "removeMark", "strong", "7@u", "7@u")])]


def tiny_patches(batch):
    """tiny_log's patch stream written by hand (the link's two patches are made up, to pin their order); the pool shuffled."""
    E, N = 0x80000000, 0xFFFFFFFF
    recs = np.array([(0 | E, 0, N, 0), (1 | E, 0, N, 0), (2 | E, 0, N, 0), (1 | E, SPAN_COMMENT | (1 << 8), N, 0), (0 | E, 0, N, 0)],
                    dtype=[("index", "<u4"), ("flags", "<u4"), ("link_attr", "<u4"), ("reserved", "<u4")])
    items = np.array([(0, 1 | E, 2, 3), (0, 3, 0, 0), (0, 0 | E, 0, 2), (0, 1 | E, 0, 1)],
                     dtype=[("log", "<u4"), ("tag", "<u4"), ("a", "<u4"), ("b", "<u4")])
    assert batch.desc[0]["n_insdel"] == 5 and batch.desc[0]["n_mark"] == 3 and batch.marks["arrival"].tolist() == [3, 3, 5]
    return DevicePatches(recs, items, np.zeros(1, np.uint32))


TINY = (b'[[{"action":"insert","index":0,"marks":{},"path":["text"],"values":["a"]}],'
        b'[{"action":"insert","index":1,"marks":{},"path":["text"],"values":["\\ud83d"]}],'
        b'[{"action":"insert","index":2,"marks":{},"path":["text"],"values":["\\""]}],'
        b'[{"action":"addMark","attrs":{"id":"c\xc3\xa9"},"endIndex":2,"markType":"comment","path":["text"],"startIndex":0}],'
        b'[{"action":"addMark","attrs":{"url":"u"},"endIndex":1,"markType":"link","path":["text"],"startIndex":0},'
        b'{"action":"addMark","attrs":{"url":"u"},"endIndex":3,"markType":"link","path":["text"],"startIndex":2}],'
        b'[{"action":"insert","index":1,"marks":{"comment":[{"id":"c\xc3\xa9"}]},"path":["text"],"values":["\\ude00"]}],'
        b'[{"action":"delete","count":1,"index":0,"path":["text"]}],'
        b'[]]')


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_spec_emits_hand_written_bytes_on_a_tiny_log():
    """Keys sorted; every value its own string (a surrogate pair split over two elements is two escapes); mark ops before the
    ins/del record their arrival names; a mark's patches by startIndex whatever the pool order; a mark op without patches []."""
    log = tiny_log()
    batch = pack_logs([log])
    dp = tiny_patches(batch)
    pools = json_pools(batch)
    out = render_patches_json(batch, dp, 0, pools)
    assert out == TINY
    assert json.loads(out) == patch_stream(batch, dp, 0, list_ops(log))
    # a failed or not-computed log is zero bytes; a log without list ops is []
    dp.status[0] = 1
    assert render_patches_json(batch, dp, 0, pools) == b""
    e = O("doc1")
    empty = [e.change([{"path": [], "action": "makeList", "key": "text"}])["change"]]
    eb = pack_logs([empty])
    assert render_patches_json(eb, DevicePatches(dp.recs[:0], dp.items[:0], np.zeros(1, np.uint32)), 0, json_pools(eb)) == b"[]"


def patch_kat_logs():
    """The reference's four exact Patch KATs (test/micromerge.ts:915-1029): (log, expected patches of its last change)."""
    out = []
    for kat in [k for k in load_kats() if k["kind"] == "script" and any("expectPatches" in st for st in k["steps"])]:
        docs, _, init = generateDocs(O, kat["initialText"])
        logs, saved = [[init], [init]], {}
        for st in kat["steps"]:
            d = st["doc"] - 1
            if st["do"] == "change":
                ch = docs[d].change(st["ops"])["change"]
                logs[d].append(ch)
                if "save" in st:
                    saved[st["save"]] = ch
            elif st["do"] == "applyChange":
                docs[d].applyChange(saved[st["change"]])
                logs[d].append(saved[st["change"]])
                if "expectPatches" in st:
                    out.append((list(logs[d]), st["expectPatches"]))
    return out


def test_spec_parses_to_patch_stream_and_the_oracle_on_encoded_patch_kats():
    cases = patch_kat_logs()
    assert len(cases) == 4
    logs = [l for l, _ in cases]
    batch = pack_logs(logs)
    dp = encoded_patches(batch, logs, seed=1)
    pools = json_pools(batch)
    for i, (log, want) in enumerate(cases):
        got = json.loads(render_patches_json(batch, dp, i, pools))
        assert got == patch_stream(batch, dp, i, list_ops(log))
        assert per_change(log, got) == oracle_per_change(log)
        assert per_change(log, got)[-1] == want


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pjengine():
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0, emit_patches=True)
    yield e
    e.close()


def assert_patches_render(engine, batch, dp, pools=None):
    """Device bytes of every log == the spec over `dp` (the engine's own patch stream)."""
    p = json_pools(batch) if pools is None else pools
    data, off = engine.render_patches_json(batch, p)
    assert len(off) == batch.n_logs + 1 and int(off[0]) == 0 and int(off[-1]) == len(data)
    raw = data.tobytes()
    bad = [i for i in range(batch.n_logs) if raw[int(off[i]): int(off[i + 1])] != render_patches_json(batch, dp, i, p)]
    assert not bad, (len(bad), bad[:5], raw[int(off[bad[0]]): int(off[bad[0] + 1])][:300] if bad else None)
    return [raw[int(off[i]): int(off[i + 1])] for i in range(batch.n_logs)]


def check_against_decoder_and_oracle(engine, logs, min_oracle=None):
    batch = pack_logs(logs)
    merged, dp = engine.run_with_patches(batch)
    assert (merged.results["status"] == 0).all() and (dp.status == 0).all()
    per = assert_patches_render(engine, batch, dp)
    checked = 0
    for i, log in enumerate(logs):
        got = json.loads(per[i])
        assert got == patch_stream(batch, dp, i, list_ops(log)), i
        want = oracle_per_change(log)
        if want is not None:
            assert per_change(log, got) == want, i
            checked += 1
    assert checked >= (len(logs) if min_oracle is None else min_oracle)
    return batch, dp, per


@pytest.mark.gpu
def test_kats_render_patches_on_the_device(pjengine):
    check_against_decoder_and_oracle(pjengine, kat_logs())


@pytest.mark.gpu
def test_patch_kats_render_on_the_device(pjengine):
    cases = patch_kat_logs()
    _, _, per = check_against_decoder_and_oracle(pjengine, [l for l, _ in cases])
    for (log, want), b in zip(cases, per):
        assert per_change(log, json.loads(b))[-1] == want


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(6))
def test_fuzz_sessions_render_patches_on_the_device(pjengine, seed):
    # the sessions of test_gpu_patches.py: unconverged replicas, zero-width marks, removed comments
    _, logs, _ = fuzz_session(O, 7000 + seed, 120, sync_prob=0.6 if seed % 3 else 1.0,
                              zero_width_prob=0.1 if seed % 2 else 0.0, full_sync_at_end=bool(seed % 4), remove_comments=bool(seed % 2))
    check_against_decoder_and_oracle(pjengine, logs)


@pytest.mark.gpu
def test_render_json_fuzz_corpus_renders_patches(pjengine):
    check_against_decoder_and_oracle(pjengine, fuzz_logs(range(8500, 8504)))


@pytest.mark.gpu
def test_unicode_corpus_renders_patches_on_the_device(pjengine):
    logs = unicode_logs()
    batch, dp, per = check_against_decoder_and_oracle(pjengine, logs, min_oracle=3)    # the others hold lone surrogates
    # a pair split over two elements: two values, two escapes
    assert b'"values":["\\ud83d"]' in per[2] and b'"values":["\\ude00"]' in per[2]
    assert b"\\u001f" in per[0] and b"\\u001F" not in per[0]
    assert b'"attrs":{"url":"lone\\udc01"}' in per[7] and b"\\ud800" in per[7]
    for b in per:
        b.decode("utf-8")
    # the raw ingest pools give the same bytes
    data, off = pjengine.render_patches_json(batch)
    data2, off2 = pjengine.render_patches_json(batch, ingest_pools(logs))
    assert data2.tobytes() == data.tobytes() and off2.tolist() == off.tolist()


@pytest.mark.gpu
def test_c4_batch_renders_patches(pjengine):
    from peritext_b200 import workload
    batch = dense_comments(workload.generate("c4", n_docs=1000))
    merged, dp = pjengine.run_with_patches(batch)
    assert batch.n_logs == 3000 and (merged.results["status"] == 0).all() and (dp.status == 0).all()
    per = assert_patches_render(pjengine, batch, dp)
    for i in (0, 1500, 2999):
        assert len(json.loads(per[i])) == int(batch.desc[i]["n_insdel"]) + int(batch.desc[i]["n_mark"])


@pytest.mark.gpu
def test_c3_logs_and_a_c2_log_left_to_the_host(pjengine):
    from peritext_b200 import workload
    batch = dense_comments(workload.generate("c3", n_docs=3, ops_per_doc=10000))
    merged, dp = pjengine.run_with_patches(batch)
    assert (merged.results["status"] == 0).all() and (dp.status == 0).sum() >= 1, dp.status
    per = assert_patches_render(pjengine, batch, dp)
    for i in np.nonzero(dp.status == 0)[0]:
        assert len(json.loads(per[i])) == int(batch.desc[i]["n_insdel"]) + int(batch.desc[i]["n_mark"])
    big = dense_comments(workload.generate("c2", n_docs=1, ops_per_doc=40000))
    merged, dp = pjengine.run_with_patches(big)
    assert (merged.results["status"] == 0).all() and (dp.status == 1).all()
    data, off = pjengine.render_patches_json(big)
    assert len(data) == 0 and set(off.tolist()) == {0}


@pytest.mark.gpu
def test_failed_logs_render_patches_as_nothing():
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_admission import tampered_logs
    from tests.test_gpu_routes import FAULTS, Log, batch_of, marks_over, route_base, typing_forward, with_fault
    logs = []
    for k, f in enumerate(f for f in FAULTS if f != "clean"):
        logs += [route_base("compact"), with_fault(route_base("direct" if k % 2 else "packed3"), f)]
    logs.append(route_base("direct"))
    batch = batch_of(logs)
    e = BatchEngine(0, emit_patches=True)
    try:
        merged, dp = e.run_with_patches(batch)
        st = merged.results["status"]
        assert (st[0::2] == 0).all() and (st[1::2] != 0).all() and len(set(st[1::2].tolist())) >= 3
        per = assert_patches_render(e, batch, dp)
        assert all(per[i] == b"" for i in range(1, batch.n_logs, 2))
        assert all(int(dp.status[i]) != 0 or len(per[i]) > 2 for i in range(0, batch.n_logs, 2))
        # admission-rejected logs (status 6 / 7)
        ab = pack_logs([l for _, l in tampered_logs()], with_changes=True)
        merged, dp = e.run_with_patches(ab)
        st = merged.results["status"]
        assert {6, 7} <= set(st.tolist()) and (st == 0).any()
        per = assert_patches_render(e, ab, dp)
        assert all(per[i] == b"" for i in range(ab.n_logs) if st[i] != 0)
        assert all(per[i] != b"" for i in range(ab.n_logs) if st[i] == 0 and dp.status[i] == 0)
        lg = []
        for k in range(12):
            x = Log(2)
            ids = typing_forward(x, 80, [0, 1])
            marks_over(x, ids, 40 if k % 3 == 0 else 2, seed=k, types=(2,), n_ids=40)
            lg.append(x)
        ob = batch_of(lg)
    finally:
        e.close()
    # PT_LOG_OVERFLOW logs (status 4): a comment pool too small for some logs, no re-merge
    e = BatchEngine(0, comment_pool_entries=300, emit_patches=True)
    try:
        e.upload(ob); e.merge()
        merged = e.download()
        recs, items, status, needed = e.download_patches()
        assert needed <= len(items) or needed == 0
        st = merged.results["status"]
        assert (st == 4).any() and (st == 0).any(), st
        dp = DevicePatches(recs, items, status)
        per = assert_patches_render(e, ob, dp)
        assert all(per[i] == b"" for i in range(ob.n_logs) if st[i] == 4)
    finally:
        e.close()


@pytest.mark.gpu
def test_two_merges_render_identical_bytes():
    from peritext_b200.engine import BatchEngine
    logs = fuzz_logs(range(8600, 8606)) + [l for l, _ in patch_kat_logs()]
    batch = pack_logs(logs)
    outs = []
    for _ in range(2):
        e = BatchEngine(0, emit_patches=True)
        try:
            merged, dp = e.run_with_patches(batch)
            outs.append(e.render_patches_json(batch))
            e.merge()                                         # the same handle again (its launch sequence as a graph)
            outs.append(e.render_patches_json(batch))
            assert_patches_render(e, batch, dp)
        finally:
            e.close()
    for d, o in outs[1:]:
        assert d.tobytes() == outs[0][0].tobytes() and o.tobytes() == outs[0][1].tobytes()


@pytest.mark.gpu
def test_render_patches_edge_cases():
    from peritext_b200.engine import BatchEngine, EngineError, _JsonPools, _JsonView, _PatchView, _check, _json_pools
    logs = unicode_logs()
    batch = pack_logs(logs)
    # a handle without PT_FLAG_EMIT_PATCHES
    e = BatchEngine(0)
    try:
        e.run(batch)
        with pytest.raises(EngineError, match="out of order.*PT_FLAG_EMIT_PATCHES"):
            e.render_patches_json(batch)
    finally:
        e.close()
    e = BatchEngine(0, emit_patches=True)
    try:
        # before any merge, and after an upload without a merge
        with pytest.raises(EngineError, match="out of order"):
            e.render_patches_json(batch)
        e.upload(batch)
        with pytest.raises(EngineError, match="out of order"):
            e.render_patches_json(batch)
        # a truncated item pool: PT_ERR_STATE with the demand; one re-merge with that pool size renders
        e.set_patch_pool(4)
        e.merge(); e.download()
        _, items, _, needed = e.download_patches()
        assert len(items) == 4 and needed > 4
        with pytest.raises(EngineError, match="out of order.*needs %d patch items" % needed):
            e.render_patches_json(batch)
        e.set_patch_pool(needed)
        with pytest.raises(EngineError, match="out of order.*replaced after the last merge"):
            e.render_patches_json(batch)
        e.merge()
        merged = e.download()
        recs, items, pst, need = e.download_patches()
        assert need == len(items) == needed
        dp = DevicePatches(recs, items, pst)
        assert_patches_render(e, batch, dp)
        digests = merged.results["digest"].copy()
        # null arguments
        v, st = _JsonView(), _JsonPools()
        L = e._L
        assert L.pt_batch_render_patches_json(e._h, None, ctypes.byref(v)) == 1
        assert L.pt_batch_render_patches_json(e._h, ctypes.byref(st), None) == 1
        assert L.pt_batch_render_patches_json(None, ctypes.byref(st), ctypes.byref(v)) == 1
        # a missing value, link or comment entry: PT_ERR_INVALID naming it
        full = json_pools(batch)
        for k, what in ((0, "value"), (2, "link"), (4, "comment")):
            p = list(full)
            p[k + 1] = p[k + 1][:-1]
            p[k] = p[k][: int(p[k + 1][-1])]
            with pytest.raises(EngineError, match="pt_batch_render_patches_json: log \\d+ names %s pool entry %d" % (what, len(p[k + 1]) - 1)):
                e.render_patches_json(batch, tuple(p))
        # the two renders interleaved: each view stays valid and unchanged; the spans, digests and patch view too
        spans = e.download(copy=False)
        spans_copy = [spans.canonical(i) for i in range(batch.n_logs)]
        pv = _PatchView()
        _check(L.pt_batch_download_patches(e._h, ctypes.byref(pv)), "pt_batch_download_patches")
        pv_recs = ctypes.string_at(pv.recs, len(recs) * 16)
        st, _keep = _json_pools(batch, full)
        vs, vp = _JsonView(), _JsonView()
        assert L.pt_batch_render_json(e._h, ctypes.byref(st), ctypes.byref(vs)) == 0
        spans_json = ctypes.string_at(vs.bytes, vs.n_bytes)
        assert L.pt_batch_render_patches_json(e._h, ctypes.byref(st), ctypes.byref(vp)) == 0
        patches_json = ctypes.string_at(vp.bytes, vp.n_bytes)
        assert vp.bytes != vs.bytes and vp.off != vs.off
        assert L.pt_batch_render_json(e._h, ctypes.byref(st), ctypes.byref(_JsonView())) == 0
        assert ctypes.string_at(vp.bytes, vp.n_bytes) == patches_json
        vp2 = _JsonView()
        assert L.pt_batch_render_patches_json(e._h, ctypes.byref(st), ctypes.byref(vp2)) == 0
        assert ctypes.string_at(vp2.bytes, vp2.n_bytes) == patches_json                 # twice: identical bytes
        assert ctypes.string_at(vs.bytes, vs.n_bytes) == spans_json
        assert spans_json == b"".join(e.render_json_list(batch))
        assert [spans.canonical(i) for i in range(batch.n_logs)] == spans_copy
        assert (e.results()["digest"] == digests).all()
        assert ctypes.string_at(pv.recs, len(recs) * 16) == pv_recs
        r2, i2, s2, n2 = e.download_patches()
        assert r2.tobytes() == recs.tobytes() and i2.tobytes() == items.tobytes() and s2.tobytes() == pst.tobytes() and n2 == need
        # a batch of zero logs
        empty = batch.select([])
        e.run(empty)
        data, off = e.render_patches_json(empty)
        assert len(data) == 0 and off.tolist() == [0]
    finally:
        e.close()
