"""pt_batch_render_json: every merged document's FormatSpanWithText[] (reference src/peritext.ts:35-38, 337-455) as UTF-8
JSON text, rendered on the device.

`render_spans_json` below is the readable specification of the output (include/peritext_b200.h, DESIGN.md §4.6), built from
`packing.decode_spans` and JSON.stringify's string rules.  CPU: it agrees with `decode_spans` on the reference's shapes, it
emits the bytes a JS engine would on hand-written cases, and `packing.json_pools` agrees byte for byte with the pools the
native ingest hands out.  GPU: the device bytes equal the spec on KATs, fuzz sessions, a unicode corpus, every merge-kernel
route case, c2 / c3 / c4 / c5 shapes and batches with failed logs; plus the entry point's edge cases."""
import json
import os
import re

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200.packing import (SPAN_COMMENT, SPAN_EM, SPAN_LINK, SPAN_STRONG, TOKEN_POOLED, decode_spans,
                                   json_pools, pack_logs)
from tests.harness import GOLDEN, fuzz_session, generateDocs, load_kats, run_concurrent


# ------------------------------------------------------------------------------------------------------------------
# The specification
# ------------------------------------------------------------------------------------------------------------------
_ESC = {0x22: b'\\"', 0x5C: b"\\\\", 0x08: b"\\b", 0x09: b"\\t", 0x0A: b"\\n", 0x0C: b"\\f", 0x0D: b"\\r"}
_LONE = re.compile(rb"\xed[\xa0-\xbf][\x80-\xbf]")


def json_string(units) -> bytes:
    """JSON.stringify of a string given as UTF-16 code units (the well-formed form: lone surrogates as \\udxxx)."""
    out = bytearray(b'"')
    k, n = 0, len(units)
    while k < n:
        u = units[k]
        if 0xD800 <= u < 0xDC00 and k + 1 < n and 0xDC00 <= units[k + 1] < 0xE000:
            out += chr(0x10000 + ((u - 0xD800) << 10) + (units[k + 1] - 0xDC00)).encode("utf-8")
            k += 2
            continue
        if u in _ESC:
            out += _ESC[u]
        elif u < 0x20 or 0xD800 <= u < 0xE000:
            out += b"\\u%04x" % u
        else:
            out += chr(u).encode("utf-8")
        k += 1
    return bytes(out + b'"')


def fragment(b: bytes) -> bytes:
    """A pool fragment as written: verbatim, the 3-byte encoding of a lone surrogate as \\udxxx."""
    return _LONE.sub(lambda m: b"\\u%04x" % (0xD000 | ((m[0][1] & 0x3F) << 6) | (m[0][2] & 0x3F)), b)


def _entry(data, off, k):
    return bytes(data[int(off[k]): int(off[k + 1])])


def token_units(tok, vals, voff):
    tok = int(tok)
    if tok & TOKEN_POOLED:
        return np.frombuffer(_entry(vals, voff, tok & (TOKEN_POOLED - 1)), "<u2").tolist()
    if tok >= 0x10000:
        return [0xD800 + ((tok - 0x10000) >> 10), 0xDC00 + ((tok - 0x10000) & 0x3FF)]
    return [tok]


def render_spans_json(batch, merged, i, pools) -> bytes:
    """Log i's getTextWithFormatting result as the engine renders it: b"" for a failed log, else
    [{"marks":{sorted marks},"text":T},...] with T = JSON.stringify of the span's concatenated UTF-16 text."""
    vals, voff, links, loff, coms, coff = pools
    r = merged.results[i]
    if int(r["status"]) != 0:
        return b""
    toks, sp = merged.tokens(i), merged.span_records(i)
    parts = []
    for j, s in enumerate(sp):
        a = int(s["start"])
        b = int(sp[j + 1]["start"]) if j + 1 < len(sp) else int(r["n_visible"])
        f = int(s["flags"])
        marks = []
        if f & SPAN_COMMENT:
            co = int(s["comment_off"])
            marks.append(b'"comment":[' + b",".join(fragment(_entry(coms, coff, int(c))) for c in merged.comment_pool[co: co + (f >> 8)]) + b"]")
        if f & SPAN_EM:
            marks.append(b'"em":{"active":true}')
        if f & SPAN_LINK:
            marks.append(b'"link":' + fragment(_entry(links, loff, int(s["link_attr"]))))
        if f & SPAN_STRONG:
            marks.append(b'"strong":{"active":true}')
        units = []
        for t in toks[a:b]:
            units += token_units(t, vals, voff)
        parts.append(b'{"marks":{' + b",".join(marks) + b'},"text":' + json_string(units) + b"}")
    return b"[" + b",".join(parts) + b"]"


def utf16_normalised(spans):
    """Span texts through a UTF-16 round trip, so that adjacent surrogate halves compare as one character."""
    return [{"marks": s["marks"], "text": s["text"].encode("utf-16-le", "surrogatepass").decode("utf-16-le", "surrogatepass")} for s in spans]


# ------------------------------------------------------------------------------------------------------------------
# Corpora
# ------------------------------------------------------------------------------------------------------------------
def text_log(values, marks=(), actor="u"):
    """One replica typing `values` (one element each) and then applying `marks` = (action, markType, first, last, attrs):
    mark ops from before element `first` to after element `last`."""
    lid = "1@" + actor
    ops = [{"opId": lid, "action": "makeList", "obj": "_root", "key": "text"}]
    prev, ids = "_head", []
    for k, v in enumerate(values):
        oid = "%d@%s" % (k + 2, actor)
        ops.append({"opId": oid, "action": "set", "obj": lid, "elemId": prev, "insert": True, "value": v})
        prev = oid
        ids.append(oid)
    ctr = len(values) + 2
    for action, mt, a, b, attrs in marks:
        op = {"opId": "%d@%s" % (ctr, actor), "action": action, "obj": lid, "markType": mt,
              "start": {"type": "before", "elemId": ids[a]}, "end": {"type": "after", "elemId": ids[b]}}
        if attrs is not None:
            op["attrs"] = attrs
        ops.append(op)
        ctr += 1
    return [{"actor": actor, "seq": 1, "deps": {}, "startOp": 1, "ops": ops}]


HI, LO = "\ud83d", "\ude00"
ODD_COMMENTS = [{"id": 'q"uote'}, {"id": "back\\slash"}, {"id": "é中\U0001F600"}, {"id": "lone\ud800x"}, {"id": "ctl\x01\n\x7f"}]
ODD_LINKS = [{"url": 'https://x.y/?q="1"&r=\\'}, {"url": "https://é.example/\U0001F600"}, {"url": "lone\udc01"}]


def unicode_logs():
    """Control characters, escapes, non-BMP text, lone surrogates, pairs split across elements, across an empty value and
    across a mark boundary, multi-character values, and attrs with quotes, backslashes, non-ASCII and lone surrogates."""
    controls = [chr(c) for c in range(0x20)]
    plain = ['"', "\\", "/", "\x7f", "\u2028", "\u2029", "é", "中", "\U0001F600", "a"]
    logs = [
        text_log(controls + plain),
        text_log(["a", HI, "b", LO, "c", HI]),                                    # lone high, lone low, trailing high
        text_log(["x", HI, LO, "y"]),                                             # a pair split across two elements
        text_log(["x", HI, "", LO, "y"]),                                         # ... with an empty value between
        text_log(["x", HI, LO, "y"], [("addMark", "strong", 0, 1, None)]),        # ... split by a mark boundary
        text_log(["p" + HI, LO + "q", "", "mid" + HI, HI + "Z" + LO, LO, "r" + HI, LO]),   # pairs across multi-character values
        text_log(["", "", "a", ""]),                                              # empty values
        text_log(list("abcdef"), [("addMark", "comment", 0, 3, ODD_COMMENTS[k]) for k in range(5)] +
                 [("addMark", "link", 1, 4, ODD_LINKS[k]) for k in range(3)] + [("addMark", "em", 2, 5, None)]),
        text_log(list("abcdef"), [("removeMark", "comment", 1, 2, {"id": "x"})]),  # {comment: []} (quirk Q3)
        text_log(list("0123456789"), [("addMark", "link", 0, 9, ODD_LINKS[2]), ("addMark", "comment", 3, 6, ODD_COMMENTS[3])]),
    ]
    # a long span whose pairs straddle the 32-element trips, and all-empty trips between the halves
    long_vals = []
    for k in range(150):
        long_vals += ["w", HI, LO] if k % 3 else [HI + "v", "", LO]
    long_vals += [HI] + [""] * 70 + [LO] + [""] * 40 + [HI] + [""] * 64 + ["z"] + [HI] + [""] * 95
    logs.append(text_log(long_vals))
    logs.append(text_log(long_vals, [("addMark", "strong", 31, 200, None), ("addMark", "comment", 60, 64, ODD_COMMENTS[0])]))
    return logs


def kat_logs(with_expected=False):
    """Both replicas of all 46 KATs: the concurrent ones as testConcurrentWrites runs them, the scripted ones by replaying
    their change / applyChange steps (expected spans: the concurrent KATs' expectedResult, None for the scripted ones)."""
    logs, expected = [], []
    for kat in load_kats():
        if kat["kind"] == "concurrent":
            rec = []
            run_concurrent(O, kat, record=rec)
            logs += rec
            expected += [kat["expectedResult"]] * 2
            continue
        docs, _, init = generateDocs(O, kat["initialText"])
        lg, saved = [[init], [init]], {}
        for st in kat["steps"]:
            d = st["doc"] - 1
            if st["do"] == "change":
                ch = docs[d].change(st["ops"])["change"]
                lg[d].append(ch)
                if "save" in st:
                    saved[st["save"]] = ch
            elif st["do"] == "applyChange":
                docs[d].applyChange(saved[st["change"]])
                lg[d].append(saved[st["change"]])
        logs += lg
        expected += [None, None]
    return (logs, expected) if with_expected else logs


def fuzz_logs(seeds):
    logs = []
    for seed in seeds:
        _, lg, _ = fuzz_session(O, seed, 120, max_chars=3, zero_width_prob=0.2)
        logs += lg
    return logs


def links_minimal_logs():
    q = json.load(open(os.path.join(GOLDEN, "links_minimal_queues.json")))["queues"]
    return [[q["doc0"][0], q["doc0"][1], q["doc1"][0], q["doc2"][0]], [q["doc0"][0], q["doc2"][0], q["doc1"][0], q["doc0"][1]]]


def check_spec_against_decode(logs):
    batch = pack_logs(logs)
    ref, _ = replay_packed(batch)
    pools = json_pools(batch)
    for i in range(batch.n_logs):
        assert int(ref.results[i]["status"]) == 0
        got = json.loads(render_spans_json(batch, ref, i, pools).decode("utf-8"))
        assert utf16_normalised(got) == utf16_normalised(decode_spans(batch, ref, i)), i
    return batch, ref


# ------------------------------------------------------------------------------------------------------------------
# CPU: the spec against decode_spans, against JS, and the two pool sources
# ------------------------------------------------------------------------------------------------------------------
def test_kats_agree_with_the_reference_shapes():
    logs, expected = kat_logs(with_expected=True)
    assert len(logs) == 2 * 46
    batch, ref = check_spec_against_decode(logs)
    # the concurrent KATs' own expected spans (the reference's values), through JSON.parse of the rendered text
    pools = json_pools(batch)
    for i in range(batch.n_logs):
        if expected[i] is not None:
            assert json.loads(render_spans_json(batch, ref, i, pools)) == expected[i]
    assert sum(e is not None for e in expected) == 62


@pytest.mark.parametrize("seeds", [range(8400, 8406), range(8406, 8412)])
def test_fuzz_sessions_agree_with_decode(seeds):
    check_spec_against_decode(fuzz_logs(seeds))


def test_links_minimal_trace_agrees_with_decode():
    batch, ref = check_spec_against_decode(links_minimal_logs())
    pools = json_pools(batch)
    assert render_spans_json(batch, ref, 0, pools) == b'[{"marks":{"link":{"url":"https://inkandswitch.com/pushpin"}},"text":"ABC9ee09150DE"}]'


def test_unicode_corpus_agrees_with_decode():
    check_spec_against_decode(unicode_logs())


def rendered(logs):
    batch = pack_logs(logs)
    ref, _ = replay_packed(batch)
    pools = json_pools(batch)
    return [render_spans_json(batch, ref, i, pools) for i in range(batch.n_logs)]


def test_spec_emits_what_json_stringify_writes():
    """Expected bytes written by hand from ECMA-262 JSON.stringify / QuoteJSONString (well-formed JSON.stringify)."""
    ctl = b"".join({8: b"\\b", 9: b"\\t", 10: b"\\n", 12: b"\\f", 13: b"\\r"}.get(c, b"\\u%04x" % c) for c in range(0x20))
    assert ctl[:12] == b"\\u0000\\u0001" and b"\\u001f" in ctl and b"\\u000b" in ctl
    out = rendered([text_log([chr(c) for c in range(0x20)] + ['"', "\\", "/", "\x7f", "\u2028", "\u2029", "\U0001F600"]),
                    text_log(["a", HI, "b", LO, "c"]),
                    text_log(["x", HI, LO, "y"]),
                    text_log(["x", HI, "", LO, "y"]),
                    text_log(["x", HI, LO, "y"], [("addMark", "strong", 0, 1, None)]),
                    text_log(["", "a", ""]),
                    text_log(list("abcdef"), [("removeMark", "comment", 1, 2, {"id": "x"})])])
    assert out[0] == (b'[{"marks":{},"text":"' + ctl + b'\\"\\\\/\x7f\xe2\x80\xa8\xe2\x80\xa9\xf0\x9f\x98\x80"}]')
    assert out[1] == b'[{"marks":{},"text":"a\\ud83db\\ude00c"}]'
    assert out[2] == b'[{"marks":{},"text":"x\xf0\x9f\x98\x80y"}]'                 # pair across two elements
    assert out[3] == b'[{"marks":{},"text":"x\xf0\x9f\x98\x80y"}]'                 # ... with "" between them
    assert out[4] == b'[{"marks":{"strong":{"active":true}},"text":"x\\ud83d"},{"marks":{},"text":"\\ude00y"}]'
    assert out[5] == b'[{"marks":{},"text":"a"}]'
    assert out[6] == b'[{"marks":{},"text":"a"},{"marks":{"comment":[]},"text":"bc"},{"marks":{},"text":"def"}]'
    for b in out:
        b.decode("utf-8")                                                         # always valid UTF-8
    # an empty document, and every mark at once in sorted key order
    e = O("doc1")
    empty = [e.change([{"path": [], "action": "makeList", "key": "text"}])["change"]]
    out = rendered([empty, text_log(list("ab"), [("addMark", "strong", 0, 1, None), ("addMark", "link", 0, 1, {"url": "u"}),
                                                 ("addMark", "comment", 0, 1, {"id": "b"}), ("addMark", "em", 0, 1, None),
                                                 ("addMark", "comment", 0, 1, {"id": "a"})])])
    assert out[0] == b"[]"
    assert out[1] == (b'[{"marks":{"comment":[{"id":"a"},{"id":"b"}],"em":{"active":true},"link":{"url":"u"},'
                      b'"strong":{"active":true}},"text":"ab"}]')
    # lone surrogates inside attrs fragments
    assert fragment('{"id":"x\ud800"}'.encode("utf-8", "surrogatepass")) == b'{"id":"x\\ud800"}'
    assert fragment("é\U0001F600".encode("utf-8")) == "é\U0001F600".encode("utf-8")


def ingest_pools(logs):
    """pt_ingest_pool kinds 0 / 1 / 3 of the logs, raw (data, offsets) as the native ingest hands them out."""
    import ctypes
    from peritext_b200.engine import _check, _view, load_library
    L = load_library()
    blobs = [json.dumps(l).encode("utf-8") for l in logs]
    ptrs = (ctypes.c_char_p * len(blobs))(*blobs)
    lens = (ctypes.c_uint64 * len(blobs))(*[len(b) for b in blobs])
    h = ctypes.c_void_p()
    _check(L.pt_ingest_create(ctypes.byref(h)), "pt_ingest_create")
    try:
        assert L.pt_ingest_parse(h, ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(lens, ctypes.c_void_p), len(blobs), 1) == 0
        out = []
        for kind in (0, 1, 3):
            data, off, cnt, first = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_void_p()
            _check(L.pt_ingest_pool(h, kind, ctypes.byref(data), ctypes.byref(off), ctypes.byref(cnt), ctypes.byref(first)), "pt_ingest_pool")
            o = _view(off.value, cnt.value + 1, np.uint64) if off.value else np.zeros(1, np.uint64)
            d = _view(data.value, o[-1], np.uint8)
            out += [d, o]
        return tuple(out)
    finally:
        L.pt_ingest_destroy(h)


@pytest.mark.parametrize("corpus", ["kats", "fuzz", "unicode"])
def test_json_pools_equal_the_ingest_pools(corpus):
    logs = {"kats": kat_logs, "fuzz": lambda: fuzz_logs(range(8420, 8424)), "unicode": unicode_logs}[corpus]()
    mine = json_pools(pack_logs(logs))
    raw = ingest_pools(logs)
    for k, (a, b) in enumerate(zip(mine, raw)):
        assert a.tobytes() == b.tobytes(), k
    if corpus == "unicode":
        assert len(mine[0]) and b"\xed\xa0\x80" in mine[4].tobytes() and b"\xed\xb0\x81" in mine[2].tobytes()


def test_json_pools_needs_real_comment_ids():
    from peritext_b200 import workload
    batch = workload.generate("c4", n_docs=2)
    with pytest.raises(ValueError, match="comment_ids"):
        json_pools(batch)
    dense_comments(batch)
    assert len(json_pools(batch)) == 6


def dense_comments(batch):
    """A generated batch's synthetic comment attrs (sparse integers) re-ranked densely in the same order, with attrs objects
    {"id": "comment-%010d"}: the merge results are unchanged apart from the rank numbers."""
    mk = batch.marks
    is_c = ((mk["kind"] >> 1) & 3) == 2
    ids = np.unique(mk["attr"][is_c])
    if len(mk):
        mk = mk.copy()
        mk["attr"][is_c] = np.searchsorted(ids, mk["attr"][is_c])
        batch.marks = mk
    batch.comment_ids = [{"id": "comment-%010d" % int(x)} for x in ids]
    return batch


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rengine():
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0)
    yield e
    e.close()


def assert_render_matches(engine, batch, merged, pools=None):
    """Device bytes of every log == the spec over `merged` (the oracle's replay or the engine's own download)."""
    p = json_pools(batch) if pools is None else pools
    data, off = engine.render_json(batch, p)
    assert len(off) == batch.n_logs + 1 and int(off[0]) == 0 and int(off[-1]) == len(data)
    raw = data.tobytes()
    bad = []
    for i in range(batch.n_logs):
        want = render_spans_json(batch, merged, i, p)
        if raw[int(off[i]): int(off[i + 1])] != want:
            bad.append(i)
    assert not bad, (len(bad), bad[:5], raw[int(off[bad[0]]): int(off[bad[0] + 1])][:300] if bad else None)
    return raw, off


@pytest.mark.gpu
def test_kats_render_on_the_device(rengine):
    batch = pack_logs(kat_logs())
    got = rengine.run(batch)
    ref, _ = replay_packed(batch)
    assert (ref.results["status"] == 0).all()
    assert_render_matches(rengine, batch, ref)
    _, expected = kat_logs(with_expected=True)
    for i, b in enumerate(rengine.render_json_list(batch)):
        if expected[i] is not None:
            assert json.loads(b) == expected[i]


@pytest.mark.gpu
def test_fuzz_sessions_render_on_the_device(rengine):
    batch = pack_logs(fuzz_logs(range(8500, 8516)))
    rengine.run(batch)
    ref, _ = replay_packed(batch, threads=4)
    assert_render_matches(rengine, batch, ref)


@pytest.mark.gpu
def test_unicode_corpus_renders_on_the_device(rengine):
    logs = unicode_logs()
    batch = pack_logs(logs)
    rengine.run(batch)
    ref, _ = replay_packed(batch)
    raw, off = assert_render_matches(rengine, batch, ref)
    per = [raw[int(off[i]): int(off[i + 1])] for i in range(batch.n_logs)]
    assert per[2] == b'[{"marks":{},"text":"x\xf0\x9f\x98\x80y"}]' and per[3] == per[2]
    assert b'\\ud83d"},{' in per[4] and b'"text":"\\ude00y"' in per[4]
    assert b'\\u00' in per[0] and b"\\u001f" in per[0] and b"\\u001F" not in per[0]
    assert b"\\ud800" in per[7] and b"\\udc01" in per[7]
    for i, b in enumerate(per):
        assert utf16_normalised(json.loads(b)) == utf16_normalised(decode_spans(batch, ref, i)), i
    # the raw ingest pools give the same bytes
    data, off2 = rengine.render_json(batch, ingest_pools(logs))
    assert data.tobytes() == raw and off2.tolist() == off.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["default", "block-only"])
def test_route_cases_render_on_the_device(config):
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_routes import all_cases, joint_batch, kernel_config
    batch = joint_batch(all_cases())
    ref, _ = replay_packed(batch, threads=8)
    with kernel_config("default" if config == "default" else "cta-only"):
        e = BatchEngine(0)
        try:
            got = e.run(batch)
            for i in range(batch.n_logs):
                assert got.canonical(i) == ref.canonical(i)
            assert_render_matches(e, batch, ref)
        finally:
            e.close()


@pytest.mark.gpu
def test_c4_batch_renders_on_the_device(rengine):
    from peritext_b200 import workload
    batch = dense_comments(workload.generate("c4", n_docs=1000))
    got = rengine.run(batch)
    assert batch.n_logs == 3000 and (got.results["status"] == 0).all()
    ref, _ = replay_packed(batch, threads=8)
    raw, off = assert_render_matches(rengine, batch, ref)
    assert (np.diff(off.astype(np.int64)) >= 2).all()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["c2", "c3", "c5"])
def test_large_shapes_render_on_the_device(rengine, shape):
    from peritext_b200 import workload
    batch = dense_comments(workload.generate(shape, n_docs=1) if shape == "c5" else workload.generate(shape, n_docs=3, ops_per_doc=10000))
    got = rengine.run(batch)
    assert (got.results["status"] == 0).all()
    if shape == "c5":
        assert int(got.results["n_visible"][0]) > 100000 and int(got.results["n_spans"][0]) > 1000
    raw, off = assert_render_matches(rengine, batch, got)
    json.loads(raw[int(off[0]): int(off[1])])


@pytest.mark.gpu
def test_failed_logs_render_as_nothing():
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_admission import tampered_logs
    from tests.test_gpu_routes import FAULTS, route_base, with_fault, Log, batch_of, marks_over, typing_forward
    # merge faults of several types between clean logs
    logs = []
    for k, f in enumerate(f for f in FAULTS if f != "clean"):
        logs += [route_base("compact"), with_fault(route_base("direct" if k % 2 else "packed3"), f)]
    logs.append(route_base("direct"))
    batch = batch_of(logs)
    e = BatchEngine(0)
    try:
        got = e.run(batch)
        st = got.results["status"]
        assert (st[0::2] == 0).all() and (st[1::2] != 0).all() and len(set(st[1::2].tolist())) >= 3
        raw, off = assert_render_matches(e, batch, got)
        assert (np.diff(off.astype(np.int64))[1::2] == 0).all() and (np.diff(off.astype(np.int64))[0::2] > 2).all()
        # admission-rejected logs (status 6 / 7)
        cases = tampered_logs()
        ab = pack_logs([l for _, l in cases], with_changes=True)
        got = e.run(ab)
        st = got.results["status"]
        assert {6, 7} <= set(st.tolist()) and (st == 0).any()
        raw, off = assert_render_matches(e, ab, got)
        assert all(int(off[i + 1]) == int(off[i]) for i in range(ab.n_logs) if st[i] != 0)
        # PT_LOG_OVERFLOW logs: a comment pool too small for some logs, no re-merge
        lg = []
        for k in range(12):
            x = Log(2)
            ids = typing_forward(x, 80, [0, 1])
            marks_over(x, ids, 40 if k % 3 == 0 else 2, seed=k, types=(2,), n_ids=40)
            lg.append(x)
        ob = batch_of(lg)
    finally:
        e.close()
    e = BatchEngine(0, comment_pool_entries=300)
    try:
        e.upload(ob); e.merge()
        got = e.download()
        st = got.results["status"]
        assert (st == 4).any() and (st == 0).any(), st
        raw, off = assert_render_matches(e, ob, got)
        assert all(int(off[i + 1]) == int(off[i]) for i in range(ob.n_logs) if st[i] == 4)
    finally:
        e.close()


@pytest.mark.gpu
def test_render_edge_cases():
    import ctypes
    from peritext_b200.engine import BatchEngine, EngineError, _JsonPools, _JsonView, _json_pools
    logs = unicode_logs()
    batch = pack_logs(logs)
    e = BatchEngine(0, emit_patches=True)
    try:
        # before any merge, and after an upload without a merge
        with pytest.raises(EngineError, match="out of order"):
            e.render_json(batch)
        e.upload(batch)
        with pytest.raises(EngineError, match="out of order"):
            e.render_json(batch)
        merged, dp = e.run_with_patches(batch)
        recs, items, pst, need = e.download_patches()
        digests = merged.results["digest"].copy()
        # null arguments
        v = _JsonView()
        assert e._L.pt_batch_render_json(e._h, None, ctypes.byref(v)) == 1
        st = _JsonPools()
        assert e._L.pt_batch_render_json(e._h, ctypes.byref(st), None) == 1
        # a missing value, link or comment entry: PT_ERR_INVALID naming it, no view
        full = json_pools(batch)
        for k, what in ((0, "value"), (2, "link"), (4, "comment")):
            p = list(full)
            p[k + 1] = p[k + 1][:-1]
            p[k] = p[k][: int(p[k + 1][-1])]
            with pytest.raises(EngineError, match="names %s pool entry %d" % (what, len(p[k + 1]) - 1)):
                e.render_json(batch, tuple(p))
        # twice: identical bytes; the spans view, digests and the patch view are unchanged
        a = e.render_json(batch)
        b = e.render_json(batch)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        again = e.download()
        for i in range(batch.n_logs):
            assert again.canonical(i) == merged.canonical(i)
        assert (again.results["digest"] == digests).all()
        r2, i2, s2, n2 = e.download_patches()
        assert r2.tobytes() == recs.tobytes() and i2.tobytes() == items.tobytes() and s2.tobytes() == pst.tobytes() and n2 == need
    finally:
        e.close()
    # no pooled values, null value pointers; a batch of zero logs
    e = BatchEngine(0)
    try:
        plain = pack_logs(kat_logs()[:4])
        assert plain.values == []
        e.run(plain)
        p = json_pools(plain)
        assert len(p[0]) == 0
        ref, _ = replay_packed(plain)
        assert_render_matches(e, plain, ref, p)
        st, _keep = _json_pools(plain, p)
        st.values = st.values_off = None
        v = _JsonView()
        assert e._L.pt_batch_render_json(e._h, ctypes.byref(st), ctypes.byref(v)) == 0 and v.n_logs == plain.n_logs
        empty = batch.select([])
        e.run(empty)
        data, off = e.render_json(empty)
        assert len(data) == 0 and off.tolist() == [0]
    finally:
        e.close()
