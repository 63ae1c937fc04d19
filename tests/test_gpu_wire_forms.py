"""Every way a batch reaches the device, against the oracle.

The engine takes a batch in five forms: plain records (`upload`), run-compressed records expanded on the device
(`upload_runs`), 8/16-byte compact records expanded on the device (`upload_compact`), records already in device memory
(`adopt_device`), and `PipelinedEngine`, which cuts the batch into chunks and sends each through one of the others.  One
corpus (KATs, fuzz sessions, quirks, every route case, the status matrix, generated workloads, empty and marks-only logs)
goes through every form, and every output array is compared with `oracle.packed.replay_packed`.  On top of that: the
compact form's field widths on the exact edge and one past it, the run expander's shapes, the outputs that read the
records again after the merge (Patch stream, element queries, both JSON renders), one handle cycling through the forms,
admission and the comment-pool retry through the pipeline, and a batch of more than 2^20 logs (the output scan's
chunked carry)."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200 import workload
from peritext_b200.packing import TOKEN_POOLED, PackedBatch, decode_spans, pack_logs
from tests.harness import fuzz_session, generateDocs, load_kats, run_concurrent
from tests.test_gpu_routes import (AFTER, END_OF_TEXT, FAULTS, LINK, ORACLE_DEFINES, STRONG, Log, all_cases, batch_of, chains, concurrent_blocks,
                                   joint_batch, route_base, status_matrix, typing_forward)

FORMS = ("plain", "runs", "compact", "adopt")


# ------------------------------------------------------------------------------------------------------------------
# Corpus
# ------------------------------------------------------------------------------------------------------------------
class Corpus:
    """A batch, which of its logs the oracle defines (the others are compared by status), and expected spans where known."""

    def __init__(self, batch, defined=None, spans=None, statuses=None):
        self.batch = batch
        self.defined = np.ones(batch.n_logs, bool) if defined is None else np.asarray(defined, bool)
        self.spans = spans or {}           # log -> (batch whose pools decode it, getTextWithFormatting)
        self.statuses = statuses           # expected status per log, where the oracle does not define the output


def kat_corpus():
    logs, spans = [], {}
    for kat in [k for k in load_kats() if k["kind"] == "concurrent"]:
        rec = []
        run_concurrent(O, kat, record=rec)
        for r in rec:
            spans[len(logs)] = kat["expectedResult"]
            logs.append(r)
    b = pack_logs(logs)
    return Corpus(b, spans={i: (b, s) for i, s in spans.items()})


def fuzz_corpus():
    logs, spans = [], []
    for seed, kw in [(11, {}), (12, {}), (2011, dict(replicas=2, max_chars=6, initial="The Peritext editor")),
                     (1011, dict(sync_prob=0.3, full_sync_at_end=False)), (3011, dict(zero_width_prob=0.3)), (3012, dict(zero_width_prob=0.3))]:
        docs, lg, _ = fuzz_session(O, seed, 120, **kw)
        logs += lg
        spans += [d.getTextWithFormatting() for d in docs]
    b = pack_logs(logs)
    return Corpus(b, spans={i: (b, s) for i, s in enumerate(spans)})


def quirk_corpus():
    """Multi-code-point values, emoji, an empty list, a fully deleted text, a removeMark-only comment, a zero-width mark."""
    logs = []
    docs, _, init = generateDocs(O, "abcdef", 1)
    logs.append([init, docs[0].change([{"path": ["text"], "action": "removeMark", "startIndex": 1, "endIndex": 3, "markType": "comment", "attrs": {"id": "x"}}])["change"]])
    e = O("doc1")
    logs.append([e.change([{"path": [], "action": "makeList", "key": "text"}])["change"]])
    docs, _, init = generateDocs(O, "abc", 1)
    c1 = docs[0].change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 3, "markType": "em"}])["change"]
    logs.append([init, c1, docs[0].change([{"path": ["text"], "action": "delete", "index": 0, "count": 3}])["change"]])
    docs, _, init = generateDocs(O, "ab", 1)
    logs.append([init, docs[0].change([{"path": ["text"], "action": "insert", "index": 1, "values": [" is great!", "é", "\U0001F600", "\U0010FFFF", "中"]}])["change"]])
    docs, _, init = generateDocs(O, "abcdef", 1)
    logs.append([init, docs[0].change([{"path": ["text"], "action": "addMark", "startIndex": 2, "endIndex": 2, "markType": "strong"}])["change"]])
    b = pack_logs(logs)
    return Corpus(b, spans={1: (b, []), 2: (b, [])})


def route_corpus():
    cases = all_cases()
    return Corpus(joint_batch(cases), spans={i: (c.batch, c.spans) for i, c in enumerate(cases) if c.spans is not None})


def status_corpus():
    rows, batch = status_matrix()
    return Corpus(batch, defined=[f in ORACLE_DEFINES for _, f in rows], statuses=[FAULTS[f] for _, f in rows])


def generated_corpus():
    parts = [workload.generate(cfg, n_docs=n, ops_per_doc=ops) for cfg, n, ops in [("c2", 4, 1500), ("c3", 6, 1500), ("c4", 40, 1000)]]
    return Corpus(concat([p for p in parts]))


def concat(batches):
    desc, ins, mk = [], [], []
    io = mo = 0
    for b in batches:
        d = b.desc.copy()
        d["insdel_off"] += io; d["mark_off"] += mo
        desc.append(d); ins.append(b.insdel); mk.append(b.marks)
        io += len(b.insdel); mo += len(b.marks)
    return PackedBatch(np.concatenate(desc), np.concatenate(ins), np.concatenate(mk))


def marks_only_log(n_marks):
    """No ins/del records: every mark spans startOfText .. endOfText."""
    lg = Log(2)
    for k in range(n_marks):
        c = lg._use(lg.ctr + 1)
        lg.mk.append((c, k % 2, (k % 2) | ((k % 4) << 1), 2 | (END_OF_TEXT << 2), 0, 0, 0, 0, (k % 3) if k % 4 in (2, 3) else 0xFFFFFFFF, 0, 0))
    return lg


def empty_corpus():
    """Empty logs and marks-only logs between ordinary ones."""
    plain = Log(1)
    ids = typing_forward(plain, 12)
    plain.mark(0, STRONG, ids[2], ids[7])
    return Corpus(batch_of([Log(1), marks_only_log(3), plain, Log(2), Log(1), marks_only_log(1), Log(1)]))


def only_empty_corpus():
    return Corpus(batch_of([Log(1), Log(3), Log(1)]))


def no_logs_corpus():
    return Corpus(batch_of([]))


def run_shapes_corpus():
    """What the run expander (one warp per log, one lane per run) has to get right: more than 32 runs (several trips of the
    warp), one insert run of more than 2048 records (one lane writes it alone), delete runs, runs interleaved between actors,
    pooled tokens inside runs, kind-2/3 records (each its own run; the log reports status 3), logs with zero runs between
    non-empty ones."""
    logs = []
    lg = Log(3); chains(lg, 70, 3, [0, 1, 2]); logs.append(lg)                       # 70 runs
    lg = Log(1); typing_forward(lg, 3000); logs.append(lg)                           # one 3000-record run
    logs.append(Log(2))
    lg = Log(2); ids = typing_forward(lg, 200, [0])
    for e in ids[20:150]:
        lg.delete(1, e)                                                              # one 130-record delete run
    for e in ids[160:170]:
        lg.delete(0, e)
    logs.append(lg)
    lg = Log(4); concurrent_blocks(lg, 400, [0, 1, 2, 3], 5); logs.append(lg)        # runs of 5, interleaved between actors
    logs.append(marks_only_log(2))
    lg = Log(2); ids = typing_forward(lg, 60, [1])
    for k in range(10, 40):                                                          # pooled tokens inside one run
        c, rc, a, ra, p = lg.ins[k]
        lg.ins[k] = (c, rc, a, ra, TOKEN_POOLED | (k % 3))
    logs.append(lg)
    lg = Log(2); ids = typing_forward(lg, 30, [0])
    lg.insert(0, ids[-1], kind=2)
    typing_forward(lg, 5, [1], start=ids[3])
    logs.append(lg)
    lg = Log(1); ids = typing_forward(lg, 8)
    lg.insert(0, ids[-1], kind=3); lg.insert(0, ids[-1], kind=3)
    logs.append(lg)
    batch = batch_of(logs)
    batch.values = ["ab", "\U0001F600\U0001F600", "xyz"]
    statuses = [0, 0, 0, 0, 0, 0, 0, 3, 3]
    return Corpus(batch, statuses=statuses)


CORPORA = {"kats": kat_corpus, "fuzz": fuzz_corpus, "quirks": quirk_corpus, "routes": route_corpus, "status": status_corpus,
           "generated": generated_corpus, "empty-and-marks-only": empty_corpus, "only-empty": only_empty_corpus,
           "no-logs": no_logs_corpus, "run-shapes": run_shapes_corpus}
_BUILT = {}


def corpus(name):
    if name not in _BUILT:
        c = CORPORA[name]()
        c.ref, _ = replay_packed(c.batch, threads=8)
        _BUILT[name] = c
    return _BUILT[name]


# ------------------------------------------------------------------------------------------------------------------
# The compact form's widths, restated
# ------------------------------------------------------------------------------------------------------------------
def compact_fits(batch, i):
    """Whether log i of `batch` is representable in the compact wire form (include/peritext_b200.h)."""
    d = batch.desc[i]
    if int(d["max_ctr"]) >= 65536 or int(d["n_insdel"]) >= 65536 or int(d["n_actors"]) > 16:
        return False
    ins, mk = batch.log_slice(i)
    tok = ins["payload"] & 0x3FFFFFFF
    if len(ins) and (((tok & (TOKEN_POOLED - 1)) >= 0x200000).any() or (ins["ctr"] >= 65536).any() or (ins["ref_ctr"] >= 65536).any()
                     or (ins["actor"] >= 16).any() or (ins["ref_actor"] >= 16).any()):
        return False
    if len(mk) and any((mk[f] >= 65536).any() for f in ("ctr", "start_ctr", "end_ctr", "arrival")):
        return False
    if len(mk) and (any((mk[f] >= 16).any() for f in ("actor", "start_actor", "end_actor")) or (mk["kind"] >= 8).any() or (mk["bounds"] >= 16).any()):
        return False
    return True


def compact_split(batch):
    """(indices of the representable logs, indices of the others); asserts that the converter refuses each of the others."""
    from peritext_b200.engine import EngineError
    from tests.test_compact_format import convert
    fits = [i for i in range(batch.n_logs) if compact_fits(batch, i)]
    unfit = [i for i in range(batch.n_logs) if i not in set(fits)]
    for i in unfit:
        with pytest.raises(EngineError):
            convert(batch.select([i]))
    return fits, unfit


# ------------------------------------------------------------------------------------------------------------------
# Running one form
# ------------------------------------------------------------------------------------------------------------------
def to_device(a):
    """A packed array as a CUDA tensor (at least 16 bytes, so that an empty array still has an address)."""
    import torch
    raw = np.ascontiguousarray(a).view(np.uint8) if a.nbytes else np.zeros(16, np.uint8)
    t = torch.from_numpy(raw.copy()).cuda()
    torch.cuda.synchronize()
    return t


def upload_as(e, batch, form):
    """Upload `batch` to handle `e` in wire form `form`, with its change table; returns what must stay alive until the
    merge has read it."""
    from peritext_b200.engine import compress_runs
    keep = None
    if form == "plain":
        e.upload(batch)
    elif form == "runs":
        keep = compress_runs(batch)
        e.upload_runs(keep)
    elif form == "compact":
        e.upload_compact(batch)
    elif form == "adopt":
        keep = (to_device(batch.insdel), to_device(batch.marks))
        e.adopt_device(batch.desc, keep[0].data_ptr(), len(batch.insdel), keep[1].data_ptr(), len(batch.marks))
    else:
        raise ValueError(form)
    if batch.changes is not None:
        e.upload_changes(batch.changes)
    return keep


def run_as(e, batch, form, merges=1):
    keep = upload_as(e, batch, form)
    for _ in range(merges):
        e.merge()
    out = e.download()
    del keep
    return out


def pipelined(batch, chunks, form):
    """PipelinedEngine over `batch` in `form` ('plain', 'runs' or 'compact'); one MergedBatch per chunk."""
    from peritext_b200.engine import PipelinedEngine, compress_runs
    p = PipelinedEngine(0, chunks=chunks)
    try:
        return p.run(compress_runs(batch) if form == "runs" else batch, copy=True, compact=form == "compact")
    finally:
        p.close()


def canon_all(parts):
    """Canonical forms of every log of a list of MergedBatch (or of one)."""
    parts = parts if isinstance(parts, list) else [parts]
    return [p.canonical(i) for p in parts for i in range(len(p.results))]


def check_against_oracle(c, got, logs, what):
    """got: canonical forms of the logs `logs` of corpus c."""
    assert len(got) == len(logs), what
    for k, i in enumerate(logs):
        want = c.ref.canonical(i)
        if c.defined[i] and (c.statuses is None or c.statuses[i] == want[0]):
            assert got[k] == want, (what, i)
        else:
            assert got[k][0] == c.statuses[i], (what, i, got[k][0])


# ------------------------------------------------------------------------------------------------------------------
# GPU: the corpus through every form
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CORPORA))
def test_every_form_matches_the_oracle(name):
    from peritext_b200.engine import BatchEngine
    c = corpus(name)
    batch = c.batch
    n = batch.n_logs
    every = list(range(n))
    if c.statuses is not None:
        assert [int(s) for s in c.ref.results["status"][c.defined]] == [s for s, d in zip(c.statuses, c.defined) if d], name
    fits, unfit = compact_split(batch)
    sub = batch.select(fits)
    e = BatchEngine(0)
    try:
        for form in ("plain", "runs", "adopt"):
            got = run_as(e, batch, form)
            check_against_oracle(c, canon_all(got), every, (name, form))
            for i, (pools, spans) in c.spans.items():
                assert decode_spans(pools, got, i) == spans, (name, form, i)
        got = run_as(e, sub, "compact")
        check_against_oracle(c, canon_all(got), fits, (name, "compact"))
    finally:
        e.close()
    for chunks in (1, 2, 3, 7):
        for form in ("plain", "runs", "compact"):
            parts = pipelined(sub if form == "compact" else batch, chunks, form)
            check_against_oracle(c, canon_all(parts), fits if form == "compact" else every, (name, "pipelined", chunks, form))


def test_which_logs_the_compact_form_refuses():
    """Only logs outside the compact widths are refused, and they are the ones expected."""
    refused = {name: compact_split(CORPORA[name]().batch)[1] for name in ("routes", "status", "kats", "run-shapes")}
    assert refused["kats"] == [] and refused["status"] == [] and refused["run-shapes"] == []
    names = [c.name for c in all_cases()]
    assert sorted(names[i] for i in refused["routes"]) == sorted(
        n for n, c in zip(names, all_cases()) if int(c.batch.desc[0]["n_actors"]) > 16 or int(c.batch.desc[0]["max_ctr"]) >= 65536)
    assert "30actors" in [names[i] for i in refused["routes"]]


# ------------------------------------------------------------------------------------------------------------------
# The compact widths on the exact edge and one past it
# ------------------------------------------------------------------------------------------------------------------
def edge_65535_log():
    """n_insdel = 65535, max_ctr = 65535: the last insert has counter 65535, and the last mark arrives after every record
    (arrival 65535), has opId counter 65535 and ends at the element with counter 65535."""
    lg = Log(2)
    ids = typing_forward(lg, 65534, [0])
    last = lg.insert(0, ids[-1], "z")
    assert last == (65535, 0) and lg.n == 65535
    lg.mk.append((101, 1, STRONG << 1, 0 | (0 << 2), ids[50][0], ids[90][0], 0, 0, 0xFFFFFFFF, 100, 0))
    lg.mk.append((65535, 1, LINK << 1, 0 | (AFTER << 2), ids[-20][0], 65535, 0, 0, 1, 65535, 0))
    lg.max_ctr = 65535
    return lg


def edge_16_actor_log():
    """n_actors = 16 with rank 15 in every actor field; pooled value 0x1FFFFF and code point U+10FFFF; a mark of kind 7
    (removeMark link) and one with bounds 15 (endOfText .. endOfText)."""
    lg = Log(16)
    ids = typing_forward(lg, 40, [15])
    c, rc, a, ra, p = lg.ins[5]
    lg.ins[5] = (c, rc, a, ra, TOKEN_POOLED | 0x1FFFFF)
    c, rc, a, ra, p = lg.ins[6]
    lg.ins[6] = (c, rc, a, ra, 0x10FFFF)
    for e in ids[30:35]:
        lg.delete(15, e)
    lg.mark(15, LINK, ids[2], ids[20], attr=0)
    lg.mark(15, LINK, ids[4], ids[10], add=False)                     # kind 7
    lg.mark(15, STRONG, None, None, sb=END_OF_TEXT, eb=END_OF_TEXT)   # bounds 15
    lg.mark(15, STRONG, ids[1], ids[8])
    return lg


@pytest.fixture(scope="module")
def edge():
    logs = [edge_65535_log(), edge_16_actor_log()]
    batch = batch_of(logs)
    d, m = batch.desc, batch.marks
    assert int(d[0]["n_insdel"]) == 65535 == int(d[0]["max_ctr"]) and int(m["arrival"].max()) == 65535 and int(m["ctr"].max()) == 65535
    assert int(d[1]["n_actors"]) == 16 and int(m["kind"].max()) == 7 and int(m["bounds"].max()) == 15
    ins1, mk1 = batch.log_slice(1)
    assert (ins1["actor"] == 15).all() and (ins1["ref_actor"][ins1["ref_ctr"] > 0] == 15).all() and (mk1["actor"] == 15).all()
    ref, _ = replay_packed(batch, threads=2)
    assert (ref.results["status"] == 0).all()
    return batch, ref


@pytest.mark.gpu
def test_compact_edge_merges_like_the_oracle(edge):
    from peritext_b200.engine import BatchEngine
    batch, ref = edge
    assert compact_split(batch) == ([0, 1], [])
    e = BatchEngine(0)
    try:
        for form in FORMS:
            got = run_as(e, batch, form)
            for i in range(batch.n_logs):
                assert got.canonical(i) == ref.canonical(i), (form, i)
    finally:
        e.close()


def test_one_past_the_compact_edge_is_refused():
    from peritext_b200.engine import EngineError
    from tests.test_compact_format import convert
    lg = edge_16_actor_log()
    lg.R = 17
    with pytest.raises(EngineError):
        convert(batch_of([lg]))
    lg = edge_16_actor_log()
    c, rc, a, ra, p = lg.ins[5]
    lg.ins[5] = (c, rc, a, ra, TOKEN_POOLED | 0x200000)
    with pytest.raises(EngineError, match="value token"):
        convert(batch_of([lg]))
    lg = Log(1)
    typing_forward(lg, 65536)
    with pytest.raises(EngineError):
        convert(batch_of([lg]))


# ------------------------------------------------------------------------------------------------------------------
# Records that do not fit the compact widths: the plain form reports the fault, the compact form refuses
# ------------------------------------------------------------------------------------------------------------------
def with_wide_fault(lg, fault):
    """A real record pushed out of the compact widths: a delete of a real counter + 65536, an insert by actor rank 16 + a real
    rank, a mark starting at a real counter + 65536."""
    last = (lg.ins[-1][0], lg.ins[-1][2])
    if fault == "delete-ref-ctr-past-width":
        lg.delete(0, (last[0] + 65536, last[1]))
    elif fault == "insert-actor-past-width":
        lg.insert(16 + 1, last)
    elif fault == "mark-start-past-width":
        lg.mark(0, STRONG, (last[0] - 5 + 65536, last[1]), last)
    return lg


WIDE_FAULTS = {"delete-ref-ctr-past-width": 1, "insert-actor-past-width": 2, "mark-start-past-width": 0}


def wide_fault_batch():
    rows = [(r, f) for r in ("packed3", "compact", "direct", "cta-u16") for f in WIDE_FAULTS]
    return rows, batch_of([with_wide_fault(route_base(r), f) for r, f in rows] + [route_base("direct")])


@pytest.mark.gpu
def test_out_of_width_records_plain_reports_compact_refuses():
    from peritext_b200.engine import BatchEngine, EngineError
    rows, batch = wide_fault_batch()
    ref, _ = replay_packed(batch, threads=4)
    fits, unfit = compact_split(batch)
    assert fits == [len(rows)] and unfit == list(range(len(rows)))
    e = BatchEngine(0)
    try:
        got = run_as(e, batch, "plain")
        for i, (r, f) in enumerate(rows):
            assert int(got.results[i]["status"]) == WIDE_FAULTS[f], (r, f)
            if f != "insert-actor-past-width":            # the oracle does not check actor ranks against n_actors
                assert got.canonical(i) == ref.canonical(i), (r, f)
        assert got.canonical(len(rows)) == ref.canonical(len(rows))
        for form in ("runs", "adopt"):
            assert canon_all(run_as(e, batch, form)) == canon_all(got), form
        with pytest.raises(EngineError, match="ref_ctr"):
            e.upload_compact(batch)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# A bad run table is refused on the host
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bad_run_tables_are_refused_before_any_copy():
    from peritext_b200.engine import BatchEngine, EngineError, PackedRuns, compress_runs
    batch = run_shapes_corpus().batch
    good = compress_runs(batch)

    def tampered(fn):
        r = PackedRuns(good.desc.copy(), good.run_off.copy(), good.tok_off.copy(), good.runs.copy(), good.tokens.copy(), good.marks, good.n_insdel_total)
        fn(r)
        return r

    def count(r, k, add):
        r.runs["kind_count"][k] = int(r.runs["kind_count"][k]) + add

    def grow_desc(r):
        r.desc["n_insdel"][1] += 1

    def to_delete_run(r):
        k = int(r.run_off[1])
        r.runs["kind_count"][k] = (1 << 30) | (int(r.runs["kind_count"][k]) & 0x3FFFFFFF)

    bad = {"count-plus-one": tampered(lambda r: count(r, 0, 1)),
           "count-zero": tampered(lambda r: count(r, 3, -(int(r.runs["kind_count"][3]) & 0x3FFFFFFF))),
           "long-run-overruns-the-buffer": tampered(lambda r: count(r, int(r.run_off[1]), 1 << 20)),
           "run-off-decreases": tampered(lambda r: r.run_off.__setitem__(2, r.run_off[1] - 1)),
           "tok-off-decreases": tampered(lambda r: r.tok_off.__setitem__(2, r.tok_off[1] - 1)),
           "tokens-short": tampered(lambda r: r.tok_off.__setitem__(slice(2, None), r.tok_off[2:] - 1)),
           "descriptor-grows": tampered(grow_desc),
           "kind-changed": tampered(to_delete_run)}
    e = BatchEngine(0)
    try:
        for name, r in bad.items():
            with pytest.raises(EngineError, match="run table|out of range"):
                e.upload_runs(r)
        e.upload_runs(good); e.merge()
        out = e.download()
        ref, _ = replay_packed(batch)
        assert canon_all(out) == canon_all(ref)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# Outputs that read the records after the merge
# ------------------------------------------------------------------------------------------------------------------
def patches_as(e, batch, form):
    keep = upload_as(e, batch, form)
    e.merge(); out = e.download()
    recs, items, status, needed = e.download_patches()
    if needed > len(items):
        e.set_patch_pool(needed + 16)
        e.merge(); out = e.download()
        recs, items, status, needed = e.download_patches()
    items = np.sort(items, order=["log", "tag", "a", "b"])
    pj = e.render_patches_json_list(batch)
    sj = e.render_json_list(batch)
    ins_q = [(i, int(r["ctr"]), int(r["actor"])) for i in range(batch.n_logs) for r in batch.log_slice(i)[0] if int(r["payload"]) >> 30 == 0]
    ins_q += [(i, 0xFFFF, 0) for i in range(batch.n_logs)]                  # an opId no log has
    found = e.find_elements([q[0] for q in ins_q], [q[1] for q in ins_q], [q[2] for q in ins_q]) if ins_q else None
    vis = [(i, k) for i in range(batch.n_logs) for k in range(int(out.results[i]["n_visible"]) + 1)]
    queried = [e.query_elements(np.array([v[0] for v in vis], np.uint32), np.array([v[1] for v in vis], np.uint32), flag) for flag in (False, True)]
    del keep
    return dict(canon=canon_all(out), recs=recs.tobytes(), items=items.tobytes(), status=status.tolist(), patches_json=pj, spans_json=sj,
                found=found.tobytes() if found is not None else b"", queried=[q.tobytes() for q in queried])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kats", "fuzz", "quirks", "empty-and-marks-only"])
def test_patch_stream_and_queries_are_the_same_in_every_form(name):
    from peritext_b200.engine import BatchEngine
    c = corpus(name)
    batch = c.batch
    e = BatchEngine(0, emit_patches=True)
    try:
        base = patches_as(e, batch, "plain")
        assert base["canon"] == canon_all(c.ref)
        assert batch.n_logs == 0 or any(s == 0 for s in base["status"])
        for form in ("runs", "compact", "adopt"):
            got = patches_as(e, batch, form)
            for k in base:
                assert got[k] == base[k], (name, form, k)
    finally:
        e.close()


@pytest.mark.gpu
def test_download_patches_on_a_fresh_handle_after_runs():
    """The Patch view is sized by the uploaded batch whichever form uploaded it, also on a handle that never saw a plain
    upload, and after a plain upload of a different size."""
    from peritext_b200.engine import BatchEngine, compress_runs
    small, big = corpus("quirks").batch, corpus("fuzz").batch
    want = {}
    e = BatchEngine(0, emit_patches=True)
    for b in (small, big):
        e.upload(b); e.merge(); e.download()
        want[id(b)] = e.download_patches()
    e.close()
    for first, second in ((None, small), (big, small), (small, big)):
        for form in ("runs", "adopt"):
            e = BatchEngine(0, emit_patches=True)
            try:
                if first is not None:
                    e.upload(first); e.merge(); e.download()
                keep = upload_as(e, second, form)
                e.merge(); e.download()
                recs, items, status, _ = e.download_patches()
                w = want[id(second)]
                assert len(recs) == len(second.insdel) and recs.tobytes() == w[0].tobytes(), form
                assert status.tolist() == w[2].tolist()
                del keep
            finally:
                e.close()


# ------------------------------------------------------------------------------------------------------------------
# One handle through every form
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_handle_cycles_through_the_forms():
    """plain -> compact -> runs -> adopt -> plain on one handle with batches that grow and shrink, three merges each on a
    user stream (the CUDA-graph replay): every step equals the oracle, nothing of an earlier batch leaks into a later one."""
    import torch
    from peritext_b200.engine import BatchEngine
    steps = [("plain", "quirks"), ("compact", "generated"), ("runs", "kats"), ("adopt", "routes"), ("plain", "empty-and-marks-only"),
             ("runs", "fuzz"), ("compact", "quirks"), ("adopt", "only-empty"), ("plain", "kats")]
    s = torch.cuda.Stream()
    e = BatchEngine(0, stream=s.cuda_stream, emit_sequence=True)
    try:
        for form, name in steps:
            c = corpus(name)
            batch = c.batch
            logs = list(range(batch.n_logs))
            if form == "compact":
                logs = compact_split(batch)[0]
                batch = batch.select(logs)
            got = run_as(e, batch, form, merges=3)
            s.synchronize()
            check_against_oracle(c, canon_all(got), logs, (form, name))
            assert len(got.seq) == int(batch.desc["n_insdel"].sum()), (form, name)
            for k, i in enumerate(logs):
                if c.ref.results[i]["status"] == 0:
                    assert len(got.sequence(k)) == int(got.results[k]["n_elems"])
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# Admission and the comment-pool retry through the pipeline
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "runs"])
def test_pipeline_admits_like_the_single_handle(form):
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_admission import oracle_admission, tampered_logs
    cases = tampered_logs()
    want = [oracle_admission(l) for _, l in cases]
    batch = pack_logs([l for _, l in cases], with_changes=True)
    e = BatchEngine(0)
    whole = e.run(batch)
    e.close()
    ref, _ = replay_packed(batch)
    for chunks in (2, 3, 7, 40):
        parts = pipelined(batch, chunks, form)
        got = canon_all(parts)
        for i, ((name, _), (st, idx)) in enumerate(zip(cases, want)):
            assert got[i] == whole.canonical(i), (chunks, name)
            if st:
                assert got[i][:4] == (st, idx, 0, 0), (chunks, name)
            else:
                assert got[i] == ref.canonical(i), (chunks, name)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "runs", "compact"])
def test_pipeline_retries_an_overflowing_comment_pool(form):
    from peritext_b200.engine import BatchEngine
    from tests.test_gpu_round2 import overlapping_comments_log
    big, big_spans = overlapping_comments_log(150, 400)
    small, small_spans = overlapping_comments_log(3, 10)
    batch = pack_logs([small, big, small, big, small])
    e = BatchEngine(0)
    whole = e.run(batch)
    e.close()
    assert (whole.results["status"] == 0).all()
    for chunks in (1, 2, 5):
        parts = pipelined(batch, chunks, form)
        assert canon_all(parts) == canon_all(whole), (form, chunks)
        k = 0
        for p in parts:
            for i in range(len(p.results)):
                assert decode_spans(batch, p, i) == (big_spans if k % 2 else small_spans), (form, chunks, k)
                k += 1


# ------------------------------------------------------------------------------------------------------------------
# More than 2^20 logs: the output scan's chunks of 1024 x 1024 logs and the carry between them
# ------------------------------------------------------------------------------------------------------------------
def template_logs():
    """8 tiny logs: 0-5 visible characters, some with a mark, one that fails (a reference to an element never inserted)."""
    logs = []
    e = O("doc1")
    logs.append([e.change([{"path": [], "action": "makeList", "key": "text"}])["change"]])
    for text, op in [("a", None), ("ab", {"action": "addMark", "startIndex": 0, "endIndex": 2, "markType": "strong"}),
                     ("abc", {"action": "delete", "index": 1, "count": 1}),
                     ("abcd", {"action": "addMark", "startIndex": 1, "endIndex": 3, "markType": "link", "attrs": {"url": "a.com"}}),
                     ("héllo", {"action": "addMark", "startIndex": 0, "endIndex": 5, "markType": "comment", "attrs": {"id": "c1"}}),
                     ("xy", {"action": "delete", "index": 0, "count": 2})]:
        docs, _, init = generateDocs(O, text, 1)
        chs = [init]
        if op is not None:
            chs.append(docs[0].change([{"path": ["text"], **op}])["change"])
        logs.append(chs)
    t = pack_logs(logs)
    bad = Log(2)
    typing_forward(bad, 3)
    bad.insert(1, (bad.ctr + 5, 0), ctr=bad.ctr + 6)
    fail = batch_of([bad])
    return concat_pools(t, fail)


def concat_pools(t, fail):
    b = concat([t, fail])
    b.values, b.link_attrs, b.comment_ids = t.values, t.link_attrs, t.comment_ids
    return b


def tile(t, n):
    """n logs: log j is template log j % t.n_logs."""
    k = t.n_logs
    reps = -(-n // k)
    ni, nm = len(t.insdel), len(t.marks)
    desc = np.tile(t.desc, reps)
    r = np.repeat(np.arange(reps, dtype=np.uint64), k)
    desc["insdel_off"] += r * np.uint64(ni); desc["mark_off"] += r * np.uint64(nm)
    b = PackedBatch(desc, np.tile(t.insdel, reps), np.tile(t.marks, reps), t.values, t.link_attrs, t.comment_ids)
    return b.slice_logs(0, n)


@pytest.mark.gpu
def test_more_than_2_pow_20_logs():
    from peritext_b200.engine import BatchEngine
    from peritext_b200.packing import json_pools
    from tests.test_gpu_render_json import render_spans_json
    t = template_logs()
    tref, _ = replay_packed(t)
    assert tref.results["status"].tolist() == [0] * 7 + [1]
    assert sorted(int(v) for v in tref.results["n_visible"][:7]) == [0, 0, 1, 2, 2, 4, 5]
    N = 2 ** 20 + 2 ** 10 + 3
    batch = tile(t, N)
    K = t.n_logs
    e = BatchEngine(0)
    try:
        e.upload(batch); e.merge()
        got = e.download()
        want = np.tile(tref.results, -(-N // K))[:N]
        assert got.results.tobytes() == want.tobytes()
        ok = want["status"] == 0
        for off, cnt in ((got.text_off, want["n_visible"]), (got.span_off, want["n_spans"])):
            c = np.zeros(N + 1, np.uint64)
            c[1:] = np.cumsum(np.where(ok, cnt, 0).astype(np.uint64))
            assert np.array_equal(off, c)
        edges = sorted({j for m in (1, 2, 511, 512, 1023, 1024, 1025) for j in (m * 1024 - 1, m * 1024, m * 1024 + 1)} |
                       {2 ** 20 - 2, 2 ** 20 - 1, 2 ** 20, 2 ** 20 + 1, N - 2, N - 1, 0, 1})
        for j in edges:
            assert got.canonical(j) == tref.canonical(j % K), j
        pools = json_pools(t)
        tj = [render_spans_json(t, tref, i, pools) for i in range(K)]
        data, off = e.render_json(batch)
        lens = np.array([len(b) for b in tj], np.uint64)
        c = np.zeros(N + 1, np.uint64)
        c[1:] = np.cumsum(np.tile(lens, -(-N // K))[:N])
        assert np.array_equal(off, c)
        raw = data.tobytes()
        for j in edges:
            assert raw[int(off[j]): int(off[j + 1])] == tj[j % K], j
    finally:
        e.close()
