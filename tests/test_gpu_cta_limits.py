"""The CTA-per-log kernel at its limits: key space max_ctr * n_actors up to 2^31 - 1, 2^22 - 1 elements, 524 285 runs.

Only `merge_one_log` (peritext_b200/csrc/merge_kernel.cuh) reaches these limits; the warp and team kernels take key spaces below
0xFFFF.  Its id table T has one entry per key, so a key space near 2^31 needs a 4 GiB (u16 indices) or 8 GiB (u32) table in
the global spill slab, and the arena must count those bytes in 64 bits.  Its Euler-tour nodes hold a 20-bit successor and
22-bit element and visible weights, so a log merges with at most 2^22 - 1 elements and 2M + 4 < 2^20 (M <= 524 285 runs) and
reports PT_LOG_OVERFLOW past either.

The logs are numpy record arrays built whole.  The key-space logs are small, so the oracle replays them.  The element and run
limits need logs of millions of records, which the oracle cannot replay (its element lookup is linear); their results are
written in closed form instead, and the CPU tests check each closed form against the oracle at small sizes.  Every batch also
holds ordinary warp- and team-routed logs, which must merge as the oracle merges them.  One huge-key-space log per batch
(except the two-slot batch) and one engine at a time keep the device memory of the module below about 10 GB."""
import numpy as np
import pytest

from oracle.packed import replay_packed
from peritext_b200.packing import (ATTR_NONE, INSDEL_DT, MARK_DT, SPAN_COMMENT, SPAN_EM, SPAN_LINK, SPAN_STRONG, PackedBatch,
                                   pack_logs)
from tests.test_gpu_routes import AFTER, BEFORE, COMMENT, EM, END_OF_TEXT, LINK, STRONG, batch_of, expected_route, lamport_forward

START_OF_TEXT = 2
OK, ELEM_NOT_FOUND, BAD_OPID, OVERFLOW = 0, 1, 2, 4
INSERT, DELETE = 0, 1 << 30
MAX_ELEMS = (1 << 22) - 1          # N >= 2^22 overflows the 22-bit weights of an Euler-tour node
MAX_RUNS = (1 << 19) - 3           # 2M + 4 >= 2^20 overflows its 20-bit successor (2(M + 1) + 1 nodes plus the terminator)


class ArrayLog:
    """A packed log as whole record arrays (INSDEL_DT / MARK_DT), with the descriptor fields `batch_of` reads."""

    def __init__(self, ins, mk, R, max_ctr):
        self.ins, self.mk, self.R, self.max_ctr = ins, mk, R, int(max_ctr)

    @property
    def n(self):
        return len(self.ins)

    @property
    def m(self):
        return len(self.mk)


def batch(logs):
    """`batch_of` for a mix of ArrayLogs and tests.test_gpu_routes.Log logs (record arrays are concatenated, not iterated)."""
    return concat([batch_of_arrays(lg) if isinstance(lg, ArrayLog) else batch_of([lg]) for lg in logs])


def batch_of_arrays(lg):
    b = batch_of([])
    b.desc = np.zeros(1, b.desc.dtype)
    b.desc[0] = (0, 0, lg.n, lg.m, lg.R, lg.max_ctr)
    b.insdel, b.marks = lg.ins, lg.mk
    return b


def concat(batches):
    """One batch of every batch's logs, in order; pools are placeholders (the comparisons are of canonical forms)."""
    batches = [b for b in batches if b.n_logs]
    desc = np.concatenate([b.desc for b in batches])
    desc["insdel_off"] = np.concatenate([[0], np.cumsum(desc["n_insdel"].astype(np.uint64))[:-1]])
    desc["mark_off"] = np.concatenate([[0], np.cumsum(desc["n_mark"].astype(np.uint64))[:-1]])
    ins = np.concatenate([b.insdel for b in batches]).astype(INSDEL_DT)
    mk = np.concatenate([b.marks for b in batches]).astype(MARK_DT)
    n_attr = max([8] + [len(b.comment_ids) for b in batches] + [len(b.link_attrs) for b in batches])
    return PackedBatch(desc, ins, mk, link_attrs=[{"url": "%d.com" % k} for k in range(n_attr)],
                       comment_ids=[{"id": "c%03d" % k} for k in range(n_attr)])


def ordinary():
    """A log on the warp route and one on the team route."""
    return [lamport_forward(300, 2, 10), lamport_forward(3000, 2)]


def tokens(k):
    return (0x4E00 + np.asarray(k, np.int64) % 0x5000).astype(np.uint32)


def insdel(ctr, ref_ctr, actor, ref_actor, payload):
    a = np.zeros(len(ctr), INSDEL_DT)
    a["ctr"], a["ref_ctr"], a["actor"], a["ref_actor"], a["payload"] = ctr, ref_ctr, actor, ref_actor, payload
    return a


def mark(ctr, actor, typ, start, end, sb, eb, attr=ATTR_NONE, arrival=0, add=True):
    """One mark record; `start` / `end` are (ctr, actor), ignored for startOfText / endOfText."""
    r = np.zeros(1, MARK_DT)
    s, e = (start or (0, 0)), (end or (0, 0))
    r[0] = (ctr, actor, (0 if add else 1) | (typ << 1), sb | (eb << 2), s[0], e[0], s[1], e[1], attr, arrival, 0)
    return r


# ------------------------------------------------------------------------------------------------------------------
# Key-space logs: a few hundred records (u16 indices) or 32 000 (u32) with ids spread over a key space of up to 2^31 - 1
# ------------------------------------------------------------------------------------------------------------------
# (key space, actors, u32 indices), KS = R * C: either side of where a 32-bit byte count of the id table wraps (u16 indices
# above 0x7FFFFFF8, u32 above 0x3FFFFFFC), a wrapped count larger than shared memory (u32 at 2^30 + 2^24) and the largest key
# space the planner accepts
KEYSPACES = [
    (0x7FFFFFF8, 8, False),
    (0x7FFFFFF9, 2699, False),
    (0x7FFFFFFF, 1, False),
    (0x3FFFFFFC, 4, True),
    (0x3FFFFFFD, 23, True),
    ((1 << 30) + (1 << 24), 65, True),
    (0x7FFFFFFF, 1, True),
]
GROUP = 40                    # children of the first element besides its chain successor: a sibling group above kBigGroup (32)
VARIANTS = ("clean", "missing-reference", "duplicate-top")


def ks_name(ks, R, wide):
    return "%s-0x%08X-R%d" % ("u32" if wide else "u16", ks, R)


def keyspace_log(KS, R, wide, variant="clean"):
    """Element e0 at key 0 (a child of HEAD); a typing chain after it and GROUP more children of e0, their keys spread over
    [2, KS - 10]; the top key KS - 1 typed after the chain's end and then deleted; mark ops with opIds at key 1 and in
    KS - 8 .. KS - 2 whose boundaries are e0, the top element, a group child and endOfText.  Variants: an insert after an
    unused key (ELEM_NOT_FOUND), or a second insert with the top key (BAD_OPID)."""
    assert KS % R == 0
    C = KS // R
    n_chain = 32000 if wide else 300
    spread = np.unique(np.linspace(2, KS - 10, n_chain + GROUP).astype(np.int64))
    assert len(spread) == n_chain + GROUP
    grp = np.zeros(len(spread), bool)
    grp[np.linspace(0, len(spread) - 1, GROUP).astype(np.int64)] = True
    chain_keys, group_keys = spread[~grp], spread[grp]
    ctr_of = lambda k: np.asarray(k, np.int64) // R + 1
    act_of = lambda k: np.asarray(k, np.int64) % R
    ident = lambda k: (int(ctr_of(k)), int(act_of(k)))

    top = KS - 1
    keys = np.concatenate([[0], chain_keys, group_keys, [top]])
    refs = np.concatenate([[-1], [0], chain_keys[:-1], np.zeros(GROUP, np.int64), [chain_keys[-1]]])
    head = refs < 0
    ins = insdel(ctr_of(keys), np.where(head, 0, ctr_of(refs)), act_of(keys), np.where(head, 0, act_of(refs)),
                 INSERT | tokens(np.arange(len(keys))))
    extra = [insdel([ctr_of(KS - 3)], [ctr_of(top)], [act_of(KS - 3)], [act_of(top)], [DELETE])]     # delete the top element
    if variant == "missing-reference":
        unused = KS // 2 + 1
        while unused in set(keys.tolist()):
            unused += 1
        extra.append(insdel([ctr_of(KS - 9)], [ctr_of(unused)], [act_of(KS - 9)], [act_of(unused)], [INSERT | 0x41]))
    elif variant == "duplicate-top":
        extra.append(insdel([ctr_of(top)], [0], [act_of(top)], [0], [INSERT | 0x42]))
    elif variant != "clean":
        raise ValueError(variant)
    ins = np.concatenate([ins] + extra)
    n = len(ins)
    g = ident(group_keys[GROUP // 2])
    mk = np.concatenate([
        mark(*ident(KS - 2), STRONG, ident(0), ident(top), BEFORE, AFTER, arrival=n),
        mark(*ident(1), STRONG, ident(chain_keys[len(chain_keys) // 2]), None, BEFORE, END_OF_TEXT, arrival=n, add=False),
        mark(*ident(KS - 4), LINK, ident(0), ident(chain_keys[10]), AFTER, BEFORE, attr=1, arrival=n),
        mark(*ident(KS - 6), COMMENT, g, None, BEFORE, END_OF_TEXT, attr=0, arrival=n),
        mark(*ident(KS - 7), COMMENT, ident(0), g, BEFORE, AFTER, attr=2, arrival=n),
        mark(*ident(KS - 8), EM, None, ident(top), START_OF_TEXT, BEFORE, arrival=n),
    ])
    return ArrayLog(ins, mk, R, C)


def forty_thousand_actors():
    """One document of 40 000 one-character changes, each by its own actor with a Lamport counter, typed at the start: it
    packs without re-ranking as n_actors = max_ctr = 40 000 (KS = 1.6e9, u32 indices) and one sibling group of 40 000 runs."""
    n = 40000
    changes = [{"actor": "a%05d" % k, "seq": 1, "deps": {}, "startOp": k + 1,
                "ops": [{"action": "set", "obj": "L", "elemId": "_head", "insert": True, "value": chr(0x4E00 + k % 0x5000),
                         "opId": "%d@a%05d" % (k + 1, k)}]} for k in range(n)]
    return pack_logs([changes], list_ids=["L"])


TWO_SLOTS_KS = 9 << 27        # u32: a 4.5 GiB id table, so a second spill slot starts past 2^32 bytes


# ------------------------------------------------------------------------------------------------------------------
# Element and run limits, with their results in closed form
# ------------------------------------------------------------------------------------------------------------------
def forward_log(N, deletes=0, marks=False):
    """N characters typed forward by one actor (one run); then `deletes` deletes of elements spread over the text (first and
    last included); then, with `marks`, four mark ops: strong [first, last), em [last, end), link on the first element,
    comment from after the first element to endOfText."""
    k = np.arange(N, dtype=np.int64)
    ins = insdel(k + 1, k, 0, 0, INSERT | tokens(k))
    dele = np.unique(np.linspace(0, N - 1, deletes).astype(np.int64)) if deletes else np.zeros(0, np.int64)
    ctr = N + np.arange(1, len(dele) + 1)
    ins = np.concatenate([ins, insdel(ctr, dele + 1, 0, 0, np.full(len(dele), DELETE))])
    mk = np.zeros(0, MARK_DT)
    c = N + len(dele)
    if marks:
        n, first, last = len(ins), (1, 0), (N, 0)
        mk = np.concatenate([mark(c + 1, 0, STRONG, first, last, BEFORE, BEFORE, arrival=n),
                             mark(c + 2, 0, EM, last, None, BEFORE, END_OF_TEXT, arrival=n),
                             mark(c + 3, 0, LINK, first, first, BEFORE, AFTER, attr=0, arrival=n),
                             mark(c + 4, 0, COMMENT, first, None, AFTER, END_OF_TEXT, attr=1, arrival=n)])
    return ArrayLog(ins, mk, 1, c + len(mk))


def wide_log(M):
    """M characters each typed at the start of the text: one sibling group of M runs under HEAD."""
    k = np.arange(M, dtype=np.int64)
    return ArrayLog(insdel(k + 1, 0, 0, 0, INSERT | tokens(k)), np.zeros(0, MARK_DT), 1, M)


def deep_log(M):
    """M characters, each typed after the previous one with a delete of the first character between them, so no insert
    continues its predecessor's run: M runs of one element on a path of depth M."""
    ins = np.zeros(2 * M - 1, INSDEL_DT)
    k = np.arange(M, dtype=np.int64)
    ins["ctr"][0::2] = 2 * k + 1
    ins["ref_ctr"][2::2] = 2 * k[1:] - 1
    ins["payload"][0::2] = INSERT | tokens(k)
    ins["ctr"][1::2] = 2 * k[1:]
    ins["ref_ctr"][1::2] = 1
    ins["payload"][1::2] = DELETE
    return ArrayLog(ins, np.zeros(0, MARK_DT), 1, 2 * M - 1)


SHAPES = {
    "forward": lambda K: forward_log(K),
    "forward-marks": lambda K: forward_log(K, marks=True),
    "forward-deletes": lambda K: forward_log(K, deletes=64),
    "wide": wide_log,
    "deep": deep_log,
}


# pt_digest.h restated over uint64 arrays (wrap-around arithmetic)
def _mix64(z):
    z = z ^ (z >> np.uint64(30)); z = z * np.uint64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> np.uint64(27)); z = z * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _u64(x):
    return np.atleast_1d(np.asarray(x, np.uint64))


def _pair(hi, lo):
    return (_u64(hi) << np.uint64(32)) | _u64(lo)


def term_text(i, tok):
    return _mix64(_pair(i, tok) + np.uint64(0x9E3779B97F4A7C15))


def term_span(j, start, flags, link):
    return _mix64(_mix64(_pair(j, start) ^ np.uint64(0xA5A5A5A55A5A5A5A)) + _pair(flags, link))


def term_comment(j, k, cid):
    return _mix64(_mix64(_pair(j, k) ^ np.uint64(0x5BD1E9955BD1E995)) + _u64(cid))


def term_counts(nvis, nspans):
    return _mix64(_pair(nvis, nspans) ^ np.uint64(0xC3C3C3C33C3C3C3C))


def digest(terms):
    t = np.concatenate([_u64(x) for x in terms])
    hi = (t << np.uint64(23)) | (t >> np.uint64(41))
    return int(t.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(hi)) if len(hi) else 0


FLAG = {STRONG: SPAN_STRONG, EM: SPAN_EM, LINK: SPAN_LINK, COMMENT: SPAN_COMMENT}


def spans_of(nvis, intervals):
    """Spans of `nvis` visible characters under mark intervals (type, a, b, attr) over visible positions [a, b), none of
    which conflict: (start, flags, link_attr, comment ids)."""
    cuts = sorted({0} | {x for (_, a, b, _) in intervals for x in (a, b) if 0 < x < nvis}) if nvis else []
    out = []
    for s in cuts:
        on = [(t, at) for (t, a, b, at) in intervals if a <= s < b]
        comments = tuple(sorted(at for t, at in on if t == COMMENT))
        flags = 0
        for t, _ in on:
            flags |= FLAG[t]
        link = next((at for t, at in on if t == LINK), ATTR_NONE)
        sp = (s, flags | (len(comments) << 8), link, comments)
        if not out or out[-1][1:] != sp[1:]:
            out.append(sp)
    return out


class Closed:
    """A log's result in closed form: status, counts, visible tokens, spans (start, flags, link, comment ids), digest."""

    def __init__(self, status, n_elems=0, toks=None, spans=()):
        self.status, self.n_elems = status, n_elems
        self.toks = np.zeros(0, np.uint32) if toks is None else toks.astype(np.uint32)
        self.spans = list(spans)
        self.n_visible, self.n_spans = len(self.toks), len(self.spans)
        if status:
            self.digest = (0, 0)
            return
        terms = [term_text(np.arange(self.n_visible), self.toks), term_counts(self.n_visible, self.n_spans)]
        for j, (start, flags, link, comments) in enumerate(self.spans):
            terms.append(term_span(j, start, flags, link))
            terms += [term_comment(j, x, c) for x, c in enumerate(comments)]
        self.digest = digest(terms)

    def canonical(self):
        return (self.status, self.n_elems, self.n_visible, self.n_spans, tuple(int(t) for t in self.toks),
                tuple(self.spans), self.digest)


def closed_form(shape, K):
    """The result of SHAPES[shape](K), or the failed-log result past the element or run limit."""
    if shape.startswith("forward"):
        if K > MAX_ELEMS:
            return Closed(OVERFLOW)
        k = np.arange(K)
        vis = np.ones(K, bool)
        if shape == "forward-deletes":
            vis[np.unique(np.linspace(0, K - 1, 64).astype(np.int64))] = False
        toks = tokens(k[vis])
        intervals = [(STRONG, 0, K - 1, ATTR_NONE), (EM, K - 1, K, ATTR_NONE), (LINK, 0, 1, 0), (COMMENT, 1, K, 1)] \
            if shape == "forward-marks" else []
        return Closed(OK, K, toks, spans_of(len(toks), intervals))
    if K > MAX_RUNS:
        return Closed(OVERFLOW)
    k = np.arange(K)
    toks = tokens(k[::-1]) if shape == "wide" else tokens(k[1:] if K > 1 else k)
    return Closed(OK, K, toks, spans_of(len(toks), []))


def limit_cases():
    """(shape, size) of every element- and run-limit case: each limit and one past it."""
    return [("forward-marks", MAX_ELEMS), ("forward", MAX_ELEMS + 1), ("forward-deletes", MAX_ELEMS),
            ("wide", MAX_RUNS), ("wide", MAX_RUNS + 1), ("deep", MAX_RUNS), ("deep", MAX_RUNS + 1)]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the closed forms agree with the oracle, and every limit case takes the CTA kernel's largest bin
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(SHAPES))
def test_closed_form_matches_the_oracle(shape):
    for K in (2, 3, 33, 70, 1000):
        b = batch([SHAPES[shape](K)])
        ref, _ = replay_packed(b)
        assert closed_form(shape, K).canonical() == ref.canonical(0), (shape, K)


def test_closed_form_shapes_are_exact():
    lg = forward_log(MAX_ELEMS, deletes=64)
    assert (int((lg.ins["payload"] >> 30 == 0).sum()), lg.n >= 1 << 22) == (MAX_ELEMS, True)
    for M in (MAX_RUNS, MAX_RUNS + 1):
        for lg in (wide_log(M), deep_log(M)):
            ins = lg.ins
            isins = ins["payload"] >> 30 == 0
            prev_ins = np.concatenate([[False], isins[:-1]])
            prev_ctr = np.concatenate([[0], ins["ctr"][:-1]])
            chained = isins & (ins["ref_ctr"] != 0) & prev_ins & (ins["ref_ctr"] == prev_ctr)
            assert int((isins & ~chained).sum()) == M
    assert 2 * MAX_RUNS + 4 < 1 << 20 <= 2 * (MAX_RUNS + 1) + 4


def test_limit_cases_take_the_largest_cta_bin():
    for shape, K in limit_cases():
        assert expected_route(batch([SHAPES[shape](K)]).desc[0]) == "cta4-u32", (shape, K)
    for ks, R, wide in KEYSPACES:
        for v in VARIANTS:
            d = batch([keyspace_log(ks, R, wide, v)]).desc[0]
            assert int(d["max_ctr"]) * int(d["n_actors"]) == ks
            assert expected_route(d) == ("cta4-u32" if wide else "cta4-u16"), (ks, R, v)
    d = forty_thousand_actors().desc[0]
    assert (int(d["n_actors"]), int(d["max_ctr"]), expected_route(d)) == (40000, 40000, "cta4-u32")
    d = batch([keyspace_log(TWO_SLOTS_KS, 9, True)]).desc[0]
    assert expected_route(d) == "cta4-u32" and 4 * TWO_SLOTS_KS > 1 << 32


def test_keyspace_logs_reach_both_ends_of_the_key_space():
    for ks, R, wide in KEYSPACES:
        lg = keyspace_log(ks, R, wide)
        key = lambda c, a: (c.astype(np.int64) - 1) * R + a
        ins_keys = key(lg.ins["ctr"], lg.ins["actor"])[lg.ins["payload"] >> 30 == 0]
        mk_keys = key(lg.mk["ctr"], lg.mk["actor"])
        assert ins_keys.min() == 0 and ins_keys.max() == ks - 1 and len(set(ins_keys.tolist())) == len(ins_keys)
        assert mk_keys.min() == 1 and mk_keys.max() == ks - 2 and not set(mk_keys.tolist()) & set(ins_keys.tolist())
        assert int(lg.ins["ctr"].max()) == ks // R


@pytest.mark.parametrize("variant", VARIANTS)
def test_keyspace_logs_replay_on_the_oracle(variant):
    """A key-space log replays on the oracle with the status its variant is built for (the oracle accepts a duplicate)."""
    lg = keyspace_log(0x7FFFFFF8, 8, False, variant)
    ref, _ = replay_packed(batch([lg]))
    want = {"clean": OK, "missing-reference": ELEM_NOT_FOUND, "duplicate-top": OK}[variant]
    assert int(ref.results[0]["status"]) == want


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def run(b):
    """Merges `b` on a fresh engine and closes it before returning: (output, stats, merge calls)."""
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0)
    try:
        calls = []
        merge = e.merge
        e.merge = lambda: (calls.append(1), merge())[1]
        out = e.run(b)
        return out, e.stats(), len(calls)
    finally:
        e.close()


def check_against_oracle(b, got, skip=()):
    ref, _ = replay_packed(b, threads=8)
    for i in range(b.n_logs):
        if i not in skip:
            assert got.canonical(i) == ref.canonical(i), i


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("ks,R,wide", KEYSPACES, ids=[ks_name(*k) for k in KEYSPACES])
def test_keyspace_limit_matches_the_oracle(ks, R, wide, variant):
    b = batch(ordinary() + [keyspace_log(ks, R, wide, variant)])
    got, st, _ = run(b)
    assert st["logs_spill_path"] == 1
    if variant == "duplicate-top":          # the oracle does not check duplicate opIds
        assert int(got.results[2]["status"]) == BAD_OPID
        check_against_oracle(b, got, skip={2})
    else:
        assert int(got.results[2]["status"]) == (OK if variant == "clean" else ELEM_NOT_FOUND)
        check_against_oracle(b, got)


@pytest.mark.gpu
def test_forty_thousand_actor_document_matches_the_oracle():
    b = concat([batch(ordinary()), forty_thousand_actors()])
    got, st, _ = run(b)
    assert st["logs_spill_path"] == 1 and int(got.results[2]["status"]) == OK
    check_against_oracle(b, got)


@pytest.mark.gpu
def test_two_spill_slots_past_four_gib():
    b = batch(ordinary() + [keyspace_log(TWO_SLOTS_KS, 9, True), keyspace_log(TWO_SLOTS_KS, 9, True, "missing-reference")])
    got, st, _ = run(b)
    assert st["logs_spill_path"] == 2
    assert [int(s) for s in got.results["status"]] == [OK, OK, OK, ELEM_NOT_FOUND]
    check_against_oracle(b, got)


@pytest.mark.gpu
def test_keyspace_of_2_pow_31_is_refused_and_the_engine_still_merges():
    from peritext_b200.engine import BatchEngine, EngineError
    lg = ArrayLog(insdel([1, 1 << 30], [0, 1], [0, 1], [0, 0], INSERT | tokens([0, 1])), np.zeros(0, MARK_DT), 2, 1 << 30)
    e = BatchEngine(0)
    try:
        with pytest.raises(EngineError) as err:
            e.upload(batch(ordinary() + [lg]))
        assert err.value.status == 1                          # PT_ERR_INVALID
        b = batch(ordinary() + [keyspace_log(0x7FFFFFFF, 1, False)])
        got = e.run(b)
    finally:
        e.close()
    check_against_oracle(b, got)


def check_closed(got, i, want):
    r = got.results[i]
    assert (int(r["status"]), int(r["n_elems"]), int(r["n_visible"]), int(r["n_spans"])) == \
        (want.status, want.n_elems, want.n_visible, want.n_spans), i
    assert (int(r["digest"][0]), int(r["digest"][1])) == want.digest, i
    assert np.array_equal(got.tokens(i), want.toks), i
    sp = got.span_records(i)
    assert [(int(s["start"]), int(s["flags"]), int(s["link_attr"])) for s in sp] == [s[:3] for s in want.spans], i
    for s, w in zip(sp, want.spans):
        o = int(s["comment_off"])
        assert tuple(int(x) for x in got.comment_pool[o: o + (int(s["flags"]) >> 8)]) == w[3], i


@pytest.mark.gpu
@pytest.mark.parametrize("limit", ["elements", "runs"])
def test_element_and_run_limits_match_the_closed_forms(limit):
    cases = [c for c in limit_cases() if c[0].startswith("forward") == (limit == "elements")]
    small = ordinary()
    b = batch(small + [SHAPES[s](K) for s, K in cases])
    got, st, merges = run(b)
    assert merges == 1                    # an overflow at a limit is not a full comment pool: no re-merge
    assert st["logs_spill_path"] == len(cases)
    check_against_oracle(batch(small), got)
    for i, (s, K) in enumerate(cases):
        check_closed(got, len(small) + i, closed_form(s, K))
