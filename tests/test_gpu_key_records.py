"""The warp kernel's key records at every key and sentinel boundary.

The warp kernel (packed3 / compact / direct id tables) reads 4-byte ins/del and 8-byte mark records that the engine derives
from the resident records wherever they change (peritext_b200/csrc/upload_kernel.cuh).  Each id (ctr, actor) is stored as its
16-bit opId key (ctr - 1) * R + actor, which is at most 0xFFFD on a warp route; 0xFFFE and 0xFFFF are sentinels for the head,
an out-of-range id, a delete, a bad kind and an invalid bound.  A mark's arrival is stored as min(arrival, n) in 11 bits, so a
log with marks and more than 2047 ins/del records is deferred to the CTA kernel.  Link and comment attrs are read from the full
mark records for the ops that survive.  Every log below must merge as the oracle merges it and as the CTA-per-log kernel
(PT_WARP=0) merges it, through every upload form and after an append."""
import numpy as np
import pytest

from oracle.packed import replay_packed
from tests.harness import environ
from tests.test_gpu_append import record_split
from tests.test_gpu_merge_copy import ROUTES, base, canon, cta_only, next_ctr, raw_insdel, raw_mark
from tests.test_gpu_routes import AFTER, BEFORE, COMMENT, END_OF_TEXT, HEAD, LINK, STRONG, Log, batch_of, expected_route, typing_forward
from tests.test_gpu_wire_forms import compact_split, run_as

OK, NOT_FOUND, BAD_OPID, BAD_KIND = 0, 1, 2, 3
ATTR_NONE = 0xFFFFFFFF
TOP_ATTR = 4095                                         # batch_of interns TOP_ATTR + 1 links and comments: the largest valid id
WIDE = {"PT_WARP": "2048:2:113:1", "PT_WARP_FORCE": "1"}   # 113 KB per warp, host estimate skipped: the large key spaces fit


def past_c(lg):
    return lg.max_ctr + 1


def mark_then(lg, **kw):
    """A mark op with its own fresh counter; the other ids are chosen after it, so 'one past C' is past the mark's counter."""
    c = next_ctr(lg)
    raw_mark(lg, ctr=c, **{k: (v(lg) if callable(v) else v) for k, v in kw.items()})


def arrivals(lg, at):
    """Only two marks, both arriving at `at`: [ids[280], last) ends at the last element only if it arrived, and [last, last]
    (same slot, bounds before / after) covers the last character only if it arrived."""
    lg.mk.clear()
    last = lg.ids[-1]
    mark_then(lg, start=lg.ids[280], end=last, arrival=at(lg))
    mark_then(lg, start=last, end=last, bounds=BEFORE | (AFTER << 2), arrival=at(lg))


def attr_marks(lg, attr):
    lg.mark(0, LINK, lg.ids[20], lg.ids[40], attr=attr)
    lg.mark(1, COMMENT, lg.ids[30], lg.ids[60], attr=attr)
    lg.mark(0, COMMENT, lg.ids[50], lg.ids[70], attr=attr)
    lg.mark(1, COMMENT, lg.ids[65], lg.ids[90], add=False, attr=attr)


# (name, builder, status, oracle-safe: every actor field < n_actors and every attr interned)
def variants():
    out = [
        ("ins-ctr-0", lambda lg: raw_insdel(lg, 0, lg.ids[-1], 0), BAD_OPID, True),
        ("ins-ctr-past-C", lambda lg: raw_insdel(lg, past_c(lg), lg.ids[-1], 0), BAD_OPID, True),
        ("ins-actor-past-R", lambda lg: raw_insdel(lg, next_ctr(lg), lg.ids[-1], lg.R), BAD_OPID, False),
        ("ins-ref-ctr-past-C", lambda lg: raw_insdel(lg, next_ctr(lg), (past_c(lg), 0), 0), NOT_FOUND, True),
        ("ins-ref-actor-past-R", lambda lg: raw_insdel(lg, next_ctr(lg), (lg.ids[-1][0], lg.R), 0), NOT_FOUND, False),
        ("ins-head", lambda lg: lg.insert(0, HEAD, "!"), OK, True),
        ("del-head", lambda lg: raw_insdel(lg, next_ctr(lg), (0, 0), 0, kind=1), NOT_FOUND, True),
        ("del-ref-ctr-past-C", lambda lg: raw_insdel(lg, next_ctr(lg), (past_c(lg), 0), 0, kind=1), NOT_FOUND, True),
        ("del-ref-actor-past-R", lambda lg: raw_insdel(lg, next_ctr(lg), (lg.ids[-1][0], lg.R), 0, kind=1), NOT_FOUND, False),
        ("kind-2", lambda lg: raw_insdel(lg, next_ctr(lg), lg.ids[-1], 0, kind=2), BAD_KIND, True),
        ("kind-3-ctr-past-C", lambda lg: raw_insdel(lg, past_c(lg), lg.ids[-1], 0, kind=3), BAD_KIND, True),
        ("kind-2-actor-past-R", lambda lg: raw_insdel(lg, next_ctr(lg), lg.ids[-1], lg.R, kind=2), BAD_KIND, False),
        ("mark-ctr-past-C", lambda lg: raw_mark(lg, ctr=past_c(lg)), BAD_OPID, True),
        ("mark-actor-past-R", lambda lg: raw_mark(lg, actor=lg.R), BAD_OPID, False),
        ("mark-start-ctr-past-C", lambda lg: mark_then(lg, start=lambda lg: (past_c(lg), 0)), OK, True),
        ("mark-start-actor-past-R", lambda lg: mark_then(lg, start=(lg.ids[20][0], lg.R)), OK, False),
        ("mark-end-ctr-past-C", lambda lg: mark_then(lg, end=lambda lg: (past_c(lg), 0)), OK, True),
        ("mark-end-actor-past-R", lambda lg: mark_then(lg, end=(lg.ids[40][0], lg.R)), OK, False),
        ("mark-opid-of-an-insert", lambda lg: raw_mark(lg, ctr=lg.ids[5][0], actor=lg.ids[5][1]), BAD_OPID, True),
        ("same-slot-equal-bounds", lambda lg: mark_then(lg, start=lg.ids[30], end=lg.ids[30], bounds=AFTER | (AFTER << 2)), OK, True),
        ("same-slot-unequal-bounds", lambda lg: mark_then(lg, start=lg.ids[30], end=lg.ids[30], bounds=BEFORE | (AFTER << 2)), OK, True),
    ]
    for b in (2, END_OF_TEXT):
        out += [(f"mark-start-bound-{b}", lambda lg, b=b: mark_then(lg, bounds=b), OK, True),
                (f"mark-end-bound-{b}", lambda lg, b=b: mark_then(lg, bounds=b << 2), OK, True)]
    for tag, at in (("n-1", lambda lg: lg.n - 1), ("n", lambda lg: lg.n), ("n+1", lambda lg: lg.n + 1),
                    ("0xFFFF", lambda lg: 0xFFFF), ("0xFFFFFFFF", lambda lg: 0xFFFFFFFF)):
        out.append((f"arrival-{tag}", lambda lg, at=at: arrivals(lg, at), OK, True))
    for tag, a in (("0", 0), ("top", TOP_ATTR), ("none", ATTR_NONE)):
        out.append((f"attr-{tag}", lambda lg, a=a: attr_marks(lg, a), OK, a != ATTR_NONE))
    return out


def boundary_cases(keep=lambda name: True):
    rows, logs = [], []
    for route in ROUTES:
        for name, build, status, safe in variants():
            if not keep(name):
                continue
            lg = base(route)
            build(lg)
            rows.append((route, name, status, safe))
            logs.append(lg)
    return rows, batch_of(logs)


# ---- the largest keys: key spaces up to C * R = 0xFFFE (the WIDE configuration's slice holds their id tables) ------------
TOP = {"packed3": (3, 20000), "compact": (14, 4681), "direct": (2, 20000)}   # (R, C): packed3's top key is 3 * C - 1


def spread(R, C, n=300):
    """R actors typing forward with counters spread over [1, C - 1]: the top counter C is left for the records under test."""
    lg = Log(R)
    lg.ids, prev = [], HEAD
    for k in range(n):
        prev = lg.insert(k % R, prev, chr(97 + k % 26), ctr=1 + (k * (C - 2)) // (n - 1))
        lg.ids.append(prev)
    lg.max_ctr = C
    return lg


def top_variants(R, C):
    top = (C, R - 1)                                 # key C * R - 1, the largest of the log
    ins_top = lambda lg: lg.ids.append(lg.insert(R - 1, lg.ids[-1], "T", ctr=C))
    return [
        ("top-own-start-end", lambda lg: (ins_top(lg), raw_mark(lg, ctr=C, actor=R - 2, start=top, end=top, bounds=BEFORE | (AFTER << 2))), OK),
        ("top-ref", lambda lg: (ins_top(lg), raw_insdel(lg, C, top, R - 2, kind=1)), OK),
        ("top-mark-own", lambda lg: raw_mark(lg, ctr=C, actor=R - 1), OK),
        # the first ids past the key space: their unchecked keys would be C * R, a sentinel on compact
        ("top-ins-actor-past-R", lambda lg: raw_insdel(lg, C, lg.ids[-1], R), BAD_OPID),
        ("top-ins-ctr-past-C", lambda lg: raw_insdel(lg, C + 1, lg.ids[-1], 0), BAD_OPID),
        ("top-ref-past-C", lambda lg: raw_insdel(lg, C, (C + 1, 0), 0, kind=1), NOT_FOUND),
        ("top-start-past-C", lambda lg: raw_mark(lg, ctr=C, actor=0, start=(C + 1, 0)), OK),
        ("top-end-past-C", lambda lg: raw_mark(lg, ctr=C, actor=0, end=(C + 1, 0)), OK),
    ]


def top_cases():
    rows, logs = [], []
    for route, (R, C) in TOP.items():
        for name, build, status in top_variants(R, C):
            lg = spread(R, C)
            build(lg)
            rows.append((route, name, status, "actor-past-R" not in name))
            logs.append(lg)
    return rows, batch_of(logs)


def arrival_limit_log(n):
    """n ins/del records and one mark op whose start is the last of them: only an arrival of n reaches it."""
    lg = Log(2)
    ids = typing_forward(lg, n, [0, 1])
    lg.mark(0, STRONG, ids[-1], None, eb=END_OF_TEXT)
    return lg


# ---- helpers -------------------------------------------------------------------------------------------------------------
def merged(batch, env=None, form="plain"):
    """Canonical outputs and the number of logs deferred from the warp kernel."""
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0)
    try:
        with environ(env or {}):
            out = canon(run_as(e, batch, form))
            return out, e.stats()["logs_deferred_to_big_bin"]
    finally:
        e.close()


def check_oracle(rows, batch, got):
    safe = [i for i, r in enumerate(rows) if r[3]]
    ref, _ = replay_packed(batch.select(safe), threads=4)
    for k, i in enumerate(safe):
        want = ref.canonical(k)
        if want[0] == rows[i][2]:
            assert got[i] == want, rows[i]


# ---- tests ---------------------------------------------------------------------------------------------------------------
def test_key_record_logs_take_their_warp_routes():
    rows, batch = boundary_cases()
    for (route, name, _, _), d in zip(rows, batch.desc):
        assert expected_route(d) == route, (route, name)
    rows, batch = top_cases()
    for (route, name, _, _), d in zip(rows, batch.desc):
        assert expected_route(d, "wide") == route, (route, name)
        assert int(d["max_ctr"]) * int(d["n_actors"]) <= 0xFFFE
    assert [int(d["max_ctr"]) * int(d["n_actors"]) for d in batch.desc if int(d["n_actors"]) == 14][0] == 0xFFFE


@pytest.mark.gpu
def test_key_records_merge_like_the_oracle_and_the_cta_kernel():
    rows, batch = boundary_cases()
    got, deferred = merged(batch)
    assert deferred == 0
    assert [g[0] for g in got] == [r[2] for r in rows]
    assert got == cta_only(batch)
    check_oracle(rows, batch, got)


@pytest.mark.gpu
def test_largest_keys_merge_like_the_oracle_and_the_cta_kernel():
    rows, batch = top_cases()
    got, deferred = merged(batch, WIDE)
    assert deferred == 0
    assert [g[0] for g in got] == [r[2] for r in rows]
    assert got == cta_only(batch)
    check_oracle(rows, batch, got)


@pytest.mark.gpu
def test_arrival_field_limit():
    """2047 ins/del records and a mark stay on the warp kernel; 2048 (max_recs raised) are deferred, with the same results."""
    for n, env, want_deferred in ((2047, WIDE, 0), (2048, {"PT_WARP": "4096:2:113:1", "PT_WARP_FORCE": "1"}, 1)):
        batch = batch_of([arrival_limit_log(n)])
        if n == 2047:
            assert expected_route(batch.desc[0], "wide") == "direct"
        got, deferred = merged(batch, env)
        assert deferred == want_deferred, n
        ref, _ = replay_packed(batch, threads=1)
        assert got == [ref.canonical(0)] == cta_only(batch), n


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["runs", "compact", "adopt"])
def test_every_upload_form_derives_the_same_key_records(form):
    rows, batch = boundary_cases()
    keep = list(range(len(rows)))
    if form == "compact":
        keep = compact_split(batch)[0]
        assert keep
        batch = batch.select(keep)
    plain, _ = merged(batch)
    got, deferred = merged(batch, form=form)
    assert got == plain and deferred == 0
    assert [g[0] for g in plain] == [rows[i][2] for i in keep]


@pytest.mark.gpu
def test_merge_after_append_reads_the_new_key_records():
    """A prefix of every log is uploaded and merged, the rest appended (an append takes no mark arriving after its own
    records): the re-merge gives what one upload of the whole logs gives."""
    from peritext_b200.engine import BatchEngine
    rows, batch = boundary_cases(lambda name: not name.startswith("arrival-") or name in ("arrival-n-1", "arrival-n"))
    pre, delta = record_split(batch, batch.desc["n_insdel"].astype(np.int64) // 2)
    whole, _ = merged(batch)
    e = BatchEngine(0)
    try:
        e.upload(pre)
        e.merge()
        before = canon(e.download())
        e.append(delta)
        e.merge()
        after = canon(e.download())
        assert e.stats()["logs_deferred_to_big_bin"] == 0
    finally:
        e.close()
    assert after == whole
    assert before != after
