"""The warp kernel's half-width copy of the records, at each field's boundary.

The warp kernel (packed3 / compact / direct id tables) reads 8-byte ins/del and 16-byte mark records that the engine derives
from the resident records wherever they change (peritext_b200/csrc/upload_kernel.cuh): 16-bit counters and arrival, 8-bit
actors, 2-bit ins/del kind, 3-bit mark kind, 4-bit bounds.  A value too wide for its field saturates (counters and arrival at
0xFFFF, actors at 255); since every warp-routed log has max_ctr * n_actors < 0xFFFF, fewer than 0xFFFF records and at most
255 actors, a saturated value is rejected, or compared, exactly like the original.  Each log below is a clean log on one warp
route plus ONE record whose field holds the widest value that fits, the first that saturates, or a far-out value; every log
must merge as the oracle merges it, as the CTA-per-log kernel (PT_WARP=0) merges it, and with the status the full-width
records gave.  Then the same batch through every upload form, and after an append (the copy must follow the new records),
and a log with more actors than the copy's actor field holds (it must not take a warp route)."""
import numpy as np
import pytest

from oracle.packed import replay_packed
from tests.harness import environ
from tests.test_gpu_append import record_split
from tests.test_gpu_routes import BEFORE, HEAD, LINK, STRONG, Log, batch_of, expected_route, lamport_forward
from tests.test_gpu_wire_forms import compact_split, run_as

ROUTES = {"packed3": 3, "compact": 4, "direct": 2}      # route -> actors of its base log
CTR = {"fit": 0xFFFF, "sat": 0x10000, "far": 0xFFFFFFFF}  # 16-bit counter / arrival fields
ACT = {"fit": 255, "sat": 256, "far": 0xFFFF}             # 8-bit actor fields
OK, NOT_FOUND, BAD_OPID, BAD_KIND = 0, 1, 2, 3


def base(route):
    lg = Log(ROUTES[route])
    lg.ids = []
    prev = None
    for k in range(300):
        prev = lg.insert(k % lg.R, prev, chr(97 + k % 26))
        lg.ids.append(prev)
    lg.mark(0, STRONG, lg.ids[3], lg.ids[9])
    return lg


def raw_insdel(lg, ctr, ref, actor, kind=0):
    """An ins/del record with exactly these fields; max_ctr is not widened (the descriptor keeps the route)."""
    lg.ins.append((ctr, ref[0], actor, ref[1], (kind << 30) | (0 if kind else ord("!"))))


def raw_mark(lg, ctr=None, actor=0, kind=STRONG << 1, bounds=BEFORE, start=None, end=None, arrival=None):
    c = ctr if ctr is not None else lg.max_ctr + 1
    if ctr is None:
        lg.max_ctr = c
    s, e = start or lg.ids[20], end or lg.ids[40]
    lg.mk.append((c, actor, kind, bounds, s[0], e[0], s[1], e[1], 0xFFFFFFFF, len(lg.ins) if arrival is None else arrival, 0))


def next_ctr(lg):
    lg.max_ctr += 1
    return lg.max_ctr


# (name, builder, status of the full-width records, oracle-safe: every actor field < n_actors)
def variants():
    out = []
    for tag, v in CTR.items():
        out += [(f"ins-ctr-{tag}", lambda lg, v=v: raw_insdel(lg, v, lg.ids[-1], 0), BAD_OPID, True),
                (f"ins-ref-ctr-{tag}", lambda lg, v=v: raw_insdel(lg, next_ctr(lg), (v, 0), 0), NOT_FOUND, True),
                (f"del-ref-ctr-{tag}", lambda lg, v=v: raw_insdel(lg, next_ctr(lg), (v, 0), 0, kind=1), NOT_FOUND, True),
                (f"mark-ctr-{tag}", lambda lg, v=v: raw_mark(lg, ctr=v), BAD_OPID, True),
                (f"mark-start-ctr-{tag}", lambda lg, v=v: raw_mark(lg, start=(v, 0)), OK, True),
                (f"mark-end-ctr-{tag}", lambda lg, v=v: raw_mark(lg, end=(v, 0)), OK, True),
                (f"mark-arrival-{tag}", lambda lg, v=v: raw_mark(lg, arrival=v), OK, True)]
    for tag, v in ACT.items():
        out += [(f"ins-actor-{tag}", lambda lg, v=v: raw_insdel(lg, next_ctr(lg), lg.ids[-1], v), BAD_OPID, False),
                (f"ins-ref-actor-{tag}", lambda lg, v=v: raw_insdel(lg, next_ctr(lg), (lg.ids[-1][0], v), 0), NOT_FOUND, False),
                (f"del-ref-actor-{tag}", lambda lg, v=v: raw_insdel(lg, next_ctr(lg), (lg.ids[-1][0], v), 0, kind=1), NOT_FOUND, False),
                (f"mark-actor-{tag}", lambda lg, v=v: raw_mark(lg, actor=v), BAD_OPID, False),
                (f"mark-start-actor-{tag}", lambda lg, v=v: raw_mark(lg, start=(lg.ids[20][0], v)), OK, False),
                (f"mark-end-actor-{tag}", lambda lg, v=v: raw_mark(lg, end=(lg.ids[40][0], v)), OK, False)]
    out += [(f"ins-kind-{k}", lambda lg, k=k: raw_insdel(lg, next_ctr(lg), lg.ids[-1], 0, kind=k), BAD_KIND, True) for k in (2, 3)]
    # mark kind bits above 2 and bound bits above 3 are not read: these are a strong add and a link remove over [20, 40)
    out += [("mark-kind-high-bits", lambda lg: raw_mark(lg, kind=0xF8 | (STRONG << 1)), OK, True),
            ("mark-kind-high-bit-3", lambda lg: raw_mark(lg, kind=0x08 | (LINK << 1) | 1), OK, True),
            ("mark-bounds-high-bits", lambda lg: raw_mark(lg, bounds=0xF0 | BEFORE), OK, True),
            ("mark-bounds-far", lambda lg: raw_mark(lg, bounds=0xFF), OK, True)]
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


def canon(out):
    return [out.canonical(i) for i in range(len(out.results))]


def test_boundary_logs_take_their_warp_routes():
    rows, batch = boundary_cases()
    for (route, name, _, _), d in zip(rows, batch.desc):
        assert expected_route(d) == route, (route, name)


def cta_only(batch):
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0)
    try:
        with environ({"PT_WARP": "0"}):
            return canon(run_as(e, batch, "plain"))
    finally:
        e.close()


@pytest.mark.gpu
def test_boundary_records_merge_like_the_oracle_and_the_cta_kernel():
    from peritext_b200.engine import BatchEngine
    rows, batch = boundary_cases()
    e = BatchEngine(0)
    try:
        got = canon(run_as(e, batch, "plain"))
        assert e.stats()["logs_deferred_to_big_bin"] == 0
    finally:
        e.close()
    assert [g[0] for g in got] == [r[2] for r in rows]
    assert got == cta_only(batch)
    safe = [i for i, r in enumerate(rows) if r[3]]
    ref, _ = replay_packed(batch.select(safe), threads=4)
    for k, i in enumerate(safe):
        want = ref.canonical(k)
        if want[0] == rows[i][2]:
            assert got[i] == want, rows[i]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["runs", "compact", "adopt"])
def test_every_upload_form_derives_the_same_copy(form):
    """The copy is derived after each form's records are in place: the same outputs as the plain upload.  The compact form
    carries only 16-bit counters and 4-bit actors, so it gets the logs that fit them."""
    from peritext_b200.engine import BatchEngine
    rows, batch = boundary_cases()
    keep = list(range(len(rows)))
    if form == "compact":
        keep = compact_split(batch)[0]
        assert len(keep) == 9 * len(ROUTES)     # the counter fields at 0xFFFF, both ins/del kinds
        batch = batch.select(keep)
    e = BatchEngine(0)
    try:
        plain = canon(run_as(e, batch, "plain"))
        assert canon(run_as(e, batch, form)) == plain
    finally:
        e.close()
    assert [g[0] for g in plain] == [rows[i][2] for i in keep]


@pytest.mark.gpu
def test_merge_after_append_reads_the_new_copy():
    """A prefix of every boundary log is uploaded and merged, the rest appended: the re-merge must read a copy of the spliced
    records, and give what one upload of the whole logs gives (an append takes no mark arriving after its own records)."""
    from peritext_b200.engine import BatchEngine
    rows, batch = boundary_cases(lambda name: "arrival" not in name)
    pre, delta = record_split(batch, batch.desc["n_insdel"].astype(np.int64) // 2)
    e = BatchEngine(0)
    try:
        whole = canon(run_as(e, batch, "plain"))
        e.upload(pre)
        e.merge()
        before = canon(e.download())
        e.append(delta)
        e.merge()
        after = canon(e.download())
    finally:
        e.close()
    assert after == whole
    assert before != after


def many_actors_log(R):
    """R actors each insert one character at the head, concurrently (counter 1): the text order is the actor order, and the
    key space C * R = R is a direct-table shape.  Read through 8-bit actors, actors 255 and up would collide."""
    lg = Log(R)
    for a in range(R):
        lg.insert(a, HEAD, chr(0x100 + a), ctr=1)
    return lg


def test_many_actors_log_would_fit_the_direct_table():
    d = batch_of([many_actors_log(256)]).desc[0]
    assert expected_route(d) == "direct"       # the route before the actor-count rule


@pytest.mark.gpu
def test_more_than_255_actors_merge_on_the_cta_kernel():
    """255 actors stay on the warp route, 256 go to the CTA kernel (PT_WARP_FORCE skips only the footprint estimate)."""
    from peritext_b200.engine import BatchEngine
    batch = batch_of([many_actors_log(256), many_actors_log(255), lamport_forward(300, 3, 10)])
    ref, _ = replay_packed(batch, threads=4)
    e = BatchEngine(0)
    try:
        with environ({"PT_WARP_FORCE": "1"}):
            got = canon(run_as(e, batch, "plain"))
    finally:
        e.close()
    assert got == [ref.canonical(i) for i in range(batch.n_logs)]
    assert got == cta_only(batch)
