"""The warp kernel's mark pass at the edges of its duplicate test and of its boundary lookups.

The mark pass (phase G, peritext_b200/csrc/warp_kernel.cuh) takes 32 mark records per trip.  Its duplicate-opId test is one
atomicOr on a key-space bitmap that the record pass seeded with every insert key, so a mark whose opId is an insert's is a
duplicate even when that insert arrives after the mark, and a repeated mark opId is one whether the two marks share a trip or
not.  Both boundary lookups run for every mark: a start or end that names no insert reads the element table's entry n, and
the hit rules (the element must have arrived before the mark, quirk Q2 for a start and end in one slot) are applied after the
loads.  The link and comment survivors of a trip send their attr lines to L2 inside the pass.  Each log below is a clean log
on one warp route plus the marks under test; every log must merge as the oracle merges it and as the CTA-per-log kernel
(PT_WARP=0) merges it."""
import pytest

from tests.test_gpu_key_records import check_oracle, merged
from tests.test_gpu_merge_copy import ROUTES, base, cta_only, raw_insdel, raw_mark
from tests.test_gpu_routes import AFTER, BEFORE, COMMENT, EM, LINK, STRONG, batch_of, expected_route

OK, BAD_OPID = 0, 2


def missing(lg, t):
    """An id inside the key space that names no insert: element t's counter with the next actor (actors type in turn)."""
    c, a = lg.ids[t]
    return (c, (a + 1) % lg.R)


def fillers(lg, count, first=0):
    """`count` valid mark ops with fresh opIds over short ranges, arriving after every ins/del record."""
    for k in range(count):
        s = (first + 7 * k) % 250
        lg.mark(k % lg.R, (STRONG, EM)[k % 2], lg.ids[s], lg.ids[s + 1 + k % 40])


def later_insert_twin(lg):
    """A mark op whose opId is that of an insert arriving after it."""
    c = lg.max_ctr + 1
    raw_mark(lg, ctr=c, actor=0, start=lg.ids[20], end=lg.ids[40])
    raw_insdel(lg, c, lg.ids[-1], 0)
    lg.max_ctr = c


def repeated_mark(lg, a, b, count):
    """`count` marks; mark b repeats mark a's opId."""
    fillers(lg, count)
    r = list(lg.mk[1 + b])
    r[0], r[1] = lg.mk[1 + a][0], lg.mk[1 + a][1]
    lg.mk[1 + b] = tuple(r)


def early(lg, arrival, **kw):
    """A mark arriving at `arrival`, placed first: a log's marks are in arrival order."""
    raw_mark(lg, arrival=arrival, **kw)
    lg.mk.insert(0, lg.mk.pop())


def at_arrival(lg, which, t, arrival):
    """A mark whose start (or end) is element t (record t), arriving at `arrival`."""
    if which == "start":
        early(lg, arrival, start=lg.ids[t], end=lg.ids[t + 30])
    else:
        early(lg, arrival, start=lg.ids[t - 30], end=lg.ids[t])


def attr_survivors(lg, count):
    """A link and a comment survivor in the first trip of marks and in the last one (a partial trip)."""
    lg.mark(0, LINK, lg.ids[2], lg.ids[50], attr=1)
    lg.mark(1, COMMENT, lg.ids[5], lg.ids[60], attr=2)
    fillers(lg, count - 5, first=3)
    lg.mark(2 % lg.R, LINK, lg.ids[100], lg.ids[180], attr=3)
    lg.mark(0, COMMENT, lg.ids[120], lg.ids[200], attr=4)


# (name, builder, status, compared with the oracle: the oracle does not check duplicate opIds)
def variants():
    out = [
        ("opid-of-a-later-insert", later_insert_twin, BAD_OPID, False),
        ("repeated-opid-one-trip", lambda lg: repeated_mark(lg, 3, 17, 40), BAD_OPID, False),
        ("repeated-opid-across-trips", lambda lg: repeated_mark(lg, 3, 45, 60), BAD_OPID, False),
        ("repeated-opid-first-and-last", lambda lg: repeated_mark(lg, 0, 69, 70), BAD_OPID, False),
        ("start-misses", lambda lg: raw_mark(lg, start=missing(lg, 20), end=lg.ids[40]), OK, True),
        ("end-misses", lambda lg: raw_mark(lg, start=lg.ids[20], end=missing(lg, 40)), OK, True),
        ("both-miss", lambda lg: raw_mark(lg, start=missing(lg, 20), end=missing(lg, 40)), OK, True),
        ("end-misses-many-trips", lambda lg: (fillers(lg, 50), raw_mark(lg, start=lg.ids[60], end=missing(lg, 70))), OK, True),
        ("same-slot-missing-equal-bounds",
         lambda lg: raw_mark(lg, start=missing(lg, 30), end=missing(lg, 30), bounds=BEFORE | (BEFORE << 2)), OK, True),
        ("same-slot-missing-unequal-bounds",
         lambda lg: raw_mark(lg, start=missing(lg, 30), end=missing(lg, 30), bounds=BEFORE | (AFTER << 2)), OK, True),
        # start and end in one slot that has not arrived (its record == the arrival), then one that has
        ("same-slot-late-equal-bounds",
         lambda lg: early(lg, 150, start=lg.ids[150], end=lg.ids[150], bounds=AFTER | (AFTER << 2)), OK, True),
        ("same-slot-late-unequal-bounds",
         lambda lg: early(lg, 150, start=lg.ids[150], end=lg.ids[150], bounds=BEFORE | (AFTER << 2)), OK, True),
        ("same-slot-arrived-unequal-bounds",
         lambda lg: early(lg, 151, start=lg.ids[150], end=lg.ids[150], bounds=BEFORE | (AFTER << 2)), OK, True),
        ("attr-survivors-first-and-last-trip", lambda lg: attr_survivors(lg, 70), OK, True),
        ("attr-survivors-one-trip", lambda lg: attr_survivors(lg, 20), OK, True),
    ]
    for which in ("start", "end"):
        for tag, d in (("arrival", 0), ("arrival-1", 1)):
            out.append((f"{which}-at-{tag}", lambda lg, which=which, d=d: at_arrival(lg, which, 150, 150 + d), OK, True))
    return out


def cases():
    rows, logs = [], []
    for route in ROUTES:
        for name, build, status, safe in variants():
            lg = base(route)
            build(lg)
            rows.append((route, name, status, safe))
            logs.append(lg)
    return rows, batch_of(logs)


def test_mark_pass_logs_take_their_warp_routes():
    rows, batch = cases()
    for (route, name, _, _), d in zip(rows, batch.desc):
        assert expected_route(d) == route, (route, name)


@pytest.mark.gpu
def test_mark_pass_merges_like_the_oracle_and_the_cta_kernel():
    rows, batch = cases()
    got, deferred = merged(batch)
    assert deferred == 0
    assert [g[0] for g in got] == [r[2] for r in rows]
    assert got == cta_only(batch)
    check_oracle(rows, batch, got)
