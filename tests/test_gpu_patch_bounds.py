"""The device Patch stream (`patch_logs_kernel`, csrc/patch_kernel.cuh) at its capacity boundaries and on the reference's
arrival-dependent corners, against the oracle's `applyChange` return values.

The kernel runs one warp per log over 16-bit shared-memory tables.  Two guards decide whether a log is computed:
* the key space: `max_ctr * n_actors >= 0xFFFF` is not computed (the id table holds 16-bit keys);
* shared memory: the host sizes the launch (`Plan::patch_smem`, plan.cpp) by the largest HOST estimate among the
  logs that is <= 200 KB, rounded up to 1 KB; the kernel compares its own, smaller, footprint `need` with that size.
So a log too large to be computed alone may be computed next to a log that raised the launch's shared memory: its status
depends on the batch.  `expected_patch_status` restates both sides.  The `n >= 0xFFFF` / `m >= 0xFFFF` guards cannot be
reached: the 200 KB cap binds first (`test_the_16_bit_count_guards_are_unreachable`).

Every case is compared at two levels: the decoded `patch_stream`, patch for patch, and the raw arrays (`pt_patch_rec` per
ins/del record, the multiset of `pt_patch_item`s per log, the pool demand `n_items_needed`), which an encoder derives from
the oracle's patches and the batch's comment / link pools.  CPU parts: the exact-shape converter, the status mirror's sides
of every threshold, and the host closed forms (peritext_b200/patches.py) on the same logs."""
from collections import Counter

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import DESC_DT, PackedBatch, _root_text_list, canon, pack_logs, patch_stream
from tests.harness import fuzz_session, generateDocs
from tests.test_gpu_adversarial import SESSIONS
from tests.test_gpu_admission import tampered_logs
from tests.test_gpu_round2 import overlapping_comments_log
from tests.test_gpu_routes import (COMMENT, EM, FAULTS, HEAD, LINK, STRONG, Log, batch_of, kernel_config, lamport_forward, marks_over,
                                   typing_forward, with_fault)
from tests.test_patch_closed_form import closed_form_patches
from tests.test_semantic_corners import noncausal_logs, q4_logs

HOST_CAP = 200 * 1024
SPAN_STRONG, SPAN_EM, SPAN_LINK, SPAN_COMMENT = 1, 2, 4, 8
ATTR_NONE = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------------------------
# The status mirror: restates the host budget (plan.cpp make_plan) and the kernel's check (patch_kernel.cuh)
# ------------------------------------------------------------------------------------------------------------------
def _a16(x):
    return (x + 15) & ~15


def _shape(d):
    return int(d["n_insdel"]), int(d["n_mark"]), int(d["max_ctr"]) * (int(d["n_actors"]) or 1)


def host_need(d):
    """The host's per-log estimate: every per-element table sized by n_insdel, 256 bytes of slack."""
    n, m, KS = _shape(d)
    return _a16(2 * KS) + 3 * _a16(2 * n) + _a16(4 * n) + 6 * _a16(4 * m) + _a16(2 * m) + 256


def device_need(d, n_elems):
    """The kernel's footprint: T u16[KS] | PosOf u16[n] | TIns u16[N] | TDel u32[N] | six u32[m] | CList u16[m] | 64."""
    n, m, KS = _shape(d)
    N = int(n_elems)
    return _a16(2 * KS) + _a16(2 * n) + _a16(2 * N) + _a16(4 * N) + 6 * _a16(4 * m) + _a16(2 * m) + 64


def patch_smem(desc):
    """Dynamic shared memory of the patch launch: the largest host estimate <= 200 KB (at least 4 KB), rounded up to 1 KB."""
    need = max([4096] + [h for h in (host_need(d) for d in desc) if h <= HOST_CAP])
    return (need + 1023) & ~1023


def expected_patch_status(batch, n_elems, merge_status=None):
    """Per log: 0 computed on the device, 1 left to the host (merge failed, key space, or footprint over the launch's smem)."""
    smem = patch_smem(batch.desc)
    out = []
    for k, d in enumerate(batch.desc):
        n, m, KS = _shape(d)
        failed = merge_status is not None and int(merge_status[k]) != 0
        out.append(int(failed or KS >= 0xFFFF or n >= 0xFFFF or m >= 0xFFFF or device_need(d, n_elems[k]) > smem))
    return out


def insert_counts(batch):
    """n_elems of a log that merges: one element per insert record."""
    return [int(((batch.log_slice(i)[0]["payload"] >> 30) == 0).sum()) for i in range(batch.n_logs)]


# ------------------------------------------------------------------------------------------------------------------
# Exact-shape logs as JSON changes: one op per change, per-actor seq, startOp = ctr, the makeList by one of the log's actors
# ------------------------------------------------------------------------------------------------------------------
BOUND_NAMES = ["before", "after", "startOfText", "endOfText"]
MARK_NAMES = ["strong", "em", "comment", "link"]


def actor_name(a):
    return "a%02d" % a                      # JS string order == rank order


def log_changes(lg):
    """`lg` (test_gpu_routes.Log, a causal log) as the Change objects one replica applied, in arrival order."""
    used = {(r[0], r[2]) for r in lg.ins} | {(r[0], r[1]) for r in lg.mk}
    lc = next(c for c in range(1, lg.max_ctr + 2) if (c, 0) not in used)
    lid = "%d@%s" % (lc, actor_name(0))
    seq = Counter()

    def change(actor, ctr, op):
        seq[actor] += 1
        return {"actor": actor_name(actor), "seq": seq[actor], "deps": {}, "startOp": ctr,
                "ops": [{"opId": "%d@%s" % (ctr, actor_name(actor)), **op}]}
    out = [change(0, lc, {"action": "makeList", "obj": "_root", "key": "text"})]
    eid = lambda c, a: "%d@%s" % (c, actor_name(a))

    def ins_op(r):
        c, rc, a, ra, p = r
        if p >> 30 == 0:
            return change(a, c, {"action": "set", "obj": lid, "elemId": eid(rc, ra) if rc else "_head", "insert": True, "value": chr(p & 0xFFFF)})
        return change(a, c, {"action": "del", "obj": lid, "elemId": eid(rc, ra)})

    def mark_op(r):
        c, a, kind, bounds, sc, ec, sa, ea, attr, _arr, _ = r
        typ = MARK_NAMES[(kind >> 1) & 3]
        bnd = lambda t, bc, ba: {"type": BOUND_NAMES[t], "elemId": eid(bc, ba)} if t <= 1 else {"type": BOUND_NAMES[t]}
        op = {"action": "removeMark" if kind & 1 else "addMark", "obj": lid, "start": bnd(bounds & 3, sc, sa),
              "end": bnd(bounds >> 2, ec, ea), "markType": typ}
        if typ == "link" and not kind & 1:
            op["attrs"] = {"url": "%d.com" % attr}
        elif typ == "comment":
            op["attrs"] = {"id": "c%03d" % attr}
        return change(a, c, op)
    mi = 0
    for k, r in enumerate(lg.ins):
        while mi < lg.m and lg.mk[mi][9] <= k:
            out.append(mark_op(lg.mk[mi])); mi += 1
        out.append(ins_op(r))
    out += [mark_op(r) for r in lg.mk[mi:]]
    return out


def spread_log(R, C, n, m=0, seed=0):
    """R actors typing forward, counters spread so that max_ctr is exactly C after m trailing mark ops; n + m is kept large
    enough that the packer does not re-rank the counters."""
    lg = Log(R)
    prev, top = HEAD, C - m
    ids = []
    for k in range(n):
        prev = lg.insert(k % R, prev, chr(97 + k % 26), ctr=1 + (k * (top - 1)) // (n - 1))
        ids.append(prev)
    if m:
        marks_over(lg, ids, m, seed, width=6)
    assert lg.max_ctr == C
    return lg


def marks_then_edits(n_text, n_marks, types, seed, n_ids=8):
    """n_text characters, n_marks mark ops over them, then inserts inside the ranges and a few deletes (second deletes
    included): the insert patches inherit what the marks left."""
    lg = Log(2)
    ids = typing_forward(lg, n_text, [0, 1])
    marks_over(lg, ids, n_marks, seed, types=types, n_ids=n_ids, width=12)
    rng = np.random.default_rng(seed + 1)
    for k in range(24):
        lg.insert(k % 2, ids[int(rng.integers(0, n_text))], "+")
    for k in range(6):
        e = ids[int(rng.integers(0, n_text))]
        lg.delete(0, e); lg.delete(1, e)
    return lg


def cap_log(n, m=200):
    return lamport_forward(n, 1, m, seed=11, width=4)


def cap_sizes():
    """(largest n whose host estimate is <= 200 KB, smallest n whose estimate is above) for a one-actor log with 200 marks."""
    def need(n, m=200):
        d = np.zeros(1, DESC_DT)[0]
        d["n_insdel"], d["n_mark"], d["n_actors"], d["max_ctr"] = n, m, 1, n + m      # cap_log(n)'s descriptor
        return host_need(d)
    lo = max(n for n in range(16000, 17200) if need(n) <= HOST_CAP)
    hi = min(n for n in range(lo, 17200) if need(n) > HOST_CAP)
    return lo, hi


# ------------------------------------------------------------------------------------------------------------------
# The cases
# ------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, changes, shape=None, status=None):
        self.name, self.changes = name, changes
        self.shape = shape              # (n_insdel, n_mark, n_actors, max_ctr) the log must pack to
        self.status = status            # the patch status of the log alone in its batch


def exact_case(name, lg, status=0):
    return Case(name, log_changes(lg), (lg.n, lg.m, lg.R, lg.max_ctr), status)


def q4_extended_logs():
    """Q4 with four concurrent ops of one comment id (add, remove, re-add, remove again) and an insert inside the range, in
    several causal arrival orders: the "last-arrived covering op of the id decides" folds see two or more earlier ops."""
    docs, _, init = generateDocs(O, "abcdef", 3)
    cm = lambda d, act, a, b: docs[d].change([{"path": ["text"], "action": act, "startIndex": a, "endIndex": b, "markType": "comment",
                                              "attrs": {"id": "k"}}])["change"]
    a1 = cm(2, "addMark", 0, 5)
    r1 = cm(1, "removeMark", 0, 3)
    a2 = cm(0, "addMark", 1, 6)
    r2 = cm(2, "removeMark", 2, 4)
    ins = docs[0].change([{"path": ["text"], "action": "insert", "index": 3, "values": ["Z", "Y"]}])["change"]
    out = []
    for k, order in enumerate([(a1, r1, a2, r2, ins), (r1, a1, r2, a2, ins), (a2, ins, r1, a1, r2), (a1, r2, r1, a2, ins)]):
        out.append(("q4-four-ops-%d" % k, [init, *order]))
    return out


def quirk_logs():
    docs, _, init = generateDocs(O, "abcdefgh", 1)
    d = docs[0]
    chs = [init]
    do = lambda op: chs.append(d.change([{"path": ["text"], **op}])["change"])
    # Q3: removeMark of a comment id nobody added: `comment: []` on the range and on inserts inside it
    do(dict(action="removeMark", startIndex=1, endIndex=5, markType="comment", attrs={"id": "ghost"}))
    do(dict(action="insert", index=3, values=list("QR")))
    do(dict(action="addMark", startIndex=2, endIndex=4, markType="comment", attrs={"id": "real"}))
    do(dict(action="insert", index=3, values=["S"]))
    q3 = chs
    docs, _, init = generateDocs(O, "abcdefgh", 1)
    d = docs[0]
    chs = [init]
    # Q2: zero-width marks — start and end in one slot: the start wins and the mark never ends
    do(dict(action="addMark", startIndex=2, endIndex=2, markType="strong"))
    do(dict(action="addMark", startIndex=5, endIndex=5, markType="link", attrs={"url": "z.com"}))
    do(dict(action="insert", index=3, values=list("xy")))
    do(dict(action="addMark", startIndex=4, endIndex=4, markType="comment", attrs={"id": "zw"}))
    do(dict(action="insert", index=7, values=["w"]))
    do(dict(action="removeMark", startIndex=6, endIndex=6, markType="em"))
    do(dict(action="insert", index=9, values=["v"]))
    return [("q3-remove-only-comment", q3), ("q2-zero-width", chs)]


def corner_cases():
    out = [Case("noncausal-" + name, log) for name, log, _ in noncausal_logs()]
    out += [Case("q4-%d" % k, log) for k, (log, _) in enumerate(q4_logs())]
    out += [Case(name, log) for name, log in q4_extended_logs()]
    out += [Case(name, log) for name, log in quirk_logs()]
    return out


_ADV = None


def adversarial_cases():
    global _ADV
    if _ADV is None:
        _ADV = []
        for name, build in SESSIONS.items():
            _, logs = build()
            _ADV += [Case("%s-r%d" % (name, r), log) for r, log in enumerate(logs)]
    return _ADV


def trip_cases():
    out = []
    for m in (31, 32, 33, 64, 65):
        out.append(exact_case("marks-%d" % m, marks_then_edits(80, m, (STRONG, EM, LINK, COMMENT), seed=m)))
        out.append(exact_case("comments-%d" % m, marks_then_edits(80, m, (COMMENT,), seed=100 + m, n_ids=6)))
    for n in (32, 33):
        lg = lamport_forward(n, 1, 5, seed=n)
        out.append(exact_case("elements-%d" % n, lg))
    return out


def ks_cases():
    return [exact_case("keyspace-65520", spread_log(15, 4368, 2380, 20, seed=1), 0),
            exact_case("keyspace-65534", spread_log(14, 4681, 2380, 20, seed=2), 0),
            exact_case("keyspace-65535", spread_log(15, 4369, 2380, 20, seed=3), 1)]


_CAP = {}


def cap_cases():
    if not _CAP:
        lo, hi = cap_sizes()
        _CAP["below"] = exact_case("host-cap-below", cap_log(lo), 0)
        _CAP["above"] = exact_case("host-cap-above", cap_log(hi), 1)
    return _CAP["below"], _CAP["above"]


def small_cases():
    return corner_cases() + adversarial_cases() + trip_cases()


# ------------------------------------------------------------------------------------------------------------------
# The oracle's patches, per list op, and the raw arrays they imply
# ------------------------------------------------------------------------------------------------------------------
def list_ops(log):
    lid = _root_text_list(log)
    return [op for ch in log for op in ch["ops"] if op.get("obj") == lid]


_ORACLE = {}


def oracle_per_op(log):
    """(the patches the oracle's applyChange returned, one list per list op in arrival order, the oracle's final elements)."""
    hit = _ORACLE.get(id(log))
    if hit is None or hit[0] is not log:
        hit = _ORACLE[id(log)] = (log, _oracle_per_op(log))
    return hit[1]


def _oracle_per_op(log):
    lid = _root_text_list(log)
    fresh = O("observer")
    out, deleted = [], set()
    for ch in log:
        ps = [p for p in fresh.applyChange(ch) if p["action"] != "makeList"]
        ops = [op for op in ch["ops"] if op.get("obj") == lid]
        k = 0
        for j, op in enumerate(ops):
            a = op["action"]
            if a == "set":
                take = 1
            elif a == "del":
                take = 0 if op["elemId"] in deleted else 1
                deleted.add(op["elemId"])
            else:
                # consecutive mark ops of one type and action in one change would make the split ambiguous
                assert not (j + 1 < len(ops) and ops[j + 1]["action"] == a and ops[j + 1].get("markType") == op["markType"])
                take = 0
                while k + take < len(ps) and ps[k + take]["action"] == a and ps[k + take]["markType"] == op["markType"]:
                    take += 1
            out.append(ps[k:k + take]); k += take
        assert k == len(ps)
    return out, fresh.elements()


def encode(batch, i, ops, per_op, elements):
    """Expected (pt_patch_rec rows of log i, Counter of its pt_patch_items) from the oracle's patches."""
    link = {canon(a): k for k, a in enumerate(batch.link_attrs)}
    crank = {c["id"]: k for k, c in enumerate(batch.comment_ids)}
    pos = {e["elemId"]: k for k, e in enumerate(elements)}
    N = len(elements)
    t_ins = np.full(N, 1 << 40, np.int64)
    t_del = np.full(N, 1 << 40, np.int64)
    recs, items = [], Counter()
    ri = mi = 0
    for op, ps in zip(ops, per_op):
        if op["action"] in ("addMark", "removeMark"):
            for p in ps:
                items[(i, mi | 0x80000000, p["startIndex"], p["endIndex"])] += 1
            mi += 1
            continue
        if op["action"] == "set":
            (p,) = ps
            t_ins[pos[op["opId"]]] = ri
            mk = p["marks"]
            flags = (SPAN_STRONG if "strong" in mk else 0) | (SPAN_EM if "em" in mk else 0) | (SPAN_LINK if "link" in mk else 0)
            com = mk.get("comment")
            if com is not None:
                flags |= SPAN_COMMENT | (len(com) << 8)
                for c in com:
                    items[(i, ri, crank[c["id"]], 0)] += 1
            recs.append((p["index"] | 0x80000000, flags, link[canon(mk["link"])] if "link" in mk else ATTR_NONE, 0))
        else:
            x = pos[op["elemId"]]
            if ps:
                t_del[x] = min(t_del[x], ri)
                recs.append((ps[0]["index"] | 0x80000000, 0, ATTR_NONE, 0))
            else:
                # a second delete emits nothing; its record still carries the element's visible index at its arrival
                idx = int(((t_ins[:x] < ri) & ~(t_del[:x] < ri)).sum())
                recs.append((idx, 0, ATTR_NONE, 0))
        ri += 1
    return recs, items


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def exact_cases():
    return trip_cases() + ks_cases() + list(cap_cases())


def test_exact_shape_logs_pack_to_their_descriptors_and_replay_on_the_oracle():
    for c in exact_cases():
        b = pack_logs([c.changes])
        d = b.desc[0]
        assert (int(d["n_insdel"]), int(d["n_mark"]), int(d["n_actors"]), int(d["max_ctr"])) == c.shape, c.name
        assert b.log_counters[0] is None, c.name                 # no dense re-ranking: the counters are the Log's own
        if c.shape[0] < 3000:
            per_op, elements = oracle_per_op(c.changes)
            assert len(elements) == insert_counts(b)[0] and len(per_op) == c.shape[0] + c.shape[1], c.name


def test_status_mirror_puts_every_named_case_on_its_side():
    cases = exact_cases()
    for c in cases:
        b = pack_logs([c.changes])
        assert expected_patch_status(b, insert_counts(b)) == [c.status], c.name
    ks = {c.name: pack_logs([c.changes]).desc[0] for c in ks_cases()}
    assert [_shape(ks[k])[2] for k in ("keyspace-65520", "keyspace-65534", "keyspace-65535")] == [65520, 65534, 65535]
    below, above = cap_cases()
    db, da = pack_logs([below.changes]).desc[0], pack_logs([above.changes]).desc[0]
    assert host_need(db) <= HOST_CAP < host_need(da) and host_need(db) > HOST_CAP - 64
    # neighbour dependence: next to `below` the launch has 200 KB and `above` fits the kernel's own, smaller, footprint
    pair = pack_logs([above.changes, below.changes])
    assert patch_smem(pair.desc) == HOST_CAP
    assert expected_patch_status(pair, insert_counts(pair)) == [0, 0]
    assert device_need(da, int(da["n_insdel"])) < HOST_CAP < host_need(da)


def test_host_estimate_bounds_the_kernel_footprint():
    # the host estimate is never below the kernel's need (n_elems <= n_insdel), so a log that sets the launch's size fits it
    rng = np.random.default_rng(0)
    for _ in range(2000):
        d = np.zeros(1, DESC_DT)[0]
        d["n_insdel"], d["n_mark"] = rng.integers(0, 40000), rng.integers(0, 5000)
        d["n_actors"], d["max_ctr"] = rng.integers(1, 20), rng.integers(1, 5000)
        N = int(rng.integers(0, int(d["n_insdel"]) + 1))
        assert device_need(d, N) < host_need(d)


def test_the_16_bit_count_guards_are_unreachable():
    # every record and mark op has its own opId key, so KS >= n + m; n = 0xFFFF (or m = 0xFFFF) needs more than 200 KB of
    # the kernel's own tables even with no elements, so the launch size (<= 200 KB) rejects such a log first
    for n, m in ((0xFFFF, 0), (0, 0xFFFF)):
        d = np.zeros(1, DESC_DT)[0]
        d["n_insdel"], d["n_mark"], d["n_actors"], d["max_ctr"] = n, m, 1, n + m
        assert device_need(d, 0) > HOST_CAP


def test_log_changes_round_trips_the_records():
    lg = marks_then_edits(40, 9, (STRONG, EM, LINK, COMMENT), seed=3)
    b = pack_logs([log_changes(lg)])
    ref = batch_of([lg])
    assert b.insdel.tolist() == ref.insdel.tolist()
    for f in ("ctr", "actor", "kind", "bounds", "start_ctr", "end_ctr", "start_actor", "end_actor", "arrival"):
        assert b.marks[f].tolist() == ref.marks[f].tolist(), f


@pytest.mark.parametrize("group", ["corners", "adversarial", "trips"])
def test_host_closed_forms_equal_the_oracle(group):
    cases = {"corners": corner_cases, "adversarial": adversarial_cases, "trips": trip_cases}[group]()
    for c in cases:
        fresh = O("observer")
        got = []
        for ch in c.changes:
            got += [p for p in fresh.applyChange(ch) if p["action"] != "makeList"]
        assert closed_form_patches(c.changes, fresh.elements(), _root_text_list(c.changes)) == got, c.name


def test_q4_extended_orders_differ_in_the_reference():
    spans = set()
    for _, log in q4_extended_logs():
        fresh = O("r")
        for ch in log:
            fresh.applyChange(ch)
        spans.add(canon(fresh.getTextWithFormatting()))
    assert len(spans) > 1           # the arrival order decides: the fold over several ops of one id is observable


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pengine():
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0, emit_patches=True)
    yield e
    e.close()


def patch_pass(e, batch, retry=True):
    """One device pass: (merged, recs, items, status, n_items_needed), re-merged once with the reported pool demand."""
    merged = e.run(batch)
    recs, items, status, needed = e.download_patches()
    if retry and needed > len(items):
        e.set_patch_pool(needed + 16)
        e.merge(); merged = e.download()
        recs, items, status, needed = e.download_patches()
    return merged, recs, items, status, needed


def check_pass(batch, logs, out, names=None):
    """Status == the mirror; every computed log equal to the oracle, decoded and raw; demand == the oracle's item count."""
    from peritext_b200.packing import DevicePatches
    merged, recs, items, status, needed = out
    names = names or [str(i) for i in range(batch.n_logs)]
    want = expected_patch_status(batch, merged.results["n_elems"], merged.results["status"])
    assert status.tolist() == want, [(n, int(s), w) for n, s, w in zip(names, status, want) if s != w]
    assert len(items) == needed
    got_items = Counter(tuple(int(x) for x in it) for it in items.tolist())
    dp = DevicePatches(recs, items, status)
    total = 0
    for i, log in enumerate(logs):
        mine = Counter({k: v for k, v in got_items.items() if k[0] == i})
        if status[i]:
            assert not mine, names[i]                        # a log that is not computed leaves no items behind
            continue
        ops = list_ops(log)
        per_op, elements = oracle_per_op(log)
        assert patch_stream(batch, dp, i, ops) == per_op, names[i]
        want_recs, want_items = encode(batch, i, ops, per_op, elements)
        o, n = int(batch.desc[i]["insdel_off"]), int(batch.desc[i]["n_insdel"])
        assert [tuple(int(x) for x in r) for r in recs[o:o + n].tolist()] == want_recs, names[i]
        assert mine == want_items, names[i]
        total += sum(want_items.values())
    assert needed == total
    return want


def run_cases(e, cases):
    logs = [c.changes for c in cases]
    batch = pack_logs(logs)
    for c, d in zip(cases, batch.desc):
        if c.shape is not None:
            assert (int(d["n_insdel"]), int(d["n_mark"]), int(d["n_actors"]), int(d["max_ctr"])) == c.shape, c.name
    return batch, logs, patch_pass(e, batch)


_NAMED = {}


def named_cases():
    """The corner, adversarial, multi-trip and key-space cases by name."""
    if not _NAMED:
        for c in corner_cases() + adversarial_cases() + trip_cases() + ks_cases():
            assert c.name not in _NAMED
            _NAMED[c.name] = c
    return _NAMED


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(named_cases()))
def test_each_case_alone(pengine, name):
    c = named_cases()[name]
    batch, logs, out = run_cases(pengine, [c])
    st = check_pass(batch, logs, out, [c.name])
    if c.status is not None:
        assert st == [c.status], c.name


@pytest.mark.gpu
def test_all_cases_in_one_mixed_batch(pengine):
    cases = list(named_cases().values())
    batch, logs, out = run_cases(pengine, cases)
    st = check_pass(batch, logs, out, [c.name for c in cases])
    for c, s in zip(cases, st):
        if c.status is not None:
            assert s == c.status, c.name


@pytest.mark.gpu
def test_host_cap_and_neighbour_dependence(pengine):
    below, above = cap_cases()
    for cases, want in (([below], [0]), ([above], [1]), ([above, below], [0, 0]), ([below, above], [0, 0])):
        batch, logs, out = run_cases(pengine, cases)
        assert check_pass(batch, logs, out, [c.name for c in cases]) == want, [c.name for c in cases]


@pytest.mark.gpu
def test_grid_stride_over_more_logs_than_ctas(pengine):
    # a ~200 KB launch fits one CTA per SM: the grid is one CTA per SM and every CTA takes several logs
    below, _ = cap_cases()
    logs = []
    seed = 0
    while len(logs) < 300:
        _, ls, _ = fuzz_session(O, 3100 + seed, 30, remove_comments=bool(seed % 2))
        logs += ls; seed += 1
    logs.insert(len(logs) // 2, below.changes)
    batch = pack_logs(logs)
    assert patch_smem(batch.desc) == HOST_CAP and batch.n_logs > 300
    check_pass(batch, logs, patch_pass(pengine, batch))


def splice(parts):
    """One batch of the logs (batch, i) in `parts` order; pools of the first batch (the failed logs' pools do not matter)."""
    desc, ins, mk = [], [], []
    io = mo = 0
    for b, i in parts:
        a, m = b.log_slice(i)
        d = b.desc[i:i + 1].copy()
        d["insdel_off"] = io; d["mark_off"] = mo
        desc.append(d); ins.append(a); mk.append(m)
        io += len(a); mo += len(m)
    b0 = parts[0][0]
    return PackedBatch(np.concatenate(desc), np.concatenate(ins), np.concatenate(mk), b0.values, b0.link_attrs, b0.comment_ids,
                       b0.other_attrs)


@pytest.mark.gpu
def test_failed_logs_are_not_computed_and_leave_no_items(pengine):
    faults = [f for f in FAULTS if f != "clean"]
    clean_logs = []
    for s in range(len(faults) + 1):
        clean_logs.append(fuzz_session(O, 3500 + s, 40)[1][s % 3])
    clean = pack_logs(clean_logs)
    bad = batch_of([with_fault(lamport_forward(120, 2, 8, seed=k), f) for k, f in enumerate(faults)])
    parts, logs = [], []
    for k in range(len(faults)):
        parts += [(clean, k), (bad, k)]; logs += [clean_logs[k], None]
    parts.append((clean, len(faults))); logs.append(clean_logs[-1])
    batch = splice(parts)
    out = patch_pass(pengine, batch)
    merged = out[0]
    assert [int(s) for s in merged.results["status"][1::2]] == [FAULTS[f] for f in faults]
    st = check_pass(batch, logs, out)
    assert st[1::2] == [1] * len(faults) and set(st[0::2]) == {0}
    # admission-rejected logs (status 6 / 7 from the pre-pass) next to valid ones
    cases = tampered_logs()
    logs = [log for _, log in cases]
    batch = pack_logs(logs, with_changes=True)
    out = patch_pass(pengine, batch)
    rs = out[0].results["status"]
    assert {6, 7} <= set(rs.tolist()) and 0 in rs.tolist()
    st = check_pass(batch, [log if s == 0 else None for log, s in zip(logs, rs)], out, [n for n, _ in cases])
    assert st == [int(s != 0) for s in rs]


@pytest.mark.gpu
def test_merge_kernel_configuration_does_not_change_the_patch_arrays(pengine):
    from peritext_b200.engine import BatchEngine
    cases = corner_cases() + adversarial_cases()
    batch = pack_logs([c.changes for c in cases])
    outs = {}
    for cfg in ("default", "cta-only"):
        with kernel_config(cfg):
            e = BatchEngine(0, emit_patches=True)
            try:
                outs[cfg] = patch_pass(e, batch)
            finally:
                e.close()
    check_pass(batch, [c.changes for c in cases], outs["default"], [c.name for c in cases])
    (_, r0, i0, s0, n0), (_, r1, i1, s1, n1) = outs["default"], outs["cta-only"]
    assert r0.tobytes() == r1.tobytes() and s0.tobytes() == s1.tobytes() and n0 == n1
    assert np.sort(i0, order=("log", "tag", "a", "b")).tobytes() == np.sort(i1, order=("log", "tag", "a", "b")).tobytes()


def comments_and_inserts_log(n_inserts=100):
    """overlapping_comments_log(150, 400), then n_inserts inserts inside the comments (each inherits ~75 comment ids)."""
    chs, _ = overlapping_comments_log(150, 400)
    d = O("doc2")
    for ch in chs:
        d.applyChange(ch)
    chs = list(chs)
    for k in range(n_inserts):
        chs.append(d.change([{"path": ["text"], "action": "insert", "index": 150 + (k * 7) % 240, "values": ["i"]}])["change"])
    return chs


@pytest.mark.gpu
def test_item_pool_overflow_with_comment_pool_overflow_retries_to_exact():
    from peritext_b200.engine import BatchEngine
    big = comments_and_inserts_log()
    small, _ = overlapping_comments_log(3, 10)
    logs = [small, big, small, big, small]
    batch = pack_logs(logs)
    e = BatchEngine(0, emit_patches=True)
    try:
        # first pass, no retries: the logs whose comment lists overflow report PT_LOG_OVERFLOW and are not computed
        e.upload(batch); e.merge(); merged = e.download()
        recs, items, status, needed = e.download_patches()
        rs = merged.results["status"]
        assert (rs == 4).any() and set(rs.tolist()) <= {0, 4}
        assert all(int(status[i]) == 1 for i in np.nonzero(rs == 4)[0])
        assert status.tolist() == expected_patch_status(batch, merged.results["n_elems"], rs)
        assert not any(int(it["log"]) in set(np.nonzero(rs == 4)[0].tolist()) for it in items)
        # BatchEngine.run retries the comment pool, run_with_patches the item pool: afterwards every log is exact
        merged, dp = e.run_with_patches(batch)
        assert (merged.results["status"] == 0).all() and (dp.status == 0).all()
        _, _, _, needed = e.download_patches()
        first_cap = 4 * (len(batch.insdel) + len(batch.marks)) + 1024
        assert needed > first_cap                             # the item pool did overflow its default size
        check_pass(batch, logs, (merged, dp.recs, dp.items, dp.status, needed))
    finally:
        e.close()


@pytest.mark.gpu
def test_truncated_pass_and_engine_reuse_after_set_patch_pool():
    from peritext_b200.engine import BatchEngine
    big = comments_and_inserts_log(60)
    cases = corner_cases()
    logs = [c.changes for c in cases] + [big]
    batch = pack_logs(logs)
    e = BatchEngine(0, emit_patches=True)
    try:
        full = patch_pass(e, batch)
        check_pass(batch, logs, full)
        _, frecs, fitems, fstatus, fneeded = full
        # a pool smaller than the demand: the pool is full, the records are untouched, the items are a sub-multiset
        cap = fneeded // 3
        e.set_patch_pool(cap)
        e.merge(); e.download()
        recs, items, status, needed = e.download_patches()
        assert len(items) == cap and needed == fneeded
        assert recs.tobytes() == frecs.tobytes() and status.tobytes() == fstatus.tobytes()
        sub, whole = Counter(map(tuple, items.tolist())), Counter(map(tuple, fitems.tolist()))
        assert not (sub - whole)
        # the same engine, its pool size set by the calls above, on a batch that needs more: one retry, exact
        logs2 = logs + [comments_and_inserts_log(120), big]
        batch2 = pack_logs(logs2)
        out2 = patch_pass(e, batch2)
        assert out2[4] > fneeded
        check_pass(batch2, logs2, out2)
        # ... and a smaller batch afterwards
        out3 = patch_pass(e, batch)
        check_pass(batch, logs, out3)
    finally:
        e.close()


@pytest.mark.gpu
def test_facade_switches_to_the_host_closed_forms_at_the_key_space_guard():
    from peritext_b200 import Micromerge
    c = named_cases()["keyspace-65535"]
    chs = c.changes
    tail = 40                                               # the 20 mark ops and the last 20 inserts
    want, _ = oracle_per_op(chs)
    want = [p for ps in want for p in ps]
    doc = Micromerge("reader")
    head_patches = doc.applyChanges(chs[:-tail])
    assert int(doc._cache[2].status[0]) == 0                # below the guard: the device computed the patches
    tail_patches = doc.applyChanges(chs[-tail:])
    assert int(doc._cache[2].status[0]) == 1                # at KS = 65535 the device declines and the host derives them
    assert [p for p in head_patches if p["action"] != "makeList"] + tail_patches == want
