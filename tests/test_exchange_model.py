"""The host specification of pt_batch_exchange: ``packing.exchange_maps`` + ``packing.apply_exchange`` against the reference's
sync (getMissingChanges then applyChanges, reference test/merge.ts:4-38) as the harness's fuzz sessions run it.

A session is recorded through a Micromerge subclass that notes whose clock getMissingChanges read (target first, then source)
and what each replica applied; the replay makes every local change with ``pack_append`` and every two-way sync with one
``apply_exchange`` of {a->b, b->a} on a batch holding one log per replica.  After every sync the batch must equal
``pack_logs`` of the replicas' logs, and the delivered indices must name the changes in the order the harness applied them.
tests/test_gpu_exchange.py runs the same replays on the device."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import (ACTOR_UNMAPPED, CTR_UNUSED, EXCHANGE_BAD_TABLE, EXCHANGE_OK, EXCHANGE_STUCK, EXCHANGE_UNMAPPED,
                                   ChangeTable, ExchangeMaps, PackedBatch, apply_append, apply_exchange, exchange_maps, pack_append, pack_logs)
from tests.harness import fuzz_session, generateDocs
from tests.test_append_packing import assert_same_batch, sparse_peer

SESSIONS = [(5, dict(replicas=3)), (6, dict(replicas=5)), (7, dict(replicas=3, sync_prob=0.3)), (8, dict(replicas=5, sync_prob=0.3))]


# ------------------------------------------------------------------------------------------------------------------
# Recording a session
# ------------------------------------------------------------------------------------------------------------------
def record_session(seed, n_steps, **kw):
    """(replica actor ids, the initial change, events, the session's final logs) of ``fuzz_session(seed, n_steps, **kw)``.
    Events: ("change", replica, change) and ["sync", src, dst, [the changes dst applied, in order]], one per direction."""
    ids = [f"doc{i + 1}" for i in range(kw.get("replicas", 3))]       # generateDocs' names
    events, asked = [], []

    class Spy(O):
        @property
        def clock(self):
            asked.append(self.actorId)
            if len(asked) == 2:                       # getMissingChanges reads target.clock, then source.clock
                events.append(["sync", ids.index(asked[1]), ids.index(asked[0]), []])
                asked.clear()
            return super().clock

        def change(self, ops):
            r = super().change(ops)
            events.append(("change", ids.index(self.actorId), r["change"]))
            return r

        def applyChange(self, change):
            out = super().applyChange(change)         # a change that is not admitted raises and is not recorded
            if events[-1][0] == "sync" and events[-1][2] == ids.index(self.actorId):
                events[-1][3].append(change)
            return out

    _, logs, _ = fuzz_session(Spy, seed, n_steps, **kw)
    assert events[0][0] == "change" and events[0][1] == 0             # generateDocs' initial change
    return ids, events[0][2], events[1:], logs


def final_logs_match(ids, init, events, logs):
    mine = [[init] for _ in ids]
    for e in events:
        if e[0] == "change":
            mine[e[1]].append(e[2])
        else:
            mine[e[2]] += e[3]
    assert mine == logs


# ------------------------------------------------------------------------------------------------------------------
# Replay
# ------------------------------------------------------------------------------------------------------------------
def two_way(events):
    """The events with the two directions of each sync joined: ("change", r, change) | ("sync", [(src, dst, applied), ...])."""
    out = []
    for e in events:
        if e[0] == "sync" and out and out[-1][0] == "sync" and len(out[-1][1]) == 1 and out[-1][1][0][:2] == (e[2], e[1]):
            out[-1][1].append((e[1], e[2], e[3]))
        elif e[0] == "sync":
            out.append(("sync", [(e[1], e[2], e[3])]))
        else:
            out.append(e)
    return out


def key(change):
    return (change["actor"], change["seq"])


def replay(ids, init, events, on_change, on_sync):
    """Drives `on_change(cur, mlogs, r, change) -> cur` and `on_sync(cur, mlogs, pairs) -> (cur, status, delivered)` through the
    session, checking what each sync delivered; returns the final (batch, logs)."""
    mlogs = [[init] for _ in ids]
    cur = pack_logs(mlogs, with_changes=True)
    for e in two_way(events):
        if e[0] == "change":
            cur = on_change(cur, mlogs, e[1], e[2])
            mlogs[e[1]].append(e[2])
            continue
        pairs = [(s, d) for s, d, _ in e[1]]
        cur, status, delivered = on_sync(cur, mlogs, pairs)
        assert (np.asarray(status) == EXCHANGE_OK).all()
        got = [[mlogs[s][int(k)] for k in delivered[p]] for p, (s, d) in enumerate(pairs)]
        for p, (s, d, applied) in enumerate(e[1]):
            assert [key(c) for c in got[p]] == [key(c) for c in applied], (s, d)
        for p, (s, d) in enumerate(pairs):
            mlogs[d] += got[p]
        assert_same_batch(cur, pack_logs(mlogs, with_changes=True))
    return cur, mlogs


def model_change(cur, mlogs, r, change):
    delta, remap = pack_append(cur, [[change] if i == r else [] for i in range(cur.n_logs)], with_changes=True)
    return apply_append(cur, delta, remap)


def model_sync(cur, mlogs, pairs):
    maps, pre = exchange_maps(cur, pairs)
    if pre is not None:
        cur = apply_append(cur, *pre)
    new, status, delivered, _ = apply_exchange(cur, pairs, maps)
    return new, status, delivered


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions_replayed_through_the_model(seed, kw):
    ids, init, events, logs = record_session(seed, 60, **kw)
    final_logs_match(ids, init, events, logs)
    syncs = [e for e in two_way(events) if e[0] == "sync"]
    assert any(len(applied) > 1 for e in syncs for _, _, applied in e[1])          # several changes queued up
    cur, mlogs = replay(ids, init, events, model_change, model_sync)
    assert mlogs == logs


# ------------------------------------------------------------------------------------------------------------------
# Hand-made cases
# ------------------------------------------------------------------------------------------------------------------
def typed(doc, text, index=0):
    return doc.change([{"path": ["text"], "action": "insert", "index": index, "values": list(text)}])["change"]


def three_replicas():
    """x, y, z share the initial text.  z types; y applies that and marks over z's characters; x applies both in order."""
    docs, _, init = generateDocs(O, "abc", 3)
    x, y, z = docs
    cz = typed(z, "ZZ", 1)
    y.applyChange(cz)
    cy = y.change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 4, "markType": "strong"}])["change"]
    return init, cz, cy


def sync_once(logs, pairs):
    cur = pack_logs(logs, with_changes=True)
    maps, pre = exchange_maps(cur, pairs)
    if pre is not None:
        cur = apply_append(cur, *pre)
    return (cur, maps) + apply_exchange(cur, pairs, maps)


def test_missing_order_that_is_not_causal_needs_a_second_pass():
    """src saw y's actor before z's, and y's second change depends on z's: for a dst that holds y's first change,
    getMissingChanges lists y's second change before z's.  The queue front is requeued once and z's change is delivered first."""
    docs, _, init = generateDocs(O, "abc", 3)
    x, y, z = docs
    y1 = typed(y, "y", 0)
    cz = typed(z, "ZZ", 1)
    y.applyChange(cz)
    y2 = y.change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 4, "markType": "strong"}])["change"]
    assert y2["deps"].get("doc3") == 1
    logs = [[init, y1, cz, y2], [init, y1]]               # dst has y's first change: the missing set is [y2, cz] in that order
    cur, maps, new, status, delivered, ddesc = sync_once(logs, [(0, 1)])
    assert status.tolist() == [EXCHANGE_OK] and delivered == [[2, 3]]
    assert_same_batch(new, pack_logs([logs[0], [init, y1, cz, y2]], with_changes=True))
    assert int(ddesc[1]["n_insdel"]) == 2 and int(ddesc[1]["n_mark"]) == 1 and int(ddesc[0]["n_insdel"]) == 0
    # without the first change in dst the order is causal already: y1, then y2 requeued behind cz
    logs = [[init, y1, cz, y2], [init]]
    _, _, new, status, delivered, _ = sync_once(logs, [(0, 1)])
    assert delivered == [[1, 2, 3]]
    assert_same_batch(new, pack_logs([logs[0], logs[0]], with_changes=True))


def test_dst_lacks_an_actor_unmapped_unless_pre_appended():
    init, cz, cy = three_replicas()
    logs = [[init, cz, cy], [init]]
    cur = pack_logs(logs, with_changes=True)
    assert cur.log_actors[1] == ["doc1"]
    maps, pre = exchange_maps(cur, [(0, 1)])
    assert pre is not None and pre[0].log_actors[1] == ["doc1", "doc2", "doc3"]
    # on the batch as it is, dst has no rank for doc2 / doc3
    bare = ExchangeMaps.of([np.array([0, ACTOR_UNMAPPED, ACTOR_UNMAPPED], np.uint16)])
    new, status, delivered, ddesc = apply_exchange(cur, [(0, 1)], bare)
    assert status.tolist() == [EXCHANGE_UNMAPPED] and delivered == [[]]
    assert_same_batch(new, cur)
    new, status, delivered, _ = apply_exchange(apply_append(cur, *pre), [(0, 1)], maps)
    assert status.tolist() == [EXCHANGE_OK] and delivered == [[1, 2]]
    assert_same_batch(new, pack_logs([logs[0], logs[0]], with_changes=True))


def test_stuck_pair_and_seq_gap_deliver_nothing_and_leave_the_other_pair_alone():
    init, cz, cy = three_replicas()
    logs = [[init, cy], [init], [init, cz], [init]]       # log 0 holds y's change without z's, which it depends on
    cur = pack_logs(logs, with_changes=True)
    maps, pre = exchange_maps(cur, [(0, 1), (2, 3)])
    cur = apply_append(cur, *pre)
    new, status, delivered, _ = apply_exchange(cur, [(0, 1), (2, 3)], maps)
    assert status.tolist() == [EXCHANGE_STUCK, EXCHANGE_OK] and delivered == [[], [1]]
    want = pack_logs([logs[0], logs[1], logs[2], logs[2]], with_changes=True)
    assert new.log_slice(3)[0].tobytes() == want.log_slice(3)[0].tobytes()
    assert int(new.desc[1]["n_insdel"]) == int(cur.desc[1]["n_insdel"])
    # a seq gap in either table
    for log in (0, 1):
        t = cur.changes
        bad = ChangeTable(t.desc, t.changes.copy(), t.deps)
        bad.changes[int(t.desc[log]["change_off"])]["seq"] = 2
        broken = PackedBatch(cur.desc, cur.insdel, cur.marks, cur.values, cur.link_attrs, cur.comment_ids, cur.other_attrs, {}, cur.log_actors,
                             cur.log_counters, bad, cur.log_lists)
        _, status, delivered, _ = apply_exchange(broken, [(0, 1), (2, 3)], maps)
        assert status.tolist() == [EXCHANGE_BAD_TABLE, EXCHANGE_OK] and delivered == [[], [1]]
    # n_ops that do not sum to the log's records
    bad = ChangeTable(t.desc, t.changes.copy(), t.deps)
    bad.changes[int(t.desc[2]["change_off"]) + 1]["n_ops"] += 1
    broken = PackedBatch(cur.desc, cur.insdel, cur.marks, changes=bad, log_actors=cur.log_actors, log_counters=cur.log_counters)
    _, status, _, _ = apply_exchange(broken, [(2, 3)], ExchangeMaps.of([maps.actor(1)]))
    assert status.tolist() == [EXCHANGE_BAD_TABLE]


def dense_logs():
    """(logs, pairs): a dense src into a plain dst that turns dense, and a plain src into a dense dst."""
    d1, init, big = sparse_peer()
    c = d1.change([{"path": ["text"], "action": "insert", "index": 1, "values": ["Z"]}])["change"]
    return [[init, big, c], [init], [init, big], [init, big, c]], [(0, 1), (3, 2)]


def test_dense_counters_on_either_side():
    logs, pairs = dense_logs()
    cur = pack_logs(logs, with_changes=True)
    assert cur.log_counters[0] is not None and cur.log_counters[1] is None
    maps, pre = exchange_maps(cur, [pairs[0]])
    assert pre is not None and maps.ctr(0) is not None
    new, status, delivered, _ = apply_exchange(apply_append(cur, *pre), [pairs[0]], maps)
    assert status.tolist() == [EXCHANGE_OK] and delivered == [[1, 2]]
    assert_same_batch(new, pack_logs([logs[0], logs[0], logs[2], logs[3]], with_changes=True))
    # without a counter map the dense ranks of src would be read as dst's plain counters: a wrong batch, so the map matters
    maps, pre = exchange_maps(cur, [pairs[1]])
    cur2 = apply_append(cur, *pre) if pre is not None else cur
    new, status, delivered, _ = apply_exchange(cur2, [pairs[1]], maps)
    assert status.tolist() == [EXCHANGE_OK] and delivered == [[2]]
    assert_same_batch(new, pack_logs([logs[0], logs[1], logs[3], logs[3]], with_changes=True))
    # a counter without an image
    cm = maps.ctr(0).copy() if maps.ctr(0) is not None else np.arange(int(cur2.desc[3]["max_ctr"]) + 1, dtype=np.uint32)
    cm[-1] = CTR_UNUSED
    _, status, delivered, _ = apply_exchange(cur2, [pairs[1]], ExchangeMaps.of([maps.actor(0)], [cm]))
    assert status.tolist() == [EXCHANGE_UNMAPPED] and delivered == [[]]


def test_two_way_and_chain_read_the_state_before_the_call():
    docs, _, init = generateDocs(O, "abc", 3)
    a, b, c = docs
    ca, cb = typed(a, "A", 1), typed(b, "B", 2)
    logs = [[init, ca], [init, cb], [init]]
    _, _, new, status, delivered, _ = sync_once(logs, [(0, 1), (1, 0)])
    assert status.tolist() == [EXCHANGE_OK, EXCHANGE_OK] and delivered == [[1], [1]]
    assert_same_batch(new, pack_logs([[init, ca, cb], [init, cb, ca], [init]], with_changes=True))
    # a chain: C receives what B held before the call, not what B receives from A in it
    _, _, new, status, delivered, _ = sync_once(logs, [(0, 1), (1, 2)])
    assert delivered == [[1], [1]]
    assert_same_batch(new, pack_logs([[init, ca], [init, cb, ca], [init, cb]], with_changes=True))


def test_empty_missing_set_and_refused_pairs():
    docs, _, init = generateDocs(O, "abc", 2)
    ca = typed(docs[0], "A", 1)
    logs = [[init, ca], [init, ca]]
    cur, maps, new, status, delivered, ddesc = sync_once(logs, [(0, 1)])
    assert status.tolist() == [EXCHANGE_OK] and delivered == [[]]
    assert_same_batch(new, cur) and int(ddesc["n_insdel"].sum()) == 0
    for bad in ([(0, 0)], [(0, 2)], [(0, 1), (0, 1)]):
        with pytest.raises(ValueError):
            apply_exchange(cur, bad, ExchangeMaps.of([maps.actor(0)] * len(bad)))
