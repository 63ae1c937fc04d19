"""pt_batch_sync_pairs on the device: the sync of the reference's fuzz loop with the exchange maps and the actor growth derived
from the handle's actor tables, so the caller sends nothing but the pair list.

The expected batch, statuses, delivery order and pre-append are always ``packing.sync_maps`` + ``apply_append`` +
``apply_exchange`` (tests/test_sync_model.py pins them against the harness's logs)."""
import ctypes

import numpy as np
import pytest

from peritext_b200 import workload
from peritext_b200.packing import (CDESC_DT, CHANGE_DT, CHANGE_NO_ACTOR, DEP_DT, DESC_DT, EXCHANGE_BAD_TABLE, EXCHANGE_DENSE, EXCHANGE_OK,
                                   EXCHANGE_STUCK, INPUT_OP_DT, AppendRemap, ChangeTable, PackedBatch, add_actors, apply_append, pack_append,
                                   pack_logs, range_requests, string_pools)
from tests.test_exchange_model import SESSIONS, dense_logs, record_session, replay, three_replicas
from tests.test_gpu_append import canon, merged
from tests.test_gpu_exchange import engine, packed_change, same_as_upload, upload
from tests.test_change_spec import replica
from tests.test_sync_model import spec_sync, turning_dense

PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def upload_all(e, batch):
    upload(e, batch)
    e.upload_actors(batch)


def device_sync(e, cur, pairs):
    """pt_batch_sync_pairs on `e` (holding `cur`), checked against the specification: statuses, delivered order, delta, the
    pre-append's actor maps and the actor tables.  Returns (the batch the handle must now hold, status, delivered)."""
    want, status, delivered, ddesc, pre = spec_sync(cur, pairs)
    got_status, (off, flat), got_desc, (aoff, amap) = e.sync_pairs(pairs)
    assert got_status.tolist() == status.tolist()
    assert [flat[int(off[p]): int(off[p + 1])].tolist() for p in range(len(pairs))] == delivered
    live = [p for p in range(len(pairs)) if status[p] != EXCHANGE_DENSE]
    if live:
        for f in ("n_insdel", "n_mark", "n_actors", "max_ctr"):
            assert np.array_equal(got_desc[f], ddesc[f]), f
    r = pre[1] if pre is not None else None
    if r is None or r.actor_off is None:
        assert int(aoff[-1]) == 0
    else:
        assert aoff.tolist() == r.actor_off.tolist() and amap.tolist() == r.actor_map.tolist()
    assert e.actors() == [list(a) for a in want.log_actors]
    return want, status, delivered


def device_add(e, cur, names):
    """pt_batch_add_actors on `e` (holding `cur`) against packing.add_actors; returns the batch the handle must now hold."""
    delta, remap, ranks = add_actors(cur, names)
    got, (aoff, amap) = e.add_actors(names)
    assert got == ranks
    if remap.actor_off is None:
        assert int(aoff[-1]) == 0
    else:
        assert aoff.tolist() == remap.actor_off.tolist() and amap.tolist() == remap.actor_map.tolist()
    new = apply_append(cur, delta, remap)
    assert e.actors() == [list(a) for a in new.log_actors]
    return new


# ------------------------------------------------------------------------------------------------------------------
# 1. The fuzz sessions: every first change by an actor through pt_batch_add_actors, every sync through pt_batch_sync_pairs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions_synced_on_the_device(seed, kw):
    ids, init, events, logs = record_session(seed, 40, **kw)
    e, u = engine(), engine()
    n_sync = [0]

    def on_change(cur, mlogs, r, change):
        cur = device_add(e, cur, [[change["actor"]] if i == r else [] for i in range(cur.n_logs)])
        delta, remap = pack_append(cur, [[change] if i == r else [] for i in range(cur.n_logs)], with_changes=True)
        assert remap.actor_off is None
        e.append(delta, remap)                     # no actor map, no new actor: the tables stay
        return apply_append(cur, delta, remap)

    def on_sync(cur, mlogs, pairs):
        new, status, delivered = device_sync(e, cur, pairs)
        n_sync[0] += 1
        if n_sync[0] % 4 == 1:
            same_as_upload(e, u, new)
        return new, status, delivered

    try:
        upload_all(e, pack_logs([[init] for _ in ids], with_changes=True))
        cur, mlogs = replay(ids, init, events, on_change, on_sync)
        assert mlogs == logs
        got = same_as_upload(e, u, cur)
        assert (got.results["status"] == 0).all()
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. Actor growth
# ------------------------------------------------------------------------------------------------------------------
def renamed(logs, names):
    """The logs with every actor id replaced through `names` (change actors, deps, op ids and references)."""
    import json
    text = json.dumps(logs)
    for old, new in names.items():
        text = text.replace(f'"{old}"', json.dumps(new)).replace(f'@{old}"', "@" + json.dumps(new)[1:])
    return json.loads(text)


@pytest.mark.gpu
@pytest.mark.parametrize("names", [{}, {"doc3": "0first"}, {"doc2": "\U0001F600", "doc3": "｡"}, {"doc3": "\ud800x"}])
def test_actor_growth_two_way_and_chain(names):
    """x, y, z share the initial text; z types, y marks over it.  Renaming z's actor to sort first moves every rank of the
    logs that learn it; non-BMP and lone-surrogate ids order by UTF-16 code units."""
    init, cz, cy = three_replicas()
    logs = renamed([[init, cz, cy], [init], [init, cz], [init], [init], [init, cz, cy]], names)
    cur = pack_logs(logs, with_changes=True)
    e, u = engine(), engine()
    try:
        upload_all(e, cur)
        cur, status, delivered = device_sync(e, cur, [(0, 1), (1, 0), (2, 3), (3, 4)])           # two-way, and a chain
        assert status.tolist() == [EXCHANGE_OK] * 4 and delivered[0] == [1, 2] and delivered[3] == []
        cur, status, delivered = device_sync(e, cur, [(3, 4), (4, 5), (5, 2)])
        assert delivered[0] == [1]
        same_as_upload(e, u, cur)
        assert cur.log_actors[1] == cur.log_actors[0]
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_src_rank_without_a_name_and_statuses_as_exchange():
    """A log with no actor ids (n_actors 1, count 0) as src and dst; a stuck pair and a broken table beside good pairs."""
    init, cz, cy = three_replicas()
    logs = [[init, cy], [init], [init, cz], [init], [init, cz, cy], [init]]
    cur = pack_logs(logs + [[]], with_changes=True)
    assert cur.log_actors[6] == [] and int(cur.desc[6]["n_actors"]) == 1
    ch = cur.changes.changes.copy()
    c3 = int(cur.changes.desc[2]["change_off"]) + 1
    ch["seq"][c3] = 5                                      # log 2: seq gap
    cur = PackedBatch(cur.desc, cur.insdel, cur.marks, cur.values, cur.link_attrs, cur.comment_ids, cur.other_attrs, cur.meta,
                      cur.log_actors, cur.log_counters, ChangeTable(cur.changes.desc, ch, cur.changes.deps), cur.log_lists)
    e = engine()
    try:
        upload_all(e, cur)
        cur, status, _ = device_sync(e, cur, [(0, 1), (2, 3), (4, 5), (6, 0), (5, 6)])
        assert status.tolist() == [EXCHANGE_STUCK, EXCHANGE_BAD_TABLE, EXCHANGE_OK, EXCHANGE_OK, EXCHANGE_OK]
        assert cur.log_actors[6] == ["doc1"]                  # what log 5 held before the call
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. DENSE pairs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dense_pairs_deliver_nothing_and_leave_the_others_as_specified():
    logs, pairs = dense_logs()
    init, cz, cy = three_replicas()
    cur = pack_logs(logs + [[init, cz, cy], [init]], with_changes=True)
    e, u = engine(), engine()
    try:
        upload(e, cur)
        e.upload_actors(string_pools(cur))
        cur, status, delivered = device_sync(e, cur, pairs + [(4, 5)])
        assert status.tolist() == [EXCHANGE_DENSE, EXCHANGE_DENSE, EXCHANGE_OK]
        same_as_upload(e, u, cur)
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_dst_turning_dense_is_decided_on_the_device():
    """Two plain logs whose missing change has counters far past the op count: the derive kernel's _wants_dense test."""
    cur, pairs = turning_dense()
    e, u = engine(), engine()
    try:
        upload_all(e, cur)
        new, status, delivered = device_sync(e, cur, pairs)
        assert status.tolist() == [EXCHANGE_DENSE, EXCHANGE_OK, EXCHANGE_OK] and delivered == [[], [], [1, 2]]
        assert new.log_actors[1] == cur.log_actors[1]
        same_as_upload(e, u, new)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Table lifetime
# ------------------------------------------------------------------------------------------------------------------
def raw_sync(e, pairs, null=False):
    from peritext_b200.engine import _SyncView, _pairs, _ptr
    pr = _pairs(pairs)
    return e._L.pt_batch_sync_pairs(e._h, None if null else _ptr(pr), len(pr), ctypes.byref(_SyncView()))


@pytest.mark.gpu
def test_table_lifetime():
    init, cz, cy = three_replicas()
    logs = [[init, cz], [init], [init]]
    cur = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload(e, cur)
        assert raw_sync(e, [(0, 1)]) == PT_ERR_STATE                       # no tables yet
        e.upload_actors(cur)
        upload(e, cur)
        assert raw_sync(e, [(0, 1)]) == PT_ERR_STATE                       # an upload drops them
        e.upload_actors(cur)
        # an exchange and an append without maps keep them
        cur, _, _ = device_sync(e, cur, [(0, 1)])
        delta, remap = pack_append(cur, [[], [], [cz]], with_changes=True)
        e.append(delta, remap)                                             # log 2 learns z: its n_actors grows, which drops them
        assert raw_sync(e, [(0, 1)]) == PT_ERR_STATE
        cur = apply_append(cur, delta, remap)
        e.upload_actors(cur)
        nomap = PackedBatch(np.zeros(cur.n_logs, DESC_DT), cur.insdel[:0], cur.marks[:0], cur.values, cur.link_attrs, cur.comment_ids,
                            cur.other_attrs, dict(cur.meta), cur.log_actors, cur.log_counters,
                            ChangeTable(np.zeros(cur.n_logs, cur.changes.desc.dtype), cur.changes.changes[:0], cur.changes.deps[:0]), cur.log_lists)
        nomap.desc["n_actors"], nomap.desc["max_ctr"] = cur.desc["n_actors"], cur.desc["max_ctr"]
        e.append(nomap)
        assert e.actors() == [list(a) for a in cur.log_actors]
        e.append(nomap, AppendRemap(comment_map=np.arange(len(cur.comment_ids), dtype=np.uint32)))     # a comment-only remap keeps them
        assert e.actors() == [list(a) for a in cur.log_actors]
        cur, status, _ = device_sync(e, cur, [(2, 1)])
        assert status.tolist() == [EXCHANGE_OK]
        aoff = np.array([0, int(cur.desc[0]["n_actors"])] + [int(cur.desc[0]["n_actors"])] * (cur.n_logs - 1), np.uint64)
        e.append(nomap, AppendRemap(actor_off=aoff, actor_map=np.arange(int(aoff[1]), dtype=np.uint16)))   # an actor map drops them
        assert raw_sync(e, [(0, 1)]) == PT_ERR_STATE
        # pt_batch_adopt_device drops them too
        import torch
        e.upload_actors(cur)
        ins = torch.from_numpy(cur.insdel.view(np.uint8).copy()).cuda()
        mk = torch.from_numpy(cur.marks.view(np.uint8).copy()).cuda() if len(cur.marks) else torch.zeros(16, dtype=torch.uint8, device="cuda")
        e.adopt_device(cur.desc, ins.data_ptr(), len(cur.insdel), mk.data_ptr(), len(cur.marks))
        e.upload_changes(cur.changes)
        assert raw_sync(e, [(0, 1)]) == PT_ERR_STATE
        torch.cuda.synchronize()
    finally:
        e.close()


@pytest.mark.gpu
def test_add_actors_on_the_device():
    from peritext_b200.engine import BatchEngine
    """Unsorted ids with duplicates and known ones, non-BMP and lone-surrogate ids, a new id sorting first (every rank moves),
    empty lists; then the refusals, which change nothing."""
    init, cz, cy = three_replicas()
    cur = pack_logs([[init, cz, cy], [init], [], [init, cz]], with_changes=True)
    e, u = engine(), engine()
    try:
        upload_all(e, cur)
        cur = device_add(e, cur, [["\U0001F600", "｡", "doc2", "\U0001F600"], ["0first"], [], ["\ud800x", "doc1", "zz", "a"]])
        cur = device_add(e, cur, [[], [], ["doc1"], []])                 # a log without ids gains one, n_actors stays 1
        cur = device_add(e, cur, [[f"id{k:04d}" for k in range(999, -1, -1)], [], [], []])   # a long list, reversed
        assert len(e.actors()[0]) == 1005
        same_as_upload(e, u, cur)
        from peritext_b200.engine import _ActorInput, _ActorView
        f = BatchEngine(0)
        try:
            f.upload(cur)
            with pytest.raises(Exception, match="pt_batch_add_actors"):
                f.add_actors([[], [], [], []])                           # no tables
        finally:
            f.close()
        data = np.frombuffer("ab".encode("utf-16-le"), np.uint8)
        for off, first in (([0, 3], [0, 1, 1, 1, 1]), ([0, 4], [0, 1, 1]), ([0, 4], [0, 2, 1, 1, 1])):
            o, fi = np.array(off, np.uint64), np.array(first, np.uint64)
            inp = _ActorInput(len(fi) - 1, data.ctypes.data, o.ctypes.data, 1, fi.ctypes.data)
            assert e._L.pt_batch_add_actors(e._h, ctypes.byref(inp), ctypes.byref(_ActorView())) == PT_ERR_INVALID
        assert e.actors() == [list(a) for a in cur.log_actors]
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. A closed loop that keeps no records on the host: add_actors, change_packed, two-way sync, merge
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_records_free_closed_loop():
    """Documents with two replicas each, logs 2d and 2d + 1.  Per round one replica of every document inserts a character: its
    actor is introduced with pt_batch_add_actors (the second replica's id sorts before the first's, so ranks move), the change
    goes through pt_batch_change from arrays (InputOperations, the change record, dep ranks from pt_batch_download_actors), then both
    replicas sync both ways with pt_batch_sync_pairs and the batch merges.  The host keeps only the reference replicas, which
    replay the same calls; at the end the handle equals their pack_logs, the replicas' digests agree, and the Change JSON
    rendered with the downloaded tables equals the one rendered with string_pools of that batch."""
    from peritext_b200.engine import BatchEngine
    from oracle.oracle import Micromerge as O
    from tests.harness import generateDocs
    n_docs, ids = 4, ["doc1", "b-second"]
    inits = [generateDocs(O, "abcdef"[: 3 + d % 3], 1)[2] for d in range(n_docs)]
    mlogs = [[inits[d]] for d in range(n_docs) for _ in range(2)]
    n = len(mlogs)
    e, u = BatchEngine(0, emit_patches=True), engine()
    try:
        upload_all(e, pack_logs(mlogs, with_changes=True))
        for rnd in range(4):
            r = 1 - rnd % 2                                              # replica 1 changes first: a new actor
            logs = [2 * d + r for d in range(n_docs)]
            ranks, _ = e.add_actors([[ids[r]] if i in logs else [] for i in range(n)])
            tables = e.actors()
            e.merge()                                                    # pt_batch_change resolves indices against a merge
            actor = np.full(n, CHANGE_NO_ACTOR, np.uint32)
            off = np.zeros(n + 1, np.uint64)
            ops = np.zeros(n_docs, INPUT_OP_DT)
            cd = np.zeros(n, CDESC_DT)
            ch = np.zeros(n_docs, CHANGE_DT)
            deps = []
            for k, i in enumerate(logs):
                c = replica(mlogs[i], ids[r]).change([{"path": ["text"], "action": "insert", "index": 0, "values": ["xyz"[rnd % 3]]}])["change"]
                c["seq"] = 1 + sum(x["actor"] == ids[r] for x in mlogs[i])       # a replica rebuilt from its log restarts its own seq
                mlogs[i].append(c)
                actor[i] = ranks[i][0]
                ops[k] = (0, 0, 0, 0, 1, 0xFFFFFFFF, c["startOp"], 0, k)      # insert one value at index 0
                dl = sorted(c["deps"].items())
                ch[k] = (c["seq"], ranks[i][0], len(dl), 0, 1)
                cd[i]["n_changes"], cd[i]["n_deps"] = 1, len(dl)
                deps += [(s, tables[i].index(a), 0) for a, s in dl]
            off[1:] = np.cumsum(actor != CHANGE_NO_ACTOR)
            cd["change_off"] = np.cumsum(cd["n_changes"]) - cd["n_changes"]; cd["dep_off"] = np.cumsum(cd["n_deps"]) - cd["n_deps"]
            table = ChangeTable(cd, ch, np.array(deps, DEP_DT) if deps else np.zeros(0, DEP_DT))
            tokens = np.array([ord("xyz"[rnd % 3])] * n_docs, np.uint32)
            e.change_packed(actor, off, ops, tokens, 0, 0, 0, table)
            pairs = [(2 * d + r, 2 * d + 1 - r) for d in range(n_docs)] + [(2 * d + 1 - r, 2 * d + r) for d in range(n_docs)]
            status, (doff, flat), _, _ = e.sync_pairs(pairs)
            assert (status == EXCHANGE_OK).all() and np.diff(doff.astype(np.int64)).tolist() == [1] * n_docs + [0] * n_docs
            for d in range(n_docs):
                mlogs[2 * d + 1 - r].append(mlogs[2 * d + r][-1])
        want = pack_logs(mlogs, with_changes=True)
        assert e.actors() == [list(a) for a in want.log_actors]
        got = same_as_upload(e, u, want)
        dig = got.results["digest"].reshape(n_docs, 2, -1)
        assert (dig[:, 0] == dig[:, 1]).all() and (got.results["status"] == 0).all()
        held = PackedBatch(want.desc, want.insdel, want.marks, want.values, want.link_attrs, want.comment_ids, want.other_attrs, want.meta,
                           e.actors(), want.log_counters, want.changes, want.log_lists)
        req = range_requests(list(range(n)))
        a, b_ = e.render_changes_json(held, req), e.render_changes_json(want, req)
        assert a[0].tobytes() == b_[0].tobytes() and a[1].tolist() == b_[1].tolist() and len(a[0])
    finally:
        e.close(); u.close()



# ------------------------------------------------------------------------------------------------------------------
# 6. Refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_leave_the_batch_untouched():
    init, cz, cy = three_replicas()
    cur = pack_logs([[init, cz, cy], [init], [init, cz]], with_changes=True)
    e = engine()
    try:
        upload_all(e, cur)
        before = merged(e)
        good = string_pools(cur)

        def tables(**kw):
            p = {k: np.array(v, copy=True) for k, v in good.items()}
            p.update(kw)
            return p
        names = [a for acts in cur.log_actors for a in acts]
        enc = lambda ids: (np.frombuffer(b"".join(x.encode("utf-16-le", "surrogatepass") for x in ids), np.uint8),
                           np.concatenate([[0], np.cumsum([len(x.encode("utf-16-le", "surrogatepass")) for x in ids])]).astype(np.uint64))
        swapped = list(names)
        swapped[0], swapped[1] = swapped[1], swapped[0]
        d, o = enc(swapped)
        odd_o = good["actors_off"].copy(); odd_o[1:] += 1; odd_o[-1] -= 1
        first = good["actors_first"].copy(); first[1] += 1
        bad = {"unsorted": tables(actors=d, actors_off=o), "odd length": tables(actors=np.concatenate([good["actors"], [0]]).astype(np.uint8), actors_off=odd_o),
               "wrong count": tables(actors_first=first)}
        for name, t in bad.items():
            with pytest.raises(Exception, match="pt_batch_upload_actors: "):
                e.upload_actors(t)
        for pairs in ([(0, 3)], [(1, 1)], [(0, 1), (2, 1)]):
            assert raw_sync(e, pairs) == PT_ERR_INVALID
            assert e._L.pt_last_error().decode().startswith("pt_batch_sync_pairs: ")
        assert raw_sync(e, [(0, 1)], null=True) == PT_ERR_INVALID
        assert raw_sync(e, []) == 0
        assert e.actors() == [list(a) for a in cur.log_actors]
        assert canon(merged(e)) == canon(before)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 7. A c4-shaped batch of 300 000 logs: one change and one two-way sync per document, maps derived on the device
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c4_300k_logs_sync_pairs_equals_exchange_with_host_maps():
    from peritext_b200.engine import BatchEngine
    base = workload.generate("c4", n_docs=100_000, ops_per_doc=120)
    base.changes = workload.history_table(base)
    base.log_actors = [[f"a{k}" for k in range(int(x))] for x in base.desc["n_actors"]]
    actor, off, ops, tokens, table, pairs, maps = workload.sync_round(base)
    e, f = BatchEngine(0, emit_sequence=True), BatchEngine(0, emit_sequence=True)
    try:
        for h in (e, f):
            h.upload(base); h.upload_changes(base.changes); h.merge()
            packed_change(h, base, actor, off, ops, tokens, table)
        e.upload_actors(base)
        s1, (o1, d1), desc1, (aoff, _) = e.sync_pairs(pairs)
        s2, (o2, d2), desc2 = f.exchange(pairs, maps)
        assert (s1 == 0).all() and s1.tolist() == s2.tolist() and int(aoff[-1]) == 0
        assert o1.tolist() == o2.tolist() and d1.tolist() == d2.tolist() and desc1.tobytes() == desc2.tobytes()
        e.merge(); f.merge()
        assert e.results().tobytes() == f.results().tobytes()
    finally:
        e.close(); f.close()
