"""pt_batch_exchange on the device: the sync of the reference's fuzz loop (getMissingChanges + applyChanges, reference
test/merge.ts:4-38) between logs of one resident batch.

The expected batch, statuses and delivery order are always ``packing.apply_exchange`` (the host specification, which
tests/test_exchange_model.py pins against ``pack_logs`` of the harness's logs); after an exchange and a merge every output must
equal a fresh upload of that batch."""
import ctypes
import random

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200 import workload
from peritext_b200.packing import (ACTOR_UNMAPPED, CTR_UNUSED, DESC_DT, EXCHANGE_BAD_TABLE, EXCHANGE_OK, EXCHANGE_STUCK, EXCHANGE_UNMAPPED, INSDEL_DT,
                                   MARK_DT, ChangeTable, ExchangeMaps, PackedBatch, _ranges, apply_append, apply_exchange, decode_spans,
                                   exchange_maps, pack_append, pack_logs)
from tests.harness import generateDocs
from tests.test_change_spec import next_op, replica
from tests.test_exchange_model import (SESSIONS, dense_logs, record_session, replay, three_replicas, typed)
from tests.test_gpu_append import canon, everything, merged, record_split, route_crossings
from tests.test_gpu_change import change_table, empty_table
from tests.test_gpu_routes import batch_of, expected_route

PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_patches=True, **kw)


def upload(e, batch):
    e.upload(batch)
    e.upload_changes(batch.changes)


def device_sync(e, cur, pairs):
    """exchange_maps, its pre-append and the exchange on handle `e` (holding `cur`); checks the view against the model and
    returns (the batch the handle must now hold, status, delivered per pair)."""
    maps, pre = exchange_maps(cur, pairs)
    if pre is not None:
        e.append(*pre)
        cur = apply_append(cur, *pre)
    want, status, delivered, ddesc = apply_exchange(cur, pairs, maps)
    got_status, (off, flat), got_desc = e.exchange(pairs, maps)
    assert got_status.tolist() == status.tolist()
    assert [flat[int(off[p]): int(off[p + 1])].tolist() for p in range(len(pairs))] == delivered
    for f in ("n_insdel", "n_mark", "n_actors", "max_ctr"):
        assert np.array_equal(got_desc[f], ddesc[f]), f
    return want, status, delivered


def same_as_upload(e, u, batch, window=None):
    """A merge on `e` against a fresh upload of `batch` on `u`, under the same patch window: results, text, spans, comment pool,
    element sequence, Patch stream, element queries and both JSON renders."""
    upload(u, batch)
    e.set_patch_window(window); u.set_patch_window(window)       # None: whole logs (an earlier compare may have left a window on `e`)
    got, want = merged(e), merged(u)
    assert canon(got) == canon(want)
    ok = [i for i in range(batch.n_logs) if int(got.results[i]["status"]) == 0]
    assert [got.sequence(i).tobytes() for i in ok] == [want.sequence(i).tobytes() for i in ok]
    assert everything(e, batch, got) == everything(u, batch, want)
    return got


# ------------------------------------------------------------------------------------------------------------------
# 1. The fuzz sessions of the model tests, on the device
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions_replayed_on_the_device(seed, kw):
    ids, init, events, logs = record_session(seed, 40, **kw)
    e, u = engine(), engine()
    n_sync = [0]

    def on_change(cur, mlogs, r, change):
        delta, remap = pack_append(cur, [[change] if i == r else [] for i in range(cur.n_logs)], with_changes=True)
        e.append(delta, remap)
        return apply_append(cur, delta, remap)

    def on_sync(cur, mlogs, pairs):
        old = (cur.desc["n_insdel"].astype(np.int64) + cur.desc["n_mark"]).astype(np.uint32)
        new, status, delivered = device_sync(e, cur, pairs)
        n_sync[0] += 1
        if n_sync[0] % 4 == 1:                      # the window of the delivered ops: the Patches applyChanges returned
            same_as_upload(e, u, new, window=old)
        return new, status, delivered

    try:
        upload(e, pack_logs([[init] for _ in ids], with_changes=True))
        cur, mlogs = replay(ids, init, events, on_change, on_sync)
        assert mlogs == logs
        got = same_as_upload(e, u, cur)
        assert (got.results["status"] == 0).all()
        for i, lg in enumerate(mlogs):
            assert decode_spans(cur, got, i) == replica(lg, "~reader").getTextWithFormatting()
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. A closed device loop: change, two-way exchange, merge
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_closed_loop_of_change_exchange_and_merge():
    rng = random.Random(3)
    n_docs, R = 5, 3
    ids = [f"doc{i + 1}" for i in range(R)]
    inits = [generateDocs(O, "abcdef"[: 3 + d % 3], 1)[2] for d in range(n_docs)]
    mlogs = [[inits[d]] for d in range(n_docs) for _ in range(R)]
    n = len(mlogs)
    cur = pack_logs(mlogs, with_changes=True)
    e, u = engine(), engine()
    try:
        upload(e, cur)
        # every replica's actor gets its rank in every log up front (doc1 < doc2 < doc3: the old rank stays)
        desc = np.zeros(n, DESC_DT)
        desc["n_actors"], desc["max_ctr"] = R, cur.desc["max_ctr"]
        intro = PackedBatch(desc, np.zeros(0, INSDEL_DT), np.zeros(0, MARK_DT), cur.values, cur.link_attrs, cur.comment_ids, cur.other_attrs, {},
                            [list(ids) for _ in range(n)], cur.log_counters, empty_table(n), cur.log_lists)
        e.append(intro)
        cur = apply_append(cur, intro)
        synced = [set() for _ in range(n_docs)]
        for step in range(6):
            merged(e)
            r = [rng.randrange(R) for _ in range(n_docs)]
            inputs, ranks = [None] * n, [None] * n
            for d in range(n_docs):
                i = d * R + r[d]
                doc = replica(mlogs[i], ids[r[d]])
                length = len(doc.root["text"])
                op = {"path": ["text"], "action": "insert", "index": rng.randrange(length + 1), "values": [rng.choice("xyz")]} if step % 2 == 0 or length < 2 else \
                    {"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": rng.randrange(1, length), "markType": rng.choice(["strong", "em"])}
                inputs[i] = {"actor": ids[r[d]], "seq": 1 + sum(c["actor"] == ids[r[d]] for c in mlogs[i]), "deps": doc.clock, "startOp": next_op(mlogs[i]), "ops": [op]}
                ranks[i] = r[d]
            some = [i for i in range(n) if inputs[i] is not None]
            table = change_table(cur.select(some), [inputs[i] for i in some], [ranks[i] for i in some])
            full = empty_table(n)
            full.desc["n_changes"][some] = 1; full.desc["n_deps"][some] = table.desc["n_deps"]
            full.desc["change_off"][some] = table.desc["change_off"]; full.desc["dep_off"][some] = table.desc["dep_off"]
            cur, dicts, status = e.change(cur, inputs, ranks, ChangeTable(full.desc, table.changes, table.deps))
            assert (status["status"] == 0).all()
            for i in some:
                mlogs[i].append(dicts[i])
            pairs = []
            for d in range(n_docs):
                a, b = rng.sample(range(R), 2)
                pairs += [(d * R + a, d * R + b), (d * R + b, d * R + a)]
                synced[d] |= {a, b}
            before = [list(lg) for lg in mlogs]
            cur, status, delivered = device_sync(e, cur, pairs)
            assert (status == EXCHANGE_OK).all()
            for p, (s, t) in enumerate(pairs):
                mlogs[t] += [before[s][k] for k in delivered[p]]
        # a last round brings every document's replicas together
        for a, b in ((0, 1), (1, 2), (0, 1)):
            pairs = [q for d in range(n_docs) for q in ((d * R + a, d * R + b), (d * R + b, d * R + a))]
            before = [list(lg) for lg in mlogs]
            cur, status, delivered = device_sync(e, cur, pairs)
            for p, (s, t) in enumerate(pairs):
                mlogs[t] += [before[s][k] for k in delivered[p]]
        got = same_as_upload(e, u, cur)
        for d in range(n_docs):
            digests = {bytes(got.results[d * R + k]["digest"]) for k in range(R)}
            assert len(digests) == 1, d
            for k in range(R):
                assert decode_spans(cur, got, d * R + k) == replica(mlogs[d * R + k], "~reader").getTextWithFormatting()
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. Per-pair statuses, dense counters, refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_failing_pairs_deliver_nothing_and_do_not_disturb_the_others():
    init, cz, cy = three_replicas()
    logs = [[init, cy], [init], [init, cz], [init], [init, cz, cy], [init]]     # 0 -> 1 is stuck; 4 -> 5 is not pre-appended
    cur = pack_logs(logs, with_changes=True)
    pairs = [(0, 1), (2, 3), (4, 5)]
    e, u = engine(), engine()
    try:
        upload(e, cur)
        maps, pre = exchange_maps(cur, pairs[:2])
        e.append(*pre)
        cur = apply_append(cur, *pre)
        bare = ExchangeMaps.of([maps.actor(0), maps.actor(1), np.array([0, ACTOR_UNMAPPED, ACTOR_UNMAPPED], np.uint16)])
        want, status, delivered, _ = apply_exchange(cur, pairs, bare)
        assert status.tolist() == [EXCHANGE_STUCK, EXCHANGE_OK, EXCHANGE_UNMAPPED]
        got_status, (off, flat), _ = e.exchange(pairs, bare)
        assert got_status.tolist() == status.tolist() and off.tolist() == [0, 0, 1, 1] and flat.tolist() == [1]
        upload(u, want)                             # (log 0 fails admission: its patch records are not computed, so no Patch compare)
        got, ref = merged(e), merged(u)
        assert canon(got) == canon(ref) and [int(s) for s in got.results["status"]] == [7, 0, 0, 0, 0, 0]
        assert e.render_json_list(want) == u.render_json_list(want)
        # a seq gap in src's table, and a counter of a delivered record without an image (found by the gather kernel)
        bad = ChangeTable(want.changes.desc, want.changes.changes.copy(), want.changes.deps)
        bad.changes[int(bad.desc[4]["change_off"])]["seq"] = 3
        broken = PackedBatch(want.desc, want.insdel, want.marks, want.values, want.link_attrs, want.comment_ids, want.other_attrs, {}, want.log_actors,
                             want.log_counters, bad, want.log_lists)
        upload(e, broken)
        pairs2 = [(4, 5), (2, 1)]
        maps2, pre2 = exchange_maps(broken, pairs2)
        e.append(*pre2)
        broken = apply_append(broken, *pre2)
        cm = np.arange(int(broken.desc[2]["max_ctr"]) + 1, dtype=np.uint32)
        cm[-1] = CTR_UNUSED
        maps2 = ExchangeMaps.of([maps2.actor(0), maps2.actor(1)], [None, cm])
        want2, status2, delivered2, _ = apply_exchange(broken, pairs2, maps2)
        assert status2.tolist() == [EXCHANGE_BAD_TABLE, EXCHANGE_UNMAPPED]
        got_status, (off, flat), desc = e.exchange(pairs2, maps2)
        assert got_status.tolist() == status2.tolist() and int(off[-1]) == 0 and int(desc["n_insdel"].sum()) == 0
        e.merge()
        assert canon(e._download_with_pool_retry()) == canon(u.run(broken))
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_dense_counters_on_either_side():
    logs, pairs = dense_logs()
    cur = pack_logs(logs, with_changes=True)
    e, u = engine(), engine()
    try:
        upload(e, cur)
        cur, status, delivered = device_sync(e, cur, pairs)
        assert status.tolist() == [EXCHANGE_OK, EXCHANGE_OK] and delivered == [[1, 2], [2]]
        same_as_upload(e, u, cur)
    finally:
        e.close(); u.close()


def raw_exchange(e, pairs, aoff, amap, coff=None, cmap=None, null=()):
    """pt_batch_exchange's status; `null` = the positions among (pairs, actor_off, actor_map, ctr_off, ctr_map) passed as NULL."""
    from peritext_b200.engine import _ExchangeInput, _ExchangeView, _map_arrays, _pairs, _ptr
    arrs = [_pairs(pairs), *_map_arrays(ExchangeMaps(aoff, amap, coff, cmap))]
    inp = _ExchangeInput(len(arrs[0]), *[None if k in null else _ptr(a) for k, a in enumerate(arrs)])
    return e._L.pt_batch_exchange(e._h, ctypes.byref(inp), ctypes.byref(_ExchangeView()))


@pytest.mark.gpu
def test_refusals_leave_the_batch_untouched():
    from peritext_b200.engine import BatchEngine
    docs, _, init = generateDocs(O, "abc", 3)
    ca, cb = typed(docs[0], "A", 1), typed(docs[1], "B", 2)
    init2 = generateDocs(O, "xy", 1)[2]
    cur = pack_logs([[init, ca, cb], [init, cb], [init, ca], [init2]], with_changes=True)
    na = [int(x) for x in cur.desc["n_actors"]]
    assert na == [2, 2, 1, 1]
    ident = lambda k: list(range(k))
    e = engine()
    try:
        upload(e, cur)
        before = merged(e)
        snap = everything(e, cur, before)
        bad = {
            "null pairs": lambda: raw_exchange(e, [(0, 1)], [0, 2], ident(2), null=(0,)),
            "null actor_off": lambda: raw_exchange(e, [(0, 1)], [0, 2], ident(2), null=(1,)),
            "null actor_map": lambda: raw_exchange(e, [(0, 1)], [0, 2], ident(2), null=(2,)),
            "src outside": lambda: raw_exchange(e, [(4, 1)], [0, 2], ident(2)),
            "dst outside": lambda: raw_exchange(e, [(0, 9)], [0, 2], ident(2)),
            "src == dst": lambda: raw_exchange(e, [(1, 1)], [0, 2], ident(2)),
            "dst twice": lambda: raw_exchange(e, [(0, 1), (2, 1)], [0, 2, 3], ident(2) + [0]),
            "actor map length": lambda: raw_exchange(e, [(0, 1)], [0, 1], [0]),
            "actor map order": lambda: raw_exchange(e, [(0, 1)], [0, 2], [1, 0]),
            "actor map bound": lambda: raw_exchange(e, [(0, 2)], [0, 2], [0, 1]),
            "ctr_map[0]": lambda: raw_exchange(e, [(0, 1)], [0, 2], ident(2), [0, 3], [1, 2, 3]),
            "ctr map order": lambda: raw_exchange(e, [(0, 1)], [0, 2], ident(2), [0, 4], [0, 2, 2, 3]),
        }
        for name, call in bad.items():
            assert call() == PT_ERR_INVALID, name
            assert e._L.pt_last_error().decode().startswith("pt_batch_exchange: "), name
        after = merged(e)
        assert canon(after) == canon(before) and everything(e, cur, after) == snap
        assert raw_exchange(e, [], [0], []) == 0                             # no pairs: nothing changes, the merge stays valid
        assert everything(e, cur, e.download()) == snap
        # the valid exchange still goes through afterwards
        want, status, delivered = device_sync(e, cur, [(0, 1), (1, 2)])
        assert delivered == [[1], [1]]
        f, g = BatchEngine(0), BatchEngine(0)
        try:
            assert raw_exchange(f, [(0, 1)], [0, 2], ident(2)) == PT_ERR_STATE          # no batch
            g.upload(cur)
            assert raw_exchange(g, [(0, 1)], [0, 2], ident(2)) == PT_ERR_STATE          # no change table
        finally:
            f.close(); g.close()
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Logs on different routes
# ------------------------------------------------------------------------------------------------------------------
def one_change_tables(batch, actors):
    """Every log's records as one change (seq 1) by the given actor rank."""
    t = workload.history_table(batch)
    t.changes["actor"] = actors
    return t


@pytest.mark.gpu
def test_exchanges_between_and_across_routes():
    """Deliveries that move the dst across a route boundary, from a src on another route: the prefixes of
    tests/test_gpu_append.py's route crossings (warp, team and CTA routes) receive their suffixes from the full logs, which hold
    them as a second change."""
    cases = route_crossings()
    full = batch_of([lg for lg, _ in cases])
    pre, _ = record_split(full, [k for _, k in cases])
    n = full.n_logs
    # logs 0..n-1: the full logs as two changes (prefix, suffix) by actor 0; logs n..2n-1: the prefixes as one change
    both = PackedBatch(np.concatenate([full.desc, pre.desc]), np.concatenate([full.insdel, pre.insdel]), np.concatenate([full.marks, pre.marks]))
    both.desc["insdel_off"] = np.cumsum(both.desc["n_insdel"].astype(np.uint64)) - both.desc["n_insdel"]
    both.desc["mark_off"] = np.cumsum(both.desc["n_mark"].astype(np.uint64)) - both.desc["n_mark"]
    cd = np.zeros(2 * n, workload.CDESC_DT)
    cd["n_changes"] = [2] * n + [1] * n
    cd["change_off"] = np.cumsum(cd["n_changes"]) - cd["n_changes"]
    ch = np.zeros(3 * n, workload.CHANGE_DT)
    pre_ops = pre.desc["n_insdel"].astype(np.int64) + pre.desc["n_mark"]
    all_ops = full.desc["n_insdel"].astype(np.int64) + full.desc["n_mark"]
    for i in range(n):
        ch[2 * i] = (1, 0, 0, 0, pre_ops[i]); ch[2 * i + 1] = (2, 0, 0, 0, all_ops[i] - pre_ops[i]); ch[2 * n + i] = (1, 0, 0, 0, pre_ops[i])
    both.changes = ChangeTable(cd, ch, np.zeros(0, workload.DEP_DT))
    both.log_actors = [[f"a{k}" for k in range(int(x))] for x in both.desc["n_actors"]]
    pairs = [(i, n + i) for i in range(n)]
    maps = ExchangeMaps.of([np.arange(int(both.desc[i]["n_actors"]), dtype=np.uint16) for i in range(n)])
    want, status, delivered, _ = apply_exchange(both, pairs, maps)
    assert status.tolist() == [EXCHANGE_OK] * n and delivered == [[1]] * n
    for i in range(n):
        assert want.log_slice(n + i)[0].tobytes() == full.log_slice(i)[0].tobytes() and want.log_slice(n + i)[1].tobytes() == full.log_slice(i)[1].tobytes()
        assert expected_route(both.desc[n + i]) != expected_route(want.desc[n + i]) and expected_route(both.desc[n + i]) != expected_route(both.desc[i])
    e, u = engine(), engine()
    try:
        upload(e, both)
        got_status, (off, flat), _ = e.exchange(pairs, maps)
        assert got_status.tolist() == [0] * n and flat.tolist() == [1] * n
        upload(u, want)
        assert canon(merged(e)) == canon(merged(u))
        # back the other way nothing is missing
        back = [(n + i, i) for i in range(n)]
        gs, (off, flat), _ = e.exchange(back, maps)
        assert gs.tolist() == [0] * n and int(off[-1]) == 0
        assert canon(merged(e)) == canon(merged(u))
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. A c4-shaped batch of 300 000 logs: one change and one two-way sync per document
# ------------------------------------------------------------------------------------------------------------------
def packed_change(e, batch, actor, off, ops, tokens, table):
    """``change_packed`` of a ``workload.sync_round``; returns its delta as a PackedBatch with the round's change table."""
    _, desc, insdel, marks = e.change_packed(actor, off, ops, tokens, 0, len(batch.link_attrs), 0, table)
    return PackedBatch(desc, insdel, marks, changes=table)


@pytest.mark.gpu
def test_c4_300k_logs_one_change_and_one_two_way_sync_per_document():
    from peritext_b200.engine import BatchEngine
    base = workload.generate("c4", n_docs=100_000, ops_per_doc=120)
    assert base.n_logs >= 300_000
    base.changes = workload.history_table(base)
    actor, off, ops, tokens, table, pairs, maps = workload.sync_round(base)
    e = BatchEngine(0, emit_sequence=True)
    try:
        e.upload(base); e.upload_changes(base.changes)
        e.merge()
        delta = packed_change(e, base, actor, off, ops, tokens, table)
        changed = apply_append(base, delta)
        status, (doff, flat), desc = e.exchange(pairs, maps)
        assert (status == 0).all()
        # the changer's new change (its last) reaches the other replica; nothing comes back
        src, dst = pairs[0::2, 0], pairs[0::2, 1]
        assert np.array_equal(np.diff(doff.astype(np.int64)), np.tile([1, 0], len(src)))
        assert np.array_equal(flat, changed.changes.desc["n_changes"][src] - 1)
        # the expected batch: every dst gains its src's generated records, the mark-free insert's ids unchanged (identity maps)
        d2 = np.zeros(base.n_logs, DESC_DT)
        d2["n_actors"] = base.desc["n_actors"]
        d2["max_ctr"] = changed.desc["max_ctr"]; d2["max_ctr"][dst] = changed.desc["max_ctr"][src]
        d2["n_insdel"][dst] = delta.desc["n_insdel"][src]
        d2["insdel_off"] = np.cumsum(d2["n_insdel"].astype(np.uint64)) - d2["n_insdel"]
        order = np.argsort(dst)
        recs = delta.insdel[_ranges(delta.desc["insdel_off"][src[order]], delta.desc["n_insdel"][src[order]])]
        cd = np.zeros(base.n_logs, workload.CDESC_DT)
        cd["n_changes"][dst] = 1; cd["n_deps"][dst] = table.desc["n_deps"][src]
        cd["change_off"] = np.cumsum(cd["n_changes"]) - cd["n_changes"]; cd["dep_off"] = np.cumsum(cd["n_deps"]) - cd["n_deps"]
        chs = table.changes[table.desc["change_off"][src[order]].astype(np.int64)]
        dps = table.deps[_ranges(table.desc["dep_off"][src[order]], table.desc["n_deps"][src[order]])]
        want = apply_append(changed, PackedBatch(d2, recs, np.zeros(0, MARK_DT), changes=ChangeTable(cd, chs, dps)))
        assert np.array_equal(desc["n_insdel"], d2["n_insdel"]) and np.array_equal(desc["max_ctr"], d2["max_ctr"])
        e.merge()
        got = e.results()
        e.upload(want); e.upload_changes(want.changes)
        e.merge()
        ref = e.results()
        assert got.tobytes() == ref.tobytes()
        assert (ref["status"] == 0).all()
        docs = base.n_logs // 3
        dig = ref["digest"].reshape(docs, 3, 2)
        s, d = src % 3, dst % 3
        assert (dig[np.arange(docs), s] == dig[np.arange(docs), d]).all()          # the synced replicas converged
    finally:
        e.close()
