"""The host specification of pt_batch_sync_pairs: ``packing.sync_maps`` (the DENSE pairs, then ``exchange_maps`` of the others),
its pre-append and ``apply_exchange`` against the reference's sync as the harness's fuzz sessions run it.
tests/test_gpu_sync.py runs the same replays on the device with nothing but the pair list."""
import numpy as np
import pytest

from peritext_b200.packing import (EXCHANGE_DENSE, EXCHANGE_OK, ChangeTable, PackedBatch, add_actors, apply_append, apply_exchange, exchange_maps,
                                   pack_append, pack_logs, sync_maps)
from tests.test_append_packing import assert_same_batch
from tests.test_exchange_model import SESSIONS, dense_logs, record_session, replay, three_replicas


def spec_sync(cur, pairs):
    """(the batch after the sync, per-pair status, delivered per pair, the DESC_DT delta, the pre-append or None)."""
    status, live, maps, pre = sync_maps(cur, pairs)
    if pre is not None:
        cur = apply_append(cur, *pre)
    new, st, dl, ddesc = apply_exchange(cur, live, maps)
    delivered, k = [], 0
    for p in range(len(pairs)):
        if status[p] == EXCHANGE_DENSE:
            delivered.append([])
        else:
            status[p] = st[k]; delivered.append(dl[k]); k += 1
    return new, status, delivered, ddesc, pre


def change_through_add_actors(cur, mlogs, r, change):
    """A local change as pt_batch_add_actors then an append whose actor map is the identity: the add introduces the actor."""
    delta, remap, ranks = add_actors(cur, [[change["actor"]] if i == r else [] for i in range(cur.n_logs)])
    cur = apply_append(cur, delta, remap)
    assert cur.log_actors[r][ranks[r][0]] == change["actor"]
    delta, remap = pack_append(cur, [[change] if i == r else [] for i in range(cur.n_logs)], with_changes=True)
    assert remap.actor_off is None and remap.ctr_off is None
    return apply_append(cur, delta, remap)


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions_replayed_through_sync_maps(seed, kw):
    ids, init, events, logs = record_session(seed, 60, **kw)

    def on_sync(cur, mlogs, pairs):
        new, status, delivered, _, _ = spec_sync(cur, pairs)
        assert (status != EXCHANGE_DENSE).all()
        return new, status, delivered
    cur, mlogs = replay(ids, init, events, change_through_add_actors, on_sync)
    assert mlogs == logs
    assert_same_batch(cur, pack_logs(logs, with_changes=True))


def test_dense_rule_flags_exactly_the_pairs_that_need_counter_maps():
    logs, pairs = dense_logs()
    cur = pack_logs(logs, with_changes=True)
    init, cz, cy = three_replicas()
    plain = pack_logs([[init, cz, cy], [init]], with_changes=True)
    for batch, prs in ((cur, pairs + [(1, 2)]), (plain, [(0, 1), (1, 0)])):
        status, live, _, _ = sync_maps(batch, prs)
        for p, pr in enumerate(prs):
            maps, pre = exchange_maps(batch, [pr])
            needs = maps.ctr(0) is not None or (pre is not None and (pre[1].ctr_off is not None or any(t is not None for t in pre[0].log_counters)))
            assert (status[p] == EXCHANGE_DENSE) == needs, pr
        assert live == [pr for p, pr in enumerate(prs) if status[p] != EXCHANGE_DENSE]


def test_dense_pairs_leave_the_other_pairs_as_exchange_maps_does():
    logs, pairs = dense_logs()
    init, cz, cy = three_replicas()
    cur = pack_logs(logs + [[init, cz, cy], [init]], with_changes=True)
    prs = pairs + [(4, 5)]
    new, status, delivered, _, pre = spec_sync(cur, prs)
    assert status.tolist() == [EXCHANGE_DENSE, EXCHANGE_DENSE, EXCHANGE_OK] and delivered[:2] == [[], []]
    assert new.log_actors[5] == cur.log_actors[4] and pre is not None
    assert new.log_actors[:4] == cur.log_actors[:4]


def turning_dense():
    """(batch, pairs): logs 0 and 1 are plain, but log 0's second change has counters far past its op count (as a
    pt_batch_change with a large first_ctr leaves them), so log 1, grown by it, would be re-ranked densely; logs 2 -> 3 are a
    plain pair beside it."""
    init, cz, cy = three_replicas()
    cur = pack_logs([[init, cz], [init], [init, cz, cy], [init]], with_changes=True)
    ins = cur.insdel.copy()
    z = cur.log_actors[0].index(cz["actor"])
    lo, hi = int(cur.desc[0]["insdel_off"]), int(cur.desc[0]["insdel_off"]) + int(cur.desc[0]["n_insdel"])
    mine = (ins["actor"][lo:hi] == z) & (ins["ctr"][lo:hi] != 0)
    ref = (ins["ref_actor"][lo:hi] == z) & (ins["ref_ctr"][lo:hi] != 0)
    ins["ctr"][lo:hi][mine] += 500; ins["ref_ctr"][lo:hi][ref] += 500
    desc = cur.desc.copy()
    desc[0]["max_ctr"] = int(ins["ctr"][lo:hi].max())
    batch = PackedBatch(desc, ins, cur.marks, cur.values, cur.link_attrs, cur.comment_ids, cur.other_attrs, cur.meta, cur.log_actors,
                        cur.log_counters, ChangeTable(cur.changes.desc, cur.changes.changes, cur.changes.deps), cur.log_lists)
    return batch, [(0, 1), (1, 0), (2, 3)]


def test_dst_turning_dense_is_a_dense_pair():
    batch, pairs = turning_dense()
    assert batch.log_counters[0] is None and batch.log_counters[1] is None
    maps, pre = exchange_maps(batch, [pairs[0]])
    assert pre is not None and pre[0].log_counters[1] is not None          # the host maps would re-rank log 1
    new, status, delivered, _, pre = spec_sync(batch, pairs)
    assert status.tolist() == [EXCHANGE_DENSE, EXCHANGE_OK, EXCHANGE_OK] and delivered == [[], [], [1, 2]]
    assert new.log_actors[1] == batch.log_actors[1] and new.log_slice(1)[0].tobytes() == batch.log_slice(1)[0].tobytes()


def test_add_actors_orders_by_utf16_code_units_and_moves_ranks():
    """A surrogate pair (U+1F600, code units D83D DE00) sorts before U+FF61 in JS order, after it by code point; duplicates and
    known ids are allowed; a new id sorting first moves every old rank."""
    init, cz, cy = three_replicas()
    cur = pack_logs([[init, cz, cy], [init], []], with_changes=True)
    names = [["\U0001F600", "｡", "doc2", "\U0001F600"], ["0first"], []]
    delta, remap, ranks = add_actors(cur, names)
    new = apply_append(cur, delta, remap)
    assert new.log_actors[0] == ["doc1", "doc2", "doc3", "\U0001F600", "｡"] and ranks[0] == [3, 4, 1, 3]
    assert new.log_actors[1] == ["0first", "doc1"] and ranks[1] == [0]
    assert remap.actor_map[int(remap.actor_off[1]): int(remap.actor_off[2])].tolist() == [1]
    assert int(remap.actor_off[1]) == int(remap.actor_off[0])                # log 0's ids all sort after its old ones
    assert new.desc["n_actors"].tolist() == [5, 2, 1] and new.desc["max_ctr"].tolist() == cur.desc["max_ctr"].tolist()
    old, got = cur.log_slice(1)[0], new.log_slice(1)[0]
    assert (got["actor"][old["ctr"] != 0] == 1).all() and np.array_equal(got["ctr"], old["ctr"])     # doc1's ids moved to rank 1
