"""pt_batch_select_logs on the device: after a select the handle must hold exactly what an upload of the selected batch (with
its change table and actor tables) would hold, so every output of a merge after it equals the output of that upload.

The expected batch is always ``packing.apply_select``, which tests/test_select_packing.py pins against ``pack_logs`` and the
oracle."""
import numpy as np
import pytest

from oracle.packed import replay_packed
from peritext_b200 import workload
from peritext_b200.packing import (SELECT_ADDED, SELECT_DROPPED, ChangeTable, PackedBatch, apply_select, change_extras, decode_spans, pack_logs,
                                   pack_select, range_requests)
from tests.test_append_packing import comment_and_link_logs, fuzz_logs
from tests.test_gpu_append import canon, engine, everything, merged
from tests.test_gpu_routes import batch_of, expected_route
from tests.test_gpu_sync import device_sync, upload_all
from tests.test_gpu_wire_forms import FORMS, upload_as
from tests.test_select_packing import oracle_spans, select_corpora, selected, wanted_logs

pytestmark = pytest.mark.gpu
A = SELECT_ADDED
PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def outputs(e, batch, logs=None):
    """Every output of a merge of `batch` on `e`: canonical spans, statuses and digests, the Patch stream, element queries, both
    span renders and, with a change table, the Change JSON of every log (with the extras of its Change logs `logs`, which a
    change without list ops needs)."""
    got = merged(e)
    out = (canon(got), got.results.tobytes(), everything(e, batch, got))
    if batch.changes is not None:
        j = e.render_changes_json(batch, range_requests(list(range(batch.n_logs))), change_extras(logs)[0] if logs is not None else None)
        out += (j[0].tobytes(), j[1].tobytes())
    return out


def uploaded(u, batch, logs=None):
    upload_as(u, batch, "plain")
    return outputs(u, batch, logs)


# ------------------------------------------------------------------------------------------------------------------
# 1. Every upload form, then a select that drops, permutes, duplicates and adds
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", ["kats", "fuzz", "quirks", "early-actor", "comments-links", "sparse", "only-added", "nothing"])
def test_select_after_every_form_equals_the_upload(name, form):
    logs, from_, new_logs = select_corpora()[name]
    prev, added, cmap, want = selected(logs, from_, new_logs, with_changes=True)
    want_logs = wanted_logs(logs, from_, new_logs)
    spans = oracle_spans(want_logs)
    e, u = engine(patches=True), engine(patches=True)
    try:
        keep = upload_as(e, prev, form)
        merged(e)
        e.select_logs(from_, added if len(new_logs) else None, cmap)
        del keep
        assert e.n_logs == want.n_logs
        got = outputs(e, want, want_logs)
        assert got == uploaded(u, want, want_logs), (name, form)
        ref, _ = replay_packed(want)
        out = merged(e)
        assert canon(out) == canon(ref)
        for i in range(want.n_logs):
            assert decode_spans(want, out, i) == spans[i], (name, form, i)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. Route crossings: the plan and the key records are rebuilt
# ------------------------------------------------------------------------------------------------------------------
def test_selects_that_cross_routes():
    from tests.test_gpu_append import route_crossings
    big = batch_of([lg for lg, _ in route_crossings()])              # a warp-past log, a team log, a spill-bin log
    small = pack_logs(fuzz_logs()[:4])                               # warp-route logs
    assert all(expected_route(d) in ("packed3", "compact", "direct") for d in small.desc)
    assert any(expected_route(d) not in ("packed3", "compact", "direct") for d in big.desc)
    e, u = engine(), engine()
    try:
        cases = [(small, [A, 0, A, 3], PackedBatch(big.desc[[0, 2]].copy(), big.insdel, big.marks)),   # big logs join a warp-only batch
                 (big, [2, 0], None),                                                                 # keep only CTA-route logs
                 (big, [1, 1, 0], None)]                                                              # fork across the team kernel
        for prev, from_, added in cases:
            e.upload(prev)
            merged(e)
            e.select_logs(from_, added)
            want = apply_select(prev, from_, added)
            got = merged(e)
            u.upload(want)
            ref = merged(u)
            assert canon(got) == canon(ref) and got.results.tobytes() == ref.results.tobytes(), from_
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. State that lives only on the device: change, sync, then a select and a new peer that syncs
# ------------------------------------------------------------------------------------------------------------------
def test_device_only_state_and_a_new_replica_that_syncs():
    from oracle.oracle import Micromerge as O
    from tests.harness import generateDocs
    docs = []
    for d, text in enumerate(["abcd", "efghij", "klm"]):
        reps, _, init = generateDocs(O, text, 2)
        c = reps[1].change([{"path": ["text"], "action": "insert", "index": 1, "values": list("xy"[: 1 + d % 2])}])["change"]
        c2 = reps[0].change([{"path": ["text"], "action": "delete", "index": 0, "count": 1}])["change"]
        docs.append(([init, c2], [init, c]))
    logs = [lg for pair in docs for lg in pair]                       # document d: logs 2d, 2d + 1
    cur = pack_logs(logs, with_changes=True)
    e, u = engine(patches=True), engine(patches=True)
    try:
        upload_all(e, cur)
        merged(e)
        for pairs in ([(0, 1), (1, 0), (2, 3)], [(3, 2), (4, 5), (5, 4)]):          # two sync rounds on the device
            cur, status, _ = device_sync(e, cur, pairs)
            merged(e)
        # retire document 1, fork log 0, add an empty replica with its own actor id, then sync document 0 into it
        newcomer = [[]]
        from_ = [0, 1, 0, 4, 5, A]
        added, cmap = pack_select(cur, from_, newcomer, with_changes=True)
        added.log_actors = [["peer-new"]]                             # the new peer's own actor id
        e.select_logs(from_, added, cmap)
        cur = apply_select(cur, from_, added, cmap)
        assert e.actors() == [list(a) for a in cur.log_actors]
        assert outputs(e, cur) == uploaded(u, cur)
        cur, status, _ = device_sync(e, cur, [(0, 5), (1, 2)])
        assert outputs(e, cur) == uploaded(u, cur)
        out = merged(e)
        assert (out.results["status"] == 0).all()
        dig = out.results["digest"]
        assert (dig[5] == dig[0]).all() and (dig[2] == dig[1]).all() and (dig[0] == dig[1]).all()
        # the Change JSON renders with the downloaded tables (device_sync checked them against the specification)
        assert "peer-new" in e.actors()[5]
        held = PackedBatch(cur.desc, cur.insdel, cur.marks, cur.values, cur.link_attrs, cur.comment_ids, cur.other_attrs, cur.meta,
                           e.actors(), cur.log_counters, cur.changes, cur.log_lists)
        req = range_requests(list(range(cur.n_logs)))
        a, b = e.render_changes_json(held, req), e.render_changes_json(cur, req)
        assert a[0].tobytes() == b[0].tobytes() and len(a[0])
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Change tables follow their logs
# ------------------------------------------------------------------------------------------------------------------
def test_admission_statuses_follow_their_logs():
    logs = fuzz_logs()[:4]
    prev = pack_logs(logs, with_changes=True)
    bad = ChangeTable(prev.changes.desc.copy(), prev.changes.changes.copy(), prev.changes.deps.copy())
    k = int(bad.desc[1]["change_off"]) + 2
    bad.changes[k]["seq"] += 7                                        # log 1: a sequence gap at its change 2
    prev.changes = bad
    added, cmap = pack_select(prev, [A], [logs[2]], with_changes=True)
    gap = ChangeTable(added.changes.desc.copy(), added.changes.changes.copy(), added.changes.deps.copy())
    gap.changes[1]["seq"] += 3                                        # the added log: a gap at its change 1
    added.changes = gap
    from_ = [3, 1, A, 1]
    e, u = engine(), engine()
    try:
        upload_as(e, prev, "plain")
        before = merged(e)
        assert int(before.results[1]["status"]) == 6 and int(before.results[1]["n_elems"]) == 2
        e.select_logs(from_, added, cmap)
        want = apply_select(prev, from_, added, cmap)
        got = merged(e)
        st = [(int(r["status"]), int(r["n_elems"])) for r in got.results]
        assert st[1] == st[3] == (6, 2) and st[2] == (6, 1) and st[0][0] == 0
        upload_as(u, want, "plain")
        assert canon(got) == canon(merged(u))
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 5-6. Comment maps and refusals
# ------------------------------------------------------------------------------------------------------------------
def test_comment_map_drops_a_rank_and_refuses_a_kept_one():
    from peritext_b200.engine import EngineError
    logs, _ = comment_and_link_logs()                                 # c-d is named only by log 0
    prev = pack_logs(logs, with_changes=True)
    e, u = engine(patches=True), engine(patches=True)
    try:
        upload_as(e, prev, "plain")
        before = outputs(e, prev)
        for cm in ([0, 1, SELECT_DROPPED], [0, 1]):                    # log 0 kept: a dropped rank, a rank outside the map
            with pytest.raises(EngineError) as err:
                e.select_logs([1, 0], None, cm)
            assert err.value.status == PT_ERR_INVALID
            assert outputs(e, prev) == before
        e.select_logs([1, 1], None, [0, 1, SELECT_DROPPED])
        want = apply_select(prev, [1, 1], None, [0, 1, SELECT_DROPPED])
        assert [c["id"] for c in want.comment_ids] == ["c-b", "c-c"]
        assert outputs(e, want) == uploaded(u, want)
    finally:
        e.close(); u.close()


def raw_select(e, from_, added=None, changes=None, actors=None, cm=None, n=None):
    """pt_batch_select_logs with exactly the given structs (None = NULL)."""
    import ctypes
    from peritext_b200.engine import _ptr
    frm = np.ascontiguousarray(from_, np.uint32)
    ref = lambda s: ctypes.byref(s) if s is not None else None
    c = None if cm is None else np.ascontiguousarray(cm, np.uint32)
    return e._L.pt_batch_select_logs(e._h, _ptr(frm), len(frm) if n is None else n, ref(added), ref(changes), ref(actors),
                                     None if c is None else c.ctypes.data, 0 if c is None else len(c))


def test_refusals_leave_the_batch_untouched():
    from peritext_b200.engine import EngineError, _ActorTables, _change_struct, _packed_ops
    from peritext_b200.packing import string_pools
    logs = fuzz_logs()[:3]
    prev = pack_logs(logs, with_changes=True)
    added, _ = pack_select(prev, [A], [logs[0]], with_changes=True)
    desc, ins, mk = np.ascontiguousarray(added.desc), np.ascontiguousarray(added.insdel), np.ascontiguousarray(added.marks)
    ops = _packed_ops(desc, ins, len(ins), mk, len(mk))
    far = desc.copy(); far["insdel_off"] += 1000
    ops_far = _packed_ops(far, ins, len(ins), mk, len(mk))
    ct, _k1 = _change_struct(added.changes)
    p = string_pools(added)
    acts = [np.ascontiguousarray(p[k], dt) for k, dt in (("actors", np.uint8), ("actors_off", np.uint64), ("actors_first", np.uint64))]
    at = _ActorTables(1, _ptr_of(acts[0]), _ptr_of(acts[1]), len(acts[1]) - 1, _ptr_of(acts[2]), None)
    bad_first = np.array([0, len(acts[1])], np.uint64)               # per_log_first does not end at count
    at_bad = _ActorTables(1, _ptr_of(acts[0]), _ptr_of(acts[1]), len(acts[1]) - 1, _ptr_of(bad_first), None)
    e, u = engine(patches=True), engine(patches=True)
    try:
        upload_as(e, prev, "plain")
        e.upload_actors(prev)
        e.set_patch_window([1] * prev.n_logs)
        before = outputs(e, prev, logs)
        cases = {
            "index past the batch": dict(from_=[0, 3]),
            "added count": dict(from_=[0, A, A], added=ops, changes=ct, actors=at),
            "added descriptor": dict(from_=[A], added=ops_far, changes=ct, actors=at),
            "change table on one side": dict(from_=[A], added=ops, actors=at),
            "actor tables on one side": dict(from_=[A], added=ops, changes=ct),
            "bad actor tables": dict(from_=[A], added=ops, changes=ct, actors=at_bad),
            "comment map order": dict(from_=[0], cm=[1, 0]),
            "null from": dict(from_=[], n=2),
        }
        for name, kw in cases.items():
            assert raw_select(e, **kw) == PT_ERR_INVALID, name
            assert outputs(e, prev, logs) == before, name
        assert e.patch_window is not None
        e.select_logs([2, A], added)
        assert e.patch_window is None
        want = apply_select(prev, [2, A], added)
        assert e.actors() == [list(a) for a in want.log_actors]
        assert outputs(e, want, [logs[2], logs[0]]) == uploaded(u, want, [logs[2], logs[0]])
        f = engine()
        try:
            with pytest.raises(EngineError) as err:
                f.select_logs([])
            assert err.value.status == PT_ERR_STATE
        finally:
            f.close()
    finally:
        e.close(); u.close()


def _ptr_of(a):
    return a.ctypes.data if a.size else None


def test_pool_settings_persist_and_zero_logs():
    logs = fuzz_logs()[:3]
    prev = pack_logs(logs)
    e = engine(patches=True)
    try:
        e.set_patch_pool(1)                                          # too small: the merge reports the demand
        e.upload(prev)
        e.merge()
        _, items, _, need = e.download_patches()
        assert need > 1 and len(items) <= 1
        e.select_logs([0, 1, 2])
        e.merge()
        _, items, _, again = e.download_patches()
        assert again == need and len(items) <= 1                    # the one-item pool persisted across the select
        e.select_logs([])
        e.merge()
        assert len(e.results()) == 0
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 7. Full size: c4 with 300 000 logs, 1 % retired and 1 % admitted
# ------------------------------------------------------------------------------------------------------------------
def test_c4_300k_logs_retire_and_admit_one_percent():
    full = workload.generate("c4", n_docs=101_000, ops_per_doc=120)
    R = int(full.meta["replicas"])
    n_docs = full.n_logs // R
    resident, fresh = full.slice_logs(0, 100_000 * R), full.slice_logs(100_000 * R, 101_000 * R)
    assert resident.n_logs >= 300_000
    retired = set(range(0, 100_000, 100))                            # 1 % of the documents, every replica of each
    from_ = [d * R + r for d in range(100_000) if d not in retired for r in range(R)] + [A] * fresh.n_logs
    want = apply_select(resident, from_, fresh)
    e = engine()
    try:
        e.upload(resident)
        merged(e)
        e.select_logs(from_, fresh)
        e.merge()
        got = e.results()
        e.upload(want)
        e.merge()
        ref = e.results()
        assert got.tobytes() == ref.tobytes()
        assert (ref["status"] == 0).all()
    finally:
        e.close()
