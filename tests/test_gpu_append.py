"""pt_batch_append on the device: after an append the handle must hold exactly the batch an upload of the concatenated logs
would hold, so every output of a merge after it equals the output of that upload.

The expected batch is always ``packing.apply_append`` (the host specification of the splice), which
tests/test_append_packing.py pins against ``pack_logs`` of the full Change logs.  Batches built from records (the route
and status builders, generated workloads) are split record-wise: each log's first k ins/del records and the marks that
arrived before them stay resident, the rest is the delta, with identity maps or with maps chosen here."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200 import workload
from peritext_b200.packing import (DESC_DT, AppendRemap, ChangeTable, PackedBatch, apply_append, decode_spans, pack_append, pack_logs,
                                   split_records)
from tests.test_append_packing import (assert_same_batch, comment_and_link_logs, early_actor_logs, fraction_splits, fuzz_logs, kat_logs, quirk_logs, sparse_logs,
                                       split)
from tests.test_gpu_routes import (COMMENT, STRONG, Log, batch_of, expected_route, marks_over, status_matrix, typing_forward)
from tests.test_gpu_wire_forms import FORMS, upload_as

PT_ERR_INVALID, PT_ERR_STATE = 1, 4


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def engine(patches=False):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_patches=patches)


def merged(e):
    e.merge()
    return e._download_with_pool_retry()


def canon(out):
    return [out.canonical(i) for i in range(len(out.results))]


def oracle_spans(logs):
    """getTextWithFormatting of each full Change log replayed by the oracle."""
    out = []
    for lg in logs:
        m = O("~reader")
        for ch in lg:
            m.applyChange(ch)
        out.append(m.getTextWithFormatting())
    return out


def everything(e, batch, out):
    """The merge's outputs that read the records again: Patch stream, element queries, both JSON renders."""
    recs, items, status, _ = e.download_patches()
    order = np.lexsort((items["b"], items["a"], items["tag"], items["log"])) if len(items) else np.zeros(0, np.int64)
    ok = [i for i in range(batch.n_logs) if out.results[i]["status"] == 0]
    logs = np.array([i for i in ok for _ in range(int(out.results[i]["n_visible"]) + 1)], np.uint32)
    idx = np.array([k for i in ok for k in range(int(out.results[i]["n_visible"]) + 1)], np.uint32)
    q = e.query_elements(logs, idx, look_after_tombstones=True) if len(logs) else np.zeros(0, np.uint32)
    ins = batch.insdel
    li = np.repeat(np.arange(batch.n_logs), batch.desc["n_insdel"].astype(np.int64))
    f = e.find_elements(li, ins["ctr"], ins["actor"]) if len(ins) else np.zeros(0)
    return (recs.tobytes(), items[order].tobytes(), status.tobytes(), q.tobytes(), np.asarray(f).tobytes(),
            e.render_json_list(batch), e.render_patches_json_list(batch))


def append(e, delta, remap=None, changes=None):
    e.append(delta, remap, changes)


def record_split(batch, cuts):
    """(prefix, delta) of a record-built batch: log i keeps its first cuts[i] ins/del records and the marks that arrived
    before them.  The prefix's max_ctr is the largest counter its records name, the delta's descriptors are the full log's, so
    the identity maps apply."""
    from peritext_b200.packing import _excl_scan, _ranges
    d = batch.desc
    n_ins = d["n_insdel"].astype(np.int64)
    cuts = np.minimum(np.asarray(cuts, np.int64), n_ins)
    m_pre = np.zeros(batch.n_logs, np.int64)
    max_pre = np.zeros(batch.n_logs, np.int64)
    for i in range(batch.n_logs):
        ins, mk = batch.log_slice(i)
        assert (np.diff(mk["arrival"].astype(np.int64)) >= 0).all()
        m_pre[i] = int((mk["arrival"] < cuts[i]).sum())
        used = [ins["ctr"][:cuts[i]], ins["ref_ctr"][:cuts[i]]] + [mk[f][:m_pre[i]] for f in ("ctr", "start_ctr", "end_ctr")]
        max_pre[i] = max([0] + [int(u.max()) for u in used if len(u)])
    max_pre = np.minimum(max_pre, d["max_ctr"].astype(np.int64))     # a faulty record may name more than the descriptor

    def part(first_ins, cnt_ins, first_mk, cnt_mk, max_ctr):
        desc = np.zeros(batch.n_logs, DESC_DT)
        desc["n_insdel"], desc["n_mark"] = cnt_ins, cnt_mk
        desc["insdel_off"], desc["mark_off"] = _excl_scan(cnt_ins), _excl_scan(cnt_mk)
        desc["n_actors"], desc["max_ctr"] = d["n_actors"], max_ctr
        return PackedBatch(desc, batch.insdel[_ranges(d["insdel_off"].astype(np.int64) + first_ins, cnt_ins)],
                           batch.marks[_ranges(d["mark_off"].astype(np.int64) + first_mk, cnt_mk)], batch.values, batch.link_attrs,
                           batch.comment_ids, batch.other_attrs)
    pre = part(np.zeros_like(cuts), cuts, np.zeros_like(m_pre), m_pre, max_pre)
    delta = part(cuts, n_ins - cuts, m_pre, d["n_mark"].astype(np.int64) - m_pre, d["max_ctr"])
    return pre, delta


# ------------------------------------------------------------------------------------------------------------------
# 1. Change logs through every upload form
# ------------------------------------------------------------------------------------------------------------------
def change_corpora():
    out = {"kats": (kat_logs(), None), "fuzz": (fuzz_logs(), None), "quirks": (quirk_logs(), [1]), "early-actor": (early_actor_logs(), [2, 1])}
    logs, ks = comment_and_link_logs(); out["comments-links"] = (logs, ks)
    logs, ks = sparse_logs(); out["sparse"] = (logs, ks)
    return out


_CORPORA = None


def corpora():
    global _CORPORA
    if _CORPORA is None:
        _CORPORA = change_corpora()
    return _CORPORA


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", ["kats", "fuzz", "quirks", "early-actor", "comments-links", "sparse"])
def test_append_after_every_form_equals_the_upload(name, form):
    logs, ks = corpora()[name]
    splits = [ks] if ks is not None else fraction_splits(logs, (0.0, 0.5))[:2] + [fraction_splits(logs)[-1]]
    want_spans = oracle_spans(logs)
    e, u = engine(patches=True), engine(patches=True)
    try:
        for cut in splits:
            prefix, suffix = split(logs, cut)
            prev = pack_logs(prefix)
            delta, remap = pack_append(prev, suffix)
            full = apply_append(prev, delta, remap)
            keep = upload_as(e, prev, form)
            merged(e)
            append(e, delta, remap)
            del keep
            got = merged(e)
            u.upload(full)
            want = merged(u)
            assert canon(got) == canon(want), (name, form, cut)
            ref, _ = replay_packed(full)
            assert canon(got) == canon(ref), (name, form, cut)
            for i in range(full.n_logs):
                assert decode_spans(full, got, i) == want_spans[i], (name, form, cut, i)
            assert everything(e, full, got) == everything(u, full, want), (name, form, cut)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2-3. Chains, empty deltas, one log of many
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_three_chained_appends_equal_one_upload():
    logs = fuzz_logs()
    cuts = [[int(f * len(lg)) for lg in logs] for f in (0.25, 0.5, 0.75, 1.0)]
    cur = pack_logs([lg[:k] for lg, k in zip(logs, cuts[0])])
    e, u = engine(patches=True), engine(patches=True)
    try:
        e.upload(cur)
        for a, b in zip(cuts, cuts[1:]):
            delta, remap = pack_append(cur, [lg[x:y] for lg, x, y in zip(logs, a, b)])
            append(e, delta, remap)
            cur = apply_append(cur, delta, remap)
        got = merged(e)
        u.upload(cur)
        want = merged(u)
        assert canon(got) == canon(want)
        assert everything(e, cur, got) == everything(u, cur, want)
        assert_same_batch(cur, pack_logs(logs))               # the batch of one pack, up to pool order
        spans = oracle_spans(logs)
        assert [decode_spans(cur, got, i) for i in range(cur.n_logs)] == spans
    finally:
        e.close(); u.close()


@pytest.mark.gpu
def test_empty_delta_and_one_log_of_many():
    logs = fuzz_logs()
    prev = pack_logs(logs)
    e = engine(patches=True)
    try:
        e.upload(prev)
        before = merged(e)
        b_all = everything(e, prev, before)
        delta, remap = pack_append(prev, [[] for _ in logs])
        append(e, delta, remap)
        after = merged(e)
        assert canon(after) == canon(before) and everything(e, prev, after) == b_all
        # one log of many gains the second half of its changes
        j = len(logs) // 2
        cut = [len(lg) if i != j else len(lg) // 2 for i, lg in enumerate(logs)]
        prefix, suffix = split(logs, cut)
        p2 = pack_logs(prefix)
        d2, r2 = pack_append(p2, suffix)
        assert sum(int(x) for x in d2.desc["n_insdel"] + d2.desc["n_mark"]) == int(d2.desc[j]["n_insdel"]) + int(d2.desc[j]["n_mark"]) > 0
        e.upload(p2)
        append(e, d2, r2)
        got = merged(e)
        assert canon(got) == canon(replay_packed(apply_append(p2, d2, r2))[0])
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Appends that move a log across routes
# ------------------------------------------------------------------------------------------------------------------
def route_crossings():
    """(log, cut, prefix route, full route): past the warp kernel's 2048 records, a team log gaining its first mark, and a log
    growing into the spill-capable size."""
    warp = Log(3)
    typing_forward(warp, 2400, [0, 1, 2])
    team = Log(4)
    ids = typing_forward(team, 3000, [0, 1, 2, 3])
    team.mark(1, STRONG, ids[10], ids[900])
    team.mark(2, COMMENT, ids[5], ids[2000], attr=1)
    spill = Log(2)
    ids = typing_forward(spill, 40000, [0, 1])
    marks_over(spill, ids, 300, seed=5)
    return [(warp, 600), (team, 3000), (spill, 6000)]


@pytest.mark.gpu
def test_appends_that_cross_routes():
    cases = route_crossings()
    full = batch_of([lg for lg, _ in cases])
    pre, delta = record_split(full, [k for _, k in cases])
    moved = [(expected_route(pre.desc[i]), expected_route(full.desc[i])) for i in range(full.n_logs)]
    assert moved[0][0] in ("packed3", "compact", "direct") and moved[0][1] not in ("packed3", "compact", "direct"), moved
    assert moved[1] == ("team", "cta2-u16") or (moved[1][0] == "team" and moved[1][1] != "team"), moved
    assert moved[2][0] != "cta4-u32" and moved[2][1] == "cta4-u32", moved          # the last bin: the only one that can spill
    want_batch = apply_append(pre, delta)
    assert want_batch.insdel.tobytes() == full.insdel.tobytes() and want_batch.marks.tobytes() == full.marks.tobytes()
    ref, _ = replay_packed(full)
    for form in ("plain", "adopt"):
        e = engine()
        try:
            keep = upload_as(e, pre, form)
            merged(e)
            append(e, delta)
            del keep
            got = merged(e)
            assert canon(got) == canon(ref), form
        finally:
            e.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. Change tables
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_change_tables_admit_resident_deps_and_report_gaps_at_the_full_index():
    logs = fuzz_logs()
    cut = [len(lg) // 2 for lg in logs]
    prefix, suffix = split(logs, cut)
    prev = pack_logs(prefix, with_changes=True)
    delta, remap = pack_append(prev, suffix, with_changes=True)
    e, u = engine(), engine()
    try:
        e.run(prev)
        append(e, delta, remap)
        got = merged(e)
        assert (got.results["status"] == 0).all()            # every suffix change's deps are resident changes
        assert any(len(c["deps"]) for lg in suffix for c in lg)
        full = apply_append(prev, delta, remap)
        assert canon(got) == canon(u.run(full))
        # a sequence gap in the delta of log j: reported with the index of the change in the whole log
        j = 1
        bad = ChangeTable(delta.changes.desc.copy(), delta.changes.changes.copy(), delta.changes.deps.copy())
        k = int(bad.desc[j]["change_off"]) + 1
        bad.changes[k]["seq"] += 5
        e.run(prev)
        append(e, delta, remap, changes=bad)
        got = merged(e)
        assert int(got.results[j]["status"]) == 6 and int(got.results[j]["n_elems"]) == int(prev.changes.desc[j]["n_changes"]) + 1
        tampered = apply_append(prev, PackedBatch(delta.desc, delta.insdel, delta.marks, delta.values, delta.link_attrs, delta.comment_ids,
                                                  delta.other_attrs, log_actors=delta.log_actors, log_counters=delta.log_counters, changes=bad), remap)
        assert canon(got) == canon(u.run(tampered))
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 6. Faulty logs through identity and non-identity maps
# ------------------------------------------------------------------------------------------------------------------
def shifted_remap(pre):
    """Every log gains an actor that sorts first (old rank r -> r + 1) and its counters double (c -> 2c)."""
    n = pre.n_logs
    na = pre.desc["n_actors"].astype(np.int64); nc = pre.desc["max_ctr"].astype(np.int64) + 1
    aoff = np.concatenate([[0], np.cumsum(na)]).astype(np.uint64)
    coff = np.concatenate([[0], np.cumsum(nc)]).astype(np.uint64)
    amap = np.concatenate([np.arange(a) + 1 for a in na] + [np.zeros(0)]).astype(np.uint16)
    cmap = np.concatenate([2 * np.arange(c) for c in nc] + [np.zeros(0)]).astype(np.uint32)
    return AppendRemap(aoff, amap, coff, cmap, None), n


@pytest.mark.gpu
def test_status_corpus_through_identity_and_shifting_maps():
    rows, full = status_matrix()
    pre, delta = record_split(full, (full.desc["n_insdel"].astype(np.int64) * 2) // 3)
    remap, _ = shifted_remap(pre)
    grown = PackedBatch(delta.desc.copy(), delta.insdel, delta.marks, delta.values, delta.link_attrs, delta.comment_ids)
    grown.desc["n_actors"] += 1; grown.desc["max_ctr"] *= 2       # the delta keeps old-space ids: those records turn faulty too
    e, u = engine(), engine()
    try:
        for dl, rm in ((delta, None), (grown, remap)):
            want = apply_append(pre, dl, rm)
            e.upload(pre)
            merged(e)
            append(e, dl, rm)
            got = merged(e)
            ref = merged_upload(u, want)
            assert canon(got) == canon(ref), rm is None
        # identity maps: the statuses are the full batch's
        assert [int(s) for s in merged_upload(u, apply_append(pre, delta)).results["status"]] == [int(s) for s in merged_upload(u, full).results["status"]]
    finally:
        e.close(); u.close()


def merged_upload(u, batch):
    u.upload(batch)
    return merged(u)


# ------------------------------------------------------------------------------------------------------------------
# 7. Refusals
# ------------------------------------------------------------------------------------------------------------------
def refusal_cases(prev, delta, remap):
    """name -> (delta, remap, change table or None) that pt_batch_append must refuse (the logs have one actor each)."""
    n = prev.n_logs
    m0 = int(prev.desc[0]["max_ctr"]) + 1
    ident = np.arange(m0).astype(np.uint32)
    swapped = ident.copy(); swapped[[1, 2]] = swapped[[2, 1]]

    def with_remap(**kw):
        r = AppendRemap(remap.actor_off, remap.actor_map, remap.ctr_off, remap.ctr_map, remap.comment_map)
        for k, v in kw.items():
            setattr(r, k, v)
        return delta, r, delta.changes

    log0 = lambda k: np.array([0] + [k] * n, np.uint64)      # log 0 gets k entries, the others none
    late = PackedBatch(delta.desc, delta.insdel, delta.marks.copy())
    late.marks["arrival"] = 0
    return {
        "n_logs": (PackedBatch(delta.desc[:1].copy(), delta.insdel[:0], delta.marks[:0]), None, delta.changes.slice_logs(0, 1)),
        "actor map length": with_remap(actor_off=log0(2), actor_map=np.array([0, 1], np.uint16)),
        "actor bound": with_remap(actor_off=log0(1), actor_map=np.array([5], np.uint16)),
        "ctr map order": with_remap(ctr_off=log0(m0), ctr_map=swapped),
        "ctr_map[0]": with_remap(ctr_off=log0(m0), ctr_map=ident + 1),
        "ctr bound": with_remap(ctr_off=log0(m0), ctr_map=ident * 1000),
        "arrival": (late, remap, delta.changes),
        "comment rank on the device": with_remap(comment_map=np.array([0], np.uint32)),      # rank 1 (c-d) is outside
    }


@pytest.mark.gpu
def test_refusals_leave_the_batch_untouched():
    from peritext_b200.engine import EngineError
    logs, ks = comment_and_link_logs()
    prefix, suffix = split(logs, ks)
    prev = pack_logs(prefix, with_changes=True)
    delta, remap = pack_append(prev, suffix, with_changes=True)
    assert remap.comment_map is not None and len(delta.marks)
    e = engine(patches=True)
    try:
        e.run(prev)
        before = canon(merged(e))
        before_all = everything(e, prev, merged(e))
        for name, (d, r, t) in refusal_cases(prev, delta, remap).items():
            with pytest.raises(EngineError, match="invalid argument"):
                e.append(d, r, t)
            assert canon(merged(e)) == before, name
        assert no_table_append(e, delta, remap) == PT_ERR_INVALID
        assert canon(merged(e)) == before
        assert everything(e, prev, merged(e)) == before_all
        e.append(delta, remap)                                  # the valid append still goes through afterwards
        assert canon(merged(e)) == canon(replay_packed(apply_append(prev, delta, remap))[0])
        f = engine()
        try:
            with pytest.raises(EngineError, match="call out of order"):
                f.append(delta, remap)
        finally:
            f.close()
    finally:
        e.close()


def no_table_append(e, d, r):
    """pt_batch_append with no delta change table (NULL) on a handle that has one."""
    import ctypes
    from peritext_b200.engine import _AppendRemap, _packed_ops
    desc, ins, mk = np.ascontiguousarray(d.desc), np.ascontiguousarray(d.insdel), np.ascontiguousarray(d.marks)
    ops = _packed_ops(desc, ins, len(ins), mk, len(mk))
    st = _AppendRemap(None, None, None, None, None, 0)          # identity maps: only the missing table is wrong
    return e._L.pt_batch_append(e._h, ctypes.byref(ops), ctypes.byref(st), None)


@pytest.mark.gpu
def test_an_empty_comment_map_is_not_the_identity():
    """pt_append_remap: a NULL comment_map is the identity, an empty one maps no comment rank, so on a batch with comment marks
    the device refuses the append."""
    from peritext_b200.engine import EngineError
    logs, ks = comment_and_link_logs()
    prev = pack_logs(split(logs, ks)[0], with_changes=True)
    assert (prev.marks["kind"] >> 1 & 3 == 2).any()                   # a comment mark
    delta, _ = pack_append(prev, [[] for _ in logs], with_changes=True)
    e = engine()
    try:
        e.run(prev)
        before = canon(merged(e))
        with pytest.raises(EngineError) as err:
            e.append(delta, AppendRemap(comment_map=np.zeros(0, np.uint32)))
        assert err.value.status == PT_ERR_INVALID
        assert canon(merged(e)) == before
        e.append(delta, AppendRemap())
        assert canon(merged(e)) == before
    finally:
        e.close()


@pytest.mark.gpu
def test_patch_records_after_splicing_an_upload_with_slack():
    """An upload whose ins/del array holds one record no descriptor covers has one patch record per uploaded record; the splice
    of an append rebuilds the records from the descriptors, so afterwards there is one per record of the spliced batch."""
    import copy
    logs, ks = comment_and_link_logs()
    prefix, suffix = split(logs, ks)
    prev = pack_logs(prefix)
    delta, remap = pack_append(prev, suffix)
    slack = copy.copy(prev)
    slack.insdel = np.concatenate([prev.insdel, prev.insdel[-1:]])
    want = apply_append(prev, delta, remap)
    e, u = engine(patches=True), engine(patches=True)
    try:
        e.upload(slack); e.merge()
        assert len(e.download_patches()[0]) == len(slack.insdel)
        e.append(delta, remap); e.merge()
        recs = e.download_patches()[0]
        assert len(recs) == len(want.insdel)
        u.upload(want); u.merge()
        assert recs.tobytes() == u.download_patches()[0].tobytes()
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 8. A c4-shaped batch of 300 000 logs with a 1 % suffix
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c4_300k_logs_one_percent_suffix():
    full = workload.generate("c4", n_docs=100_000, ops_per_doc=120)
    assert full.n_logs >= 300_000
    n_ins = full.desc["n_insdel"].astype(np.int64)
    pre, delta = split_records(full, (n_ins * 99) // 100)
    e = engine()
    try:
        e.upload(pre)
        merged(e)
        append(e, delta)
        e.merge()
        got = e.results()
        e.upload(full)
        e.merge()
        want = e.results()
        assert got.tobytes() == want.tobytes()
        assert (want["status"] == 0).all()
    finally:
        e.close()


@pytest.mark.gpu
def test_refusals_of_actor_order_and_a_one_sided_change_table():
    """An actor map that is not strictly increasing, and a delta change table for a batch without one: refused, and a merge
    right after equals the merge before."""
    from peritext_b200.engine import EngineError
    logs = fuzz_logs()[:3]
    prefix, suffix = split(logs, [len(lg) // 2 for lg in logs])
    prev = pack_logs(prefix)
    delta, remap = pack_append(prev, suffix)
    with_table, _ = pack_append(pack_logs(prefix, with_changes=True), suffix, with_changes=True)
    na = [int(x) for x in prev.desc["n_actors"]]
    assert na[0] >= 2
    bad_order = np.concatenate([np.arange(a)[::-1] if i == 0 else np.arange(a) for i, a in enumerate(na)]).astype(np.uint16)
    r = AppendRemap(np.concatenate([[0], np.cumsum(na)]).astype(np.uint64), bad_order, remap.ctr_off, remap.ctr_map, remap.comment_map)
    e = engine()
    try:
        e.upload(prev)
        before = canon(merged(e))
        for name, (d, rm, t) in {"actor map order": (delta, r, None), "change table on the delta only": (delta, remap, with_table.changes)}.items():
            with pytest.raises(EngineError, match="invalid argument"):
                e.append(d, rm, t)
            assert canon(merged(e)) == before, name
    finally:
        e.close()
