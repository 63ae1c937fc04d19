"""pt_batch_restore on the device.  Each request's appended records and change record must equal what pt_batch_change generates
on a twin handle from the specification's InputOperations (``restore.restore_inputs``, as runs of value tokens) under the
specification's change record (``restore.restore_change_record``): the twins' merges, Patch streams and Change JSON are
compared byte for byte.  After the restore and a merge, every restored log's visible text is its version's, and the new change
rendered as Change JSON applies in the oracle.  tests/test_restore_spec.py pins the specification against the oracle's change()."""
import json

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import (CHANGE_NO_ACTOR, DESC_DT, INPUT_OP_DT, INSDEL_DT, PackedBatch, apply_append, apply_checkout,
                                   decode_spans, pack_logs, range_requests)
from peritext_b200.restore import (RESTORE, RESTORE_BAD_TABLE, RESTORE_FOREIGN, RESTORE_LOG_FAILED, RESTORE_MARKS, RESTORE_OK,
                                   RESTORE_TEXT_DIFFERS, restore_change_table, restore_inputs, restore_mark_records, restore_tokens)
from tests.test_append_packing import kat_logs, sparse_logs
from peritext_b200.packing import canon as canon_json
from tests.harness import generateDocs
from tests.test_attribution_spec import deletes_cases
from tests.test_checkout_model import SESSIONS, session
from tests.test_gpu_append import canon, merged
from tests.test_gpu_wire_forms import FORMS, upload_as
from tests.test_restore_spec import tombstone_boundary_log

pytestmark = pytest.mark.gpu
PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_patches=True, **kw)


def text_of(batch, got, i):
    return "".join(s["text"] for s in decode_spans(batch, got, i))


def checkout_all(e, batch, n_changes):
    """Every log checked out at n_changes[i] on the device; the host batch of the same.  Returns (batch, its merge)."""
    logs = list(range(batch.n_logs))
    assert (e.checkout(logs, n_changes=n_changes) == 0).all()
    co, st = apply_checkout(batch, logs, n_changes=n_changes)
    assert (st == 0).all()
    return co, merged(e)


def requests_for(co, pairs):
    """(log, version, actor = the log's newest change's actor, first_ctr = max_ctr + 1) per (log, version) pair."""
    out = []
    for log, ver in pairs:
        cd = co.changes.desc[log]
        a = int(co.changes.changes[int(cd["change_off"]) + int(cd["n_changes"]) - 1]["actor"]) if int(cd["n_changes"]) else 0
        out.append((log, ver, a, int(co.desc[log]["max_ctr"]) + 1))
    return out


def twin_change(u, co, got, reqs, n_ops):
    """The specification's InputOperations of every OK request through pt_batch_change on twin handle `u` (merged over co)."""
    n = co.n_logs
    actor = np.full(n, CHANGE_NO_ACTOR, np.uint32)
    per = {}
    for (log, ver, a, f), k in zip(reqs, n_ops):
        if int(k):
            actor[log] = a
            per[log] = (restore_tokens(co, got, log, ver), f)
    rows, toks, off = [], [], np.zeros(n + 1, np.uint64)
    for i in range(n):
        if i in per:
            runs, f = per[i]
            for action, v, arg in runs:
                if action == RESTORE:
                    rows.append((0, 0, 0, v, len(arg), 0xFFFFFFFF, f, 0, len(toks)))
                    toks += arg; f += len(arg)
                else:
                    rows.append((1, 0, 0, v, arg, 0xFFFFFFFF, f, 0, 0))
                    f += arg
        off[i + 1] = len(rows)
    ops = np.array(rows, INPUT_OP_DT) if rows else np.zeros(0, INPUT_OP_DT)
    dch = restore_change_table(co, np.array(reqs, dtype=REQ_DT), n_ops)
    st, desc, insdel, marks = u.change_packed(actor, off, ops, np.array(toks, np.uint32), len(co.values), len(co.link_attrs), len(co.comment_ids), dch)
    assert (st["status"] == 0).all()
    return apply_append(co, delta_of(co, desc, insdel, marks, dch))


REQ_DT = [("log", "<u4"), ("version", "<u4"), ("actor", "<u4"), ("first_ctr", "<u4")]


def delta_of(co, desc, insdel, marks, dch):
    return PackedBatch(desc, insdel, marks, co.values, co.link_attrs, co.comment_ids, co.other_attrs, dict(co.meta), list(co.log_actors),
                       co.log_counters, dch, list(co.log_lists))


def twin_marks(u, co, got, reqs, n_ops):
    """The specification's MARKS records of every request with ops, appended on twin `u` (merged over co) with pt_batch_append."""
    desc = np.zeros(co.n_logs, DESC_DT)
    desc["n_actors"], desc["max_ctr"] = co.desc["n_actors"], co.desc["max_ctr"]
    recs = [None] * co.n_logs
    for (log, ver, a, f), k in zip(reqs, n_ops):
        if int(k):
            st, ops = restore_inputs(co, got, log, ver, RESTORE_MARKS)
            recs[log] = restore_mark_records(co, got, log, ops, a, f)
            assert len(recs[log]) == int(k)
            desc[log]["n_mark"], desc[log]["max_ctr"] = len(ops), f + len(ops) - 1
    desc["mark_off"] = np.concatenate([[0], np.cumsum(desc["n_mark"])[:-1]]) if co.n_logs else 0
    marks = np.concatenate([r for r in recs if r is not None]) if any(r is not None for r in recs) else restore_mark_records(co, got, 0, [], 0, 0)
    dch = restore_change_table(co, np.array(reqs, dtype=REQ_DT), n_ops)
    delta = delta_of(co, desc, np.zeros(0, INSDEL_DT), marks, dch)
    u.append(delta, changes=dch)
    return apply_append(co, delta)


def new_changes(co, logs):
    """RANGE requests for the change each of `logs` appended after `co`'s table."""
    req = range_requests(logs, count=1)
    if len(logs):
        req["first"] = co.changes.desc["n_changes"][np.asarray(logs, np.int64)]
    return req


def restore_and_compare(e, u, co, got, pairs, json_logs=True):
    """Restore `pairs` on `e` and the specification on twin `u` (both merged over `co`); the checks of the module docstring.
    Returns (statuses, n_ops, seq, the merge after the restore)."""
    reqs = requests_for(co, pairs)
    want = [restore_inputs(co, got, log, ver) for log, ver in pairs]
    old_first = (co.desc["n_insdel"].astype(np.int64) + co.desc["n_mark"]).astype(np.uint32)
    st, n_ops, seq = e.restore(reqs)
    assert st.tolist() == [s for s, _ in want]
    assert [int(k) for k in n_ops] == [sum(len(op.get("values", ())) + op.get("count", 0) for op in ops) for _, ops in want]
    new = twin_change(u, co, got, reqs, n_ops)
    after, ref = merged(e), merged(u)
    assert canon(after) == canon(ref)
    if json_logs:                                   # the new changes: seq, deps in their order, opIds and references
        req = new_changes(co, [r[0] for r, k in zip(reqs, n_ops) if k])
        assert e.render_changes_json_list(co, req) == u.render_changes_json_list(co, req)
    for (log, ver), s in zip(pairs, st):
        if s == RESTORE_OK:
            assert text_of(co, after, log) == text_of(co, got, ver), (log, ver)
    # the Patches of the new ops alone, against the twin's (which pt_batch_change pins against the oracle's change())
    e.set_patch_window(old_first); u.set_patch_window(old_first)
    e.merge(); u.merge()
    assert e.render_patches_json_list(co) == u.render_patches_json_list(co)
    return st, n_ops, seq, after, new


def marks_and_compare(e, u, batch, pairs):
    """MARKS of `pairs` on `e` and the specification's records appended on twin `u` (both holding `batch`, unmerged): statuses,
    merges and the new changes' JSON equal; afterwards no OK request's log differs from its version in formatting."""
    got, ref = merged(e), merged(u)
    assert canon(got) == canon(ref)
    reqs = requests_for(batch, pairs)
    want = [restore_inputs(batch, got, log, ver, RESTORE_MARKS) for log, ver in pairs]
    st, n_ops, seq = e.restore(reqs, RESTORE_MARKS)
    assert st.tolist() == [s for s, _ in want] and n_ops.tolist() == [len(ops) for _, ops in want]
    new = twin_marks(u, batch, got, reqs, n_ops)
    after, ref = merged(e), merged(u)
    assert canon(after) == canon(ref)
    req = new_changes(batch, [r[0] for r, k in zip(reqs, n_ops) if k])
    assert e.render_changes_json_list(batch, req) == u.render_changes_json_list(batch, req)
    for (log, ver), s in zip(pairs, st):
        if s == RESTORE_OK:
            assert restore_inputs(new, after, log, ver, RESTORE_MARKS) == (RESTORE_OK, []), (log, ver)
    return st, n_ops, new, after


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("seed,kw", SESSIONS[:3])
def test_every_form_restores_every_log_to_half_its_table(seed, kw, form):
    _, logs = session(seed, kw, steps=40)
    batch = pack_logs(logs, with_changes=True)
    e, u = engine(), engine()
    try:
        keep = upload_as(e, batch, form)
        merged(e)
        del keep
        half = [int(batch.changes.desc[i]["n_changes"]) // 2 for i in range(batch.n_logs)]
        co, got = checkout_all(e, batch, half)
        upload_as(u, co, "plain")
        ref = merged(u)
        assert canon(ref) == canon(got)
        n = batch.n_logs
        st, n_ops, seq, _, new = restore_and_compare(e, u, co, got, [(i, n + i) for i in range(n)])
        assert (st == RESTORE_OK).all() and n_ops.sum() > 0
        # MARKS on the restored logs (built by the restore on the device) against the specification's records on the twin
        e.set_patch_window(); u.set_patch_window()
        marks_and_compare(e, u, new, [(i, n + i) for i in range(n)])
    finally:
        e.close(); u.close()


def test_kats_sparse_counters_concurrent_deletes_and_the_tombstone_corner():
    for logs, js in ((kat_logs(), True), (sparse_logs()[0], False), (deletes_cases(), True), ([tombstone_boundary_log()], True)):
        batch = pack_logs(logs, with_changes=True)
        e, u = engine(), engine()
        try:
            upload_as(e, batch, "plain")
            merged(e)
            n = batch.n_logs
            prefix = [max(1, int(batch.changes.desc[i]["n_changes"]) - 1 - (i % 3)) for i in range(n)]
            if n == 1:                                            # the tombstone corner: the version before the delete
                prefix = [2]
            co, got = checkout_all(e, batch, prefix)
            upload_as(u, co, "plain")
            merged(u)
            st, _, _, _, _ = restore_and_compare(e, u, co, got, [(i, n + i) for i in range(n)], json_logs=js)
            assert (st == RESTORE_OK).all()
        finally:
            e.close(); u.close()


def test_nothing_to_do_mixed_statuses_and_many_requests():
    _, logs = session(2007, SESSIONS[1][1], steps=40)
    other = kat_logs()[:2]
    batch = pack_logs(logs + other, with_changes=True)
    e, u = engine(), engine()
    try:
        upload_as(e, batch, "plain")
        merged(e)
        n = batch.n_logs
        co, got = checkout_all(e, batch, [int(batch.changes.desc[i]["n_changes"]) // 2 for i in range(n)])
        upload_as(u, co, "plain")
        merged(u)
        # itself: nothing to do; a version; a checkout restored to its source's later elements: FOREIGN (packed ids of another
        # document would collide with the log's, so a version must come from the log's own id space)
        grown = next(i for i in range(1, n) if got.results["n_elems"][i] > got.results["n_elems"][n + i])
        pairs = [(0, 0), (1, n + 1), (n + grown, grown)]
        st, n_ops, seq, _, _ = restore_and_compare(e, u, co, got, pairs)
        assert st.tolist() == [RESTORE_OK, RESTORE_OK, RESTORE_FOREIGN]
        assert n_ops[0] == 0 and seq[0] == 0 and n_ops[2] == 0 and seq[2] == 0 and n_ops[1] > 0 and seq[1] > 0
    finally:
        e.close(); u.close()
    # more requests than resident warps: many small documents, each restored to its first change
    many = [kat_logs()[0]] * 9000                                 # above 132 SMs x 16 CTAs x 4 warps
    batch = pack_logs(many, with_changes=True)
    e, u = engine(), engine()
    try:
        upload_as(e, batch, "compact")
        merged(e)
        n = batch.n_logs
        co, got = checkout_all(e, batch, [1] * n)
        upload_as(u, co, "plain")
        merged(u)
        st, n_ops, _, _, _ = restore_and_compare(e, u, co, got, [(i, n + i) for i in range(n)], json_logs=False)
        assert (st == RESTORE_OK).all()
    finally:
        e.close(); u.close()


def test_the_restore_change_syncs_to_the_oracle():
    """The new change, rendered as Change JSON, applies in the oracle on a replica of the log and gives the version's text."""
    _, logs = session(7, {}, steps=40)
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_as(e, batch, "plain")
        merged(e)
        n = batch.n_logs
        co, got = checkout_all(e, batch, [2] * n)
        reqs = requests_for(co, [(i, n + i) for i in range(n)])
        st, n_ops, seq = e.restore(reqs)
        assert (st == RESTORE_OK).all()
        rendered = e.render_changes_json_list(co, new_changes(co, list(range(n))))
        for i in range(n):
            new, = json.loads(rendered[i].decode("utf-8", "surrogatepass"))
            assert new["seq"] == int(seq[i]) and len(new["ops"]) == int(n_ops[i])
            d = O("~reader")
            for ch in logs[i] + [new]:
                d.applyChange(ch)
            v = O("~reader")
            for ch in logs[i][:2]:
                v.applyChange(ch)
            assert d.getTextWithFormatting() and "".join(s["text"] for s in d.getTextWithFormatting()) == "".join(s["text"] for s in v.getTextWithFormatting())
    finally:
        e.close()


def test_log_failed_bad_table_and_refusals_leave_the_batch_and_its_merge():
    from peritext_b200.engine import EngineError
    _, logs = session(7, {}, steps=30)
    batch = pack_logs(logs, with_changes=True)
    n = batch.n_logs
    e = engine()
    try:
        upload_as(e, batch, "plain")
        got = merged(e)
        before = canon(got)
        reqs = requests_for(batch, [(i, i) for i in range(n)])
        bad = [
            ([(n, 0, 0, 10 ** 6)], 1, PT_ERR_INVALID),                        # log outside the batch
            ([(0, n, 0, 10 ** 6)], 1, PT_ERR_INVALID),                        # version outside the batch
            ([reqs[0], reqs[0]], 1, PT_ERR_INVALID),                          # a log named twice
            ([reqs[0]], 0, PT_ERR_INVALID),                                   # mode: no flag
            ([reqs[0]], 3, PT_ERR_INVALID),                                   # mode: both flags
            ([(0, 0, 999, 10 ** 6)], 1, PT_ERR_INVALID),                      # actor
            ([(0, 0, 0, int(batch.desc[0]["max_ctr"]))], 1, PT_ERR_INVALID),  # first_ctr not above max_ctr
        ]
        for r, mode, code in bad:
            with pytest.raises(EngineError) as ex:
                e.restore(r, mode)
            assert ex.value.status == code
        import ctypes
        from peritext_b200.restore import RESTORE_REQUEST_DT, _RestoreView
        v = _RestoreView()
        one = np.array([reqs[0]], RESTORE_REQUEST_DT)
        assert e._L.pt_batch_restore(e._h, None, 1, 1, ctypes.byref(v)) == PT_ERR_INVALID       # null requests
        assert e._L.pt_batch_restore(e._h, one.ctypes.data, 1, 1, None) == PT_ERR_INVALID      # null view
        assert e._L.pt_batch_restore(e._h, one.ctypes.data, 1, 3, ctypes.byref(v)) == PT_ERR_INVALID   # both flags
        # the generated counters would pass 2^32 - 1: refused after the count pass, nothing changed
        actor0 = requests_for(batch, [(0, 0)])[0][2]
        ver = batch.n_logs
        e.checkout([0], n_changes=[1]); merged(e)
        with pytest.raises(EngineError) as ex:
            e.restore([(0, ver, actor0, 0xFFFFFFFF)])
        assert ex.value.status == PT_ERR_INVALID
        after = merged(e)
        assert canon(after)[:n] == before
        # max_ctr x n_actors would reach 2^31 (the log has 3 actors): refused after the count pass, nothing changed
        R = int(batch.desc[0]["n_actors"])
        assert R >= 2
        with pytest.raises(EngineError) as ex:
            e.restore([(0, ver, actor0, 0x7FFFFFFF // R + 1)])
        assert ex.value.status == PT_ERR_INVALID and "2^31" in str(ex.value)
        assert canon(merged(e))[:n] == before
    finally:
        e.close()
    # a status per request: LOG_FAILED (admission-rejected log), BAD_TABLE (n_ops that do not sum to the records)
    bad = pack_logs(logs, with_changes=True)
    bad.changes.changes["n_ops"][int(bad.changes.desc[1]["change_off"])] += 1
    rej = pack_logs(logs, with_changes=True)
    rej.changes.changes["seq"][int(rej.changes.desc[0]["change_off"]) + 1] += 5
    for b, want in ((bad, [RESTORE_OK, RESTORE_BAD_TABLE]), (rej, [RESTORE_LOG_FAILED, RESTORE_OK])):
        e = engine()
        try:
            upload_as(e, b, "plain")
            merged(e)
            st, n_ops, _ = e.restore(requests_for(b, [(0, 0), (1, 1)]))
            assert st.tolist() == want and (n_ops == 0).all()
        finally:
            e.close()
    # no merge since the last change to the batch, and a handle without the element sequence
    e = engine()
    try:
        upload_as(e, batch, "plain")
        with pytest.raises(EngineError) as ex:
            e.restore(requests_for(batch, [(0, 0)]))
        assert ex.value.status == PT_ERR_STATE
    finally:
        e.close()
    from peritext_b200.engine import BatchEngine
    e = BatchEngine(0)
    try:
        upload_as(e, batch, "plain")
        merged(e)
        with pytest.raises(EngineError) as ex:
            e.restore(requests_for(batch, [(0, 0)]))
        assert ex.value.status == PT_ERR_STATE
    finally:
        e.close()


def q3_normalised(batch, got, i):
    """Per visible position its canonical marks, the `comment` key without ids (quirk Q3) dropped."""
    out = []
    for sp in decode_spans(batch, got, i):
        m = {k: v for k, v in sp["marks"].items() if not (k == "comment" and v == [])}
        out += [canon_json(m)] * len(sp["text"])
    return out


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_restore_version_renders_like_the_version(seed, kw):
    """TEXT, merge, MARKS, merge: every restored log renders as its version, per position with Q3 normalised, and byte for byte
    where no Q3 corner occurs.  A log whose text already differs gets TEXT_DIFFERS from MARKS alone."""
    _, logs = session(seed, kw, steps=40)
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_as(e, batch, "runs")
        merged(e)
        n = batch.n_logs
        co, got = checkout_all(e, batch, [max(1, int(batch.changes.desc[i]["n_changes"]) // 3) for i in range(n)])
        differs = [i for i in range(n) if not np.array_equal(got.tokens(i), got.tokens(n + i))]
        if differs:
            st, n_ops, _ = e.restore(requests_for(co, [(differs[0], n + differs[0])]), RESTORE_MARKS)
            assert st.tolist() == [RESTORE_TEXT_DIFFERS] and n_ops.tolist() == [0]
            got = merged(e)
        (st_t, _, _), (st_m, ops_m, _) = e.restore_version(list(range(n)), [n + i for i in range(n)], [requests_for(co, [(i, i)])[0][2] for i in range(n)])
        assert (st_t == RESTORE_OK).all() and (st_m == RESTORE_OK).all()
        after = e.download()
        js = e.render_json_list(co)
        for i in range(n):
            assert q3_normalised(co, after, i) == q3_normalised(co, after, n + i), i
            if b'"comment":[]' not in js[i] and b'"comment":[]' not in js[n + i]:
                assert js[i] == js[n + i], i
    finally:
        e.close()


def test_restore_change_reaches_other_replicas_through_sync():
    """A restore on one replica, delivered to the others by pt_batch_sync_pairs: after a two-way sync every replica converges
    (equal digests and text) on the restored document; a second restore then runs on a log the sync built."""
    _, logs = session(7, {}, steps=40)
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_as(e, batch, "plain")
        e.upload_actors(batch)
        merged(e)
        n = batch.n_logs
        co, got = checkout_all(e, batch, [2] + [1] * (n - 1))
        actor0 = requests_for(co, [(0, 0)])[0][2]
        (st, n_ops, _), _ = e.restore_version([0], [n], [actor0])
        assert st.tolist() == [RESTORE_OK] and n_ops[0] > 0
        for pairs in ([(0, j) for j in range(1, n)], [(1, 0)]):         # a dst once per call
            status, *_ = e.sync_pairs(pairs)
            assert (status == 0).all()
        after = merged(e)
        res = after.results
        assert all((res["digest"][j] == res["digest"][0]).all() for j in range(n))
        assert all(np.array_equal(after.tokens(j), got.tokens(n)) for j in range(n))
        # log 1 now holds the restore it received; restoring it to its own first-change checkout is an ordinary request
        (st, _, _), _ = e.restore_version([1], [n + 1], [requests_for(co, [(1, 1)])[0][2]])
        assert st.tolist() == [RESTORE_OK]
        final = e.download()
        assert np.array_equal(final.tokens(1), final.tokens(n + 1))
    finally:
        e.close()


def test_empty_and_mark_only_logs():
    """A log whose version is empty loses all its text; a log restored to itself, and a mark-only difference, by MARKS."""
    d, _, init = generateDocs(O, "abcdef", 1)
    d = d[0]
    bold = d.change([{"path": ["text"], "action": "addMark", "startIndex": 1, "endIndex": 4, "markType": "strong"}])["change"]
    link = d.change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 3, "markType": "link", "attrs": {"url": "x.org"}}])["change"]
    logs = [[init, bold, link], [init]]
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_as(e, batch, "plain")
        merged(e)
        co, got = checkout_all(e, batch, [1, 0])                          # log 3: the empty version of log 1
        st, n_ops, _ = e.restore(requests_for(co, [(0, 2), (1, 3)]))      # log 0: same text, nothing to do; log 1: delete all
        assert st.tolist() == [RESTORE_OK, RESTORE_OK] and n_ops.tolist() == [0, 6]
        got = merged(e)
        reqs = [(log, ver, a, f + int(k)) for (log, ver, a, f), k in zip(requests_for(co, [(0, 2), (1, 3)]), n_ops)]
        st, n_ops, _ = e.restore(reqs, RESTORE_MARKS)
        assert st.tolist() == [RESTORE_OK, RESTORE_OK] and n_ops.tolist() == [2, 0]   # removeMark strong, removeMark link
        after = merged(e)
        assert q3_normalised(co, after, 0) == q3_normalised(co, after, 2)
    finally:
        e.close()


def test_logs_built_by_select():
    """Forks made by pt_batch_select_logs, checked out and restored, against the twin holding apply_select's batch."""
    from peritext_b200.packing import apply_select
    _, logs = session(1007, SESSIONS[2][1], steps=40)
    batch = pack_logs(logs, with_changes=True)
    e, u = engine(), engine()
    try:
        upload_as(e, batch, "compact")
        merged(e)
        frm = list(range(batch.n_logs))[::-1] + [0, 1]
        e.select_logs(frm)
        sel = apply_select(batch, frm)
        merged(e)
        n = sel.n_logs
        co, got = checkout_all(e, sel, [max(1, int(sel.changes.desc[i]["n_changes"]) // 2) for i in range(n)])
        upload_as(u, co, "plain")
        merged(u)
        st, n_ops, _, _, _ = restore_and_compare(e, u, co, got, [(i, n + i) for i in range(n)])
        assert (st == RESTORE_OK).all() and n_ops.sum() > 0
    finally:
        e.close(); u.close()
