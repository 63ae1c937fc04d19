"""pt_batch_checkout and pt_batch_download_clocks on the device.  After a checkout the handle must hold exactly what an upload of
``packing.apply_checkout``'s batch (with its change table and actor tables) would hold, so every output of a merge after it
equals the output of that upload; tests/test_checkout_model.py pins ``apply_checkout`` against the oracle."""
import json

import numpy as np
import pytest

from peritext_b200 import workload
from peritext_b200.packing import (CDESC_DT, CHANGE_DT, CHECKOUT_BAD_TABLE, CHECKOUT_NOT_CLOSED, CHECKOUT_OK, CHECKOUT_UNKNOWN, CLOCK_DT, DEP_DT, SELECT_ADDED,
                                   ChangeTable, apply_checkout, apply_select, checkout_clocks, clocks, pack_logs)
from tests.test_append_packing import kat_logs, sparse_logs
from tests.test_checkout_model import SESSIONS, clock_of, cross_clocks, session, two_replicas
from tests.test_gpu_append import canon, engine, merged, route_crossings
from tests.test_gpu_routes import batch_of, expected_route
from tests.test_gpu_select import outputs, uploaded
from tests.test_gpu_sync import device_sync, upload_all
from tests.test_gpu_wire_forms import FORMS, upload_as

pytestmark = pytest.mark.gpu
PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def requests(logs, stride=3):
    """A prefix request at every stride-th prefix of every log, and the full table of log 0 twice."""
    lg = [r for r, log in enumerate(logs) for j in range(0, len(log) + 1, stride)] + [0, 0]
    nch = [j for log in logs for j in range(0, len(log) + 1, stride)] + [len(logs[0])] * 2
    return lg, nch


def prefix_logs(logs, lg, nch):
    """The Change logs of a batch after prefix checkouts: the resident ones, then logs[r][:j] per request."""
    return list(logs) + [logs[r][:j] for r, j in zip(lg, nch)]


def same_clocks(e, batch):
    off, seq, st = e.clocks()
    w_off, w_seq, w_st = clocks(batch)
    assert off.tolist() == w_off.tolist() and seq.tolist() == w_seq.tolist() and st.tolist() == w_st.tolist()


# ------------------------------------------------------------------------------------------------------------------
# 1. Every upload form, prefix and clock checkouts, against the specification
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("seed,kw", SESSIONS[:3])
def test_checkout_after_every_form_equals_the_upload(seed, kw, form):
    _, logs = session(seed, kw, steps=40)
    prev = pack_logs(logs, with_changes=True)
    lg, nch = requests(logs)
    want, status = apply_checkout(prev, lg, n_changes=nch)
    e, u = engine(patches=True), engine(patches=True)
    try:
        keep = upload_as(e, prev, form)
        merged(e)
        got = e.checkout(lg, n_changes=nch)
        del keep
        assert got.tolist() == status.tolist() and (got == CHECKOUT_OK).all()
        assert e.n_logs == want.n_logs
        want_logs = prefix_logs(logs, lg, nch)
        assert outputs(e, want, want_logs) == uploaded(u, want, want_logs), form
        same_clocks(e, want)
        # clock mode on the result: the other replicas' prefix clocks
        cl, ck, _ = cross_clocks(logs, stride=7)
        have = [clock_of(x) for x in logs]
        ok = [k for k, (r, c) in enumerate(zip(cl, ck)) if all(s <= have[r].get(a, 0) for a, s in c.items())]
        ck = [{a: s for a, s in ck[k].items() if a in want.log_actors[cl[k]] or s} for k in ok]
        cr = checkout_clocks(want, [cl[k] for k in ok], ck)
        want2, status2 = apply_checkout(want, [cl[k] for k in ok], clock=cr)
        assert e.checkout([cl[k] for k in ok], clock=cr).tolist() == status2.tolist()
        logs2 = want_logs + [[ch for ch in want_logs[cl[k]] if ch["seq"] <= c.get(ch["actor"], 0)] if st == CHECKOUT_OK else []
                             for k, c, st in zip(ok, ck, status2)]
        assert outputs(e, want2, logs2) == uploaded(u, want2, logs2)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. State that lives only on the device: syncs, then clocks named from the device and checked out
# ------------------------------------------------------------------------------------------------------------------
def test_after_device_syncs_the_clocks_name_the_version():
    from oracle.oracle import Micromerge as O
    from tests.harness import generateDocs
    logs = []
    for d, text in enumerate(["abcd", "efghij", "klm"]):
        reps, _, init = generateDocs(O, text, 2)
        c = reps[1].change([{"path": ["text"], "action": "insert", "index": 1, "values": list("xy"[: 1 + d % 2])}])["change"]
        c2 = reps[0].change([{"path": ["text"], "action": "delete", "index": 0, "count": 1}])["change"]
        c3 = reps[1].change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 2, "markType": "strong"}])["change"]
        logs += [[init, c2], [init, c, c3]]                   # document d: logs 2d, 2d + 1; every change has list ops
    cur = pack_logs(logs, with_changes=True)
    e, u = engine(patches=True), engine(patches=True)
    try:
        upload_all(e, cur)
        merged(e)
        cur, _, _ = device_sync(e, cur, [(1, 0), (2, 3), (4, 5)])             # device-only changes to logs 0, 3 and 5
        same_clocks(e, cur)
        off, seq, st = e.clocks()
        # check out every log at its own clock (a fork) and at the clock log 0 holds now
        lg = list(range(cur.n_logs)) * 2
        ent = [(r, int(seq[int(off[i]) + r])) for i in range(cur.n_logs) for r in range(int(off[i + 1] - off[i]))]
        ids0 = {cur.log_actors[0][r]: int(seq[int(off[0]) + r]) for r in range(int(off[1] - off[0]))}
        c_off, c_ent = checkout_clocks(cur, lg[cur.n_logs:], [{a: s for a, s in ids0.items() if a in cur.log_actors[r]} for r in range(cur.n_logs)])
        own_off = np.concatenate([[0], np.cumsum(off[1:] - off[:-1])]).astype(np.uint64)
        clk = (np.concatenate([own_off, c_off[1:] + own_off[-1]]).astype(np.uint64), np.concatenate([np.array(ent, CLOCK_DT), c_ent]))
        want, status = apply_checkout(cur, lg, clock=clk)
        got = e.checkout(lg, clock=clk)
        assert got.tolist() == status.tolist()
        assert (got[: cur.n_logs] == CHECKOUT_OK).all()
        assert e.actors() == [list(a) for a in want.log_actors]
        assert outputs(e, want) == uploaded(u, want)
        same_clocks(e, want)
        g_off, g_seq, _ = e.clocks()                   # each OK checkout's clock is its request clock
        for k in range(cur.n_logs):
            i = cur.n_logs + k
            assert g_seq[int(g_off[i]): int(g_off[i + 1])].tolist() == seq[int(off[k]): int(off[k + 1])].tolist()
        res = merged(e).results
        assert (res["digest"][cur.n_logs: 2 * cur.n_logs] == res["digest"][: cur.n_logs]).all()
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. Prefixes: the Patch stream and its render are the source's first ops; a full checkout is a fork; empty is empty
# ------------------------------------------------------------------------------------------------------------------
def test_prefix_patches_are_the_sources_first_ops():
    _, logs = session(7, {}, steps=40)
    prev = pack_logs(logs, with_changes=True)
    lg, nch = requests(logs, stride=4)
    want, _ = apply_checkout(prev, lg, n_changes=nch)
    e, f = engine(patches=True), engine(patches=True)
    try:
        e.upload(prev); e.upload_changes(prev.changes)
        e.checkout(lg, n_changes=nch)
        out = merged(e)
        recs, _, pst, _ = e.download_patches()
        js = [json.loads(x) for x in e.render_patches_json_list(want)]
        for k, (r, j) in enumerate(zip(lg, nch)):
            i = prev.n_logs + k
            assert pst[i] == 0 and out.results[i]["status"] == 0
            d, s = want.desc[i], want.desc[r]
            a, b = int(d["insdel_off"]), int(s["insdel_off"])
            assert recs[a: a + int(d["n_insdel"])].tobytes() == recs[b: b + int(d["n_insdel"])].tobytes(), (r, j)
            assert js[i] == js[r][: int(d["n_insdel"]) + int(d["n_mark"])], (r, j)
            if j == 0:
                assert out.results[i]["n_visible"] == 0 and out.results[i]["n_spans"] == 0
        # a checkout of the full table is a select_logs fork
        full = [r for r in range(prev.n_logs)]
        e.select_logs(list(range(prev.n_logs)))
        e.checkout(full, n_changes=[len(x) for x in logs])
        f.upload(prev); f.upload_changes(prev.changes)
        f.select_logs(list(range(prev.n_logs)) * 2)
        fork = apply_select(prev, list(range(prev.n_logs)) * 2)
        assert outputs(e, fork, logs * 2) == outputs(f, fork, logs * 2)
    finally:
        e.close(); f.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Statuses, mixed calls and refusals
# ------------------------------------------------------------------------------------------------------------------
def computed_outputs(e, batch):
    """``outputs`` with the patch records of logs whose patch status is not 0 cleared: the device does not compute them."""
    from peritext_b200.engine import PATCH_REC_DT
    o = list(outputs(e, batch))
    ev = list(o[2])
    recs, st = np.frombuffer(ev[0], PATCH_REC_DT).copy(), np.frombuffer(ev[2], np.uint32)
    for i in np.nonzero(st)[0]:
        a = int(batch.desc[i]["insdel_off"])
        recs[a: a + int(batch.desc[i]["n_insdel"])] = 0
    ev[0] = recs.tobytes()
    o[2] = tuple(ev)
    return tuple(o)


def raw_checkout(e, logs, n_changes=None, clock_off=None, clock_=None, n=None, status=True):
    arr = lambda a, dt: None if a is None else np.ascontiguousarray(a, dt)
    lg, nc, co, ce = arr(logs, np.uint32), arr(n_changes, np.uint32), arr(clock_off, np.uint64), arr(clock_, CLOCK_DT)
    st = np.zeros(max(1, len(logs or [])), np.uint32)
    p = lambda a: None if a is None else a.ctypes.data
    return e._L.pt_batch_checkout(e._h, p(lg), len(lg) if n is None else n, p(nc), p(co), p(ce), st.ctypes.data if status else None)


def test_statuses_mix_and_refusals_leave_the_batch_untouched():
    from peritext_b200.engine import EngineError
    log, good = two_replicas()
    _, bad = two_replicas()
    bad.changes.changes["seq"][1] = 2
    rev = pack_logs([log], with_changes=True)
    rev.changes.changes = rev.changes.changes[::-1].copy()
    both = apply_select(good, [0, SELECT_ADDED, SELECT_ADDED], apply_select(bad, [0, SELECT_ADDED], rev))
    e, u = engine(patches=True), engine(patches=True)
    try:
        e.upload(both); e.upload_changes(both.changes); e.upload_actors(both)
        before = outputs(e, both)
        cases = {
            "null logs": dict(logs=None, n_changes=[1], n=1),
            "null status": dict(logs=[0], n_changes=[1], status=False),
            "log past the batch": dict(logs=[0, 3], n_changes=[1, 1]),
            "neither mode": dict(logs=[0]),
            "both modes": dict(logs=[0], n_changes=[1], clock_off=[0, 0]),
            "clock_off from 1": dict(logs=[0], clock_off=[1, 1], clock_=[(0, 1)]),
            "clock_off decreases": dict(logs=[0, 0], clock_off=[0, 2, 1], clock_=[(0, 1), (1, 1)]),
            "actor past n_actors": dict(logs=[0], clock_off=[0, 1], clock_=[(2, 1)]),
            "actor twice": dict(logs=[0], clock_off=[0, 2], clock_=[(1, 1), (1, 1)]),
        }
        for name, kw in cases.items():
            assert raw_checkout(e, **kw) == PT_ERR_INVALID, name
            assert outputs(e, both) == before, name
        assert raw_checkout(e, [], n_changes=[]) == 0 and outputs(e, both) == before
        # OK, UNKNOWN, NOT_CLOSED (a dep of doc1 uncovered, and table order in log 2), BAD_TABLE, several on one log
        lg = [0, 0, 0, 1, 2, 0]
        co = [0, 2, 3, 4, 4, 6, 6]
        ce = [(0, 1), (1, 1), (0, 2), (1, 1), (0, 1), (1, 1)]
        want, status = apply_checkout(both, lg, clock=(np.array(co, np.uint64), np.array(ce, CLOCK_DT)))
        assert status.tolist() == [CHECKOUT_OK, CHECKOUT_UNKNOWN, CHECKOUT_NOT_CLOSED, CHECKOUT_BAD_TABLE, CHECKOUT_NOT_CLOSED, CHECKOUT_OK]
        assert e.checkout(lg, clock=(co, np.array(ce, CLOCK_DT))).tolist() == status.tolist()
        assert e.actors() == [list(a) for a in want.log_actors]
        upload_as(u, want, "plain")
        assert computed_outputs(e, want) == computed_outputs(u, want)
        same_clocks(e, want)
        e.select_logs([0, 1, 2])                        # retires the checkouts
        assert outputs(e, both) == before
        f = engine()
        try:
            with pytest.raises(EngineError) as err:
                f.checkout([0], n_changes=[0])
            assert err.value.status == PT_ERR_STATE
            f.upload(both)
            with pytest.raises(EngineError) as err:
                f.checkout([0], n_changes=[0])
            assert err.value.status == PT_ERR_STATE
            with pytest.raises(EngineError) as err:
                f.clocks()
            assert err.value.status == PT_ERR_STATE
        finally:
            f.close()
    finally:
        e.close(); u.close()


def two_change_table(batch):
    """Every log's list ops as two changes by actor rank 0: the first half and the rest."""
    n = batch.n_logs
    ops = (batch.desc["n_insdel"] + batch.desc["n_mark"]).astype(np.int64)
    cd = np.zeros(n, CDESC_DT)
    cd["change_off"] = 2 * np.arange(n); cd["n_changes"] = 2
    ch = np.zeros(2 * n, CHANGE_DT)
    ch["seq"] = np.tile([1, 2], n)
    ch["n_ops"][0::2] = ops // 2; ch["n_ops"][1::2] = ops - ops // 2
    return ChangeTable(cd, ch, np.zeros(0, DEP_DT))


def test_checkouts_cross_routes_and_dense_counters():
    big = batch_of([x[0] for x in route_crossings()])
    big.changes = two_change_table(big)
    sp, _ = sparse_logs()
    dense = pack_logs(sp, with_changes=True)
    assert any(c is not None for c in dense.log_counters)
    kats = pack_logs(kat_logs()[:6], with_changes=True)
    e, u = engine(patches=True), engine(patches=True)
    try:
        for prev, lg, nch, src_logs in [(big, [0, 1, 2, 0, 1, 2], [1, 1, 1, 2, 2, 0], None),
                                        (dense, [0, 1, 0, 1], [1, 2, 3, 3], sp),
                                        (kats, [5, 4, 3], [2, 1, 0], kat_logs()[:6])]:
            upload_as(e, prev, "plain")
            merged(e)
            want, status = apply_checkout(prev, lg, n_changes=nch)
            assert (status == CHECKOUT_OK).all()
            assert (e.checkout(lg, n_changes=nch) == CHECKOUT_OK).all()
            if prev is big:                             # no pools: the merge outputs only
                routes = {expected_route(d) for d in want.desc}
                assert len(routes) >= 2, routes
                got = merged(e)
                u.upload(want); u.upload_changes(want.changes)
                ref = merged(u)
                assert canon(got) == canon(ref) and got.results.tobytes() == ref.results.tobytes()
            else:
                want_logs = prefix_logs(src_logs, lg, nch)
                assert outputs(e, want, want_logs) == uploaded(u, want, want_logs)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. Scale
# ------------------------------------------------------------------------------------------------------------------
def test_c4_300k_logs_at_empty_and_full_clocks():
    from tests.test_gpu_exchange import one_change_tables
    full = workload.generate("c4")
    assert full.n_logs >= 300_000
    full.changes = one_change_tables(full, np.zeros(full.n_logs, np.uint16))
    lg = list(range(0, full.n_logs, 100))
    e = engine()
    try:
        e.upload(full); e.upload_changes(full.changes)
        n0 = full.n_logs
        st = e.checkout(lg + lg, n_changes=[0] * len(lg) + [1] * len(lg))
        assert (st == CHECKOUT_OK).all()
        e.merge()
        res = e.results()
        assert (res["status"] == 0).all()
        assert (res["n_visible"][n0: n0 + len(lg)] == 0).all()
        assert res[n0 + len(lg):].tobytes() == res[lg].tobytes()
        e.select_logs(list(range(n0)))
        e.merge()
        again = e.results()
        assert again.tobytes() == res[:n0].tobytes()
    finally:
        e.close()


def test_c4_slice_through_the_native_ingest():
    from peritext_b200.engine import pack_logs_native
    gen = workload.generate("c4", n_docs=3000, ops_per_doc=60)
    prev = pack_logs_native([workload.to_change_json(gen, i) for i in range(gen.n_logs)])
    n_ch = prev.changes.desc["n_changes"].astype(np.int64)
    assert n_ch.max() > 1
    lg = list(range(0, prev.n_logs, 7))
    nch = [int(n_ch[i]) // 2 for i in lg]
    want, status = apply_checkout(prev, lg, n_changes=nch)
    assert (status == CHECKOUT_OK).all()
    e, u = engine(), engine()
    try:
        e.upload(prev); e.upload_changes(prev.changes)
        assert (e.checkout(lg, n_changes=nch) == CHECKOUT_OK).all()
        got = merged(e)
        u.upload(want); u.upload_changes(want.changes)
        ref = merged(u)
        assert canon(got) == canon(ref) and got.results.tobytes() == ref.results.tobytes()
        same_clocks(e, want)
    finally:
        e.close(); u.close()
