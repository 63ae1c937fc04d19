"""pt_batch_attribute on the device.  Its runs must equal ``attribution.attribution_runs`` byte for byte, read from the batch the
handle holds (the upload, or the host specification of the calls that built it on the device) and the element sequence of its
last merge; tests/test_attribution_spec.py pins ``attribution_runs`` against the Change dicts and the oracle."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.attribution import ATTR_BAD_TABLE, ATTR_LOG_FAILED, ATTR_OK, attribution_runs
from peritext_b200.packing import CLOCK_DT, SELECT_ADDED, apply_checkout, apply_select, checkout_clocks, pack_logs
from tests.harness import generateDocs
from tests.test_append_packing import kat_logs, sparse_logs
from tests.test_attribution_spec import deletes_cases, prefix_clocks
from tests.test_checkout_model import SESSIONS, clock_of, session
from tests.test_gpu_append import merged
from tests.test_gpu_change import change_table, header, replica
from tests.test_gpu_exchange import device_sync as device_exchange
from tests.test_gpu_sync import device_sync, upload_all
from tests.test_gpu_wire_forms import FORMS, empty_corpus, upload_as

pytestmark = pytest.mark.gpu
PT_ERR_INVALID, PT_ERR_STATE = 1, 4


def engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, emit_sequence=True, **kw)


def same(e, batch, logs, clock=None, got=None):
    """The device's attribution of `logs` equals the specification over the handle's last merge (merging first unless `got`)."""
    got = merged(e) if got is None else got
    want = attribution_runs(batch, got, logs, clock)
    have = e.attribute(logs, clock)
    for w, h in zip(want, have):
        assert w.dtype == h.dtype and w.tobytes() == h.tobytes()
    return have


def clocks_for(batch, logs, clks):
    """checkout_clocks of clocks by actor id, dropping the zero entries of actors a log does not know."""
    keep = [{a: s for a, s in c.items() if a in batch.log_actors[i] or s} for i, c in zip(logs, clks)]
    ok = [k for k, i in enumerate(logs) if all(a in batch.log_actors[i] for a in keep[k])]
    return [logs[k] for k in ok], checkout_clocks(batch, [logs[k] for k in ok], [keep[k] for k in ok])


def all_clock_requests(batch, logs):
    """Every log at every prefix clock of every log (prefix and cross clocks), one request list."""
    clks = prefix_clocks(logs, stride=3)
    lg = [i for _ in clks for i in range(len(logs))]
    return clocks_for(batch, lg, [c for c in clks for _ in range(len(logs))])


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("seed,kw", SESSIONS[:3])
def test_every_form_and_clock_equals_the_specification(seed, kw, form):
    _, logs = session(seed, kw, steps=40)
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        keep = upload_as(e, batch, form)
        got = merged(e)
        del keep
        st, _, runs = same(e, batch, list(range(batch.n_logs)) * 2, got=got)   # every log twice
        assert (st == ATTR_OK).all() and len(runs)
        lg, clk = all_clock_requests(batch, logs)
        st, _, runs = same(e, batch, lg, clk, got=got)
        assert (st == ATTR_OK).all() and (runs["flags"] != 0).any()
    finally:
        e.close()


def test_kats_sparse_counters_and_concurrent_deletes():
    for logs in (kat_logs(), sparse_logs()[0], deletes_cases()):
        batch = pack_logs(logs, with_changes=True)
        e = engine()
        try:
            upload_as(e, batch, "plain")
            got = merged(e)
            st, _, _ = same(e, batch, list(range(batch.n_logs)), got=got)
            assert (st == ATTR_OK).all()
            lg, clk = all_clock_requests(batch, logs)
            same(e, batch, lg, clk, got=got)
        finally:
            e.close()


def one_change_tables(batch):
    """Each log's records as one change of actor rank 0."""
    from peritext_b200.packing import CDESC_DT, CHANGE_DT, DEP_DT, ChangeTable
    cd = np.zeros(batch.n_logs, CDESC_DT)
    cd["change_off"] = np.arange(batch.n_logs); cd["n_changes"] = 1
    ch = np.zeros(batch.n_logs, CHANGE_DT)
    ch["seq"] = 1; ch["n_ops"] = batch.desc["n_insdel"] + batch.desc["n_mark"]
    return ChangeTable(cd, ch, np.zeros(0, DEP_DT))


def test_empty_and_mark_only_logs_and_slot_reuse():
    """Logs without elements have no runs; more requests than the resident warps (grid-stride slots) agree too."""
    batch = empty_corpus().batch
    batch.changes = one_change_tables(batch)
    e = engine()
    try:
        e.upload(batch); e.upload_changes(batch.changes)
        got = merged(e)
        st, off, runs = same(e, batch, list(range(batch.n_logs)), got=got)
        assert (st == ATTR_OK).all()
        assert [int(off[i + 1] - off[i]) for i in range(batch.n_logs)] == [int(n > 0) for n in got.results["n_elems"]]
        n = 132 * 16 * 4 + 77
        same(e, batch, [k % batch.n_logs for k in range(n)], got=got)
    finally:
        e.close()


def test_logs_built_on_the_device():
    """pt_batch_checkout (prefix and clock forks), pt_batch_select_logs (forks), pt_batch_sync_pairs, pt_batch_exchange and
    pt_batch_change: the runs follow the batch the handle holds."""
    _, logs = session(2007, dict(replicas=2, max_chars=6, initial="The Peritext editor"), steps=40)
    cur = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_all(e, cur)
        merged(e)
        lg = [r for r in range(cur.n_logs) for _ in range(3)]
        nch = [j for lg_ in logs for j in (0, len(lg_) // 2, len(lg_))]
        want, status = apply_checkout(cur, lg, n_changes=nch)
        assert e.checkout(lg, n_changes=nch).tolist() == status.tolist()
        cur = want
        same(e, cur, list(range(cur.n_logs)))
        frm = [0, 1, 0, cur.n_logs - 1, 1]
        e.select_logs(frm)
        cur = apply_select(cur, frm)
        same(e, cur, list(range(cur.n_logs)))
        merged(e)
        cur, _, _ = device_sync(e, cur, [(0, 1), (3, 2)])
        got = merged(e)
        same(e, cur, list(range(cur.n_logs)), got=got)
        lg2, clk = clocks_for(cur, list(range(cur.n_logs)), [clock_of(logs[0][:5])] * cur.n_logs)
        same(e, cur, lg2, clk, got=got)
        cur, _, _ = device_exchange(e, cur, [(1, 4)])
        same(e, cur, list(range(cur.n_logs)))
    finally:
        e.close()


def test_local_changes_on_the_device():
    reps, _, init = generateDocs(O, "abcdef", 2)
    c1 = reps[1].change([{"path": ["text"], "action": "delete", "index": 2, "count": 2}])["change"]
    logs = [[init, c1], [init]]
    cur = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        e.upload(cur); e.upload_changes(cur.changes)
        merged(e)
        ops = [[{"path": ["text"], "action": "insert", "index": 1, "values": list("xyz")}, {"path": ["text"], "action": "delete", "index": 0, "count": 1}]] * 2
        inputs = [{**header(log, "doc1"), "seq": replica(log, "doc1").clock.get("doc1", 0) + 1, "ops": o} for log, o in zip(logs, ops)]
        ranks = [cur.log_actors[i].index("doc1") for i in range(2)]
        table = change_table(cur, inputs, ranks)
        table.changes["n_ops"] = 4                                # the generated list ops: three inserts and one delete
        new, _, status = e.change(cur, inputs, ranks, table)
        assert (status["status"] == 0).all()
        st, _, runs = same(e, new, [0, 1])
        assert (st == ATTR_OK).all() and len(set(runs["ins_seq"].tolist())) > 1
    finally:
        e.close()


def test_c5_shaped_log_and_user_stream():
    import torch
    from peritext_b200 import workload
    from peritext_b200.packing import ChangeTable, CDESC_DT, CHANGE_DT, DEP_DT
    b = workload.generate("c5", n_docs=1, ops_per_doc=110_000).select([0])
    n_ops = int(b.desc[0]["n_insdel"] + b.desc[0]["n_mark"])
    per = 97                                                  # many changes of one actor, seq 1 .. n, covering every list op
    cnt = (n_ops + per - 1) // per
    ch = np.zeros(cnt, CHANGE_DT)
    ch["seq"] = np.arange(1, cnt + 1); ch["actor"] = 0; ch["n_ops"] = per
    ch["n_ops"][-1] = n_ops - per * (cnt - 1)
    cd = np.zeros(1, CDESC_DT); cd["n_changes"] = cnt
    b.changes = ChangeTable(cd, ch, np.zeros(0, DEP_DT))
    s = torch.cuda.Stream()
    e = engine(stream=s.cuda_stream)
    try:
        e.upload(b); e.upload_changes(b.changes)
        got = merged(e)
        assert int(got.results["n_elems"][0]) > 10_000
        clk = (np.array([0, 1], np.uint64), np.array([(0, cnt // 2)], CLOCK_DT))
        st, _, runs = same(e, b, [0, 0], got=got)
        assert (st == ATTR_OK).all() and len(runs) > 64
        same(e, b, [0], clk, got=got)
    finally:
        e.close()


def test_statuses():
    logs = kat_logs()[:4]
    batch = pack_logs(logs, with_changes=True)
    bad = pack_logs(logs, with_changes=True)
    bad.changes.changes["n_ops"][int(bad.changes.desc[1]["change_off"])] += 1    # log 1's n_ops no longer sum
    rej = pack_logs(logs, with_changes=True)
    rej.changes.changes["seq"][int(rej.changes.desc[2]["change_off"])] += 5     # admission rejects log 2
    for b, log, want in ((bad, 1, ATTR_BAD_TABLE), (rej, 2, ATTR_LOG_FAILED)):
        e = engine()
        try:
            e.upload(b); e.upload_changes(b.changes)
            got = merged(e)
            st, _, _ = same(e, b, [0, log, 3], got=got)
            assert st.tolist() == [ATTR_OK, want, ATTR_OK]
        finally:
            e.close()
    fault = pack_logs(logs, with_changes=True)
    fault.insdel["ref_ctr"][int(fault.desc[3]["insdel_off"]) + 1] = 0xFFFF              # a reference no element has
    e = engine()
    try:
        e.upload(fault); e.upload_changes(fault.changes)
        got = merged(e)
        assert int(got.results["status"][3]) != 0
        assert same(e, fault, [3], got=got)[0].tolist() == [ATTR_LOG_FAILED]
    finally:
        e.close()


def test_refusals_leave_everything_unchanged():
    from peritext_b200.engine import EngineError
    _, logs = session(7, {}, steps=20)
    batch = pack_logs(logs, with_changes=True)
    e = engine()
    try:
        upload_as(e, batch, "plain")
        with pytest.raises(EngineError) as x:
            e.attribute([0])                                     # no merge yet
        assert x.value.status == PT_ERR_STATE
        got = merged(e)
        ref = e.attribute([0, 1])
        spans = e.download()
        bad = [([batch.n_logs], None), ([0], (np.array([1, 1], np.uint64), np.zeros(1, CLOCK_DT))),
               ([0, 1], (np.array([0, 1, 0], np.uint64), np.zeros(1, CLOCK_DT))),
               ([0], (np.array([0, 1], np.uint64), np.array([(int(batch.desc[0]["n_actors"]), 1)], CLOCK_DT))),
               ([0], (np.array([0, 2], np.uint64), np.array([(0, 1), (0, 2)], CLOCK_DT)))]
        for lg, clk in bad:
            with pytest.raises(EngineError) as x:
                e.attribute(lg, clk)
            assert x.value.status == PT_ERR_INVALID, (lg, clk)
        st, off, runs = e.attribute([])
        assert len(st) == 0 and off.tolist() == [0] and len(runs) == 0
        after = e.download()
        assert [after.canonical(i) for i in range(batch.n_logs)] == [spans.canonical(i) for i in range(batch.n_logs)]
        for w, h in zip(ref, e.attribute([0, 1])):
            assert w.tobytes() == h.tobytes()
        same(e, batch, [0, 1], got=got)
    finally:
        e.close()
    from peritext_b200.engine import BatchEngine
    for kw, table in ((dict(), True), (dict(emit_sequence=True), False)):
        h = BatchEngine(0, **kw)
        try:
            h.upload(batch)
            if table:
                h.upload_changes(batch.changes)
            merged(h)
            with pytest.raises(EngineError) as x:
                h.attribute([0])
            assert x.value.status == PT_ERR_STATE
        finally:
            h.close()
