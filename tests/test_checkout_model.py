"""The host side of pt_batch_checkout and pt_batch_download_clocks: ``apply_checkout``, ``checkout_clocks`` and ``clocks``.

A version of a log is what a fresh Micromerge holds after applyChange of exactly the changes it covers.  So every checkout that
``apply_checkout`` reports OK must replay (oracle.packed) to the spans the oracle gives for those changes applied in table
order, at every prefix of the fuzz sessions' and the KATs' logs and at the clocks of the other replicas' prefixes.
tests/test_gpu_checkout.py reuses the cases here."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200.packing import (CHECKOUT_BAD_TABLE, CHECKOUT_NOT_CLOSED, CHECKOUT_OK, CHECKOUT_UNKNOWN, CLOCK_DT, apply_checkout, checkout_clocks,
                                   clocks, decode_spans, pack_logs)
from tests.harness import fuzz_session, generateDocs
from tests.test_append_packing import kat_logs

SESSIONS = [(7, {}), (2007, dict(replicas=2, max_chars=6, initial="The Peritext editor")), (1007, dict(sync_prob=0.3, full_sync_at_end=False)),
            (3007, dict(zero_width_prob=0.3))]


def session(seed, kw, steps=60):
    """(final docs, per-replica Change logs) of a harness fuzz session."""
    docs, logs, _ = fuzz_session(O, seed, steps, **kw)
    return docs, logs


def prefix_spans(log):
    """The spans of a fresh Micromerge after each prefix log[:j], j = 0 .. len(log)."""
    m, out = O("~reader"), [[]]
    for ch in log:
        m.applyChange(ch)
        out.append(m.getTextWithFormatting())
    return out


def clock_of(changes) -> dict:
    """Micromerge.clock after applying `changes`: per actor id the highest seq."""
    clk: dict = {}
    for ch in changes:
        clk[ch["actor"]] = max(clk.get(ch["actor"], 0), ch["seq"])
    return clk


def covered(log, clk):
    return [ch for ch in log if ch["seq"] <= clk.get(ch["actor"], 0)]


def oracle_of(changes):
    m = O("~reader")
    for ch in changes:
        m.applyChange(ch)
    return m.getTextWithFormatting() if changes else []


def spans_of(batch, first):
    """decode_spans of logs first .. of `batch`, replayed by the oracle's packed replay."""
    ref, _ = replay_packed(batch)
    return [decode_spans(batch, ref, i) for i in range(first, batch.n_logs)]


def every_prefix(logs):
    """(logs, n_changes) of a checkout of every prefix of every log."""
    req = [(r, j) for r, lg in enumerate(logs) for j in range(len(lg) + 1)]
    return [r for r, _ in req], [j for _, j in req]


def cross_clocks(logs, stride=5):
    """(logs, clocks by actor id, the covered Change lists): log r at the clock of logs[t][:j], every stride-th j."""
    out_l, out_c, out_w = [], [], []
    for t, lt in enumerate(logs):
        for j in range(0, len(lt) + 1, stride):
            clk = clock_of(lt[:j])
            for r, lr in enumerate(logs):
                out_l.append(r); out_c.append(clk); out_w.append(covered(lr, clk))
    return out_l, out_c, out_w


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_every_prefix_replays_to_the_oracle(seed, kw):
    _, logs = session(seed, kw)
    batch = pack_logs(logs, with_changes=True)
    lg, nch = every_prefix(logs)
    got, status = apply_checkout(batch, lg, n_changes=nch)
    assert (status == CHECKOUT_OK).all()
    want = [s for log in logs for s in prefix_spans(log)]
    assert spans_of(got, batch.n_logs) == want
    for k, (r, j) in enumerate(zip(lg, nch)):         # the prefix's records are the source's first records
        d, s = got.desc[batch.n_logs + k], batch.desc[r]
        ins = got.insdel[int(d["insdel_off"]): int(d["insdel_off"]) + int(d["n_insdel"])]
        assert ins.tobytes() == batch.insdel[int(s["insdel_off"]): int(s["insdel_off"]) + len(ins)].tobytes()
        assert int(got.changes.desc[batch.n_logs + k]["n_changes"]) == j


def test_every_prefix_of_the_kat_logs():
    logs = kat_logs()
    batch = pack_logs(logs, with_changes=True)
    lg, nch = every_prefix(logs)
    got, status = apply_checkout(batch, lg, n_changes=nch)
    assert (status == CHECKOUT_OK).all()
    assert spans_of(got, batch.n_logs) == [s for log in logs for s in prefix_spans(log)]


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_cross_replica_clocks(seed, kw):
    docs, logs = session(seed, kw)
    batch = pack_logs(logs, with_changes=True)
    lg, clk, want = cross_clocks(logs)
    have = [clock_of(lr) for lr in logs]
    known = [all(seq <= have[r].get(a, 0) for a, seq in c.items()) for r, c in zip(lg, clk)]
    # an actor the log never saw may only come with seq 0
    clk = [{a: s for a, s in c.items() if a in batch.log_actors[r] or s} for r, c in zip(lg, clk)]
    ok_idx = [k for k, kn in enumerate(known) if kn]
    got, status = apply_checkout(batch, [lg[k] for k in ok_idx], clock=checkout_clocks(batch, [lg[k] for k in ok_idx], [clk[k] for k in ok_idx]))
    assert (status == CHECKOUT_OK).all()
    assert spans_of(got, batch.n_logs) == [oracle_of(want[k]) for k in ok_idx]
    # the covered changes replayed give replica t's document after j arrivals when the session converged
    if kw.get("full_sync_at_end", True):
        finals = [d.getTextWithFormatting() for d in docs]
        assert all(f == finals[0] for f in finals)
        t_of = [(t, j) for t, lt in enumerate(logs) for j in range(0, len(lt) + 1, 5) for _ in logs]
        ps = [prefix_spans(lt) for lt in logs]
        got_spans = spans_of(got, batch.n_logs)
        for g, k in zip(got_spans, ok_idx):
            t, j = t_of[k]
            assert g == ps[t][j], (t, j, lg[k])


def test_unknown_when_the_log_lacks_changes_of_the_clock():
    _, logs = session(1007, dict(sync_prob=0.3, full_sync_at_end=False))
    batch = pack_logs(logs, with_changes=True)
    lg, clk, _ = cross_clocks(logs, stride=1)
    have = [clock_of(lr) for lr in logs]
    unknown = [k for k, (r, c) in enumerate(zip(lg, clk)) if any(s > have[r].get(a, 0) for a, s in c.items()) and all(a in batch.log_actors[r] for a in c)]
    assert unknown
    pick = unknown[:20]
    _, status = apply_checkout(batch, [lg[k] for k in pick], clock=checkout_clocks(batch, [lg[k] for k in pick], [clk[k] for k in pick]))
    assert (status == CHECKOUT_UNKNOWN).all()


def two_replicas():
    """A Change log with [init by doc1 (seq 1), doc2's seq 1 that depends on doc1's seq 1], packed with its change table."""
    docs, _, init = generateDocs(O, "abc", 2)
    c2 = docs[1].change([{"path": ["text"], "action": "insert", "index": 1, "values": ["x"]}])["change"]
    assert c2["deps"] == {"doc1": 1}
    return [init, c2], pack_logs([[init, c2]], with_changes=True)


def clock(entries):
    """A single request's clock-mode arrays from [(actor rank, seq)]."""
    return np.array([0, len(entries)], np.uint64), np.array(entries, CLOCK_DT) if entries else np.zeros(0, CLOCK_DT)


def test_not_closed_against_the_covered_changes():
    log, batch = two_replicas()
    assert batch.log_actors[0] == ["doc1", "doc2"]
    _, st = apply_checkout(batch, [0], clock=clock([(1, 1)]))                 # doc2's change without doc1's
    assert st.tolist() == [CHECKOUT_NOT_CLOSED]
    got, st = apply_checkout(batch, [0], clock=clock([(0, 1), (1, 0)]))       # a seq of 0 is allowed
    assert st.tolist() == [CHECKOUT_OK]
    assert spans_of(got, 1) == [oracle_of(log[:1])]
    # a dep (doc1, 0) with nothing of doc1 covered: applyChange refuses a zero clock entry
    batch.changes.deps["seq"][:] = 0
    _, st = apply_checkout(batch, [0], clock=clock([(1, 1)]))
    assert st.tolist() == [CHECKOUT_NOT_CLOSED]


def test_not_closed_is_computed_in_table_order():
    _, batch = two_replicas()
    ch = batch.changes.changes
    assert ch["dep_off"].tolist() == [0, 0]
    batch.changes.changes = ch[::-1].copy()                                 # doc2's change first: admission rejects the table
    _, st = apply_checkout(batch, [0], clock=clock([(0, 1), (1, 1)]))       # the clock alone holds doc2's dep
    assert st.tolist() == [CHECKOUT_NOT_CLOSED]
    _, st = apply_checkout(batch, [0], n_changes=[1])
    assert st.tolist() == [CHECKOUT_NOT_CLOSED]


def test_bad_table():
    _, batch = two_replicas()
    batch.changes.changes["seq"][1] = 2                                     # doc2's seq 2 without a seq 1
    got, st = apply_checkout(batch, [0, 0], n_changes=[0, 2])
    assert st.tolist() == [CHECKOUT_BAD_TABLE] * 2
    assert got.n_logs == 3 and got.desc[1:]["n_insdel"].tolist() == [0, 0] and got.changes.desc[1:]["n_changes"].tolist() == [0, 0]
    _, batch = two_replicas()
    batch.changes.changes["n_ops"][0] += 1                                  # n_ops do not sum to the records
    _, st = apply_checkout(batch, [0], n_changes=[1])
    assert st.tolist() == [CHECKOUT_BAD_TABLE]


def test_clocks_model():
    _, logs = session(1007, dict(sync_prob=0.3, full_sync_at_end=False))
    batch = pack_logs(logs, with_changes=True)
    off, seq, st = clocks(batch)
    assert (st == CHECKOUT_OK).all()
    for i, lg in enumerate(logs):
        c = clock_of(lg)
        assert {a: int(seq[int(off[i]) + r]) for r, a in enumerate(batch.log_actors[i]) if seq[int(off[i]) + r]} == c
    batch.changes.changes["seq"][0] = 9
    off, seq, st = clocks(batch)
    assert st[0] == CHECKOUT_BAD_TABLE and not seq[int(off[0]): int(off[1])].any() and (st[1:] == CHECKOUT_OK).all()


def test_helper_refusals():
    _, batch = two_replicas()
    with pytest.raises(ValueError, match="exactly one"):
        apply_checkout(batch, [0])
    with pytest.raises(ValueError, match="exactly one"):
        apply_checkout(batch, [0], n_changes=[1], clock=clock([]))
    with pytest.raises(ValueError, match="no log"):
        apply_checkout(batch, [1], n_changes=[1])
    with pytest.raises(ValueError, match="n_actors"):
        apply_checkout(batch, [0], clock=clock([(2, 1)]))
    with pytest.raises(ValueError, match="twice"):
        apply_checkout(batch, [0], clock=clock([(0, 1), (0, 1)]))
    with pytest.raises(ValueError, match="offsets"):
        apply_checkout(batch, [0], clock=(np.array([1, 1], np.uint64), np.zeros(1, CLOCK_DT)))
    with pytest.raises(ValueError, match="offsets"):
        apply_checkout(batch, [0, 0], clock=(np.array([0, 2, 1], np.uint64), np.zeros(2, CLOCK_DT)))
    with pytest.raises(ValueError, match="change table"):
        apply_checkout(pack_logs([[]]), [0], n_changes=[0])
    with pytest.raises(ValueError, match="does not know"):
        checkout_clocks(batch, [0], [{"doc9": 1}])
    off, ent = checkout_clocks(batch, [0, 0], [{"doc9": 0, "doc2": 1}, {}])
    assert off.tolist() == [0, 1, 1] and ent.tolist() == [(1, 1)]
