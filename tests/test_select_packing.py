"""The host side of pt_batch_select_logs: ``pack_select`` + ``apply_select`` against the oracle and ``pack_logs``.

``apply_select(pack_logs(L), from_, *pack_select(pack_logs(L), from_, new_logs))`` must hold, per new log, what ``pack_logs`` of
the selected or added Change log holds (descriptor, records, actor ranks, counters, change table), with value tokens, link ids
and comment ranks compared through their pools, and the oracle's packed replay of it must give the spans the oracle's replay of
that Change log gives.  The corpora are tests/test_append_packing.py's; tests/test_gpu_select.py reuses the cases here."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200.packing import (ATTR_NONE, SELECT_ADDED, SELECT_DROPPED, apply_select, canon, decode_spans, pack_logs, pack_select)
from tests.harness import generateDocs
from tests.test_append_packing import (comment_and_link_logs, early_actor_logs, fuzz_logs, kat_logs, quirk_logs, sparse_logs, token_strs)

A = SELECT_ADDED


def select_corpora():
    """name -> (resident Change logs, from_, the added Change logs): drops, permutations, duplicates and additions."""
    kats, fuzz = kat_logs(), fuzz_logs()
    early = early_actor_logs()
    cl, _ = comment_and_link_logs()
    sp, _ = sparse_logs()
    n = len(kats)
    return {
        "kats": (kats, [n - 1, 0, 0, A, n // 2, A], [fuzz[0], kats[1][:1]]),
        "fuzz": (fuzz, [A] + list(range(len(fuzz)))[::-2] + [1, 1], [kats[3]]),
        "quirks": (quirk_logs() + early, [2, A, 0, 0], quirk_logs()),
        "early-actor": (early, [A, 1, A], [early[0], early[1][:1]]),
        "comments-links": (cl, [1, A, 0], [cl[0][:2]]),
        "sparse": (sp, [1, A, 1], [sp[0]]),
        "only-added": (kats[:3], [A, A], [kats[4], []]),
        "nothing": (kats[:3], [], []),
    }


def wanted_logs(logs, from_, new_logs):
    it = iter(new_logs)
    return [next(it) if f == A else logs[f] for f in from_]


def oracle_spans(logs):
    out = []
    for lg in logs:
        m = O("~reader")
        for ch in lg:
            m.applyChange(ch)
        out.append(m.getTextWithFormatting() if lg else [])     # an empty replica has no text list yet
    return out


def attr_names(batch):
    """Each mark's attr as the string it names: a comment id, a link url, or None."""
    kind = (batch.marks["kind"] >> 1) & 3
    out = []
    for k, a in zip(kind.tolist(), batch.marks["attr"].tolist()):
        out.append(None if a == ATTR_NONE else batch.comment_ids[a]["id"] if k == 2 else canon(batch.link_attrs[a]) if k == 3 else a)
    return out


def assert_same_logs(got, want, what=""):
    """Log by log the same packing; value tokens, link ids and comment ranks through their pools."""
    assert got.desc.tobytes() == want.desc.tobytes(), what
    for f in ("ctr", "ref_ctr", "actor", "ref_actor"):
        assert np.array_equal(got.insdel[f], want.insdel[f]), (what, f)
    assert np.array_equal(got.insdel["payload"] >> 30, want.insdel["payload"] >> 30), what
    ins = (got.insdel["payload"] >> 30) == 0
    assert [s for s, k in zip(token_strs(got), ins) if k] == [s for s, k in zip(token_strs(want), ins) if k], what
    for f in ("ctr", "actor", "kind", "bounds", "start_ctr", "end_ctr", "start_actor", "end_actor", "arrival", "reserved"):
        assert np.array_equal(got.marks[f], want.marks[f]), (what, f)
    assert attr_names(got) == attr_names(want), what
    assert got.log_actors == want.log_actors and got.log_lists == want.log_lists, what
    assert len(got.log_counters) == len(want.log_counters), what
    for a, b in zip(got.log_counters, want.log_counters):
        assert (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b)), what
    assert (got.changes is None) == (want.changes is None), what
    if want.changes is not None:
        for f in ("desc", "changes", "deps"):
            assert getattr(got.changes, f).tobytes() == getattr(want.changes, f).tobytes(), (what, f)


def selected(logs, from_, new_logs, with_changes=False):
    prev = pack_logs(logs, with_changes=with_changes)
    added, cmap = pack_select(prev, from_, new_logs, with_changes=with_changes)
    return prev, added, cmap, apply_select(prev, from_, added if len(new_logs) else None, cmap)


@pytest.mark.parametrize("with_changes", [False, True])
@pytest.mark.parametrize("name", ["kats", "fuzz", "quirks", "early-actor", "comments-links", "sparse", "only-added", "nothing"])
def test_select_equals_packing_the_selected_logs(name, with_changes):
    logs, from_, new_logs = select_corpora()[name]
    _, _, _, got = selected(logs, from_, new_logs, with_changes)
    want_logs = wanted_logs(logs, from_, new_logs)
    assert_same_logs(got, pack_logs(want_logs, with_changes=with_changes), name)
    ref, _ = replay_packed(got)
    spans = oracle_spans(want_logs)
    for i in range(got.n_logs):
        assert decode_spans(got, ref, i) == spans[i], (name, i)


def test_an_added_comment_that_sorts_first_shifts_the_kept_ranks():
    logs, _ = comment_and_link_logs()                      # log 0 names c-b and c-d, log 1 c-c and c-b
    docs, _, init = generateDocs(O, "wxyz", 1)
    early = docs[0].change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 2, "markType": "comment", "attrs": {"id": "c-a"}}])["change"]
    prev = pack_logs(logs)
    assert [c["id"] for c in prev.comment_ids] == ["c-b", "c-c", "c-d"]
    added, cmap = pack_select(prev, [0, A], [[init, early]], with_changes=False)
    assert cmap.tolist() == [1, 2, 3]
    assert [c["id"] for c in added.comment_ids] == ["c-a", "c-b", "c-c", "c-d"]
    got = apply_select(prev, [0, A], added, cmap)
    assert attr_names(got) == attr_names(pack_logs([logs[0], [init, early]]))
    kept = got.marks[: int(got.desc[0]["n_mark"])]
    com = ((kept["kind"] >> 1) & 3) == 2
    old = prev.marks[: int(prev.desc[0]["n_mark"])]
    assert (kept["attr"][com] == old["attr"][com] + 1).all()
    _, none = pack_select(prev, [1, 0], [], with_changes=False)
    assert none is None                                    # nothing moves: the identity


def test_a_dropped_comment_rank_shrinks_the_order_and_a_kept_one_refuses():
    logs, _ = comment_and_link_logs()
    prev = pack_logs(logs)                                 # c-d is named only by log 0
    got = apply_select(prev, [1], None, [0, 1, SELECT_DROPPED])
    assert [c["id"] for c in got.comment_ids] == ["c-b", "c-c"]
    assert_same_logs(got, pack_logs([logs[1]]))
    with pytest.raises(ValueError, match="comment"):
        apply_select(prev, [0], None, [0, 1, SELECT_DROPPED])
    with pytest.raises(ValueError, match="comment"):
        apply_select(prev, [0], None, [0, 1])              # rank 2 is outside the map


def test_mismatched_entries_are_refused():
    logs = kat_logs()[:2]
    prev = pack_logs(logs)
    added, _ = pack_select(prev, [A], [logs[0]], with_changes=False)
    with pytest.raises(ValueError):
        pack_select(prev, [A, A], [logs[0]], with_changes=False)
    with pytest.raises(ValueError):
        apply_select(prev, [0, A, A], added)
    with pytest.raises(ValueError):
        apply_select(prev, [2], None)
