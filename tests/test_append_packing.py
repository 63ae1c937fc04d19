"""The host side of pt_batch_append: ``pack_append`` + ``apply_append`` against ``pack_logs`` of the concatenated logs.

``apply_append(pack_logs(prefix), *pack_append(pack_logs(prefix), suffix))`` must equal ``pack_logs(prefix + suffix)`` in
every field: descriptors, actor ranks, counters, arrival, kinds, comment ranks, log_actors, log_counters and the change
table.  Value tokens and link ids may differ (append keeps the old pool indices and gives new strings the next ones), so
they are compared through their pools.  The corpora here are reused by tests/test_gpu_append.py."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import (ATTR_NONE, CTR_UNUSED, TOKEN_POOLED, AppendRemap, PackedBatch, apply_append, canon, pack_append,
                                   pack_logs)
from tests.harness import fuzz_session, generateDocs, load_kats, run_concurrent


# ------------------------------------------------------------------------------------------------------------------
# Corpora of Change logs, each with the split points worth testing
# ------------------------------------------------------------------------------------------------------------------
def kat_logs():
    logs = []
    for kat in [k for k in load_kats() if k["kind"] == "concurrent"]:
        rec = []
        run_concurrent(O, kat, record=rec)
        logs += rec
    return logs


def fuzz_logs():
    logs = []
    for seed, kw in [(11, {}), (2011, dict(replicas=2, max_chars=6, initial="The Peritext editor")),
                     (1011, dict(sync_prob=0.3, full_sync_at_end=False)), (3011, dict(zero_width_prob=0.3))]:
        _, lg, _ = fuzz_session(O, seed, 80, **kw)
        logs += lg
    return logs


def quirk_logs():
    """Multi-code-point values, emoji, U+10FFFF, and a value that only the suffix interns."""
    docs, _, init = generateDocs(O, "ab", 1)
    c1 = docs[0].change([{"path": ["text"], "action": "insert", "index": 1, "values": [" is great!", "é", "\U0001F600"]}])["change"]
    c2 = docs[0].change([{"path": ["text"], "action": "insert", "index": 2, "values": ["\U0010FFFF", "中", "new value", " is great!"]}])["change"]
    return [[init, c1, c2]]


def early_actor_logs():
    """A peer whose actor id sorts before every other ("0peer" < "doc1") arrives in the suffix, in both logs."""
    docs, _, init = generateDocs(O, "abcd", 2)
    p = O("0peer")
    p.applyChange(init)
    c = p.change([{"path": ["text"], "action": "insert", "index": 2, "values": ["x", "y"]},
                  {"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 3, "markType": "strong"}])["change"]
    own = docs[0].change([{"path": ["text"], "action": "delete", "index": 0, "count": 1}])["change"]
    return [[init, own, c], [init, c]]


def comment_and_link_logs():
    """Log 1's suffix adds a comment id that sorts between log 0's; log 0's suffix adds a link url that log 1 already has."""
    d0, _, i0 = generateDocs(O, "abcdefgh", 1)
    d1, _, i1 = generateDocs(O, "ijklmnop", 1)
    a = [d0[0].change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 4, "markType": "comment", "attrs": {"id": "c-b"}}])["change"],
         d0[0].change([{"path": ["text"], "action": "addMark", "startIndex": 2, "endIndex": 6, "markType": "comment", "attrs": {"id": "c-d"}}])["change"]]
    b = [d1[0].change([{"path": ["text"], "action": "addMark", "startIndex": 1, "endIndex": 3, "markType": "link", "attrs": {"url": "y.com"}}])["change"]]
    a2 = [d0[0].change([{"path": ["text"], "action": "addMark", "startIndex": 1, "endIndex": 5, "markType": "link", "attrs": {"url": "z.com"}}])["change"],
          d0[0].change([{"path": ["text"], "action": "addMark", "startIndex": 3, "endIndex": 7, "markType": "link", "attrs": {"url": "y.com"}}])["change"]]
    b2 = [d1[0].change([{"path": ["text"], "action": "addMark", "startIndex": 0, "endIndex": 5, "markType": "comment", "attrs": {"id": "c-c"}}])["change"],
          d1[0].change([{"path": ["text"], "action": "removeMark", "startIndex": 2, "endIndex": 3, "markType": "comment", "attrs": {"id": "c-b"}}])["change"]]
    return [[i0] + a + a2, [i1] + b + b2], [1 + len(a), 1 + len(b)]


def sparse_peer(start=5_000_000):
    """A peer that picks startOp `start` (reference src/micromerge.ts:511 only takes the max)."""
    docs, _, init = generateDocs(O, "abc", 2)
    d1 = docs[0]
    s = str(start)
    big = {"actor": "doc2", "seq": 1, "deps": {"doc1": 1}, "startOp": start, "ops": [
        {"opId": f"{s}@doc2", "action": "set", "obj": "1@doc1", "elemId": "2@doc1", "insert": True, "value": "X"},
        {"opId": f"{start + 1}@doc2", "action": "set", "obj": "1@doc1", "elemId": f"{s}@doc2", "insert": True, "value": "Y"},
        {"opId": f"{start + 2}@doc2", "action": "addMark", "obj": "1@doc1", "start": {"type": "before", "elemId": f"{s}@doc2"},
         "end": {"type": "after", "elemId": "3@doc1"}, "markType": "link", "attrs": {"url": "u"}}]}
    d1.applyChange(big)
    return d1, init, big


def sparse_logs():
    """Plain -> dense (the sparse peer arrives in the suffix) and dense -> plain (200 typed characters bring the op count
    past the counters' spread)."""
    d1, init, big = sparse_peer()
    c = d1.change([{"path": ["text"], "action": "insert", "index": 1, "values": ["Z"]}])["change"]
    e1, init2, big2 = sparse_peer(200)
    grow = e1.change([{"path": ["text"], "action": "insert", "index": 2, "values": list("q" * 200)}])["change"]
    return [[init, big, c], [init2, big2, grow]], [1, 2]


def split(logs, ks):
    return [lg[:k] for lg, k in zip(logs, ks)], [lg[k:] for lg, k in zip(logs, ks)]


def fraction_splits(logs, fracs=(0.0, 0.3, 0.7, 1.0)):
    """Per-log split points: the same fraction of every log (0 and 1 included), and one mixed set."""
    out = [[int(round(f * len(lg))) for lg in logs] for f in fracs]
    out.append([(7 * i) % (len(lg) + 1) for i, lg in enumerate(logs)])
    return out


# ------------------------------------------------------------------------------------------------------------------
# Comparison
# ------------------------------------------------------------------------------------------------------------------
def token_strs(batch):
    tok = batch.insdel["payload"] & 0x3FFFFFFF
    return [batch.values[t & (TOKEN_POOLED - 1)] if t & TOKEN_POOLED else chr(t) for t in tok.tolist()]


def assert_same_batch(got, want, what=""):
    """Field-by-field equality; value tokens and link ids through their pools."""
    assert got.desc.tobytes() == want.desc.tobytes(), what
    for f in ("ctr", "ref_ctr", "actor", "ref_actor"):
        assert np.array_equal(got.insdel[f], want.insdel[f]), (what, f)
    assert np.array_equal(got.insdel["payload"] >> 30, want.insdel["payload"] >> 30), what
    ins = (got.insdel["payload"] >> 30) == 0
    assert [s for s, k in zip(token_strs(got), ins) if k] == [s for s, k in zip(token_strs(want), ins) if k], what
    for f in ("ctr", "actor", "kind", "bounds", "start_ctr", "end_ctr", "start_actor", "end_actor", "arrival", "reserved"):
        assert np.array_equal(got.marks[f], want.marks[f]), (what, f)
    link = ((want.marks["kind"] >> 1) & 3) == 3
    assert np.array_equal(got.marks["attr"][~link], want.marks["attr"][~link]), what

    def url(b, a):
        return None if a == ATTR_NONE else canon(b.link_attrs[a])
    assert [url(got, int(a)) for a in got.marks["attr"][link]] == [url(want, int(a)) for a in want.marks["attr"][link]], what
    assert [canon(c) for c in got.comment_ids] == [canon(c) for c in want.comment_ids], what
    assert sorted(got.values) == sorted(want.values) and sorted(map(canon, got.link_attrs)) == sorted(map(canon, want.link_attrs)), what
    assert got.log_actors == want.log_actors, what
    assert len(got.log_counters) == len(want.log_counters), what
    for a, b in zip(got.log_counters, want.log_counters):
        assert (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b)), what
    assert got.log_lists == want.log_lists, what
    assert (got.changes is None) == (want.changes is None), what
    if want.changes is not None:
        for f in ("desc", "changes", "deps"):
            assert getattr(got.changes, f).tobytes() == getattr(want.changes, f).tobytes(), (what, f)


def appended(prefix, suffix, with_changes=False):
    """(pack_logs(prefix), delta, remap, apply_append of them)."""
    prev = pack_logs(prefix, with_changes=with_changes)
    delta, remap = pack_append(prev, suffix, with_changes=with_changes)
    return prev, delta, remap, apply_append(prev, delta, remap)


def check_split(logs, ks, with_changes=False, what=""):
    prefix, suffix = split(logs, ks)
    _, _, remap, got = appended(prefix, suffix, with_changes)
    assert_same_batch(got, pack_logs(logs, with_changes=with_changes), what)
    return remap


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_changes", [False, True])
@pytest.mark.parametrize("name", ["kats", "fuzz"])
def test_append_equals_packing_the_concatenation(name, with_changes):
    logs = kat_logs() if name == "kats" else fuzz_logs()
    for ks in fraction_splits(logs):
        check_split(logs, ks, with_changes, (name, ks))


@pytest.mark.parametrize("with_changes", [False, True])
def test_quirk_values(with_changes):
    logs = quirk_logs()
    for k in range(len(logs[0]) + 1):
        check_split(logs, [k], with_changes, k)


@pytest.mark.parametrize("with_changes", [False, True])
def test_new_actor_that_sorts_first_renumbers_the_old(with_changes):
    logs = early_actor_logs()
    remap = check_split(logs, [2, 1], with_changes)
    assert remap.actor_map is not None and list(remap.actor_map[:1]) == [1]        # doc1: rank 0 -> 1


def test_new_comment_between_old_ones_and_new_link_in_an_earlier_log():
    logs, ks = comment_and_link_logs()
    prefix, suffix = split(logs, ks)
    prev, delta, remap, got = appended(prefix, suffix)
    assert [c["id"] for c in prev.comment_ids] == ["c-b", "c-d"]
    assert remap.comment_map is not None and list(remap.comment_map) == [0, 2]
    assert [canon(a) for a in delta.link_attrs] == ['{"url":"y.com"}', '{"url":"z.com"}']
    want = pack_logs(logs)
    assert [canon(a) for a in want.link_attrs] == ['{"url":"z.com"}', '{"url":"y.com"}']
    assert_same_batch(got, want)


@pytest.mark.parametrize("with_changes", [False, True])
def test_sparse_counters_switch_between_dense_and_plain(with_changes):
    logs, ks = sparse_logs()
    prev = pack_logs(split(logs, ks)[0], with_changes=with_changes)
    full = pack_logs(logs, with_changes=with_changes)
    assert prev.log_counters[0] is None and full.log_counters[0] is not None          # plain -> dense
    assert prev.log_counters[1] is not None and full.log_counters[1] is None          # dense -> plain
    remap = check_split(logs, ks, with_changes)
    c0 = remap.ctr_map[int(remap.ctr_off[0]): int(remap.ctr_off[1])]
    assert len(c0) == int(prev.desc[0]["max_ctr"]) + 1 and c0[0] == 0
    c1 = remap.ctr_map[int(remap.ctr_off[1]): int(remap.ctr_off[2])]
    assert list(c1) == [int(c) for c in prev.log_counters[1][: int(prev.desc[1]["max_ctr"]) + 1]]
    for ks2 in ([0, 0], [3, 3], [1, 1]):
        check_split(logs, ks2, with_changes, ks2)


def test_unused_plain_counters_map_to_the_unused_marker():
    """A plain log turning dense: old counters that no record names have no dense rank."""
    d1, init, big = sparse_peer()
    gap = d1.change([{"path": ["text"], "action": "insert", "index": 0, "values": ["G"]}])["change"]
    gap = {**gap, "startOp": 9, "ops": [{**gap["ops"][0], "opId": "9@doc1"}]}       # counters 5..8 unused
    prev = pack_logs([[init, gap]])
    assert prev.log_counters[0] is None and int(prev.desc[0]["max_ctr"]) == 9
    delta, remap = pack_append(prev, [[big]])
    cm = list(remap.ctr_map)
    assert cm == [0, CTR_UNUSED, 1, 2, 3] + [CTR_UNUSED] * 4 + [4]        # 1 is the makeList, 5..8 are nobody's
    assert_same_batch(apply_append(prev, delta, remap), pack_logs([[init, gap, big]]))


def test_chained_appends_equal_one_pack():
    logs = fuzz_logs()[:6]
    cuts = [[int(f * len(lg)) for lg in logs] for f in (0.25, 0.5, 0.75, 1.0)]
    cur = pack_logs([lg[:k] for lg, k in zip(logs, cuts[0])])
    for a, b in zip(cuts, cuts[1:]):
        delta, remap = pack_append(cur, [lg[x:y] for lg, x, y in zip(logs, a, b)])
        cur = apply_append(cur, delta, remap)
    assert_same_batch(cur, pack_logs(logs))


def test_identity_append_of_nothing():
    logs = kat_logs()[:4]
    prev = pack_logs(logs)
    delta, remap = pack_append(prev, [[] for _ in logs])
    assert remap == AppendRemap() and len(delta.insdel) == 0 and len(delta.marks) == 0
    assert_same_batch(apply_append(prev, delta, remap), prev)


def test_apply_append_maps_faulty_values_to_all_ones():
    """A resident value outside its map's domain becomes 0xFFFF / 0xFFFFFFFF; HEAD ids keep their actor."""
    logs = early_actor_logs()
    prev = pack_logs(split(logs, [2, 1])[0])
    delta, remap = pack_append(prev, split(logs, [2, 1])[1])
    bad = pack_logs(split(logs, [2, 1])[0])
    i0 = int(bad.desc[0]["insdel_off"])
    bad.insdel[i0]["actor"] = 7                        # >= old n_actors
    bad.insdel[i0 + 1]["ref_ctr"] = 10_000             # > old max_ctr, with a non-identity counter map below
    remap2 = AppendRemap(remap.actor_off, remap.actor_map, np.array([0, int(bad.desc[0]["max_ctr"]) + 1, int(bad.desc[0]["max_ctr"]) + 1 + int(bad.desc[1]["max_ctr"]) + 1], np.uint64),
                         np.concatenate([np.arange(int(bad.desc[0]["max_ctr"]) + 1), np.arange(int(bad.desc[1]["max_ctr"]) + 1)]).astype(np.uint32) * 1)
    got = apply_append(bad, delta, remap2)
    assert int(got.insdel[0]["actor"]) == 0xFFFF and int(got.insdel[1]["ref_ctr"]) == 0xFFFFFFFF
    head = [k for k in range(int(bad.desc[0]["n_insdel"])) if int(bad.insdel[i0 + k]["ref_ctr"]) == 0]
    assert head and all(int(got.insdel[k]["ref_actor"]) == int(bad.insdel[i0 + k]["ref_actor"]) for k in head)


def test_pack_append_refuses_a_mismatched_change_table_setting():
    prev = pack_logs(kat_logs()[:2])
    with pytest.raises(ValueError):
        pack_append(prev, [[], []], with_changes=True)


def test_append_to_sliced_and_selected_batches():
    """slice_logs / select keep each log's text list, actors and counters, so appending to a sub-batch gives the same delta
    as appending to the whole batch (pool indices aside)."""
    logs = fuzz_logs()
    prefix, suffix = split(logs, [len(lg) // 2 for lg in logs])
    prev = pack_logs(prefix)
    whole, _ = pack_append(prev, suffix)
    for sub, idx in ((prev.slice_logs(0, 4), [0, 1, 2, 3]), (prev.select([5, 1, 7]), [5, 1, 7])):
        got, _ = pack_append(sub, [suffix[i] for i in idx])
        want = whole.select(idx)
        assert int(got.desc["n_insdel"].sum()) > 0
        assert got.desc.tobytes() == want.desc.tobytes()
        assert np.array_equal(got.insdel["ctr"], want.insdel["ctr"]) and np.array_equal(got.marks["arrival"], want.marks["arrival"])
        assert got.log_actors == want.log_actors and got.log_lists == want.log_lists


def test_append_without_a_recorded_text_list_raises():
    """A batch that does not record its text lists (native ingest) needs list_ids: the new changes alone rarely name the
    list, and guessing would drop every new op."""
    logs = fuzz_logs()[:3]
    prefix, suffix = split(logs, [len(lg) // 2 for lg in logs])
    prev = pack_logs(prefix)
    bare = PackedBatch(prev.desc, prev.insdel, prev.marks, prev.values, prev.link_attrs, prev.comment_ids, prev.other_attrs,
                       log_actors=prev.log_actors, log_counters=prev.log_counters)
    with pytest.raises(ValueError, match="list_ids"):
        pack_append(bare, suffix)
    got, _ = pack_append(bare, suffix, list_ids=prev.log_lists)
    assert got.desc.tobytes() == pack_append(prev, suffix)[0].desc.tobytes()


def test_counter_map_covers_boundaries_past_the_old_max_ctr():
    """A mark boundary can name an element whose insert arrives later (past the old max_ctr): when the log turns dense its
    counter map still covers that counter, so the boundary gets its rank as in pack_logs of the full log."""
    d1, init, big = sparse_peer()
    docs, _, init = generateDocs(O, "abc", 1)
    mark = {"actor": "doc1", "seq": 2, "deps": {}, "startOp": 5, "ops": [
        {"opId": "5@doc1", "action": "addMark", "obj": "1@doc1", "start": {"type": "before", "elemId": "2@doc1"},
         "end": {"type": "after", "elemId": "7@doc1"}, "markType": "strong"}]}
    ins = {"actor": "doc1", "seq": 3, "deps": {}, "startOp": 6, "ops": [
        {"opId": "6@doc1", "action": "set", "obj": "1@doc1", "elemId": "4@doc1", "insert": True, "value": "u"},
        {"opId": "7@doc1", "action": "set", "obj": "1@doc1", "elemId": "6@doc1", "insert": True, "value": "v"}]}
    logs = [[init, mark, ins, big]]
    prev = pack_logs([[init, mark]])
    assert int(prev.marks[0]["end_ctr"]) == 7 and int(prev.desc[0]["max_ctr"]) == 5
    delta, remap = pack_append(prev, [[ins, big]])
    assert len(remap.ctr_map) == 8
    got = apply_append(prev, delta, remap)
    assert_same_batch(got, pack_logs(logs))
