"""PT_FLAG_EMIT_LARGE_PATCHES: the device Patch stream of logs too large for the warp patch kernel (`patch_large_kernel`,
csrc/patch_large_kernel.cuh), against the oracle's `applyChange` return values.

With the flag a log's patch status is 1 only if its merge failed; every other log is computed, by the warp kernel or by the
CTA-per-log arrival sweep, and the two are indistinguishable in the outputs.  `PT_PATCH_WARP=0` (read at upload) skips the
warp kernel and sends every log to the sweep, so the corner catalogue of tests/test_gpu_patch_bounds.py reaches it.  The
sweep walks the list ops in chunks of 512 (`kLargeChunk`); the chunk tests put ops on both sides of a chunk edge."""
from collections import Counter
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import pack_logs, patch_stream
from tests.harness import environ, fuzz_session
from tests.test_gpu_admission import tampered_logs
from tests.test_gpu_patch_bounds import (cap_cases, corner_cases, encode, exact_case, list_ops, log_changes, marks_then_edits, named_cases,
                                         oracle_per_op, splice)
from tests.test_gpu_patch_window import check_window, merge_all
from tests.test_gpu_routes import COMMENT, EM, FAULTS, LINK, STRONG, batch_of, lamport_forward, with_fault

CHUNK = 512


def large_engine():
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, large_patches=True)


@pytest.fixture(scope="module")
def lengine():
    e = large_engine()
    yield e
    e.close()


def large_pass(e, batch, warp=True):
    """One device pass with the flag (warp=False: every log through the sweep), re-merged once with the pool demand."""
    with environ({"PT_PATCH_WARP": None if warp else "0"}):
        merged = e.run(batch)
    recs, items, status, needed = e.download_patches()
    if needed > len(items):
        e.set_patch_pool(needed + 16)
        e.merge(); merged = e.download()
        recs, items, status, needed = e.download_patches()
    return merged, recs, items, status, needed


def check_large(batch, logs, out, names=None):
    """Status == "the merge failed"; every computed log equal to the oracle, decoded and raw; demand == the oracle's count."""
    from peritext_b200.packing import DevicePatches
    merged, recs, items, status, needed = out
    names = names or [str(i) for i in range(batch.n_logs)]
    want = [int(s != 0) for s in merged.results["status"]]
    assert status.tolist() == want, [(n, int(s), w) for n, s, w in zip(names, status, want) if s != w]
    assert len(items) == needed
    got_items = Counter(tuple(int(x) for x in it) for it in items.tolist())
    dp = DevicePatches(recs, items, status)
    total = 0
    for i, log in enumerate(logs):
        mine = Counter({k: v for k, v in got_items.items() if k[0] == i})
        if status[i]:
            assert not mine, names[i]
            continue
        ops = list_ops(log)
        per_op, elements = oracle_per_op(log)
        assert patch_stream(batch, dp, i, ops) == per_op, names[i]
        want_recs, want_items = encode(batch, i, ops, per_op, elements)
        o, n = int(batch.desc[i]["insdel_off"]), int(batch.desc[i]["n_insdel"])
        assert [tuple(int(x) for x in r) for r in recs[o:o + n].tolist()] == want_recs, names[i]
        assert mine == want_items, names[i]
        total += sum(want_items.values())
    assert needed == total
    return want


# ------------------------------------------------------------------------------------------------------------------
# 1. Every named case through the sweep, alone and in one mixed batch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(named_cases()))
def test_each_case_alone_through_the_sweep(lengine, name):
    c = named_cases()[name]
    batch = pack_logs([c.changes])
    assert check_large(batch, [c.changes], large_pass(lengine, batch, warp=False), [c.name]) == [0]


@pytest.mark.gpu
def test_all_cases_in_one_mixed_batch_through_the_sweep(lengine):
    cases = list(named_cases().values()) + list(cap_cases())
    logs = [c.changes for c in cases]
    batch = pack_logs(logs)
    assert set(check_large(batch, logs, large_pass(lengine, batch, warp=False), [c.name for c in cases])) == {0}


# ------------------------------------------------------------------------------------------------------------------
# 2. The logs the warp kernel declines, with default routing; both kernels in one batch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_declined_logs_are_computed_with_default_routing(lengine):
    below, above = cap_cases()
    ks = named_cases()["keyspace-65535"]
    for cases in ([ks], [above], [above, below], corner_cases()[:6] + [ks, above] + corner_cases()[6:]):
        logs = [c.changes for c in cases]
        batch = pack_logs(logs)
        assert set(check_large(batch, logs, large_pass(lengine, batch), [c.name for c in cases])) == {0}


@pytest.mark.gpu
def test_sweep_and_warp_kernel_give_identical_arrays(lengine):
    cases = corner_cases() + [exact_case("marks-65", marks_then_edits(80, 65, (STRONG, EM, LINK, COMMENT), seed=65))]
    batch = pack_logs([c.changes for c in cases])
    a = large_pass(lengine, batch)
    b = large_pass(lengine, batch, warp=False)
    assert a[1].tobytes() == b[1].tobytes() and a[3].tobytes() == b[3].tobytes() and a[4] == b[4]
    assert np.sort(a[2], order=("log", "tag", "a", "b")).tobytes() == np.sort(b[2], order=("log", "tag", "a", "b")).tobytes()


# ------------------------------------------------------------------------------------------------------------------
# 3. Chunk edges
# ------------------------------------------------------------------------------------------------------------------
def chunk_cases():
    out = []
    for total in (CHUNK - 1, CHUNK, CHUNK + 1):
        out.append(exact_case("typing-%d" % total, lamport_forward(total - 12, 2, 12, seed=total, width=30)))
    # marks over text typed in the first chunk, then inserts inside them and delete pairs (a delete and its second delete
    # adjacent): the covering mark ops and the inserts fall in one chunk and in different chunks
    for n_text, n_marks in ((300, 40), (700, 65), (1100, 300)):
        out.append(exact_case("marks-%d-%d" % (n_text, n_marks), marks_then_edits(n_text, n_marks, (STRONG, EM, LINK, COMMENT), seed=n_text)))
    return out


@pytest.mark.gpu
def test_chunk_edges(lengine):
    cases = chunk_cases()
    assert [c.shape[0] + c.shape[1] for c in cases[:3]] == [CHUNK - 1, CHUNK, CHUNK + 1]
    logs = [c.changes for c in cases]
    batch = pack_logs(logs)
    check_large(batch, logs, large_pass(lengine, batch, warp=False), [c.name for c in cases])
    for c in cases:
        b1 = pack_logs([c.changes])
        check_large(b1, [c.changes], large_pass(lengine, b1, warp=False), [c.name])


# ------------------------------------------------------------------------------------------------------------------
# 4. Windows on declined-size logs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_windows_on_declined_logs_equal_the_whole_log_tail():
    _, above = cap_cases()
    ks = named_cases()["keyspace-65535"]
    logs = [above.changes, ks.changes]
    batch = pack_logs(logs)
    tot = [int(d["n_insdel"]) + int(d["n_mark"]) for d in batch.desc]
    e = large_engine()
    try:
        e.upload(batch)
        whole = merge_all(e, batch)
        assert (whole[3] == 0).all()
        check_large(batch, logs, (SimpleNamespace(results=whole[0]), *whole[1:5]))
        cuts = [0, 1, CHUNK - 1, CHUNK, CHUNK + 1, 5000, None, "last", "end"]
        for cut in cuts:
            w = []
            for i in range(batch.n_logs):
                if cut is None:
                    w.append(tot[i] // 2)
                elif cut == "last":
                    w.append(tot[i] - 1)
                elif cut == "end":
                    w.append(tot[i])
                else:
                    w.append(min(cut, tot[i]))
            w = np.array(w, np.uint32)
            e.set_patch_window(w)
            win = merge_all(e, batch)
            check_window(batch, whole, win, w)
            # a pool of exactly the window's demand
            e.set_patch_pool(max(1, win[4]))
            e.merge(); e.download()
            _, items, _, needed = e.download_patches()
            assert needed == win[4] and len(items) == needed
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. Failed and admission-rejected logs; the pool overflow rule
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("warp", [True, False])
def test_failed_logs_stay_uncomputed_and_leave_no_items(lengine, warp):
    faults = [f for f in FAULTS if f != "clean"]
    clean_logs = [fuzz_session(O, 3500 + s, 40)[1][s % 3] for s in range(len(faults) + 1)]
    clean = pack_logs(clean_logs)
    bad = batch_of([with_fault(lamport_forward(120, 2, 8, seed=k), f) for k, f in enumerate(faults)])
    parts, logs = [], []
    for k in range(len(faults)):
        parts += [(clean, k), (bad, k)]; logs += [clean_logs[k], None]
    parts.append((clean, len(faults))); logs.append(clean_logs[-1])
    batch = splice(parts)
    out = large_pass(lengine, batch, warp)
    st = check_large(batch, logs, out)
    assert st[1::2] == [1] * len(faults) and set(st[0::2]) == {0}
    cases = tampered_logs()
    logs = [log for _, log in cases]
    batch = pack_logs(logs, with_changes=True)
    out = large_pass(lengine, batch, warp)
    rs = out[0].results["status"]
    assert {6, 7} <= set(rs.tolist()) and 0 in rs.tolist()
    assert check_large(batch, [log if s == 0 else None for log, s in zip(logs, rs)], out, [n for n, _ in cases]) == [int(s != 0) for s in rs]


@pytest.mark.gpu
def test_pool_overflow_reports_the_exact_demand_and_one_retry_succeeds():
    _, above = cap_cases()
    cases = corner_cases() + [above]
    logs = [c.changes for c in cases]
    batch = pack_logs(logs)
    e = large_engine()
    try:
        full = large_pass(e, batch)
        check_large(batch, logs, full)
        e.set_patch_pool(full[4] // 3)
        e.merge(); e.download()
        recs, items, status, needed = e.download_patches()
        assert needed == full[4] and len(items) == full[4] // 3 and recs.tobytes() == full[1].tobytes()
        assert not (Counter(map(tuple, items.tolist())) - Counter(map(tuple, full[2].tolist())))
        e.set_patch_pool(needed)
        e.merge(); merged = e.download()
        check_large(batch, logs, (merged, *e.download_patches()))
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 6. The facade with an opted-in engine
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_facade_takes_the_device_stream_past_the_key_space_guard():
    from peritext_b200 import Micromerge
    chs = named_cases()["keyspace-65535"].changes
    want, _ = oracle_per_op(chs)
    want = [p for ps in want for p in ps]
    e = large_engine()
    try:
        doc = Micromerge("reader", engine=e)
        head = doc.applyChanges(chs[:-40])
        tail = doc.applyChanges(chs[-40:])
        assert int(doc._cache[2].status[0]) == 0            # at KS = 65535 the device computed the patches
        assert [p for p in head if p["action"] != "makeList"] + tail == want
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------------
# 7. More candidate logs than CTAs: one scratch slot reused for several logs, skipped candidates between them
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_more_logs_than_ctas_with_failed_logs_interleaved(lengine):
    # every log through the sweep: more than one candidate per CTA, merge-failed candidates (skipped) between computed ones
    faults = [f for f in FAULTS if f != "clean"]
    bad = batch_of([with_fault(lamport_forward(120, 2, 8, seed=k), f) for k, f in enumerate(faults)])
    good, seed = [], 0
    while len(good) < 330:
        good += fuzz_session(O, 3700 + seed, 30, remove_comments=bool(seed % 2))[1]; seed += 1
    clean = pack_logs(good)
    parts, logs = [], []
    for k in range(len(good)):
        parts.append((clean, k)); logs.append(good[k])
        if k % 37 == 5:
            parts.append((bad, (k // 37) % len(faults))); logs.append(None)
    batch = splice(parts)
    st = check_large(batch, logs, large_pass(lengine, batch, warp=False))
    assert batch.n_logs > 300 and st.count(1) == sum(1 for lg in logs if lg is None)


@pytest.mark.gpu
def test_more_declined_logs_than_ctas_with_warp_computed_candidates(lengine):
    # default routing: `above` next to `below` is a candidate that the warp kernel computes (skipped by the sweep), the key-space
    # logs are computed by the sweep; the skipped ones come first, so some CTAs skip a log and then compute another
    below, above = cap_cases()
    ks = named_cases()["keyspace-65535"]
    cases = [below] + [above] * 4 + [ks] * 140
    logs = [c.changes for c in cases]
    batch = pack_logs(logs)
    out = large_pass(lengine, batch)
    assert set(check_large(batch, logs, out)) == {0}


# ------------------------------------------------------------------------------------------------------------------
# 8. The append flow on declined-size logs, the render, the true c5 shape
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("warp", [True, False])
def test_append_then_window_on_declined_logs(warp):
    import json
    from peritext_b200.packing import apply_append, pack_append
    from tests.test_append_packing import split
    from tests.test_gpu_patch_window import per_change_tail
    from tests.test_gpu_render_patches_json import oracle_per_change
    _, above = cap_cases()
    ks = named_cases()["keyspace-65535"]
    logs = [above.changes, ks.changes]
    cut = [len(above.changes) - 30, len(ks.changes) // 2]
    prefix, suffix = split(logs, cut)
    prev = pack_logs(prefix)
    delta, remap = pack_append(prev, suffix)
    full = apply_append(prev, delta, remap)
    e, u = large_engine(), large_engine()
    try:
        with environ({"PT_PATCH_WARP": None if warp else "0"}):
            e.upload(prev)
            merge_all(e, prev)
            e.append(delta, remap)
            u.upload(full)
        old = (prev.desc["n_insdel"].astype(np.int64) + prev.desc["n_mark"].astype(np.int64)).astype(np.uint32)
        e.set_patch_window(old)
        win = merge_all(e, full)
        whole = merge_all(u, full)
        assert (win[3] == 0).all() and (whole[3] == 0).all()
        check_window(full, whole, win, old)
        for i, log in enumerate(logs):
            assert per_change_tail(log, cut[i], json.loads(win[5][i])) == oracle_per_change(log)[cut[i]:], i
    finally:
        e.close(); u.close()


@pytest.mark.gpu
@pytest.mark.parametrize("warp", [True, False])
def test_declined_logs_render_the_spec_bytes(lengine, warp):
    from tests.test_gpu_render_patches_json import check_against_decoder_and_oracle
    below, above = cap_cases()
    ks = named_cases()["keyspace-65535"]
    with environ({"PT_PATCH_WARP": None if warp else "0"}):
        check_against_decoder_and_oracle(lengine, [above.changes, ks.changes, below.changes])


def c5_changes():
    """The true-shape c5 document (workload.generate("c5", n_docs=1), log 0) as JSON changes: its records as they are, insert
    values mapped to lower-case letters."""
    from peritext_b200 import workload
    b = workload.generate("c5", n_docs=1)
    a, m = b.log_slice(0)
    d = b.desc[0]
    ins = [(int(r["ctr"]), int(r["ref_ctr"]), int(r["actor"]), int(r["ref_actor"]),
            (int(r["payload"]) & 0xC0000000) | (97 + (int(r["payload"]) & 0xFFFF) % 26)) for r in a]
    mk = [tuple(int(r[f]) for f in ("ctr", "actor", "kind", "bounds", "start_ctr", "end_ctr", "start_actor", "end_actor", "attr",
                                    "arrival", "reserved")) for r in m]
    lg = SimpleNamespace(ins=ins, mk=mk, m=len(mk), n=len(ins), R=int(d["n_actors"]), max_ctr=int(d["max_ctr"]))
    return log_changes(lg), (int(d["n_insdel"]), int(d["n_mark"]))


@pytest.mark.gpu
def test_true_shape_c5_document(lengine):
    chs, (n, m) = c5_changes()
    batch = pack_logs([chs])
    d = batch.desc[0]
    assert (int(d["n_insdel"]), int(d["n_mark"])) == (n, m) and n > 100000 and m == 10000
    assert int(d["max_ctr"]) * int(d["n_actors"]) >= 0xFFFF          # declined by the warp kernel
    assert check_large(batch, [chs], large_pass(lengine, batch), ["c5"]) == [0]
