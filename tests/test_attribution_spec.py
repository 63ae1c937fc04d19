"""The host specification of pt_batch_attribute, ``attribution.attribution_runs``, against an independent statement of the same
semantics built from the Change dicts and the oracle's element sequence.

The independent statement: replay the log in a fresh oracle replica; element ``ctr@actor`` was inserted by the change of
``actor`` whose [startOp, startOp + len(ops)) holds ``ctr``; its deletes are the ``del`` ops naming it, matched to their
changes the same way, and the attributed one has the smallest opId in compareOpIds order.  ``attribution_runs`` reads the
packed batch instead (ranks, list-op positions, records), over an element sequence made from the oracle's ``elements()``, so
the two agree only if the packed form carries the attribution.  tests/test_gpu_attribution.py reuses the cases here."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.attribution import (ATTR_BAD_TABLE, ATTR_DELETED_SINCE, ATTR_INSERTED_SINCE, ATTR_LOG_FAILED, ATTR_OK, ATTR_RUN_DT, _AttrView,
                                       attribution_runs)
from peritext_b200.packing import RESULT_DT, MergedBatch, checkout_clocks, elem_refs, pack_logs, parse_op_id
from tests.harness import generateDocs
from tests.test_append_packing import kat_logs, sparse_logs
from tests.test_checkout_model import SESSIONS, clock_of, session

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# The independent statement
# ------------------------------------------------------------------------------------------------------------------
def replay(log):
    d = O("~reader")
    for ch in log:
        d.applyChange(ch)
    return d


def _op_key(op_id):
    ctr, actor = parse_op_id(op_id)
    return ctr, actor.encode("utf-16-be")          # compareOpIds: counter, then actor id in JS string order


def semantic_runs(log, clock=None):
    """Runs of `log` by actor id: [(elem, visible, n, flags, (ins actor, ins seq), (del actor, del seq) or None)]."""
    owner = lambda actor, ctr: next(ch for ch in log if ch["actor"] == actor and ch["startOp"] <= ctr < ch["startOp"] + len(ch["ops"]))
    covered = lambda ch: clock is None or ch["seq"] <= clock.get(ch["actor"], 0)
    dels: dict = {}
    for ch in log:
        for j, op in enumerate(ch["ops"]):
            if op["action"] == "del":
                dels.setdefault(op["elemId"], []).append((_op_key(f"{ch['startOp'] + j}@{ch['actor']}"), ch))
    runs, prev, visible = [], None, 0
    for e, el in enumerate(replay(log).elements()):
        ctr, actor = parse_op_id(el["elemId"])
        ic = owner(actor, ctr)
        ds = dels.get(el["elemId"], [])
        dc = min(ds, key=lambda x: x[0])[1] if ds else None
        flags = (0 if covered(ic) else ATTR_INSERTED_SINCE) | (ATTR_DELETED_SINCE if ds and not any(covered(c) for _, c in ds) else 0)
        tup = ((ic["actor"], ic["seq"]), None if dc is None else (dc["actor"], dc["seq"]), flags)
        assert (dc is not None) == el["deleted"]
        if tup != prev:
            runs.append([e, visible, 0, flags, tup[0], tup[1]])
            prev = tup
        runs[-1][2] += 1
        visible += not el["deleted"]
    return [tuple(r) for r in runs]


def by_id(batch, i, rows):
    """ATTR_RUN_DT rows of log i in the semantic form (actor ranks -> ids)."""
    ids = batch.log_actors[i]
    return [(int(r["elem"]), int(r["visible"]), int(r["n"]), int(r["flags"]), (ids[int(r["ins_actor"])], int(r["ins_seq"])),
             None if int(r["del_seq"]) == 0 else (ids[int(r["del_actor"])], int(r["del_seq"]))) for r in rows]


def oracle_merged(batch, logs):
    """A MergedBatch holding only what attribution reads, the element sequences, made from the oracle's elements()."""
    seqs = []
    for i, log in enumerate(logs):
        els = replay(log).elements()
        refs, ok = elem_refs(batch, [i] * len(els), [e["elemId"] for e in els])
        assert ok.all()
        ins, _ = batch.log_slice(i)
        at = {(int(r["ctr"]), int(r["actor"])): j for j, r in enumerate(ins) if int(r["payload"]) >> 30 == 0}
        seqs.append(np.array([at[(int(f["ctr"]), int(f["actor"]))] | (int(e["deleted"]) << 31) for f, e in zip(refs, els)], np.uint32))
    res = np.zeros(len(logs), RESULT_DT)
    res["n_elems"] = [len(s) for s in seqs]
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.uint64)
    seq = np.concatenate(seqs + [np.zeros(0, np.uint32)])
    z = np.zeros(0, np.uint32)
    return MergedBatch(res, off[:-1], off[:-1], z, np.zeros(0, np.uint8), z, seq=seq, seq_off=off[:-1])


def check(logs, clocks=None):
    """attribution_runs == semantic_runs for every log, without a clock and at each clock of `clocks` (by actor id)."""
    batch = pack_logs(logs, with_changes=True)
    merged = oracle_merged(batch, logs)
    lg = list(range(len(logs)))
    st, off, runs = attribution_runs(batch, merged, lg)
    assert (st == ATTR_OK).all()
    for i in lg:
        assert by_id(batch, i, runs[int(off[i]): int(off[i + 1])]) == semantic_runs(logs[i]), i
    for clk in clocks or []:
        keep = [{a: s for a, s in clk.items() if a in batch.log_actors[i] or s} for i in lg]
        ok = [i for i in lg if all(a in batch.log_actors[i] for a in keep[i])]
        st, off, runs = attribution_runs(batch, merged, ok, clock=checkout_clocks(batch, ok, [keep[i] for i in ok]))
        assert (st == ATTR_OK).all()
        for k, i in enumerate(ok):
            assert by_id(batch, i, runs[int(off[k]): int(off[k + 1])]) == semantic_runs(logs[i], keep[i]), (i, clk)
    return batch, merged


# ------------------------------------------------------------------------------------------------------------------
# Cases
# ------------------------------------------------------------------------------------------------------------------
def concurrent_deletes(order):
    """One element deleted by three actors concurrently (and a neighbour by one), delivered in the given arrival order."""
    reps, _, init = generateDocs(O, "abcd", 3)
    cs = [reps[r].change([{"path": ["text"], "action": "delete", "index": 1, "count": 1 + (r == 2)}])["change"] for r in range(3)]
    return [init] + [cs[r] for r in order]


def deletes_cases():
    return [concurrent_deletes(o) for o in ((0, 1, 2), (2, 1, 0), (1, 2, 0))]


def prefix_clocks(logs, stride=4):
    return [clock_of(lg[:j]) for lg in logs for j in range(0, len(lg) + 1, stride)]


def test_kat_logs_both_replicas():
    logs = kat_logs()
    check(logs, prefix_clocks(logs, stride=3)[:40])


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions(seed, kw):
    _, logs = session(seed, kw)
    check(logs, prefix_clocks(logs, stride=9))


def test_sparse_and_dense_counters():
    logs, _ = sparse_logs()
    batch, _ = check(logs, prefix_clocks(logs, stride=1))
    assert any(c is not None for c in batch.log_counters)


def test_concurrent_deletes_take_the_smallest_opid_in_either_arrival_order():
    logs = deletes_cases()
    batch, merged = check(logs, [clock_of(lg[:2]) for lg in logs])
    st, off, runs = attribution_runs(batch, merged, range(len(logs)))
    per = [by_id(batch, i, runs[int(off[i]): int(off[i + 1])]) for i in range(len(logs))]
    assert per[0] == per[1] == per[2]
    # all three deletes are 6@docN, so 6@doc1 (doc1 seq 2, uncovered) is attributed; doc3's covered delete still clears the flag
    clk = {"doc1": 1, "doc3": 1}
    keep = checkout_clocks(batch, [0], [clk])
    st, off, runs = attribution_runs(batch, merged, [0], clock=keep)
    assert [int(r["flags"]) & ATTR_DELETED_SINCE for r in runs if int(r["del_seq"])] == [0] * sum(1 for r in runs if int(r["del_seq"]))


def test_converged_replicas_give_identical_runs():
    _, logs = session(7, {})
    batch, merged = check(logs)
    st, off, runs = attribution_runs(batch, merged, range(len(logs)))
    per = [by_id(batch, i, runs[int(off[i]): int(off[i + 1])]) for i in range(len(logs))]
    assert all(p == per[0] for p in per)


def test_statuses_and_refusals():
    logs = kat_logs()[:2]
    batch = pack_logs(logs, with_changes=True)
    merged = oracle_merged(batch, logs)
    merged.results["status"][1] = 7
    bad = pack_logs(logs, with_changes=True)
    bad.changes.changes["n_ops"][int(bad.changes.desc[0]["change_off"])] += 1
    assert attribution_runs(batch, merged, [0, 1, 1])[0].tolist() == [ATTR_OK, ATTR_LOG_FAILED, ATTR_LOG_FAILED]
    assert attribution_runs(bad, merged, [0])[0].tolist() == [ATTR_BAD_TABLE]
    with pytest.raises(ValueError):
        attribution_runs(batch, merged, [2])
    with pytest.raises(ValueError):
        attribution_runs(batch, merged, [0], clock=(np.array([0, 2], np.uint64), np.array([(0, 1), (0, 2)], [("actor", "<u4"), ("seq", "<u4")])))
    st, off, runs = attribution_runs(batch, merged, [])
    assert len(st) == 0 and off.tolist() == [0] and len(runs) == 0


def test_struct_layouts_match_header(tmp_path):
    """ATTR_RUN_DT and _AttrView have the header's sizes and offsets, checked by the C compiler."""
    lines = ['#include "peritext_b200.h"']
    dt_fields = [(f, ATTR_RUN_DT.fields[f][1], ATTR_RUN_DT.fields[f][0].itemsize) for f in ATTR_RUN_DT.names]
    view_fields = [(f, getattr(_AttrView, f).offset, getattr(_AttrView, f).size) for f, *_ in _AttrView._fields_]
    for t, size, fields in (("pt_attr_run", ATTR_RUN_DT.itemsize, dt_fields), ("pt_attr_view", ctypes.sizeof(_AttrView), view_fields)):
        lines.append(f'_Static_assert(sizeof({t}) == {size}, "sizeof({t}) is not {size}");')
        for f, o, s in fields:
            lines.append(f'_Static_assert(offsetof({t}, {f}) == {o}, "offsetof({t}, {f}) is not {o}");')
            lines.append(f'_Static_assert(sizeof((({t}*)0)->{f}) == {s}, "sizeof({t}.{f}) is not {s}");')
    src = tmp_path / "attr_layouts.c"
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run(["gcc", "-std=c11", "-fsyntax-only", "-include", "stddef.h", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
