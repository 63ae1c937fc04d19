"""The host specification of pt_batch_restore, ``restore.restore_inputs``, against the oracle.

A version is checked out with ``packing.apply_checkout`` (so it keeps its source's packed ids, as pt_batch_checkout does), the
element sequences come from the oracle's ``elements()``, and the InputOperations ``restore_inputs`` returns are fed through the
oracle's own ``Micromerge.change`` on a replica of the log: its visible text must then equal the version's, token for token.
tests/test_gpu_restore.py reuses the cases here."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from peritext_b200.packing import apply_checkout, checkout_clocks, pack_logs
from oracle.packed import replay_packed
from peritext_b200.packing import canon
from peritext_b200.restore import (DELETE, KEEP, NOTHING, RESTORE, RESTORE_BAD_TABLE, RESTORE_FOREIGN, RESTORE_LOG_FAILED, RESTORE_MARKS, RESTORE_OK,
                                   RESTORE_REQUEST_DT, RESTORE_TEXT_DIFFERS, _RestoreView, marks_inputs, restore_change_record, restore_inputs,
                                   restore_runs)
from tests.harness import generateDocs
from tests.test_append_packing import kat_logs, sparse_logs
from tests.test_attribution_spec import deletes_cases, oracle_merged
from tests.test_checkout_model import SESSIONS, clock_of, covered, session

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def replay(changes, actor="~reader"):
    d = O(actor)
    for ch in changes:
        d.applyChange(ch)
    return d


def text(d):
    return "".join(s["text"] for s in d.getTextWithFormatting())


def versions_of(logs, stride=1, cross=True):
    """(source log, covered changes, prefix length or clock by actor id) of every non-empty prefix of every log, and, with
    `cross`, of every log at every other log's final clock that it holds."""
    out = [(i, lg[:j], j) for i, lg in enumerate(logs) for j in range(1, len(lg) + 1, stride)]
    if cross:
        out += [(i, covered(lg, clock_of(other)), clock_of(other)) for i, lg in enumerate(logs) for other in logs
                if other is not lg and all(clock_of(lg).get(a, 0) >= s for a, s in clock_of(other).items())]
    return [v for v in out if v[1]]                       # the empty version has no text list to replay


def checked_out(logs, versions):
    """(batch with the versions added behind the logs by apply_checkout, the oracle's merge of it, the version logs' indices)."""
    batch = pack_logs(logs, with_changes=True)
    prefix = [(i, v) for i, _, v in versions if isinstance(v, int)]
    clocks = [(i, v) for i, _, v in versions if not isinstance(v, int)]
    co, st = apply_checkout(batch, [i for i, _ in prefix], n_changes=[v for _, v in prefix]) if prefix else (batch, np.zeros(0))
    assert (st == 0).all()
    if clocks:
        keep = [{a: s for a, s in c.items() if a in batch.log_actors[i]} for i, c in clocks]
        co, st = apply_checkout(co, [i for i, _ in clocks], clock=checkout_clocks(co, [i for i, _ in clocks], keep))
        assert (st == 0).all()
    order = [v for v in versions if isinstance(v[2], int)] + [v for v in versions if not isinstance(v[2], int)]
    merged = oracle_merged(co, list(logs) + [cov for _, cov, _ in order])
    return co, merged, [(src, len(logs) + k, cov) for k, (src, cov, _) in enumerate(order)]


def actor_of(batch, i):
    """The actor that makes the restore on log i: its newest change's actor (a replica's own actor after a fuzz session)."""
    cd = batch.changes.desc[i]
    if int(cd["n_changes"]) == 0:
        return batch.log_actors[i][0] if batch.log_actors[i] else "~restorer"
    return batch.log_actors[i][int(batch.changes.changes[int(cd["change_off"]) + int(cd["n_changes"]) - 1]["actor"])]


def check(logs, versions):
    """Every version's restore, through the oracle's change(), gives the version's visible text.  Returns the cases."""
    batch, merged, reqs = checked_out(logs, versions)
    out = []
    for src, ver, cov in reqs:
        st, ops = restore_inputs(batch, merged, src, ver)
        assert st == RESTORE_OK
        actor = actor_of(batch, src)
        d = replay(logs[src], actor)
        want = text(replay(cov))
        if ops:
            r = d.change(ops)
            seq, deps = restore_change_record(batch, src, batch.log_actors[src].index(actor), len(r["change"]["ops"]))
            assert list(r["change"]["deps"].items()) == [(batch.log_actors[src][a], s) for a, s in deps]
            assert seq == clock_of(logs[src]).get(actor, 0) + 1      # a replica that made its own changes (the oracle's applyChange
                                                                    # replay does not advance its seq)
        else:
            assert text(d) == want
        assert text(d) == want, (src, ver, ops)
        out.append((src, ver, ops))
    return batch, merged, out


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_fuzz_sessions_every_prefix_and_cross_clock(seed, kw):
    _, logs = session(seed, kw, steps=40)
    _, _, cases = check(logs, versions_of(logs, stride=2))
    assert any(op["action"] == "insert" for _, _, ops in cases for op in ops)
    assert any(op["action"] == "delete" for _, _, ops in cases for op in ops)


def test_kat_logs():
    logs = kat_logs()
    check(logs, versions_of(logs, cross=False))


def test_sparse_counters_and_concurrent_deletes():
    for logs in (sparse_logs()[0], deletes_cases()):
        check(logs, versions_of(logs))


def tombstone_boundary_log():
    """The "growth behavior for spans where the boundary is a tombstone" corner: a link ends after an element that is then
    deleted, so lookAfterTombstones moves an insert at that index right of the restored elements."""
    d, _, init = generateDocs(O, "abcdefg", 1)
    d = d[0]
    log = [init]
    for inp in ([{"path": ["text"], "action": "addMark", "startIndex": 1, "endIndex": 4, "markType": "link", "attrs": {"url": "a.com"}}],
                [{"path": ["text"], "action": "delete", "index": 2, "count": 3}],
                [{"path": ["text"], "action": "insert", "index": 2, "values": ["X"]}]):
        log.append(d.change(inp)["change"])
    return log


def test_look_after_tombstones_picks_a_tombstone_right_of_restored_elements():
    log = tombstone_boundary_log()
    batch, merged, cases = check([log], versions_of([log], cross=False))
    # the sequence is a b c d X e f g with c d e deleted and d's after slot defined (the link's end).  Restoring the version
    # before the delete re-inserts "cd" at index 2: its reference is the last tombstone with a defined after slot, "d", right
    # of the old "c"; then X goes and "e" comes back after it
    ops = dict(((s, v), o) for s, v, o in cases)[(0, 2)]
    assert ops == [{"path": ["text"], "action": "insert", "index": 2, "values": list("cd")},
                   {"path": ["text"], "action": "delete", "index": 4, "count": 1},
                   {"path": ["text"], "action": "insert", "index": 4, "values": ["e"]}]
    d = replay(log, "doc1")
    els = d.elements()
    assert [e["deleted"] for e in els[2:6]] == [True, True, False, True] and els[3]["after"]
    assert d.change(ops)["change"]["ops"][0]["elemId"] == els[3]["elemId"]


def test_version_equal_to_log_is_nothing_to_do():
    _, logs = session(7, {}, steps=30)
    batch = pack_logs(logs, with_changes=True)
    merged = oracle_merged(batch, logs)
    for i in range(len(logs)):
        assert restore_inputs(batch, merged, i, i) == (RESTORE_OK, [])


def test_run_formation_and_op_order():
    c = lambda s: [({"k": KEEP, "d": DELETE, "r": RESTORE, "n": NOTHING}[ch], k) for k, ch in enumerate(s)]
    assert restore_runs(c("")) == []
    assert restore_runs(c("kkk")) == []
    assert restore_runs(c("dndd")) == [(DELETE, 0, 3)]                      # "nothing" does not break a run
    assert restore_runs(c("rnrkr")) == [(RESTORE, 0, [0, 2]), (RESTORE, 3, [4])]   # a kept element does
    assert restore_runs(c("kdrdk")) == [(DELETE, 1, 1), (RESTORE, 1, [2]), (DELETE, 2, 1)]
    assert restore_runs(c("rrddrr")) == [(RESTORE, 0, [0, 1]), (DELETE, 2, 2), (RESTORE, 2, [4, 5])]


def test_foreign_and_statuses():
    _, logs = session(7, {}, steps=30)
    other = kat_logs()[:1]
    batch = pack_logs(logs + other, with_changes=True)
    merged = oracle_merged(batch, logs + other)
    n = len(logs)
    assert restore_inputs(batch, merged, 0, n)[0] == RESTORE_FOREIGN              # another document's elements
    # a version whose elements are the log's in another order
    co, _, reqs = checked_out(logs, [(0, logs[0], len(logs[0]))])
    m2 = oracle_merged(co, list(logs) + [logs[0]])
    ver = reqs[0][1]
    o = int(m2.seq_off[ver]); k = int(m2.results[ver]["n_elems"])
    assert k >= 2
    m2.seq[o: o + k] = m2.seq[o: o + k][::-1].copy()
    assert restore_inputs(co, m2, 0, ver)[0] == RESTORE_FOREIGN
    merged.results["status"][1] = 7
    assert restore_inputs(batch, merged, 1, 0)[0] == RESTORE_LOG_FAILED
    assert restore_inputs(batch, merged, 0, 1)[0] == RESTORE_LOG_FAILED
    bad = pack_logs(logs + other, with_changes=True)
    bad.changes.changes["n_ops"][int(bad.changes.desc[0]["change_off"])] += 1
    assert restore_inputs(bad, merged, 0, 0)[0] == RESTORE_BAD_TABLE
    with pytest.raises(ValueError):
        restore_inputs(batch, merged, 0, 0, mode=3)


def test_struct_layouts_match_header(tmp_path):
    """RESTORE_REQUEST_DT and _RestoreView have the header's sizes and offsets, checked by the C compiler."""
    lines = ['#include "peritext_b200.h"']
    dt_fields = [(f, RESTORE_REQUEST_DT.fields[f][1], RESTORE_REQUEST_DT.fields[f][0].itemsize) for f in RESTORE_REQUEST_DT.names]
    view_fields = [(f, getattr(_RestoreView, f).offset, getattr(_RestoreView, f).size) for f, *_ in _RestoreView._fields_]
    for t, size, fields in (("pt_restore_request", RESTORE_REQUEST_DT.itemsize, dt_fields), ("pt_restore_view", ctypes.sizeof(_RestoreView), view_fields)):
        lines.append(f'_Static_assert(sizeof({t}) == {size}, "sizeof({t}) is not {size}");')
        for f, o, s in fields:
            lines.append(f'_Static_assert(offsetof({t}, {f}) == {o}, "offsetof({t}, {f}) is not {o}");')
            lines.append(f'_Static_assert(sizeof((({t}*)0)->{f}) == {s}, "sizeof({t}.{f}) is not {s}");')
    src = tmp_path / "restore_layouts.c"
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run(["gcc", "-std=c11", "-fsyntax-only", "-include", "stddef.h", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ------------------------------------------------------------------------------------------------------------------
# MARKS
# ------------------------------------------------------------------------------------------------------------------
def oracle_formats(d):
    """position_formats' tuples from the oracle's getTextWithFormatting (one position per character)."""
    out = []
    for sp in d.getTextWithFormatting():
        m = sp["marks"]
        out += [("strong" in m, "em" in m, m.get("link"), {c["id"]: c for c in m.get("comment", [])})] * len(sp["text"])
    return out


def normalised(d):
    """Per character the canonical marks, the `comment` key without ids (quirk Q3) dropped."""
    out = []
    for sp in d.getTextWithFormatting():
        m = {k: v for k, v in sp["marks"].items() if not (k == "comment" and v == [])}
        out += [canon(m)] * len(sp["text"])
    return out


def check_full(logs, versions):
    """TEXT, then MARKS from the formatting the restored text inherits, through the oracle's change(): the document then has
    the version's text and, position for position, its formatting."""
    batch, merged, reqs = checked_out(logs, versions)
    n_marks = 0
    for src, ver, cov in reqs:
        st, ops = restore_inputs(batch, merged, src, ver)
        assert st == RESTORE_OK
        d = replay(logs[src], actor_of(batch, src))
        if ops:
            d.change(ops)
        v = replay(cov)
        mops = marks_inputs(oracle_formats(d), oracle_formats(v))
        if mops:
            d.change(mops)
            n_marks += len(mops)
        assert text(d) == text(v) and normalised(d) == normalised(v), (src, ver, mops)
        assert not marks_inputs(oracle_formats(d), oracle_formats(v))
    return n_marks


@pytest.mark.parametrize("seed,kw", SESSIONS)
def test_marks_after_text_give_the_version_formatting(seed, kw):
    _, logs = session(seed, kw, steps=40)
    assert check_full(logs, versions_of(logs, stride=3)) > 0


def test_marks_on_kat_logs_and_the_tombstone_corner():
    logs = kat_logs()
    assert check_full(logs, versions_of(logs, cross=False)) > 0
    check_full([tombstone_boundary_log()], versions_of([tombstone_boundary_log()], cross=False))


def test_marks_op_order_and_ranges():
    c = lambda *ids: {i: {"id": i} for i in ids}
    L = {"url": "a"}
    have = [(False, False, None, {}), (True, False, L, c("b")), (True, False, L, c("b")), (False, False, None, {})]
    want = [(True, False, None, c("a")), (True, False, None, c("a", "b")), (False, True, {"url": "x"}, {}), (False, False, None, {})]
    got = [(o["startIndex"], o["endIndex"], o["action"], o["markType"], (o.get("attrs") or {}).get("id", (o.get("attrs") or {}).get("url"))) for o in marks_inputs(have, want)]
    assert got == [(0, 1, "addMark", "strong", None), (0, 2, "addMark", "comment", "a"),
                   (1, 2, "removeMark", "link", None), (2, 3, "removeMark", "strong", None), (2, 3, "addMark", "em", None),
                   (2, 3, "removeMark", "comment", "b"), (2, 3, "addMark", "link", "x")]
    assert marks_inputs(want, want) == []


def test_marks_statuses_on_a_merged_batch():
    _, logs = session(7, {}, steps=30)
    batch, _, reqs = checked_out(logs, [(0, logs[0][:2], 2)])
    merged = replay_packed(batch)[0]
    assert restore_inputs(batch, merged, 0, 0, RESTORE_MARKS) == (RESTORE_OK, [])
    assert restore_inputs(batch, merged, 0, reqs[0][1], RESTORE_MARKS)[0] == RESTORE_TEXT_DIFFERS
