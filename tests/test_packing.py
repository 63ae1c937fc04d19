"""Sub-batches of a batch that carries a change table (the admission pre-pass): ``slice_logs`` and ``select`` of a
PackedBatch, and ``slice_logs`` of its run-compressed form, must give every log the same change and dependency rows as
the whole batch, with offsets re-based to the sub-batch."""
import numpy as np

from oracle.oracle import Micromerge as O
from peritext_b200.packing import pack_logs
from tests.harness import fuzz_session


def log_changes(table, i):
    d = table.desc[i]
    c0, p0 = int(d["change_off"]), int(d["dep_off"])
    return (table.changes[c0: c0 + int(d["n_changes"])].tobytes(), table.deps[p0: p0 + int(d["n_deps"])].tobytes(),
            int(d["n_changes"]), int(d["n_deps"]))


def sessions():
    logs = []
    for seed in range(3):
        _, lg, _ = fuzz_session(O, 700 + seed, 40)
        logs += lg
    return pack_logs(logs, with_changes=True)


def assert_sub_table(sub, whole, idx):
    t = sub.changes
    assert t is not None and len(t.desc) == sub.n_logs == len(idx)
    assert int(t.desc["n_changes"].sum()) == len(t.changes) and int(t.desc["n_deps"].sum()) == len(t.deps)
    if len(idx):
        assert int(t.desc[0]["change_off"]) == 0 and int(t.desc[0]["dep_off"]) == 0
    for k, i in enumerate(idx):
        assert log_changes(t, k) == log_changes(whole.changes, i), (idx, i)


def test_slice_logs_and_select_carry_the_change_table():
    b = sessions()
    n = b.n_logs
    assert n == 9 and len(b.changes.deps)
    for a, e in [(0, n), (0, 1), (2, 7), (n - 1, n), (4, 4)]:
        assert_sub_table(b.slice_logs(a, e), b, list(range(a, e)))
    for idx in ([8, 0, 5], [3], [], [1, 1, 2]):
        assert_sub_table(b.select(idx), b, idx)


def test_run_slices_carry_the_change_table():
    from peritext_b200.engine import compress_runs
    b = sessions()
    r = compress_runs(b)
    assert r.changes is b.changes
    for a, e in [(0, 4), (4, 9), (3, 3)]:
        s = r.slice_logs(a, e)
        assert_sub_table(s, b, list(range(a, e)))
        assert np.array_equal(s.desc["n_insdel"], b.desc["n_insdel"][a:e])
