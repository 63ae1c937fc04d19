"""The merge path of a handle created on a user stream, against the oracle and against a handle on the legacy default stream.

On a user stream `pt_batch_merge` takes two paths the default stream never reaches: from the second merge after an upload, a
splice or a pool change it replays its launch sequence as a CUDA graph (every pointer, capacity and launch shape baked in), and
when bin 0 and a CTA bin both hold logs, CTA bins 1-4 run their own lists on a side stream beside the warp and team kernels
(fork / join).  Every case here merges several times in a row and compares the merges byte for byte (merge 1 direct, the later
ones replayed), compares them with the oracle (``replay_packed``, or the replica's getTextWithFormatting for Change logs) and
with a default-stream handle that holds the host specification of the batch.  A ``torch.profiler`` pass proves that the graph
and the fork really ran, so the comparisons cannot silently turn into default-stream ones."""
import json
import os
import random
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200 import workload
from peritext_b200.packing import (SELECT_ADDED, ChangeTable, apply_append, apply_select, change_extras, decode_spans, pack_append, pack_logs,
                                   pack_select, range_requests)
from tests.harness import environ, fuzz_session, generateDocs
from tests.test_change_spec import next_op, replica
from tests.test_gpu_admission import oracle_admission, tampered_logs
from tests.test_gpu_append import canon, everything, route_crossings
from tests.test_gpu_change import change_table, empty_table
from tests.test_gpu_patch_bounds import log_changes, named_cases
from tests.test_gpu_patch_window import check_window, small_corpus
from tests.test_gpu_routes import (CONFIGS, FAULTS, ORACLE_DEFINES, WARP_ROUTES, Log, all_cases, batch_of, concurrent_at_one_position,
                                   expected_route, joint_batch, lamport_forward, marks_over, status_matrix, typing_backwards)
from tests.test_gpu_wire_forms import FORMS, upload_as

pytestmark = pytest.mark.gpu
A = SELECT_ADDED
PT_ERR_STATE = 4
KERNEL_ENV = ("PT_WARP", "PT_WARP_FORCE", "PT_TEAM", "PT_PATCH_WARP", "PT_WARP_FLAGS", "PT_TMA", "PT_PREFETCH")


# ------------------------------------------------------------------------------------------------------------------
# Harness
# ------------------------------------------------------------------------------------------------------------------
def stream_engine(**kw):
    """A BatchEngine on a new torch stream; the handle keeps the stream alive."""
    import torch
    from peritext_b200.engine import BatchEngine
    s = torch.cuda.Stream()
    e = BatchEngine(0, stream=s.cuda_stream, **kw)
    e.user_stream = s
    return e


def default_engine(**kw):
    from peritext_b200.engine import BatchEngine
    return BatchEngine(0, **kw)


def kernel_env(env=None):
    """The kernel-selection variables: unset, except those of `env`.  Read at upload and at capture, so held around both."""
    return environ({**{k: None for k in KERNEL_ENV}, **(env or {})})


def snapshot(e, batch, out):
    """Every output of the merge `out` on `e`: canonical spans, result rows, element sequences of the merged logs and, where the
    handle emits patches, the Patch stream, element queries, find and both JSON renders."""
    ok = [i for i in range(len(out.results)) if int(out.results[i]["status"]) == 0]
    seq = [out.sequence(i).tobytes() for i in ok] if out.seq is not None else None
    snap = (canon(out), out.results.tobytes(), seq)
    if e.emit_patches and len(out.results):
        recs, _, status, _ = e.download_patches()
        own = np.repeat(np.arange(batch.n_logs), batch.desc["n_insdel"].astype(np.int64))
        recs[status[own] != 0] = 0                      # the records of a log whose patches were not computed are undefined
        snap += (recs.tobytes(),) + everything(e, batch, out)[1:]
    return snap


def replayed(e, batch, k=3, traces=None):
    """`k` merges in a row, each downloaded and compared byte for byte with the first (merge 1 runs its launches directly, merges
    2..k replay the captured graph).  With `traces` (a list), the profiler traces of merge 1 and merge k are appended to it.
    Returns (the MergedBatch of the last merge, its snapshot)."""
    first = None
    for out in merges(e, k, traces):
        snap = snapshot(e, batch, out)
        if first is None:
            first = snap
        else:
            assert snap == first, "a replayed merge differs from merge 1"
    return out, first


def merges(e, k, traces=None):
    """Yields the download of each of `k` merges in a row (profiled as in ``replayed``)."""
    for m in range(k):
        if traces is not None and m in (0, k - 1):
            traces.append(trace(e.merge))
        else:
            e.merge()
        yield e.download()


def trace(fn):
    """The complete ("X") events of a torch.profiler trace (CPU and CUDA activities) of fn()."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return [ev for ev in events if ev.get("ph") == "X"]


def kernels(events):
    evs = [ev for ev in events if str(ev.get("cat", "")).lower() == "kernel"]
    assert evs, "the profiler recorded no CUDA kernel"
    return evs


def graph_launches(events):
    return [ev for ev in events if "cudaGraphLaunch" in ev.get("name", "")]


def assert_graph_path(traces):
    """Merge 1 launched its kernels itself; the last merge replayed the graph (and its kernels ran)."""
    first, last = traces
    kernels(first); kernels(last)
    assert not graph_launches(first), "merge 1 replayed a graph"
    assert graph_launches(last), "the repeated merge did not replay a captured graph"


def assert_forked(events):
    """The CTA-per-log bins' own launches of a direct merge ran on a stream other than the warp / team kernels'."""
    evs = kernels(events)
    stream = lambda ev: (ev.get("args") or {}).get("stream")
    bins = {stream(ev) for ev in evs if "merge_logs_kernel<" in ev["name"]}
    bin0 = {stream(ev) for ev in evs if "merge_logs_warp_kernel<" in ev["name"] or "merge_logs_team_kernel<" in ev["name"]}
    assert bins and bin0, sorted({(ev["name"][:60], stream(ev)) for ev in evs})
    assert None not in bins | bin0
    assert bins - bin0, f"the CTA bins ran on the warp / team kernels' stream {bin0}"


def oracle_equal(batch, got, statuses=None, defined=None):
    """Every log against replay_packed; where the oracle does not define a log (`defined`), its status against `statuses`."""
    ref, _ = replay_packed(batch, threads=8)
    for i in range(batch.n_logs):
        if defined is None or defined[i]:
            assert got.canonical(i) == ref.canonical(i), i
        else:
            assert int(got.results[i]["status"]) == statuses[i], i


def oracle_spans(logs):
    return [replica(lg, "~reader").getTextWithFormatting() for lg in logs]


# ------------------------------------------------------------------------------------------------------------------
# 1. The fork, with deferrals into list 3 from both streams
# ------------------------------------------------------------------------------------------------------------------
def bin2_deferral_log():
    """2200 characters typed backwards (one sibling group under HEAD) and 8 marks: the planner's estimate puts it in CTA bin 2,
    but its Euler tour does not fit bin 2's 74 KB, so bin 2's own launch defers it on the device to bin 3 (exactly once)."""
    lg = Log(1)
    ids = typing_backwards(lg, 2200, [0])
    marks_over(lg, ids, 8, seed=2200, width=8)
    return lg


def fork_batch():
    """Every route case (packed3, compact, direct, team, every CTA bin, a team log that defers on the device), the status
    matrix, the spill-slab log of the append tests and a log that CTA bin 2 defers, in one batch; (batch, defined per log,
    expected status per log)."""
    cases = list(all_cases())
    rows, sm = status_matrix()
    tail = batch_of([route_crossings()[2][0], bin2_deferral_log()])
    parts = cases + [SimpleNamespace(batch=b.select([i])) for b in (sm, tail) for i in range(b.n_logs)]
    batch = joint_batch(parts)
    defined = [True] * len(cases) + [f in ORACLE_DEFINES for _, f in rows] + [True] * 2
    statuses = [0] * len(cases) + [FAULTS[f] for _, f in rows] + [0] * 2
    return batch, defined, statuses


def deferrals(batch, env):
    """logs_deferred_to_big_bin of one default-stream merge of `batch` under `env`."""
    e = default_engine()
    try:
        with kernel_env(env):
            e.upload(batch)
            e.merge()
            return e.stats()["logs_deferred_to_big_bin"]
    finally:
        e.close()


def test_fork_with_deferrals_from_both_streams():
    """Deferral list 3 is appended to by the team kernel on the main stream and by CTA bin 2's own launch on the side stream,
    at the same time; lists 1 and 4 receive from the warp kernel and bin 3."""
    env = CONFIGS["forced-deferral"]["env"]           # the warp kernel runs out of its 4.5 KB slice and defers on the device
    batch, defined, statuses = fork_batch()
    routes = [expected_route(d, "forced-deferral") for d in batch.desc]
    assert {"packed3", "compact", "direct", "team"} <= set(routes) and {"cta2", "cta3", "cta4"} <= {r[:4] for r in routes}
    # the deferrals by where they start: the warp kernel (main stream), the team kernel (main stream, into list 3) and CTA bin
    # 2's own launch (side stream, into list 3); each part alone, then all of them in one batch
    parts = {"warp": [i for i, r in enumerate(routes) if r in WARP_ROUTES], "team": [i for i, r in enumerate(routes) if r == "team"],
             "bin2": [batch.n_logs - 1]}
    parts["rest"] = sorted(set(range(batch.n_logs)) - {i for p in parts.values() for i in p})
    assert routes[-1].startswith("cta2")
    counts = {k: deferrals(batch.select(p), env) for k, p in parts.items()}
    assert counts["bin2"] == 1 and counts["team"] > 0 and counts["warp"] > 0, counts
    e, u = stream_engine(), default_engine()
    try:
        with kernel_env(env):
            e.upload(batch)
            traces = []
            got, snap = replayed(e, batch, 3, traces)
            st = e.stats()
            u.upload(batch)
            u.merge()
            want = u.download()
            ust = u.stats()
        assert_graph_path(traces)
        assert_forked(traces[0])
        assert st == ust, (st, ust)
        assert st["logs_deferred_to_big_bin"] == sum(counts.values()), (st, counts)
        assert snap == snapshot(u, batch, want)
        oracle_equal(batch, got, statuses, defined)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 2. Admission inside the graph, with an actor table past 48 KB of shared memory
# ------------------------------------------------------------------------------------------------------------------
def many_actor_log(n_actors=6200):
    """One round of `n_actors` actors inserting at one position: admit_kernel's table of 8 bytes per actor exceeds 48 KB."""
    lg = Log(n_actors)
    concurrent_at_one_position(lg, 1, list(range(n_actors)))
    return log_changes(lg)


def test_admission_in_the_graph():
    cases = tampered_logs() + [("6200-actors", many_actor_log())]
    logs = [lg for _, lg in cases]
    want = [oracle_admission(lg) for lg in logs]
    assert {w[0] for w in want} == {0, 6, 7}
    batch = pack_logs(logs, with_changes=True)
    assert int(batch.desc["n_actors"].max()) * 8 > 48 * 1024
    e, u = stream_engine(), default_engine()
    try:
        with kernel_env():
            upload_as(e, batch, "plain")
            traces = []
            got, snap = replayed(e, batch, 3, traces)
            assert_graph_path(traces)
            for i, ((name, _), (s, idx)) in enumerate(zip(cases, want)):
                r = got.results[i]
                if s:
                    assert (int(r["status"]), int(r["n_elems"])) == (s, idx), name
                else:
                    assert int(r["status"]) == 0, name
            spans = oracle_spans([lg for lg, (s, _) in zip(logs, want) if s == 0])
            assert [decode_spans(batch, got, i) for i, (s, _) in enumerate(want) if s == 0] == spans
            upload_as(u, batch, "plain")
            u.merge()
            assert snap == snapshot(u, batch, u.download())
            # a table that admits every log: the statuses follow it through the replays, and back
            for table in (empty_table(batch.n_logs), batch.changes):
                e.upload_changes(table); u.upload_changes(table)
                got, snap = replayed(e, batch)
                u.merge()
                assert snap == snapshot(u, batch, u.download())
                rejected = [int(s) in (6, 7) for s in got.results["status"]]
                assert rejected == [s != 0 for s, _ in want] if table is batch.changes else not any(rejected)
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 3. Patch windows across replays, without a splice
# ------------------------------------------------------------------------------------------------------------------
def patch_pass(e, batch, k=3):
    """`k` merges compared with each other; the last one's MergedBatch and (results, recs, items, status, needed, per-log patch
    JSON)."""
    out, _ = replayed(e, batch, k)
    recs, items, status, needed = e.download_patches()
    assert needed == len(items)
    return out, (out.results, recs, items, status, needed, e.render_patches_json_list(batch))


@pytest.mark.parametrize("large", [False, True])
def test_patch_windows_across_replays(large):
    from peritext_b200.engine import EngineError
    ks = named_cases()["keyspace-65535"].changes          # over the warp patch kernel's key space
    logs = small_corpus() + [ks]
    batch = pack_logs(logs)
    tot = (batch.desc["n_insdel"].astype(np.int64) + batch.desc["n_mark"]).astype(np.uint32)
    w = (tot // 2).astype(np.uint32)
    w2 = np.array([(7 * i) % (int(t) + 1) for i, t in enumerate(tot)], np.uint32)
    assert (w != w2).any()
    e, u = stream_engine(large_patches=large, emit_patches=True), default_engine(large_patches=large, emit_patches=True)
    try:
        with kernel_env():
            e.upload(batch); u.upload(batch)
            out, whole = patch_pass(e, batch)
            assert int(whole[3][-1]) == (0 if large else 1)
            oracle_equal(batch, out)
            for window in (w, None, w2):
                e.set_patch_window(window)
                with pytest.raises(EngineError) as err:
                    e.download_patches()
                assert err.value.status == PT_ERR_STATE
                traces = []
                out, snap = replayed(e, batch, 2, traces)
                assert graph_launches(traces[0]) and graph_launches(traces[1]), "the window re-captured the graph"
                _, win = patch_pass(e, batch, 1)
                check_window(batch, whole, win, np.zeros(batch.n_logs, np.uint32) if window is None else window)
                u.set_patch_window(window)
                u.merge()
                assert snap == snapshot(u, batch, u.download())
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 4. Patch and comment pools across replays
# ------------------------------------------------------------------------------------------------------------------
def test_pools_across_replays():
    logs = small_corpus()
    batch = pack_logs(logs)
    spans = oracle_spans(logs)
    e, u = stream_engine(emit_patches=True), default_engine(emit_patches=True)
    try:
        with kernel_env():
            e.upload(batch); u.upload(batch)
            _, full = replayed(e, batch)
            u.merge()
            assert full == snapshot(u, batch, u.download())
            need = None
            # the patch pool: too small reports the demand, exactly the demand fits; shrink and re-grow.  Which items an
            # overflowing merge keeps depends on the order the logs run in, so there only the counts are compared.
            for cap in (1, None, -1, None):
                cap = need if cap is None else need + cap if cap < 0 else cap
                e.set_patch_pool(cap)
                for _ in merges(e, 2):
                    _, items, _, got_need = e.download_patches()
                    need = got_need if cap == 1 else need
                    assert got_need == need and len(items) == min(cap, need), cap
                assert need > 1
                if cap == need:
                    u.set_patch_pool(cap)
                    _, snap = replayed(e, batch)
                    u.merge()
                    assert snap == snapshot(u, batch, u.download()) == full, cap
            # the comment pool: too small gives status 4 and reports the demand, which then fits; shrink and re-grow
            e.set_comment_pool(1)
            out = list(merges(e, 2))[-1]
            demand = e.stats()["comment_pool_needed"]
            assert demand > 1 and (out.results["status"] == 4).any()
            for cap in (demand, demand - 1, demand):
                e.set_comment_pool(cap)
                if cap < demand:
                    for out in merges(e, 3):
                        st = out.results["status"]
                        assert (st == 4).any() and e.stats()["comment_pool_needed"] == demand, cap
                        assert [c for c, s in zip(canon(out), st) if s != 4] == [c for c, s in zip(full[0], st) if s != 4]
                    continue
                u.set_comment_pool(cap)
                out, snap = replayed(e, batch)
                u.merge()
                assert snap == snapshot(u, batch, u.download()) == full, cap
            assert [decode_spans(batch, out, i) for i in range(batch.n_logs)] == spans
    finally:
        e.close(); u.close()


# ------------------------------------------------------------------------------------------------------------------
# 5. A seeded lifecycle of one handle, mirrored by uploads of the host specification on a default-stream handle
# ------------------------------------------------------------------------------------------------------------------
IDS = ["doc1", "doc2", "doc3"]


class Lifecycle:
    """One user-stream handle `e` holding `cur` (the host specification) whose log i is the Change log `mlogs[i]` of replica
    `owner[i]` = (document, replica) or, for an admitted large log, (None, None).  With `patches` the handles emit the Patch
    stream (and the element sequence that pt_batch_change needs), which sends every log to the CTA bins: no fork; without,
    the small logs take the warp kernel and the admitted large ones a CTA bin: the fork."""

    def __init__(self, seed, patches):
        self.rng = random.Random(seed)
        self.patches = patches
        self.e, self.u = stream_engine(emit_patches=patches), default_engine(emit_patches=patches)
        if patches:
            for h in (self.e, self.u):
                h.set_patch_pool(1 << 22)                       # room for every step's Patch stream
        self.mlogs = []
        self.owner = []
        for d, text in enumerate(["abcdef", "xyz", "peritext", "hello"]):
            init = generateDocs(O, text, 1)[2]
            for r in range(len(IDS)):
                self.mlogs.append([init]); self.owner.append((d, r))
        self.cur = pack_logs(self.mlogs, with_changes=True)
        self.keep = None
        self.big = [log_changes(lamport_forward(3000, 2, 300, seed=seed)), log_changes(lamport_forward(1000, 1, 536, seed=seed))]
        self.traces = None

    def small(self):
        return [i for i, (d, _) in enumerate(self.owner) if d is not None]

    # --- steps -------------------------------------------------------------------------------------------------------
    def upload(self, form=None):
        form = form or self.rng.choice(FORMS)
        self.keep = upload_as(self.e, self.cur, form)
        self.e.upload_actors(self.cur)
        return form

    def tables(self):
        if not self.e._has_actors:
            self.e.upload_actors(self.cur)

    def add_actors(self):
        from tests.test_gpu_sync import device_add
        self.tables()
        names = [list(IDS) if d is not None else [] for d, _ in self.owner]
        self.cur = device_add(self.e, self.cur, names)

    def edit(self, i):
        d, r = self.owner[i]
        doc = replica(self.mlogs[i], IDS[r])
        n = len(doc.root["text"])
        if n < 2 or self.rng.random() < 0.6:
            return {"path": ["text"], "action": "insert", "index": self.rng.randrange(n + 1), "values": [self.rng.choice("uvw")]}
        a = self.rng.randrange(n - 1)
        op = {"path": ["text"], "action": "addMark", "startIndex": a, "endIndex": self.rng.randrange(a + 1, n + 1),
              "markType": self.rng.choice(["strong", "em", "comment"])}
        if op["markType"] == "comment":
            op["attrs"] = {"id": "c%d" % self.rng.randrange(9)}
        return op

    def append(self):
        i = self.rng.choice(self.small())
        actor = IDS[self.owner[i][1]]
        ch = replica(self.mlogs[i], actor).change([self.edit(i)])["change"]
        ch["seq"] = 1 + sum(c["actor"] == actor for c in self.mlogs[i])     # a fresh replica would number it 1
        delta, remap = pack_append(self.cur, [[ch] if j == i else [] for j in range(self.cur.n_logs)], with_changes=True)
        self.e.append(delta, remap)
        self.cur = apply_append(self.cur, delta, remap)
        self.mlogs[i].append(ch)

    def change(self):
        n = self.cur.n_logs
        inputs, ranks = [None] * n, [None] * n
        for i in self.small():
            actor = IDS[self.owner[i][1]]
            if actor not in self.cur.log_actors[i] or self.rng.random() < 0.3:
                continue
            op = self.edit(i)
            if op["action"] == "addMark" and op["markType"] == "comment":
                op = {**op, "markType": "em"}
                op.pop("attrs", None)
            doc = replica(self.mlogs[i], actor)
            inputs[i] = {"actor": actor, "seq": 1 + sum(c["actor"] == actor for c in self.mlogs[i]), "deps": doc.clock,
                         "startOp": next_op(self.mlogs[i]), "ops": [op]}
            ranks[i] = self.cur.log_actors[i].index(actor)
        some = [i for i in range(n) if inputs[i] is not None]
        if not some:
            return False
        table = change_table(self.cur.select(some), [inputs[i] for i in some], [ranks[i] for i in some])
        full = empty_table(n)
        full.desc["n_changes"][some] = 1; full.desc["n_deps"][some] = table.desc["n_deps"]
        full.desc["change_off"][some] = table.desc["change_off"]; full.desc["dep_off"][some] = table.desc["dep_off"]
        self.cur, dicts, status = self.e.change(self.cur, inputs, ranks, ChangeTable(full.desc, table.changes, table.deps))
        assert (status["status"][some] == 0).all()
        for i in some:
            self.mlogs[i].append(dicts[i])
        return True

    def pairs(self):
        by_doc = {}
        for i, (d, _) in enumerate(self.owner):
            if d is not None:
                by_doc.setdefault(d, []).append(i)
        out = []
        for slots in by_doc.values():
            if len(slots) >= 2:
                a, b = self.rng.sample(slots, 2)
                out += [(a, b), (b, a)]
        return out

    def deliver(self, pairs, delivered):
        before = [list(lg) for lg in self.mlogs]
        for p, (s, t) in enumerate(pairs):
            self.mlogs[t] += [before[s][k] for k in delivered[p]]

    def exchange(self):
        from tests.test_gpu_exchange import device_sync
        pairs = self.pairs()
        if pairs:
            self.cur, _, delivered = device_sync(self.e, self.cur, pairs)
            self.deliver(pairs, delivered)

    def sync(self):
        from tests.test_gpu_sync import device_sync
        self.tables()
        pairs = self.pairs()
        if pairs:
            self.cur, _, delivered = device_sync(self.e, self.cur, pairs)
            self.deliver(pairs, delivered)

    def select(self, from_, new_logs=(), owners=()):
        self.tables()
        new_logs = list(new_logs)
        added, cmap = pack_select(self.cur, from_, new_logs, with_changes=True)
        self.e.select_logs(from_, added if new_logs else None, cmap)
        self.cur = apply_select(self.cur, from_, added if new_logs else None, cmap)
        it, own = iter(new_logs), iter(owners)
        self.mlogs = [list(next(it)) if f == A else self.mlogs[f] for f in from_]
        self.owner = [next(own) if f == A else self.owner[f] for f in from_]

    def admit_big(self):
        n = self.cur.n_logs
        self.select([A] + list(range(n))[::-1] + [A], self.big, [(None, None)] * 2)
        assert all(expected_route(self.cur.desc[i])[:3] == "cta" for i in (0, n + 1))
        self.traces = []                                        # the next check proves the fork

    def fork_big(self):
        big = [i for i, (d, _) in enumerate(self.owner) if d is None]
        self.select(list(range(self.cur.n_logs)) + big[:1])

    def drop_big(self):
        keep = self.small()
        self.select(keep[1:] + keep[:1])
        self.traces = []                                        # the next check proves the fork is gone

    def to_zero_and_back(self):
        saved, owners = [list(lg) for lg in self.mlogs], list(self.owner)
        self.select([])
        self.check()
        self.select([A] * len(saved), saved, owners)

    def window(self):
        tot = self.cur.desc["n_insdel"].astype(np.int64) + self.cur.desc["n_mark"]
        self.e.set_patch_window(np.array([self.rng.randrange(int(t) + 1) for t in tot], np.uint32))

    def changes(self):
        self.e.upload_changes(self.cur.changes)

    # --- the check after every step -----------------------------------------------------------------------------------
    def check(self):
        e, u, cur = self.e, self.u, self.cur
        traces, self.traces = self.traces, None
        out, snap = replayed(e, cur, 3, traces)
        if traces is not None:
            assert_graph_path(traces)
            if self.forks():
                assert_forked(traces[0])
            else:
                assert len({(ev.get("args") or {}).get("stream") for ev in kernels(traces[0]) if "merge_logs_" in ev["name"]}) == 1
        if not cur.n_logs:
            return
        assert canon(out) == canon(replay_packed(cur)[0])
        assert [decode_spans(cur, out, i) for i in range(cur.n_logs)] == oracle_spans(self.mlogs)
        upload_as(u, cur, "plain")
        if self.patches:
            u.set_patch_window(e.patch_window)
        u.merge()
        assert snap == snapshot(u, cur, u.download())
        req, extras = range_requests(list(range(cur.n_logs))), change_extras(self.mlogs)[0]
        a, b = e.render_changes_json(cur, req, extras), u.render_changes_json(cur, req, extras)
        assert [x.tobytes() for x in a] == [x.tobytes() for x in b]

    def forks(self):
        return not self.patches and any(d is None for d, _ in self.owner)

    def close(self):
        self.e.close(); self.u.close()


STEPS = ("upload", "append", "change", "exchange", "sync", "window", "changes", "add_actors")


@pytest.mark.parametrize("seed,patches", [(1, True), (2, False), (3, False)])
def test_seeded_lifecycle(seed, patches):
    lc = Lifecycle(seed, patches)
    steps = [x for x in STEPS if patches or x not in ("change", "window")]
    done = []
    lc.traces = []                                              # the first check: the graph, and no fork on a warp-only batch
    try:
        with kernel_env():
            # every step at least once, every upload form once; a warp-only batch (no fork) until large logs are admitted
            # (fork), forked, and dropped again (no fork); the other steps drawn by the seed
            first = ["append", "change", "window", "exchange", "sync", "changes"]
            plan = (["upload-plain", "add_actors"] + [x for x in first if x in steps] + ["upload-runs", None, None, "admit_big", "fork_big",
                    "upload-compact"] + [None] * 5 + ["drop_big", "zero", "upload-adopt"] + [None] * 8)
            for step in plan:
                step = step or lc.rng.choice(steps)
                if step == "zero":
                    lc.to_zero_and_back()
                elif step.startswith("upload"):
                    step = "upload-" + lc.upload(step[len("upload-"):] or None)
                elif step == "change":
                    step = "change" if lc.change() else "change (nothing to change)"
                else:
                    getattr(lc, step)()
                done.append(step)
                assert lc.forks() == (not patches and "admit_big" in done and "drop_big" not in done)
                lc.check()
            want = {"upload-" + f for f in FORMS} | {"add_actors", "append", "exchange", "sync", "changes", "admit_big", "fork_big", "drop_big", "zero"}
            assert want | ({"change", "window"} if patches else set()) <= set(done), done
    except BaseException:
        print("steps:", done)
        raise
    finally:
        lc.close()


# ------------------------------------------------------------------------------------------------------------------
# 6. Two handles on two user streams, interleaved
# ------------------------------------------------------------------------------------------------------------------
def mixed_batch():
    """Record-built logs on every kind of route for a handle without the element sequence: packed3, compact, direct, team, CTA
    bins 1, 2 (with a device-side deferral) and 4 (the spill-slab log)."""
    return batch_of([lamport_forward(300, 3, 10), lamport_forward(300, 4, 10), lamport_forward(300, 2, 10), lamport_forward(3000, 2),
                     lamport_forward(1000, 1, 536), bin2_deferral_log(), route_crossings()[2][0]])


def streams_of(events, *names):
    return {(ev.get("args") or {}).get("stream") for ev in kernels(events) if any(n in ev["name"] for n in names)}


def test_two_handles_on_two_streams_interleaved():
    """A patch-emitting handle (every log in the CTA bins, no fork) and a plain one whose mixed batch forks, merging side by
    side with no host synchronisation; then the batches swap handles."""
    import torch
    a_logs = small_corpus() + [named_cases()["keyspace-65535"].changes]
    batches = [pack_logs(a_logs), mixed_batch()]
    spans = [oracle_spans(a_logs), None]
    e1, e2 = stream_engine(large_patches=True), stream_engine()
    e1.set_patch_pool(1 << 22)
    try:
        with kernel_env():
            for order in ((0, 1), (1, 0)):
                hs = [e1, e2]
                for h, j in zip(hs, order):
                    h.upload(batches[j])
                traces = []
                for m in range(3):
                    both = lambda: [h.merge() for h in hs]      # no host synchronisation between the two streams
                    if m in (0, 2):
                        traces.append(trace(both))
                    else:
                        both()
                torch.cuda.synchronize()
                assert not graph_launches(traces[0]) and len(graph_launches(traces[1])) >= 2
                if order == (0, 1):
                    # e2's CTA bins on its side stream, apart from e2's warp / team kernels and from e1's stream
                    side = streams_of(traces[0], "merge_logs_kernel<") - streams_of(traces[0], "merge_logs_warp_kernel<", "merge_logs_team_kernel<") \
                        - streams_of(traces[0], "patch_logs_kernel", "patch_large_kernel")
                    assert side, "the plain handle's CTA bins did not run on a stream of their own"
                for h, j in zip(hs, order):
                    out = h.download()
                    oracle_equal(batches[j], out)
                    if spans[j] is not None:
                        assert [decode_spans(batches[j], out, i) for i in range(batches[j].n_logs)] == spans[j]
                    if h.emit_patches:
                        _, items, _, needed = h.download_patches()
                        assert needed == len(items)
                    u = default_engine(emit_patches=h.emit_patches, large_patches=h.large_patches)
                    try:
                        u.set_patch_pool(1 << 22)
                        u.upload(batches[j]); u.merge()
                        assert snapshot(h, batches[j], out) == snapshot(u, batches[j], u.download())
                    finally:
                        u.close()
    finally:
        e1.close(); e2.close()


# ------------------------------------------------------------------------------------------------------------------
# 7. Full size: c4 with 300 000 logs, then 1 % retired and 1 % admitted
# ------------------------------------------------------------------------------------------------------------------
def test_c4_300k_logs_replayed_on_a_user_stream():
    full = workload.generate("c4", n_docs=101_000, ops_per_doc=120)
    R = int(full.meta["replicas"])
    resident, fresh = full.slice_logs(0, 100_000 * R), full.slice_logs(100_000 * R, 101_000 * R)
    assert resident.n_logs >= 300_000
    retired = set(range(0, 100_000, 100))
    from_ = [d * R + r for d in range(100_000) if d not in retired for r in range(R)] + [A] * fresh.n_logs
    want = apply_select(resident, from_, fresh)
    refs = []
    with kernel_env():
        u = default_engine()                                    # one handle at a time
        try:
            for b in (resident, want):
                u.upload(b); u.merge()
                r = u.results()
                assert (r["status"] == 0).all()
                refs.append(r.tobytes())
        finally:
            u.close()
        e = stream_engine()
        try:
            e.upload(resident)
            for step in range(2):
                if step:
                    e.select_logs(from_, fresh)
                traces = []
                for m in range(3):
                    if m in (0, 2):
                        traces.append(trace(e.merge))
                    else:
                        e.merge()
                    assert e.results().tobytes() == refs[step], (step, m + 1)
                assert_graph_path(traces)
                # every c4 log takes the warp kernel: no CTA bin holds a log, so nothing forks
                assert len(streams_of(traces[0], "merge_logs_")) == 1
        finally:
            e.close()
