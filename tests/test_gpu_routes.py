"""Every merge-kernel route at its dispatch and capacity boundaries, against the oracle.

The planner (`ptp::route_of`, peritext_b200/csrc/plan.cpp) sends each log, by its shape, to the warp kernel (packed3 / compact / direct id
table), the 8-warp team kernel, or one of four CTA bins (u16 or u32 indices); the warp and team kernels defer what they cannot
finish to the CTA bins on the device.  The logs here are built record by record with numpy, so that n_insdel, n_mark,
n_actors, max_ctr, run structure and counter collisions are exact and each one sits on a named side of one threshold.
`expected_route` restates the host's decision; the CPU tests pin every case to its side, the GPU tests check that every
route, every kernel configuration and the forced device-side deferral give the oracle's results bit for bit.
Valid logs are causal: every reference was inserted earlier and has a lower counter than the insert naming it."""
import numpy as np
import pytest

from oracle.oracle import Micromerge as O
from oracle.packed import replay_packed
from peritext_b200.packing import DESC_DT, INSDEL_DT, MARK_DT, PackedBatch, decode_spans, pack_logs
from tests.harness import environ, generateDocs

STRONG, EM, COMMENT, LINK = 0, 1, 2, 3
BEFORE, AFTER, END_OF_TEXT = 0, 1, 3
HEAD = None


# ------------------------------------------------------------------------------------------------------------------
# Exact-shape logs
# ------------------------------------------------------------------------------------------------------------------
class Log:
    """One packed log under construction.  Element ids are (ctr, actor); `ctr` is a Lamport clock unless a structure
    reuses a counter on purpose (concurrent inserts of several actors)."""

    def __init__(self, n_actors):
        self.R = n_actors
        self.ins, self.mk = [], []
        self.ctr = 0            # highest counter used so far
        self.max_ctr = 0        # descriptor max_ctr (>= every counter in the log)

    def _use(self, c):
        self.ctr = max(self.ctr, c)
        self.max_ctr = max(self.max_ctr, c)
        return c

    def insert(self, actor, ref, ch="x", ctr=None, kind=0):
        c = self._use(self.ctr + 1 if ctr is None else ctr)
        rc, ra = ref if ref is not None else (0, 0)
        self.ins.append((c, rc, actor, ra, (kind << 30) | ord(ch)))
        return (c, actor)

    def delete(self, actor, ref, ctr=None):
        c = self._use(self.ctr + 1 if ctr is None else ctr)
        rc, ra = ref if ref is not None else (0, 0)
        self.ins.append((c, rc, actor, ra, 1 << 30))
        return (c, actor)

    def mark(self, actor, typ, start, end, add=True, attr=0xFFFFFFFF, sb=BEFORE, eb=BEFORE):
        """A mark op arriving after every ins/del record so far; `start` / `end` are element ids (or None with
        sb / eb = startOfText / endOfText)."""
        c = self._use(self.ctr + 1)
        s, e = start or (0, 0), end or (0, 0)
        self.mk.append((c, actor, (0 if add else 1) | (typ << 1), sb | (eb << 2), s[0], e[0], s[1], e[1], attr, len(self.ins), 0))
        return (c, actor)

    @property
    def n(self):
        return len(self.ins)

    @property
    def m(self):
        return len(self.mk)


def batch_of(logs):
    desc = np.zeros(len(logs), DESC_DT)
    io = mo = 0
    n_attr = 1
    for k, lg in enumerate(logs):
        desc[k] = (io, mo, lg.n, lg.m, lg.R, lg.max_ctr)
        io += lg.n; mo += lg.m
        n_attr = max([n_attr] + [r[8] + 1 for r in lg.mk if r[8] != 0xFFFFFFFF])
    ins = np.array([r for lg in logs for r in lg.ins], INSDEL_DT) if io else np.zeros(0, INSDEL_DT)
    mk = np.array([r for lg in logs for r in lg.mk], MARK_DT) if mo else np.zeros(0, MARK_DT)
    return PackedBatch(desc, ins, mk, link_attrs=[{"url": "%d.com" % k} for k in range(n_attr)],
                       comment_ids=[{"id": "c%03d" % k} for k in range(n_attr)])


def typing_forward(lg, n, actors=None, start=HEAD, ch=97):
    """n characters, each typed after the previous one (one chain), by `actors` in turn; returns the element ids."""
    actors = actors or [0]
    ids, prev = [], start
    for k in range(n):
        prev = lg.insert(actors[k % len(actors)], prev, chr(ch + k % 26))
        ids.append(prev)
    return ids


def typing_backwards(lg, n, actors=None):
    """n characters, each typed at the start of the text: one sibling group of n children of HEAD."""
    actors = actors or [0]
    return [lg.insert(actors[k % len(actors)], HEAD, chr(65 + k % 26)) for k in range(n)]


def concurrent_blocks(lg, n, actors, blk):
    """Each round, every actor appends `blk` characters to its own chain with the SAME counters as the others (concurrent
    edits): runs of `blk`, and every counter is shared by len(actors) inserts."""
    tails = {a: HEAD for a in actors}
    ids = []
    while len(ids) < n:
        base = lg.ctr + 1
        for a in actors:
            for j in range(min(blk, n - len(ids))):
                tails[a] = lg.insert(a, tails[a], chr(97 + j % 26), ctr=base + j)
                ids.append(tails[a])
    return ids


def concurrent_at_one_position(lg, rounds, actors):
    """An anchor, then round after round every actor inserts right after the previous round's first insert, all with one
    counter: len(actors) - 1 counter collisions per round."""
    anchor = lg.insert(actors[0], HEAD, "#")
    ids = [anchor]
    for _ in range(rounds):
        c = lg.ctr + 1
        row = [lg.insert(a, anchor, chr(48 + a % 10), ctr=c) for a in actors]
        anchor = row[0]
        ids += row
    return ids


def delete_all_then_retype(lg, n, actors):
    ids = typing_forward(lg, n, actors)
    for k, e in enumerate(ids):
        lg.delete(actors[k % len(actors)], e)
    return typing_forward(lg, n, actors, ch=65)


def chains(lg, runs, length, actors=None):
    """`runs` chains of `length` characters, each started at HEAD: exactly `runs` runs (no element has a second child)."""
    actors = actors or [0]
    ids = []
    for r in range(runs):
        ids += typing_forward(lg, length, [actors[r % len(actors)]])
    return ids


def marks_over(lg, ids, count, seed, types=(STRONG, EM, LINK, COMMENT), n_ids=8, actor=0, width=None):
    """`count` mark ops with random ranges over the elements `ids` (all visible), at most `width` elements wide."""
    rng = np.random.default_rng(seed)
    L = len(ids)
    for k in range(count):
        a = int(rng.integers(0, L - 1)); b = int(rng.integers(a + 1, L + 1 if width is None else min(L, a + width) + 1))
        t = types[k % len(types)]
        add = bool(rng.random() < 0.75)
        attr = 0xFFFFFFFF
        if t == LINK:
            attr = int(rng.integers(0, 4))
        elif t == COMMENT:
            attr = int(rng.integers(0, n_ids))
        end, eb = (ids[b], BEFORE) if b < L else (None, END_OF_TEXT)
        lg.mark(actor, t, ids[a], end, add=add, attr=attr, eb=eb)


# ------------------------------------------------------------------------------------------------------------------
# The route mirror: restates the planner's decision (ptp::route_of, peritext_b200/csrc/plan.cpp)
# ------------------------------------------------------------------------------------------------------------------
CTA_BINS = [(1536, 31 * 1024), (4096, 74 * 1024), (12288, 112 * 1024), (0xFFFFFFFF, 226 * 1024)]   # (max records, smem)
TEAM_SMEM = 55 * 1024
# kernel configurations: PT_WARP (None: the default 2048-record bin with a 7136-byte slice per warp), force = PT_WARP_FORCE
CONFIGS = {
    "default": dict(env={}, warp=(2048, 7136), team=True, force=False),
    "team-off": dict(env={"PT_TEAM": "0"}, warp=(2048, 7136), team=False, force=False),
    "cta-only": dict(env={"PT_WARP": "0"}, warp=None, team=False, force=False),
    # a 4.5 KB slice with the host estimate skipped: logs run out of shared memory part-way and are deferred on the device
    "forced-deferral": dict(env={"PT_WARP": "2048:4:4608:4", "PT_WARP_FORCE": "1"}, warp=(2048, 4608), team=True, force=True),
    # a 113 KB slice (2 warps per CTA) with the host estimate skipped: the warp kernel's own limits, not its memory, decide
    "wide": dict(env={"PT_WARP": "2048:2:113:1", "PT_WARP_FORCE": "1"}, warp=(2048, 113 * 1024), team=True, force=True),
}
WARP_ROUTES = ("packed3", "compact", "direct")


def expected_route(d, config="default"):
    """Where the planner sends the log with descriptor row `d`: 'packed3' / 'compact' / 'direct' (warp kernel), 'team', or
    'cta<k>-u16' / 'cta<k>-u32' (CTA bin k = 1..4, 16- or 32-bit indices)."""
    cfg = CONFIGS[config]
    n, m, C = int(d["n_insdel"]), int(d["n_mark"]), int(d["max_ctr"])
    R = int(d["n_actors"]) or 1
    recs, KS = n + m, C * R
    I = 2 if (n < 32000 and m < 32000) else 4
    b = 0
    while recs > CTA_BINS[b][0]:
        b += 1
    seg = min(2 * m + 2, n // 2 + 2)
    typical = KS * I + (14 * n) // 10 + max(5 * n, m * (6 * I + 13) + 18 * seg if m else 0) + 2048
    while b < len(CTA_BINS) - 1 and typical > CTA_BINS[b][1]:
        b += 1
    packed3 = R == 3 and n <= 1022
    compact = 3 <= R <= 30 and n <= 2046
    if cfg["warp"] and recs <= cfg["warp"][0] and KS < 0xFFFF:
        idbytes = 4 * C if packed3 else 2 * C + 512 if compact else 2 * KS
        rest = n // 2 + 32 + 14 * (n // 4) + (KS // 32 + 2) * 6 + 512 if packed3 else n // 2 + 16 * n // 3 + 1024
        if cfg["force"] or idbytes + rest <= cfg["warp"][1]:
            return "packed3" if packed3 else "compact" if compact else "direct"
    if cfg["team"] and m == 0 and KS < 0xFFFF and n < 0xFFFF and (3 * n) // 4 + 2 * KS + 2 * n + 1024 <= TEAM_SMEM:
        return "team"
    return "cta%d-u%d" % (b + 1, 8 * I)


def team_footprint(d):
    n, KS = int(d["n_insdel"]), int(d["max_ctr"]) * (int(d["n_actors"]) or 1)
    return (3 * n) // 4 + 2 * KS + 2 * n + 1024


# ------------------------------------------------------------------------------------------------------------------
# The boundary table
# ------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, log, routes, defer=None, spans=None):
        self.name, self.log, self.routes = name, log, routes      # routes: config -> expected route
        self.defer = defer or {}                                  # config -> 0 (no deferral) / 1 (at least one)
        self.spans = spans                                        # getTextWithFormatting of a Micromerge-built log


def lamport_forward(n, R, marks=0, seed=0, width=None):
    lg = Log(R)
    ids = typing_forward(lg, n, list(range(R)))
    if marks:
        marks_over(lg, ids, marks, seed, width=width)
    return lg


def shared_counter_forward(n, R, marks=0, blk=32, seed=0):
    lg = Log(R)
    ids = concurrent_blocks(lg, n, list(range(R)), blk)
    if marks:
        marks_over(lg, ids[:blk], marks, seed)
    return lg


def ks_log(R, C, n=400):
    """R actors typing forward with counters spread up to exactly max_ctr = C (key space C * R)."""
    lg = Log(R)
    prev = HEAD
    for k in range(n):
        c = 1 + (k * (C - 1)) // (n - 1)
        prev = lg.insert(k % R, prev, chr(97 + k % 26), ctr=c)
    assert lg.max_ctr == C
    return lg


def collisions_log(n_ov, R=4, n=300):
    """Typing forward by actor 0 (distinct counters), then n_ov inserts by the other actors that reuse counters already
    taken (each after an element with a lower counter): n_ov entries in the compact id table's overflow."""
    lg = Log(R)
    ids = typing_forward(lg, n, [0])
    made = 0
    for a in range(1, R):
        for k in range(1, n):
            if made == n_ov:
                return lg
            lg.insert(a, ids[k - 1], "+", ctr=ids[k][0])
            made += 1
    assert made == n_ov
    return lg


def micromerge_case(name, text, ops, routes, defer=None):
    docs, _, init = generateDocs(O, text, 1)
    d = docs[0]
    chs = [init] + [d.change([{"path": ["text"], **op}])["change"] for op in ops]
    return ("mm", name, chs, d.getTextWithFormatting(), routes, defer)


def comment_ops(k, L, distinct=True):
    return [dict(action="addMark", startIndex=j % (L - 1), endIndex=min(L, j % (L - 1) + 1 + (j * 5) % 7), markType="comment",
                 attrs={"id": "id%02d" % (j if distinct else 0)}) for j in range(k)]


def short_text_ops(L):
    ops = []
    for j in range(12):
        a = (j * 5) % (L - 1); b = min(L, a + 1 + (j * 3) % 9)
        t = ["strong", "em", "link", "comment"][j % 4]
        op = dict(action="addMark" if j % 5 != 4 else "removeMark", startIndex=a, endIndex=b, markType=t)
        if t == "link" and op["action"] == "addMark":
            op["attrs"] = {"url": "%d.com" % (j % 3)}
        if t == "comment":
            op["attrs"] = {"id": "k%d" % (j % 3)}
        ops.append(op)
    return ops


def seg_work_log(n_survivors):
    """n_survivors mark ops over 200 visible characters with boundaries at 5 * k (k < 36): S = 36 segments, so the warp kernel's
    segment work ceil(S / 32) * nS is 2 * n_survivors."""
    lg = Log(1)
    ids = typing_forward(lg, 200)
    for k in range(n_survivors):
        a = 5 * (k % 35); b = a + 5 * (1 + (k * 7) % 3)
        b = min(b, 175)
        lg.mark(0, (STRONG, EM, LINK)[k % 3], ids[a], ids[b], attr=(k % 3) if k % 3 == 2 else 0xFFFFFFFF)
    return lg


def backwards_log(n, R):
    lg = Log(R)
    typing_backwards(lg, n, list(range(R)))
    return lg


def structure_log(kind, R, size):
    lg = Log(R)
    actors = list(range(R))
    if kind == "forward":
        typing_forward(lg, size, actors)
    elif kind == "backwards":
        typing_backwards(lg, size, actors)
    elif kind == "one-char-interleaved":
        concurrent_blocks(lg, size, actors, 1)
    elif kind == "one-position":
        concurrent_at_one_position(lg, max(1, size // R), actors)
    elif kind == "delete-all-retype":
        delete_all_then_retype(lg, size // 3, actors)
    return lg


def build_cases():
    W = "wide"
    cases = []
    add = lambda *a, **k: cases.append(Case(*a, **k))
    # packed3 <-> compact: 3 actors, 1022 / 1023 ins/del records, with and without marks
    for mk in (0, 20):
        add(f"3actors-1022-m{mk}", lamport_forward(1022, 3, mk), {W: "packed3"}, defer={W: 0})
        add(f"3actors-1023-m{mk}", lamport_forward(1023, 3, mk), {W: "compact"}, defer={W: 0})
    # ... and a 1022-record packed3 log that fits the default slice (three replicas typing concurrently)
    add("3actors-1022-shared-counters", shared_counter_forward(1022, 3), {"default": "packed3", W: "packed3"}, defer={W: 0})
    add("3actors-1023-shared-counters", shared_counter_forward(1023, 3), {"default": "team", W: "compact"}, defer={W: 1})
    # compact <-> direct: 30 / 31 actors
    add("30actors", lamport_forward(600, 30), {"default": "compact", W: "compact"}, defer={W: 0})
    add("31actors", lamport_forward(600, 31), {"default": "team", W: "direct"}, defer={W: 0})
    # compact <-> direct: 2046 / 2047 ins/del records with 5 actors
    add("5actors-2046", lamport_forward(2046, 5, 2), {W: "compact"}, defer={W: 0})
    add("5actors-2047", lamport_forward(2047, 5, 1), {W: "direct"}, defer={W: 0})
    # warp bin <-> CTA / team: 2048 / 2049 records
    add("2048-records-marks", lamport_forward(1900, 2, 148), {W: "direct"})
    add("2049-records-marks", lamport_forward(1900, 2, 149), {W: "cta2-u16"})
    add("2048-records", lamport_forward(2048, 2), {W: "direct"})
    add("2049-records", lamport_forward(2049, 2), {W: "team", "default": "team"})
    # the CTA bins' record limits, with marks
    add("cta-1536", lamport_forward(1000, 1, 536), {"default": "cta1-u16"})
    add("cta-1537", lamport_forward(1000, 1, 537), {"default": "cta2-u16"})
    add("cta-4096", lamport_forward(3000, 1, 1096), {"default": "cta2-u16"})
    add("cta-4097", lamport_forward(3000, 1, 1097), {"default": "cta3-u16"})
    add("cta-12288", lamport_forward(12000, 1, 288), {"default": "cta3-u16"})
    add("cta-12289", lamport_forward(12000, 1, 289), {"default": "cta4-u16"})
    # u16 <-> u32 indices from the mark count alone
    add("marks-31999", lamport_forward(2000, 2, 31999, seed=3, width=4), {"default": "cta4-u16"})
    add("marks-32000", lamport_forward(2000, 2, 32000, seed=3, width=4), {"default": "cta4-u32"})
    # team footprint: 2 actors typing forward, 6.75 n + 1024 bytes: n = 8192 is exactly 55 KB
    add("team-footprint-inside", lamport_forward(8192, 2), {"default": "team"}, defer={"default": 0})
    add("team-footprint-outside", lamport_forward(8193, 2), {"default": "cta3-u16"})
    # ... and a team log that must defer on the device: 8000 children of HEAD need 8001 Euler-tour nodes of 8 B
    add("team-typing-backwards-8000", backwards_log(8000, 1), {"default": "team"}, defer={"default": 1})
    # the warp kernel's Euler-tour splitters: 8k - 1, 8k, 8k + 1 runs
    for runs in (127, 128, 129):
        lg = Log(3)
        chains(lg, runs, 3, [0, 1, 2])
        add(f"runs-{runs}", lg, {"default": "packed3"}, defer={"default": 0})
    # the compact id table's overflow: 96 / 97 inserts that share a counter with an earlier insert
    add("overflow-96", collisions_log(96), {"default": "compact", W: "compact"}, defer={W: 0})
    add("overflow-97", collisions_log(97), {"default": "compact", W: "compact"}, defer={W: 1})
    # segment work ceil(S/32) * nS: 1536 / 1538
    add("segment-work-1536", seg_work_log(768), {W: "direct"}, defer={W: 0})
    add("segment-work-1538", seg_work_log(769), {W: "direct"}, defer={W: 1})
    # the 16-bit key-space guard: max_ctr * n_actors = 65534 / 65535
    add("keyspace-65534", ks_log(14, 4681), {W: "compact"}, defer={W: 0})
    add("keyspace-65535", ks_log(15, 4369), {W: "cta4-u16"})
    # team-sized repeats of the adversarial structures (with Lamport counters the key space grows with the actors: fewer
    # records for 8 and 30 actors keep them inside the team kernel's 55 KB)
    for R in (2, 3, 8, 30):
        for kind in ("forward", "backwards", "one-char-interleaved", "one-position", "delete-all-retype"):
            size = 3000 if R <= 3 or kind in ("one-char-interleaved", "one-position") else {8: 2900, 30: 850}[R]
            add(f"team-{kind}-{R}actors", structure_log(kind, R, size if kind != "backwards" else min(size, 1500)), {"default": "team"})
    # run counts across the team kernel's 256-record trips
    for n in (255, 256, 257, 4095, 4096, 4097):
        add(f"forward-{n}", lamport_forward(n, 2), {"default": expected_route(batch_of([lamport_forward(n, 2)]).desc[0])})
    return cases


def build_mm_cases():
    """Micromerge-built logs (spans also checked against getTextWithFormatting): the warp kernel's phase I forms."""
    W = "wide"
    out = []
    # short text: <= 32 visible characters (and <= 32 surviving comment ops) take the per-position form
    for L in (32, 33):
        out.append(micromerge_case(f"visible-{L}", "abcdefghijklmnopqrstuvwxyz0123456789"[:L], short_text_ops(L), {"default": "direct"}))
    # surviving comment ops: 32 / 33 (short text / segments), 48 / 49 (segments / deferred); 32 distinct ids = mask bit 31
    for k in (32, 33):
        out.append(micromerge_case(f"comments-{k}-distinct", "x" * 30, comment_ops(k, 30), {"default": "direct"}))
    out.append(micromerge_case("comments-32-one-id", "x" * 30, comment_ops(32, 30, distinct=False), {"default": "direct"}))
    for k in (48, 49):
        out.append(micromerge_case(f"comments-{k}", "y" * 60, comment_ops(k, 60), {"default": "direct", W: "direct"},
                                   defer={W: 0 if k == 48 else 1}))
    return out


_CASES = None


def all_cases():
    global _CASES
    if _CASES is None:
        cases = build_cases()
        for _, name, chs, spans, routes, defer in build_mm_cases():
            b = pack_logs([chs])
            c = Case(name, None, routes, defer, spans)
            c.batch = b
            cases.append(c)
        for c in cases:
            if c.log is not None:
                c.batch = batch_of([c.log])
        _CASES = cases
    return _CASES


def case_ids():
    return [c.name for c in all_cases()]


def joint_batch(cases):
    """One batch holding every case's log (pools of the Micromerge-built cases stay valid: each case's own batch is kept
    for decoding)."""
    desc, ins, mk = [], [], []
    io = mo = 0
    for c in cases:
        d = c.batch.desc.copy()
        d["insdel_off"] = io; d["mark_off"] = mo
        desc.append(d); ins.append(c.batch.insdel); mk.append(c.batch.marks)
        io += len(c.batch.insdel); mo += len(c.batch.marks)
    n_attr = max(max(len(c.batch.comment_ids), len(c.batch.link_attrs)) for c in cases)
    return PackedBatch(np.concatenate(desc), np.concatenate(ins), np.concatenate(mk),
                       link_attrs=[{"url": "%d.com" % k} for k in range(n_attr)], comment_ids=[{"id": "c%03d" % k} for k in range(n_attr)])


# ------------------------------------------------------------------------------------------------------------------
# CPU: every case lands on the side of the threshold it is named for
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", case_ids())
def test_case_takes_its_route(name):
    c = next(c for c in all_cases() if c.name == name)
    d = c.batch.desc[0]
    for cfg, route in c.routes.items():
        assert expected_route(d, cfg) == route, (name, cfg)
    assert expected_route(d, "cta-only").startswith("cta")
    if c.log is not None:
        assert (c.log.n, c.log.m) == (int(d["n_insdel"]), int(d["n_mark"]))


def test_threshold_shapes_are_exact():
    by = {c.name: c.batch.desc[0] for c in all_cases()}
    n = lambda k: int(by[k]["n_insdel"])
    m = lambda k: int(by[k]["n_mark"])
    R = lambda k: int(by[k]["n_actors"])
    assert (n("3actors-1022-m0"), n("3actors-1023-m0"), R("3actors-1022-m20")) == (1022, 1023, 3)
    assert (R("30actors"), R("31actors")) == (30, 31)
    assert (n("5actors-2046"), n("5actors-2047")) == (2046, 2047)
    for k, v in [("2048-records-marks", 2048), ("2049-records-marks", 2049), ("cta-1536", 1536), ("cta-1537", 1537),
                 ("cta-4096", 4096), ("cta-4097", 4097), ("cta-12288", 12288), ("cta-12289", 12289)]:
        assert n(k) + m(k) == v and m(k) > 0, k
    assert (m("marks-31999"), m("marks-32000")) == (31999, 32000)
    assert team_footprint(by["team-footprint-inside"]) == TEAM_SMEM and team_footprint(by["team-footprint-outside"]) > TEAM_SMEM
    ks = lambda k: int(by[k]["max_ctr"]) * R(k)
    assert (ks("keyspace-65534"), ks("keyspace-65535")) == (65534, 65535)
    # the compact table's overflow: inserts whose counter an earlier insert already holds
    for k, v in [("overflow-96", 96), ("overflow-97", 97)]:
        c = next(c for c in all_cases() if c.name == k)
        ctrs = [r[0] for r in c.log.ins if r[4] >> 30 == 0]
        assert len(ctrs) - len(set(ctrs)) == v
    # the Euler-tour splitter cases: exactly 8k - 1, 8k, 8k + 1 runs
    for runs in (127, 128, 129):
        c = next(c for c in all_cases() if c.name == f"runs-{runs}")
        heads = sum(1 for i, r in enumerate(c.log.ins) if r[1] == 0 or (r[1], r[3]) != c.log.ins[i - 1][0:3:2])
        assert heads == runs
    # segment work: 36 segments (35 distinct boundaries inside the text) and 768 / 769 surviving ops
    for k, ns in [("segment-work-1536", 768), ("segment-work-1538", 769)]:
        c = next(c for c in all_cases() if c.name == k)
        ids = {(r[0], r[2]): i for i, r in enumerate(c.log.ins)}
        bnd = {ids[(r[4], r[6])] for r in c.log.mk} | {ids[(r[5], r[7])] for r in c.log.mk}
        S = len(bnd - {0}) + 1
        assert c.log.m == ns and -(-S // 32) * ns in (1536, 1538)


def test_logs_are_causal():
    for c in all_cases():
        if c.log is None:
            continue
        seen = set()
        for (ctr, rc, a, ra, p) in c.log.ins:
            if rc:
                assert (rc, ra) in seen and rc < ctr or p >> 30 == 1 and (rc, ra) in seen, c.name
            if p >> 30 == 0:
                assert (ctr, a) not in seen, c.name
                seen.add((ctr, a))


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def kernel_config(config):
    return environ({"PT_WARP": None, "PT_WARP_FORCE": None, "PT_TEAM": None, **CONFIGS[config]["env"]})


def run_config(batch, config):
    from peritext_b200.engine import BatchEngine
    with kernel_config(config):
        e = BatchEngine(0)
        try:
            out = e.run(batch)
            st = e.stats()
        finally:
            e.close()
    return out, st


def assert_same(batch, got, ref, what, logs=None):
    for i in (range(batch.n_logs) if logs is None else logs):
        assert got.results[i]["status"] == ref.results[i]["status"], (what, i)
        assert got.canonical(i) == ref.canonical(i), (what, i)


@pytest.fixture(scope="module")
def merged():
    cases = all_cases()
    batch = joint_batch(cases)
    ref, _ = replay_packed(batch, threads=8)
    assert (ref.results["status"] == 0).all()
    return cases, batch, ref, {cfg: run_config(batch, cfg) for cfg in CONFIGS}


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_case_matches_the_oracle(merged, config):
    cases, batch, ref, outs = merged
    got, st = outs[config]
    for i, c in enumerate(cases):
        assert got.canonical(i) == ref.canonical(i), (c.name, config)
        if c.spans is not None:
            assert decode_spans(c.batch, got, i) == c.spans, (c.name, config)
    if config == "forced-deferral":
        assert st["logs_deferred_to_big_bin"] > 0


def defer_cases():
    return [(c.name, cfg) for c in all_cases() for cfg in c.defer]


@pytest.mark.gpu
@pytest.mark.parametrize("name,config", defer_cases())
def test_deferral_on_the_named_side(name, config):
    c = next(c for c in all_cases() if c.name == name)
    got, st = run_config(c.batch, config)
    ref, _ = replay_packed(c.batch)
    assert_same(c.batch, got, ref, (name, config))
    if c.defer[config]:
        assert st["logs_deferred_to_big_bin"] >= 1, (name, config, st)
    else:
        assert st["logs_deferred_to_big_bin"] == 0, (name, config, st)


@pytest.mark.gpu
def test_route_mirror_counts_the_warp_routed_logs():
    # a 256-byte slice holds nothing: with the host estimate skipped, every log the mirror sends to the warp kernel is deferred
    # to the first CTA bin exactly once (only logs that then fit that bin are taken, so no CTA bin defers them again)
    tiny = dict(env={"PT_WARP": "2048:8:256:4", "PT_WARP_FORCE": "1"}, warp=(2048, 256), team=True, force=True)
    CONFIGS["tiny"] = tiny
    try:
        cases = [c for c in all_cases() if int(c.batch.desc[0]["n_insdel"]) + int(c.batch.desc[0]["n_mark"]) <= 1100
                 and expected_route(c.batch.desc[0], "cta-only") == "cta1-u16"]
        cases += [c for c in all_cases() if c.name == "keyspace-65535"]
        batch = joint_batch(cases)
        want = sum(expected_route(d, "tiny") in WARP_ROUTES for d in batch.desc)
        assert 0 < want < batch.n_logs
        got, st = run_config(batch, "tiny")
    finally:
        del CONFIGS["tiny"]
    ref, _ = replay_packed(batch, threads=8)
    assert_same(batch, got, ref, "tiny")
    assert st["logs_deferred_to_big_bin"] == want


# ------------------------------------------------------------------------------------------------------------------
# Status matrix: one fault per log, in every route, next to clean logs
# ------------------------------------------------------------------------------------------------------------------
def route_base(route):
    """A clean log on `route` (default configuration) with room for the fault records appended below."""
    if route == "packed3":
        return lamport_forward(300, 3, 10)
    if route == "compact":
        return lamport_forward(300, 4, 10)
    if route == "direct":
        return lamport_forward(300, 2, 10)
    if route == "team":
        return lamport_forward(3000, 2)
    if route == "cta-u16":
        return lamport_forward(3000, 2, 300)
    return lamport_forward(1500, 2, 32000, seed=5, width=4)        # cta-u32: the mark count alone


def with_fault(lg, fault):
    """Appends the fault's records (fresh counters above everything in the log)."""
    c = lg.ctr
    last = (lg.ins[-1][0], lg.ins[-1][2])
    if fault == "missing-reference":
        lg.insert(1, (c + 1, 0), ctr=c + 2)                       # (c + 1, 0) is never inserted
    elif fault == "delete-head":
        lg.delete(0, HEAD)
    elif fault == "kind-2":
        lg.insert(0, last, kind=2)
    elif fault == "duplicate-opid":
        lg.insert(1, HEAD, ctr=c + 1); lg.insert(0, last, ctr=c + 2); lg.insert(1, HEAD, ctr=c + 1)   # unreferenced
    elif fault == "low-counter":
        x = lg.insert(1, HEAD, ctr=c + 1)
        lg.insert(0, x, ctr=c + 1)                                # opId (c+1, 0) is below its reference (c+1, 1)
    elif fault == "duplicate-and-missing":
        lg.insert(1, HEAD, ctr=c + 1); lg.insert(1, HEAD, ctr=c + 1)
        lg.insert(0, (c + 2, 1), ctr=c + 3)
    elif fault != "clean":
        raise ValueError(fault)
    return lg


FAULTS = {"clean": 0, "missing-reference": 1, "delete-head": 1, "kind-2": 3, "duplicate-opid": 2, "low-counter": 5,
          "duplicate-and-missing": 1}
ORACLE_DEFINES = {"clean", "missing-reference", "delete-head", "kind-2", "duplicate-and-missing"}
ROUTES = ["packed3", "compact", "direct", "team", "cta-u16", "cta-u32"]


def status_matrix():
    rows = [(r, f) for r in ROUTES for f in FAULTS]
    logs = [with_fault(route_base(r), f) for r, f in rows]
    return rows, batch_of(logs)


def test_status_matrix_logs_take_their_routes():
    rows, batch = status_matrix()
    for (r, f), d in zip(rows, batch.desc):
        got = expected_route(d)
        assert got == r if r in WARP_ROUTES + ("team",) else got.endswith(r[-4:]) and got.startswith("cta"), (r, f, got)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["default", "team-off", "cta-only", "forced-deferral"])
def test_status_matrix(config):
    rows, batch = status_matrix()
    got, _ = run_config(batch, config)
    ref, _ = replay_packed(batch, threads=8)
    for i, (r, f) in enumerate(rows):
        assert int(got.results[i]["status"]) == FAULTS[f], (config, r, f)
        if f in ORACLE_DEFINES:
            assert got.canonical(i) == ref.canonical(i), (config, r, f)
