"""Python restatements of the reference's TEST HARNESS helpers (not of the product path):

* generateDocs      — reference test/generateDocs.ts:11-42
* accumulatePatches — reference test/accumulatePatches.ts:9-80   (second oracle for the Patch stream)
* applyChanges / getMissingChanges — reference test/merge.ts:4-38
* run_concurrent    — testConcurrentWrites, reference test/micromerge.ts:46-86

They are written against the reference's `Micromerge` class surface, so they drive either the CPU oracle
(`oracle.oracle.Micromerge`) or the engine facade (`peritext_b200.Micromerge`) unchanged.  `environ` sets the engine's
kernel-selection variables around a block.
"""
from __future__ import annotations

import copy
import json
import os
from contextlib import contextmanager

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@contextmanager
def environ(env):
    """Sets the variables of `env` (None: unset) for the block, then restores their earlier values."""
    old = {k: os.environ.get(k) for k in env}

    def apply(values):
        for k, v in values.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    try:
        apply(env)
        yield
    finally:
        apply(old)


def load_kats():
    with open(os.path.join(GOLDEN, "kats.json"), encoding="utf-8") as f:
        return json.load(f)["kats"]


def generateDocs(Micromerge, text="The Peritext editor", count=2):
    docs = [Micromerge(f"doc{i + 1}") for i in range(count)]
    patches = [[] for _ in range(count)]
    r = docs[0].change([
        {"path": [], "action": "makeList", "key": "text"},
        {"path": ["text"], "action": "insert", "index": 0, "values": list(text)},
    ])
    patches[0] = r["patches"]
    for i, doc in enumerate(docs):
        if i == 0:
            continue
        patches[i] = doc.applyChange(r["change"])
    return docs, patches, r["change"]


def addCharactersToSpans(characters, marks, spans):
    """reference src/peritext.ts:438-455 (harness copy: accumulatePatches imports it)."""
    if not characters:
        return
    if spans and spans[-1]["marks"] == marks:
        spans[-1]["text"] += "".join(characters)
    else:
        spans.append({"text": "".join(characters), "marks": marks})


def accumulatePatches(patches):
    metadata = []
    for patch in patches:
        assert patch["path"] == ["text"]
        a = patch["action"]
        if a == "insert":
            for vi, ch in enumerate(patch["values"]):
                metadata.insert(patch["index"] + vi, {"character": ch, "marks": copy.copy(patch["marks"])})
        elif a == "delete":
            del metadata[patch["index"]: patch["index"] + patch["count"]]
        elif a == "addMark":
            for index in range(patch["startIndex"], patch["endIndex"]):
                mt = patch["markType"]
                if mt != "comment":
                    metadata[index]["marks"][mt] = dict(patch.get("attrs") or {"active": True})
                else:
                    arr = metadata[index]["marks"].get(mt)
                    if arr is None:
                        metadata[index]["marks"][mt] = [dict(patch["attrs"])]
                    elif not any(c["id"] == patch["attrs"]["id"] for c in arr):
                        metadata[index]["marks"][mt] = sorted(arr + [dict(patch["attrs"])], key=lambda c: c["id"])
        elif a == "removeMark":
            for index in range(patch["startIndex"], patch["endIndex"]):
                metadata[index]["marks"].pop(patch["markType"], None)
        elif a == "makeList":
            pass
        else:
            raise AssertionError(a)
    spans = []
    for m in metadata:
        addCharactersToSpans([m["character"]], m["marks"], spans)
    return spans


def applyChanges(document, changes):
    """reference test/merge.ts:4-23 (causal retry by requeue)."""
    changes = list(changes)
    iterations = 0
    patches = []
    while changes:
        change = changes.pop(0)
        try:
            patches.extend(document.applyChange(change))
        except Exception:
            changes.append(change)
        iterations += 1
        if iterations > 10000:
            raise RuntimeError("applyChanges did not converge")
    return patches


def getMissingChanges(source, target, queues):
    """reference test/merge.ts:25-38"""
    changes = []
    tclock = target.clock
    for actor, number in source.clock.items():
        if actor not in tclock:
            changes.extend(queues[actor][0:number])
        elif tclock[actor] < number:
            changes.extend(queues[actor][tclock[actor]:number])
    return changes


def with_path(ops):
    return [{**op, "path": ["text"]} for op in ops]


def run_concurrent(Micromerge, kat, record=None):
    """testConcurrentWrites (reference test/micromerge.ts:46-86).  Returns (docs, patchLists).
    `record`, if given, collects every Change each doc applied in arrival order: record[docIndex] = [change...]."""
    docs, patches, initial = generateDocs(Micromerge, kat["initialText"])
    doc1, doc2 = docs
    p1, p2 = list(patches[0]), list(patches[1])
    log = [[initial], [initial]]
    if kat.get("preOps"):
        r0 = doc1.change(with_path(kat["preOps"]))
        p1 += r0["patches"]
        p2 += doc2.applyChange(r0["change"])
        log[0].append(r0["change"]); log[1].append(r0["change"])
    r1 = doc1.change(with_path(kat["inputOps1"])); p1 += r1["patches"]; log[0].append(r1["change"])
    r2 = doc2.change(with_path(kat["inputOps2"])); p2 += r2["patches"]; log[1].append(r2["change"])
    p2 += doc2.applyChange(r1["change"]); log[1].append(r1["change"])
    p1 += doc1.applyChange(r2["change"]); log[0].append(r2["change"])
    if record is not None:
        record.extend(log)
    return docs, [p1, p2]


# ------------------------------------------------------------------------------------------------------------------
# Seeded fuzz sessions in the shape of reference test/fuzz.ts:23-199 (driven through any Micromerge class).
# Deviations (SURVEY.md §8d): seeded RNG; removeMark really emits removeMark (fuzz.ts:80 emits addMark);
# removeMark/comment reuses an id the acting replica has already seen, so no concurrent add/remove of one id (Q4).
# ------------------------------------------------------------------------------------------------------------------
import random as _random

_URLS = [f"{c}.com" for c in "ABCDEFGHIJKLMNOPQRSTUVWXYZ"]
_MARKS = ["strong", "em", "link", "comment"]


def fuzz_session(Micromerge, seed, n_steps, replicas=3, initial="ABCDE", sync_prob=1.0, full_sync_at_end=True,
                 max_chars=2, zero_width_prob=0.0, remove_comments=True, on_patches=None):
    """Returns (docs, logs, queues): logs[r] = Changes replica r applied (own + remote) in arrival order."""
    rng = _random.Random(seed)
    docs, _, init = generateDocs(Micromerge, initial, replicas)
    ids = [d.actorId for d in docs]
    queues = {a: [] for a in ids}
    queues[ids[0]].append(init)
    logs = [[init] for _ in docs]
    seen_comments = [[] for _ in docs]   # comment ids each replica has seen (own adds + synced)
    comment_owner = {}
    n_comment = 0

    def sync(li, ri):
        for src, dst in ((li, ri), (ri, li)):
            missing = getMissingChanges(docs[src], docs[dst], queues)
            pending = list(missing)
            it = 0
            while pending:
                ch = pending.pop(0)
                try:
                    ps = docs[dst].applyChange(ch)
                    if on_patches is not None:
                        on_patches(dst, ps)
                    logs[dst].append(ch)
                    for op in ch["ops"]:
                        if op["action"] == "addMark" and op.get("markType") == "comment":
                            seen_comments[dst].append(op["attrs"]["id"])
                except Exception:
                    pending.append(ch)
                it += 1
                assert it < 10000

    for _ in range(n_steps):
        t = rng.randrange(replicas)
        doc = docs[t]
        length = len(doc.root["text"])
        kind = rng.choice(["insert", "remove", "addMark", "removeMark"])
        op = None
        if kind == "insert" or length == 0:
            index = rng.randrange(length) if length else 0
            nchars = rng.randrange(max_chars) if length else 1     # fuzz.ts:111-113: randomBytes(n).toString("hex")
            vals = [rng.choice("0123456789abcdef") for _ in range(2 * nchars)]
            op = {"path": ["text"], "action": "insert", "index": index, "values": vals}
        elif kind == "remove":
            index = rng.randrange(length) + 1
            count = -(-rng.random() * (length - index) // 1)
            count = int(count)
            op = {"path": ["text"], "action": "delete", "index": index, "count": count}
        else:
            start = rng.randrange(length)
            end = start + rng.randrange(length - start) + 1
            mt = rng.choice(_MARKS)
            if zero_width_prob and rng.random() < zero_width_prob and not (start == 0 and mt in ("link", "comment")):
                end = start   # (a zero-width non-inclusive mark at index 0 throws in the reference: getListElementId(-1))
            op = {"path": ["text"], "action": kind, "startIndex": start, "endIndex": end, "markType": mt}
            if mt == "link" and kind == "addMark":
                op["attrs"] = {"url": rng.choice(_URLS)}
            elif mt == "comment":
                if kind == "addMark":
                    n_comment += 1
                    cid = "comment-%04x-%d" % (rng.randrange(65536), n_comment)
                    op["attrs"] = {"id": cid}
                    seen_comments[t].append(cid)
                else:
                    if not seen_comments[t] or not remove_comments:
                        continue
                    op["attrs"] = {"id": rng.choice(seen_comments[t])}
        r = doc.change([op])
        if on_patches is not None:
            on_patches(t, r["patches"])
        queues[ids[t]].append(r["change"])
        logs[t].append(r["change"])
        if rng.random() < sync_prob:
            li = rng.randrange(replicas)
            ri = rng.randrange(replicas)
            while ri == li:
                ri = rng.randrange(replicas)
            sync(li, ri)
    if full_sync_at_end:
        for _ in range(2):
            for a in range(replicas):
                for b in range(a + 1, replicas):
                    sync(a, b)
    return docs, logs, queues
