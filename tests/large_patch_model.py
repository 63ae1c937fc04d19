"""Host model of `patch_large_kernel` (csrc/patch_large_kernel.cuh): the chunked arrival sweep, with the chunk size B as a
parameter, over one log's list ops and the final positions of its elements.  It keeps the kernel's state and corrections:
present / visible bitmaps with prefixes as of the chunk's start, plus the chunk's earlier ins/del ops; one insertion-only
max tree per mark type over the ranked boundary slots, plus the chunk's earlier mark ops; the comment ops sorted by
(id, op); FirstDef per boundary for the mark walk.  It returns the Patch dicts of `peritext_b200.patches.derive_patch`, so
tests/test_large_patch_model.py compares it with the host closed forms and the oracle."""
from __future__ import annotations

import numpy as np

from peritext_b200.packing import js_key, parse_op_id

INF = 1 << 62
TYPES = ["strong", "em", "comment", "link"]


class MaxTree:
    """Insertion-only max tree over `n` leaves: range update, point query (tree_update / tree_query)."""

    def __init__(self, n):
        self.P2 = 1
        while self.P2 < max(n, 1):
            self.P2 <<= 1
        self.t = [None] * (2 * self.P2)

    def update(self, l, r, v):
        l += self.P2; r += self.P2
        while l < r:
            if l & 1:
                self.t[l] = v if self.t[l] is None else max(self.t[l], v); l += 1
            if r & 1:
                r -= 1; self.t[r] = v if self.t[r] is None else max(self.t[r], v)
            l >>= 1; r >>= 1

    def query(self, leaf):
        x, v = leaf + self.P2, None
        while x:
            if self.t[x] is not None and (v is None or self.t[x] > v):
                v = self.t[x]
            x >>= 1
        return v


def op_key(op_id):
    c, a = parse_op_id(op_id)
    return (c, js_key(a))


def sweep_patches(ops, pos, B):
    """Patch list per op of `ops` (the log's list ops in arrival order); `pos`: elemId -> final position."""
    N = len(pos)
    recs, marks, order = [], [], []               # order: ("r", i) / ("m", k) in arrival order
    t_ins_of = {}
    for op in ops:
        a = op["action"]
        if a in ("addMark", "removeMark"):
            marks.append(dict(op=op, arrival=len(recs))); order.append(("m", len(marks) - 1))
        elif a == "set" or a == "del":
            i = len(recs)
            if a == "set":
                t_ins_of[op["opId"]] = i
                recs.append(dict(op=op, ins=True, p=pos[op["opId"]]))
            else:
                recs.append(dict(op=op, ins=False, p=pos[op["elemId"]]))
            order.append(("r", i))
        else:
            order.append(("x", None))
    n, m = len(recs), len(marks)
    TIns = np.full(N, INF, np.int64)
    TDel = np.full(N, INF, np.int64)
    for i, r in enumerate(recs):
        if r["ins"]:
            TIns[r["p"]] = i
        else:
            TDel[r["p"]] = min(TDel[r["p"]], i)

    def slot(b, arrival):                         # the arrived-before rule (src/peritext.ts:236-241)
        if b["type"] not in ("before", "after") or b["elemId"] not in t_ins_of or not t_ins_of[b["elemId"]] < arrival:
            return INF
        return 2 * pos[b["elemId"]] + (1 if b["type"] == "after" else 0)
    for mk in marks:
        op = mk["op"]
        mk["ps"], mk["raw"] = slot(op["start"], mk["arrival"]), slot(op["end"], mk["arrival"])
        mk["pe"] = INF if mk["raw"] == mk["ps"] else mk["raw"]
        mk["type"], mk["remove"], mk["key"] = op["markType"], op["action"] == "removeMark", op_key(op["opId"])
    bnd = sorted({s for mk in marks for s in (mk["ps"], mk["raw"]) if s != INF})
    rank = {s: r for r, s in enumerate(bnd)}
    D = len(bnd)
    srank_le = lambda s: int(np.searchsorted(np.array(bnd, np.int64), s, side="right"))     # boundaries <= s
    first_def = [INF] * D
    for y, mk in enumerate(marks):
        if mk["ps"] != INF and mk["ps"] <= mk["pe"]:
            first_def[rank[mk["ps"]]] = min(first_def[rank[mk["ps"]]], y)
        if mk["raw"] != INF and mk["raw"] != mk["ps"]:
            first_def[rank[mk["raw"]]] = min(first_def[rank[mk["raw"]]], y)
    csort = sorted((js_key(mk["op"]["attrs"]["id"]), k) for k, mk in enumerate(marks) if mk["type"] == "comment")
    cidx = {k: x for x, (_, k) in enumerate(csort)}
    trees = {t: MaxTree(D) for t in TYPES}

    def covers(mk, s):
        return mk["ps"] <= s < mk["pe"]

    out = [None] * len(order)
    pres = np.zeros(N, bool)
    vis = np.zeros(N, bool)
    for c0 in range(0, len(order), B):
        chunk = order[c0:c0 + B]
        pres_pre = np.concatenate([[0], np.cumsum(pres)])       # prefixes as of the chunk's start
        vis_pre = np.concatenate([[0], np.cumsum(vis)])
        crecs = [i for kind, i in chunk if kind == "r"]
        cmarks = [k for kind, k in chunk if kind == "m"]

        def vis_below(q, upto):                   # visible below position q after the chunk's records before `upto`
            v = int(vis_pre[q])
            for j in crecs:
                if j >= upto:
                    break
                r = recs[j]
                if r["p"] < q:
                    v += 1 if r["ins"] else (-1 if TDel[r["p"]] == j else 0)
            return v

        def lww(t, s, before):                    # the winner among the tree and the chunk's mark ops before `before`
            leaf1 = srank_le(s)
            w = trees[t].query(leaf1 - 1) if leaf1 else None
            for k in cmarks:
                if not before(k):
                    break
                mk = marks[k]
                if mk["type"] == t and covers(mk, s) and (w is None or (mk["key"], k) > w):
                    w = (mk["key"], k)
            return w

        for pos_in_chunk, (kind, idx) in enumerate(chunk):
            at = c0 + pos_in_chunk
            if kind == "x":
                out[at] = []
                continue
            if kind == "r":
                i, r = idx, recs[idx]
                op, p = r["op"], r["p"]
                index = vis_below(p, i)
                if not r["ins"]:
                    out[at] = [{"path": ["text"], "action": "delete", "index": index, "count": 1}] if TDel[p] == i else []
                    continue
                rk = int(pres_pre[p])
                py = int(np.flatnonzero(pres[:p])[rk - 1]) if rk else -1           # select(rank - 1)
                for j in crecs:
                    if j >= i:
                        break
                    if recs[j]["ins"] and recs[j]["p"] < p:
                        py = max(py, recs[j]["p"])
                marks_out = {}
                if py >= 0:
                    s = 2 * py + 1
                    before = lambda k: marks[k]["arrival"] <= i
                    for t in ("strong", "em", "link"):
                        w = lww(t, s, before)
                        if w is not None and not marks[w[1]]["remove"]:
                            marks_out[t] = marks[w[1]]["op"].get("attrs") or {"active": True}
                    if lww("comment", s, before) is not None:
                        ids, x = [], len(csort)
                        while x > 0:
                            cid = csort[x - 1][0]
                            decided = False
                            while x > 0 and csort[x - 1][0] == cid:
                                x -= 1
                                k = csort[x][1]
                                if not decided and marks[k]["arrival"] <= i and covers(marks[k], s):
                                    decided = True
                                    if not marks[k]["remove"]:
                                        ids.append(marks[k]["op"]["attrs"])
                        marks_out["comment"] = sorted(ids, key=lambda c: js_key(c["id"]))
                out[at] = [{"path": ["text"], "action": "insert", "index": index, "values": [op["value"]], "marks": marks_out}]
                continue
            X, mk = idx, marks[idx]
            op, ps, pe = mk["op"], mk["ps"], mk["pe"]
            res = []
            if ps != INF and ps < pe:
                upto = mk["arrival"]
                length = vis_below(N, upto)
                vis_at = lambda s: vis_below((s + 1) >> 1, upto)
                rend = D if pe == INF else rank[pe]
                cur, rc, start_i = ps, rank[ps], vis_at(ps)
                add = op["action"] == "addMark"
                while True:
                    nxt = pe
                    for r in range(rc + 1, rend):
                        if first_def[r] < X:
                            rc, nxt = r, bnd[r]
                            break
                    if mk["type"] != "comment":
                        w = lww(mk["type"], cur, lambda k: k < X)
                        if w is not None and w[0] > mk["key"]:
                            changed = False
                        else:
                            old_on = w is not None and not marks[w[1]]["remove"]
                            changed = old_on != add or (old_on and add and mk["type"] == "link" and marks[w[1]]["op"]["attrs"] != op["attrs"])
                    else:
                        any_c = lww("comment", cur, lambda k: k < X) is not None
                        has = False
                        x = cidx[X]
                        while x > 0 and csort[x - 1][0] == csort[cidx[X]][0]:
                            Y = csort[x - 1][1]
                            if covers(marks[Y], cur):
                                has = not marks[Y]["remove"]
                                break
                            x -= 1
                        changed = (not has) if add else (not any_c or has)
                    end_i = length if nxt == INF else vis_at(nxt)
                    if changed and end_i > start_i and start_i < length:
                        patch = {"action": op["action"], "markType": mk["type"], "path": ["text"], "startIndex": start_i}
                        if add and mk["type"] in ("link", "comment"):
                            patch["attrs"] = op["attrs"]
                        patch["endIndex"] = end_i
                        res.append(patch)
                    if nxt == pe:
                        break
                    cur, start_i = nxt, end_i
            out[at] = res
        # advance the state past the chunk: bitmaps, then the trees
        for j in crecs:
            r = recs[j]
            if r["ins"]:
                pres[r["p"]] = True
                if not TDel[r["p"]] <= crecs[-1]:
                    vis[r["p"]] = True
            elif TDel[r["p"]] == j and TIns[r["p"]] < crecs[0]:
                vis[r["p"]] = False
        for k in cmarks:
            mk = marks[k]
            if mk["ps"] != INF and mk["ps"] < mk["pe"]:
                trees[mk["type"]].update(rank[mk["ps"]], D if mk["pe"] == INF else rank[mk["pe"]], (mk["key"], k))
    return out
