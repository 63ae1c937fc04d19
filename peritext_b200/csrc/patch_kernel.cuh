// patch_kernel.cuh — the reference's Patch stream for whole logs, on the device (sm_90a).
//
// Micromerge.applyChange returns, for every op it applies, the Patch the editor needs (reference src/micromerge.ts:659-671
// insert {index, marks}, :689-703 delete {index}, src/peritext.ts:175-220, 251-281 mark patches).  Sequentially these depend
// on the replica's state at apply time; they are functions of (a) the FINAL position of every element in the sequence —
// which the merge kernels materialise (PT_FLAG_EMIT_SEQUENCE) — and (b) the ARRIVAL index of every op (SURVEY.md §9.5;
// proven against the oracle's patch stream by tests/test_patch_closed_form.py on the host model peritext_b200/patches.py):
//   insert / delete index = #{ e : pos(e) < pos(x), e inserted before t, not deleted before t }      (2-D dominance count)
//   insert marks          = opsToMarks of the mark ops that arrived before t and cover the slot after the nearest element
//                           left of x that was present at t (getActiveMarksAtIndex, src/peritext.ts:328-330, 405-436)
//   mark patches          = one per maximal visible range between consecutive slots DEFINED at time t inside the op's range
//                           where adding the op changes the effective marks (src/peritext.ts:198-220)
// One warp per log; every count is a uniform loop over shared-memory tables (lane = one op, broadcast reads).  The loops
// are quadratic in the log's size, which is what a document under interactive editing needs (the facade's use); logs
// beyond PT_PATCH_MAX_* are reported as "not computed" and the host closed forms take over.
//
// Patch window (pt_batch_set_patch_window).  Every op's patch is a function of the two inputs above alone, so the ops of a
// suffix of the log can be computed without the others.  The tables (T, PosOf, TIns, TDel, the mark slots) still cover the
// whole log, because the window's ops count and cover elements of every age; only the per-op loops start at the window:
// ins/del records [j0, n) and mark ops [k0, m), where k0 mark records and j0 ins/del records lie before list-op position
// first_op (patch_window.cuh).  The records before the window are written as {0, 0, PT_ATTR_NONE, 0} and emit no items.  The
// quadratic part becomes O(window x log) per log; the linear table phase is unchanged.
#pragma once
#include "warp_kernel.cuh"
#include "patch_window.cuh"

namespace ptk {

constexpr uint32_t kInfSlot = 0xFFFFFFFFu;

struct PatchParams {
    const pt_log_desc* __restrict__ desc;
    const pt_insdel_rec* __restrict__ insdel;
    const pt_mark_rec* __restrict__ marks;
    const pt_log_result* __restrict__ results;
    const uint64_t* __restrict__ text_off;      // capacity layout: where the log's element sequence starts
    const uint32_t* __restrict__ seq;           // element sequence (record index | deleted << 31)
    const uint32_t* __restrict__ first_op;      // per log: list-op position of the window's first op (0: the whole log)
    uint32_t n_logs;
    uint32_t smem_bytes;                        // dynamic shared memory of the CTA (one warp)
    pt_patch_rec* recs;                         // one per ins/del record (same offsets as the records)
    pt_patch_item* items;                       // pool: mark patches and the comment ids of insert patches, any order
    unsigned long long* item_cursor;            // counts past item_cap: the batch's demand
    unsigned long long item_cap;
    uint32_t* status;                           // per log: 0 computed, 1 not computed (too large / merge failed)
};

__device__ __forceinline__ void patch_emit(const PatchParams& P, uint32_t log, uint32_t tag, uint32_t a, uint32_t b) {
    const unsigned long long at = atomicAdd(P.item_cursor, 1ull);
    if (at < P.item_cap) { pt_patch_item it; it.log = log; it.tag = tag; it.a = a; it.b = b; P.items[at] = it; }
}

__global__ void __launch_bounds__(32) patch_logs_kernel(const PatchParams P) {
    const uint32_t lane = threadIdx.x;
    for (uint32_t li = blockIdx.x; li < P.n_logs; li += gridDim.x) {
        const pt_log_desc L = P.desc[li];
        const pt_log_result RS = P.results[li];
        const uint32_t n = L.n_insdel, m = L.n_mark, R = L.n_actors ? L.n_actors : 1u, C = L.max_ctr, N = RS.n_elems;
        const unsigned long long KS64 = (unsigned long long)C * R;
        // footprint: T u16[KS] | PosOf u16[n] | TIns u16[N] | TDel u32[N] | Ps, Pe, PeRaw, MInfo, MAttr, MArr u32[m] | CList u16[m]
        const unsigned long long need = ((KS64 * 2 + 15) & ~15ull) + ((n * 2ull + 15) & ~15ull) + ((N * 2ull + 15) & ~15ull) + ((N * 4ull + 15) & ~15ull) +
                                        6 * ((m * 4ull + 15) & ~15ull) + ((m * 2ull + 15) & ~15ull) + 64;
        if (RS.status != 0 || KS64 >= 0xFFFFull || n >= 0xFFFFu || m >= 0xFFFFu || need > P.smem_bytes) {
            if (lane == 0) P.status[li] = 1;
            continue;
        }
        const uint32_t KS = (uint32_t)KS64;
        const pt_insdel_rec* __restrict__ ins = P.insdel + L.insdel_off;
        const pt_mark_rec* __restrict__ mk = P.marks + L.mark_off;
        const uint32_t* __restrict__ seq = P.seq + P.text_off[li];
        pt_patch_rec* out = P.recs + L.insdel_off;
        WArena A; A.base = 0; A.used = 0; A.cap = P.smem_bytes;
        uint16_t* T = A.alloc<uint16_t>(KS);
        uint16_t* PosOf = A.alloc<uint16_t>(n);        // record -> sequence position of the element it inserts / deletes
        uint16_t* TIns = A.alloc<uint16_t>(N);         // position -> arrival index of the insert
        uint32_t* TDel = A.alloc<uint32_t>(N);         // position -> arrival index of the FIRST delete (kInfSlot: never)
        uint32_t* Ps = A.alloc<uint32_t>(m);           // start slot (kInfSlot: never matched)
        uint32_t* Pe = A.alloc<uint32_t>(m);           // effective end slot (kInfSlot: never ends; same slot as start: start wins)
        uint32_t* PeRaw = A.alloc<uint32_t>(m);        // end slot as written by the walk (defines a slot even when the start was missed)
        uint32_t* MInfo = A.alloc<uint32_t>(m);        // opId key | type << 16 | remove << 18
        uint32_t* MAttr = A.alloc<uint32_t>(m);
        uint32_t* MArr = A.alloc<uint32_t>(m);         // ins/del records that arrived before the mark op
        uint16_t* CList = A.alloc<uint16_t>(m);        // indices of the comment mark ops, arrival order
        auto keyOf = [&](uint32_t ctr, uint32_t actor) -> uint32_t { return (ctr - 1u) * R + actor; };
        auto badId = [&](uint32_t ctr, uint32_t actor) -> bool { return ctr - 1u >= C || actor >= R; };
        wfill<uint16_t>(T, KS, (uint16_t)kNone16, lane);
        wfill<uint32_t>(TDel, N, kInfSlot, lane);
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) {
            const uint4 r = ld_rec(ins + i);
            if ((r.w >> 30) == PT_KIND_INSERT) T[keyOf(r.x, r.z & 0xFFFFu)] = (uint16_t)i;
        }
        for (uint32_t p = lane; p < N; p += 32) { const uint32_t rec = seq[p] & 0x3FFFFFFFu; PosOf[rec] = (uint16_t)p; TIns[p] = (uint16_t)rec; }
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) {
            const uint4 r = ld_rec(ins + i);
            if ((r.w >> 30) == PT_KIND_DELETE) {
                const uint32_t p = PosOf[T[keyOf(r.y, r.z >> 16)]];        // the merge succeeded: the target exists and arrived earlier
                PosOf[i] = (uint16_t)p;
                atomicMin(&TDel[p], i);
            }
        }
        // mark ops -> slots (2 * position + after), with the reference's rule that a boundary element must have arrived
        // before the op (src/peritext.ts:236-241); comment ops also go to CList
        uint32_t mc = 0;
        for (uint32_t kb = 0; kb < m; kb += 32) {
            const uint32_t k = kb + lane;
            bool isC = false;
            if (k < m) {
                const uint4* q = reinterpret_cast<const uint4*>(mk + k);
                const uint4 a0 = __ldg(q), a1 = __ldg(q + 1);
                const uint32_t kind = (a0.y >> 16) & 0xFFu, bounds = a0.y >> 24, arrival = a1.z;
                const uint32_t sb = bounds & 3u, eb = (bounds >> 2) & 3u;
                uint32_t ps = kInfSlot, pr = kInfSlot;
                if (sb <= PT_BOUND_AFTER && !badId(a0.z, a1.x & 0xFFFFu)) { const uint32_t j = T[keyOf(a0.z, a1.x & 0xFFFFu)]; if (j != kNone16 && j < arrival) ps = 2u * PosOf[j] + sb; }
                if (eb <= PT_BOUND_AFTER && !badId(a0.w, a1.x >> 16)) { const uint32_t j = T[keyOf(a0.w, a1.x >> 16)]; if (j != kNone16 && j < arrival) pr = 2u * PosOf[j] + eb; }
                Ps[k] = ps; PeRaw[k] = pr; Pe[k] = pr == ps ? kInfSlot : pr;
                MInfo[k] = keyOf(a0.x, a0.y & 0xFFFFu) | (((kind >> 1) & 3u) << 16) | ((kind & 1u) << 18);
                MAttr[k] = a1.y; MArr[k] = arrival;
                isC = ((kind >> 1) & 3u) == PT_MARK_COMMENT;
            }
            const uint32_t bal = __ballot_sync(kFull, isC);
            if (isC) CList[mc + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)k;
            mc += __popc(bal);
        }
        __syncwarp();
        const uint32_t w0 = P.first_op[li], k0 = ptw::marks_before(mk, n, m, w0, lane), j0 = w0 - k0;
        for (uint32_t i = lane; i < j0; i += 32) { pt_patch_rec z; z.index = 0; z.flags = 0; z.link_attr = PT_ATTR_NONE; z.reserved = 0; out[i] = z; }

        // ---- insert / delete patches: one lane per record, uniform loops over the elements / the mark ops -------------------
        for (uint32_t ib = j0; ib < n; ib += 32) {
            const uint32_t i = ib + lane;
            const bool live = i < n;
            uint32_t p = 0; bool isIns = false;
            if (live) { p = PosOf[i]; isIns = (__ldg(&ins[i].payload) >> 30) == PT_KIND_INSERT; }
            uint32_t cnt = 0, py = kInfSlot;
            for (uint32_t q = 0; q < N; q++) {
                const uint32_t ti = TIns[q], td = TDel[q];
                if (live && q < p && ti < i) { py = q; if (!(td < i)) cnt++; }      // present at time i / visible at time i
            }
            uint32_t flags = 0, link = PT_ATTR_NONE, ncom = 0;
            if (__any_sync(kFull, live && isIns && py != kInfSlot)) {
                // marks inherited by the new element: ops that arrived before record i and cover the slot after element py
                const uint32_t s = 2u * py + 1u;
                const bool want = live && isIns && py != kInfSlot;
                uint32_t w0 = 0, w1 = 0, w2 = 0;
                for (uint32_t k = 0; k < m; k++) {
                    const uint32_t info = MInfo[k], t = (info >> 16) & 3u;
                    if (want && MArr[k] <= i && Ps[k] <= s && s < Pe[k]) {
                        const uint32_t val = (((info & 0xFFFFu) << 16) | k) + 1u;       // LWW by opId (src/peritext.ts:304-313)
                        if (t == PT_MARK_STRONG) w0 = max(w0, val); else if (t == PT_MARK_EM) w1 = max(w1, val);
                        else if (t == PT_MARK_LINK) w2 = max(w2, val); else flags |= PT_SPAN_COMMENT;
                    }
                }
                if (w0 && !((MInfo[(w0 - 1u) & 0xFFFFu] >> 18) & 1u)) flags |= PT_SPAN_STRONG;
                if (w1 && !((MInfo[(w1 - 1u) & 0xFFFFu] >> 18) & 1u)) flags |= PT_SPAN_EM;
                if (w2) { const uint32_t k2 = (w2 - 1u) & 0xFFFFu; if (!((MInfo[k2] >> 18) & 1u)) { flags |= PT_SPAN_LINK; link = MAttr[k2]; } }
                if (__any_sync(kFull, (flags & PT_SPAN_COMMENT) != 0)) {
                    // comment ids: the last-arrived covering op of an id decides (fold in arrival order, src/peritext.ts:314-322)
                    for (uint32_t c1 = 0; c1 < mc; c1++) {
                        const uint32_t k = CList[c1];
                        const bool cov = want && (flags & PT_SPAN_COMMENT) && MArr[k] <= i && Ps[k] <= s && s < Pe[k];
                        if (!__any_sync(kFull, cov)) continue;
                        const uint32_t id = MAttr[k];
                        bool later = false;
                        for (uint32_t c2 = c1 + 1; c2 < mc; c2++) {
                            const uint32_t k2 = CList[c2];
                            if (MAttr[k2] != id) continue;
                            if (MArr[k2] <= i && Ps[k2] <= s && s < Pe[k2]) later = true;
                        }
                        if (cov && !later && !((MInfo[k] >> 18) & 1u)) { patch_emit(P, li, i, id, 0); ncom++; }
                    }
                }
            }
            if (live) {
                pt_patch_rec pr;
                const bool emits = isIns || TDel[p] == i;          // a delete emits a patch only if it is the element's first
                pr.index = cnt | (emits ? 0x80000000u : 0u); pr.flags = flags | (ncom << 8); pr.link_attr = link; pr.reserved = 0;
                out[i] = pr;
            }
        }

        // ---- mark patches: one lane per mark op X; intervals between consecutive slots defined at its arrival time ---------
        for (uint32_t xb = k0; xb < m; xb += 32) {
            const uint32_t X = xb + lane;
            if (X >= m) continue;
            const uint32_t ps = Ps[X], pe = Pe[X];
            if (ps == kInfSlot || ps >= pe) continue;
            const uint32_t tX = MArr[X], infoX = MInfo[X], typeX = (infoX >> 16) & 3u, keyX = infoX & 0xFFFFu, attrX = MAttr[X];
            const bool addX = !((infoX >> 18) & 1u);
            uint32_t length = 0;
            for (uint32_t q = 0; q < N; q++) if (TIns[q] < tX && !(TDel[q] < tX)) length++;
            uint32_t cur = ps, start_i = 0;
            for (uint32_t q = 0; q < N && 2u * q + 1u <= cur; q++) if (TIns[q] < tX && !(TDel[q] < tX)) start_i++;
            for (;;) {
                // next slot after `cur` that an earlier op defined (its start if the walk reached it, its end), else the op's end
                uint32_t nxt = pe;
                for (uint32_t Y = 0; Y < X; Y++) {
                    const uint32_t ys = Ps[Y], ye = Pe[Y], yr = PeRaw[Y];
                    if (ys != kInfSlot && ys <= ye && ys > cur && ys < nxt) nxt = ys;
                    if (yr != kInfSlot && yr != ys && yr > cur && yr < nxt) nxt = yr;
                }
                // does adding X change the effective marks on [cur, nxt)?
                bool changed;
                if (typeX != PT_MARK_COMMENT) {
                    uint32_t w = 0;
                    for (uint32_t Y = 0; Y < X; Y++) {
                        const uint32_t inf = MInfo[Y];
                        if (((inf >> 16) & 3u) == typeX && Ps[Y] != kInfSlot && Ps[Y] <= cur && cur < Pe[Y]) w = max(w, (((inf & 0xFFFFu) << 16) | Y) + 1u);
                    }
                    if (w && (w - 1u) >> 16 > keyX) changed = false;                       // an earlier-arrived op with a larger opId keeps winning
                    else {
                        const uint32_t Yw = (w - 1u) & 0xFFFFu;
                        const bool oldOn = w && !((MInfo[Yw] >> 18) & 1u);
                        changed = oldOn != addX || (oldOn && addX && typeX == PT_MARK_LINK && MAttr[Yw] != attrX);
                    }
                } else {
                    bool any = false, has = false;
                    for (uint32_t Y = 0; Y < X; Y++) {
                        const uint32_t inf = MInfo[Y];
                        if (((inf >> 16) & 3u) == PT_MARK_COMMENT && Ps[Y] != kInfSlot && Ps[Y] <= cur && cur < Pe[Y]) {
                            any = true;
                            if (MAttr[Y] == attrX) has = !((inf >> 18) & 1u);               // arrival order: the last one decides
                        }
                    }
                    changed = addX ? !has : (!any || has);      // a remove on a range without the `comment` key creates `comment: []`
                }
                uint32_t end_i = length;
                if (nxt != kInfSlot) { end_i = 0; for (uint32_t q = 0; q < N && 2u * q + 1u <= nxt; q++) if (TIns[q] < tX && !(TDel[q] < tX)) end_i++; }
                if (changed && end_i > start_i && start_i < length) patch_emit(P, li, X | 0x80000000u, start_i, end_i);
                if (nxt == pe) break;
                cur = nxt; start_i = end_i;
            }
        }
        if (lane == 0) P.status[li] = 0;
        __syncwarp();
    }
}

}  // namespace ptk
