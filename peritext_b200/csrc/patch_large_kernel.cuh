// patch_large_kernel.cuh — the Patch stream of logs too large for patch_logs_kernel (PT_FLAG_EMIT_LARGE_PATCHES), sm_90a.
//
// Same closed forms and the same outputs as patch_kernel.cuh (records, items, item demand, window), for the logs the warp
// kernel declines: max_ctr x n_actors >= 0xFFFF, or a footprint above its shared memory.  One CTA per log, tables in a
// global scratch slot per resident CTA (32-bit indices; several MB per c5 log, so in L2 and HBM).  Instead of the warp kernel's per-op
// loops over every element and every earlier mark op, the CTA sweeps the log's list ops in ARRIVAL order, kLargeChunk ops
// at a time (one op per thread), holding the state "as of the chunk's start":
//   * present / visible bitmaps over final positions with exclusive per-word popcount prefixes: an index is a prefix read
//     plus the corrections of the chunk's earlier ins/del ops (O(chunk) from shared memory); an insert's present
//     predecessor is a select on the present prefix (binary search over the word prefixes, then an in-word select);
//   * one insertion-only max tree per mark type over the compressed boundary slots (every finite start / end slot of the
//     log's mark ops, ranked by a slot bitmap + prefix): a mark op is a range update of (opId key, op) when the sweep
//     passes it, a lookup at a slot is a point query; the chunk's own earlier mark ops are a loop over shared memory.  The
//     comment tree answers "does an earlier comment op cover this slot";
//   * comment ids: the comment ops sorted once by (id, op) — every id's ops in arrival order — so an insert covered by a
//     comment op finds each id's last covering op in one pass over the log's comment ops, and a comment op's `has` is a
//     backward scan of its own id;
//   * defined slots: FirstDef[b] = the first mark op whose walk defines boundary b (the rules of patch_kernel.cuh:198-201),
//     so a mark op X steps over the boundaries inside its range and keeps those with FirstDef < X.
// Cost per log: O(N/32) per chunk (bitmap prefixes), O(chunk + log N) per ins/del op, O(log D) per tree update / query,
// O(comment ops) per insert covered by a comment op, and per mark op O(boundaries inside its range x (chunk + log D)).
// No per-op loop runs over all elements or all earlier mark ops of the log.  DESIGN.md §4.9.
#pragma once
#include "patch_kernel.cuh"
#include "plan.h"

namespace ptk {

constexpr int kLargeThreads = 512;        // one list op per thread per chunk
constexpr uint32_t kLargeChunk = kLargeThreads;
constexpr uint32_t kLargeNone = 0xFFFFFFFFu;

struct LargePatchParams {
    const pt_log_desc* __restrict__ desc;
    const pt_insdel_rec* __restrict__ insdel;
    const pt_mark_rec* __restrict__ marks;
    const pt_log_result* __restrict__ results;
    const uint64_t* __restrict__ text_off;
    const uint32_t* __restrict__ seq;
    const uint32_t* __restrict__ first_op;
    const uint32_t* __restrict__ cand;          // candidate logs (plan.h Plan::large_cand)
    uint32_t n_cand;
    uint32_t after_warp;                        // patch_logs_kernel ran first: take only the candidates it left at status 1
    char* scratch;                              // one slot of slot_bytes per CTA
    unsigned long long slot_bytes;
    pt_patch_rec* recs;
    pt_patch_item* items;
    unsigned long long* item_cursor;
    unsigned long long item_cap;
    uint32_t* status;
};

__device__ __forceinline__ void large_emit(const LargePatchParams& P, uint32_t log, uint32_t tag, uint32_t a, uint32_t b) {
    const unsigned long long at = atomicAdd(P.item_cursor, 1ull);
    if (at < P.item_cap) { pt_patch_item it; it.log = log; it.tag = tag; it.a = a; it.b = b; P.items[at] = it; }
}

// Block-wide exclusive scan of per-thread pairs; sh holds 2 x 32 words.  Returns the pair's exclusive prefix; tot = totals.
__device__ __forceinline__ uint2 block_scan2(uint2 v, uint32_t* sh, uint2& tot) {
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    uint2 inc = v;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t a = __shfl_up_sync(kFull, inc.x, d), b = __shfl_up_sync(kFull, inc.y, d);
        if (lane >= (uint32_t)d) { inc.x += a; inc.y += b; }
    }
    if (lane == 31) { sh[w] = inc.x; sh[32 + w] = inc.y; }
    __syncthreads();
    if (w == 0) {
        constexpr uint32_t nw = kLargeThreads / 32;
        uint32_t a = lane < nw ? sh[lane] : 0u, b = lane < nw ? sh[32 + lane] : 0u;
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t x = __shfl_up_sync(kFull, a, d), y = __shfl_up_sync(kFull, b, d);
            if (lane >= (uint32_t)d) { a += x; b += y; }
        }
        if (lane < nw) { sh[lane] = a; sh[32 + lane] = b; }
    }
    __syncthreads();
    constexpr uint32_t last = kLargeThreads / 32 - 1;
    tot = make_uint2(sh[last], sh[32 + last]);
    const uint2 base = w ? make_uint2(sh[w - 1], sh[32 + w - 1]) : make_uint2(0u, 0u);
    __syncthreads();                                   // sh is reused by the next scan
    return make_uint2(base.x + inc.x - v.x, base.y + inc.y - v.y);
}

// Exclusive popcount prefixes of two bitmaps of nw words (b may be null): pa[w], pb[w] for w in [0, nw], contiguous word
// ranges per thread.
__device__ void prefix_words(const uint32_t* a, uint32_t* pa, const uint32_t* b, uint32_t* pb, uint32_t nw, uint32_t* sh) {
    const uint32_t per = (nw + kLargeThreads - 1) / kLargeThreads, lo = min(nw, threadIdx.x * per), hi = min(nw, lo + per);
    uint2 s = make_uint2(0u, 0u);
    for (uint32_t w = lo; w < hi; w++) { s.x += __popc(a[w]); if (b) s.y += __popc(b[w]); }
    uint2 tot;
    uint2 run = block_scan2(s, sh, tot);
    for (uint32_t w = lo; w < hi; w++) {
        pa[w] = run.x; run.x += __popc(a[w]);
        if (b) { pb[w] = run.y; run.y += __popc(b[w]); }
    }
    if (threadIdx.x == 0) { pa[nw] = tot.x; if (b) pb[nw] = tot.y; }
}

__device__ __forceinline__ uint32_t rank_below(const uint32_t* bits, const uint32_t* pre, uint32_t p) {
    return pre[p >> 5] + __popc(bits[p >> 5] & ((1u << (p & 31u)) - 1u));
}

// Position of the r-th (0-based) set bit; r < the bitmap's population.
__device__ __forceinline__ uint32_t select_bit(const uint32_t* bits, const uint32_t* pre, uint32_t nw, uint32_t r) {
    uint32_t lo = 0, hi = nw;                           // largest w with pre[w] <= r
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (pre[mid] <= r) lo = mid; else hi = mid; }
    uint32_t word = bits[lo];
    for (uint32_t k = r - pre[lo]; k; k--) word &= word - 1u;
    return lo * 32u + (uint32_t)(__ffs(word) - 1);
}

__device__ __forceinline__ void tree_update(unsigned long long* t, uint32_t P2, uint32_t l, uint32_t r, unsigned long long v) {
    for (l += P2, r += P2; l < r; l >>= 1, r >>= 1) {
        if (l & 1u) atomicMax(&t[l++], v);
        if (r & 1u) atomicMax(&t[--r], v);
    }
}

__device__ __forceinline__ unsigned long long tree_query(const unsigned long long* t, uint32_t P2, uint32_t leaf) {
    unsigned long long v = 0;
    for (uint32_t x = leaf + P2; x; x >>= 1) v = max(v, t[x]);
    return v;
}

__global__ void __launch_bounds__(kLargeThreads, 1) patch_large_kernel(const LargePatchParams P) {
    __shared__ uint32_t sh[64];
    __shared__ uint32_t s_mc, s_take;
    // the current chunk: its ins/del records (position | kind << 30: 0 insert, 1 first delete, 2 other delete) and mark ops
    __shared__ uint32_t CRec[kLargeChunk];
    __shared__ uint32_t CPs[kLargeChunk], CPe[kLargeChunk], CKey[kLargeChunk], CInf[kLargeChunk];
    const uint32_t tid = threadIdx.x;
    char* slot = P.scratch + (size_t)blockIdx.x * P.slot_bytes;
    for (uint32_t ci = blockIdx.x; ci < P.n_cand; ci += gridDim.x) {
        const uint32_t li = P.cand[ci];
        const pt_log_desc L = P.desc[li];
        const pt_log_result RS = P.results[li];
        const uint32_t n = L.n_insdel, m = L.n_mark, R = L.n_actors ? L.n_actors : 1u, C = L.max_ctr, N = RS.n_elems;
        const unsigned long long KS = (unsigned long long)C * R;
        if (tid == 0) {
            const bool take = RS.status == 0 && !(P.after_warp && P.status[li] == 0) && ptp::large_patch_bytes(n, m, KS, N) <= P.slot_bytes;
            if (!(RS.status == 0 && P.after_warp && P.status[li] == 0)) P.status[li] = take ? 0u : 1u;
            s_take = take;
        }
        __syncthreads();
        const bool take = s_take;
        __syncthreads();                                   // every thread has read s_take before thread 0 writes the next one
        if (!take) continue;
        const pt_insdel_rec* __restrict__ ins = P.insdel + L.insdel_off;
        const pt_mark_rec* __restrict__ mk = P.marks + L.mark_off;
        const uint32_t* __restrict__ seq = P.seq + P.text_off[li];
        pt_patch_rec* out = P.recs + L.insdel_off;
        // ---- tables: the layout of ptp::large_patch_bytes ---------------------------------------------------------------
        const ptp::LargeLayout G = ptp::large_layout(n, m, KS, N);
        uint32_t* T = (uint32_t*)(slot + G.T);
        uint32_t* PosOf = (uint32_t*)(slot + G.PosOf);     // record -> sequence position of the element it inserts / deletes
        uint32_t* TIns = (uint32_t*)(slot + G.TIns);       // position -> the insert record
        uint32_t* TDel = (uint32_t*)(slot + G.TDel);       // position -> the FIRST delete record (kLargeNone: never)
        uint32_t* Ps = (uint32_t*)(slot + G.Ps);
        uint32_t* Pe = (uint32_t*)(slot + G.Pe);
        uint32_t* PeRaw = (uint32_t*)(slot + G.PeRaw);
        uint32_t* MKey = (uint32_t*)(slot + G.MKey);       // opId key
        uint32_t* MInf = (uint32_t*)(slot + G.MInf);       // type | remove << 2
        uint32_t* MAttr = (uint32_t*)(slot + G.MAttr);
        uint32_t* MArr = (uint32_t*)(slot + G.MArr);
        uint32_t* CIdx = (uint32_t*)(slot + G.CIdx);       // comment op -> its place in CSort
        uint32_t* Pres = (uint32_t*)(slot + G.Pres);
        uint32_t* Vis = (uint32_t*)(slot + G.Vis);
        uint32_t* PresPre = (uint32_t*)(slot + G.PresPre);
        uint32_t* VisPre = (uint32_t*)(slot + G.VisPre);
        uint32_t* SBits = (uint32_t*)(slot + G.SBits);     // boundary slots
        uint32_t* SPre = (uint32_t*)(slot + G.SPre);
        uint32_t* Bnd = (uint32_t*)(slot + G.Bnd);         // rank -> boundary slot
        uint32_t* FirstDef = (uint32_t*)(slot + G.FirstDef);
        unsigned long long* Tree = (unsigned long long*)(slot + G.Tree);     // 4 trees (one per mark type) of 2 * P2 nodes
        unsigned long long* CSort = (unsigned long long*)(slot + G.CSort);  // comment ops: id << 32 | op, sorted
        const uint32_t NW = G.NW, SW = G.SW, P2 = G.P2, P2c = G.P2c;
        auto keyOf = [&](uint32_t ctr, uint32_t actor) -> uint32_t { return (ctr - 1u) * R + actor; };
        auto badId = [&](uint32_t ctr, uint32_t actor) -> bool { return ctr - 1u >= C || actor >= R; };

        for (uint64_t k = tid; k < KS; k += kLargeThreads) T[k] = kLargeNone;
        for (uint32_t p = tid; p < N; p += kLargeThreads) TDel[p] = kLargeNone;
        for (uint32_t w = tid; w < SW; w += kLargeThreads) SBits[w] = 0u;
        for (uint32_t x = tid; x < 8u * P2; x += kLargeThreads) Tree[x] = 0ull;
        for (uint32_t x = tid; x < P2c; x += kLargeThreads) CSort[x] = ~0ull;
        for (uint32_t x = tid; x < 2u * m + 2u; x += kLargeThreads) FirstDef[x] = kLargeNone;
        if (tid == 0) s_mc = 0;
        __syncthreads();
        for (uint32_t i = tid; i < n; i += kLargeThreads) {
            const uint4 r = ld_rec(ins + i);
            if ((r.w >> 30) == PT_KIND_INSERT) T[keyOf(r.x, r.z & 0xFFFFu)] = i;
        }
        for (uint32_t p = tid; p < N; p += kLargeThreads) { const uint32_t rec = seq[p] & 0x3FFFFFFFu; PosOf[rec] = p; TIns[p] = rec; }
        __syncthreads();
        for (uint32_t i = tid; i < n; i += kLargeThreads) {
            const uint4 r = ld_rec(ins + i);
            if ((r.w >> 30) == PT_KIND_DELETE) {
                const uint32_t p = PosOf[T[keyOf(r.y, r.z >> 16)]];        // the merge succeeded: the target exists and arrived earlier
                PosOf[i] = p;
                atomicMin(&TDel[p], i);
            }
        }
        // mark ops -> slots, with the reference's rule that a boundary element must have arrived before the op
        // (src/peritext.ts:236-241); every finite slot is a boundary; comment ops go to CSort
        for (uint32_t k = tid; k < m; k += kLargeThreads) {
            const uint4* q = reinterpret_cast<const uint4*>(mk + k);
            const uint4 a0 = __ldg(q), a1 = __ldg(q + 1);
            const uint32_t kind = (a0.y >> 16) & 0xFFu, bounds = a0.y >> 24, arrival = a1.z;
            const uint32_t sb = bounds & 3u, eb = (bounds >> 2) & 3u, type = (kind >> 1) & 3u;
            uint32_t ps = kInfSlot, pr = kInfSlot;
            if (sb <= PT_BOUND_AFTER && !badId(a0.z, a1.x & 0xFFFFu)) { const uint32_t j = T[keyOf(a0.z, a1.x & 0xFFFFu)]; if (j != kLargeNone && j < arrival) ps = 2u * PosOf[j] + sb; }
            if (eb <= PT_BOUND_AFTER && !badId(a0.w, a1.x >> 16)) { const uint32_t j = T[keyOf(a0.w, a1.x >> 16)]; if (j != kLargeNone && j < arrival) pr = 2u * PosOf[j] + eb; }
            Ps[k] = ps; PeRaw[k] = pr; Pe[k] = pr == ps ? kInfSlot : pr;
            MKey[k] = keyOf(a0.x, a0.y & 0xFFFFu); MInf[k] = type | ((kind & 1u) << 2); MAttr[k] = a1.y; MArr[k] = arrival;
            if (ps != kInfSlot) atomicOr(&SBits[ps >> 5], 1u << (ps & 31u));
            if (pr != kInfSlot) atomicOr(&SBits[pr >> 5], 1u << (pr & 31u));
            if (type == PT_MARK_COMMENT) CSort[atomicAdd(&s_mc, 1u)] = ((unsigned long long)a1.y << 32) | k;
        }
        __syncthreads();
        prefix_words(SBits, SPre, nullptr, nullptr, SW, sh);
        __syncthreads();
        // comment ops by (id, op): a bitonic sort over P2c entries (the padding sorts last)
        const uint32_t mc = s_mc;
        const uint32_t len = mc > 1 ? 1u << (32 - __clz(mc - 1u)) : 1u;
        for (uint32_t kk = 2; kk <= len; kk <<= 1) {
            for (uint32_t jj = kk >> 1; jj; jj >>= 1) {
                for (uint32_t x = tid; x < len; x += kLargeThreads) {
                    const uint32_t y = x ^ jj;
                    if (y > x) {
                        const unsigned long long a = CSort[x], b = CSort[y];
                        if ((a > b) == ((x & kk) == 0)) { CSort[x] = b; CSort[y] = a; }
                    }
                }
                __syncthreads();
            }
        }
        __syncthreads();
        for (uint32_t x = tid; x < mc; x += kLargeThreads) CIdx[(uint32_t)CSort[x]] = x;
        // boundaries by rank, and the first mark op whose walk defines each of them (patch_kernel.cuh:198-201)
        const uint32_t D = SPre[SW];
        for (uint32_t w = tid; w < SW; w += kLargeThreads) {
            uint32_t bits = SBits[w], r = SPre[w];
            while (bits) { Bnd[r++] = w * 32u + (uint32_t)(__ffs(bits) - 1); bits &= bits - 1u; }
        }
        auto srank = [&](uint32_t s) -> uint32_t { return rank_below(SBits, SPre, s); };
        for (uint32_t y = tid; y < m; y += kLargeThreads) {
            const uint32_t ys = Ps[y], ye = Pe[y], yr = PeRaw[y];
            if (ys != kInfSlot && ys <= ye) atomicMin(&FirstDef[srank(ys)], y);
            if (yr != kInfSlot && yr != ys) atomicMin(&FirstDef[srank(yr)], y);
        }
        // ---- the window: records [0, j0) and mark ops [0, k0) lie before first_op -----------------------------------------
        const uint32_t total = n + m, w0 = min(P.first_op[li], total);
        auto marks_below = [&](uint32_t pos) -> uint32_t {        // #{k : min(arrival_k, n) + k < pos}: increasing in k
            uint32_t lo = 0, hi = m;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (min(MArr[mid], n) + mid < pos) lo = mid + 1; else hi = mid; }
            return lo;
        };
        __syncthreads();
        const uint32_t k0 = marks_below(w0), j0 = w0 - k0;
        for (uint32_t i = tid; i < j0; i += kLargeThreads) { pt_patch_rec z; z.index = 0; z.flags = 0; z.link_attr = PT_ATTR_NONE; z.reserved = 0; out[i] = z; }
        // the state as of first_op
        for (uint32_t w = tid; w < NW; w += kLargeThreads) {
            uint32_t pres = 0, vis = 0;
            for (uint32_t b = 0; b < 32u && w * 32u + b < N; b++) {
                const uint32_t p = w * 32u + b;
                if (TIns[p] < j0) { pres |= 1u << b; if (!(TDel[p] < j0)) vis |= 1u << b; }
            }
            Pres[w] = pres; Vis[w] = vis;
        }
        auto tree_add = [&](uint32_t k) {
            const uint32_t ps = Ps[k], pe = Pe[k];
            if (ps == kInfSlot || ps >= pe) return;
            const uint32_t l = srank(ps), r = pe == kInfSlot ? D : srank(pe);
            tree_update(Tree + (size_t)(MInf[k] & 3u) * 2u * P2, P2, l, r, ((unsigned long long)MKey[k] << 32 | k) + 1ull);
        };
        for (uint32_t k = tid; k < k0; k += kLargeThreads) tree_add(k);
        __syncthreads();
        prefix_words(Pres, PresPre, Vis, VisPre, NW, sh);
        __syncthreads();

        // ---- the sweep: list ops [c0, c1), one per thread ---------------------------------------------------------------
        uint32_t k_lo = k0;
        for (uint32_t c0 = w0; c0 < total; c0 += kLargeChunk) {
            const uint32_t c1 = min(total, c0 + kLargeChunk), k_hi = marks_below(c1), j_lo = c0 - k_lo, j_hi = c1 - k_hi;
            const uint32_t nrec = j_hi - j_lo, nmk = k_hi - k_lo;
            if (tid < nrec) {
                const uint32_t j = j_lo + tid, p = PosOf[j];
                const bool isIns = (__ldg(&ins[j].payload) >> 30) == PT_KIND_INSERT;
                CRec[tid] = p | (isIns ? 0u : TDel[p] == j ? 1u << 30 : 2u << 30);
            }
            if (tid < nmk) {
                const uint32_t k = k_lo + tid;
                CPs[tid] = Ps[k]; CPe[tid] = Pe[k]; CKey[tid] = MKey[k]; CInf[tid] = MInf[k];
            }
            __syncthreads();
            // visible elements below position q at the time the first `upto` records of the chunk have arrived
            auto vis_below = [&](uint32_t q, uint32_t upto) -> uint32_t {
                int v = (int)rank_below(Vis, VisPre, q);
                for (uint32_t u = 0; u < upto; u++) {
                    const uint32_t cr = CRec[u], kd = cr >> 30;
                    if ((cr & 0x3FFFFFFFu) < q) v += kd == 0 ? 1 : kd == 1 ? -1 : 0;
                }
                return (uint32_t)v;
            };
            // LWW winner of `type` among the ops before the chunk and the chunk's first `upto` mark ops covering slot s
            auto lww = [&](uint32_t type, uint32_t s, uint32_t upto, uint32_t leaf1) -> unsigned long long {
                unsigned long long w = leaf1 ? tree_query(Tree + (size_t)type * 2u * P2, P2, leaf1 - 1u) : 0ull;
                for (uint32_t u = 0; u < upto; u++)
                    if ((CInf[u] & 3u) == type && CPs[u] <= s && s < CPe[u]) w = max(w, ((unsigned long long)CKey[u] << 32 | (k_lo + u)) + 1ull);
                return w;
            };
            if (tid < nrec) {
                // ---- an insert / delete record ------------------------------------------------------------------------
                const uint32_t i = j_lo + tid, p = CRec[tid] & 0x3FFFFFFFu, kd = CRec[tid] >> 30;
                const uint32_t cnt = vis_below(p, tid);
                uint32_t flags = 0, link = PT_ATTR_NONE, ncom = 0;
                if (kd == 0) {
                    // the nearest element left of p present at time i: the present bitmap, or an earlier insert of the chunk
                    const uint32_t r = rank_below(Pres, PresPre, p);
                    int py = r ? (int)select_bit(Pres, PresPre, NW, r - 1u) : -1;
                    for (uint32_t u = 0; u < tid; u++) { const uint32_t cr = CRec[u], q = cr & 0x3FFFFFFFu; if ((cr >> 30) == 0 && q < p) py = max(py, (int)q); }
                    if (py >= 0) {
                        const uint32_t s = 2u * (uint32_t)py + 1u, leaf1 = srank(s + 1u);
                        uint32_t upto = 0;                          // the chunk's mark ops that arrived before record i
                        while (upto < nmk && MArr[k_lo + upto] <= i) upto++;
                        const unsigned long long w0s = lww(PT_MARK_STRONG, s, upto, leaf1), w1 = lww(PT_MARK_EM, s, upto, leaf1), w2 = lww(PT_MARK_LINK, s, upto, leaf1);
                        if (w0s && !((MInf[(uint32_t)(w0s - 1ull)] >> 2) & 1u)) flags |= PT_SPAN_STRONG;
                        if (w1 && !((MInf[(uint32_t)(w1 - 1ull)] >> 2) & 1u)) flags |= PT_SPAN_EM;
                        if (w2) { const uint32_t k2 = (uint32_t)(w2 - 1ull); if (!((MInf[k2] >> 2) & 1u)) { flags |= PT_SPAN_LINK; link = MAttr[k2]; } }
                        if (lww(PT_MARK_COMMENT, s, upto, leaf1)) {
                            flags |= PT_SPAN_COMMENT;
                            // comment ids: per id, the last covering op that arrived before record i decides
                            uint32_t x = mc;
                            while (x > 0) {
                                const uint32_t id = (uint32_t)(CSort[x - 1] >> 32);
                                bool decided = false;
                                while (x > 0 && (uint32_t)(CSort[x - 1] >> 32) == id) {
                                    const uint32_t k = (uint32_t)CSort[--x];
                                    if (!decided && MArr[k] <= i && Ps[k] <= s && s < Pe[k]) {
                                        decided = true;
                                        if (!((MInf[k] >> 2) & 1u)) { large_emit(P, li, i, id, 0); ncom++; }
                                    }
                                }
                            }
                        }
                    }
                }
                pt_patch_rec pr;
                const bool emits = kd != 2;                    // a delete emits a patch only if it is the element's first
                pr.index = cnt | (emits ? 0x80000000u : 0u); pr.flags = flags | (ncom << 8); pr.link_attr = link; pr.reserved = 0;
                out[i] = pr;
            } else if (tid < nrec + nmk) {
                // ---- a mark op X: intervals between consecutive slots defined at its arrival time ------------------------
                const uint32_t u = tid - nrec, X = k_lo + u, ps = CPs[u], pe = CPe[u];
                if (ps != kInfSlot && ps < pe) {
                    const uint32_t upto = min(MArr[X], j_hi) - min(MArr[X], j_lo), typeX = CInf[u] & 3u, keyX = CKey[u], attrX = MAttr[X];
                    const bool addX = !((CInf[u] >> 2) & 1u);
                    auto vis_at = [&](uint32_t s) -> uint32_t { return vis_below((s + 1u) >> 1, upto); };   // #{visible q : 2q + 1 <= s}
                    const uint32_t length = vis_below(N, upto);
                    const uint32_t rend = pe == kInfSlot ? D : srank(pe);
                    uint32_t cur = ps, rc = srank(ps), start_i = vis_at(ps);
                    for (;;) {
                        uint32_t nxt = pe;
                        for (uint32_t r = rc + 1; r < rend; r++) if (FirstDef[r] < X) { rc = r; nxt = Bnd[r]; break; }
                        bool changed;
                        const uint32_t leaf1 = srank(cur + 1u);
                        if (typeX != PT_MARK_COMMENT) {
                            const unsigned long long w = lww(typeX, cur, u, leaf1);
                            if (w && (uint32_t)((w - 1ull) >> 32) > keyX) changed = false;     // an earlier op with a larger opId keeps winning
                            else {
                                const uint32_t Yw = (uint32_t)(w - 1ull);
                                const bool oldOn = w && !((MInf[Yw] >> 2) & 1u);
                                changed = oldOn != addX || (oldOn && addX && typeX == PT_MARK_LINK && MAttr[Yw] != attrX);
                            }
                        } else {
                            const bool any = lww(PT_MARK_COMMENT, cur, u, leaf1) != 0ull;
                            bool has = false;
                            for (uint32_t x = CIdx[X]; x > 0 && (uint32_t)(CSort[x - 1] >> 32) == attrX; x--) {
                                const uint32_t Y = (uint32_t)CSort[x - 1];
                                if (Ps[Y] <= cur && cur < Pe[Y]) { has = !((MInf[Y] >> 2) & 1u); break; }   // arrival order: the last one decides
                            }
                            changed = addX ? !has : (!any || has);      // a remove on a range without the `comment` key creates `comment: []`
                        }
                        const uint32_t end_i = nxt == kInfSlot ? length : vis_at(nxt);
                        if (changed && end_i > start_i && start_i < length) large_emit(P, li, X | 0x80000000u, start_i, end_i);
                        if (nxt == pe) break;
                        cur = nxt; start_i = end_i;
                    }
                }
            }
            __syncthreads();
            // ---- advance the state past the chunk ---------------------------------------------------------------------------
            if (tid < nrec) {
                const uint32_t cr = CRec[tid], p = cr & 0x3FFFFFFFu, kd = cr >> 30;
                // an element inserted and first deleted inside the chunk never turns visible: no order between the two atomics
                if (kd == 0) { atomicOr(&Pres[p >> 5], 1u << (p & 31u)); if (!(TDel[p] < j_hi)) atomicOr(&Vis[p >> 5], 1u << (p & 31u)); }
                else if (kd == 1 && TIns[p] < j_lo) atomicAnd(&Vis[p >> 5], ~(1u << (p & 31u)));
            }
            if (tid < nmk) tree_add(k_lo + tid);
            __syncthreads();
            prefix_words(Pres, PresPre, Vis, VisPre, NW, sh);
            __syncthreads();
            k_lo = k_hi;
        }
    }
}

}  // namespace ptk
