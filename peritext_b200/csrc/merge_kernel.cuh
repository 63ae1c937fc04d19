// merge_kernel.cuh — the op-log apply + flatten kernel (sm_90a).
//
// One CTA materialises one LOG (one replica's op log of one document) end to end:
//   packed records in HBM  ->  element sequence (RGA order)  ->  visible text + formatted spans + digest in HBM.
// It computes the ORDER-INDEPENDENT CLOSED FORM of what the reference does sequentially in
//   Micromerge.applyOp / applyListInsert / applyListUpdate     (reference src/micromerge.ts:534-724)
//   applyAddRemoveMark                                          (reference src/peritext.ts:154-249)
//   getTextWithFormatting / opsToMarks / addCharactersToSpans   (reference src/peritext.ts:294-455)
// (SURVEY.md §9.2; proven equal to the sequential oracle by tests/test_closed_form.py on the CPU model
//  tests/kernel_model.py, whose phase names A..I this file follows).
//
// No floating point, no tensor cores: integer/index work bounded by HBM traffic and shared-memory latency.
// Layout of the per-record state: BITMAPS over record indices (insert / chain-continuation / head / visible) with
// popcount prefixes per 32-record word, instead of per-record index arrays; everything per-element is derived as
//   run(i)  = popcount(head bits <= i) - 1
//   pos(i)  = PosBase[run(i)] + i                 (runs are contiguous in the log AND in the sequence)
//   vis(i)  = VisBase[run(i)] + popcount(visible bits < i)
// Working arrays live in a per-CTA stack-like ARENA.  The pipeline is instantiated twice: SH=true keeps every array in
// dynamic shared memory (LDS/STS with 32-bit addresses); a log that does not fit is deferred to a launch with a larger
// budget, and only the largest one falls back to SH=false, which spills to a per-CTA global slab (L2 resident).
// Index arrays are u16 when the log is small enough (halves the footprint).  The record stream of phase A is staged
// through shared memory with TMA bulk copies (cp.async.bulk + mbarrier), double buffered.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/peritext_b200.h"
#include "../../include/pt_digest.h"

namespace ptk {

struct BatchParams {
    const pt_log_desc* __restrict__ desc;
    const pt_insdel_rec* __restrict__ insdel;
    const pt_mark_rec* __restrict__ marks;
    const uint32_t* __restrict__ key_insdel;   // the warp kernel's key-record copy of insdel / marks (upload_kernel.cuh); null
    const uint2* __restrict__ key_marks;       // when no log is on a warp route
    const uint32_t* __restrict__ order;   // log indices of this launch (bin), largest first
    uint32_t n_work;
    uint32_t* work_counter;               // persistent-CTA work queue head
    pt_log_result* results;
    const uint64_t* __restrict__ text_off;
    const uint64_t* __restrict__ span_off;
    uint32_t* text;
    pt_span* spans;
    uint32_t* comment_pool;
    unsigned long long* comment_used;
    unsigned long long comment_cap;
    char* slab;                           // spill: slab_bytes per SPILLING CTA (a CTA takes a slot the first time it spills)
    unsigned long long slab_bytes;
    uint32_t* slab_counter;               // next free slab slot
    uint32_t slab_slots;                  // slots allocated: min(logs that can spill, grid)
    uint32_t smem_arena_bytes;            // dynamic shared memory given to the arena
    unsigned long long* stats;            // [0] logs finished on the shared-only path, [1] on the spill path, [2] deferred
    uint32_t* retry_list;                 // non-null: logs that do not fit this bin's shared memory are deferred here
    uint32_t* retry_count;
    const uint32_t* n_work_dev;           // non-null: number of work items is read from device memory (retry launch)
    uint32_t prefetch_next;               // CTA-per-log kernel: prefetch the next log's records into L2 while working on the current one
    uint32_t warp_flags;                  // warp-per-log kernel (PT_WARP_FLAGS, default 0x704): bit0 prefetch this log's marks, bit1 the next round's
                                          // records, bit2 round-aligned warps, bits 8-11 skip in-log phase barrier 2 / 3 / 4 / 5
    uint32_t use_tma;                     // stage the record stream through shared memory with cp.async.bulk (shared-only path)
    uint32_t* seq;                        // optional: element sequence output (record index | after-slot defined << 30 | deleted << 31), text offsets
    const uint32_t* admit;                // optional: per-log admission status (pre-pass); non-zero: the log is not merged
};

// ---------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_rec(const pt_insdel_rec* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- TMA (cp.async.bulk, 1-D) + mbarrier helpers: global -> shared staging of the record stream ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int BLOCK>
struct BlockCtx {
    unsigned long long tma_bar[2];      // mbarriers of the two staging buffers (initialised once per CTA)
    uint32_t warp_a[32], warp_b[32];
    uint32_t tot_a, tot_b;
    uint32_t status;
    uint32_t work, work_next;
    uint32_t misc[4];
    uint32_t dup_cnt;                   // occupied id-table entries (must equal the number of inserts)
    uint32_t slab_slot;                 // this CTA's slot of the global spill slab (0xFFFFFFFF: none taken yet)
    unsigned long long dig0, dig1;
    unsigned long long pool_base;
};

// exclusive block scan of a PAIR of values per thread (two independent sums in one pass)
template <int BLOCK>
__device__ __forceinline__ void block_scan2(uint32_t va, uint32_t vb, BlockCtx<BLOCK>& c, uint32_t& ea, uint32_t& eb,
                                            uint32_t& ta, uint32_t& tb) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t xa = va, xb = vb;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t ya = __shfl_up_sync(0xffffffffu, xa, o), yb = __shfl_up_sync(0xffffffffu, xb, o);
        if (lane >= (uint32_t)o) { xa += ya; xb += yb; }
    }
    if (lane == 31) { c.warp_a[warp] = xa; c.warp_b[warp] = xb; }
    __syncthreads();
    if (warp == 0) {
        uint32_t wa = lane < (BLOCK / 32) ? c.warp_a[lane] : 0, wb = lane < (BLOCK / 32) ? c.warp_b[lane] : 0;
        uint32_t sa = wa, sb = wb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t ya = __shfl_up_sync(0xffffffffu, sa, o), yb = __shfl_up_sync(0xffffffffu, sb, o);
            if (lane >= (uint32_t)o) { sa += ya; sb += yb; }
        }
        if (lane < (BLOCK / 32)) { c.warp_a[lane] = sa - wa; c.warp_b[lane] = sb - wb; }
        if (lane == 31) { c.tot_a = sa; c.tot_b = sb; }
    }
    __syncthreads();
    ea = c.warp_a[warp] + xa - va; eb = c.warp_b[warp] + xb - vb;
    ta = c.tot_a; tb = c.tot_b;
    __syncthreads();
}
template <int BLOCK>
__device__ __forceinline__ uint32_t block_scan_excl(uint32_t v, BlockCtx<BLOCK>& c, uint32_t& total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
    if (BLOCK == 32) { total = __shfl_sync(0xffffffffu, x, 31); return x - v; }
    if (lane == 31) c.warp_a[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < (BLOCK / 32) ? c.warp_a[lane] : 0, s2 = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, s2, o); if (lane >= (uint32_t)o) s2 += y; }
        if (lane < (BLOCK / 32)) c.warp_a[lane] = s2 - w;
        if (lane == 31) c.tot_a = s2;
    }
    __syncthreads();
    const uint32_t res = c.warp_a[warp] + x - v;
    total = c.tot_a;
    __syncthreads();
    return res;
}

extern __shared__ __align__(16) char ptk_smem[];   // dynamic shared memory = the arena's fast region

// SH = true : every array must fit in dynamic shared memory; pointers are derived from the __shared__ symbol so the
//             compiler emits LDS/STS with 32-bit addresses.  An allocation that does not fit sets `overflow` and the
//             caller restarts the log in the SH = false instantiation.
// SH = false: shared memory first, then the per-CTA global slab (generic pointers).
template <bool SH>
struct Arena {
    uint32_t sm_cap, sm_used;
    char* gm; unsigned long long gm_cap, gm_used;
    bool overflow;
    // bytes in 64 bits: the id table of a key space near 2^31 is 4-8 GiB, and a 32-bit count would wrap to a size that fits
    template <class T> __device__ __forceinline__ T* alloc(uint32_t count) {
        const unsigned long long bytes = ((unsigned long long)count * sizeof(T) + 15ull) & ~15ull;
        if (SH) {
            if (sm_used + bytes > sm_cap) { overflow = true; return reinterpret_cast<T*>(ptk_smem); }
            const uint32_t off = sm_used; sm_used += (uint32_t)bytes;
            return reinterpret_cast<T*>(ptk_smem + off);
        }
        if (sm_used + bytes <= sm_cap) { T* p = reinterpret_cast<T*>(ptk_smem + sm_used); sm_used += (uint32_t)bytes; return p; }
        if (gm_used + bytes > gm_cap) { overflow = true; return reinterpret_cast<T*>(gm); }
        T* p = reinterpret_cast<T*>(gm + gm_used); gm_used += bytes; return p;
    }
};
#define PT_ALLOC(var, T, count) T* var = A.template alloc<T>(count); if (SH && A.overflow) return 1

// fill `count` elements (allocation is padded to 16 B, so whole uint4 stores are safe)
template <class T, int BLOCK>
__device__ __forceinline__ void fill(T* p, uint32_t count, T v) {
    uint32_t nvec = (uint32_t)((count * sizeof(T) + 15u) >> 4);
    uint32_t w;
    if (sizeof(T) == 1) w = 0x01010101u * (uint32_t)(uint8_t)v;
    else if (sizeof(T) == 2) w = 0x00010001u * (uint32_t)(uint16_t)v;
    else w = (uint32_t)v;
    uint4 q = make_uint4(w, w, w, w);
    uint4* d = reinterpret_cast<uint4*>(p);
    for (uint32_t i = threadIdx.x; i < nvec; i += BLOCK) d[i] = q;
}

// 32 byte-flags (0/1) -> one 32-bit word
__device__ __forceinline__ uint32_t pack32(const uint8_t* b) {
    const uint4* q = reinterpret_cast<const uint4*>(b);
    uint4 x = q[0], y = q[1];
    auto nib = [](uint32_t v) -> uint32_t { return ((v * 0x00204081u) >> 21) & 0xFu; };
    return nib(x.x) | (nib(x.y) << 4) | (nib(x.z) << 8) | (nib(x.w) << 12) | (nib(y.x) << 16) | (nib(y.y) << 20) | (nib(y.z) << 24) | (nib(y.w) << 28);
}

__device__ __forceinline__ void digest_add(unsigned long long& d0, unsigned long long& d1, uint64_t t) { d0 += t; d1 ^= pt_term_hi(t); }
template <int BLOCK>
__device__ __forceinline__ void digest_flush(BlockCtx<BLOCK>& c, unsigned long long d0, unsigned long long d1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 ^= __shfl_xor_sync(0xffffffffu, d1, o); }
    if ((threadIdx.x & 31) == 0 && (d0 | d1)) { atomicAdd(&c.dig0, d0); atomicXor(&c.dig1, d1); }
}

// Comment-pool reservation: ONE fire-and-forget style atomicAdd on the batch-wide cursor (a CAS loop on a hot global word
// serialises the whole GPU at one success per round trip — measured: 6x slower c4 merges).  The cursor keeps counting past
// the capacity, so after the merge it holds the batch's exact DEMAND: logs that found the pool full report PT_LOG_OVERFLOW,
// the host sees demand > capacity (pt_spans_view.comment_pool_needed), resizes once and re-merges — then every log fits.
template <class Params>
__device__ __forceinline__ unsigned long long pool_reserve(const Params& P, uint32_t count, uint32_t& status) {
    const unsigned long long base = atomicAdd(P.comment_used, (unsigned long long)count);
    if (base + count > P.comment_cap) { status = PT_LOG_OVERFLOW; return 0; }
    return base;
}

// Euler-tour node: next (20 bits) | element weight (22 bits) | visible weight (22 bits)
constexpr uint32_t kNodeNxtBits = 20;
constexpr unsigned long long kNodeNxtMask = (1ull << kNodeNxtBits) - 1;
__device__ __forceinline__ unsigned long long node_make(uint32_t nxt, uint32_t wel, uint32_t wvis) {
    return (unsigned long long)nxt | ((unsigned long long)wel << 20) | ((unsigned long long)wvis << 42);
}

// =========================================================================================================
// The per-log pipeline.  Idx = uint16_t (logs with < 32000 records) or uint32_t.
// =========================================================================================================
template <class Idx, int BLOCK, bool SH>
__device__ int merge_one_log(const BatchParams& P, uint32_t li, BlockCtx<BLOCK>& c, uint32_t& tma_parity) {
    constexpr Idx NONE = (Idx)~(Idx)0;
    const uint32_t tid = threadIdx.x, lane = tid & 31;

    const pt_log_desc L = P.desc[li];
    const uint32_t n = L.n_insdel, m = L.n_mark, R = L.n_actors ? L.n_actors : 1, C = L.max_ctr;
    const uint32_t KS = C * R;
    const pt_insdel_rec* __restrict__ ins = P.insdel + L.insdel_off;
    const pt_mark_rec* __restrict__ mk = P.marks + L.mark_off;
    uint32_t* text_out = P.text + P.text_off[li];
    uint32_t* seq_out = P.seq ? P.seq + P.text_off[li] : nullptr;
    pt_span* span_out = P.spans + P.span_off[li];
    pt_log_result* res = P.results + li;

    Arena<SH> A;
    A.sm_cap = P.smem_arena_bytes; A.sm_used = 0;
    A.gm = P.slab; A.gm_cap = 0; A.gm_used = 0; A.overflow = false;
    if (!SH) {
        // the global slab has one slot per CTA that ever spills (only logs whose worst case exceeds the shared-memory budget can)
        if (tid == 0 && c.slab_slot == 0xFFFFFFFFu) c.slab_slot = atomicAdd(P.slab_counter, 1u);
        __syncthreads();
        if (c.slab_slot < P.slab_slots) { A.gm = P.slab + (unsigned long long)c.slab_slot * P.slab_bytes; A.gm_cap = P.slab_bytes; }
    }

    if (tid == 0) { c.status = 0; c.misc[0] = 0; c.misc[2] = 0; c.misc[3] = 0; c.dup_cnt = 0; c.dig0 = 0; c.dig1 = 0; c.pool_base = 0; }

    auto keyOf = [&](uint32_t ctr, uint32_t actor) -> uint32_t { return (ctr - 1u) * R + actor; };
    auto badId = [&](uint32_t ctr, uint32_t actor) -> bool { return ctr - 1u >= C || actor >= R; };
    auto fail = [&](uint32_t code) { atomicMax(&c.status, code); };
    auto bail = [&]() { if (tid == 0) { pt_log_result r{}; r.status = c.status; *res = r; } __syncthreads(); };

    const uint32_t NWr = (n + 31) / 32 + 1;     // words over record indices (+1 zero pad word)

    // ---- arrays that live to the end (allocation order = smem priority) --------------------------------------
    PT_ALLOC(T, Idx, KS);                    // A: opId key -> insert record index
    PT_ALLOC(InsBits, uint32_t, NWr);   // record is an insert
    PT_ALLOC(HeadBits, uint32_t, NWr);  // record starts a run (first: chain-continuation bits)
    PT_ALLOC(VisBits, uint32_t, NWr);   // record is a visible element
    PT_ALLOC(HeadPre, Idx, NWr);             // heads in words < w
    PT_ALLOC(VisPre, Idx, NWr);              // visible elements in words < w
    // byte flags, dead after phase C (released)
    const uint32_t mark_sm = A.sm_used; const unsigned long long mark_gm = A.gm_used;
    PT_ALLOC(Other, uint8_t, NWr * 32 + 32);   // element has a child that is not its log successor
    PT_ALLOC(Del, uint8_t, NWr * 32 + 32);     // tombstone

    fill<Idx, BLOCK>(T, KS, NONE);
    fill<uint8_t, BLOCK>(Other, NWr * 32 + 32, (uint8_t)0);
    fill<uint8_t, BLOCK>(Del, NWr * 32 + 32, (uint8_t)0);
    if (tid == 0) { InsBits[NWr - 1] = 0; HeadBits[NWr - 1] = 0; }
    __syncthreads();

    if (m) {   // number of comment mark ops (sizes the comment tables); issued first so the marks' HBM latency overlaps phase A
        uint32_t ccnt = 0;
        for (uint32_t k = tid; k < m; k += BLOCK) ccnt += (((uint32_t)mk[k].kind >> 1) & 3u) == PT_MARK_COMMENT ? 1u : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ccnt += __shfl_xor_sync(0xffffffffu, ccnt, o);
        if (lane == 0 && ccnt) atomicAdd(&c.misc[2], ccnt);
    }

    // ---- A+B, fused per chunk of records (the only pass over the records before the text pass) ---------------------------
    // A: id table T[K(opId)] and the insert / chain-link bitmaps.  cand(i): record i is an insert whose reference element
    //    is the insert at record i-1 (a typing chain link) — decided by comparing with the left neighbour, no lookup.
    // B: after the chunk's ids are in the table: parents of chain heads (-> "has another child" flags) and deletes
    //    (-> tombstones), one code path for both.  A referenced element must arrive EARLIER in the log, as in the
    //    reference, where applyOp throws "List element not found" otherwise (src/micromerge.ts:752).
    {
        const uint4 zero4 = make_uint4(0, 0, 0, 0xC0000000u);     // kind 3: neither insert nor delete
        auto stepA = [&](uint32_t i, const uint4 r, const uint4 rp) -> uint32_t {   // returns bit0: record needs a table lookup in B, bit1: it is a valid insert
            const uint32_t ctr = r.x, actor = r.z & 0xFFFFu, ref_ctr = r.y, ref_actor = r.z >> 16, kind = r.w >> 30;
            bool isIns = false, valid = false;
            if (i < n) {
                if (kind > 1u) fail(PT_LOG_BAD_KIND);
                else if (badId(ctr, actor)) fail(PT_LOG_BAD_OPID);
                else {
                    valid = true;
                    if (kind == PT_KIND_INSERT) {
                        isIns = true;
                        T[keyOf(ctr, actor)] = (Idx)i;
                    }
                }
            }
            // reference element == the insert at record i-1 ?
            bool cand = isIns && ref_ctr != 0 && ref_ctr == rp.x && ref_actor == (rp.z & 0xFFFFu) && (rp.w >> 30) == PT_KIND_INSERT;
            if (cand && keyOf(ref_ctr, ref_actor) >= keyOf(ctr, actor)) { fail(PT_LOG_CYCLE); cand = false; }
            const uint32_t insW = __ballot_sync(0xffffffffu, isIns), candW = __ballot_sync(0xffffffffu, cand);
            if (lane == 0 && i < n) { InsBits[i >> 5] = insW; HeadBits[i >> 5] = candW; }
            return ((valid && !cand) ? 1u : 0u) | (isIns ? 2u : 0u);
        };
        auto stepB = [&](uint32_t i, bool live, const uint4 r) {
            if (!live) return;
            const uint32_t ctr = r.x, ref_ctr = r.y, actor = r.z & 0xFFFFu, ref_actor = r.z >> 16;
            const bool isIns = (r.w >> 30) == PT_KIND_INSERT;
            if (ref_ctr == 0) { if (!isIns) fail(PT_LOG_ELEM_NOT_FOUND); return; }        // insert: child of HEAD
            const Idx j = badId(ref_ctr, ref_actor) ? NONE : T[keyOf(ref_ctr, ref_actor)];
            if (j == NONE || (uint32_t)j >= i) { fail(PT_LOG_ELEM_NOT_FOUND); return; }   // must have arrived earlier (deterministic)
            if (isIns && keyOf(ref_ctr, ref_actor) >= keyOf(ctr, actor)) { fail(PT_LOG_CYCLE); return; }
            (isIns ? Other : Del)[j] = 1;        // deletes: OR, idempotent (micromerge.ts:689)
        };
        if (SH && P.use_tma) {
            // TMA-staged record stream: chunks of 2*BLOCK records land in a double-buffered shared-memory stage
            // (cp.async.bulk + mbarrier complete_tx); chunk k+2 is in flight while chunk k is decoded.
            constexpr uint32_t CH = 2 * BLOCK;
            const uint32_t stage_mark = A.sm_used;
            PT_ALLOC(Stage, uint4, 2 * CH);
            const uint32_t nch = (n + CH - 1) / CH;
            auto issue = [&](uint32_t k) {
                const uint32_t b = k & 1u, cnt = min(CH, n - k * CH);
                mbar_expect_tx(&c.tma_bar[b], cnt * 16u);
                tma_load_1d(Stage + b * CH, ins + (size_t)k * CH, cnt * 16u, &c.tma_bar[b]);
            };
            if (tid == 0) { fence_proxy_async(); if (nch > 0) issue(0); if (nch > 1) issue(1); }
            for (uint32_t k = 0; k < nch; k++) {
                const uint32_t b = k & 1u;
                mbar_wait(&c.tma_bar[b], (tma_parity >> b) & 1u);
                tma_parity ^= 1u << b;
                const uint4* st = Stage + b * CH;
                const uint32_t i0 = k * CH + tid, i1 = i0 + BLOCK;
                const uint4 r0 = i0 < n ? st[tid] : zero4, r1 = i1 < n ? st[BLOCK + tid] : zero4;
                uint4 p0 = zero4, p1 = zero4;
                if (i0 < n) { if (tid > 0) p0 = st[tid - 1]; else if (i0 > 0) p0 = ld_rec(ins + i0 - 1); }
                if (i1 < n) p1 = st[BLOCK + tid - 1];
                const uint32_t l0 = stepA(i0, r0, p0);
                const uint32_t l1 = stepA(i1, r1, p1);
                __syncthreads();                                   // the chunk's ids are in T; everyone is done with buffer b
                if (tid == 0 && k + 2 < nch) { fence_proxy_async(); issue(k + 2); }
                stepB(i0, l0 & 1u, r0);
                stepB(i1, l1 & 1u, r1);
            }
            A.sm_used = stage_mark;                                // release the stage
        } else
        for (uint32_t base = 0; base < n; base += 2 * BLOCK) {     // two records per thread per trip: 4 loads in flight
            const uint32_t i0 = base + tid, i1 = i0 + BLOCK;
            const uint4 r0 = i0 < n ? ld_rec(ins + i0) : zero4, r1 = i1 < n ? ld_rec(ins + i1) : zero4;
            // the left neighbours (same cache lines, L1 hits)
            const uint4 p0 = (i0 > 0 && i0 < n) ? ld_rec(ins + i0 - 1) : zero4, p1 = i1 < n ? ld_rec(ins + i1 - 1) : zero4;
            const uint32_t l0 = stepA(i0, r0, p0);
            const uint32_t l1 = stepA(i1, r1, p1);
            __syncthreads();                                       // the trip's ids are in T
            stepB(i0, l0 & 1u, r0);
            stepB(i1, l1 & 1u, r1);
        }
    }
    __syncthreads();
    if (c.status) { bail(); return 0; }
    {   // two inserts with one opId leave ONE table entry: the number of occupied entries must equal the number of inserts
        // (checked after phase C); a vectorised count over the table instead of a second look at every insert
        const uint32_t nvec = (uint32_t)((KS * sizeof(Idx) + 15u) >> 4);
        const uint4* tv = reinterpret_cast<const uint4*>(T);
        uint32_t occ = 0;
        for (uint32_t v = tid; v < nvec; v += BLOCK) {
            const uint4 q = tv[v];
            if (sizeof(Idx) == 2) {
                const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int k = 0; k < 4; k++) occ += ((w[k] & 0xFFFFu) != 0xFFFFu) + ((w[k] >> 16) != 0xFFFFu);
            } else occ += (q.x != 0xFFFFFFFFu) + (q.y != 0xFFFFFFFFu) + (q.z != 0xFFFFFFFFu) + (q.w != 0xFFFFFFFFu);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) occ += __shfl_xor_sync(0xffffffffu, occ, o);
        if (lane == 0 && occ) atomicAdd(&c.dup_cnt, occ);
    }

    // ---- C: runs, bit-parallel: head = insert & (!chain-link | predecessor has another child); visible = insert & !deleted
    uint32_t M, nvis;
    {
        uint32_t carryH = 0, carryV = 0;
        for (uint32_t base = 0; base < NWr; base += BLOCK) {
            const uint32_t w = base + tid;
            uint32_t head = 0, vis = 0;
            if (w < NWr) {
                const uint32_t insW = InsBits[w], candW = HeadBits[w];
                const uint32_t otherW = pack32(Other + 32 * w), delW = pack32(Del + 32 * w);
                const uint32_t otherPrev = (otherW << 1) | (w ? (uint32_t)Other[32 * w - 1] : 0u);
                head = insW & (~candW | otherPrev);
                vis = insW & ~delW;
            }
            uint32_t eh, ev, th, tv;
            block_scan2<BLOCK>(__popc(head), __popc(vis), c, eh, ev, th, tv);
            if (w < NWr) { HeadBits[w] = head; VisBits[w] = vis; HeadPre[w] = (Idx)(carryH + eh); VisPre[w] = (Idx)(carryV + ev); }
            carryH += th; carryV += tv;
        }
        M = carryH; nvis = carryV;
    }
    A.sm_used = mark_sm; A.gm_used = mark_gm;      // release Other / Del
    uint32_t N = 0;
    {
        uint32_t cnt = 0;
        for (uint32_t w = tid; w < NWr; w += BLOCK) cnt += __popc(InsBits[w]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0 && cnt) atomicAdd(&c.misc[0], cnt);
    }
    __syncthreads();
    N = c.misc[0];
    if (c.dup_cnt != N) { __syncthreads(); if (tid == 0) c.status = PT_LOG_BAD_OPID; __syncthreads(); bail(); return 0; }
    const uint32_t McBound = c.misc[2];
    if (2ull * M + 4 >= (1ull << kNodeNxtBits) || N >= (1u << 22)) { if (tid == 0) c.status = PT_LOG_OVERFLOW; __syncthreads(); bail(); return 0; }

    auto runOf = [&](uint32_t i) -> uint32_t {     // run id of element record i
        return (uint32_t)HeadPre[i >> 5] + __popc(HeadBits[i >> 5] & (0xFFFFFFFFu >> (31 - (i & 31)))) - 1u;
    };
    auto visBefore = [&](uint32_t i) -> uint32_t {  // visible element records with index < i   (i in 0..n)
        return (uint32_t)VisPre[i >> 5] + __popc(VisBits[i >> 5] & ((1u << (i & 31)) - 1u));
    };

    // ---- D: run tree; children of every node ordered by DESCENDING opId of the run head ---------------------------------
    const uint32_t E = 2 * (M + 1), END = E;
    if (SH) {   // will everything fit in shared memory?  (upper bound on the peak of the stack-like arena; avoids wasted attempts)
        auto al = [](unsigned long long b) -> unsigned long long { return (b + 15ull) & ~15ull; };
        const unsigned long long I = sizeof(Idx);
        const unsigned long long base = (unsigned long long)A.sm_used + 2 * al((M + 2) * 4ull);
        unsigned long long peak = base + al((E + 1) * 8ull) + 2 * al(((E + 7) / 8 + 3) * 8ull) + 5 * al((M + 1) * I) + al((M + 1) * 4ull) + al((M + 2) * I)
                                 + al((M / 33 + 2) * I) + al(((KS + 31) / 32 + 1) * 4ull) + al(((KS + 31) / 32 + 1) * I);
        if (m) {
            const unsigned long long NWp_ = (N + 32) / 32 + 1, KW_ = (KS + 31) / 32;
            const unsigned long long Sb = (2ull * m + 2 < (unsigned long long)N + 2 ? 2ull * m + 2 : (unsigned long long)N + 2) + 1;
            // spans: at most one per visible element and per mark boundary; typically far fewer — guess half, a log that needs
            // more fails its allocation in phase I and is deferred then (nothing irreversible has happened by that point)
            const unsigned long long Mcb = McBound, Hb = 4 * Mcb + 8, VWb = (nvis + 31) / 32, nsp = (nvis < 2ull * m + 1 ? nvis : 2ull * m + 1) / 2 + 16;
            const unsigned long long Pm = base + 6 * al((m + 1) * I) + al(m + 1) + 2 * al((m + 1) * 4ull) + al((NWp_ + 1) * 4) + al((NWp_ + 1) * I);
            const unsigned long long pG2 = Pm + al((KW_ + 1) * 4) + al((KW_ + 1) * I);
            const unsigned long long Q = Pm + 2 * al((Sb + 1) * 4);
            const unsigned long long pG3 = Q + al((2 * Sb + 2) * 4) + al((Sb + 2) * 4);
            const unsigned long long Rr = Q + al((nvis / 32 + 2) * 4ull) + al((Mcb + 1) * 4) + 3 * al((Mcb + 1) * I) + 2 * al((2 * Mcb + 1) * I);
            const unsigned long long pH = Rr + 2 * al((Hb + 1) * 4) + al((Hb + 1) * I) + al((Mcb + 1) * I);
            const unsigned long long pI = Rr + al((nvis + 1ull) * I) + al((VWb + 1) * 4) + al((VWb + 1) * I) + al((nsp + 1) * I) + 3 * al((nsp + 1) * 4);
            if (pG2 > peak) peak = pG2;
            if (pG3 > peak) peak = pG3;
            if (pH > peak) peak = pH;
            if (pI > peak) peak = pI;
        }
        if (peak > A.sm_cap) return 1;
    }
    PT_ALLOC(PosBase, uint32_t, M + 2);   // pos(i) = PosBase[run] + i        (wrap-around arithmetic)
    PT_ALLOC(VisBase, uint32_t, M + 2);   // vis(i) = VisBase[run] + visBefore(i)
    const uint32_t mark2_sm = A.sm_used; const unsigned long long mark2_gm = A.gm_used;   // run-tree temporaries, released after E
    PT_ALLOC(Node, unsigned long long, E + 1);   // E: Euler-tour nodes
    PT_ALLOC(Sub, unsigned long long, (E + 7) / 8 + 3);   // splitter sublist summaries
    PT_ALLOC(Sub2, unsigned long long, (E + 7) / 8 + 3);  // second buffer for the jumping rounds
    PT_ALLOC(RunHead, Idx, M + 1);
    PT_ALLOC(Prun, Idx, M + 1);
    PT_ALLOC(Key, uint32_t, M + 1);
    uint32_t* GrpCnt = VisBase;                     // children per node (node M = HEAD); dead before VisBase is written
    uint32_t* GrpCur = PosBase;                     // fill cursors; dead before PosBase is written
    PT_ALLOC(GrpOff, Idx, M + 2);
    PT_ALLOC(Unsorted, Idx, M + 1);
    PT_ALLOC(Sorted, Idx, M + 1);
    PT_ALLOC(SPos, Idx, M + 1);
    PT_ALLOC(BigList, Idx, M / 33 + 2);
    PT_ALLOC(GBits, uint32_t, (KS + 31) / 32 + 1);
    PT_ALLOC(GPre, Idx, (KS + 31) / 32 + 1);
    fill<uint32_t, BLOCK>(GrpCnt, M + 2, 0u);
    fill<uint32_t, BLOCK>(GrpCur, M + 2, 0u);
    __syncthreads();
    for (uint32_t w = tid; w < NWr; w += BLOCK) {      // compact the run heads: RunHead[run] = record index (one bit word per thread)
        uint32_t hb = HeadBits[w], rid = HeadPre[w];
        while (hb) { const uint32_t b = __ffs(hb) - 1; hb &= hb - 1; RunHead[rid++] = (Idx)(w * 32 + b); }
    }
    __syncthreads();
    for (uint32_t rid = tid; rid < M; rid += BLOCK) {  // one thread per run
        const uint32_t i = RunHead[rid], w = i >> 5, b = i & 31;
        // run = insert records from i up to the next head or non-insert record
        uint32_t stop = (HeadBits[w] | ~InsBits[w]) & ~(0xFFFFFFFFu >> (31 - b));
        uint32_t ww = w;
        while (!stop) { ww++; stop = HeadBits[ww] | ~InsBits[ww]; }     // pad word: InsBits == 0 -> stops
        const uint32_t end = ww * 32 + (__ffs(stop) - 1);
        const uint4 rec = ld_rec(ins + i);
        const uint32_t p = rec.y == 0 ? n : (uint32_t)T[keyOf(rec.y, rec.z >> 16)];
        const uint32_t q = p == n ? M : runOf(p);
        Node[rid] = node_make(0, end - i, visBefore(end) - visBefore(i));   // weights now, successor in phase E
        Prun[rid] = (Idx)q;
        Key[rid] = keyOf(rec.x, rec.z & 0xFFFFu);
        atomicAdd(&GrpCnt[q], 1u);
    }
    __syncthreads();
    {
        uint32_t carry = 0;
        for (uint32_t base = 0; base < M + 1; base += BLOCK) {
            uint32_t q = base + tid, total;
            uint32_t ex = block_scan_excl<BLOCK>(q < M + 1 ? GrpCnt[q] : 0u, c, total);
            if (q < M + 1) { GrpOff[q] = (Idx)(carry + ex); if (GrpCnt[q] > 32u) BigList[atomicAdd(&c.misc[3], 1u)] = (Idx)q; }
            carry += total;
        }
    }
    __syncthreads();
    for (uint32_t r = tid; r < M; r += BLOCK) {
        uint32_t q = Prun[r];
        Unsorted[(uint32_t)GrpOff[q] + atomicAdd(&GrpCur[q], 1u)] = (Idx)r;
    }
    __syncthreads();
    constexpr uint32_t kBigGroup = 32;                 // larger sibling groups are ranked with a key-space bitmap, not by counting
    for (uint32_t r = tid; r < M; r += BLOCK) {
        uint32_t q = Prun[r], cnt = GrpCnt[q], off = GrpOff[q];
        if (cnt > kBigGroup) continue;
        uint32_t rank = 0;
        if (cnt > 1) { uint32_t kr = Key[r]; for (uint32_t s = 0; s < cnt; s++) rank += Key[Unsorted[off + s]] > kr ? 1u : 0u; }
        Sorted[off + rank] = (Idx)r;
        SPos[r] = (Idx)(off + rank);
    }
    const uint32_t nBig = c.misc[3];
    if (nBig) {
        // rank inside a big group = number of members with a larger opId key = members' bits above mine in a bitmap over
        // the key space (unique keys: a counting sort).  One group at a time, all threads cooperate.
        const uint32_t KWg = (KS + 31) / 32;
        for (uint32_t g = 0; g < nBig; g++) {
            const uint32_t q = BigList[g], cnt = GrpCnt[q], off = GrpOff[q];
            fill<uint32_t, BLOCK>(GBits, KWg + 1, 0u);
            __syncthreads();
            for (uint32_t s2 = tid; s2 < cnt; s2 += BLOCK) { const uint32_t k = Key[Unsorted[off + s2]]; atomicOr(&GBits[k >> 5], 1u << (k & 31)); }
            __syncthreads();
            {
                uint32_t carry = 0;
                for (uint32_t base = 0; base < KWg; base += BLOCK) {
                    uint32_t w = base + tid, total;
                    uint32_t ex = block_scan_excl<BLOCK>(w < KWg ? __popc(GBits[w]) : 0u, c, total);
                    if (w < KWg) GPre[w] = (Idx)(carry + ex);
                    carry += total;
                }
            }
            __syncthreads();
            for (uint32_t s2 = tid; s2 < cnt; s2 += BLOCK) {
                const uint32_t r = Unsorted[off + s2], k = Key[r];
                const uint32_t below = (uint32_t)GPre[k >> 5] + __popc(GBits[k >> 5] & ((1u << (k & 31)) - 1u));
                const uint32_t rank = cnt - 1u - below;          // members with a larger key come first
                Sorted[off + rank] = (Idx)r;
                SPos[r] = (Idx)(off + rank);
            }
            __syncthreads();
        }
    }
    __syncthreads();

    // ---- E: Euler tour (enter r = r, exit r = (M+1)+r, r in 0..M) + weighted pointer-jumping list ranking ------------------
    // One 64-bit word per node: next | element weight | visible weight; invariant: the weights of x cover the nodes from
    // x up to (excluding) next(x).
    for (uint32_t r = tid; r <= M; r += BLOCK) {
        const uint32_t ent = r, ext = (M + 1) + r;
        const uint32_t cnt = GrpCnt[r];
        const uint32_t first = cnt ? (uint32_t)Sorted[GrpOff[r]] : ext;
        Node[ent] = (r < M ? (Node[ent] & ~kNodeNxtMask) : 0ull) | first;
        uint32_t nx;
        if (r == M) nx = END;
        else {
            const uint32_t q = Prun[r], sp = SPos[r];
            const bool last = sp + 1 == (uint32_t)GrpOff[q] + GrpCnt[q];
            nx = last ? (M + 1) + q : (uint32_t)Sorted[sp + 1];
        }
        Node[ext] = node_make(nx, 0, 0);
    }
    if (tid == 0) Node[END] = node_make(END, 0, 0);
    __syncthreads();
    // Work-efficient ranking: every 8th node id (and the list head) is a SPLITTER.  (1) each splitter walks its sublist
    // once, leaving in every visited node (owner splitter, weight prefix inside the sublist); (2) only the ~E/8 splitter
    // summaries are ranked by pointer jumping; (3) suffix(x) = suffix(owner sublist) - prefix(x).
    const uint32_t headNode = M;                              // enter(HEAD) starts the tour
    const uint32_t nSp = (E + 7) / 8 + 1;                     // splitter ids: k < nSp-1 -> node 8k ; nSp-1 -> headNode (if not a multiple of 8)
    const uint32_t SPEND = nSp;                               // terminator of the splitter list
    auto spOf = [&](uint32_t x) -> uint32_t { return (x & 7u) == 0 ? (x >> 3) : nSp - 1; };
    auto isSp = [&](uint32_t x) -> bool { return (x & 7u) == 0 || x == headNode; };
    for (uint32_t k = tid; k < nSp; k += BLOCK) {
        uint32_t cur = k + 1 < nSp ? 8 * k : headNode;
        unsigned long long acc = 0;
        bool valid = cur < E && (k + 1 < nSp || (headNode & 7u) != 0);
        uint32_t nx = END;
        if (valid) {
            for (;;) {
                const unsigned long long a = Node[cur];
                nx = (uint32_t)(a & kNodeNxtMask);
                Node[cur] = acc | k;                          // (owner, prefix before this node)
                acc += a & ~kNodeNxtMask;
                if (nx == END || isSp(nx)) break;
                cur = nx;
            }
        }
        Sub[k] = valid ? (acc | (nx == END ? SPEND : spOf(nx))) : (unsigned long long)SPEND;
    }
    if (tid == 0) { Sub[SPEND] = SPEND; Sub2[SPEND] = SPEND; }
    __syncthreads();
    {   // pointer jumping over the splitter summaries only, double buffered (race-free)
        unsigned long long *cur = Sub, *nxt2 = Sub2;
        for (uint32_t span = 1; span < nSp + 1; span <<= 1) {
            for (uint32_t x = tid; x < nSp; x += BLOCK) {
                const unsigned long long a = cur[x];
                const unsigned long long b = cur[(uint32_t)(a & kNodeNxtMask)];      // cur[SPEND] = {SPEND, 0, 0}
                nxt2[x] = ((a & ~kNodeNxtMask) + (b & ~kNodeNxtMask)) | (b & kNodeNxtMask);
            }
            __syncthreads();
            unsigned long long* t = cur; cur = nxt2; nxt2 = t;
        }
        Sub = cur;
    }
    for (uint32_t r = tid; r < M; r += BLOCK) {
        const unsigned long long loc = Node[r];
        const unsigned long long a = (Sub[(uint32_t)(loc & kNodeNxtMask)] & ~kNodeNxtMask) - (loc & ~kNodeNxtMask);   // elements / visible from run r to the end
        const uint32_t sufEl = (uint32_t)(a >> 20) & 0x3FFFFFu, sufVis = (uint32_t)(a >> 42);
        const uint32_t h = RunHead[r];
        PosBase[r] = (N - sufEl) - h;
        VisBase[r] = (nvis - sufVis) - visBefore(h);
    }
    __syncthreads();
    A.sm_used = mark2_sm; A.gm_used = mark2_gm;     // release the run-tree temporaries
    auto posOf = [&](uint32_t i) -> uint32_t { return PosBase[runOf(i)] + i; };                    // sequence position of element record i
    auto visOf = [&](uint32_t i) -> uint32_t { return VisBase[runOf(i)] + visBefore(i); };         // visible elements before it in the sequence
    auto isVis = [&](uint32_t i) -> bool { return (VisBits[i >> 5] >> (i & 31)) & 1u; };

    // ---- F: text out (visible index = prefix count of non-deleted elements, micromerge.ts:747-750) ------------------------------
    // only VISIBLE elements are touched (4 bytes of their record: the value token); the element sequence, when requested,
    // needs every insert
    {
        unsigned long long d0 = 0, d1 = 0;
        auto stepF = [&](uint32_t i, bool live) {
            if (!live) return;
            const bool vis = isVis(i);
            if (seq_out) seq_out[posOf(i)] = i | (vis ? 0u : 0x80000000u);
            if (!vis) return;
            const uint32_t tok = PT_PAYLOAD_TOKEN(__ldg(&ins[i].payload));
            const uint32_t vr = visOf(i);
            text_out[vr] = tok;
            digest_add(d0, d1, pt_term_text(vr, tok));
        };
        const uint32_t* LiveBits = seq_out ? InsBits : VisBits;
        for (uint32_t base = 0; base < n; base += 2 * BLOCK) {
            const uint32_t i0 = base + tid, i1 = i0 + BLOCK;
            stepF(i0, i0 < n && ((LiveBits[i0 >> 5] >> (i0 & 31)) & 1u));
            stepF(i1, i1 < n && ((LiveBits[i1 >> 5] >> (i1 & 31)) & 1u));
        }
        digest_flush<BLOCK>(c, d0, d1);
    }

    uint32_t nspans = 0;
    if (m == 0) {
        // no marks: one span {} covering all visible text (peritext.ts:392), none if the text is empty
        if (nvis && tid == 0) {
            pt_span s; s.start = 0; s.flags = 0; s.link_attr = PT_ATTR_NONE; s.comment_off = 0;
            span_out[0] = s;
            unsigned long long d0 = 0, d1 = 0;
            digest_add(d0, d1, pt_term_span(0, 0, 0, PT_ATTR_NONE));
            atomicAdd(&c.dig0, d0); atomicXor(&c.dig1, d1);
        }
        nspans = nvis ? 1u : 0u;
    } else {
        // ---- G: marks ---------------------------------------------------------------------------------------------------
        // G1: rank mark ops by opId: bitmap over the key space + prefix popcount (a counting sort with unique keys)
        const uint32_t NWp = (N + 32) / 32 + 1;          // words over sequence positions 0..N
        const uint32_t KW = (KS + 31) / 32;
        PT_ALLOC(ByRank, Idx, m + 1);
        PT_ALLOC(MRank, Idx, m + 1);
        PT_ALLOC(IvA, Idx, m + 1);         // element interval [a,b) per mark op; a == b: covers nothing
        PT_ALLOC(IvB, Idx, m + 1);
        PT_ALLOC(IvVA, Idx, m + 1);        // visible rank of positions a and b
        PT_ALLOC(IvVB, Idx, m + 1);
        PT_ALLOC(MKind, uint8_t, m + 1);   // pt_mark_rec.kind (bit0 remove, bits2:1 type)
        PT_ALLOC(MAttr, uint32_t, m + 1);
        PT_ALLOC(CompactC, uint32_t, m + 1);     // indices of non-empty comment ops
        PT_ALLOC(BndBits, uint32_t, NWp + 1);
        PT_ALLOC(SegPre, Idx, NWp + 1);
        const uint32_t mark3_sm = A.sm_used; const unsigned long long mark3_gm = A.gm_used;
        PT_ALLOC(KBits, uint32_t, KW + 1);       // temporaries of G1/G2
        PT_ALLOC(KPre, Idx, KW + 1);
        fill<uint32_t, BLOCK>(KBits, KW + 1, 0u);
        fill<uint32_t, BLOCK>(BndBits, NWp + 1, 0u);
        if (tid == 0) { c.misc[1] = 0; }
        __syncthreads();
        for (uint32_t k = tid; k < m; k += BLOCK) {
            uint32_t ctr = mk[k].ctr, actor = mk[k].actor;
            if (badId(ctr, actor)) { fail(PT_LOG_BAD_OPID); continue; }
            uint32_t key = keyOf(ctr, actor);
            uint32_t old = atomicOr(&KBits[key >> 5], 1u << (key & 31));
            if ((old >> (key & 31)) & 1u) fail(PT_LOG_BAD_OPID);
            if (T[key] != NONE) fail(PT_LOG_BAD_OPID);
        }
        __syncthreads();
        if (c.status) { bail(); return 0; }
        {
            uint32_t carry = 0;
            for (uint32_t base = 0; base < KW; base += BLOCK) {
                uint32_t w = base + tid, total;
                uint32_t ex = block_scan_excl<BLOCK>(w < KW ? __popc(KBits[w]) : 0u, c, total);
                if (w < KW) KPre[w] = (Idx)(carry + ex);
                carry += total;
            }
        }
        __syncthreads();
        // G2: boundary slots -> element intervals (SURVEY.md §9.2 item 3); comment ops are compacted on the side
        for (uint32_t k = tid; k < m; k += BLOCK) {
            const uint4* q = reinterpret_cast<const uint4*>(mk + k);
            const uint4 r0 = __ldg(q), r1 = __ldg(q + 1);
            // r0 = {ctr, actor|kind<<16|bounds<<24, start_ctr, end_ctr}; r1 = {start_actor|end_actor<<16, attr, arrival, reserved}
            const uint32_t ctr = r0.x, actor = r0.y & 0xFFFFu, kind = (r0.y >> 16) & 0xFFu, bounds = r0.y >> 24;
            const uint32_t start_ctr = r0.z, end_ctr = r0.w, start_actor = r1.x & 0xFFFFu, end_actor = r1.x >> 16, attr = r1.y, arrival = r1.z;
            uint32_t key = keyOf(ctr, actor);
            uint32_t rank = (uint32_t)KPre[key >> 5] + __popc(KBits[key >> 5] & ((1u << (key & 31)) - 1u));
            MRank[k] = (Idx)rank; ByRank[rank] = (Idx)k; MKind[k] = (uint8_t)kind; MAttr[k] = attr;
            uint32_t sb = bounds & 3u, eb = (bounds >> 2) & 3u;
            // a slot is 2*pos + (after ? 1 : 0); NOSLOT: the walk never matches this boundary (peritext.ts:236-241)
            const uint32_t NOSLOT = 0xFFFFFFFFu;
            uint32_t ps = NOSLOT, pe = NOSLOT, vs = 0, ve = nvis;
            if (sb <= PT_BOUND_AFTER && !badId(start_ctr, start_actor)) {
                // the boundary element must have ARRIVED before the mark op: the reference's walk at apply time never matches
                // an element that is inserted later (peritext.ts:236-241) — a missing start is a no-op, a missing end never ends
                Idx j = T[keyOf(start_ctr, start_actor)];
                if (j != NONE && (uint32_t)j < arrival) {
                    ps = 2u * posOf(j) + sb; vs = visOf(j) + ((sb && isVis(j)) ? 1u : 0u);
                    if (seq_out && sb == PT_BOUND_AFTER) atomicOr(&seq_out[posOf(j)], 0x40000000u);    // the element's markOpsAfter slot is defined
                }
            }
            if (eb <= PT_BOUND_AFTER && !badId(end_ctr, end_actor)) {
                Idx j = T[keyOf(end_ctr, end_actor)];
                if (j != NONE && (uint32_t)j < arrival) {
                    pe = 2u * posOf(j) + eb; ve = visOf(j) + ((eb && isVis(j)) ? 1u : 0u);
                    if (seq_out && eb == PT_BOUND_AFTER) atomicOr(&seq_out[posOf(j)], 0x40000000u);    // (src/peritext.ts:239-241 writes the end slot whenever the walk reaches it)
                }
            }
            uint32_t a = 0, b = 0;
            if (ps != NOSLOT) {
                if (pe == ps || pe == NOSLOT) { pe = 2u * N; ve = nvis; }   // same slot: start branch wins, never ends (quirk Q2)
                a = (ps + 1u) >> 1; b = (pe + 1u) >> 1; if (b > N) b = N;
                if (a >= b) { a = 0; b = 0; }
            }
            IvA[k] = (Idx)a; IvB[k] = (Idx)b; IvVA[k] = (Idx)vs; IvVB[k] = (Idx)ve;
            if (a < b) {
                atomicOr(&BndBits[a >> 5], 1u << (a & 31)); atomicOr(&BndBits[b >> 5], 1u << (b & 31));
                if (((kind >> 1) & 3u) == PT_MARK_COMMENT) CompactC[atomicAdd(&c.misc[1], 1u)] = k;
            }
        }
        __syncthreads();
        A.sm_used = mark3_sm; A.gm_used = mark3_gm;     // release KBits / KPre
        const uint32_t Mc = c.misc[1];
        uint32_t S;   // number of segment ids: seg(x) in [0, S)
        {
            uint32_t carry = 0;
            for (uint32_t base = 0; base < NWp; base += BLOCK) {
                uint32_t w = base + tid, total;
                uint32_t ex = block_scan_excl<BLOCK>(w < NWp ? __popc(BndBits[w]) : 0u, c, total);
                if (w < NWp) SegPre[w] = (Idx)(carry + ex);
                carry += total;
            }
            S = carry + 1;
        }
        __syncthreads();
        auto segOf = [&](uint32_t x) -> uint32_t {    // popcount(boundary bits[0..x]) inclusive
            uint32_t w = x >> 5, b = x & 31;
            return (uint32_t)SegPre[w] + __popc(BndBits[w] & (0xFFFFFFFFu >> (31 - b)));
        };
        // G3: stabbing max per LWW type: an iterative segment tree over segment ids (range atomicMax, point query), ONE type at
        // a time in the same buffer (three trees at once were the peak of the whole pipeline's shared-memory footprint and
        // pushed 10K-record logs with ~1K marks into the one-CTA-per-SM bin)
        const uint32_t TS = 2 * S + 2;
        PT_ALLOC(SegFlags, uint32_t, S + 1);
        PT_ALLOC(SegLink, uint32_t, S + 1);
        const uint32_t mark4_sm = A.sm_used; const unsigned long long mark4_gm = A.gm_used;
        PT_ALLOC(Tree, uint32_t, TS);          // temporaries of G3
        PT_ALLOC(CDiff, int, S + 2);
        fill<uint32_t, BLOCK>(SegFlags, S + 1, 0u);
        fill<uint32_t, BLOCK>(SegLink, S + 1, PT_ATTR_NONE);
        fill<int, BLOCK>(CDiff, S + 2, 0);
#pragma unroll 1
        for (uint32_t pass = 0; pass < 3; pass++) {
            const uint32_t ptype = pass == 0 ? PT_MARK_STRONG : pass == 1 ? PT_MARK_EM : PT_MARK_LINK;
            fill<uint32_t, BLOCK>(Tree, TS, 0u);
            __syncthreads();
            for (uint32_t k = tid; k < m; k += BLOCK) {
                const uint32_t a = IvA[k], b = IvB[k];
                if (a >= b) continue;
                const uint32_t t = ((uint32_t)MKind[k] >> 1) & 3u;
                if (t == PT_MARK_COMMENT) { if (pass == 0) { atomicAdd(&CDiff[segOf(a)], 1); atomicAdd(&CDiff[segOf(b)], -1); } continue; }   // G4 difference array
                if (t != ptype) continue;
                const uint32_t sa = segOf(a), sb2 = segOf(b);
                const uint32_t v = (uint32_t)MRank[k] + 1u;
                for (uint32_t l = sa + S, r = sb2 + S; l < r; l >>= 1, r >>= 1) {
                    if (l & 1u) atomicMax(&Tree[l++], v);
                    if (r & 1u) atomicMax(&Tree[--r], v);
                }
            }
            __syncthreads();
            // LWW winner of this type per segment (peritext.ts:304-313): present iff the max-opId covering op is an addMark
            for (uint32_t s2 = tid; s2 < S; s2 += BLOCK) {
                uint32_t w = 0;
                for (uint32_t p = s2 + S; p >= 1; p >>= 1) w = max(w, Tree[p]);
                if (w) {
                    const uint32_t kk = ByRank[w - 1];
                    if (!(MKind[kk] & 1u)) {
                        SegFlags[s2] |= pass == 0 ? PT_SPAN_STRONG : pass == 1 ? PT_SPAN_EM : PT_SPAN_LINK;
                        if (pass == 2) SegLink[s2] = MAttr[kk];
                    }
                }
            }
            __syncthreads();
        }
        // G4: `comment` key present iff >= 1 comment op covers the segment (quirk Q3): running sum of the difference array
        {
            int carry = 0;
            for (uint32_t base = 0; base < S; base += BLOCK) {
                const uint32_t s2 = base + tid;
                const int v = s2 < S ? CDiff[s2] : 0;
                uint32_t total;
                const uint32_t ex = block_scan_excl<BLOCK>((uint32_t)v, c, total);   // two's complement sums are fine
                if (s2 < S && carry + (int)ex + v > 0) SegFlags[s2] |= PT_SPAN_COMMENT;
                carry += (int)total;
            }
        }
        A.sm_used = mark4_sm; A.gm_used = mark4_gm;     // release Tree / CDiff (the scan above ended with a barrier)

        // ---- H: comment presence pieces (per comment id an LWW channel, peritext.ts:314-322 folded in opId order) ----------
        // comment ops sorted by (id, op index) by counting; a piece = elementary interval of one id where an add wins
        const uint32_t HW = nvis / 32 + 1;
        PT_ALLOC(CHead, uint32_t, HW + 1);
        PT_ALLOC(CId, uint32_t, Mc + 1);        // sorted by (id, k)
        PT_ALLOC(CK, Idx, Mc + 1);                   // mark op index
        PT_ALLOC(CG0, Idx, Mc + 1);                  // first sorted position of the op's id group
        PT_ALLOC(CGn, Idx, Mc + 1);                  // group size
        PT_ALLOC(PcA, Idx, 2 * Mc + 1);
        PT_ALLOC(PcB, Idx, 2 * Mc + 1);              // PcA == PcB: dead piece
        // group the comment ops by id: open-addressing hash of the ids, bucket counts, scan, fill (O(Mc))
        uint32_t Hbits = 1; while ((1u << Hbits) < 2 * Mc + 2) Hbits++;
        const uint32_t H = 1u << Hbits;
        const uint32_t mark5_sm = A.sm_used; const unsigned long long mark5_gm = A.gm_used;
        PT_ALLOC(HTab, uint32_t, H);                      // id + 1 (0 = empty); later the fill cursor   (temporaries)
        PT_ALLOC(HCnt, uint32_t, H + 1);
        PT_ALLOC(HOff, Idx, H + 1);
        PT_ALLOC(CSlot, Idx, Mc + 1);
        fill<uint32_t, BLOCK>(CHead, HW + 1, 0u);
        fill<uint32_t, BLOCK>(HTab, H, 0u);
        fill<uint32_t, BLOCK>(HCnt, H + 1, 0u);
        __syncthreads();
        for (uint32_t ci = tid; ci < Mc; ci += BLOCK) {
            const uint32_t id = MAttr[CompactC[ci]];
            uint32_t slot = (id * 2654435761u) >> (32 - Hbits);
            for (;;) {
                const uint32_t old = atomicCAS(&HTab[slot], 0u, id + 1u);
                if (old == 0u || old == id + 1u) break;
                slot = (slot + 1) & (H - 1);
            }
            CSlot[ci] = (Idx)slot;
            atomicAdd(&HCnt[slot], 1u);
        }
        __syncthreads();
        {
            uint32_t carry = 0;
            for (uint32_t base = 0; base < H; base += BLOCK) {
                uint32_t q = base + tid, total;
                uint32_t ex = block_scan_excl<BLOCK>(q < H ? HCnt[q] : 0u, c, total);
                if (q < H) HOff[q] = (Idx)(carry + ex);
                carry += total;
            }
        }
        __syncthreads();
        for (uint32_t ci = tid; ci < Mc; ci += BLOCK) {
            const uint32_t k = CompactC[ci], id = MAttr[k], slot = CSlot[ci];
            const uint32_t pos = (uint32_t)HOff[slot] + (atomicAdd(&HTab[slot], 1u) - (id + 1u));
            CId[pos] = id; CK[pos] = (Idx)k; CG0[pos] = HOff[slot]; CGn[pos] = (Idx)HCnt[slot];
        }
        __syncthreads();
        A.sm_used = mark5_sm; A.gm_used = mark5_gm;     // release the hash temporaries
        for (uint32_t e = tid; e < 2 * Mc; e += BLOCK) {
            const uint32_t ci = e >> 1, which = e & 1u, k = CK[ci];
            const uint32_t g0 = CG0[ci], g1 = g0 + (uint32_t)CGn[ci];
            const uint32_t x = which ? (uint32_t)IvB[k] : (uint32_t)IvA[k];
            const uint32_t xv = which ? (uint32_t)IvVB[k] : (uint32_t)IvVA[k];
            bool dup = false; uint32_t nextEnd = 0xFFFFFFFFu, nextV = 0;
            for (uint32_t cj = g0; cj < g1; cj++) {
                const uint32_t j = CK[cj];
                const uint32_t ja = IvA[j], jb = IvB[j];
                if (ja == x && (cj < ci || (cj == ci && 0u < which))) dup = true;
                if (jb == x && (cj < ci || (cj == ci && 1u < which))) dup = true;
                if (ja > x && ja < nextEnd) { nextEnd = ja; nextV = IvVA[j]; }
                if (jb > x && jb < nextEnd) { nextEnd = jb; nextV = IvVB[j]; }
            }
            uint32_t va = 0, vb = 0;
            if (!dup && nextEnd != 0xFFFFFFFFu) {
                uint32_t best = 0; bool bestAdd = false;
                for (uint32_t cj = g0; cj < g1; cj++) {
                    const uint32_t j = CK[cj];
                    if ((uint32_t)IvA[j] <= x && nextEnd <= (uint32_t)IvB[j]) {
                        // comment ops fold in Set order = ARRIVAL order, no opId comparison (peritext.ts:314-322, quirk Q4): the
                        // last-arrived covering op of this id decides; mark records are stored in arrival order
                        const uint32_t rk = j + 1u;
                        if (rk > best) { best = rk; bestAdd = (MKind[j] & 1u) == 0; }
                    }
                }
                if (best && bestAdd) { va = xv; vb = nextV; if (va >= vb) { va = 0; vb = 0; } }
            }
            PcA[e] = (Idx)va; PcB[e] = (Idx)vb;
        }
        __syncthreads();
        for (uint32_t e = tid; e < 2 * Mc; e += BLOCK) {
            const uint32_t va = PcA[e], vb = PcB[e];
            if (va >= vb) continue;
            const uint32_t ci = e >> 1, g0 = CG0[ci], g1 = g0 + (uint32_t)CGn[ci];
            bool startTouch = false, endTouch = false;
            for (uint32_t f = 2 * g0; f < 2 * g1; f++) {
                const uint32_t fa = PcA[f], fb = PcB[f];
                if (fa >= fb) continue;
                if (fb == va) startTouch = true;
                if (fa == vb) endTouch = true;
            }
            if (!startTouch) atomicOr(&CHead[va >> 5], 1u << (va & 31));
            if (!endTouch) atomicOr(&CHead[vb >> 5], 1u << (vb & 31));
        }

        // ---- I: spans ---------------------------------------------------------------------------------------------------
        PT_ALLOC(VisSeg, Idx, nvis + 1);
        const uint32_t VW = (nvis + 31) / 32;
        PT_ALLOC(HeadB, uint32_t, VW + 1);
        PT_ALLOC(HeadP, Idx, VW + 1);
        for (uint32_t i = tid; i < n; i += BLOCK) {
            if (!isVis(i)) continue;
            VisSeg[visOf(i)] = (Idx)segOf(posOf(i));
        }
        __syncthreads();
        for (uint32_t base = 0; base < VW * 32; base += BLOCK) {       // head flags: one thread per visible position, ballot -> word
            const uint32_t v = base + tid;
            bool h = false;
            if (v < nvis) {
                if (v == 0) h = true;
                else {
                    const uint32_t s1 = VisSeg[v - 1], s2 = VisSeg[v];
                    h = ((CHead[v >> 5] >> (v & 31)) & 1u) || (s1 != s2 && (SegFlags[s1] != SegFlags[s2] || SegLink[s1] != SegLink[s2]));
                }
            }
            const uint32_t bits = __ballot_sync(0xffffffffu, h);
            if (lane == 0 && (v >> 5) < VW) HeadB[v >> 5] = bits;
        }
        __syncthreads();
        {
            uint32_t carry = 0;
            for (uint32_t base = 0; base < VW; base += BLOCK) {
                uint32_t w = base + tid, total;
                uint32_t ex = block_scan_excl<BLOCK>(w < VW ? __popc(HeadB[w]) : 0u, c, total);
                if (w < VW) HeadP[w] = (Idx)(carry + ex);
                carry += total;
            }
            nspans = carry;
        }
        __syncthreads();
        auto headRank = [&](uint32_t v) -> uint32_t {   // number of span heads at visible positions < v  (v in 0..nvis)
            uint32_t w = v >> 5, b = v & 31;
            if (w >= VW) return nspans;
            return (uint32_t)HeadP[w] + __popc(HeadB[w] & ((1u << b) - 1u));
        };
        // comment lists per span: count, reserve pool space, fill, sort; span start positions for the per-span pass
        PT_ALLOC(SpanStart, Idx, nspans + 1);
        PT_ALLOC(SpanCC, uint32_t, nspans + 1);
        PT_ALLOC(SpanCO, uint32_t, nspans + 1);
        PT_ALLOC(SpanCur, uint32_t, nspans + 1);
        fill<uint32_t, BLOCK>(SpanCC, nspans + 1, 0u);
        fill<uint32_t, BLOCK>(SpanCur, nspans + 1, 0u);
        for (uint32_t v = tid; v < nvis; v += BLOCK)
            if ((HeadB[v >> 5] >> (v & 31)) & 1u) SpanStart[headRank(v)] = (Idx)v;
        __syncthreads();
        // many spans per piece: one warp per piece, lanes over the spans it covers; few spans: one thread per piece
        const bool wpp = nspans >= 256;
        const uint32_t pe0 = wpp ? (tid >> 5) : tid, peStep = wpp ? BLOCK / 32 : BLOCK, pj0 = wpp ? lane : 0u, pjStep = wpp ? 32u : 1u;
        for (uint32_t e = pe0; e < 2 * Mc; e += peStep) {
            uint32_t va = PcA[e], vb = PcB[e];
            if (va >= vb) continue;
            for (uint32_t j = headRank(va) + pj0, j1 = headRank(vb); j < j1; j += pjStep) atomicAdd(&SpanCC[j], 1u);
        }
        __syncthreads();
        uint32_t totalC;
        {
            uint32_t carry = 0;
            for (uint32_t base = 0; base < nspans; base += BLOCK) {
                uint32_t j = base + tid, total;
                uint32_t ex = block_scan_excl<BLOCK>(j < nspans ? SpanCC[j] : 0u, c, total);
                if (j < nspans) SpanCO[j] = carry + ex;
                carry += total;
            }
            totalC = carry;
        }
        if (tid == 0) {
            unsigned long long base = 0;
            if (totalC) base = pool_reserve(P, totalC, c.status);
            c.pool_base = base;
        }
        __syncthreads();
        if (c.status) { bail(); return 0; }
        uint32_t* pool = P.comment_pool + c.pool_base;
        // build and sort the lists in shared memory when they fit (latency of the per-span sort), else in the pool itself
        const unsigned long long slBytes = ((unsigned long long)totalC * 4u + 15u) & ~15ull;
        const bool staged = totalC > 0 && A.sm_used + slBytes <= A.sm_cap;
        uint32_t* SL = staged ? reinterpret_cast<uint32_t*>(ptk_smem + A.sm_used) : pool;
        for (uint32_t e = pe0; e < 2 * Mc; e += peStep) {
            uint32_t va = PcA[e], vb = PcB[e];
            if (va >= vb) continue;
            const uint32_t id = CId[e >> 1];
            for (uint32_t j = headRank(va) + pj0, j1 = headRank(vb); j < j1; j += pjStep)
                SL[SpanCO[j] + atomicAdd(&SpanCur[j], 1u)] = id;
        }
        __syncthreads();
        {
            unsigned long long d0 = 0, d1 = 0;
            for (uint32_t j = tid; j < nspans; j += BLOCK) {                // one thread per span
                const uint32_t v = SpanStart[j], s2 = VisSeg[v];
                const uint32_t cnt = SpanCC[j];
                uint32_t* lst = SL + SpanCO[j];
                for (uint32_t x = 1; x < cnt; x++) {                        // insertion sort: ascending comment id
                    uint32_t key = lst[x]; uint32_t y = x;
                    while (y > 0 && lst[y - 1] > key) { lst[y] = lst[y - 1]; y--; }
                    lst[y] = key;
                }
                pt_span sp; sp.start = v; sp.flags = SegFlags[s2] | (cnt << 8); sp.link_attr = SegLink[s2];
                sp.comment_off = cnt ? (uint32_t)(c.pool_base + SpanCO[j]) : 0u;
                span_out[j] = sp;
                for (uint32_t x = 0; x < cnt; x++) digest_add(d0, d1, pt_term_comment(j, x, lst[x]));
                digest_add(d0, d1, pt_term_span(j, sp.start, sp.flags, sp.link_attr));
            }
            if (staged) {
                __syncthreads();
                for (uint32_t x = tid; x < totalC; x += BLOCK) pool[x] = SL[x];   // coalesced copy to the comment pool
            }
            digest_flush<BLOCK>(c, d0, d1);
        }
    }
    __syncthreads();
    if (tid == 0) {
        pt_log_result r;
        r.status = A.overflow ? PT_LOG_OVERFLOW : c.status;
        r.n_elems = N; r.n_visible = nvis; r.n_spans = nspans;
        uint64_t t = pt_term_counts(nvis, nspans);
        r.digest[0] = c.dig0 + t; r.digest[1] = c.dig1 ^ pt_term_hi(t);
        if (r.status) { r.n_elems = r.n_visible = r.n_spans = 0; r.digest[0] = r.digest[1] = 0; }
        *res = r;
    }
    __syncthreads();
    return 0;
}

// Persistent CTAs pull logs from the bin's work queue; the next log's records are prefetched into L2 while the
// current one is processed.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (BLOCK == 512 ? 2 : BLOCK == 256 ? 3 : BLOCK == 128 ? 7 : BLOCK == 64 ? 8 : BLOCK == 32 ? 8 : 1)) merge_logs_kernel(const BatchParams P) {
    __shared__ BlockCtx<BLOCK> ctx;
    const uint32_t n_work = P.n_work_dev ? *P.n_work_dev : P.n_work;
    uint32_t tma_parity = 0;                // bit b: parity to wait for on staging barrier b (uniform across the CTA)
    if (threadIdx.x == 0) { ctx.work_next = atomicAdd(P.work_counter, 1u); ctx.slab_slot = 0xFFFFFFFFu; mbar_init(&ctx.tma_bar[0], 1); mbar_init(&ctx.tma_bar[1], 1); mbar_fence_init(); }
    __syncthreads();
    for (;;) {
        const uint32_t w = ctx.work_next;
        __syncthreads();
        if (w >= n_work) break;
        if (threadIdx.x == 0) ctx.work_next = atomicAdd(P.work_counter, 1u);
        __syncthreads();
        const uint32_t wn = ctx.work_next;
        if (P.prefetch_next && wn < n_work) {
            const pt_log_desc& Ln = P.desc[P.order[wn]];
            const char* p0 = reinterpret_cast<const char*>(P.insdel + Ln.insdel_off);
            const uint32_t lines = (uint32_t)(((unsigned long long)Ln.n_insdel * sizeof(pt_insdel_rec) + 127) >> 7);
            for (uint32_t l = threadIdx.x; l < lines; l += BLOCK) prefetch_l2(p0 + ((size_t)l << 7));
        }
        const uint32_t li = P.order[w];
        if (P.admit && P.admit[li]) continue;      // rejected by the admission pre-pass (its status is already in the result header)
        const pt_log_desc& L = P.desc[li];
        const bool small = L.n_insdel < 32000u && L.n_mark < 32000u;
        // optimistic: everything in shared memory (LDS/STS); restart with the spill-capable variant if it does not fit
        int spill;
        if (small) spill = merge_one_log<uint16_t, BLOCK, true>(P, li, ctx, tma_parity); else spill = merge_one_log<uint32_t, BLOCK, true>(P, li, ctx, tma_parity);
        if (spill) {
            __syncthreads();
            if (P.retry_list) {            // defer to the next bin (larger shared-memory budget)
                if (threadIdx.x == 0) { P.retry_list[atomicAdd(P.retry_count, 1u)] = li; atomicAdd(&P.stats[2], 1ull); }
                continue;
            }
            if (small) merge_one_log<uint16_t, BLOCK, false>(P, li, ctx, tma_parity); else merge_one_log<uint32_t, BLOCK, false>(P, li, ctx, tma_parity);
        }
        if (threadIdx.x == 0) atomicAdd(&P.stats[spill ? 1 : 0], 1ull);
    }
}

}  // namespace ptk
