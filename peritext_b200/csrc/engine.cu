// engine.cu — C-ABI of the batch CRDT-merge engine (include/peritext_b200.h) over the sm_90a kernels.
//
// Host responsibilities (all per batch, none per op): size the output regions from the descriptors, bin the logs
// by size (block size + shared-memory budget per bin), order each bin largest-first for the persistent-CTA work
// queue, launch, and move results.  There is NO CPU fallback: without a CUDA device every entry point fails.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "merge_kernel.cuh"
#include "warp_kernel.cuh"
#include "patch_kernel.cuh"
#include "team_kernel.cuh"
#include "render_kernel.cuh"

namespace {

thread_local std::string g_last_error;

#define PT_CUDA(call)                                                                                   \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) {                                                                       \
            g_last_error = std::string(#call) + ": " + cudaGetErrorString(e__);                        \
            return PT_ERR_CUDA;                                                                         \
        }                                                                                               \
    } while (0)

struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return PT_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { g_last_error = std::string("cudaMalloc: ") + cudaGetErrorString(e); return PT_ERR_NOMEM; }
        cap = want; return PT_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct HostBuf {   // pinned
    void* p = nullptr; size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return PT_OK;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e != cudaSuccess) { g_last_error = std::string("cudaMallocHost: ") + cudaGetErrorString(e); return PT_ERR_NOMEM; }
        cap = want; return PT_OK;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

constexpr int kNumBins = 5;
struct BinCfg { uint32_t max_recs; int block; uint32_t smem; int ctas_per_sm; };
// shared memory per SM: 228 KB, 1 KB reserved per resident CTA, 227 KB max per CTA.
// Bin 0 is the WARP-PER-LOG kernel (warp_kernel.cuh): block = warps per CTA * 32, smem = bytes PER WARP; a log it cannot
// finish is deferred on the device to bin 1.  Bins 1..4 are the CTA-per-log kernel (merge_kernel.cuh).
BinCfg kBins[kNumBins] = {
    {2048u, 8 * 32, 7136u, 4},
    {1536u, 128, 31u * 1024u, 7},
    {4096u, 256, 74u * 1024u, 3},
    {12288u, 512, 112u * 1024u, 2},
    {0xFFFFFFFFu, 1024, 226u * 1024u, 1},
};
constexpr int kTeamWarps = 8;                 // team kernel (team_kernel.cuh): 8 warps per log, 4 logs per SM
constexpr uint32_t kTeamSmem = 55u * 1024u;
bool g_team_bin = true;
bool g_warp_bin = true, g_warp_force = false;   // force: skip the host-side footprint estimate (tests of the device-side deferral)

inline size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }

// Worst-case arena bytes of one log: an upper bound on the sum of every Arena::alloc in merge_one_log with
// M <= N <= n, S <= 2m+2, nvis <= n, Mc <= m, nspans <= 2m+1 (released arrays are counted too).
size_t arena_worst_bytes(uint64_t n, uint64_t m, uint64_t KS) {
    const size_t I = (n < 32000 && m < 32000) ? 2 : 4;
    size_t b = 0;
    auto A = [&](uint64_t count, size_t sz) { b += al16((size_t)count * sz); };
    const uint64_t NWr = (n + 31) / 32 + 1;
    A(KS, I); A(NWr, 4); A(NWr, 4); A(NWr, 4); A(NWr, I); A(NWr, I);               // T InsBits HeadBits VisBits HeadPre VisPre
    A(NWr * 32 + 32, 1); A(NWr * 32 + 32, 1);                                      // Other Del
    A(2 * n + 3, 8); A((2 * n + 9) / 8 + 3, 8); A((2 * n + 9) / 8 + 3, 8);         // Node Sub Sub2
    A(n + 1, I); A(n + 2, 4); A(n + 2, 4); A(n + 1, I); A(n + 1, 4); A(n + 2, I);  // RunHead PosBase VisBase Prun Key GrpOff
    A(n + 1, I); A(n + 1, I); A(n + 1, I);                                         // Unsorted Sorted SPos
    A(n / 33 + 2, I); A(KS / 32 + 2, 4); A(KS / 32 + 2, I);                        // BigList GBits GPre
    if (m) {
        const uint64_t KW = KS / 32 + 2, S = 2 * m + 2, Mc = m, nsp = 2 * m + 1, NWp = (n + 32) / 32 + 1;
        A(KW + 1, 4); A(KW + 1, I); for (int k = 0; k < 6; k++) A(m + 1, I);       // KBits KPre ByRank MRank IvA IvB IvVA IvVB
        A(m + 1, 1); A(m + 1, 4); A(m + 1, 4);                                     // MKind MAttr CompactC
        A(NWp + 1, 4); A(NWp + 1, I);                                              // BndBits SegPre
        A(2 * S + 2, 4); A(S + 1, 4); A(S + 1, 4); A(S + 2, 4);                    // Tree SegFlags SegLink CDiff
        A(n / 32 + 3, 4); A(Mc + 1, 4); A(Mc + 1, I); A(Mc + 1, I); A(Mc + 1, I);  // CHead CId CK CG0 CGn
        A(2 * Mc + 1, I); A(2 * Mc + 1, I);                                        // PcA PcB
        A(4 * Mc + 8, 4); A(4 * Mc + 9, 4); A(4 * Mc + 9, I); A(Mc + 1, I);        // HTab HCnt HOff CSlot
        A(n + 1, I); A(n / 32 + 2, 4); A(n / 32 + 2, I);                           // VisSeg HeadB HeadP
        A(nsp + 1, I); A(nsp + 1, 4); A(nsp + 1, 4); A(nsp + 1, 4);                // SpanStart SpanCC SpanCO SpanCur
    }
    return b + 256;
}

// Expands run-compressed ins/del streams into pt_insdel_rec records (one warp per log, lanes over the runs; a run's
// records are written by its lane — runs are short, and the expanded array is consumed from L2/HBM by the merge kernel).
__global__ void expand_runs_kernel(const pt_log_desc* __restrict__ desc, const unsigned long long* __restrict__ run_off,
                                   const unsigned long long* __restrict__ tok_off, const pt_run_rec* __restrict__ runs,
                                   const uint32_t* __restrict__ tokens, pt_insdel_rec* __restrict__ out, uint32_t n_logs) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        const unsigned long long r0 = run_off[li], r1 = run_off[li + 1];
        pt_insdel_rec* o = out + desc[li].insdel_off;
        const uint32_t* tk = tokens + tok_off[li];
        uint32_t rec_base = 0, tok_base = 0;
        for (unsigned long long rb = r0; rb < r1; rb += 32) {
            const unsigned long long ri = rb + lane;
            uint4 r = make_uint4(0, 0, 0, 0);
            uint32_t cnt = 0, kind = 0;
            if (ri < r1) { r = __ldg(reinterpret_cast<const uint4*>(runs + ri)); cnt = r.w & 0x3FFFFFFFu; kind = r.w >> 30; }
            uint32_t tcnt = kind == PT_KIND_INSERT ? cnt : 0u;
            // exclusive prefix sums of the record and token counts inside the warp
            uint32_t pr = cnt, pt = tcnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t a = __shfl_up_sync(0xffffffffu, pr, d), b2 = __shfl_up_sync(0xffffffffu, pt, d); if (lane >= (uint32_t)d) { pr += a; pt += b2; } }
            const uint32_t tot_r = __shfl_sync(0xffffffffu, pr, 31), tot_t = __shfl_sync(0xffffffffu, pt, 31);
            uint32_t ro = rec_base + pr - cnt, to = tok_base + pt - tcnt;
            const uint32_t actor = r.z & 0xFFFFu;
            for (uint32_t k = 0; k < cnt; k++) {
                uint4 w;
                w.x = r.x + k;
                if (kind == PT_KIND_INSERT) {
                    w.y = k == 0 ? r.y : r.x + k - 1;
                    w.z = actor | ((k == 0 ? (r.z >> 16) : actor) << 16);
                    w.w = (PT_KIND_INSERT << 30) | tk[to + k];
                } else {
                    w.y = r.y + k; w.z = r.z; w.w = kind << 30;
                }
                reinterpret_cast<uint4*>(o)[ro + k] = w;
            }
            rec_base += tot_r; tok_base += tot_t;
        }
    }
}


// ---- compact wire format: elementwise expansion to the 16 / 32 byte records the merge kernels read -------------------------
__global__ void expand_insdel_c8_kernel(const pt_insdel_c8* __restrict__ in, pt_insdel_rec* __restrict__ out, unsigned long long n) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint2 q = __ldg(reinterpret_cast<const uint2*>(in + i));
        const uint32_t tok22 = q.y >> 10;
        uint4 o;
        o.x = q.x & 0xFFFFu; o.y = q.x >> 16;
        o.z = (q.y & 0xFu) | (((q.y >> 4) & 0xFu) << 16);
        o.w = (((q.y >> 8) & 3u) << 30) | ((tok22 & 0x200000u) ? PT_TOKEN_POOLED : 0u) | (tok22 & 0x1FFFFFu);
        reinterpret_cast<uint4*>(out)[i] = o;
    }
}
__global__ void expand_mark_c16_kernel(const pt_mark_c16* __restrict__ in, pt_mark_rec* __restrict__ out, unsigned long long n) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(in + i));
        // pt_mark_rec: {ctr, actor | kind << 16 | bounds << 24, start_ctr, end_ctr} {start_actor | end_actor << 16, attr, arrival, 0}
        uint4 a, b;
        a.x = q.x & 0xFFFFu;
        a.y = (q.w & 0xFu) | (((q.w >> 12) & 7u) << 16) | (((q.w >> 15) & 0xFu) << 24);
        a.z = q.x >> 16; a.w = q.y & 0xFFFFu;
        b.x = ((q.w >> 4) & 0xFu) | (((q.w >> 8) & 0xFu) << 16);
        b.y = q.z; b.z = q.y >> 16; b.w = 0;
        reinterpret_cast<uint4*>(out)[2 * i] = a; reinterpret_cast<uint4*>(out)[2 * i + 1] = b;
    }
}

// ---- output compaction (download path) ---------------------------------------------------------------------------------
// The merge kernels write each log's tokens / spans at offsets derived from the descriptors alone (capacity = n_insdel
// tokens, min(n_insdel, 2 n_mark + 1) spans), typically a few percent full (c4: 5 visible characters per 500-record log).
// Before the device -> host copy the used prefixes are packed back to back: exclusive scan of (n_visible, n_spans) over
// the logs (block sums -> one-block scan -> offsets), then one warp per log copies its tokens and spans.
// The scan kernels take the per-log counts from a source functor: two channels (a, c) per log.  The JSON render
// (render_kernel.cuh) scans its per-log byte counts through the same kernels, on channel a only.
constexpr uint32_t kScanBlock = 1024;
struct MergedCounts {      // (n_visible, n_spans) of the logs that merged, 0 for the others
    const pt_log_result* __restrict__ res;
    __device__ void operator()(uint32_t i, unsigned long long& a, unsigned long long& c) const {
        if (res[i].status == 0) { a = res[i].n_visible; c = res[i].n_spans; }
    }
};
struct PlainCounts {       // a u64 count per log on channel a
    const unsigned long long* __restrict__ cnt;
    __device__ void operator()(uint32_t i, unsigned long long& a, unsigned long long&) const { a = cnt[i]; }
};
template <class Src>
__global__ void out_block_sums_kernel(Src src, uint32_t n, unsigned long long* __restrict__ bsum) {
    __shared__ unsigned long long sa[32], sb[32];
    const uint32_t i = blockIdx.x * kScanBlock + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long a = 0, c = 0;
    if (i < n) src(i, a, c);
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    if (lane == 0) { sa[warp] = a; sb[warp] = c; }
    __syncthreads();
    if (warp == 0) {
        a = sa[lane]; c = sb[lane];
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
        if (lane == 0) { bsum[2 * blockIdx.x] = a; bsum[2 * blockIdx.x + 1] = c; }
    }
}
__global__ void out_scan_blocks_kernel(unsigned long long* bsum, uint32_t nb) {   // one block; exclusive scan in place, totals at [2 nb]
    __shared__ unsigned long long ca, cb;
    __shared__ unsigned long long wa[32], wb[32];
    if (threadIdx.x == 0) { ca = 0; cb = 0; }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = 0; base < nb; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long va = i < nb ? bsum[2 * i] : 0ull, vb = i < nb ? bsum[2 * i + 1] : 0ull;
        unsigned long long a = va, c = vb;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long ya = __shfl_up_sync(0xffffffffu, a, o), yb = __shfl_up_sync(0xffffffffu, c, o);
            if (lane >= (uint32_t)o) { a += ya; c += yb; }
        }
        if (lane == 31) { wa[warp] = a; wb[warp] = c; }
        __syncthreads();
        if (warp == 0) {
            unsigned long long x = wa[lane], y = wb[lane];
            const unsigned long long x0 = x, y0 = y;
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long yx = __shfl_up_sync(0xffffffffu, x, o), yy = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= (uint32_t)o) { x += yx; y += yy; }
            }
            wa[lane] = x - x0; wb[lane] = y - y0;
        }
        __syncthreads();
        const unsigned long long ea = ca + wa[warp] + a - va, eb = cb + wb[warp] + c - vb;
        if (i < nb) { bsum[2 * i] = ea; bsum[2 * i + 1] = eb; }
        __syncthreads();
        if (threadIdx.x == 1023) { ca = ea + va; cb = eb + vb; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { bsum[2 * nb] = ca; bsum[2 * nb + 1] = cb; }
}
template <class Src>   // soff may be null (one-channel sources)
__global__ void out_offsets_kernel(Src src, uint32_t n, const unsigned long long* __restrict__ bsum, uint32_t nb,
                                   unsigned long long* __restrict__ toff, unsigned long long* __restrict__ soff) {
    __shared__ unsigned long long wa[32], wb[32];
    const uint32_t i = blockIdx.x * kScanBlock + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long va = 0, vb = 0;
    if (i < n) src(i, va, vb);
    unsigned long long a = va, c = vb;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long ya = __shfl_up_sync(0xffffffffu, a, o), yb = __shfl_up_sync(0xffffffffu, c, o);
        if (lane >= (uint32_t)o) { a += ya; c += yb; }
    }
    if (lane == 31) { wa[warp] = a; wb[warp] = c; }
    __syncthreads();
    if (warp == 0) {
        unsigned long long x = wa[lane], y = wb[lane];
        const unsigned long long x0 = x, y0 = y;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long yx = __shfl_up_sync(0xffffffffu, x, o), yy = __shfl_up_sync(0xffffffffu, y, o);
            if (lane >= (uint32_t)o) { x += yx; y += yy; }
        }
        wa[lane] = x - x0; wb[lane] = y - y0;
    }
    __syncthreads();
    if (i < n) { toff[i] = bsum[2 * blockIdx.x] + wa[warp] + a - va; if (soff) soff[i] = bsum[2 * blockIdx.x + 1] + wb[warp] + c - vb; }
    if (i == 0) { toff[n] = bsum[2 * nb]; if (soff) soff[n] = bsum[2 * nb + 1]; }
}
__global__ void out_gather_kernel(const pt_log_result* __restrict__ res, uint32_t n, const uint64_t* __restrict__ cap_toff, const uint64_t* __restrict__ cap_soff,
                                  const unsigned long long* __restrict__ toff, const unsigned long long* __restrict__ soff,
                                  const uint32_t* __restrict__ text, const pt_span* __restrict__ spans, uint32_t* __restrict__ ctext, pt_span* __restrict__ cspans) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n; li += nwarps) {
        if (res[li].status != 0) continue;
        const uint32_t nv = res[li].n_visible, ns = res[li].n_spans;
        const uint32_t* ts = text + cap_toff[li]; uint32_t* td = ctext + toff[li];
        for (uint32_t k = lane; k < nv; k += 32) td[k] = ts[k];
        const uint4* ss = reinterpret_cast<const uint4*>(spans + cap_soff[li]); uint4* sd = reinterpret_cast<uint4*>(cspans + soff[li]);
        for (uint32_t k = lane; k < ns; k += 32) sd[k] = ss[k];
    }
}


// ---- admission pre-pass: Micromerge.applyChange's causal checks (reference src/micromerge.ts:499-511) for every log -------
// One warp per log, one lane per change, 32 changes per trip.  The reference keeps clock[actor] = seq of the last applied
// change; as long as every earlier change of the log was admitted that is the NUMBER of earlier changes by that actor, so
// each change can be checked independently against per-actor prefix counts (match_any groups inside the trip + running
// counts in shared memory), and the FIRST failing change — what the reference would throw at — is a min over lanes.
__global__ void admit_kernel(const pt_change_desc* __restrict__ cd, const pt_change_rec* __restrict__ ch, const pt_dep_rec* __restrict__ dp,
                             const pt_log_desc* __restrict__ desc, uint32_t n_logs, uint32_t maxR, uint32_t* __restrict__ admit, pt_log_result* __restrict__ results) {
    extern __shared__ uint32_t adm_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* cnt = adm_smem + (size_t)wib * 2 * maxR;      // changes admitted so far, per actor
    uint32_t* cmask = cnt + maxR;                           // lanes of the current trip, per actor
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t li = blockIdx.x * wpb + wib; li < n_logs; li += gridDim.x * wpb) {
        const pt_change_desc D = cd[li];
        const uint32_t R = desc[li].n_actors ? desc[li].n_actors : 1u;
        for (uint32_t a = lane; a < R; a += 32) { cnt[a] = 0; cmask[a] = 0; }
        __syncwarp();
        const pt_change_rec* c0 = ch + D.change_off; const pt_dep_rec* d0 = dp + D.dep_off;
        uint32_t fail_idx = 0xFFFFFFFFu, fail_code = 0;
        for (uint32_t base = 0; base < D.n_changes; base += 32) {
            const uint32_t k = base + lane;
            const bool valid = k < D.n_changes;
            uint4 r = make_uint4(0, 0, 0, 0);
            if (valid) r = __ldg(reinterpret_cast<const uint4*>(c0 + k));
            const uint32_t seq = r.x, actor = r.y & 0xFFFFu, n_deps = r.y >> 16, dep_off = r.z;
            const bool aok = valid && actor < R;
            const uint32_t a = aok ? actor : (0x10000u + lane);
            const uint32_t mask = __match_any_sync(0xffffffffu, a);
            const bool leader = (mask & lt) == 0;
            if (aok && leader) cmask[actor] = mask;
            __syncwarp();
            uint32_t code = 0;
            if (valid) {
                if (!aok) code = PT_LOG_BAD_OPID;
                else if (seq != cnt[actor] + __popc(mask & lt) + 1u) code = PT_LOG_SEQ_GAP;            // src/micromerge.ts:501-504
                else if (dep_off + n_deps > D.n_deps) code = PT_LOG_BAD_OPID;
                else for (uint32_t d = 0; d < n_deps; d++) {                                            // src/micromerge.ts:505-509
                    const pt_dep_rec q = d0[dep_off + d];
                    const uint32_t have = q.actor < R ? cnt[q.actor] + __popc(cmask[q.actor] & lt) : 0u;
                    if (have == 0 || have < q.seq) { code = PT_LOG_MISSING_DEP; break; }
                }
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, code != 0);
            if (bal) { const uint32_t f = __ffs(bal) - 1; fail_idx = base + f; fail_code = __shfl_sync(0xffffffffu, code, f); break; }
            __syncwarp();
            if (aok && leader) { cnt[actor] += __popc(mask); cmask[actor] = 0; }
            __syncwarp();
        }
        if (lane == 0) {
            admit[li] = fail_code;
            if (fail_code) { pt_log_result r{}; r.status = fail_code; r.n_elems = fail_idx; results[li] = r; }
        }
        __syncwarp();
    }
}


// ---- batched getListElementId (reference src/micromerge.ts:762-805) over the materialised element sequences ----------------
// One warp per query: ballot / popcount over the sequence words finds the k-th visible element; lookAfterTombstones then
// scans the run of tombstones that follows for the last one whose markOpsAfter slot is defined (bit 30).
__global__ void query_elements_kernel(const pt_elem_query* __restrict__ q, uint32_t n, const pt_log_result* __restrict__ res,
                                      const uint64_t* __restrict__ seq_off, const uint32_t* __restrict__ seq, uint32_t n_logs, uint32_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t k = warp; k < n; k += nwarps) {
        const pt_elem_query Q = q[k];
        uint32_t ans = PT_ELEM_NOT_FOUND;
        if (Q.log < n_logs && res[Q.log].status == 0) {
            const uint32_t N = res[Q.log].n_elems;
            const uint32_t* s = seq + seq_off[Q.log];
            uint32_t seen = 0, pos = 0xFFFFFFFFu;
            for (uint32_t b = 0; b < N && pos == 0xFFFFFFFFu; b += 32) {
                const uint32_t e = b + lane < N ? s[b + lane] : 0x80000000u;
                const uint32_t vis = __ballot_sync(0xffffffffu, !(e >> 31));
                const uint32_t c = __popc(vis);
                if (seen + c > Q.index) {
                    uint32_t m = vis;                                        // (index - seen)-th set bit
                    for (uint32_t r = Q.index - seen; r; r--) m &= m - 1;
                    pos = b + (__ffs(m) - 1);
                }
                seen += c;
            }
            if (pos != 0xFFFFFFFFu) {
                uint32_t best = pos;
                if (Q.flags & PT_QUERY_LOOK_AFTER_TOMBSTONES) {
                    bool open = true;
                    for (uint32_t b = pos + 1; b < N && open; b += 32) {
                        const uint32_t e = b + lane < N ? s[b + lane] : 0u;      // past the end counts as "not a tombstone"
                        const uint32_t live = __ballot_sync(0xffffffffu, !(e >> 31));
                        const uint32_t upto = live ? ((1u << (__ffs(live) - 1)) - 1u) : 0xFFFFFFFFu;    // tombstones before the next visible element
                        const uint32_t marked = __ballot_sync(0xffffffffu, (e >> 30) & 1u) & upto;
                        if (marked) best = b + (31 - __clz(marked));
                        open = live == 0;
                    }
                }
                ans = s[best] & 0x3FFFFFFFu;
            }
        }
        if (lane == 0) out[k] = ans;
    }
}

// ---- batched findListElement (reference src/micromerge.ts:731-755; resolveCursor :475 = .visible) -------------------------
// One warp per query, the inverse of query_elements_kernel.  Stage 1 finds the element's insert record: the log's ins/del
// records 32 per trip (coalesced 16-byte loads), first ballot hit (a log that merged OK has no duplicate insert opIds).
// Stage 2 finds the sequence word that names that record, 32 words per trip, and counts the visible elements before it:
// the running popcount of the live ballot plus the live lanes below the matching one.  O(n_insdel + n_elems) reads per
// query, like the reference's linear scan.
__global__ void find_elements_kernel(const pt_elem_ref* __restrict__ q, uint32_t n, const pt_log_desc* __restrict__ desc,
                                     const pt_insdel_rec* __restrict__ insdel, const pt_log_result* __restrict__ res,
                                     const uint64_t* __restrict__ seq_off, const uint32_t* __restrict__ seq, uint32_t n_logs,
                                     pt_elem_pos* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t k = warp; k < n; k += nwarps) {
        const uint4 Q = __ldg(reinterpret_cast<const uint4*>(q + k));
        const uint32_t log = Q.x, ctr = Q.y, actor = Q.z & 0xFFFFu;
        uint4 ans = make_uint4(PT_ELEM_NOT_FOUND, 0u, PT_ELEM_NOT_FOUND, 0u);      // index, visible, record, flags
        if (log >= n_logs || res[log].status != PT_LOG_OK) {
            ans.w = PT_ELEM_LOG_FAILED;
        } else if (ctr != 0) {
            const pt_log_desc D = desc[log];
            const uint4* r = reinterpret_cast<const uint4*>(insdel + D.insdel_off);
            uint32_t rec = PT_ELEM_NOT_FOUND;
            for (uint32_t b = 0; b < D.n_insdel; b += 32) {
                bool hit = false;
                if (b + lane < D.n_insdel) {
                    const uint4 w = __ldg(r + b + lane);
                    hit = w.x == ctr && (w.z & 0xFFFFu) == actor && PT_PAYLOAD_KIND(w.w) == PT_KIND_INSERT;
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, hit);
                if (bal) { rec = b + __ffs(bal) - 1; break; }
            }
            if (rec != PT_ELEM_NOT_FOUND) {
                const uint32_t N = res[log].n_elems;
                const uint32_t* s = seq + seq_off[log];
                uint32_t seen = 0;
                for (uint32_t b = 0; b < N; b += 32) {
                    const bool valid = b + lane < N;
                    const uint32_t e = valid ? s[b + lane] : 0u;
                    const uint32_t live = __ballot_sync(0xffffffffu, valid && !(e >> 31));
                    const uint32_t match = __ballot_sync(0xffffffffu, valid && (e & 0x3FFFFFFFu) == rec);
                    if (match) {
                        const uint32_t m = __ffs(match) - 1;
                        const uint32_t em = __shfl_sync(0xffffffffu, e, m);
                        ans = make_uint4(b + m, seen + __popc(live & ((1u << m) - 1u)), rec,
                                         ((em >> 31) ? PT_ELEM_DELETED : 0u) | (((em >> 30) & 1u) ? PT_ELEM_AFTER_DEFINED : 0u));
                        break;
                    }
                    seen += __popc(live);
                }
            }
        }
        if (lane == 0) reinterpret_cast<uint4*>(out)[k] = ans;
    }
}

}  // namespace

struct pt_batch {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 0;
    pt_limits limits{};
    // batch
    bool have_batch = false, merged = false, adopted = false;
    uint32_t n_logs = 0;
    uint64_t n_insdel = 0, n_mark = 0, n_text = 0, n_span = 0, pool_cap = 0;
    std::vector<pt_log_desc> h_desc;
    std::vector<uint64_t> h_text_off, h_span_off;
    std::vector<uint32_t> h_order;
    uint32_t bin_first[kNumBins + 1] = {0};
    uint32_t warp_packed = 0;               // bin 0: the first warp_packed logs use the packed3 id table (3 actors, <= 1022 records)
    uint32_t warp_compact = 0;              // bin 0: the next warp_compact logs use the compact id table
    uint32_t team_count = 0;                // bin 0: the last team_count logs run on the team kernel
    uint32_t n_spill = 0, slab_slots = 0;   // logs that can spill / slab slots allocated
    size_t bin_slab[kNumBins] = {0};
    size_t retry_slab = 0;
    // device
    DevBuf d_runs, d_tokens, d_run_off, d_tok_off, d_cins, d_cmarks;
    DevBuf d_desc, d_insdel, d_marks, d_order, d_counters, d_results, d_text_off, d_span_off, d_text, d_spans, d_pool, d_slab, d_retry, d_seq;
    DevBuf d_bsum, d_ctoff, d_csoff, d_ctext, d_cspans;   // download path: packed outputs + their offsets ([n_logs + 1])
    DevBuf d_cdesc, d_changes, d_deps, d_admit;           // admission pre-pass (optional change table)
    DevBuf d_patch_recs, d_patch_items, d_patch_status;   // PT_FLAG_EMIT_PATCHES
    HostBuf h_patch_recs, h_patch_items, h_patch_status, h_patch_misc;
    DevBuf d_jval, d_jvoff, d_jlink, d_jloff, d_jcom, d_jcoff;          // pt_batch_render_json: the caller's pools,
    DevBuf d_jsize, d_jbsum, d_joff, d_jmiss, d_jbytes;                 // per-log sizes, scan, offsets, missing-entry key, output
    HostBuf h_joff, h_jbytes, h_jmisc;
    uint64_t patch_cap = 0;
    uint32_t patch_smem = 0;
    bool have_changes = false;
    uint32_t adm_maxR = 1;
    const pt_insdel_rec* dp_insdel = nullptr;
    const pt_mark_rec* dp_marks = nullptr;
    // pinned host
    HostBuf h_stage, h_results, h_text, h_spans, h_pool, h_misc, h_seq, h_ctoff, h_csoff;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaStream_t side = nullptr, launch_stream = nullptr;   // side: the CTA-per-log bins' own launches run beside the warp / team kernels
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    uint64_t launches = 0;
    cudaGraphExec_t graph_exec = nullptr;   // the merge sequence of the current batch, captured once
    bool graph_ok = false, graph_tried = false;
    uint32_t merges_since_upload = 0;
    bool dl_begun = false;
    uint32_t kernels_per_merge = 0;
    uint64_t pool_used_host = 0;
};

namespace {

// PT_BINS="max_recs:block:smem_kb:ctas_per_sm,..." (4 entries, ascending; last max_recs ignored) overrides the CTA-per-log bins;
// PT_WARP="max_recs:warps_per_cta:slice_kb:ctas_per_sm" overrides the warp-per-log bin, PT_WARP=0 disables it (tuning)
const BinCfg kDefaultBins[kNumBins] = {kBins[0], kBins[1], kBins[2], kBins[3], kBins[4]};
void load_bins_from_env() {
    // re-read whenever the variables change (tests flip PT_WARP between uploads to cross-check the two kernels)
    static std::string last = "\x01";
    const char* we = getenv("PT_WARP"); const char* be = getenv("PT_BINS"); const char* fe = getenv("PT_WARP_FORCE"); const char* te0 = getenv("PT_TEAM");
    const std::string cur = std::string(we ? we : "") + "|" + (be ? be : "") + "|" + (fe ? fe : "") + "|" + (te0 ? te0 : "");
    if (cur == last) return;
    last = cur;
    for (int i = 0; i < kNumBins; i++) kBins[i] = kDefaultBins[i];
    g_warp_bin = true; g_warp_force = fe && atoi(fe) != 0;
    { const char* te = getenv("PT_TEAM"); g_team_bin = !(te && atoi(te) == 0); }
    if (const char* w = getenv("PT_WARP")) {
        unsigned long a, wp, sl, ct;
        if (sscanf(w, "%lu:%lu:%lu:%lu", &a, &wp, &sl, &ct) == 4 && (wp == 2 || wp == 4 || wp == 6 || wp == 8 || wp == 12 || wp == 16)) {
            if (sl < 256) sl *= 1024;                    // slice: KB, or bytes when >= 256
            sl &= ~(unsigned long)15;
            if (sl * wp <= 227 * 1024) kBins[0] = BinCfg{(uint32_t)a, (int)wp * 32, (uint32_t)sl, (int)ct};
        }
        else if (atoi(w) == 0) { g_warp_bin = false; g_team_bin = false; }      // PT_WARP=0: CTA-per-log kernels only
    }
    const char* e = getenv("PT_BINS");
    if (!e) return;
    BinCfg tmp[kNumBins];
    int k = 1;
    const char* p = e;
    while (k < kNumBins && *p) {
        unsigned long a, bl, sm, ct; int used = 0;
        if (sscanf(p, "%lu:%lu:%lu:%lu%n", &a, &bl, &sm, &ct, &used) != 4) return;
        if (bl != 32 && bl != 64 && bl != 128 && bl != 256 && bl != 512 && bl != 1024) return;
        tmp[k++] = BinCfg{(uint32_t)a, (int)bl, (uint32_t)(sm * 1024), (int)ct};
        p += used; if (*p == ',') p++;
    }
    if (k != kNumBins) return;
    tmp[kNumBins - 1].max_recs = 0xFFFFFFFFu;
    for (int i = 1; i < kNumBins; i++) kBins[i] = tmp[i];
}

int plan_batch(pt_batch* b, const pt_packed_ops* ops) {
    load_bins_from_env();
    b->n_logs = ops->n_logs;
    b->n_insdel = ops->n_insdel_total;
    b->n_mark = ops->n_mark_total;
    b->h_desc.assign(ops->logs, ops->logs + ops->n_logs);
    b->h_text_off.resize(b->n_logs); b->h_span_off.resize(b->n_logs);
    uint64_t to = 0, so = 0, ncomment_bound = 0;
    uint32_t n_packed = 0, n_compact = 0, n_team = 0, n_spill = 0;
    std::vector<uint8_t> is_team(ops->n_logs, 0);
    std::vector<uint32_t> bins[kNumBins];
    for (int k = 0; k < kNumBins; k++) b->bin_slab[k] = 0;
    for (uint32_t i = 0; i < b->n_logs; i++) {
        const pt_log_desc& L = b->h_desc[i];
        if (L.insdel_off + L.n_insdel > b->n_insdel || L.mark_off + L.n_mark > b->n_mark) { g_last_error = "log descriptor out of range"; return PT_ERR_INVALID; }
        b->h_text_off[i] = to; b->h_span_off[i] = so;
        to += L.n_insdel;
        so += std::min<uint64_t>(L.n_insdel, 2ull * L.n_mark + 1);
        ncomment_bound += L.n_mark;
        uint64_t recs = (uint64_t)L.n_insdel + L.n_mark;
        uint64_t KS = (uint64_t)L.max_ctr * (L.n_actors ? L.n_actors : 1);
        int bin = 1; while (recs > kBins[bin].max_recs) bin++;
        // typical shared-memory need (runs ~ n/6, segments ~ min(2m, n/2)); a wrong guess only costs a device-side deferral
        {
            const uint64_t I = (L.n_insdel < 32000 && L.n_mark < 32000) ? 2 : 4, n_ = L.n_insdel, m_ = L.n_mark;
            // id table + bitmaps / run offsets (~1.4 B per record) + the larger of the run-tree temporaries (~5 B per record
            // for typing-heavy logs) and the mark tables (per-op arrays + ~18 B per elementary segment)
            const uint64_t seg = std::min<uint64_t>(2 * m_ + 2, n_ / 2 + 2);
            const uint64_t typical = KS * I + (14 * n_) / 10 + std::max<uint64_t>(5 * n_, m_ ? m_ * (6 * I + 13) + 18 * seg : 0) + 2048;
            while (bin < kNumBins - 1 && typical > kBins[bin].smem) bin++;
        }
        // short logs: one warp per log (16-bit keys and indices).  Footprint estimate: id table (compact form with >= 3
        // actors: one slot per counter + overflow) + bitmaps + run-tree temporaries for ~ n/3 runs; a low guess only costs
        // a device-side deferral
        if (g_warp_bin && !(b->limits.flags & PT_FLAG_EMIT_SEQUENCE) && recs <= kBins[0].max_recs && KS < 0xFFFFull) {
            const uint64_t R_ = L.n_actors ? L.n_actors : 1, n_ = L.n_insdel;
            const bool packed3 = R_ == 3 && n_ <= 1022;
            const uint64_t idbytes = packed3 ? 4ull * L.max_ctr : (R_ >= 3 && R_ <= 30 && n_ <= 2046) ? 2ull * L.max_ctr + 512 : 2 * KS;
            // packed3 (three concurrent replicas): per-word state 16 B per 32 records, ~14 B per run for ~ n/4 runs, key bitmap + prefix
            const uint64_t rest = packed3 ? n_ / 2 + 32 + 14 * (n_ / 4) + (KS / 32 + 2) * 6 + 512 : n_ / 2 + 16 * n_ / 3 + 1024;
            if (g_warp_force || idbytes + rest <= kBins[0].smem) bin = 0;
        }
        if (bin == 0) {   // bin 0's warp launches: packed3 id table (3 actors) / compact (>= 3 actors) / direct
            const uint64_t R_ = L.n_actors ? L.n_actors : 1;
            if (R_ == 3 && L.n_insdel <= 1022) n_packed++;
            else if (R_ >= 3 && R_ <= 30 && L.n_insdel <= 2046) n_compact++;
        } else if (g_team_bin && !(b->limits.flags & PT_FLAG_EMIT_SEQUENCE) && L.n_mark == 0 && KS < 0xFFFFull && L.n_insdel < 0xFFFFu &&
                   (3ull * L.n_insdel) / 4 + 2 * KS + 2ull * L.n_insdel + 1024 <= kTeamSmem) {
            // medium logs without mark ops: a team of 8 warps per log, 4 logs per SM (team_kernel.cuh); rides in bin 0's list
            bin = 0; is_team[i] = 1; n_team++;
        }
        bins[bin].push_back(i);
        if (KS > 0x7FFFFFFFull) { g_last_error = "max_ctr * n_actors too large; re-rank counters densely on the host"; return PT_ERR_INVALID; }
        {   // only a log whose worst-case working set exceeds the largest shared-memory budget can ever spill to the global slab
            const size_t worst = arena_worst_bytes(L.n_insdel, L.n_mark, KS);
            if (worst > kBins[kNumBins - 1].smem) { b->bin_slab[kNumBins - 1] = std::max(b->bin_slab[kNumBins - 1], worst); n_spill++; }
        }
    }
    b->n_text = to; b->n_span = so;
    // default pool: 4 entries per mark op (+slack) fits the generated workloads (c3, the densest, needs < 2); a batch that needs
    // more reports its exact demand and merges again (BatchEngine.run), so the pool need not be sized for the worst case
    b->pool_cap = b->limits.comment_pool_entries ? b->limits.comment_pool_entries : 4ull * ncomment_bound + 1024;
    b->h_order.clear();
    for (int k = 0; k < kNumBins; k++) {
        b->bin_first[k] = (uint32_t)b->h_order.size();
        auto& v = bins[k];
        // bin 0's list: [warp kernel, packed3 id table | compact id table | direct id table | team kernel]
        auto cat = [&](uint32_t x) { if (is_team[x]) return 3; const pt_log_desc& D = b->h_desc[x]; const uint32_t R_ = D.n_actors ? D.n_actors : 1;
                                     return (R_ == 3 && D.n_insdel <= 1022) ? 0 : (R_ >= 3 && R_ <= 30 && D.n_insdel <= 2046) ? 1 : 2; };
        std::stable_sort(v.begin(), v.end(), [&](uint32_t x, uint32_t y) {
            if (k == 0) { const int cx = cat(x), cy = cat(y); if (cx != cy) return cx < cy; }
            return (uint64_t)b->h_desc[x].n_insdel + b->h_desc[x].n_mark > (uint64_t)b->h_desc[y].n_insdel + b->h_desc[y].n_mark; });
        b->h_order.insert(b->h_order.end(), v.begin(), v.end());
    }
    b->bin_first[kNumBins] = (uint32_t)b->h_order.size();
    b->warp_packed = n_packed; b->warp_compact = n_compact; b->team_count = n_team; b->n_spill = n_spill;
    return PT_OK;
}

int alloc_and_upload_plan(pt_batch* b) {
    int rc;
    const size_t n = b->n_logs;
    if ((rc = b->d_desc.reserve(std::max<size_t>(1, n) * sizeof(pt_log_desc)))) return rc;
    if ((rc = b->d_order.reserve(std::max<size_t>(1, n) * 4))) return rc;
    if ((rc = b->d_counters.reserve(256))) return rc;   // [0,64) stats | [64,72) pool cursor | [128,176) work/deferral counters
    if ((rc = b->d_results.reserve(std::max<size_t>(1, n) * sizeof(pt_log_result)))) return rc;
    if ((rc = b->d_text_off.reserve(std::max<size_t>(1, n) * 8))) return rc;
    if ((rc = b->d_span_off.reserve(std::max<size_t>(1, n) * 8))) return rc;
    if ((rc = b->d_text.reserve(std::max<uint64_t>(1, b->n_text) * 4))) return rc;
    if ((b->limits.flags & PT_FLAG_EMIT_SEQUENCE) && (rc = b->d_seq.reserve(std::max<uint64_t>(1, b->n_text) * 4))) return rc;
    if ((rc = b->d_spans.reserve(std::max<uint64_t>(1, b->n_span) * sizeof(pt_span)))) return rc;
    if ((rc = b->d_pool.reserve(std::max<uint64_t>(1, b->pool_cap) * 4))) return rc;
    if ((rc = b->d_retry.reserve(std::max<size_t>(1, n) * 4 * kNumBins + 16))) return rc;
    if (b->limits.flags & PT_FLAG_EMIT_PATCHES) {
        b->patch_cap = b->limits.patch_pool_items ? b->limits.patch_pool_items : 4ull * (b->n_insdel + b->n_mark) + 1024;
        if ((rc = b->d_patch_recs.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_patch_rec)))) return rc;
        if ((rc = b->d_patch_items.reserve(std::max<uint64_t>(1, b->patch_cap) * sizeof(pt_patch_item)))) return rc;
        if ((rc = b->d_patch_status.reserve(std::max<size_t>(1, n) * 4))) return rc;
        // one warp per CTA; shared memory = the largest footprint among the logs, capped (larger logs are left to the host)
        uint64_t need_max = 4096;
        for (uint32_t i = 0; i < b->n_logs; i++) {
            const pt_log_desc& L = b->h_desc[i];
            const uint64_t KS = (uint64_t)L.max_ctr * (L.n_actors ? L.n_actors : 1);
            const uint64_t need = ((KS * 2 + 15) & ~15ull) + 3 * (((uint64_t)L.n_insdel * 2 + 15) & ~15ull) / 1 + (((uint64_t)L.n_insdel * 4 + 15) & ~15ull) +
                                  6 * (((uint64_t)L.n_mark * 4 + 15) & ~15ull) + (((uint64_t)L.n_mark * 2 + 15) & ~15ull) + 256;
            if (need <= 200 * 1024) need_max = std::max(need_max, need);
        }
        b->patch_smem = (uint32_t)((need_max + 1023) & ~1023ull);
    }
    // spill slab: one slot per CTA that can ever spill = min(logs that can spill, CTAs of the last bin); a batch with one huge
    // log no longer multiplies its worst case by the whole grid
    const size_t slab_max = b->bin_slab[kNumBins - 1];
    b->slab_slots = (uint32_t)std::min<size_t>(b->n_spill, (size_t)b->num_sms * kBins[kNumBins - 1].ctas_per_sm);
    const size_t slab_total = (size_t)b->slab_slots * slab_max;
    b->retry_slab = slab_max;
    if ((rc = b->d_slab.reserve(std::max<size_t>(slab_total, 16)))) return rc;
    // stage the small host-derived arrays through pinned memory
    size_t stage = n * (sizeof(pt_log_desc) + 4 + 8 + 8) + 64;
    if ((rc = b->h_stage.reserve(stage))) return rc;
    char* s = (char*)b->h_stage.p;
    if (n) {
        memcpy(s, b->h_desc.data(), n * sizeof(pt_log_desc));
        PT_CUDA(cudaMemcpyAsync(b->d_desc.p, s, n * sizeof(pt_log_desc), cudaMemcpyHostToDevice, b->stream)); s += n * sizeof(pt_log_desc);
        memcpy(s, b->h_order.data(), n * 4);
        PT_CUDA(cudaMemcpyAsync(b->d_order.p, s, n * 4, cudaMemcpyHostToDevice, b->stream)); s += n * 4;
        memcpy(s, b->h_text_off.data(), n * 8);
        PT_CUDA(cudaMemcpyAsync(b->d_text_off.p, s, n * 8, cudaMemcpyHostToDevice, b->stream)); s += n * 8;
        memcpy(s, b->h_span_off.data(), n * 8);
        PT_CUDA(cudaMemcpyAsync(b->d_span_off.p, s, n * 8, cudaMemcpyHostToDevice, b->stream)); s += n * 8;
    }
    return PT_OK;
}

// counters: [0,kNumBins) work-queue heads of the bins' own lists, [kNumBins, 2k) heads of the retry launches,
// [2k, 3k) number of logs deferred INTO bin k (list k of d_retry)
template <int BLOCK>
int launch_bin_t(pt_batch* b, int k, ptk::BatchParams P, bool retry) {
    const BinCfg& cfg = kBins[k];
    uint32_t cnt = retry ? b->n_logs : b->bin_first[k + 1] - b->bin_first[k];
    uint32_t grid = (uint32_t)std::min<size_t>(cnt, (size_t)b->num_sms * cfg.ctas_per_sm);
    uint32_t* counters = (uint32_t*)((char*)b->d_counters.p + 128);
    uint32_t* lists = (uint32_t*)b->d_retry.p;
    if (retry) {
        P.order = lists + (size_t)k * b->n_logs; P.n_work = 0; P.n_work_dev = counters + 2 * kNumBins + k;
        P.work_counter = counters + kNumBins + k;
    } else {
        P.order = (const uint32_t*)b->d_order.p + b->bin_first[k]; P.n_work = cnt; P.n_work_dev = nullptr;
        P.work_counter = counters + k;
    }
    const bool last = k == kNumBins - 1;
    P.slab_bytes = last ? b->retry_slab : 0;
    if (retry) P.slab_counter += 1;      // the two launches of the last bin run one after the other: each counts its slots from zero
    P.retry_list = last ? nullptr : lists + (size_t)(k + 1) * b->n_logs;
    P.retry_count = last ? nullptr : counters + 2 * kNumBins + (k + 1);
    P.smem_arena_bytes = cfg.smem;
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_kernel<BLOCK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smem));
    ptk::merge_logs_kernel<BLOCK><<<grid, BLOCK, cfg.smem, b->launch_stream>>>(P);
    PT_CUDA(cudaGetLastError());
    b->launches++;
    return PT_OK;
}
template <int WARPS, int IDM>
int launch_warp_range(pt_batch* b, ptk::BatchParams P, uint32_t first, uint32_t cnt, uint32_t counter_slot) {
    if (!cnt) return PT_OK;
    const BinCfg& cfg = kBins[0];
    const uint32_t per_cta = WARPS * ptk::kWarpGrab;
    const uint32_t grid = (uint32_t)std::min<size_t>((cnt + per_cta - 1) / per_cta, (size_t)b->num_sms * cfg.ctas_per_sm);
    uint32_t* counters = (uint32_t*)((char*)b->d_counters.p + 128);
    uint32_t* lists = (uint32_t*)b->d_retry.p;
    P.order = (const uint32_t*)b->d_order.p + b->bin_first[0] + first; P.n_work = cnt; P.n_work_dev = nullptr;
    P.work_counter = counters + counter_slot;
    P.slab_bytes = 0;
    P.retry_list = lists + (size_t)1 * b->n_logs;        // deferrals go to the first CTA-per-log bin
    P.retry_count = counters + 2 * kNumBins + 1;
    P.smem_arena_bytes = cfg.smem;                       // per warp
    const int smem = (int)(cfg.smem * WARPS);
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_warp_kernel<WARPS, IDM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ptk::merge_logs_warp_kernel<WARPS, IDM><<<grid, WARPS * 32, smem, b->launch_stream>>>(P);
    PT_CUDA(cudaGetLastError());
    b->launches++;
    return PT_OK;
}
int launch_team_range(pt_batch* b, ptk::BatchParams P, uint32_t first, uint32_t cnt) {
    if (!cnt) return PT_OK;
    const uint32_t grid = (uint32_t)std::min<size_t>(cnt, (size_t)b->num_sms * 4);
    uint32_t* counters = (uint32_t*)((char*)b->d_counters.p + 128);
    uint32_t* lists = (uint32_t*)b->d_retry.p;
    P.order = (const uint32_t*)b->d_order.p + b->bin_first[0] + first; P.n_work = cnt; P.n_work_dev = nullptr;
    P.work_counter = counters + 3 * kNumBins + 1;
    P.slab_bytes = 0;
    P.retry_list = lists + (size_t)3 * b->n_logs;        // a log that does not fit goes to the 512-thread CTA bin (and on from there)
    P.retry_count = counters + 2 * kNumBins + 3;
    P.smem_arena_bytes = kTeamSmem;
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_team_kernel<kTeamWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTeamSmem));
    ptk::merge_logs_team_kernel<kTeamWarps><<<grid, kTeamWarps * 32, kTeamSmem, b->launch_stream>>>(P);
    PT_CUDA(cudaGetLastError());
    b->launches++;
    return PT_OK;
}
template <int WARPS>
int launch_warp_bin_t(pt_batch* b, const ptk::BatchParams& P) {
    const uint32_t cnt = b->bin_first[1] - b->bin_first[0] - b->team_count;
    const uint32_t np = b->warp_packed, nc = b->warp_compact;
    int rc = launch_warp_range<WARPS, ptk::kIdPacked3>(b, P, 0, np, 3 * kNumBins + 2);
    if (rc) return rc;
    if ((rc = launch_warp_range<WARPS, ptk::kIdCompact>(b, P, np, nc, 0))) return rc;
    if ((rc = launch_warp_range<WARPS, ptk::kIdDirect>(b, P, np + nc, cnt - np - nc, 3 * kNumBins))) return rc;
    return launch_team_range(b, P, cnt, b->team_count);
}
int launch_bin(pt_batch* b, int k, const ptk::BatchParams& P, bool retry) {
    if (!retry && b->bin_first[k + 1] == b->bin_first[k]) return PT_OK;
    if (k == 0) {
        switch (kBins[0].block / 32) {
            case 2: return launch_warp_bin_t<2>(b, P);
            case 4: return launch_warp_bin_t<4>(b, P);
            case 6: return launch_warp_bin_t<6>(b, P);
            case 8: return launch_warp_bin_t<8>(b, P);
            case 12: return launch_warp_bin_t<12>(b, P);
            default: return launch_warp_bin_t<16>(b, P);
        }
    }
    switch (kBins[k].block) {
        case 32: return launch_bin_t<32>(b, k, P, retry);
        case 64: return launch_bin_t<64>(b, k, P, retry);
        case 128: return launch_bin_t<128>(b, k, P, retry);
        case 256: return launch_bin_t<256>(b, k, P, retry);
        case 512: return launch_bin_t<512>(b, k, P, retry);
        default: return launch_bin_t<1024>(b, k, P, retry);
    }
}

}  // namespace

extern "C" {

int pt_batch_create(int device, const pt_limits* limits, void* cuda_stream, pt_batch** out) {
    if (!out) return PT_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0 || device < 0 || device >= count) {
        g_last_error = e != cudaSuccess ? cudaGetErrorString(e) : "no such CUDA device (this engine has no CPU fallback)";
        return PT_ERR_NO_DEVICE;
    }
    PT_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    PT_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) { g_last_error = "device is not sm_90-class (kernels are built for sm_90a only)"; return PT_ERR_NO_DEVICE; }
    pt_batch* b = new pt_batch();
    b->device = device; b->stream = (cudaStream_t)cuda_stream; b->num_sms = prop.multiProcessorCount;
    if (limits) b->limits = *limits;
    if (b->limits.flags & PT_FLAG_EMIT_PATCHES) b->limits.flags |= PT_FLAG_EMIT_SEQUENCE;
    if (cudaEventCreate(&b->ev0) != cudaSuccess || cudaEventCreate(&b->ev1) != cudaSuccess) { delete b; g_last_error = "cudaEventCreate failed"; return PT_ERR_CUDA; }
    if (b->stream != nullptr) {          // fork / join needs a real stream (not the legacy default stream)
        if (cudaStreamCreateWithFlags(&b->side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&b->ev_join, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); b->side = nullptr; }
    }
    b->launch_stream = b->stream;
    *out = b;
    return PT_OK;
}

static int upload_common(pt_batch* b, const pt_packed_ops* ops, bool adopt) {
    if (!b || !ops || (ops->n_logs && !ops->logs)) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));            // the staging buffer and the device arrays of the previous batch are reused
    b->have_batch = false; b->merged = false;
    if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }
    b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0; b->dl_begun = false; b->have_changes = false;
    int rc = plan_batch(b, ops);
    if (rc) return rc;
    if ((rc = alloc_and_upload_plan(b))) return rc;
    if (adopt) {
        b->dp_insdel = ops->insdel; b->dp_marks = ops->marks; b->adopted = true;
    } else {
        if ((rc = b->d_insdel.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_insdel_rec)))) return rc;
        if ((rc = b->d_marks.reserve(std::max<uint64_t>(1, b->n_mark) * sizeof(pt_mark_rec)))) return rc;
        if (b->n_insdel) PT_CUDA(cudaMemcpyAsync(b->d_insdel.p, ops->insdel, b->n_insdel * sizeof(pt_insdel_rec), cudaMemcpyHostToDevice, b->stream));
        if (b->n_mark) PT_CUDA(cudaMemcpyAsync(b->d_marks.p, ops->marks, b->n_mark * sizeof(pt_mark_rec), cudaMemcpyHostToDevice, b->stream));
        b->dp_insdel = (const pt_insdel_rec*)b->d_insdel.p; b->dp_marks = (const pt_mark_rec*)b->d_marks.p; b->adopted = false;
        // pageable caller buffers may be freed on return: finish the copies now (pinned ones stay asynchronous)
        auto pinned = [](const void* p) {
            cudaPointerAttributes a;
            if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
            return a.type == cudaMemoryTypeHost;
        };
        if (!((b->n_insdel == 0 || pinned(ops->insdel)) && (b->n_mark == 0 || pinned(ops->marks)))) PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    b->have_batch = true;
    return PT_OK;
}

int pt_batch_upload(pt_batch* b, const pt_packed_ops* ops) { return upload_common(b, ops, false); }

int pt_batch_upload_runs(pt_batch* b, const pt_packed_runs* rr) {
    if (!b || !rr || (rr->n_logs && (!rr->logs || !rr->run_off || !rr->tok_off))) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));            // the staging buffer and the device arrays of the previous batch are reused
    b->have_batch = false; b->merged = false;
    if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }
    b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0; b->dl_begun = false; b->have_changes = false;
    pt_packed_ops ops{rr->n_logs, rr->logs, nullptr, rr->n_insdel_total, nullptr, rr->n_mark_total};
    int rc = plan_batch(b, &ops);
    if (rc) return rc;
    if ((rc = alloc_and_upload_plan(b))) return rc;
    const size_t nl = rr->n_logs;
    const uint64_t n_runs = nl ? rr->run_off[nl] : 0, n_tok = nl ? rr->tok_off[nl] : 0;
    if ((rc = b->d_insdel.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_insdel_rec)))) return rc;
    if ((rc = b->d_marks.reserve(std::max<uint64_t>(1, b->n_mark) * sizeof(pt_mark_rec)))) return rc;
    if ((rc = b->d_runs.reserve(std::max<uint64_t>(1, n_runs) * sizeof(pt_run_rec)))) return rc;
    if ((rc = b->d_tokens.reserve(std::max<uint64_t>(1, n_tok) * 4))) return rc;
    if ((rc = b->d_run_off.reserve((nl + 1) * 8))) return rc;
    if ((rc = b->d_tok_off.reserve((nl + 1) * 8))) return rc;
    if (nl) {
        PT_CUDA(cudaMemcpyAsync(b->d_run_off.p, rr->run_off, (nl + 1) * 8, cudaMemcpyHostToDevice, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->d_tok_off.p, rr->tok_off, (nl + 1) * 8, cudaMemcpyHostToDevice, b->stream));
    }
    if (n_runs) PT_CUDA(cudaMemcpyAsync(b->d_runs.p, rr->runs, n_runs * sizeof(pt_run_rec), cudaMemcpyHostToDevice, b->stream));
    if (n_tok) PT_CUDA(cudaMemcpyAsync(b->d_tokens.p, rr->tokens, n_tok * 4, cudaMemcpyHostToDevice, b->stream));
    if (b->n_mark) PT_CUDA(cudaMemcpyAsync(b->d_marks.p, rr->marks, b->n_mark * sizeof(pt_mark_rec), cudaMemcpyHostToDevice, b->stream));
    if (nl) {
        const uint32_t threads = 128, warps_needed = (uint32_t)nl;
        const uint32_t grid = (uint32_t)std::min<uint64_t>(((uint64_t)warps_needed * 32 + threads - 1) / threads, (uint64_t)b->num_sms * 16);
        expand_runs_kernel<<<grid, threads, 0, b->stream>>>((const pt_log_desc*)b->d_desc.p, (const unsigned long long*)b->d_run_off.p,
                                                          (const unsigned long long*)b->d_tok_off.p, (const pt_run_rec*)b->d_runs.p,
                                                          (const uint32_t*)b->d_tokens.p, (pt_insdel_rec*)b->d_insdel.p, (uint32_t)nl);
        PT_CUDA(cudaGetLastError());
        b->launches++;
    }
    b->dp_insdel = (const pt_insdel_rec*)b->d_insdel.p; b->dp_marks = (const pt_mark_rec*)b->d_marks.p; b->adopted = false;
    auto pinned = [](const void* p) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return a.type == cudaMemoryTypeHost;
    };
    if (!((n_runs == 0 || pinned(rr->runs)) && (n_tok == 0 || pinned(rr->tokens)) && (b->n_mark == 0 || pinned(rr->marks)) && (nl == 0 || (pinned(rr->run_off) && pinned(rr->tok_off)))))
        PT_CUDA(cudaStreamSynchronize(b->stream));
    b->have_batch = true;
    return PT_OK;
}

int pt_compress_runs(const pt_packed_ops* ops, uint64_t* run_off, uint64_t* tok_off, pt_run_rec* runs, uint32_t* tokens,
                     uint64_t* n_runs_out, uint64_t* n_tokens_out) {
    if (!ops || !run_off || !tok_off) return PT_ERR_INVALID;
    uint64_t nr = 0, nt = 0;
    for (uint32_t li = 0; li < ops->n_logs; li++) {
        const pt_log_desc& L = ops->logs[li];
        const pt_insdel_rec* r = ops->insdel + L.insdel_off;
        run_off[li] = nr; tok_off[li] = nt;
        uint32_t i = 0;
        while (i < L.n_insdel) {
            const uint32_t kind = PT_PAYLOAD_KIND(r[i].payload);
            uint32_t j = i + 1;
            if (kind == PT_KIND_INSERT) {
                while (j < L.n_insdel && PT_PAYLOAD_KIND(r[j].payload) == PT_KIND_INSERT && r[j].actor == r[i].actor && r[j].ctr == r[j - 1].ctr + 1 &&
                       r[j].ref_ctr == r[j - 1].ctr && r[j].ref_actor == r[j - 1].actor && (j - i) < 0x3FFFFFFFu) j++;
            } else if (kind == PT_KIND_DELETE) {
                while (j < L.n_insdel && PT_PAYLOAD_KIND(r[j].payload) == PT_KIND_DELETE && r[j].actor == r[i].actor && r[j].ctr == r[j - 1].ctr + 1 &&
                       r[j].ref_ctr == r[j - 1].ref_ctr + 1 && r[j].ref_actor == r[i].ref_actor && (j - i) < 0x3FFFFFFFu) j++;
            }
            if (runs) { pt_run_rec q; q.ctr0 = r[i].ctr; q.ref_ctr = r[i].ref_ctr; q.actor = r[i].actor; q.ref_actor = r[i].ref_actor; q.kind_count = (kind << 30) | (j - i); runs[nr] = q; }
            if (kind == PT_KIND_INSERT) { if (tokens) for (uint32_t k = i; k < j; k++) tokens[nt + (k - i)] = PT_PAYLOAD_TOKEN(r[k].payload); nt += j - i; }
            nr++;
            i = j;
        }
    }
    run_off[ops->n_logs] = nr; tok_off[ops->n_logs] = nt;
    if (n_runs_out) *n_runs_out = nr;
    if (n_tokens_out) *n_tokens_out = nt;
    return PT_OK;
}
int pt_batch_adopt_device(pt_batch* b, const pt_packed_ops* ops) { return upload_common(b, ops, true); }

int pt_compact_ops(const pt_packed_ops* ops, pt_insdel_c8* io, pt_mark_c16* mo, int threads) {
    if (!ops || (ops->n_insdel_total && !io) || (ops->n_mark_total && !mo)) return PT_ERR_INVALID;
    for (uint32_t i = 0; i < ops->n_logs; i++) {
        const pt_log_desc& L = ops->logs[i];
        if (L.max_ctr >= 65536u || L.n_insdel >= 65536u || L.n_actors > 16u) { g_last_error = "log not representable in the compact wire format"; return PT_ERR_INVALID; }
    }
    int T = threads > 0 ? threads : (int)std::max(1u, std::thread::hardware_concurrency());
    std::atomic<int> bad{0};
    auto work = [&](int t) {
        const uint64_t n = ops->n_insdel_total, a = n * t / T, b2 = n * (t + 1) / T;
        for (uint64_t k = a; k < b2; k++) {
            const pt_insdel_rec& r = ops->insdel[k];
            const uint32_t tok = PT_PAYLOAD_TOKEN(r.payload), val = tok & (PT_TOKEN_POOLED - 1);
            if (val >= 0x200000u) bad = 1;
            pt_insdel_c8 o; o.ctr = (uint16_t)r.ctr; o.ref_ctr = (uint16_t)r.ref_ctr;
            o.w = (r.actor & 0xFu) | ((r.ref_actor & 0xFu) << 4) | (PT_PAYLOAD_KIND(r.payload) << 8) | (((tok & PT_TOKEN_POOLED ? 0x200000u : 0u) | (val & 0x1FFFFFu)) << 10);
            io[k] = o;
        }
        const uint64_t m = ops->n_mark_total, c = m * t / T, d = m * (t + 1) / T;
        for (uint64_t k = c; k < d; k++) {
            const pt_mark_rec& r = ops->marks[k];
            if (r.arrival >= 65536u) bad = 1;
            pt_mark_c16 o; o.ctr = (uint16_t)r.ctr; o.start_ctr = (uint16_t)r.start_ctr; o.end_ctr = (uint16_t)r.end_ctr; o.arrival = (uint16_t)r.arrival; o.attr = r.attr;
            o.w = (r.actor & 0xFu) | ((r.start_actor & 0xFu) << 4) | ((r.end_actor & 0xFu) << 8) | ((r.kind & 7u) << 12) | ((r.bounds & 0xFu) << 15);
            mo[k] = o;
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    if (bad) { g_last_error = "value token or arrival index not representable in the compact wire format"; return PT_ERR_INVALID; }
    return PT_OK;
}

int pt_batch_upload_compact(pt_batch* b, const pt_packed_compact* cc) {
    if (!b || !cc || (cc->n_logs && !cc->logs)) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->have_batch = false; b->merged = false;
    if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }
    b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0; b->dl_begun = false; b->have_changes = false;
    pt_packed_ops ops{cc->n_logs, cc->logs, nullptr, cc->n_insdel_total, nullptr, cc->n_mark_total};
    int rc = plan_batch(b, &ops);
    if (rc) return rc;
    if ((rc = alloc_and_upload_plan(b))) return rc;
    if ((rc = b->d_insdel.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_insdel_rec)))) return rc;
    if ((rc = b->d_marks.reserve(std::max<uint64_t>(1, b->n_mark) * sizeof(pt_mark_rec)))) return rc;
    if ((rc = b->d_cins.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_insdel_c8)))) return rc;
    if ((rc = b->d_cmarks.reserve(std::max<uint64_t>(1, b->n_mark) * sizeof(pt_mark_c16)))) return rc;
    const uint32_t threads = 256, gmax = (uint32_t)b->num_sms * 16;
    if (b->n_insdel) {
        PT_CUDA(cudaMemcpyAsync(b->d_cins.p, cc->insdel, b->n_insdel * sizeof(pt_insdel_c8), cudaMemcpyHostToDevice, b->stream));
        expand_insdel_c8_kernel<<<(uint32_t)std::min<uint64_t>((b->n_insdel + threads - 1) / threads, gmax), threads, 0, b->stream>>>(
            (const pt_insdel_c8*)b->d_cins.p, (pt_insdel_rec*)b->d_insdel.p, b->n_insdel);
        b->launches++;
    }
    if (b->n_mark) {
        PT_CUDA(cudaMemcpyAsync(b->d_cmarks.p, cc->marks, b->n_mark * sizeof(pt_mark_c16), cudaMemcpyHostToDevice, b->stream));
        expand_mark_c16_kernel<<<(uint32_t)std::min<uint64_t>((b->n_mark + threads - 1) / threads, gmax), threads, 0, b->stream>>>(
            (const pt_mark_c16*)b->d_cmarks.p, (pt_mark_rec*)b->d_marks.p, b->n_mark);
        b->launches++;
    }
    PT_CUDA(cudaGetLastError());
    b->dp_insdel = (const pt_insdel_rec*)b->d_insdel.p; b->dp_marks = (const pt_mark_rec*)b->d_marks.p; b->adopted = false;
    auto pinned = [](const void* p) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return a.type == cudaMemoryTypeHost;
    };
    if (!((b->n_insdel == 0 || pinned(cc->insdel)) && (b->n_mark == 0 || pinned(cc->marks)))) PT_CUDA(cudaStreamSynchronize(b->stream));
    b->have_batch = true;
    return PT_OK;
}

int pt_batch_upload_changes(pt_batch* b, const pt_change_table* t) {
    if (!b || !t) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_upload_changes before pt_batch_upload"; return PT_ERR_STATE; }
    if (t->n_logs != b->n_logs || (t->n_logs && !t->logs)) { g_last_error = "change table does not match the batch"; return PT_ERR_INVALID; }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    uint32_t maxR = 1;
    for (uint32_t i = 0; i < b->n_logs; i++) {
        const pt_change_desc& D = t->logs[i];
        if (D.change_off + D.n_changes > t->n_changes_total || D.dep_off + D.n_deps > t->n_deps_total) { g_last_error = "change descriptor out of range"; return PT_ERR_INVALID; }
        maxR = std::max<uint32_t>(maxR, b->h_desc[i].n_actors);
    }
    if ((size_t)2 * maxR * 4 > 200 * 1024) { g_last_error = "more than 25600 actors in one log: not supported by the admission pre-pass"; return PT_ERR_INVALID; }
    int rc;
    const size_t n = b->n_logs;
    if ((rc = b->d_cdesc.reserve(std::max<size_t>(1, n) * sizeof(pt_change_desc)))) return rc;
    if ((rc = b->d_changes.reserve(std::max<uint64_t>(1, t->n_changes_total) * sizeof(pt_change_rec)))) return rc;
    if ((rc = b->d_deps.reserve(std::max<uint64_t>(1, t->n_deps_total) * sizeof(pt_dep_rec)))) return rc;
    if ((rc = b->d_admit.reserve(std::max<size_t>(1, n) * 4))) return rc;
    if (n) PT_CUDA(cudaMemcpyAsync(b->d_cdesc.p, t->logs, n * sizeof(pt_change_desc), cudaMemcpyHostToDevice, b->stream));
    if (t->n_changes_total) PT_CUDA(cudaMemcpyAsync(b->d_changes.p, t->changes, t->n_changes_total * sizeof(pt_change_rec), cudaMemcpyHostToDevice, b->stream));
    if (t->n_deps_total) PT_CUDA(cudaMemcpyAsync(b->d_deps.p, t->deps, t->n_deps_total * sizeof(pt_dep_rec), cudaMemcpyHostToDevice, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));            // the caller's arrays may be freed on return
    b->adm_maxR = maxR; b->have_changes = true;
    if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }   // the launch sequence changes
    b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0;
    return PT_OK;
}

static int enqueue_merge(pt_batch* b) {
    PT_CUDA(cudaMemsetAsync(b->d_counters.p, 0, 256, b->stream));   // stats, pool cursor and queue counters in one shot
    ptk::BatchParams P{};
    P.desc = (const pt_log_desc*)b->d_desc.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.results = (pt_log_result*)b->d_results.p;
    P.text_off = (const uint64_t*)b->d_text_off.p; P.span_off = (const uint64_t*)b->d_span_off.p;
    P.text = (uint32_t*)b->d_text.p; P.spans = (pt_span*)b->d_spans.p;
    P.comment_pool = (uint32_t*)b->d_pool.p; P.comment_used = (unsigned long long*)((char*)b->d_counters.p + 64); P.comment_cap = b->pool_cap;
    P.slab = (char*)b->d_slab.p;
    P.slab_counter = (uint32_t*)((char*)b->d_counters.p + 96); P.slab_slots = b->slab_slots;
    P.seq = (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) ? (uint32_t*)b->d_seq.p : nullptr;
    P.stats = (unsigned long long*)b->d_counters.p;
    P.admit = nullptr;
    if (b->have_changes && b->n_logs) {
        // admission pre-pass: 4 warps per CTA while the per-actor tables fit, else one warp with up to 200 KB
        const size_t per_warp = (size_t)2 * b->adm_maxR * 4;
        const uint32_t wpb = per_warp * 4 <= 48 * 1024 ? 4u : 1u;
        const size_t smem = per_warp * wpb;
        if (smem > 48 * 1024) PT_CUDA(cudaFuncSetAttribute(admit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(((uint64_t)b->n_logs + wpb - 1) / wpb, (uint64_t)b->num_sms * 16);
        admit_kernel<<<grid, wpb * 32, smem, b->stream>>>((const pt_change_desc*)b->d_cdesc.p, (const pt_change_rec*)b->d_changes.p, (const pt_dep_rec*)b->d_deps.p,
                                                       (const pt_log_desc*)b->d_desc.p, b->n_logs, b->adm_maxR, (uint32_t*)b->d_admit.p, (pt_log_result*)b->d_results.p);
        PT_CUDA(cudaGetLastError());
        b->launches++;
        P.admit = (const uint32_t*)b->d_admit.p;
    }
    { const char* e = getenv("PT_PREFETCH"); P.prefetch_next = e ? (uint32_t)atoi(e) : 0u; }
    { const char* e = getenv("PT_WARP_FLAGS"); P.warp_flags = e ? (uint32_t)atoi(e) : 0x704u; }   // default: phase-aligned rounds (bit 2), the in-log phase barriers 2-4 skipped (bits 8-10: measured), no extra L2 prefetch
    { const char* e = getenv("PT_TMA"); P.use_tma = e ? (uint32_t)atoi(e) : 1u; }
    int rc;
    // ascending bins; a log whose working set does not fit bin k's shared memory is deferred (on the device) to bin k+1;
    // only the last bin can spill to the global slab
    // The CTA-per-log bins' own lists do not depend on the warp / team kernels: when both exist they are launched on a side
    // stream (fork / join, also inside the captured graph) and fill the SMs the warp kernel's tail leaves idle.  The deferral
    // launches come after the join, in ascending bin order.
    const bool have0 = b->bin_first[1] > b->bin_first[0], haveBlocks = b->bin_first[kNumBins] > b->bin_first[1];
    const bool fork = have0 && haveBlocks && b->side != nullptr;
    if (fork) {
        PT_CUDA(cudaEventRecord(b->ev_fork, b->stream));
        PT_CUDA(cudaStreamWaitEvent(b->side, b->ev_fork, 0));
        b->launch_stream = b->side;
    }
    if (fork) {
        for (int k = 1; k < kNumBins; k++) if ((rc = launch_bin(b, k, P, false))) { b->launch_stream = b->stream; return rc; }
        PT_CUDA(cudaEventRecord(b->ev_join, b->side));
        b->launch_stream = b->stream;
        if ((rc = launch_bin(b, 0, P, false))) return rc;
        PT_CUDA(cudaStreamWaitEvent(b->stream, b->ev_join, 0));
        for (int k = 1; k < kNumBins; k++) if ((rc = launch_bin(b, k, P, true))) return rc;
    } else {
        bool lower = false;
        for (int k = 0; k < kNumBins; k++) {
            if ((rc = launch_bin(b, k, P, false))) return rc;
            if (k > 0 && lower && (rc = launch_bin(b, k, P, true))) return rc;
            lower = lower || b->bin_first[k + 1] > b->bin_first[k];
        }
    }
    if ((b->limits.flags & PT_FLAG_EMIT_PATCHES) && b->n_logs) {
        ptk::PatchParams Q{};
        Q.desc = P.desc; Q.insdel = P.insdel; Q.marks = P.marks; Q.results = P.results; Q.text_off = P.text_off; Q.seq = P.seq;
        Q.n_logs = b->n_logs; Q.smem_bytes = b->patch_smem;
        Q.recs = (pt_patch_rec*)b->d_patch_recs.p; Q.items = (pt_patch_item*)b->d_patch_items.p;
        Q.item_cursor = (unsigned long long*)((char*)b->d_counters.p + 80); Q.item_cap = b->patch_cap;
        Q.status = (uint32_t*)b->d_patch_status.p;
        PT_CUDA(cudaFuncSetAttribute(ptk::patch_logs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b->patch_smem));
        const uint32_t per_sm = std::max<uint32_t>(1, std::min<uint32_t>(32, (227u * 1024u) / (b->patch_smem + 1024u)));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(b->n_logs, (uint64_t)b->num_sms * per_sm);
        ptk::patch_logs_kernel<<<grid, 32, b->patch_smem, b->stream>>>(Q);
        PT_CUDA(cudaGetLastError());
        b->launches++;
    }
    return PT_OK;
}

int pt_batch_merge(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_merge before pt_batch_upload"; return PT_ERR_STATE; }
    PT_CUDA(cudaSetDevice(b->device));
    // The launch sequence of a batch is fixed: capture it once into a CUDA graph (not possible on the legacy default
    // stream, where the launches are simply enqueued directly).
    if (!b->graph_tried && b->merges_since_upload >= 1) {   // a batch merged more than once: replay its launch sequence as a graph
        b->graph_tried = true;
        const char* eg = getenv("PT_GRAPH");
        if (b->stream != nullptr && !(eg && atoi(eg) == 0)) {
            const uint64_t l0 = b->launches;
            if (cudaStreamBeginCapture(b->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
                int rc = enqueue_merge(b);
                cudaGraph_t g = nullptr;
                cudaError_t e = cudaStreamEndCapture(b->stream, &g);
                if (rc == PT_OK && e == cudaSuccess && g && cudaGraphInstantiate(&b->graph_exec, g, 0) == cudaSuccess) {
                    b->graph_ok = true; b->kernels_per_merge = (uint32_t)(b->launches - l0);
                }
                if (g) cudaGraphDestroy(g);
                b->launches = l0;
            }
            cudaGetLastError();
        }
    }
    PT_CUDA(cudaEventRecord(b->ev0, b->stream));
    if (b->graph_ok) {
        PT_CUDA(cudaGraphLaunch(b->graph_exec, b->stream));
        b->launches += b->kernels_per_merge;
    } else {
        int rc = enqueue_merge(b);
        if (rc) return rc;
    }
    PT_CUDA(cudaEventRecord(b->ev1, b->stream));
    b->merged = true; b->merges_since_upload++; b->dl_begun = false;
    return PT_OK;
}

int pt_batch_sync(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    return PT_OK;
}

float pt_batch_last_merge_ms(pt_batch* b) {
    if (!b || !b->merged) return -1.f;
    if (cudaEventSynchronize(b->ev1) != cudaSuccess) return -1.f;
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, b->ev0, b->ev1) != cudaSuccess) return -1.f;
    return ms;
}

int pt_batch_download_results(pt_batch* b, pt_log_result* out, uint32_t n_logs) {
    if (!b || (!out && n_logs)) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    if (n_logs > b->n_logs) return PT_ERR_INVALID;
    int rc;
    if ((rc = b->h_results.reserve(std::max<size_t>(1, b->n_logs) * sizeof(pt_log_result)))) return rc;
    if (n_logs) PT_CUDA(cudaMemcpyAsync(b->h_results.p, b->d_results.p, (size_t)n_logs * sizeof(pt_log_result), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    if (n_logs) memcpy(out, b->h_results.p, (size_t)n_logs * sizeof(pt_log_result));
    return PT_OK;
}

// Pack the outputs on the device (see the compaction kernels above) and enqueue the device -> host copies of the per-log
// headers, the packed offsets and the comment-pool cursor (asynchronous, pinned destinations); pt_batch_download then
// waits, learns the packed sizes and copies exactly the used tokens / spans / comment ids.  Lets a caller overlap one
// handle's download with another handle's upload / merge.
int pt_batch_download_begin(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    int rc;
    const size_t n = b->n_logs;
    const uint32_t nb = (uint32_t)((n + kScanBlock - 1) / kScanBlock);
    if ((rc = b->h_results.reserve(std::max<size_t>(1, n) * sizeof(pt_log_result)))) return rc;
    if ((rc = b->h_ctoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->h_csoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->h_misc.reserve(16))) return rc;
    if ((rc = b->d_bsum.reserve((size_t)(2 * nb + 2) * 8))) return rc;
    if ((rc = b->d_ctoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->d_csoff.reserve((n + 1) * 8))) return rc;
    // packed outputs can never exceed the capacities; sized once per batch
    if ((rc = b->d_ctext.reserve(std::max<uint64_t>(1, b->n_text) * 4))) return rc;
    if ((rc = b->d_cspans.reserve(std::max<uint64_t>(1, b->n_span) * sizeof(pt_span)))) return rc;
    PT_CUDA(cudaMemcpyAsync(b->h_misc.p, (char*)b->d_counters.p + 64, 8, cudaMemcpyDeviceToHost, b->stream));   // pool cursor = the batch's demand
    if (n) {
        const pt_log_result* res = (const pt_log_result*)b->d_results.p;
        unsigned long long* bsum = (unsigned long long*)b->d_bsum.p;
        unsigned long long *toff = (unsigned long long*)b->d_ctoff.p, *soff = (unsigned long long*)b->d_csoff.p;
        out_block_sums_kernel<<<nb, kScanBlock, 0, b->stream>>>(MergedCounts{res}, (uint32_t)n, bsum);
        out_scan_blocks_kernel<<<1, 1024, 0, b->stream>>>(bsum, nb);
        out_offsets_kernel<<<nb, kScanBlock, 0, b->stream>>>(MergedCounts{res}, (uint32_t)n, bsum, nb, toff, soff);
        const uint32_t gthreads = 256, ggrid = (uint32_t)std::min<uint64_t>((n * 32 + gthreads - 1) / gthreads, (uint64_t)b->num_sms * 16);
        out_gather_kernel<<<ggrid, gthreads, 0, b->stream>>>(res, (uint32_t)n, (const uint64_t*)b->d_text_off.p, (const uint64_t*)b->d_span_off.p, toff, soff,
                                                           (const uint32_t*)b->d_text.p, (const pt_span*)b->d_spans.p, (uint32_t*)b->d_ctext.p, (pt_span*)b->d_cspans.p);
        PT_CUDA(cudaGetLastError());
        b->launches += 4;
        PT_CUDA(cudaMemcpyAsync(b->h_results.p, b->d_results.p, n * sizeof(pt_log_result), cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->h_ctoff.p, b->d_ctoff.p, (n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->h_csoff.p, b->d_csoff.p, (n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    } else {
        ((uint64_t*)b->h_ctoff.p)[0] = 0; ((uint64_t*)b->h_csoff.p)[0] = 0;
    }
    if (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) {
        if ((rc = b->h_seq.reserve(std::max<uint64_t>(1, b->n_text) * 4))) return rc;
        if (b->n_text) PT_CUDA(cudaMemcpyAsync(b->h_seq.p, b->d_seq.p, b->n_text * 4, cudaMemcpyDeviceToHost, b->stream));
    }
    b->dl_begun = true;
    return PT_OK;
}

int pt_batch_download(pt_batch* b, pt_spans_view* out) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    int rc;
    if (!b->dl_begun && (rc = pt_batch_download_begin(b))) return rc;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const bool want_seq = (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) != 0;
    const size_t n = b->n_logs;
    const uint64_t demand = *(unsigned long long*)b->h_misc.p;
    const uint64_t used = std::min<uint64_t>(demand, b->pool_cap);
    const uint64_t n_ctext = ((const uint64_t*)b->h_ctoff.p)[n], n_cspan = ((const uint64_t*)b->h_csoff.p)[n];
    b->pool_used_host = used;
    if ((rc = b->h_pool.reserve(std::max<uint64_t>(1, used) * 4))) return rc;
    if ((rc = b->h_text.reserve(std::max<uint64_t>(1, n_ctext) * 4))) return rc;
    if ((rc = b->h_spans.reserve(std::max<uint64_t>(1, n_cspan) * sizeof(pt_span)))) return rc;
    if (n_ctext) PT_CUDA(cudaMemcpyAsync(b->h_text.p, b->d_ctext.p, n_ctext * 4, cudaMemcpyDeviceToHost, b->stream));
    if (n_cspan) PT_CUDA(cudaMemcpyAsync(b->h_spans.p, b->d_cspans.p, n_cspan * sizeof(pt_span), cudaMemcpyDeviceToHost, b->stream));
    if (used) PT_CUDA(cudaMemcpyAsync(b->h_pool.p, b->d_pool.p, used * 4, cudaMemcpyDeviceToHost, b->stream));
    if (n_ctext || n_cspan || used) PT_CUDA(cudaStreamSynchronize(b->stream));
    out->n_logs = b->n_logs;
    out->results = (const pt_log_result*)b->h_results.p;
    out->text_off = (const uint64_t*)b->h_ctoff.p;
    out->span_off = (const uint64_t*)b->h_csoff.p;
    out->text = (const uint32_t*)b->h_text.p;
    out->spans = (const pt_span*)b->h_spans.p;
    out->comment_pool = (const uint32_t*)b->h_pool.p;
    out->comment_pool_used = used;
    out->seq = want_seq ? (const uint32_t*)b->h_seq.p : nullptr;
    out->seq_off = want_seq ? b->h_text_off.data() : nullptr;
    out->comment_pool_needed = demand;                  // the cursor counts past the capacity
    return PT_OK;
}

int pt_batch_download_patches(pt_batch* b, pt_patch_view* out) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_PATCHES)) { g_last_error = "the handle was created without PT_FLAG_EMIT_PATCHES"; return PT_ERR_STATE; }
    int rc;
    if ((rc = b->h_patch_misc.reserve(16))) return rc;
    if ((rc = b->h_patch_recs.reserve(std::max<uint64_t>(1, b->n_insdel) * sizeof(pt_patch_rec)))) return rc;
    if ((rc = b->h_patch_status.reserve(std::max<size_t>(1, b->n_logs) * 4))) return rc;
    PT_CUDA(cudaMemcpyAsync(b->h_patch_misc.p, (char*)b->d_counters.p + 80, 8, cudaMemcpyDeviceToHost, b->stream));
    if (b->n_insdel) PT_CUDA(cudaMemcpyAsync(b->h_patch_recs.p, b->d_patch_recs.p, b->n_insdel * sizeof(pt_patch_rec), cudaMemcpyDeviceToHost, b->stream));
    if (b->n_logs) PT_CUDA(cudaMemcpyAsync(b->h_patch_status.p, b->d_patch_status.p, (size_t)b->n_logs * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t demand = *(unsigned long long*)b->h_patch_misc.p, used = std::min<uint64_t>(demand, b->patch_cap);
    if ((rc = b->h_patch_items.reserve(std::max<uint64_t>(1, used) * sizeof(pt_patch_item)))) return rc;
    if (used) { PT_CUDA(cudaMemcpyAsync(b->h_patch_items.p, b->d_patch_items.p, used * sizeof(pt_patch_item), cudaMemcpyDeviceToHost, b->stream)); PT_CUDA(cudaStreamSynchronize(b->stream)); }
    out->recs = (const pt_patch_rec*)b->h_patch_recs.p; out->items = (const pt_patch_item*)b->h_patch_items.p;
    out->n_items = used; out->n_items_needed = demand; out->status = (const uint32_t*)b->h_patch_status.p;
    return PT_OK;
}

int pt_batch_set_patch_pool(pt_batch* b, uint64_t items) {
    if (!b || items > 0xFFFFFFFFull) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->limits.patch_pool_items = (uint32_t)items;
    if (b->have_batch && items && (b->limits.flags & PT_FLAG_EMIT_PATCHES)) {
        b->patch_cap = items;
        int rc;
        if ((rc = b->d_patch_items.reserve(b->patch_cap * sizeof(pt_patch_item)))) return rc;
        if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }
        b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0;
    }
    return PT_OK;
}

int pt_batch_query_elements(pt_batch* b, const pt_elem_query* queries, uint32_t n, uint32_t* out) {
    if (!b || (n && (!queries || !out))) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "query before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = "the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    if (!n) return PT_OK;
    PT_CUDA(cudaSetDevice(b->device));
    DevBuf dq, da;
    int rc;
    if ((rc = dq.reserve((size_t)n * sizeof(pt_elem_query))) || (rc = da.reserve((size_t)n * 4))) { dq.release(); da.release(); return rc; }
    cudaError_t e = cudaMemcpyAsync(dq.p, queries, (size_t)n * sizeof(pt_elem_query), cudaMemcpyHostToDevice, b->stream);
    if (e == cudaSuccess) {
        const uint32_t threads = 128, grid = (uint32_t)std::min<uint64_t>(((uint64_t)n * 32 + threads - 1) / threads, (uint64_t)b->num_sms * 16);
        query_elements_kernel<<<grid, threads, 0, b->stream>>>((const pt_elem_query*)dq.p, n, (const pt_log_result*)b->d_results.p,
                                                              (const uint64_t*)b->d_text_off.p, (const uint32_t*)b->d_seq.p, b->n_logs, (uint32_t*)da.p);
        e = cudaGetLastError();
        b->launches++;
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, da.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->stream);
    dq.release(); da.release();
    if (e != cudaSuccess) { g_last_error = std::string("pt_batch_query_elements: ") + cudaGetErrorString(e); return PT_ERR_CUDA; }
    return PT_OK;
}

int pt_batch_find_elements(pt_batch* b, const pt_elem_ref* refs, uint32_t n, pt_elem_pos* out) {
    if (!b || (n && (!refs || !out))) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "find before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = "the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    if (!n) return PT_OK;
    PT_CUDA(cudaSetDevice(b->device));
    DevBuf dq, da;
    int rc;
    if ((rc = dq.reserve((size_t)n * sizeof(pt_elem_ref))) || (rc = da.reserve((size_t)n * sizeof(pt_elem_pos)))) { dq.release(); da.release(); return rc; }
    cudaError_t e = cudaMemcpyAsync(dq.p, refs, (size_t)n * sizeof(pt_elem_ref), cudaMemcpyHostToDevice, b->stream);
    if (e == cudaSuccess) {
        const uint32_t threads = 128, grid = (uint32_t)std::min<uint64_t>(((uint64_t)n * 32 + threads - 1) / threads, (uint64_t)b->num_sms * 16);
        find_elements_kernel<<<grid, threads, 0, b->stream>>>((const pt_elem_ref*)dq.p, n, (const pt_log_desc*)b->d_desc.p, b->dp_insdel,
                                                             (const pt_log_result*)b->d_results.p, (const uint64_t*)b->d_text_off.p,
                                                             (const uint32_t*)b->d_seq.p, b->n_logs, (pt_elem_pos*)da.p);
        e = cudaGetLastError();
        b->launches++;
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, da.p, (size_t)n * sizeof(pt_elem_pos), cudaMemcpyDeviceToHost, b->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->stream);
    dq.release(); da.release();
    if (e != cudaSuccess) { g_last_error = std::string("pt_batch_find_elements: ") + cudaGetErrorString(e); return PT_ERR_CUDA; }
    return PT_OK;
}

// JSON render (render_kernel.cuh): upload the pools, size pass, scan of the sizes through the download path's scan kernels,
// read back the total and the missing-entry key (one sync), size the output exactly, write pass, copy back.
int pt_batch_render_json(pt_batch* b, const pt_json_pools* pools, pt_json_view* out) {
    if (!b || !pools || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "render before merge"; return PT_ERR_STATE; }
    struct Pool { const uint8_t* data; const uint64_t* off; uint64_t count; DevBuf* dd; DevBuf* doff; const char* name; };
    const Pool ps[3] = {{pools->values, pools->values_off, pools->n_values, &b->d_jval, &b->d_jvoff, "values"},
                        {pools->links, pools->links_off, pools->n_links, &b->d_jlink, &b->d_jloff, "links"},
                        {pools->comments, pools->comments_off, pools->n_comments, &b->d_jcom, &b->d_jcoff, "comments"}};
    for (const Pool& p : ps) {
        if (p.count && (!p.data || !p.off)) { g_last_error = std::string("pt_batch_render_json: null ") + p.name + " pool with a nonzero count"; return PT_ERR_INVALID; }
        for (uint64_t k = 0; k < p.count; k++)
            if (p.off[k + 1] < p.off[k]) { g_last_error = std::string("pt_batch_render_json: ") + p.name + " offsets decrease"; return PT_ERR_INVALID; }
    }
    PT_CUDA(cudaSetDevice(b->device));
    int rc;
    const uint32_t n = b->n_logs;
    if ((rc = b->h_joff.reserve(((size_t)n + 1) * 8)) || (rc = b->h_jbytes.reserve(1)) || (rc = b->h_jmisc.reserve(16))) return rc;
    uint64_t* hoff = (uint64_t*)b->h_joff.p;
    if (!n) {
        hoff[0] = 0;
        *out = pt_json_view{0, hoff, (const char*)b->h_jbytes.p, 0};
        return PT_OK;
    }
    ptr::JsonPools P{};
    const uint8_t** pdata[3] = {&P.val, &P.link, &P.com};
    const uint64_t** poff[3] = {&P.voff, &P.loff, &P.coff};
    uint64_t* pcount[3] = {&P.nval, &P.nlink, &P.ncom};
    for (int k = 0; k < 3; k++) {
        const Pool& p = ps[k];
        const uint64_t lo = p.count ? p.off[0] : 0, hi = p.count ? p.off[p.count] : 0;     // entries address data[lo, hi)
        if ((rc = p.dd->reserve(std::max<uint64_t>(1, hi))) || (rc = p.doff->reserve((p.count + 1) * 8))) return rc;
        if (hi > lo) PT_CUDA(cudaMemcpyAsync((uint8_t*)p.dd->p + lo, p.data + lo, hi - lo, cudaMemcpyHostToDevice, b->stream));
        if (p.count) PT_CUDA(cudaMemcpyAsync(p.doff->p, p.off, (p.count + 1) * 8, cudaMemcpyHostToDevice, b->stream));
        *pdata[k] = (const uint8_t*)p.dd->p; *poff[k] = (const uint64_t*)p.doff->p; *pcount[k] = p.count;
    }
    const uint32_t nb = (n + kScanBlock - 1) / kScanBlock;
    if ((rc = b->d_jsize.reserve((size_t)n * 8)) || (rc = b->d_jbsum.reserve((size_t)(2 * nb + 2) * 8)) || (rc = b->d_joff.reserve(((size_t)n + 1) * 8)) ||
        (rc = b->d_jmiss.reserve(8))) return rc;
    unsigned long long *sizes = (unsigned long long*)b->d_jsize.p, *bsum = (unsigned long long*)b->d_jbsum.p, *doff = (unsigned long long*)b->d_joff.p,
                       *miss = (unsigned long long*)b->d_jmiss.p;
    const pt_log_result* res = (const pt_log_result*)b->d_results.p;
    const uint64_t *toff = (const uint64_t*)b->d_text_off.p, *soff = (const uint64_t*)b->d_span_off.p;
    const uint32_t* text = (const uint32_t*)b->d_text.p;
    const pt_span* spans = (const pt_span*)b->d_spans.p;
    const uint32_t* cpool = (const uint32_t*)b->d_pool.p;
    const uint32_t threads = 128, grid = (uint32_t)std::min<uint64_t>(((uint64_t)n * 32 + threads - 1) / threads, (uint64_t)b->num_sms * 16);
    PT_CUDA(cudaMemsetAsync(miss, 0xFF, 8, b->stream));
    ptr::json_size_kernel<<<grid, threads, 0, b->stream>>>(res, n, toff, soff, text, spans, cpool, P, sizes, miss);
    out_block_sums_kernel<<<nb, kScanBlock, 0, b->stream>>>(PlainCounts{sizes}, n, bsum);
    out_scan_blocks_kernel<<<1, 1024, 0, b->stream>>>(bsum, nb);
    out_offsets_kernel<<<nb, kScanBlock, 0, b->stream>>>(PlainCounts{sizes}, n, bsum, nb, doff, (unsigned long long*)nullptr);
    PT_CUDA(cudaGetLastError());
    b->launches += 4;
    uint64_t* hm = (uint64_t*)b->h_jmisc.p;
    PT_CUDA(cudaMemcpyAsync(hm, doff + n, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(hm + 1, miss, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t total = hm[0], key = hm[1];
    if (key != ~0ull) {
        static const char* kinds[3] = {"value", "link", "comment"};
        g_last_error = "pt_batch_render_json: log " + std::to_string(key >> 34) + " names " + kinds[(key >> 32) & 3] + " pool entry " +
                       std::to_string(key & 0xFFFFFFFFull) + ", which the caller's pools do not hold";
        return PT_ERR_INVALID;
    }
    if ((rc = b->d_jbytes.reserve(std::max<uint64_t>(1, total))) || (rc = b->h_jbytes.reserve(std::max<uint64_t>(1, total)))) return rc;
    ptr::json_write_kernel<<<grid, threads, 0, b->stream>>>(res, n, toff, soff, text, spans, cpool, P, doff, (uint8_t*)b->d_jbytes.p);
    PT_CUDA(cudaGetLastError());
    b->launches++;
    PT_CUDA(cudaMemcpyAsync(hoff, doff, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    if (total) PT_CUDA(cudaMemcpyAsync(b->h_jbytes.p, b->d_jbytes.p, total, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    *out = pt_json_view{n, hoff, (const char*)b->h_jbytes.p, total};
    return PT_OK;
}

int pt_batch_device_results(pt_batch* b, void** dev_ptr, uint32_t* n_logs) {
    if (!b || !dev_ptr) return PT_ERR_INVALID;
    if (!b->have_batch) return PT_ERR_STATE;
    *dev_ptr = b->d_results.p;
    if (n_logs) *n_logs = b->n_logs;
    return PT_OK;
}

uint64_t pt_batch_launch_count(const pt_batch* b) { return b ? b->launches : 0; }

int pt_batch_stats(pt_batch* b, uint64_t out[4]) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) return PT_ERR_STATE;
    unsigned long long h[8] = {0};
    PT_CUDA(cudaMemcpyAsync(h, b->d_counters.p, 32, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    for (int i = 0; i < 3; i++) out[i] = h[i];
    out[3] = 0;
    PT_CUDA(cudaMemcpyAsync(h, (char*)b->d_counters.p + 64, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    out[3] = h[0];                                       // comment-pool entries the batch needs
    return PT_OK;
}

#ifdef PT_PHASE_CLOCKS
// Profiling build only (make PHASE_CLOCKS=1): the warp kernel's per-phase cycle sums on the current device, summed over
// its warps since the last reset: out[0..8] = log start, A+B, C, D, E, F, G, I, round wait; out[9] = logs merged.
int pt_phase_clocks(uint64_t out[ptk::kNumPhases + 1], int reset) {
    if (!out) return PT_ERR_INVALID;
    PT_CUDA(cudaDeviceSynchronize());
    PT_CUDA(cudaMemcpyFromSymbol(out, ptk::ptk_phase_clk, sizeof(ptk::ptk_phase_clk)));
    if (reset) {
        static const unsigned long long zero[ptk::kNumPhases + 1] = {};
        PT_CUDA(cudaMemcpyToSymbol(ptk::ptk_phase_clk, zero, sizeof(zero)));
    }
    return PT_OK;
}
#endif

int pt_batch_set_comment_pool(pt_batch* b, uint64_t entries) {
    if (!b) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->limits.comment_pool_entries = entries;
    if (b->have_batch && entries) {
        b->pool_cap = entries;
        int rc;
        if ((rc = b->d_pool.reserve(std::max<uint64_t>(1, b->pool_cap) * 4))) return rc;
        if (b->graph_exec) { cudaGraphExecDestroy(b->graph_exec); b->graph_exec = nullptr; }   // the pool pointer / capacity are baked in
        b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0;
    }
    return PT_OK;
}

void pt_batch_destroy(pt_batch* b) {
    if (!b) return;
    cudaSetDevice(b->device);
    cudaStreamSynchronize(b->stream);
    for (DevBuf* d : {&b->d_desc, &b->d_insdel, &b->d_marks, &b->d_order, &b->d_counters, &b->d_results, &b->d_text_off,
                      &b->d_span_off, &b->d_text, &b->d_spans, &b->d_pool, &b->d_slab, &b->d_retry, &b->d_seq,
                      &b->d_runs, &b->d_tokens, &b->d_run_off, &b->d_tok_off, &b->d_cins, &b->d_cmarks, &b->d_bsum, &b->d_ctoff, &b->d_csoff, &b->d_ctext, &b->d_cspans,
                      &b->d_cdesc, &b->d_changes, &b->d_deps, &b->d_admit, &b->d_patch_recs, &b->d_patch_items, &b->d_patch_status,
                      &b->d_jval, &b->d_jvoff, &b->d_jlink, &b->d_jloff, &b->d_jcom, &b->d_jcoff, &b->d_jsize, &b->d_jbsum, &b->d_joff,
                      &b->d_jmiss, &b->d_jbytes}) d->release();
    for (HostBuf* h : {&b->h_patch_recs, &b->h_patch_items, &b->h_patch_status, &b->h_patch_misc, &b->h_joff, &b->h_jbytes, &b->h_jmisc}) h->release();
    for (HostBuf* h : {&b->h_stage, &b->h_results, &b->h_text, &b->h_spans, &b->h_pool, &b->h_misc, &b->h_seq, &b->h_ctoff, &b->h_csoff}) h->release();
    if (b->side) cudaStreamDestroy(b->side);
    if (b->ev_fork) cudaEventDestroy(b->ev_fork);
    if (b->ev_join) cudaEventDestroy(b->ev_join);
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    if (b->graph_exec) cudaGraphExecDestroy(b->graph_exec);
    delete b;
}

const char* pt_strerror(int status) {
    switch (status) {
        case PT_OK: return "ok";
        case PT_ERR_INVALID: return "invalid argument";
        case PT_ERR_CUDA: return "CUDA runtime error";
        case PT_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (no CPU fallback)";
        case PT_ERR_STATE: return "call out of order";
        case PT_ERR_NOMEM: return "out of memory";
        default: return "unknown status";
    }
}
const char* pt_last_error(void) { return g_last_error.c_str(); }
const char* pt_version(void) { return "peritext_b200 0.1 (sm_90a)"; }

}  // extern "C"
