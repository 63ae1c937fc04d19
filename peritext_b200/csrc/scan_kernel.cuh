// scan_kernel.cuh — exclusive scans of per-log counts over the batch, and the packing of the merge outputs before download.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace pts {

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

}  // namespace pts
