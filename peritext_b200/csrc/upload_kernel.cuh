// upload_kernel.cuh — expansion of the optional upload wire forms (pt_batch_upload_runs, pt_batch_upload_compact) into the
// pt_insdel_rec / pt_mark_rec records the merge kernels read, and the warp kernel's half-width copy of those records.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace ptu {

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

// ---- the warp kernel's half-width copy of the resident records (warp_kernel.cuh reads it and nothing else on its streams) -----
// Same record positions as the full arrays, so the descriptors' offsets index it unchanged.
//   ins/del, 8 B (uint2):  x = ctr:16 | ref_ctr:16 << 16;  y = actor:8 | ref_actor:8 << 8 | kind:2 << 16   (no payload)
//   mark, 16 B (uint4):    x = ctr:16 | start_ctr:16 << 16;  y = end_ctr:16 | arrival:16 << 16;  z = attr;
//                          w = actor:8 | start_actor:8 << 8 | end_actor:8 << 16 | kind:3 << 24 | bounds:4 << 27
// A counter or arrival too wide for its field saturates at 0xFFFF, an actor at 255.  The warp routes have C * R < 0xFFFF,
// n < 0xFFFF and R <= 255 (ptp::route_of), so a saturated id fails the same range check as the original and a saturated
// arrival still exceeds every record index: the copy changes no warp-kernel result.  The warp kernel reads no mark kind bit
// above 2 and no bound bit above 3.
__device__ __forceinline__ uint32_t sat16(uint32_t v) { return min(v, 0xFFFFu); }
__device__ __forceinline__ uint32_t sat8(uint32_t v) { return min(v, 0xFFu); }
__global__ void derive_half_records_kernel(const pt_insdel_rec* __restrict__ ins, const pt_mark_rec* __restrict__ mk,
                                           uint2* __restrict__ hins, uint4* __restrict__ hmk, unsigned long long n, unsigned long long m) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n + m; i += (unsigned long long)gridDim.x * blockDim.x) {
        if (i < n) {
            const uint4 r = __ldg(reinterpret_cast<const uint4*>(ins + i));   // {ctr, ref_ctr, actor | ref_actor << 16, payload}
            hins[i] = make_uint2(sat16(r.x) | (sat16(r.y) << 16), sat8(r.z & 0xFFFFu) | (sat8(r.z >> 16) << 8) | ((r.w >> 30) << 16));
        } else {
            const uint4* q = reinterpret_cast<const uint4*>(mk + (i - n));
            // {ctr, actor | kind << 16 | bounds << 24, start_ctr, end_ctr} {start_actor | end_actor << 16, attr, arrival, reserved}
            const uint4 a = __ldg(q), b = __ldg(q + 1);
            hmk[i - n] = make_uint4(sat16(a.x) | (sat16(a.z) << 16), sat16(a.w) | (sat16(b.z) << 16), b.y,
                                    sat8(a.y & 0xFFFFu) | (sat8(b.x & 0xFFFFu) << 8) | (sat8(b.x >> 16) << 16) |
                                        (((a.y >> 16) & 7u) << 24) | (((a.y >> 24) & 0xFu) << 27));
        }
    }
}

}  // namespace ptu
