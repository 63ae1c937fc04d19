// upload_kernel.cuh — expansion of the optional upload wire forms (pt_batch_upload_runs, pt_batch_upload_compact) into the
// pt_insdel_rec / pt_mark_rec records the merge kernels read, and the warp kernel's key-record copy of those records.
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

// ---- the warp kernel's key-record copy of the resident records (warp_kernel.cuh reads it and nothing else on its streams) -----
// Same record positions as the full arrays, so the descriptors' offsets index it unchanged.  An id (c, a) of a log with
// C * R < 0xFFFF is stored as its 16-bit opId key (c - 1) * R + a, which is at most 0xFFFD; the two values above it are never
// keys and carry what the record passes branch on:
//   ins/del, 4 B (uint32):  own:16 | ref:16 << 16
//       kind > 1: own = ref = S1;  own id out of range: own = S1, ref = S0;  delete: own = S0;
//       ref = S0 at the head (ref_ctr == 0), the key of the reference if it is in range, else S1
//   mark, 8 B (uint2):      x = own:16 | start:16 << 16;  y = end:16 | arrival:11 << 16 | kind:3 << 27 | start bound:1 << 30 |
//                           end bound:1 << 31
//       own = S1: the id is out of range;  start / end = S1: the id is out of range or the bound is above PT_BOUND_AFTER (the
//       op then covers nothing / never ends);  a bound bit is kept only for a valid bound;  arrival = min(arrival, n), which
//       fits 11 bits on every log the warp kernel merges marks of (n <= 2047), and compares with every record index the same
// The warp kernel reads no mark kind bit above 2.  One warp per log; a log with C * R >= 0xFFFF is not on a warp route and
// is left unwritten.  The link and comment attrs stay in the full mark records (warp_kernel.cuh reads them for survivors).
constexpr uint32_t kKeyS0 = 0xFFFEu, kKeyS1 = 0xFFFFu;
__global__ void derive_key_records_kernel(const pt_log_desc* __restrict__ desc, const pt_insdel_rec* __restrict__ ins,
                                          const pt_mark_rec* __restrict__ mk, uint32_t* __restrict__ kins, uint2* __restrict__ kmk,
                                          uint32_t n_logs) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(desc + li)), d1 = __ldg(reinterpret_cast<const uint4*>(desc + li) + 1);
        const uint32_t n = d1.x, m = d1.y, R = d1.z ? d1.z : 1u, C = d1.w;
        if ((unsigned long long)C * R >= 0xFFFFull) continue;
        const unsigned long long io = (unsigned long long)d0.x | ((unsigned long long)d0.y << 32);
        const unsigned long long mo = (unsigned long long)d0.z | ((unsigned long long)d0.w << 32);
        auto key = [&](uint32_t c, uint32_t a) -> uint32_t { return c - 1u < C && a < R ? (c - 1u) * R + a : kKeyS1; };
        for (uint32_t i = lane; i < n; i += 32) {
            const uint4 r = __ldg(reinterpret_cast<const uint4*>(ins + io + i));   // {ctr, ref_ctr, actor | ref_actor << 16, payload}
            const uint32_t kind = r.w >> 30;
            uint32_t own = kind > 1u ? kKeyS1 : key(r.x, r.z & 0xFFFFu), ref = kKeyS1;
            if (kind <= 1u) {
                if (own == kKeyS1) ref = kKeyS0;
                else {
                    if (kind == PT_KIND_DELETE) own = kKeyS0;
                    ref = r.y == 0 ? kKeyS0 : key(r.y, r.z >> 16);
                }
            }
            kins[io + i] = own | (ref << 16);
        }
        const uint32_t narr = min(n, 0x7FFu);
        for (uint32_t k = lane; k < m; k += 32) {
            const uint4* q = reinterpret_cast<const uint4*>(mk + mo + k);
            // {ctr, actor | kind << 16 | bounds << 24, start_ctr, end_ctr} {start_actor | end_actor << 16, attr, arrival, reserved}
            const uint4 a = __ldg(q), b = __ldg(q + 1);
            const uint32_t sb = (a.y >> 24) & 3u, eb = (a.y >> 26) & 3u;
            const uint32_t s = sb <= PT_BOUND_AFTER ? key(a.z, b.x & 0xFFFFu) : kKeyS1, e = eb <= PT_BOUND_AFTER ? key(a.w, b.x >> 16) : kKeyS1;
            kmk[mo + k] = make_uint2(key(a.x, a.y & 0xFFFFu) | (s << 16),
                                     e | (min(b.z, narr) << 16) | (((a.y >> 16) & 7u) << 27) |
                                         ((sb <= PT_BOUND_AFTER ? sb : 0u) << 30) | ((eb <= PT_BOUND_AFTER ? eb : 0u) << 31));
        }
    }
}

}  // namespace ptu
