// query_kernel.cuh — element queries over the materialised element sequences of a merged batch (pt_batch_query_elements,
// pt_batch_find_elements).
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace ptq {

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

}  // namespace ptq
