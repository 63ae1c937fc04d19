// admit_kernel.cuh — causal admission of every log's change table before the merge (pt_batch_upload_changes).
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace ptadm {

// ---- admission pre-pass: Micromerge.applyChange's causal checks (reference src/micromerge.ts:499-511) for every log -------
// One warp per log, one lane per change, 32 changes per trip, against ptct::TripClock (DESIGN.md §4.3): as long as every
// earlier change of the log was admitted, the reference's clock is the per-actor count of earlier changes, so each change is
// checked on its own, and the FIRST failing change — what the reference would throw at — is a min over lanes.
__global__ void admit_kernel(const pt_change_desc* __restrict__ cd, const pt_change_rec* __restrict__ ch, const pt_dep_rec* __restrict__ dp,
                             const pt_log_desc* __restrict__ desc, uint32_t n_logs, uint32_t maxR, uint32_t* __restrict__ admit, pt_log_result* __restrict__ results) {
    extern __shared__ uint32_t adm_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* cnt = adm_smem + (size_t)wib * 2 * maxR;      // changes admitted so far, per actor
    uint32_t* cmask = cnt + maxR;                           // lanes of the current trip, per actor
    for (uint32_t li = blockIdx.x * wpb + wib; li < n_logs; li += gridDim.x * wpb) {
        const pt_change_desc D = cd[li];
        const uint32_t R = desc[li].n_actors ? desc[li].n_actors : 1u;
        for (uint32_t a = lane; a < R; a += 32) { cnt[a] = 0; cmask[a] = 0; }
        __syncwarp();
        const pt_change_rec* c0 = ch + D.change_off; const pt_dep_rec* d0 = dp + D.dep_off;
        uint32_t fail_idx = 0xFFFFFFFFu, fail_code = 0;
        ptct::TripClock clk(cnt, cmask, lane);
        for (uint32_t base = 0; base < D.n_changes; base += 32) {
            const uint32_t k = base + lane;
            const bool valid = k < D.n_changes;
            uint4 r = make_uint4(0, 0, 0, 0);
            if (valid) r = __ldg(reinterpret_cast<const uint4*>(c0 + k));
            const uint32_t seq = r.x, actor = r.y & 0xFFFFu, n_deps = r.y >> 16, dep_off = r.z;
            const bool aok = valid && actor < R;
            clk.group(aok, actor, lane);
            uint32_t code = 0;
            if (valid) {
                if (!aok) code = PT_LOG_BAD_OPID;
                else if (seq != clk.have(actor) + 1u) code = PT_LOG_SEQ_GAP;                               // src/micromerge.ts:501-504
                else if (dep_off + n_deps > D.n_deps) code = PT_LOG_BAD_OPID;
                else for (uint32_t d = 0; d < n_deps; d++) {                                            // src/micromerge.ts:505-509
                    const pt_dep_rec q = d0[dep_off + d];
                    const uint32_t have = q.actor < R ? clk.have(q.actor) : 0u;
                    if (have == 0 || have < q.seq) { code = PT_LOG_MISSING_DEP; break; }
                }
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, code != 0);
            if (bal) { const uint32_t f = __ffs(bal) - 1; fail_idx = base + f; fail_code = __shfl_sync(0xffffffffu, code, f); break; }
            clk.commit();
        }
        if (lane == 0) {
            admit[li] = fail_code;
            if (fail_code) { pt_log_result r{}; r.status = fail_code; r.n_elems = fail_idx; results[li] = r; }
        }
        __syncwarp();
    }
}

}  // namespace ptadm
