// patch_window.cuh — where a log's patch window starts (pt_batch_set_patch_window).  Shared by the patch kernel, which
// computes the Patches of the window's ops only, and the patch JSON render, which renders them: both must cut the log at the
// same record.
//
// List-op positions: mark record k sits at min(arrival_k, n) + k, right before ins/del record arrival_k; ins/del record j sits
// at j + #{k : min(arrival_k, n) <= j}.  Arrivals never decrease, so the mark positions strictly increase in k and the marks
// before position first_op are a prefix [0, k0); the ins/del records before it are [0, first_op - k0).
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace ptw {

// k0 = #{k : min(arrival_k, n) + k < first_op} over the log's m mark records mk[0 .. m).  Warp-collective (one ballot per 32
// marks, stopping at the first mark inside the window); every lane returns the same count.
__device__ __forceinline__ uint32_t marks_before(const pt_mark_rec* __restrict__ mk, uint32_t n, uint32_t m, uint32_t first_op, uint32_t lane) {
    uint32_t k0 = 0;
    for (uint32_t kb = 0; first_op && kb < m; kb += 32) {
        const uint32_t k = kb + lane;
        const uint32_t bal = __ballot_sync(0xffffffffu, k < m && min(__ldg(&mk[k].arrival), n) + k < first_op);
        k0 += __popc(bal);
        if (bal != 0xffffffffu) break;
    }
    return k0;
}

// The same count by one thread: the mark positions strictly increase, so k0 is the first k with min(arrival_k, n) + k >=
// first_op, found by bisection.  For callers whose lanes cut different logs or positions (pt_batch_exchange's select kernel).
__device__ __forceinline__ uint32_t marks_before_lane(const pt_mark_rec* __restrict__ mk, uint32_t n, uint32_t m, uint32_t first_op) {
    uint32_t lo = 0, hi = m;
    while (lo < hi) {
        const uint32_t k = lo + ((hi - lo) >> 1);
        if ((unsigned long long)min(__ldg(&mk[k].arrival), n) + k < first_op) lo = k + 1; else hi = k;
    }
    return lo;
}

}  // namespace ptw
