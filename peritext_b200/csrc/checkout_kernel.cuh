// checkout_kernel.cuh — the device side of pt_batch_checkout and pt_batch_download_clocks (include/peritext_b200.h).
//
// A version of a log is a subset of its changes: the closed form over (final position, arrival index) makes it the subset's
// records gathered in arrival order with the mark arrivals renumbered, which is what ptx::exchange_gather_kernel writes.
// The change-table rules (ptct::) are DESIGN.md §4.3's.
//
// checkout_select_kernel: one warp per request, grid-stride.  Per-warp shared memory holds two words per actor of the source
// (actor_shape's budget), A and B:
//   1. A = the source's clock: ptct::source_clock, writing each change's list-op position into the request's scratch slot.  A
//      table that fails it is BAD_TABLE.
//   2. B = the request clock: the caller's entries (clock mode), or count_clock over the table's first changes (prefix mode: in
//      a seq-contiguous table that prefix is exactly the changes with seq <= its per-actor counts).  B[a] > A[a] is UNKNOWN.
//   3. one pass over the table: cov[k] = seq_k <= B[actor_k]; a dep actor >= n_actors or record ranges that do not fit the
//      log (any change) is BAD_TABLE, as for pt_batch_exchange's src.
//   4. the in-order pass over the covered changes (ptct::TripClock on A and B): a covered change with a dep (a, d) that sees
//      fewer than max(d, 1) covered changes by a before it is NOT_CLOSED (applyChange, reference src/micromerge.ts:505-509).
//      Each covered change gets its record ranges and a ptct::Delivered entry (ptct::place_delivered).
//   5. 32 bytes of totals (ptct::PairTotals); a request that is not OK has zero counts.
// clocks_kernel: one warp per log, count_clock straight into the output.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace ptck {

struct CheckoutParams {
    const uint32_t* logs; uint32_t n; uint32_t maxR;
    const uint32_t* n_changes;                                          // [n] prefix mode, or null
    const unsigned long long* clock_off; const pt_clock_entry* clock;   // clock mode: request k's entries [clock_off[k], clock_off[k + 1])
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_mark_rec* marks;
    const unsigned long long* slot_off;   // [n + 1] a request's scratch slot: its source's n_changes entries of pos, cov and dlv
    uint32_t* pos; uint32_t* cov; ptct::Delivered* dlv;
    ptct::PairTotals* totals;
};

__global__ void checkout_select_kernel(CheckoutParams P) {
    extern __shared__ uint32_t cko_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* A = cko_smem + (size_t)wib * 2 * P.maxR;
    uint32_t* B = A + P.maxR;
    for (uint32_t k = blockIdx.x * wpb + wib; k < P.n; k += gridDim.x * wpb) {
        const uint32_t src = P.logs[k];
        const pt_log_desc S = P.desc[src];
        const pt_change_desc C = P.cdesc[src];
        const uint32_t R = S.n_actors, n = C.n_changes;
        for (uint32_t a = lane; a < R; a += 32) { A[a] = 0; B[a] = 0; }
        __syncwarp();
        const pt_change_rec* c0 = P.changes + C.change_off;
        const pt_dep_rec* d0 = P.deps + C.dep_off;
        const pt_mark_rec* mk = P.marks + S.mark_off;
        uint32_t* pos = P.pos + P.slot_off[k];
        uint32_t* cov = P.cov + P.slot_off[k];
        ptct::Delivered* dlv = P.dlv + P.slot_off[k];
        // ---- 1, 2: the source's clock and the request's ----
        uint32_t status = ptct::source_clock(c0, C, S, A, pos, lane) ? PT_CHECKOUT_OK : PT_CHECKOUT_BAD_TABLE;
        bool unknown = false;
        if (status == PT_CHECKOUT_OK) {
            if (P.n_changes) ptct::count_clock(c0, min(P.n_changes[k], n), C.n_deps, R, B, nullptr, nullptr, lane);   // a prefix of a table that passed
            else ptct::load_clock(B, P.clock, P.clock_off[k], P.clock_off[k + 1], lane);
            __syncwarp();
            for (uint32_t a = lane; a < R; a += 32) unknown |= B[a] > A[a];
            unknown = __any_sync(0xffffffffu, unknown);
        }
        // ---- 3: covered flags, and the table's dep actors and record ranges ----
        bool bad = false;
        for (uint32_t base = 0; status == PT_CHECKOUT_OK && base < n; base += 32) {
            const uint32_t c = base + lane;
            if (c >= n) continue;
            const uint4 r = __ldg(reinterpret_cast<const uint4*>(c0 + c));
            cov[c] = r.x <= B[r.y & 0xFFFFu];
            for (uint32_t d = 0; d < (r.y >> 16); d++) bad |= d0[r.z + d].actor >= R;
            bad |= !ptct::change_records(mk, S, pos[c], r.w).fits;
        }
        if (__any_sync(0xffffffffu, bad)) status = PT_CHECKOUT_BAD_TABLE;
        else if (unknown) status = PT_CHECKOUT_UNKNOWN;
        // ---- 4: closure, in table order, and the covered changes' places ----
        ptct::PairTotals t{};                                 // the covered changes' running totals; status PT_CHECKOUT_OK
        __syncwarp();
        for (uint32_t a = lane; a < R; a += 32) { A[a] = 0; B[a] = 0; }
        __syncwarp();
        ptct::TripClock clk(A, B, lane);
        for (uint32_t base = 0; status == PT_CHECKOUT_OK && base < n; base += 32) {
            const uint32_t c = base + lane;
            uint4 r = make_uint4(0, 0, 0, 0);
            bool in = false;
            if (c < n) { r = __ldg(reinterpret_cast<const uint4*>(c0 + c)); in = cov[c] != 0; }
            clk.group(in, r.y & 0xFFFFu, lane);
            bool open = false;
            for (uint32_t d = 0; in && d < (r.y >> 16); d++) {
                const pt_dep_rec q = d0[r.z + d];
                const uint32_t have = clk.have(q.actor);
                if (have == 0 || have < q.seq) { open = true; break; }
            }
            if (__any_sync(0xffffffffu, open)) { status = PT_CHECKOUT_NOT_CLOSED; break; }
            ptct::Records x{};
            if (in) x = ptct::change_records(mk, S, pos[c], r.w);
            ptct::place_delivered(dlv, in, c, x, r.y >> 16, lane, t);
            clk.commit();
        }
        if (lane == 0) P.totals[k] = status == PT_CHECKOUT_OK ? t : ptct::PairTotals{0u, 0u, 0u, 0u, 0u, status, 0u, 0u};
        __syncwarp();
    }
}

// pt_batch_download_clocks: seq[off[i] + a] = log i's changes by actor rank a; a table that fails count_clock reads as zeros
// with status PT_CHECKOUT_BAD_TABLE.
__global__ void clocks_kernel(const pt_change_desc* __restrict__ cdesc, const pt_change_rec* __restrict__ changes, const pt_log_desc* __restrict__ desc,
                              uint32_t n_logs, const unsigned long long* __restrict__ off, uint32_t* seq, uint32_t* __restrict__ status) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n_logs; i += nwarps) {
        const pt_change_desc C = cdesc[i];
        const uint32_t R = desc[i].n_actors;
        uint32_t* out = seq + off[i];
        for (uint32_t a = lane; a < R; a += 32) out[a] = 0;
        __syncwarp();
        const bool ok = ptct::count_clock(changes + C.change_off, C.n_changes, C.n_deps, R, out, nullptr, nullptr, lane);
        __syncwarp();
        if (!ok) for (uint32_t a = lane; a < R; a += 32) out[a] = 0;
        if (lane == 0) status[i] = ok ? PT_CHECKOUT_OK : PT_CHECKOUT_BAD_TABLE;
        __syncwarp();
    }
}

}  // namespace ptck
