// checkout_kernel.cuh — the device side of pt_batch_checkout and pt_batch_download_clocks (include/peritext_b200.h).
//
// A version of a log is a subset of its changes: the closed form over (final position, arrival index) makes it the subset's
// records gathered in arrival order with the mark arrivals renumbered, which is what ptx::exchange_gather_kernel writes.
//
// checkout_select_kernel: one warp per request, grid-stride.  Per-warp shared memory holds two words per actor of the source
// (actor_shape's budget), A and B:
//   1. A = the source's clock: ptx::count_clock over its table, writing each change's list-op position into the request's
//      scratch slot.  A table that fails it, or whose n_ops do not sum to the log's records, is BAD_TABLE.
//   2. B = the request clock: the caller's entries (clock mode), or count_clock over the table's first changes (prefix mode: in
//      a seq-contiguous table that prefix is exactly the changes with seq <= its per-actor counts).  B[a] > A[a] is UNKNOWN.
//   3. one pass over the table: cov[k] = seq_k <= B[actor_k]; a dep actor >= n_actors or record ranges that do not fit the
//      log (any change) is BAD_TABLE, as for pt_batch_exchange's src.
//   4. the in-order pass, 32 changes per trip: A = the covered changes by actor so far, B = the trip's covered lanes by actor
//      (match_any groups: admit_kernel's scheme).  A covered change with a dep (a, d) that sees fewer than max(d, 1) covered
//      changes by a before it is NOT_CLOSED (applyChange, reference src/micromerge.ts:505-509).  Each covered change gets a
//      ptx::Delivered entry: its record ranges (ptw::marks_before_lane) and its place among the covered records (running sums).
//   5. 32 bytes of totals (ptx::PairTotals); a request that is not OK has zero counts.
// clocks_kernel: one warp per log, count_clock straight into the output.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "exchange_kernel.cuh"
#include "patch_window.cuh"

namespace ptck {

// Step 3's checks of change r (its record: seq, actor | n_deps << 16, dep_off, n_ops) at list-op position x0 of a table that
// passed count_clock: true if a dep names an actor >= R or its record ranges do not fit log S (marks mk).  *ins_lo = its first
// ins/del record.
__device__ __forceinline__ bool change_unfit(uint4 r, uint32_t x0, const pt_dep_rec* __restrict__ d0, uint32_t R, const pt_mark_rec* __restrict__ mk,
                                             const pt_log_desc& S, uint32_t* ins_lo) {
    bool bad = false;
    for (uint32_t d = 0; d < (r.y >> 16); d++) bad |= d0[r.z + d].actor >= R;
    const uint32_t x1 = x0 + r.w;
    const uint32_t k0 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x0), k1 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x1);
    *ins_lo = x0 - k0;
    return bad || k0 > x0 || k1 > x1 || k1 < k0 || x1 - k1 > S.n_insdel || x1 - k1 < x0 - k0;   // arrivals that do not fit the table
}

struct CheckoutParams {
    const uint32_t* logs; uint32_t n; uint32_t maxR;
    const uint32_t* n_changes;                                          // [n] prefix mode, or null
    const unsigned long long* clock_off; const pt_clock_entry* clock;   // clock mode: request k's entries [clock_off[k], clock_off[k + 1])
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_mark_rec* marks;
    const unsigned long long* slot_off;   // [n + 1] a request's scratch slot: its source's n_changes entries of pos, cov and dlv
    uint32_t* pos; uint32_t* cov; ptx::Delivered* dlv;
    ptx::PairTotals* totals;
};

__global__ void checkout_select_kernel(CheckoutParams P) {
    extern __shared__ uint32_t cko_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
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
        ptx::Delivered* dlv = P.dlv + P.slot_off[k];
        // ---- 1, 2: the source's clock and the request's ----
        unsigned long long ops = 0;
        uint32_t status = PT_CHECKOUT_OK;
        if (!ptx::count_clock(c0, n, C.n_deps, R, A, pos, &ops, lane) || ops != (unsigned long long)S.n_insdel + S.n_mark || ops > 0xFFFFFFFFull)
            status = PT_CHECKOUT_BAD_TABLE;
        bool unknown = false;
        if (status == PT_CHECKOUT_OK) {
            if (P.n_changes) {
                ptx::count_clock(c0, min(P.n_changes[k], n), C.n_deps, R, B, nullptr, nullptr, lane);   // a prefix of a table that passed
            } else {
                for (unsigned long long e = P.clock_off[k] + lane; e < P.clock_off[k + 1]; e += 32) {   // actors < R and distinct (host)
                    const pt_clock_entry q = P.clock[e];
                    B[q.actor] = q.seq;
                }
            }
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
            uint32_t ins_lo;
            bad |= change_unfit(r, pos[c], d0, R, mk, S, &ins_lo);
        }
        if (__any_sync(0xffffffffu, bad)) status = PT_CHECKOUT_BAD_TABLE;
        else if (unknown) status = PT_CHECKOUT_UNKNOWN;
        // ---- 4: closure, in table order, and the covered changes' places ----
        uint32_t t_ins = 0, t_mk = 0, t_ch = 0, t_dep = 0;
        __syncwarp();
        for (uint32_t a = lane; a < R; a += 32) { A[a] = 0; B[a] = 0; }
        __syncwarp();
        for (uint32_t base = 0; status == PT_CHECKOUT_OK && base < n; base += 32) {
            const uint32_t c = base + lane;
            uint4 r = make_uint4(0, 0, 0, 0);
            bool in = false;
            if (c < n) { r = __ldg(reinterpret_cast<const uint4*>(c0 + c)); in = cov[c] != 0; }
            const uint32_t actor = r.y & 0xFFFFu;
            const uint32_t mask = __match_any_sync(0xffffffffu, in ? actor : (0x10000u + lane));
            const bool leader = (mask & lt) == 0;
            if (in && leader) B[actor] = mask;
            __syncwarp();
            bool open = false;
            for (uint32_t d = 0; in && d < (r.y >> 16); d++) {
                const pt_dep_rec q = d0[r.z + d];
                const uint32_t have = A[q.actor] + __popc(B[q.actor] & lt);
                if (have == 0 || have < q.seq) { open = true; break; }
            }
            if (__any_sync(0xffffffffu, open)) { status = PT_CHECKOUT_NOT_CLOSED; break; }
            uint32_t ins_lo = 0, ins_n = 0, mk_lo = 0, mk_n = 0;
            if (in) {
                const uint32_t x0 = pos[c], x1 = x0 + r.w;
                const uint32_t k0 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x0), k1 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x1);
                ins_lo = x0 - k0; ins_n = (x1 - k1) - ins_lo; mk_lo = k0; mk_n = k1 - k0;
            }
            const uint32_t pass = __ballot_sync(0xffffffffu, in);
            uint32_t n_i, n_m, n_d;
            const uint32_t e_i = ptx::warp_excl_scan(ins_n, lane, n_i), e_m = ptx::warp_excl_scan(mk_n, lane, n_m),
                           e_d = ptx::warp_excl_scan(in ? (r.y >> 16) : 0u, lane, n_d);
            if (in) dlv[t_ch + __popc(pass & lt)] = ptx::Delivered{c, ins_lo, mk_lo, ins_n, mk_n, t_ins + e_i, t_mk + e_m, t_dep + e_d};
            t_ins += n_i; t_mk += n_m; t_dep += n_d; t_ch += __popc(pass);
            __syncwarp();
            if (in && leader) { A[actor] += __popc(mask); B[actor] = 0; }
            __syncwarp();
        }
        if (lane == 0)
            P.totals[k] = status == PT_CHECKOUT_OK ? ptx::PairTotals{t_ins, t_mk, t_ch, t_dep, 0u, PT_CHECKOUT_OK, 0u, 0u}
                                                   : ptx::PairTotals{0u, 0u, 0u, 0u, 0u, status, 0u, 0u};
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
        const bool ok = ptx::count_clock(changes + C.change_off, C.n_changes, C.n_deps, R, out, nullptr, nullptr, lane);
        __syncwarp();
        if (!ok) for (uint32_t a = lane; a < R; a += 32) out[a] = 0;
        if (lane == 0) status[i] = ok ? PT_CHECKOUT_OK : PT_CHECKOUT_BAD_TABLE;
        __syncwarp();
    }
}

}  // namespace ptck
