// attribute_kernel.cuh — the device side of pt_batch_attribute (include/peritext_b200.h): which change inserted, and which
// change deleted, every element of a merged log, as runs over its element sequence.
//
// attribute_resolve_kernel: one warp per request, grid-stride.  Per-warp shared memory holds two words per actor of the log
// (actor_shape's budget), A and B.  Each request has its own scratch slot: per change first and cov, per ins/del record chg,
// dkey, dcov and dchg, and an opId table of 2 slots per ins/del record.
//   1. A = the log's clock: ptct::source_clock, writing each change's list-op position into first; a table that fails it, has
//      a dep actor >= n_actors or a change whose records do not fit (ptct::change_records) is BAD_TABLE (DESIGN.md §4.3's
//      change-table rules, as for pt_batch_checkout).  first[c] becomes change c's first ins/del record and
//      cov[c] = seq_c <= B[actor_c], B being the request clock (no clock: every change is covered).
//   2. records, 32 per trip: chg[r] = the last change whose first record is <= r (bisection over first); inserts go into the
//      opId table, open addressing keyed by (ctr, actor), holding the record index (the key is read back from the record).
//   3. deletes: the target's insert record through the table, then atomicMin of the delete's packed opId (ctr << 16 | actor,
//      compareOpIds order) into dkey[target] and, for a delete in a covered change, atomicOr of 1 into dcov[target].
//   4. deletes again: the one whose opId is dkey[target] writes its change into dchg[target].  A log that merged OK has no
//      duplicate opIds and no delete of an element it does not hold, so each target has exactly one winner.
// attribute_runs_kernel<kWrite>: one warp per request over the element sequence of the last merge, 32 words per trip.  An
// element's tuple is (chg, dchg, flags) of its insert record; a run starts where the tuple differs from its predecessor's
// (shfl_up inside the trip, a carry across trips).  The count pass (kWrite = false) and the write pass run the same function,
// so they cannot disagree; build with -DPT_RENDER_CHECK (make RENDER_CHECK=1) to assert it on the device.
#pragma once
#include <cassert>
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace pta {

constexpr uint32_t kNone = 0xFFFFFFFFu;

struct AttrParams {
    const uint32_t* logs; uint32_t n; uint32_t maxR;
    const unsigned long long* clock_off; const pt_clock_entry* clock;   // request k's entries [clock_off[k], clock_off[k + 1]); null: no clock
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_insdel_rec* insdel; const pt_mark_rec* marks;
    const pt_log_result* res; const uint64_t* seq_off; const uint32_t* seq;
    const unsigned long long* chg_slot;   // [n + 1] a request's per-change scratch: its log's n_changes entries of first and cov
    const unsigned long long* rec_slot;   // [n + 1] its per-record scratch: n_insdel entries of chg, dchg, dcov, dkey; 2 n_insdel of table
    uint32_t* first; uint32_t* cov;
    uint32_t* chg; uint32_t* dchg; uint32_t* dcov; unsigned long long* dkey; uint32_t* table;
    uint32_t* status;                     // [n] PT_ATTR_*
    unsigned long long* count;            // [n] runs per request (count pass)
    const unsigned long long* off;        // [n + 1] (write pass)
    pt_attr_run* runs;
};

__device__ __forceinline__ uint32_t opid_slot(uint32_t ctr, uint32_t actor, uint32_t cap) {
    uint32_t h = ctr * 0x9E3779B1u ^ (actor + 1u) * 0x85EBCA77u;
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
    return __umulhi(h, cap);
}

// The insert record of log records ins[] whose opId is (ctr, actor), or kNone.  The table's entries were written by other
// lanes of the warp before a __syncwarp: read them at L2.
__device__ __forceinline__ uint32_t opid_find(const uint32_t* T, uint32_t cap, const uint4* __restrict__ ins, uint32_t ctr, uint32_t actor) {
    for (uint32_t s = opid_slot(ctr, actor, cap);; s = s + 1 == cap ? 0 : s + 1) {
        const uint32_t v = __ldcg(T + s);
        if (v == kNone) return kNone;
        const uint4 w = __ldg(ins + v);
        if (w.x == ctr && (w.z & 0xFFFFu) == actor && PT_PAYLOAD_KIND(w.w) == PT_KIND_INSERT) return v;
    }
}

__global__ void attribute_resolve_kernel(AttrParams P) {
    extern __shared__ uint32_t attr_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* A = attr_smem + (size_t)wib * 2 * P.maxR;
    uint32_t* B = A + P.maxR;
    for (uint32_t k = blockIdx.x * wpb + wib; k < P.n; k += gridDim.x * wpb) {
        const uint32_t log = P.logs[k];
        const pt_log_desc S = P.desc[log];
        const pt_change_desc C = P.cdesc[log];
        const uint32_t R = S.n_actors, n = C.n_changes, nI = S.n_insdel;
        const pt_change_rec* c0 = P.changes + C.change_off;
        uint32_t* first = P.first + P.chg_slot[k];
        uint32_t* cov = P.cov + P.chg_slot[k];
        uint32_t status = PT_ATTR_OK;
        // ---- 1: the table's checks, each change's first record and whether the clock covers it ----
        if (P.res[log].status != PT_LOG_OK) {
            status = PT_ATTR_LOG_FAILED;
        } else {
            for (uint32_t a = lane; a < R; a += 32) { A[a] = 0; B[a] = 0; }
            __syncwarp();
            if (!ptct::source_clock(c0, C, S, A, first, lane)) status = PT_ATTR_BAD_TABLE;
            if (status == PT_ATTR_OK && P.clock) ptct::load_clock(B, P.clock, P.clock_off[k], P.clock_off[k + 1], lane);
            __syncwarp();
            const pt_dep_rec* d0 = P.deps + C.dep_off;
            bool bad = false;
            for (uint32_t base = 0; status == PT_ATTR_OK && base < n; base += 32) {
                const uint32_t c = base + lane;
                if (c >= n) continue;
                const uint4 r = __ldg(reinterpret_cast<const uint4*>(c0 + c));
                cov[c] = !P.clock || r.x <= B[r.y & 0xFFFFu];
                for (uint32_t d = 0; d < (r.y >> 16); d++) bad |= d0[r.z + d].actor >= R;
                const ptct::Records x = ptct::change_records(P.marks + S.mark_off, S, first[c], r.w);
                bad |= !x.fits;
                first[c] = x.ins_lo;
            }
            if (__any_sync(0xffffffffu, bad)) status = PT_ATTR_BAD_TABLE;
            __syncwarp();
        }
        if (status == PT_ATTR_OK && nI) {
            const unsigned long long ro = P.rec_slot[k];
            uint32_t *chg = P.chg + ro, *dchg = P.dchg + ro, *dcov = P.dcov + ro, *T = P.table + 2 * ro;
            unsigned long long* dkey = P.dkey + ro;
            const uint32_t cap = 2 * nI;
            const uint4* ins = reinterpret_cast<const uint4*>(P.insdel + S.insdel_off);
            for (uint32_t i = lane; i < nI; i += 32) { dchg[i] = kNone; dcov[i] = 0; dkey[i] = ~0ull; T[i] = kNone; T[nI + i] = kNone; }
            __syncwarp();
            // ---- 2: each record's change; the inserts into the opId table ----
            for (uint32_t base = 0; base < nI; base += 32) {
                const uint32_t r = base + lane;
                if (r >= nI) continue;
                uint32_t lo = 0, hi = n;                       // the first change whose first record is > r; first[0] = 0
                while (lo < hi) {
                    const uint32_t m = lo + ((hi - lo) >> 1);
                    if (first[m] <= r) lo = m + 1; else hi = m;
                }
                chg[r] = lo - 1;
                const uint4 w = __ldg(ins + r);
                if (PT_PAYLOAD_KIND(w.w) == PT_KIND_INSERT)
                    for (uint32_t s = opid_slot(w.x, w.z & 0xFFFFu, cap);; s = s + 1 == cap ? 0 : s + 1)
                        if (atomicCAS(T + s, kNone, r) == kNone) break;
            }
            __syncwarp();
            // ---- 3: every delete's opId and coverage into its target ----
            for (uint32_t base = 0; base < nI; base += 32) {
                const uint32_t r = base + lane;
                if (r >= nI) continue;
                const uint4 w = __ldg(ins + r);
                if (PT_PAYLOAD_KIND(w.w) != PT_KIND_DELETE) continue;
                const uint32_t t = opid_find(T, cap, ins, w.y, w.z >> 16);
                if (t == kNone) continue;
                atomicMin(dkey + t, ((unsigned long long)w.x << 16) | (w.z & 0xFFFFu));
                if (__ldcg(cov + chg[r])) atomicOr(dcov + t, 1u);
            }
            __syncwarp();
            // ---- 4: the smallest opId's change ----
            for (uint32_t base = 0; base < nI; base += 32) {
                const uint32_t r = base + lane;
                if (r >= nI) continue;
                const uint4 w = __ldg(ins + r);
                if (PT_PAYLOAD_KIND(w.w) != PT_KIND_DELETE) continue;
                const uint32_t t = opid_find(T, cap, ins, w.y, w.z >> 16);
                if (t != kNone && __ldcg(dkey + t) == (((unsigned long long)w.x << 16) | (w.z & 0xFFFFu))) dchg[t] = chg[r];
            }
        }
        if (lane == 0) P.status[k] = status;
        __syncwarp();
    }
}

// Request k's runs: their number, and with kWrite the runs themselves at out[0 ..).  Warp-collective.
template <bool kWrite>
__device__ __forceinline__ unsigned long long attribute_walk(const AttrParams& P, uint32_t k, uint32_t lane, pt_attr_run* out) {
    const uint32_t log = P.logs[k];
    const uint32_t N = P.res[log].n_elems;
    const uint32_t* s = P.seq + P.seq_off[log];
    const unsigned long long ro = P.rec_slot[k];
    const uint32_t *chg = P.chg + ro, *dchg = P.dchg + ro, *dcov = P.dcov + ro, *cov = P.cov + P.chg_slot[k];
    const pt_change_rec* c0 = P.changes + P.cdesc[log].change_off;
    const uint32_t lt = (1u << lane) - 1u;
    unsigned long long runs = 0;
    uint32_t visible = 0, last = 0;                        // visible elements before the trip; the element the open run starts at
    uint32_t p_ci = 0, p_cd = 0, p_fl = 0;                 // the tuple of the trip's predecessor
    for (uint32_t b = 0; b < N; b += 32) {
        const uint32_t e = b + lane;
        const bool valid = e < N;
        uint32_t ci = 0, cd = kNone, fl = 0;
        if (valid) {
            const uint32_t r = __ldg(s + e) & 0x3FFFFFFFu;
            ci = __ldg(chg + r); cd = __ldg(dchg + r);
            fl = (__ldg(cov + ci) ? 0u : PT_ATTR_INSERTED_SINCE) | (cd != kNone && !__ldg(dcov + r) ? PT_ATTR_DELETED_SINCE : 0u);
        }
        uint32_t u_ci = __shfl_up_sync(0xffffffffu, ci, 1), u_cd = __shfl_up_sync(0xffffffffu, cd, 1), u_fl = __shfl_up_sync(0xffffffffu, fl, 1);
        if (lane == 0) { u_ci = p_ci; u_cd = p_cd; u_fl = p_fl; }
        const bool start = valid && (e == 0 || ci != u_ci || cd != u_cd || fl != u_fl);
        const uint32_t sb = __ballot_sync(0xffffffffu, start), vb = __ballot_sync(0xffffffffu, valid && cd == kNone);
        if (kWrite && start) {
            const unsigned long long j = runs + __popc(sb & lt);
            const uint4 ci_r = __ldg(reinterpret_cast<const uint4*>(c0 + ci));
            uint32_t d_seq = 0, d_actor = 0;
            if (cd != kNone) { const uint4 cd_r = __ldg(reinterpret_cast<const uint4*>(c0 + cd)); d_seq = cd_r.x; d_actor = cd_r.y & 0xFFFFu; }
            uint32_t* o = reinterpret_cast<uint32_t*>(out + j);
            *reinterpret_cast<uint2*>(o) = make_uint2(e, visible + __popc(vb & lt));
            o[3] = fl;
            *reinterpret_cast<uint4*>(o + 4) = make_uint4(ci_r.x, d_seq, (ci_r.y & 0xFFFFu) | (d_actor << 16), 0u);
            if (j) {                                        // the previous run ends here: its n (no other lane writes that word)
                const uint32_t below = sb & lt;
                out[j - 1].n = e - (below ? b + 31 - __clz(below) : last);
            }
        }
        if (sb) last = b + 31 - __clz(sb);
        runs += __popc(sb);
        visible += __popc(vb);
        p_ci = __shfl_sync(0xffffffffu, ci, 31); p_cd = __shfl_sync(0xffffffffu, cd, 31); p_fl = __shfl_sync(0xffffffffu, fl, 31);
    }
    if (kWrite && runs && lane == 0) out[runs - 1].n = N - last;
    return runs;
}

template <bool kWrite>
__global__ void attribute_runs_kernel(AttrParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t k = warp; k < P.n; k += nwarps) {
        const bool ok = P.status[k] == PT_ATTR_OK;
        const unsigned long long runs = ok ? attribute_walk<kWrite>(P, k, lane, kWrite ? P.runs + P.off[k] : nullptr) : 0ull;
        if (!kWrite && lane == 0) P.count[k] = runs;
#ifdef PT_RENDER_CHECK
        if (kWrite) assert(P.off[k] + runs == P.off[k + 1]);
#endif
    }
}

}  // namespace pta
