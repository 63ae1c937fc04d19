// exchange_kernel.cuh — the device side of pt_batch_exchange (include/peritext_b200.h): which changes of log src log dst is
// missing, in the order applyChanges admits them, and the gather of their records into a delta in dst's id space.
//
// exchange_select_kernel: one warp per pair, grid-stride.  Per-warp shared memory holds dst's clock (by dst actor rank) and a
// per-src-actor word (first the actor's change count, then the queue slot of its first missing change).
//   1. clocks: ptct::count_clock over dst's table, ptct::source_clock over src's (with each change's list-op position into the
//      pair's scratch slot).
//   2. queue, getMissingChanges order: ptct::missing_queue, with dst's clock through the actor map.
//   3. delivery, applyChanges order (test/merge.ts:4-23): repeated in-order passes over the queue, 32 candidates per trip.
//      All lanes test seq and deps against the clock of the trip's start.  A pass is final (clocks only grow, and a
//      seq-contiguous table has no second change with the same actor and seq); a lane that failed is tested again in lane
//      order, after the clock bumps of the delivered lanes before it, so it sees exactly what the reference's queue front
//      would.  Lanes that fail stay in the queue (compacted in place) for the next pass; a pass that delivers nothing ends
//      the pair with PT_EXCHANGE_STUCK.
//    A delivered change's record ranges come from its list-op positions (ptct::change_records), and ptct::place_delivered
//    gives it its place in the delta.
// exchange_gather_kernel: one warp per delivered change (blockIdx.y slices a long change, as splice_records_kernel slices a
// long log): 16-byte coalesced copies with the pair's actor and counter maps applied (a mark is a lane pair, as in the
// splice), mark arrivals rebased onto dst's records; slice 0 also writes the change record, its deps and the delivered index.
// An id without an image sets the pair's status, and the host drops that pair's delta.  pt_batch_checkout runs it too, with
// identity maps and empty dst logs (checkout_kernel.cuh).
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace ptx {

// One pair's maps, src id space -> dst id space.  The actor map has exactly src's n_actors entries; a == null (pt_batch_checkout)
// is the identity actor map and nc == 0 the identity counter map.  No image: 0xFFFF / 0xFFFFFFFF.
struct PairMaps {
    const uint16_t* a; uint32_t na;
    const uint32_t* c; uint32_t nc;
    __device__ __forceinline__ uint32_t actor(uint32_t x) const { return a ? (x < na ? (uint32_t)__ldg(a + x) : 0xFFFFu) : x; }
    __device__ __forceinline__ uint32_t ctr(uint32_t x) const { return nc ? (x < nc ? __ldg(c + x) : 0xFFFFFFFFu) : x; }
    // the actor of an id whose counter is ctr_old: counter 0 is HEAD / a text boundary and names no actor
    __device__ __forceinline__ uint32_t id_actor(uint32_t ctr_old, uint32_t x) const { return ctr_old ? actor(x) : x; }
};

struct ExchangeParams {
    const pt_exchange_pair* pairs; uint32_t n_pairs; uint32_t maxR;
    const unsigned long long* actor_off; const uint16_t* actor_map;    // actor_off null: identity for every pair (gather only)
    const unsigned long long* ctr_off;  const uint32_t* ctr_map;       // ctr_off null: identity for every pair
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_insdel_rec* insdel; const pt_mark_rec* marks;
    const unsigned long long* slot_off;   // [n_pairs + 1] a pair's scratch slot: src's n_changes entries of queue, pos and dlv
    uint32_t* queue; uint32_t* pos; ptct::Delivered* dlv;
    ptct::PairTotals* totals;
    // gather only
    const unsigned long long* dlv_off;    // [n_pairs + 1] exclusive scan of the pairs' delivered changes
    unsigned long long n_dlv;
    const ptct::PairBase* base;
    const pt_log_desc* dst_desc;          // the descriptors a pair's dst indexes: desc, or a checkout's empty logs
    pt_insdel_rec* out_insdel; pt_mark_rec* out_marks; pt_change_rec* out_changes; pt_dep_rec* out_deps;
    uint32_t* out_delivered;              // may be null
};

__device__ __forceinline__ PairMaps pair_maps(const ExchangeParams& P, uint32_t p) {
    PairMaps m{nullptr, 0u, nullptr, 0u};
    if (P.actor_off) { const unsigned long long ao = P.actor_off[p]; m.a = P.actor_map + ao; m.na = (uint32_t)(P.actor_off[p + 1] - ao); }
    if (P.ctr_off) { const unsigned long long o = P.ctr_off[p]; m.c = P.ctr_map + o; m.nc = (uint32_t)(P.ctr_off[p + 1] - o); }
    return m;
}

// applyChange's admission test (reference src/micromerge.ts:501-509) of a src change against dst's clock; the change's and
// its deps' actors are known to have images (step 2 checked them).
__device__ __forceinline__ bool admits(const PairMaps& m, const uint32_t* clk, const pt_dep_rec* __restrict__ d0, uint4 r) {
    if (r.x != clk[m.actor(r.y & 0xFFFFu)] + 1u) return false;
    for (uint32_t d = 0; d < (r.y >> 16); d++) {
        const pt_dep_rec q = d0[r.z + d];
        const uint32_t have = clk[m.actor(q.actor)];
        if (have == 0 || have < q.seq) return false;
    }
    return true;
}

__global__ void exchange_select_kernel(ExchangeParams P) {
    extern __shared__ uint32_t xch_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t* clk = xch_smem + (size_t)wib * 2 * P.maxR;     // dst's clock, by dst actor rank
    uint32_t* cs = clk + P.maxR;                             // by src actor rank: change count, then first queue slot
    for (uint32_t p = blockIdx.x * wpb + wib; p < P.n_pairs; p += gridDim.x * wpb) {
        const pt_exchange_pair pr = P.pairs[p];
        const pt_log_desc S = P.desc[pr.src], D = P.desc[pr.dst];
        const pt_change_desc CS = P.cdesc[pr.src], CD = P.cdesc[pr.dst];
        const PairMaps m = pair_maps(P, p);
        const uint32_t Rs = S.n_actors, Rd = D.n_actors;
        for (uint32_t a = lane; a < Rd; a += 32) clk[a] = 0;
        for (uint32_t a = lane; a < Rs; a += 32) cs[a] = 0;
        __syncwarp();
        const pt_change_rec* c0 = P.changes + CS.change_off;
        const pt_dep_rec* d0 = P.deps + CS.dep_off;
        uint32_t* queue = P.queue + P.slot_off[p];
        uint32_t* pos = P.pos + P.slot_off[p];
        ptct::Delivered* dlv = P.dlv + P.slot_off[p];
        uint32_t status = PT_EXCHANGE_OK;
        if (!ptct::count_clock(P.changes + CD.change_off, CD.n_changes, CD.n_deps, Rd, clk, nullptr, nullptr, lane) ||
            !ptct::source_clock(c0, CS, S, cs, pos, lane))
            status = PT_EXCHANGE_BAD_TABLE;
        // ---- step 2: the queue ----
        uint32_t nq = 0;
        if (status == PT_EXCHANGE_OK) {
            bool bad = false, unmapped = false;
            nq = ptct::missing_queue(c0, CS.n_changes, cs,
                                     [&](uint32_t actor) { const uint32_t ma = m.actor(actor); return ma < Rd ? clk[ma] : 0u; },   // no rank in dst: 0
                                     [&](uint32_t k, uint4 r, uint32_t slot) {
                                         queue[slot] = k;
                                         if (m.actor(r.y & 0xFFFFu) >= Rd) unmapped = true;
                                         for (uint32_t d = 0; d < (r.y >> 16); d++) {
                                             const uint32_t da = d0[r.z + d].actor;
                                             if (da >= Rs) bad = true;
                                             else if (m.actor(da) >= Rd) unmapped = true;
                                         }
                                     }, lane);
            if (__any_sync(0xffffffffu, bad)) status = PT_EXCHANGE_BAD_TABLE;
            else if (__any_sync(0xffffffffu, unmapped)) status = PT_EXCHANGE_UNMAPPED;
        }
        // ---- step 3: delivery ----
        ptct::PairTotals t{};                                 // the delivered changes' running totals; status PT_EXCHANGE_OK
        const pt_mark_rec* mk = P.marks + S.mark_off;
        uint32_t remaining = nq;
        __syncwarp();
        while (status == PT_EXCHANGE_OK && remaining) {
            uint32_t kept = 0;
            const uint32_t before = t.n_changes;
            for (uint32_t base = 0; base < remaining && status == PT_EXCHANGE_OK; base += 32) {
                const bool valid = base + lane < remaining;
                const uint32_t c = valid ? queue[base + lane] : 0u;
                uint4 r = make_uint4(0, 0, 0, 0);
                if (valid) r = __ldg(reinterpret_cast<const uint4*>(c0 + c));
                const uint32_t ma = m.actor(r.y & 0xFFFFu);
                bool ok = valid && admits(m, clk, d0, r);
                const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
                uint32_t pass = __ballot_sync(0xffffffffu, ok), applied = 0;
                // failing lanes in lane order: first the bumps of the delivered lanes before them, then their test again
                for (uint32_t fail = vmask & ~pass; fail; fail &= fail - 1) {
                    const uint32_t f = __ffs(fail) - 1, due = pass & ((1u << f) - 1u) & ~applied;
                    if ((due >> lane) & 1u) atomicMax(&clk[ma], r.x);
                    applied |= due;
                    __syncwarp();
                    if (lane == f) ok = admits(m, clk, d0, r);
                    pass |= __ballot_sync(0xffffffffu, lane == f && ok);
                }
                if (((pass & ~applied) >> lane) & 1u) atomicMax(&clk[ma], r.x);
                __syncwarp();
                // the delivered lanes' record ranges and their places in the delta (pass is ballot(ok))
                ptct::Records x{};
                if (ok) x = ptct::change_records(mk, S, pos[c], r.w);
                if (__any_sync(0xffffffffu, ok && !x.fits)) { status = PT_EXCHANGE_BAD_TABLE; break; }
                ptct::place_delivered(dlv, ok, c, x, r.y >> 16, lane, t);
                // the others go back to the queue; slot kept + rank <= base + lane, which this trip has already read
                if (valid && !ok) queue[kept + __popc(vmask & ~pass & lt)] = c;
                kept += __popc(vmask & ~pass);
                __syncwarp();
            }
            if (status == PT_EXCHANGE_OK && t.n_changes == before) status = PT_EXCHANGE_STUCK;
            remaining = kept;
        }
        if (lane == 0)
            P.totals[p] = status == PT_EXCHANGE_OK ? t : ptct::PairTotals{0u, 0u, 0u, 0u, 0u, status, 0u, 0u};
        __syncwarp();
    }
}

__global__ void exchange_gather_kernel(ExchangeParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t first = blockIdx.y * 32u + lane, step = gridDim.y * 32u;       // this warp's slice of each change
    for (unsigned long long j = warp; j < P.n_dlv; j += nwarps) {
        uint32_t lo = 0, hi = P.n_pairs;                   // the pair: the last p with dlv_off[p] <= j
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (P.dlv_off[mid] <= j) lo = mid; else hi = mid; }
        const uint32_t p = lo, k = (uint32_t)(j - P.dlv_off[p]);
        const pt_exchange_pair pr = P.pairs[p];
        const pt_log_desc S = P.desc[pr.src], D = P.dst_desc[pr.dst];
        const PairMaps m = pair_maps(P, p);
        const ptct::PairBase B = P.base[p];
        const ptct::Delivered d = P.dlv[P.slot_off[p] + k];
        uint32_t top = 0;                                  // the largest mapped opId counter this lane wrote
        bool unmapped = false;
        auto ctr = [&](uint32_t c) { const uint32_t x = m.ctr(c); unmapped |= x == 0xFFFFFFFFu; return x; };
        auto id_actor = [&](uint32_t c, uint32_t a) { const uint32_t x = m.id_actor(c, a); unmapped |= c && x == 0xFFFFu; return x; };
        // ins/del records: {ctr, ref_ctr, actor | ref_actor << 16, payload}
        const uint4* is = reinterpret_cast<const uint4*>(P.insdel + S.insdel_off + d.ins_lo);
        uint4* id = reinterpret_cast<uint4*>(P.out_insdel + B.insdel + d.ins_off);
        for (uint32_t i = first; i < d.n_insdel; i += step) {
            uint4 r = __ldg(is + i);
            const uint32_t a = id_actor(r.x, r.z & 0xFFFFu), ra = id_actor(r.y, r.z >> 16);
            r.x = ctr(r.x); r.y = ctr(r.y); r.z = (a & 0xFFFFu) | (ra << 16);
            top = max(top, r.x);
            id[i] = r;
        }
        // mark records, two words each: A = {ctr, actor | kind << 16 | bounds << 24, start_ctr, end_ctr},
        // B = {start_actor | end_actor << 16, attr, arrival, reserved}
        const uint4* ms = reinterpret_cast<const uint4*>(P.marks + S.mark_off + d.mk_lo);
        uint4* md = reinterpret_cast<uint4*>(P.out_marks + B.mark + d.mk_off);
        const uint32_t nq = 2u * d.n_mark;
        for (uint32_t base = first - lane; base < nq; base += step) {             // 32-aligned: a mark's two words share a trip
            const uint32_t i = base + lane;
            const bool valid = i < nq;
            uint4 q = valid ? __ldg(ms + i) : make_uint4(0, 0, 0, 0);
            const uint32_t pz = __shfl_xor_sync(0xffffffffu, q.z, 1), pw = __shfl_xor_sync(0xffffffffu, q.w, 1);
            if (!valid) continue;
            if (!(lane & 1u)) {
                const uint32_t a = id_actor(q.x, q.y & 0xFFFFu);
                q.x = ctr(q.x); q.y = (q.y & 0xFFFF0000u) | (a & 0xFFFFu); q.z = ctr(q.z); q.w = ctr(q.w);
                top = max(top, q.x);
            } else {
                const uint32_t sa = id_actor(pz, q.x & 0xFFFFu), ea = id_actor(pw, q.x >> 16);
                q.x = (sa & 0xFFFFu) | (ea << 16);
                // arrival: dst's old records, then the delivered ins/del records before the mark
                const uint32_t within = q.z < d.ins_lo ? 0u : min(q.z - d.ins_lo, d.n_insdel);
                q.z = D.n_insdel + d.ins_off + within;
            }
            md[i] = q;
        }
        if (blockIdx.y == 0) {
            // change record {seq, actor | n_deps << 16, dep_off, n_ops} and its deps {seq, actor | reserved << 16}
            const pt_change_desc CS = P.cdesc[pr.src];
            uint4 r = __ldg(reinterpret_cast<const uint4*>(P.changes + CS.change_off + d.change));
            const uint2* ps = reinterpret_cast<const uint2*>(P.deps + CS.dep_off + r.z);
            uint2* pd = reinterpret_cast<uint2*>(P.out_deps + B.dep + d.dep_off);
            for (uint32_t t = lane; t < (r.y >> 16); t += 32) {
                uint2 q = __ldg(ps + t);
                const uint32_t a = m.actor(q.y & 0xFFFFu);
                unmapped |= a == 0xFFFFu;
                q.y = (q.y & 0xFFFF0000u) | a;
                pd[t] = q;
            }
            if (lane == 0) {
                const uint32_t a = m.actor(r.y & 0xFFFFu);
                unmapped |= a == 0xFFFFu;
                r.y = (r.y & 0xFFFF0000u) | a; r.z = d.dep_off;
                reinterpret_cast<uint4*>(P.out_changes + B.change)[k] = r;
                if (P.out_delivered) P.out_delivered[j] = d.change;
            }
        }
        for (int o = 16; o > 0; o >>= 1) top = max(top, __shfl_xor_sync(0xffffffffu, top, o));
        const bool any_unmapped = __any_sync(0xffffffffu, unmapped);
        if (lane == 0) {
            if (top) atomicMax(&P.totals[p].max_ctr, top);
            if (any_unmapped) atomicMax(&P.totals[p].status, (uint32_t)PT_EXCHANGE_UNMAPPED);
        }
    }
}

}  // namespace ptx
