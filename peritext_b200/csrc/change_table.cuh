// change_table.cuh — the rules every kernel that walks a log's change table shares (DESIGN.md §4.3, "Change-table rules"):
// admission, pt_batch_exchange, pt_batch_sync_pairs, pt_batch_render_changes_json, pt_batch_checkout / pt_batch_download_clocks
// and pt_batch_attribute.  Each rule is written here once; the kernel files keep only their own steps.  All of it is
// warp-level: one warp per log, request or pair, one lane per change, 32 changes per trip.
#pragma once
#include <cstdint>
#include <type_traits>

#include "../../include/peritext_b200.h"
#include "patch_window.cuh"

namespace ptct {

struct PairTotals { uint32_t n_insdel, n_mark, n_changes, n_deps, max_ctr, status, reserved0, reserved1; };   // 32 B per pair
struct Delivered {          // one per delivered change, in delivery order.  32 B
    uint32_t change;                    // index in src's change table
    uint32_t ins_lo, mk_lo;             // its first ins/del and mark record in src's log
    uint32_t n_insdel, n_mark;
    uint32_t ins_off, mk_off, dep_off;  // its place among the pair's delivered records
};
struct PairBase { unsigned long long insdel, mark, change, dep; };   // where a pair's records start in the delta arrays

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t lane, uint32_t& total) {
    uint32_t s = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, d); if (lane >= (uint32_t)d) s += y; }
    total = __shfl_sync(0xffffffffu, s, 31);
    return s - v;
}

// A table's clock: cnt[actor] = the actor's changes (cnt zeroed by the caller); false if a change names an actor >= R, breaks
// seq == count + 1, or its deps leave the log's dep records.  match_any groups give each change its rank among the trip's
// changes of the same actor.  cnt nullptr: no clock, only the dep-range check (told apart by type, so that the clock's callers
// carry no test of it).  With pos: pos[k] = sum of n_ops before change k (its list-op position), *ops = the sum over the table.
template <class Cnt>
__device__ __forceinline__ bool count_clock(const pt_change_rec* __restrict__ c0, uint32_t n, uint32_t n_deps, uint32_t R, Cnt cnt,
                                            uint32_t* __restrict__ pos, unsigned long long* ops, uint32_t lane) {
    constexpr bool kClock = !std::is_same_v<Cnt, std::nullptr_t>;
    uint32_t* const clk = cnt;
    const uint32_t lt = (1u << lane) - 1u;
    unsigned long long run = 0;
    bool ok = true;
    for (uint32_t base = 0; base < n && ok; base += 32) {
        const uint32_t k = base + lane;
        const bool valid = k < n;
        uint4 r = make_uint4(0, 0, 0, 0);
        if (valid) r = __ldg(reinterpret_cast<const uint4*>(c0 + k));
        const uint32_t actor = r.y & 0xFFFFu;
        const bool aok = valid && actor < R;
        const uint32_t mask = kClock ? __match_any_sync(0xffffffffu, aok ? actor : (0x10000u + lane)) : 0u;
        const bool bad = valid && ((kClock && (!aok || r.x != clk[aok ? actor : 0] + __popc(mask & lt) + 1u)) || (unsigned long long)r.z + (r.y >> 16) > n_deps);
        ok = !__any_sync(0xffffffffu, bad);
        if (pos) {
            uint32_t tot;
            const uint32_t ex = warp_excl_scan(valid ? r.w : 0u, lane, tot);   // a trip's n_ops can wrap only in a table the total check refuses
            unsigned long long wide = valid ? r.w : 0u;
            for (int o = 16; o > 0; o >>= 1) wide += __shfl_xor_sync(0xffffffffu, wide, o);
            if (valid) pos[k] = (uint32_t)run + ex;
            run += wide;
        }
        if (kClock) {
            __syncwarp();
            if (aok && (mask & lt) == 0) clk[actor] += __popc(mask);
            __syncwarp();
        }
    }
    if (ops) *ops = run;
    return ok;
}

// The checks a source table passes before its changes' records are read: count_clock of log S's table c0 (descriptor C) into
// cnt with the list-op positions into pos, and n_ops summing to S's records (so every position fits 32 bits).
__device__ __forceinline__ bool source_clock(const pt_change_rec* __restrict__ c0, const pt_change_desc& C, const pt_log_desc& S, uint32_t* cnt,
                                             uint32_t* __restrict__ pos, uint32_t lane) {
    unsigned long long ops = 0;
    return count_clock(c0, C.n_changes, C.n_deps, S.n_actors, cnt, pos, &ops, lane) &&
           ops == (unsigned long long)S.n_insdel + S.n_mark && ops <= 0xFFFFFFFFull;
}

// A change's records in log S (marks mk), from its list-op positions [x0, x0 + n_ops): the marks before position X are the
// first k with min(arrival_k, n) + k >= X (ptw::marks_before_lane), the ins/del records before it X - k.  !fits: arrivals that
// do not fit the table; the ranges are then meaningless.
struct Records { uint32_t ins_lo, n_insdel, mk_lo, n_mark; bool fits; };
__device__ __forceinline__ Records change_records(const pt_mark_rec* __restrict__ mk, const pt_log_desc& S, uint32_t x0, uint32_t n_ops) {
    const uint32_t x1 = x0 + n_ops;
    const uint32_t k0 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x0), k1 = ptw::marks_before_lane(mk, S.n_insdel, S.n_mark, x1);
    const bool fits = !(k0 > x0 || k1 > x1 || k1 < k0 || x1 - k1 > S.n_insdel || x1 - k1 < x0 - k0);
    return Records{x0 - k0, (x1 - k1) - (x0 - k0), k0, k1 - k0, fits};
}

// applyChange's clock over a table taken in order, 32 changes per trip (reference src/micromerge.ts:499-511).  As long as every
// earlier change was applied, clock[a] is the number of earlier changes by a, so each lane is checked on its own against
// cnt[a] (changes by a in earlier trips, in shared memory) plus its rank among the trip's lanes of a (cmask[a], from the
// match_any leader).  Both arrays are zeroed by the caller and left zeroed by commit.
struct TripClock {
    uint32_t* cnt; uint32_t* cmask; uint32_t lt;
    uint32_t mask, actor; bool in;
    __device__ __forceinline__ TripClock(uint32_t* cnt_, uint32_t* cmask_, uint32_t lane) : cnt(cnt_), cmask(cmask_), lt((1u << lane) - 1u), mask(0), actor(0), in(false) {}
    // this lane's change, of actor a, takes part (in) or not.  Warp-collective.
    __device__ __forceinline__ void group(bool in_, uint32_t a, uint32_t lane) {
        in = in_; actor = a;
        mask = __match_any_sync(0xffffffffu, in ? a : (0x10000u + lane));
        if (in && (mask & lt) == 0) cmask[a] = mask;
        __syncwarp();
    }
    __device__ __forceinline__ uint32_t have(uint32_t a) const { return cnt[a] + __popc(cmask[a] & lt); }
    // the trip's changes are applied.  Warp-collective.
    __device__ __forceinline__ void commit() {
        __syncwarp();
        if (in && (mask & lt) == 0) { cnt[actor] += __popc(mask); cmask[actor] = 0; }
        __syncwarp();
    }
};

// The lane's change c (if in, with records x and n_deps deps; x zero and n_deps ignored otherwise) goes to
// dlv[t.n_changes + its rank among the trip's delivered lanes]; its records' places follow the running totals t, which then
// take the trip's.  Warp-collective.
__device__ __forceinline__ void place_delivered(Delivered* dlv, bool in, uint32_t c, const Records& x, uint32_t n_deps, uint32_t lane, PairTotals& t) {
    const uint32_t pass = __ballot_sync(0xffffffffu, in);
    uint32_t n_i, n_m, n_d;
    const uint32_t e_i = warp_excl_scan(x.n_insdel, lane, n_i), e_m = warp_excl_scan(x.n_mark, lane, n_m),
                   e_d = warp_excl_scan(in ? n_deps : 0u, lane, n_d);
    if (in) dlv[t.n_changes + __popc(pass & ((1u << lane) - 1u))] = Delivered{c, x.ins_lo, x.mk_lo, x.n_insdel, x.n_mark, t.n_insdel + e_i, t.n_mark + e_m, t.n_deps + e_d};
    t.n_insdel += n_i; t.n_mark += n_m; t.n_deps += n_d; t.n_changes += __popc(pass);
}

// The actors of a seq-contiguous table c0[0 .. n) in the order it first shows them (the insertion order of Micromerge.clock): an
// actor's first change is its seq 1, so that is the table order of the seq-1 changes (missing_queue's rule).  shown(actor, k) is
// called for the k-th; returns their number.  Warp-collective.
template <class Shown>
__device__ __forceinline__ uint32_t first_shown(const pt_change_rec* __restrict__ c0, uint32_t n, Shown shown, uint32_t lane) {
    uint32_t k = 0;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t c = base + lane;
        uint4 r = make_uint4(0, 0, 0, 0);
        if (c < n) r = __ldg(reinterpret_cast<const uint4*>(c0 + c));
        const bool first = c < n && r.x == 1u;
        const uint32_t fm = __ballot_sync(0xffffffffu, first);
        if (first) shown(r.y & 0xFFFFu, k + __popc(fm & ((1u << lane) - 1u)));
        k += __popc(fm);
    }
    return k;
}

// A request's clock entries [lo, hi) into clk[actor] (actors < n_actors and distinct: the host checks them).
__device__ __forceinline__ void load_clock(uint32_t* clk, const pt_clock_entry* clock, unsigned long long lo, unsigned long long hi, uint32_t lane) {
    for (unsigned long long e = lo + lane; e < hi; e += 32) {
        const pt_clock_entry q = clock[e];
        clk[q.actor] = q.seq;
    }
}

// getMissingChanges order (reference test/merge.ts:25-38) of a seq-contiguous table c0[0 .. n) whose clock count_clock left in
// cs[actor]: actors in the order the table first shows them, then ascending seq.  have(actor) is the peer's clock entry for the
// table's actor rank.  An actor's first change is its seq 1, so one pass in table order gives every actor the slot of its first
// missing change (a warp scan over the trip's seq-1 lanes, overwriting cs), and change k = (actor, seq) with seq > have goes to
// slot cs[actor] + seq - have - 1: queued(k, its record, slot).  Returns the queue length.  Warp-collective.
template <class Have, class Queued>
__device__ __forceinline__ uint32_t missing_queue(const pt_change_rec* __restrict__ c0, uint32_t n, uint32_t* cs, Have have_of, Queued queued, uint32_t lane) {
    uint32_t nq = 0;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t k = base + lane;
        const bool valid = k < n;
        uint4 r = make_uint4(0, 0, 0, 0);
        if (valid) r = __ldg(reinterpret_cast<const uint4*>(c0 + k));
        const uint32_t actor = r.y & 0xFFFFu, have = valid ? have_of(actor) : 0u;
        const bool first = valid && r.x == 1u;
        uint32_t tot;
        const uint32_t ex = warp_excl_scan(first && cs[actor] > have ? cs[actor] - have : 0u, lane, tot);
        __syncwarp();
        if (first) cs[actor] = nq + ex;
        __syncwarp();
        nq += tot;
        if (valid && r.x > have) queued(k, r, cs[actor] + r.x - have - 1u);
    }
    return nq;
}

}  // namespace ptct
