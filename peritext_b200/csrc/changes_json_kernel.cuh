// changes_json_kernel.cuh — pt_batch_render_changes_json: the reference's Change objects (src/micromerge.ts:60-71) of resident
// logs as UTF-8 JSON text, written on the device from the change table, the op records and the caller's string pools
// (include/peritext_b200.h has the contract, DESIGN.md §4.8d the design).
//
// changes_select_kernel: one warp per request.  Every request first takes the list-op position of each change of its log's table
// (ptct::count_clock without a clock: the positions and the dep-range check) and checks that they sum to the log's records.
// RANGE selects a clipped range of the table.  MISSING counts the log's clock with ptct::count_clock (seq-contiguous per actor,
// else PT_CHANGES_BAD_TABLE), loads the peer's clock into shared memory by rank and builds the queue in getMissingChanges order
// with ptct::missing_queue (DESIGN.md §4.3's change-table rules).  The selected changes are cut into WORK ITEMS of at most kSlice list
// ops each, so one c5-sized change is not left to a single warp; an OK request without changes gets one item, which writes "[]".
//
// changes_json_size_kernel / changes_json_write_kernel: one warp per item, both through render_item<W>.  Slice 0 of a change
// writes its header and deps (lane 0), the last slice the rest of the ops array and the trailer; the request's brackets and the
// commas between changes go to its first, last and slice-0 items.  The list ops of a slice go 32 per trip, one per lane, in
// arrival order (the patch render's OR-reduced mark-slot mask says which positions are mark records); the extras anchored before
// a list op are written by that op's lane.  Every byte count comes from the same write-or-count functions as the write, so the
// two passes cannot disagree; make RENDER_CHECK=1 asserts it.
#pragma once
#include <cassert>
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "render_kernel.cuh"
#include "patch_json_kernel.cuh"
#include "change_table.cuh"
#include "patch_window.cuh"

namespace ptcj {

using ptr::kFull;
using ptr::kNoUnit;
using ptr::lane_lit;     // PTJ_LIT and PTR_LIT name them unqualified
using ptr::emit_lit;

constexpr uint32_t kSlice = 1024;   // list ops per work item

struct Sel { uint32_t change, pos, item0, reserved; };   // a selected change: table index, first list-op position, first item

struct ChangesParams {
    const pt_changes_request* req; uint32_t n_req; uint32_t maxR;
    const pt_clock_entry* clock;
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_insdel_rec* insdel; const pt_mark_rec* marks;
    const unsigned long long* slot_off;   // [n_req + 1] a request's scratch slot: its log's n_changes entries of pos and sel
    uint32_t* pos; Sel* sel;
    uint32_t* n_sel; uint32_t* status; unsigned long long* items;   // per request
    const pt_change_extra* extras; unsigned long long n_extras;
    unsigned long long* bad;              // [2] (log << 32 | change): [0] a change with no op, [1] extras past their change's ops
    // the item passes
    const unsigned long long* item_off;   // [n_req + 1]
    unsigned long long n_items;
    const uint8_t* actors; const unsigned long long* actors_off; const unsigned long long* actors_first;
    const unsigned long long* counters; const unsigned long long* counters_first;
    const uint8_t* list_ids; const unsigned long long* list_ids_off;
    const uint8_t* xops; const unsigned long long* xops_off;
};

// Missing actor / counter pool entries: (log << 34 | kind << 32 | index), kind 0 actor, 1 counter; the lowest key wins.
__device__ __forceinline__ void note_pool(unsigned long long* miss, uint32_t log, uint32_t kind, uint32_t idx) {
    if (miss) atomicMin(miss, ((unsigned long long)log << 34) | ((unsigned long long)kind << 32) | idx);
}

template <bool W> __device__ __forceinline__ uint32_t put_dec64(uint8_t* d, unsigned long long v) {
    uint32_t len = 1;
    for (unsigned long long t = v; t >= 10ull; t /= 10ull) len++;
    if (W) for (uint32_t k = len; k-- > 0; v /= 10ull) d[k] = (uint8_t)('0' + v % 10ull);
    return len;
}

// UTF-16LE units p[0 .. n) as a JSON string (quotes included), JSON.stringify's rules (render_kernel.cuh's unit_out).
template <bool W> __device__ __forceinline__ uint32_t str_out(const uint8_t* p, uint64_t n, uint8_t* d) {
    auto unit = [&](uint64_t j) { return (uint32_t)p[2 * j] | ((uint32_t)p[2 * j + 1] << 8); };
    uint32_t b = PTJ_LIT(W, d, "\"");
    uint32_t prev = kNoUnit;
    for (uint64_t j = 0; j < n; j++) {
        const uint32_t u = unit(j), nx = j + 1 < n ? unit(j + 1) : kNoUnit;
        b += ptr::unit_out<W>(u, prev, nx, d + b);
        prev = u;
    }
    return b + PTJ_LIT(W, d + b, "\"");
}

// Actor rank a of log `log` as a quoted JSON string; an actor the pool does not hold is noted and writes "".
template <bool W> __device__ __forceinline__ uint32_t actor_out(const ChangesParams& C, uint32_t log, uint32_t a, uint8_t* d, unsigned long long* miss2) {
    const unsigned long long f = C.actors_first[log];
    if (a >= C.actors_first[log + 1] - f) { if (!W) note_pool(miss2, log, 0, a); return str_out<W>(nullptr, 0, d); }
    const unsigned long long o = C.actors_off[f + a];
    return str_out<W>(C.actors + o, (C.actors_off[f + a + 1] - o) >> 1, d);
}

// The original counter of packed counter c (the counter pool's entry for a re-ranked log, else c itself).
template <bool W> __device__ __forceinline__ unsigned long long orig_ctr(const ChangesParams& C, uint32_t log, uint32_t c, unsigned long long* miss2) {
    const unsigned long long f = C.counters_first[log], n = C.counters_first[log + 1] - f;
    if (!n) return c;
    if (c >= n) { if (!W) note_pool(miss2, log, 1, c); return c; }
    return C.counters[f + c];
}

// "ctr@actor" with the original counter; counter 0 (HEAD) is "_head".
template <bool W> __device__ __forceinline__ uint32_t id_out(const ChangesParams& C, uint32_t log, uint32_t ctr, uint32_t a, uint8_t* d, unsigned long long* miss2) {
    if (!ctr) return PTJ_LIT(W, d, "\"_head\"");
    const unsigned long long f = C.actors_first[log];
    uint32_t b = PTJ_LIT(W, d, "\"");
    b += put_dec64<W>(d + b, orig_ctr<W>(C, log, ctr, miss2));
    b += PTJ_LIT(W, d + b, "@");
    if (a >= C.actors_first[log + 1] - f) { if (!W) note_pool(miss2, log, 0, a); return b + PTJ_LIT(W, d + b, "\""); }
    const unsigned long long o = C.actors_off[f + a];
    const uint8_t* p = C.actors + o;
    const uint64_t n = (C.actors_off[f + a + 1] - o) >> 1;
    uint32_t prev = '@';
    for (uint64_t j = 0; j < n; j++) {
        const uint32_t u = (uint32_t)p[2 * j] | ((uint32_t)p[2 * j + 1] << 8);
        const uint32_t nx = j + 1 < n ? (uint32_t)p[2 * j + 2] | ((uint32_t)p[2 * j + 3] << 8) : (uint32_t)'"';
        b += ptr::unit_out<W>(u, prev, nx, d + b);
        prev = u;
    }
    return b + PTJ_LIT(W, d + b, "\"");
}

template <bool W> __device__ __forceinline__ uint32_t list_id_out(const ChangesParams& C, uint32_t log, uint8_t* d) {
    const unsigned long long o = C.list_ids_off[log];
    return str_out<W>(C.list_ids + o, (C.list_ids_off[log + 1] - o) >> 1, d);
}

template <bool W> __device__ __forceinline__ uint32_t bound_out(const ChangesParams& C, uint32_t log, uint32_t t, uint32_t ctr, uint32_t a, uint8_t* d,
                                                                unsigned long long* miss2) {
    if (t >= PT_BOUND_START_OF_TEXT) return t == PT_BOUND_START_OF_TEXT ? PTJ_LIT(W, d, "{\"type\":\"startOfText\"}") : PTJ_LIT(W, d, "{\"type\":\"endOfText\"}");
    uint32_t b = PTJ_LIT(W, d, "{\"elemId\":");
    b += id_out<W>(C, log, ctr, a, d + b, miss2);
    return b + (t == PT_BOUND_BEFORE ? PTJ_LIT(W, d + b, ",\"type\":\"before\"}") : PTJ_LIT(W, d + b, ",\"type\":\"after\"}"));
}

// List op `j` of its kind (ins/del record j or mark record j of the log) as one op object.  One lane.
template <bool W>
__device__ uint32_t list_op_out(const ChangesParams& C, const ptr::JsonPools& P, const pt_log_desc& L, uint32_t log, bool is_mark, uint32_t j, uint8_t* d,
                                unsigned long long* miss, unsigned long long* miss2) {
    uint32_t n = 0;
    if (!is_mark) {
        const pt_insdel_rec r = C.insdel[L.insdel_off + j];
        const bool ins = PT_PAYLOAD_KIND(r.payload) == PT_KIND_INSERT;
        n += ins ? PTJ_LIT(W, d, "{\"action\":\"set\",\"elemId\":") : PTJ_LIT(W, d, "{\"action\":\"del\",\"elemId\":");
        n += id_out<W>(C, log, r.ref_ctr, r.ref_actor, d + n, miss2);
        n += ins ? PTJ_LIT(W, d + n, ",\"insert\":true,\"obj\":") : PTJ_LIT(W, d + n, ",\"obj\":");
        n += list_id_out<W>(C, log, d + n);
        n += PTJ_LIT(W, d + n, ",\"opId\":");
        n += id_out<W>(C, log, r.ctr, r.actor, d + n, miss2);
        if (ins) {
            n += PTJ_LIT(W, d + n, ",\"value\":\"");
            // every value is a string of its own: surrogate halves pair only inside it
            n += ptr::elem_out<W>(ptr::make_elem<W>(PT_PAYLOAD_TOKEN(r.payload), P, miss, log), kNoUnit, kNoUnit, d + n);
            n += PTJ_LIT(W, d + n, "\"");
        }
        return n + PTJ_LIT(W, d + n, "}");
    }
    const pt_mark_rec m = C.marks[L.mark_off + j];
    const uint32_t type = (m.kind >> 1) & 3u;
    n += (m.kind & 1u) ? PTJ_LIT(W, d, "{\"action\":\"removeMark\",") : PTJ_LIT(W, d, "{\"action\":\"addMark\",");
    if (m.attr != PT_ATTR_NONE) {
        n += PTJ_LIT(W, d + n, "\"attrs\":");
        n += type == PT_MARK_LINK ? ptr::pool_frag<W>(P.link, P.loff, P.nlink, m.attr, 1, d + n, miss, log)
                                  : ptr::pool_frag<W>(P.com, P.coff, P.ncom, m.attr, 2, d + n, miss, log);
        n += PTJ_LIT(W, d + n, ",");
    }
    n += PTJ_LIT(W, d + n, "\"end\":");
    n += bound_out<W>(C, log, (m.bounds >> 2) & 3u, m.end_ctr, m.end_actor, d + n, miss2);
    n += PTJ_LIT(W, d + n, ",\"markType\":\"");
    switch (type) {
        case PT_MARK_STRONG: n += PTJ_LIT(W, d + n, "strong"); break;
        case PT_MARK_EM: n += PTJ_LIT(W, d + n, "em"); break;
        case PT_MARK_COMMENT: n += PTJ_LIT(W, d + n, "comment"); break;
        default: n += PTJ_LIT(W, d + n, "link"); break;
    }
    n += PTJ_LIT(W, d + n, "\",\"obj\":");
    n += list_id_out<W>(C, log, d + n);
    n += PTJ_LIT(W, d + n, ",\"opId\":");
    n += id_out<W>(C, log, m.ctr, m.actor, d + n, miss2);
    n += PTJ_LIT(W, d + n, ",\"start\":");
    n += bound_out<W>(C, log, m.bounds & 3u, m.start_ctr, m.start_actor, d + n, miss2);
    return n + PTJ_LIT(W, d + n, "}");
}

// Extras e of x[0 .. n) as ops, each after a comma unless it is op 0.  One lane.
template <bool W> __device__ __forceinline__ uint32_t extras_out(const ChangesParams& C, const pt_change_extra* x, uint64_t n, uint8_t* d) {
    uint32_t b = 0;
    for (uint64_t e = 0; e < n; e++) {
        if (x[e].pos) b += PTJ_LIT(W, d + b, ",");
        const unsigned long long o = C.xops_off[x[e].op];
        b += ptr::frag_copy<W>(C.xops + o, C.xops_off[x[e].op + 1] - o, d + b);
    }
    return b;
}

// The first entry of the sorted extras whose (log, change) is >= key.
__device__ __forceinline__ unsigned long long extras_lower(const ChangesParams& C, unsigned long long key) {
    unsigned long long lo = 0, hi = C.n_extras;
    while (lo < hi) {
        const unsigned long long mid = lo + ((hi - lo) >> 1);
        if ((((unsigned long long)C.extras[mid].log << 32) | C.extras[mid].change) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// How many of the change's op-carrying extras x[0 .. n) sit before list op j + 1, i.e. have pos - (their rank) <= j.
__device__ __forceinline__ uint32_t extras_upto(const pt_change_extra* x, uint32_t n, long long j) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if ((long long)x[mid].pos - (long long)mid <= j) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void changes_select_kernel(ChangesParams C) {
    extern __shared__ uint32_t cj_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* clk = cj_smem + (size_t)wib * 2 * C.maxR;     // the peer's clock, by actor rank
    uint32_t* cs = clk + C.maxR;                            // by actor rank: change count, then first queue slot
    for (uint32_t r = blockIdx.x * wpb + wib; r < C.n_req; r += gridDim.x * wpb) {
        const pt_changes_request q = C.req[r];
        const pt_log_desc L = C.desc[q.log];
        const pt_change_desc CD = C.cdesc[q.log];
        const pt_change_rec* c0 = C.changes + CD.change_off;
        uint32_t* pos = C.pos + C.slot_off[r];
        Sel* sel = C.sel + C.slot_off[r];
        unsigned long long ops = 0;   // the header reads a change's deps in every mode
        const bool deps_ok = ptct::count_clock(c0, CD.n_changes, CD.n_deps, 0u, nullptr, pos, &ops, lane);
        uint32_t status = deps_ok && ops == (unsigned long long)L.n_insdel + L.n_mark ? PT_CHANGES_OK : PT_CHANGES_BAD_TABLE;
        uint32_t ns = 0;
        if (status == PT_CHANGES_OK && q.mode == PT_CHANGES_RANGE) {
            const uint32_t a = min(q.first, CD.n_changes), e = (uint32_t)min((unsigned long long)q.first + q.count, (unsigned long long)CD.n_changes);
            ns = e > a ? e - a : 0u;
            for (uint32_t k = lane; k < ns; k += 32) sel[k].change = a + k;
        } else if (status == PT_CHANGES_OK) {
            const uint32_t R = L.n_actors;
            for (uint32_t a = lane; a < R; a += 32) { clk[a] = 0; cs[a] = 0; }
            __syncwarp();
            for (uint32_t k = lane; k < q.n_clock; k += 32) { const pt_clock_entry e = C.clock[q.clock_off + k]; atomicMax(&clk[e.actor], e.seq); }
            __syncwarp();
            if (!ptct::count_clock(c0, CD.n_changes, CD.n_deps, R, cs, nullptr, nullptr, lane)) {
                status = PT_CHANGES_BAD_TABLE;
            } else {
                ns = ptct::missing_queue(c0, CD.n_changes, cs, [&](uint32_t actor) { return clk[actor]; },
                                         [&](uint32_t k, uint4, uint32_t slot) { sel[slot].change = k; }, lane);
            }
        }
        if (status != PT_CHANGES_OK) ns = 0;
        __syncwarp();
        // the selected changes' work items, and the checks that need the change's extras
        unsigned long long nitems = 0;
        for (uint32_t base = 0; base < ns; base += 32) {
            const uint32_t k = base + lane;
            const bool valid = k < ns;
            uint32_t it = 0, c = 0;
            if (valid) {
                c = sel[k].change;
                const uint32_t n_ops = c0[c].n_ops;
                it = max(1u, (n_ops + kSlice - 1u) / kSlice);
                const unsigned long long key = ((unsigned long long)q.log << 32) | c, x0 = extras_lower(C, key), x1 = extras_lower(C, key + 1);
                if (n_ops == 0 && x0 == x1) atomicMin(&C.bad[0], key);
                else if (x1 > x0 && C.extras[x0].op != PT_EXTRA_NONE && C.extras[x1 - 1].pos >= (unsigned long long)n_ops + (x1 - x0)) atomicMin(&C.bad[1], key);
            }
            uint32_t tot;
            const uint32_t ex = ptct::warp_excl_scan(it, lane, tot);
            if (valid) sel[k] = Sel{c, pos[c], (uint32_t)nitems + ex, 0u};
            nitems += tot;
        }
        if (status == PT_CHANGES_OK && ns == 0) nitems = 1;     // "[]"
        if (lane == 0) { C.n_sel[r] = ns; C.status[r] = status; C.items[r] = status == PT_CHANGES_OK ? nitems : 0ull; }
        __syncwarp();
    }
}

// Item j's bytes at d (W) or its byte count (!W).  Warp-collective; every lane returns the same count.
template <bool W>
__device__ uint64_t render_item(const ChangesParams& C, const ptr::JsonPools& P, unsigned long long j, uint8_t* d, unsigned long long* miss,
                                unsigned long long* miss2, uint32_t lane) {
    uint32_t lo = 0, hi = C.n_req;                             // the request: the last r with item_off[r] <= j
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (C.item_off[mid] <= j) lo = mid; else hi = mid; }
    const uint32_t r = lo, t = (uint32_t)(j - C.item_off[r]), ns = C.n_sel[r];
    const bool last_item = j + 1 == C.item_off[r + 1];
    uint64_t pos = 0;
    if (!ns) { PTR_LIT(W, d, pos, "[]", lane); return pos; }
    const uint32_t log = C.req[r].log;
    const Sel* sel = C.sel + C.slot_off[r];
    uint32_t a = 0, b = ns;                                    // the change: the last k with item0 <= t
    while (b - a > 1) { const uint32_t mid = (a + b) >> 1; if (sel[mid].item0 <= t) a = mid; else b = mid; }
    const uint32_t k = a, s = t - sel[k].item0;
    const Sel S = sel[k];
    const pt_log_desc L = C.desc[log];
    const pt_change_desc CD = C.cdesc[log];
    const pt_change_rec ch = C.changes[CD.change_off + S.change];
    const uint32_t n_ops = ch.n_ops, n_slices = max(1u, (n_ops + kSlice - 1u) / kSlice);
    const uint32_t j0 = s * kSlice, j1 = min(n_ops, j0 + kSlice);
    const unsigned long long key = ((unsigned long long)log << 32) | S.change, x0 = extras_lower(C, key), x1 = extras_lower(C, key + 1);
    const pt_change_extra* xs = C.extras + x0;
    const bool none = x1 > x0 && xs[0].op == PT_EXTRA_NONE;
    const uint32_t nx = none ? 0u : (uint32_t)(x1 - x0);      // the op-carrying extras
    const pt_mark_rec* mk = C.marks + L.mark_off;
    if (t == 0) PTR_LIT(W, d, pos, "[", lane);
    if (s == 0) {                                              // header and deps
        uint32_t h = 0;
        if (lane == 0) {
            uint8_t* o = W ? d + pos : nullptr;
            if (k) h += PTJ_LIT(W, o, ",");
            h += PTJ_LIT(W, o + h, "{\"actor\":");
            h += actor_out<W>(C, log, ch.actor, o + h, miss2);
            h += PTJ_LIT(W, o + h, ",\"deps\":{");
            const pt_dep_rec* dp = C.deps + CD.dep_off + ch.dep_off;
            for (uint32_t q = 0; q < ch.n_deps; q++) {
                if (q) h += PTJ_LIT(W, o + h, ",");
                h += actor_out<W>(C, log, dp[q].actor, o + h, miss2);
                h += PTJ_LIT(W, o + h, ":");
                h += put_dec64<W>(o + h, dp[q].seq);
            }
            h += PTJ_LIT(W, o + h, "},\"ops\":[");
        }
        pos += __shfl_sync(kFull, h, 0);
    }
    // the slice's list ops, at list-op positions [S.pos + j0, S.pos + j1), 32 per trip in arrival order
    const uint32_t n = L.n_insdel, m = L.n_mark, w0 = S.pos + j0, w1 = S.pos + j1;
    uint32_t mi = ptw::marks_before_lane(mk, n, m, w0), ri = w0 - mi;      // bisection: a late slice of a long change
    for (uint32_t base = w0; base < w1; base += 32) {
        uint32_t bit = 0;
        if (mi + lane < m) {
            const uint32_t p = min(mk[mi + lane].arrival, n) + mi + lane;
            if (p >= base && p < base + 32) bit = 1u << (p - base);
        }
        const uint32_t mm = __reduce_or_sync(kFull, bit), below = __popc(mm & ((1u << lane) - 1u));
        const bool is_mark = (mm >> lane) & 1u;
        const uint32_t jj = is_mark ? mi + below : ri + lane - below, p = base + lane, jl = p - S.pos;
        const bool live = p < w1 && jj < (is_mark ? m : n);
        uint32_t c = 0, e_lo = 0, e_hi = 0;
        if (live) {
            e_lo = jl ? extras_upto(xs, nx, (long long)jl - 1) : 0u;
            e_hi = extras_upto(xs, nx, jl);
            c = extras_out<false>(C, xs + e_lo, e_hi - e_lo, nullptr) + (jl + e_hi ? 1u : 0u) +
                list_op_out<false>(C, P, L, log, is_mark, jj, nullptr, miss, miss2);
        }
        const uint32_t incl = ptr::warp_incl_scan(c, lane);
        if (W && live) {
            uint8_t* o = d + pos + incl - c;
            o += extras_out<true>(C, xs + e_lo, e_hi - e_lo, o);
            if (jl + e_hi) *o++ = ',';
            list_op_out<true>(C, P, L, log, is_mark, jj, o, nullptr, nullptr);
        }
        pos += __shfl_sync(kFull, incl, 31);
        mi += __popc(mm); ri += 32u - __popc(mm);
    }
    if (s + 1 == n_slices) {                                   // the extras after the last list op, and the trailer
        uint32_t h = 0;
        if (lane == 0) {
            uint8_t* o = W ? d + pos : nullptr;
            const uint32_t e0 = n_ops ? extras_upto(xs, nx, (long long)n_ops - 1) : 0u;
            h += extras_out<W>(C, xs + e0, nx - e0, o);
            h += PTJ_LIT(W, o + h, "],\"seq\":");
            h += put_dec64<W>(o + h, ch.seq);
            h += PTJ_LIT(W, o + h, ",\"startOp\":");
            unsigned long long start = 0;
            if (x1 > x0) {
                start = xs[0].start_op;
            } else {                                           // the original counter of the change's first list op
                const uint32_t k0 = ptw::marks_before_lane(mk, n, m, S.pos);
                const bool first_mark = k0 < m && min(mk[k0].arrival, n) + k0 == S.pos;
                start = orig_ctr<W>(C, log, first_mark ? mk[k0].ctr : C.insdel[L.insdel_off + S.pos - k0].ctr, miss2);
            }
            h += put_dec64<W>(o + h, start);
            h += PTJ_LIT(W, o + h, "}");
            if (last_item) h += PTJ_LIT(W, o + h, "]");
        }
        pos += __shfl_sync(kFull, h, 0);
    }
    return pos;
}

// One warp per item, grid-stride.
__global__ void changes_json_size_kernel(const ChangesParams C, ptr::JsonPools P, unsigned long long* __restrict__ sizes, unsigned long long* __restrict__ miss,
                                         unsigned long long* __restrict__ miss2) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned long long j = warp; j < C.n_items; j += nwarps) {
        const uint64_t s = render_item<false>(C, P, j, nullptr, miss, miss2, lane);
        if (lane == 0) sizes[j] = s;
    }
}

__global__ void changes_json_write_kernel(const ChangesParams C, ptr::JsonPools P, const unsigned long long* __restrict__ off, uint8_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned long long j = warp; j < C.n_items; j += nwarps) {
        const uint64_t end = render_item<true>(C, P, j, out + off[j], nullptr, nullptr, lane);
#ifdef PT_RENDER_CHECK
        assert(end == off[j + 1] - off[j]);      // the write pass ends exactly where the size pass said
#else
        (void)end;
#endif
    }
}

// Request r's text starts where its first item does: off[r] = item byte offset of item_off[r], for r in [0, n_req].
__global__ void changes_offsets_kernel(const unsigned long long* __restrict__ item_off, const unsigned long long* __restrict__ boff, uint32_t n_req,
                                       unsigned long long* __restrict__ off) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= n_req; r += gridDim.x * blockDim.x) off[r] = boff[item_off[r]];
}

}  // namespace ptcj
