// change_kernel.cuh — the device half of pt_batch_change (include/peritext_b200.h): Micromerge.change's list ops
// (reference src/micromerge.ts:308-441, changeMark src/peritext.ts:458-501) resolved against the merged documents.
//
// change_resolve_kernel: one warp per log with InputOperations (grid-stride over the work list).  The warp copies the log's
// element sequence (the merge's PT_FLAG_EMIT_SEQUENCE words: bits29:0 insert record, bit30 after slot defined, bit31 deleted)
// into its scratch slot and replays the InputOperations in order on that copy, so each one sees the earlier ones applied:
//   * the k-th visible element: 128 words per trip (four coalesced 32-word loads in flight), ballot / popcount per load;
//   * lookAfterTombstones: the run of tombstones after it, 32 words per trip, the last one with bit 30;
//   * an insert of n values: one splice, the tail of the sequence moves n words right (backwards, 128 words per trip), and
//     the n new words name the records the change appends (old n_insdel + the ins/del records generated before);
//   * a delete sets bit 31, a non-inclusive end sets bit 30 of its element.
// A new element's opId exceeds every opId of the log (first_ctr > max_ctr), so it lands right after its reference element,
// where applyListInsert (src/micromerge.ts:630-635) puts it.  An element's opId is read from its insert record: the
// resident one, or the delta record this warp wrote earlier.  The records are written into the delta as they are generated
// (the host laid the delta out for every log succeeding); a log that fails keeps its partial records, and the host gives it
// zero new records.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace ptc {

// Per-log outcome codes beyond pt_change_status's: the host refuses the call when any log reports one of them.
constexpr uint32_t kRefuseMergeStatus = 0x100u;   // the log's merge status is not PT_LOG_OK
constexpr uint32_t kRefuseElements = 0x101u;      // n_elems + the change's insert values >= 2^22
constexpr uint32_t kNotFound = 0xFFFFFFFFu;
constexpr uint32_t kWordDeleted = 0x80000000u, kWordAfter = 0x40000000u, kWordRecord = 0x3FFFFFFFu;

struct ChangeParams {
    const uint32_t* work; uint32_t n_work;          // logs with InputOperations
    const pt_log_desc* desc;                         // resident batch
    const pt_insdel_rec* insdel;
    const pt_log_result* results;
    const uint64_t* seq_off; const uint32_t* seq;    // the last merge's element sequences
    const uint32_t* actor;                           // [n_logs]
    const unsigned long long* input_off;             // [n_logs + 1]
    const pt_input_op* ops;
    const uint32_t* tokens;
    const pt_log_desc* delta;                        // [n_logs] where each log's generated records go
    const uint32_t* new_elems;                       // [n_logs] the insert values of each log's change
    const unsigned long long* scratch_off;           // [n_logs] word offset of the log's slot (16-byte aligned)
    uint32_t* scratch;
    pt_insdel_rec* out_insdel; pt_mark_rec* out_marks;
    pt_change_status* status;                        // [n_logs]
};

// Position of the k-th visible word of s[0, len), or kNotFound.
__device__ __forceinline__ uint32_t kth_visible(const uint32_t* s, uint32_t len, uint32_t k, uint32_t lane) {
    uint32_t seen = 0;
    for (uint32_t b = 0; b < len; b += 128) {
        uint32_t e[4];
#pragma unroll
        for (int j = 0; j < 4; j++) e[j] = b + 32 * j + lane < len ? s[b + 32 * j + lane] : kWordDeleted;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t vis = __ballot_sync(0xffffffffu, !(e[j] >> 31));
            const uint32_t c = __popc(vis);
            if (seen + c > k) {
                uint32_t m = vis;                                          // the (k - seen)-th set bit
                for (uint32_t r = k - seen; r; r--) m &= m - 1;
                return b + 32 * j + (__ffs(m) - 1);
            }
            seen += c;
        }
    }
    return kNotFound;
}

// First visible position >= from, or kNotFound.
__device__ __forceinline__ uint32_t next_visible(const uint32_t* s, uint32_t len, uint32_t from, uint32_t lane) {
    for (uint32_t b = from; b < len; b += 32) {
        const uint32_t e = b + lane < len ? s[b + lane] : kWordDeleted;
        const uint32_t vis = __ballot_sync(0xffffffffu, !(e >> 31));
        if (vis) return b + (__ffs(vis) - 1);
    }
    return kNotFound;
}

// getListElementId's lookAfterTombstones step (src/micromerge.ts:775-797): the last tombstone with a defined after slot in the
// run of tombstones that follows pos, else pos.
__device__ __forceinline__ uint32_t look_after(const uint32_t* s, uint32_t len, uint32_t pos, uint32_t lane) {
    uint32_t best = pos;
    for (uint32_t b = pos + 1; b < len; b += 32) {
        const uint32_t e = b + lane < len ? s[b + lane] : 0u;               // past the end counts as "not a tombstone"
        const uint32_t live = __ballot_sync(0xffffffffu, !(e >> 31));
        const uint32_t upto = live ? ((1u << (__ffs(live) - 1)) - 1u) : 0xFFFFFFFFu;
        const uint32_t marked = __ballot_sync(0xffffffffu, (e >> 30) & 1u) & upto;
        if (marked) best = b + (31 - __clz(marked));
        if (live) break;
    }
    return best;
}

__global__ void __launch_bounds__(128) change_resolve_kernel(ChangeParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t w = warp; w < P.n_work; w += nwarps) {
        const uint32_t li = P.work[w];
        const pt_log_desc D = P.desc[li], O = P.delta[li];
        const pt_log_result R = P.results[li];
        const unsigned long long i0 = P.input_off[li], i1 = P.input_off[li + 1];
        const uint32_t A = P.actor[li];
        uint32_t code = PT_CHANGE_OK, fail = 0xFFFFFFFFu;
        if (R.status != PT_LOG_OK) code = kRefuseMergeStatus;
        else if ((unsigned long long)R.n_elems + P.new_elems[li] >= (1ull << 22)) code = kRefuseElements;
        if (code == PT_CHANGE_OK && i1 > i0) {
            uint32_t* s = P.scratch + P.scratch_off[li];
            const uint32_t* src = P.seq + P.seq_off[li];
            uint32_t len = R.n_elems, vis_len = R.n_visible;
            for (uint32_t k = lane; k < len; k += 32) s[k] = src[k];
            __syncwarp();
            const pt_insdel_rec* old = P.insdel + D.insdel_off;
            pt_insdel_rec* gi = P.out_insdel + O.insdel_off;
            pt_mark_rec* gm = P.out_marks + O.mark_off;
            uint32_t n_id = 0, n_mk = 0;                             // ins/del and mark records generated so far
            // the packed opId (ctr, actor) of the element at position p of the scratch sequence
            auto elem_id = [&](uint32_t p, uint32_t& ctr, uint32_t& act) {
                const uint32_t r = s[p] & kWordRecord;
                const pt_insdel_rec& x = r < D.n_insdel ? old[r] : gi[r - D.n_insdel];
                ctr = x.ctr; act = x.actor;
            };
            for (unsigned long long k = i0; k < i1 && code == PT_CHANGE_OK; k++) {
                const pt_input_op op = P.ops[k];
                if (op.action == PT_INPUT_INSERT) {
                    uint32_t ref_ctr = 0, ref_actor = 0, pos = 0;
                    if (op.index != 0) {
                        const uint32_t p = op.index > 0 ? kth_visible(s, len, (uint32_t)op.index - 1u, lane) : kNotFound;
                        if (p == kNotFound) { code = PT_CHANGE_OUT_OF_BOUNDS; fail = (uint32_t)(k - i0); break; }
                        const uint32_t q = look_after(s, len, p, lane);
                        elem_id(q, ref_ctr, ref_actor);
                        pos = q + 1;
                    }
                    const uint32_t n = (uint32_t)op.arg;
                    if (n == 0) continue;
                    // the splice: s[pos, len) moves n words right, backwards in trips of 128 words (all loads before all stores)
                    for (uint32_t hi = len; hi > pos;) {
                        const uint32_t lo = hi - pos > 128 ? hi - 128 : pos;
                        uint32_t e[4];
#pragma unroll
                        for (int j = 0; j < 4; j++) { const uint32_t x = lo + 32 * j + lane; e[j] = x < hi ? s[x] : 0u; }
                        __syncwarp();
#pragma unroll
                        for (int j = 0; j < 4; j++) { const uint32_t x = lo + 32 * j + lane; if (x < hi) s[x + n] = e[j]; }
                        __syncwarp();
                        hi = lo;
                    }
                    for (uint32_t j = lane; j < n; j += 32) {
                        s[pos + j] = D.n_insdel + n_id + j;
                        pt_insdel_rec r;
                        r.ctr = op.first_ctr + j; r.actor = (uint16_t)A;
                        r.ref_ctr = j ? op.first_ctr + j - 1 : ref_ctr; r.ref_actor = (uint16_t)(j ? A : ref_actor);
                        r.payload = (PT_KIND_INSERT << 30) | PT_PAYLOAD_TOKEN(P.tokens[op.tok_off + j]);
                        gi[n_id + j] = r;
                    }
                    __syncwarp();
                    n_id += n; len += n; vis_len += n;
                } else if (op.action == PT_INPUT_DELETE) {
                    uint32_t p = kNotFound;
                    for (int32_t c = 0; c < op.arg; c++) {
                        // the index-th visible element; after deleting it, the next one is the first visible element after it
                        p = c == 0 ? (op.index >= 0 ? kth_visible(s, len, (uint32_t)op.index, lane) : kNotFound)
                                   : (p == kNotFound ? kNotFound : next_visible(s, len, p + 1, lane));
                        if (p == kNotFound) { code = PT_CHANGE_OUT_OF_BOUNDS; fail = (uint32_t)(k - i0); break; }
                        uint32_t tc, ta;
                        elem_id(p, tc, ta);
                        if (lane == 0) {
                            s[p] |= kWordDeleted;
                            pt_insdel_rec r;
                            r.ctr = op.first_ctr + (uint32_t)c; r.actor = (uint16_t)A; r.ref_ctr = tc; r.ref_actor = (uint16_t)ta;
                            r.payload = PT_KIND_DELETE << 30;
                            gi[n_id] = r;
                        }
                        __syncwarp();
                        n_id++; vis_len--;
                    }
                } else {                                                 // addMark / removeMark (changeMark, src/peritext.ts:458-501)
                    const uint32_t t = op.mark_type;
                    const bool inclusive = t == PT_MARK_STRONG || t == PT_MARK_EM;
                    const uint32_t ps = op.index >= 0 ? kth_visible(s, len, (uint32_t)op.index, lane) : kNotFound;
                    uint32_t sc = 0, sa = 0, ec = 0, ea = 0, eb = PT_BOUND_END_OF_TEXT, pe = kNotFound;
                    bool ok = ps != kNotFound;
                    if (ok) {
                        elem_id(ps, sc, sa);
                        if (inclusive && (int64_t)op.arg >= (int64_t)vis_len) {
                            eb = PT_BOUND_END_OF_TEXT;
                        } else if (inclusive) {
                            eb = PT_BOUND_BEFORE;
                            pe = op.arg >= 0 ? kth_visible(s, len, (uint32_t)op.arg, lane) : kNotFound;
                            ok = pe != kNotFound;
                        } else {
                            eb = PT_BOUND_AFTER;
                            pe = op.arg >= 1 ? kth_visible(s, len, (uint32_t)op.arg - 1u, lane) : kNotFound;
                            ok = pe != kNotFound;
                        }
                    }
                    if (!ok) { code = PT_CHANGE_OUT_OF_BOUNDS; fail = (uint32_t)(k - i0); break; }
                    if (pe != kNotFound) elem_id(pe, ec, ea);
                    if (lane == 0) {
                        if (eb == PT_BOUND_AFTER) s[pe] |= kWordAfter;
                        pt_mark_rec m;
                        m.ctr = op.first_ctr; m.actor = (uint16_t)A;
                        m.kind = (uint8_t)((op.action == PT_INPUT_REMOVE_MARK ? 1u : 0u) | (t << 1));
                        m.bounds = (uint8_t)(PT_BOUND_BEFORE | (eb << 2));
                        m.start_ctr = sc; m.start_actor = (uint16_t)sa; m.end_ctr = ec; m.end_actor = (uint16_t)ea;
                        m.attr = op.attr; m.arrival = D.n_insdel + n_id; m.reserved = 0;
                        gm[n_mk] = m;
                    }
                    __syncwarp();
                    n_mk++;
                }
            }
        }
        if (lane == 0) P.status[li] = pt_change_status{code, fail};
    }
}

}  // namespace ptc
