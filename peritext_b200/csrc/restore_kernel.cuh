// restore_kernel.cuh — the device side of pt_batch_restore (include/peritext_b200.h): the change that makes a log's visible
// text (TEXT) or its formatting (MARKS) equal to an earlier version's, generated straight into the append delta.
//
// restore_kernel<kWrite>: one warp per request, grid-stride; the count pass (kWrite = false) and the write pass run the
// same function, so they cannot disagree.  Per-warp shared memory holds the log's clock (actor_shape's budget).
//   1. the table: ptct::source_clock into the clock, each change's list-op position into the request's scratch slot; a dep
//      actor >= n_actors or record ranges that do not fit (ptct::change_records) is BAD_TABLE (DESIGN.md §4.3's rules for a src).
//   2. TEXT's walk (restore_walk): 32 elements of the log per trip.  Lane l loads element b + l's opId from its insert record and the version's
//      elements [j, j + 32) of its cursor j; a log element matches iff its opId is the version element at j + its rank among
//      the trip's matching lanes (opIds are unique in a merged log, so any other position means the version is no ordered
//      subsequence: FOREIGN), and j advances by the popcount.  Each element gets its class (keep / delete / restore /
//      nothing) and, by a ballot scan, its record index; delete and restore elements write their record at once.
//   3. TEXT's run state, warp-uniform: the last visible-at-that-moment element (anchor), the last tombstone with bit 30 since it
//      (cand) and the open restore run.  A restore run closes at the next kept or deleted element (or the end); its first
//      record's reference is then HEAD (nothing visible before it), cand, or the anchor, and lane 0 patches it in.  A trip
//      without restore elements and no open run updates the state from ballots; other trips step through their event lanes.
//   2'. MARKS' walk (restore_marks_walk): the token comparison and the visible -> record table, then one lane merging the two
//      span lists (see there).
//   4. the change record and its deps: ptct::first_shown's actors with their counts.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace ptrs {

constexpr uint32_t kKeep = 0, kDel = 1, kRes = 2, kNothing = 3;

struct RestoreParams {
    const pt_restore_request* req; uint32_t n; uint32_t maxR;
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_insdel_rec* insdel; const pt_mark_rec* marks;
    const pt_log_result* res; const uint64_t* seq_off; const uint32_t* seq;
    uint32_t mode;                        // PT_RESTORE_TEXT or PT_RESTORE_MARKS
    const uint64_t* text_off; const uint32_t* text; const uint64_t* span_off; const pt_span* spans; const uint32_t* cpool;
    const unsigned long long* slot_off;   // [n + 1] a request's scratch slot: its log's n_changes list-op positions
    uint32_t* pos;
    const unsigned long long* vis_off;    // [n + 1] MARKS: a request's visible -> record table (its log's n_insdel words)
    uint32_t* vis;
    const unsigned long long* open_off;   // [n + 1] MARKS: its open comment ranges, two lists of n_mark(log) + n_mark(version)
    uint4* open;
    uint32_t* status; uint32_t* n_ops; uint32_t* n_deps; uint32_t* seq_out;   // [n] count pass
    uint32_t* elems;                      // [n] count pass: the log's n_elems after the change
    const pt_log_desc* delta;             // [n_logs] write pass: where each log's records go (insdel_off)
    const pt_change_desc* delta_cdesc;    // [n_logs] and its change record and deps (change_off, dep_off)
    pt_insdel_rec* out_insdel; pt_mark_rec* out_marks; pt_change_rec* out_changes; pt_dep_rec* out_deps;
};

// Request k's walk over its log: the number of generated records (fresh: of them inserts); foreign when the version is no
// ordered subsequence of the log.  With kWrite the records go to out[0 ..).  Warp-collective.
template <bool kWrite>
__device__ __forceinline__ uint32_t restore_walk(const RestoreParams& P, const pt_restore_request& q, uint32_t lane, pt_insdel_rec* out, bool& foreign,
                                                uint32_t& fresh) {
    const uint32_t N = P.res[q.log].n_elems, NV = P.res[q.version].n_elems;
    const uint32_t* sL = P.seq + P.seq_off[q.log];
    const uint32_t* sV = P.seq + P.seq_off[q.version];
    const uint4* insL = reinterpret_cast<const uint4*>(P.insdel + P.desc[q.log].insdel_off);
    const uint4* insV = reinterpret_cast<const uint4*>(P.insdel + P.desc[q.version].insdel_off);
    const uint32_t lt = (1u << lane) - 1u, A = q.actor, F = q.first_ctr;
    uint32_t j = 0, rec = 0;                                     // version cursor; records generated before the trip
    uint32_t prev = kNothing;                                    // the class of the last element that is not "nothing"
    bool have_anchor = false, have_cand = false, headed = false;
    uint32_t anc_c = 0, anc_a = 0, cand_c = 0, cand_a = 0, run_first = 0;
    // the open restore run ends before record r_end: its first record's reference, then the new anchor is its last value
    auto close = [&](uint32_t r_end) {
        const uint32_t rc = headed ? 0u : have_cand ? cand_c : anc_c, ra = headed ? 0u : have_cand ? cand_a : anc_a;
        if (!headed) have_cand = false;
        if (kWrite && lane == 0) { out[run_first].ref_ctr = rc; out[run_first].ref_actor = (uint16_t)ra; }
        anc_c = F + r_end - 1u; anc_a = A; have_anchor = true;
    };
    foreign = false; fresh = 0;
    for (uint32_t b = 0; b < N; b += 32) {
        const uint32_t e = b + lane;
        const bool valid = e < N;
        const uint32_t w = valid ? __ldg(sL + e) : 0u;
        uint4 x = make_uint4(0, 0, 0, 0);
        if (valid) x = __ldg(insL + (w & 0x3FFFFFFFu));
        const uint32_t ctr = x.x, act = x.z & 0xFFFFu;
        const uint32_t jv = j + lane;
        uint32_t vc = 0, va = 0, vw = 0;                        // ctr 0 matches no element
        if (jv < NV) { vw = __ldg(sV + jv); const uint4 y = __ldg(insV + (vw & 0x3FFFFFFFu)); vc = y.x; va = y.z & 0xFFFFu; }
        const uint32_t vdel = __ballot_sync(0xffffffffu, (vw >> 31) != 0);
        uint32_t r = 32;
        for (uint32_t t = 0; t < 32; t++) {
            const uint32_t c = __shfl_sync(0xffffffffu, vc, t), a = __shfl_sync(0xffffffffu, va, t);
            if (valid && c == ctr && a == act) r = t;
        }
        const uint32_t found = __ballot_sync(0xffffffffu, r < 32);
        if (__any_sync(0xffffffffu, r < 32 && r != (uint32_t)__popc(found & lt))) { foreign = true; return rec; }
        j += __popc(found);
        const bool in_vis = r < 32 && !((vdel >> r) & 1u), now_vis = valid && !(w >> 31);
        const uint32_t cls = !valid ? kNothing : now_vis ? (in_vis ? kKeep : kDel) : (in_vis ? kRes : kNothing);
        const bool b30 = valid && ((w >> 30) & 1u);
        const uint32_t gen = __ballot_sync(0xffffffffu, cls == kDel || cls == kRes);
        const uint32_t my = rec + __popc(gen & lt);
        const uint32_t nn = __ballot_sync(0xffffffffu, cls != kNothing);
        const uint32_t below = nn & lt;
        const uint32_t up = __shfl_sync(0xffffffffu, cls, below ? 31 - __clz(below) : 0);
        const uint32_t before = below ? up : prev;              // the class of the last non-"nothing" element before this one
        if (kWrite && (cls == kDel || cls == kRes)) {
            pt_insdel_rec o;
            o.ctr = F + my; o.actor = (uint16_t)A;
            if (cls == kDel) { o.ref_ctr = ctr; o.ref_actor = (uint16_t)act; o.payload = PT_KIND_DELETE << 30; }
            else {
                const bool cont = before == kRes;               // a further value of the run references the one before
                o.ref_ctr = cont ? F + my - 1u : 0u; o.ref_actor = (uint16_t)(cont ? A : 0u);
                o.payload = (PT_KIND_INSERT << 30) | PT_PAYLOAD_TOKEN(x.w);
            }
            out[my] = o;
        }
        __syncwarp();
        const uint32_t resm = __ballot_sync(0xffffffffu, cls == kRes);
        fresh += __popc(resm);
        if (!resm && prev != kRes) {                            // no run opens or closes: the state from ballots
            const uint32_t kp = __ballot_sync(0xffffffffu, cls == kKeep);
            uint32_t tail = 0xFFFFFFFFu;
            if (kp) {
                const uint32_t hk = 31 - __clz(kp);
                anc_c = __shfl_sync(0xffffffffu, ctr, hk); anc_a = __shfl_sync(0xffffffffu, act, hk);
                have_anchor = true; have_cand = false;
                tail = hk == 31 ? 0u : ~((2u << hk) - 1u);
            }
            const uint32_t cm = __ballot_sync(0xffffffffu, b30 && cls != kKeep) & tail;
            if (cm) {
                const uint32_t hc = 31 - __clz(cm);
                cand_c = __shfl_sync(0xffffffffu, ctr, hc); cand_a = __shfl_sync(0xffffffffu, act, hc); have_cand = true;
            }
        } else {                                                // step through the trip's event lanes in order
            for (uint32_t ev = __ballot_sync(0xffffffffu, cls != kNothing || b30); ev; ev &= ev - 1) {
                const uint32_t l = __ffs(ev) - 1;
                const uint32_t c_l = __shfl_sync(0xffffffffu, cls, l), b_l = __shfl_sync(0xffffffffu, (uint32_t)b30, l);
                const uint32_t k_l = __shfl_sync(0xffffffffu, ctr, l), a_l = __shfl_sync(0xffffffffu, act, l), r_l = __shfl_sync(0xffffffffu, my, l);
                if ((c_l == kKeep || c_l == kDel) && prev == kRes) close(r_l);
                if (c_l == kKeep) { anc_c = k_l; anc_a = a_l; have_anchor = true; have_cand = false; }
                else if (b_l) { cand_c = k_l; cand_a = a_l; have_cand = true; }
                if (c_l == kRes && prev != kRes) { run_first = r_l; headed = !have_anchor; }
                if (c_l != kNothing) prev = c_l;
            }
        }
        if (nn) prev = __shfl_sync(0xffffffffu, cls, 31 - __clz(nn));
        rec += __popc(gen);
    }
    if (j < NV) { foreign = true; return rec; }
    if (prev == kRes) close(rec);
    __syncwarp();
    return rec;
}

// An open range of one mark type (and comment rank): its kind (kAdd / kRemove), attr, first visible index and op slot.
constexpr uint32_t kNone = 0, kAdd = 1, kRemove = 2;
struct Open { uint32_t kind, attr, start, slot; };

// Request k's MARKS walk: the number of generated mark ops; differs when the two visible token sequences differ.  Lanes build the
// log's visible -> record table and compare the texts; then lane 0 merges the two span lists, one segment of equal formatting in
// both per step, and keeps the open ranges (strong, em, link in registers; comment ranks in two sorted lists in scratch).  A range
// reserves its op slot when it opens, so ops come out by start, then type in ALL_MARKS order, then rank; it is written when it
// closes.  With kWrite the records go to out[0 ..).  Warp-collective.
template <bool kWrite>
__device__ __forceinline__ uint32_t restore_marks_walk(const RestoreParams& P, const pt_restore_request& q, uint32_t k, uint32_t lane, pt_mark_rec* out,
                                                       bool& differs) {
    const pt_log_result RL = P.res[q.log], RV = P.res[q.version];
    const uint32_t NV = RL.n_visible;
    differs = NV != RV.n_visible;
    if (differs) return 0;
    const uint32_t* tL = P.text + P.text_off[q.log];
    const uint32_t* tV = P.text + P.text_off[q.version];
    bool bad = false;
    for (uint32_t p = lane; p < NV; p += 32) bad |= __ldg(tL + p) != __ldg(tV + p);
    differs = __any_sync(0xffffffffu, bad);
    if (differs) return 0;
    // the visible -> record table of the log
    uint32_t* vis = P.vis + P.vis_off[k];
    const uint32_t* sL = P.seq + P.seq_off[q.log];
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t b = 0, v = 0; b < RL.n_elems; b += 32) {
        const uint32_t e = b + lane;
        const uint32_t w = e < RL.n_elems ? __ldg(sL + e) : 0x80000000u;
        const uint32_t m = __ballot_sync(0xffffffffu, !(w >> 31));
        if (!(w >> 31)) vis[v + __popc(m & lt)] = w & 0x3FFFFFFFu;
        v += __popc(m);
    }
    __syncwarp();
    uint32_t ops = 0;
    if (lane == 0) {
        const pt_log_desc S = P.desc[q.log];
        const uint4* ins = reinterpret_cast<const uint4*>(P.insdel + S.insdel_off);
        const pt_span* spL = P.spans + P.span_off[q.log];
        const pt_span* spV = P.spans + P.span_off[q.version];
        const uint32_t nL = RL.n_spans, nVs = RV.n_spans;
        uint4* cur = P.open + P.open_off[k];
        const uint32_t cap = (uint32_t)((P.open_off[k + 1] - P.open_off[k]) / 2);
        uint4* nxt = cur + cap;
        uint32_t n_cur = 0;
        Open st{kNone, 0, 0, 0}, em{kNone, 0, 0, 0}, ln{kNone, 0, 0, 0};
        auto emit = [&](uint32_t type, uint32_t kind, uint32_t attr, uint32_t start, uint32_t slot, uint32_t end) {
            if (!kWrite) return;
            pt_mark_rec m;
            const uint4 a = __ldg(ins + vis[start]);
            m.ctr = q.first_ctr + slot; m.actor = (uint16_t)q.actor;
            m.kind = (uint8_t)((kind == kRemove ? 1u : 0u) | (type << 1));
            m.start_ctr = a.x; m.start_actor = (uint16_t)(a.z & 0xFFFFu);
            uint32_t eb;
            m.end_ctr = 0; m.end_actor = 0;
            if (type == PT_MARK_STRONG || type == PT_MARK_EM) {
                eb = end >= NV ? PT_BOUND_END_OF_TEXT : PT_BOUND_BEFORE;
                if (end < NV) { const uint4 z = __ldg(ins + vis[end]); m.end_ctr = z.x; m.end_actor = (uint16_t)(z.z & 0xFFFFu); }
            } else {
                eb = PT_BOUND_AFTER;
                const uint4 z = __ldg(ins + vis[end - 1]); m.end_ctr = z.x; m.end_actor = (uint16_t)(z.z & 0xFFFFu);
            }
            m.bounds = (uint8_t)(PT_BOUND_BEFORE | (eb << 2));
            m.attr = attr; m.arrival = S.n_insdel; m.reserved = 0;
            out[slot] = m;
        };
        // one range of a single-valued type: close it at p unless it continues with (kind, attr); open (kind, attr) at p
        auto step = [&](Open& o, uint32_t type, uint32_t kind, uint32_t attr, uint32_t p) {
            if (o.kind != kNone && (o.kind != kind || o.attr != attr)) { emit(type, o.kind, o.attr, o.start, o.slot, p); o.kind = kNone; }
            if (kind != kNone && o.kind == kNone) o = Open{kind, attr, p, ops++};
        };
        uint32_t iL = 0, iV = 0;
        for (uint32_t p = 0; p < NV;) {
            const pt_span A = spL[iL], B = spV[iV];
            const uint32_t eL = iL + 1 < nL ? spL[iL + 1].start : NV, eV = iV + 1 < nVs ? spV[iV + 1].start : NV;
            const uint32_t qe = min(eL, eV);
            auto diff = [](bool l, bool v) { return v && !l ? kAdd : l && !v ? kRemove : kNone; };
            step(st, PT_MARK_STRONG, diff(A.flags & PT_SPAN_STRONG, B.flags & PT_SPAN_STRONG), PT_ATTR_NONE, p);
            step(em, PT_MARK_EM, diff(A.flags & PT_SPAN_EM, B.flags & PT_SPAN_EM), PT_ATTR_NONE, p);
            // comment ranks: the sorted symmetric difference of the two sets against the open list, by rank
            const uint32_t* cA = P.cpool + A.comment_off;
            const uint32_t* cB = P.cpool + B.comment_off;
            const uint32_t na = PT_SPAN_NCOMMENTS(A.flags), nb = PT_SPAN_NCOMMENTS(B.flags);
            uint32_t ia = 0, ib = 0, io = 0, n_nxt = 0;
            while (ia < na || ib < nb || io < n_cur) {
                const uint32_t ra = ia < na ? cA[ia] : 0xFFFFFFFFu, rb = ib < nb ? cB[ib] : 0xFFFFFFFFu;
                const uint32_t ro = io < n_cur ? cur[io].x : 0xFFFFFFFFu;
                const uint32_t r = min(min(ra, rb), ro);
                const uint32_t kind = ra == r && rb == r ? kNone : rb == r ? kAdd : ra == r ? kRemove : kNone;
                if (ra == r) ia++;
                if (rb == r) ib++;
                uint4 o = make_uint4(r, kNone, 0, 0);
                if (ro == r) { o = cur[io]; io++; }
                if (o.y != kNone && o.y != kind) { emit(PT_MARK_COMMENT, o.y, r, o.z, o.w, p); o.y = kNone; }
                if (kind != kNone && o.y == kNone) o = make_uint4(r, kind, p, ops++);
                if (o.y != kNone) nxt[n_nxt++] = o;
            }
            uint4* t = cur; cur = nxt; nxt = t; n_cur = n_nxt;
            const bool hl = A.flags & PT_SPAN_LINK, hv = B.flags & PT_SPAN_LINK;
            step(ln, PT_MARK_LINK, hv && (!hl || A.link_attr != B.link_attr) ? kAdd : hl && !hv ? kRemove : kNone,
                 hv && (!hl || A.link_attr != B.link_attr) ? B.link_attr : PT_ATTR_NONE, p);
            p = qe;
            if (eL == qe) iL++;
            if (eV == qe) iV++;
        }
        if (st.kind != kNone) emit(PT_MARK_STRONG, st.kind, st.attr, st.start, st.slot, NV);
        if (em.kind != kNone) emit(PT_MARK_EM, em.kind, em.attr, em.start, em.slot, NV);
        for (uint32_t i = 0; i < n_cur; i++) emit(PT_MARK_COMMENT, cur[i].y, cur[i].x, cur[i].z, cur[i].w, NV);
        if (ln.kind != kNone) emit(PT_MARK_LINK, ln.kind, ln.attr, ln.start, ln.slot, NV);
    }
    __syncwarp();
    return __shfl_sync(0xffffffffu, ops, 0);
}

template <bool kWrite>
__global__ void restore_kernel(RestoreParams P) {
    extern __shared__ uint32_t rst_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    uint32_t* cnt = rst_smem + (size_t)wib * 2 * P.maxR;
    for (uint32_t k = blockIdx.x * wpb + wib; k < P.n; k += gridDim.x * wpb) {
        if (kWrite && (P.status[k] != PT_RESTORE_OK || P.n_ops[k] == 0)) continue;
        const pt_restore_request q = P.req[k];
        const pt_log_desc S = P.desc[q.log];
        const pt_change_desc C = P.cdesc[q.log];
        const uint32_t R = S.n_actors, n = C.n_changes;
        const pt_change_rec* c0 = P.changes + C.change_off;
        uint32_t status = PT_RESTORE_OK;
        // ---- 1: the log's clock and the table's rules ----
        if (P.res[q.log].status != PT_LOG_OK || P.res[q.version].status != PT_LOG_OK) {
            status = PT_RESTORE_LOG_FAILED;
        } else {
            for (uint32_t a = lane; a < R; a += 32) cnt[a] = 0;
            __syncwarp();
            uint32_t* pos = P.pos + P.slot_off[k];
            if (!ptct::source_clock(c0, C, S, cnt, pos, lane)) status = PT_RESTORE_BAD_TABLE;
            const pt_dep_rec* d0 = P.deps + C.dep_off;
            bool bad = false;
            for (uint32_t base = 0; status == PT_RESTORE_OK && base < n; base += 32) {
                const uint32_t c = base + lane;
                if (c >= n) continue;
                const uint4 r = __ldg(reinterpret_cast<const uint4*>(c0 + c));
                for (uint32_t d = 0; d < (r.y >> 16); d++) bad |= d0[r.z + d].actor >= R;
                bad |= !ptct::change_records(P.marks + S.mark_off, S, pos[c], r.w).fits;
            }
            if (__any_sync(0xffffffffu, bad)) status = PT_RESTORE_BAD_TABLE;
            __syncwarp();
        }
        // ---- 2, 3: the walk ----
        uint32_t ops = 0, fresh = 0;
        if (status == PT_RESTORE_OK && P.mode == PT_RESTORE_TEXT) {
            bool foreign;
            ops = restore_walk<kWrite>(P, q, lane, kWrite ? P.out_insdel + P.delta[q.log].insdel_off : nullptr, foreign, fresh);
            if (foreign) { status = PT_RESTORE_FOREIGN; ops = 0; }
        } else if (status == PT_RESTORE_OK) {
            bool differs;
            ops = restore_marks_walk<kWrite>(P, q, k, lane, kWrite ? P.out_marks + P.delta[q.log].mark_off : nullptr, differs);
            if (differs) { status = PT_RESTORE_TEXT_DIFFERS; ops = 0; }
        }
        // ---- 4: the change record: its deps are the table's seq-1 changes in table order, each actor with its count ----
        const pt_change_desc DC = kWrite ? P.delta_cdesc[q.log] : pt_change_desc{};
        const uint32_t nd = status != PT_RESTORE_OK ? 0u : ptct::first_shown(c0, n, [&](uint32_t a, uint32_t j) {
            if (kWrite) P.out_deps[DC.dep_off + j] = pt_dep_rec{cnt[a], (uint16_t)a, 0};
        }, lane);
        const uint32_t seq = status == PT_RESTORE_OK && ops ? cnt[q.actor] + 1u : 0u;
        if (lane == 0) {
            if (kWrite) P.out_changes[DC.change_off] = pt_change_rec{seq, (uint16_t)q.actor, (uint16_t)nd, 0u, ops};
            else { P.status[k] = status; P.n_ops[k] = ops; P.n_deps[k] = ops ? nd : 0u; P.seq_out[k] = seq; P.elems[k] = P.res[q.log].n_elems + fresh; }
        }
        __syncwarp();
    }
}

}  // namespace ptrs
