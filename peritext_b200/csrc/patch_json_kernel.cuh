// patch_json_kernel.cuh — pt_batch_render_patches_json: the Patch[] that Micromerge.applyChange returns for every list op of
// every log (reference src/micromerge.ts:25-31, 659-703; src/peritext.ts:175-281) as UTF-8 JSON text, written on the device
// from what the merge left behind: the op records, the patch kernel's pt_patch_rec per ins/del record and its item pool.
//
// Output of a log whose merge status and patch status are 0 (DESIGN.md §4.7 has the full contract): one inner array per list
// op, arrival order, keys sorted:
//   insert  [{"action":"insert","index":I,"marks":M,"path":["text"],"values":[V]}]
//   delete  [{"action":"delete","count":1,"index":I,"path":["text"]}], or [] when it is not the element's first delete
//   mark    [{"action":A,"attrs":F,"endIndex":b,"markType":T,"path":["text"],"startIndex":a},...] ascending startIndex; attrs
//           only for addMark of a link / comment
// M is the span render's marks object, V the element's value alone as JSON.stringify writes it (render_kernel.cuh's rules).
//
// Item order.  The patch kernel appends items to its pool in atomic order.  Every item has an owner: a comment id belongs to
// its ins/del record (insdel_off + tag), a mark patch to n_insdel_total + mark_off + its mark record.  pitem_count_kernel
// counts the items per owner, the download path's scan gives each owner a segment, pitem_scatter_kernel drops every item
// into its owner's segment (any order) and pitem_rank_kernel moves it to its rank by key inside the segment.  Keys are unique
// in a segment (a comment id is emitted once per insert; one op's mark patches start at strictly increasing indices), so the
// ordered items, and the bytes, do not depend on the pool's order.
//
// Render.  Size pass, scan, write pass, as for the span render, but one warp per log and one LANE per op, 32 ops per trip in
// arrival order: each lane counts its op with op_out<false>, a warp scan places it, and the write pass writes it with
// op_out<true> at its position.  Patches are small and independent, and a c4 log has about a thousand of them.
#pragma once
#include "render_kernel.cuh"
#include "patch_window.cuh"

namespace ptr {

struct PatchJsonIn {
    const pt_log_desc* __restrict__ desc;
    const pt_insdel_rec* __restrict__ insdel;
    const pt_mark_rec* __restrict__ marks;
    const pt_log_result* __restrict__ res;
    const pt_patch_rec* __restrict__ recs;          // one per ins/del record
    const uint32_t* __restrict__ pstatus;           // per log: 0 computed on the device
    const unsigned long long* __restrict__ seg;     // [n_owners + 1] the owners' segments of the ordered items
    const uint2* __restrict__ items;                // ordered items: (a, b)
    const uint32_t* __restrict__ first_op;          // per log: list-op position of the patch window's first op (0: whole log)
    uint64_t n_insdel;                              // the batch's ins/del records: the mark owners start here
};

__device__ __forceinline__ uint64_t item_owner(const pt_patch_item& it, const pt_log_desc* __restrict__ desc, uint64_t n_insdel) {
    const pt_log_desc& L = desc[it.log];
    return (it.tag & 0x80000000u) ? n_insdel + L.mark_off + (it.tag & 0x7FFFFFFFu) : L.insdel_off + it.tag;
}

__global__ void pitem_count_kernel(const pt_patch_item* __restrict__ items, uint64_t n, const pt_log_desc* __restrict__ desc, uint64_t n_insdel,
                                   unsigned long long* __restrict__ cnt) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(&cnt[item_owner(items[i], desc, n_insdel)], 1ull);
}

// cnt counts down to zero: each item takes one slot of its owner's segment
__global__ void pitem_scatter_kernel(const pt_patch_item* __restrict__ items, uint64_t n, const pt_log_desc* __restrict__ desc, uint64_t n_insdel,
                                     unsigned long long* __restrict__ cnt, const unsigned long long* __restrict__ seg, pt_patch_item* __restrict__ tmp) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const pt_patch_item it = items[i];
        const uint64_t o = item_owner(it, desc, n_insdel);
        tmp[seg[o] + atomicAdd(&cnt[o], ~0ull) - 1ull] = it;     // adds -1
    }
}

// an item's rank in its segment = the number of smaller keys there: O(segment) per item, no more than the patch kernel's own
// O(mark ops) / O(comment ops) loop that emitted it
__global__ void pitem_rank_kernel(const pt_patch_item* __restrict__ tmp, uint64_t n, const pt_log_desc* __restrict__ desc, uint64_t n_insdel,
                                  const unsigned long long* __restrict__ seg, uint2* __restrict__ sorted) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const pt_patch_item it = tmp[i];
        const uint64_t o = item_owner(it, desc, n_insdel), s0 = seg[o], s1 = seg[o + 1];
        uint64_t r = 0;
        for (uint64_t q = s0; q < s1; q++) r += tmp[q].a < it.a;
        sorted[s0 + r] = make_uint2(it.a, it.b);
    }
}

// One lane's literal bytes.
template <bool W> __device__ __forceinline__ uint32_t lane_lit(uint8_t* d, const char* s, uint32_t len) {
    if (W) for (uint32_t k = 0; k < len; k++) d[k] = (uint8_t)s[k];
    return len;
}
#define PTJ_LIT(W, d, s) lane_lit<W>(d, s, (uint32_t)(sizeof(s) - 1))

template <bool W> __device__ __forceinline__ uint32_t put_dec(uint8_t* d, uint32_t v) {
    uint32_t len = 1;
    for (uint32_t t = v; t >= 10u; t /= 10u) len++;
    if (W) for (uint32_t k = len; k-- > 0; v /= 10u) d[k] = (uint8_t)('0' + v % 10u);
    return len;
}

// A pool fragment by one lane, or nothing (and a note of the missing entry in the size pass) when r is beyond the pool.
template <bool W> __device__ __forceinline__ uint32_t pool_frag(const uint8_t* data, const uint64_t* off, uint64_t count, uint32_t r, uint32_t kind,
                                                                uint8_t* d, unsigned long long* miss, uint32_t log) {
    if (r >= count) { if (!W) note_missing(miss, log, kind, r); return 0; }
    return frag_copy<W>(data + off[r], off[r + 1] - off[r], d);
}

// The inner array of list op `j` of its kind (ins/del record j, or mark record j) of log `log`: its bytes at d (W) or its
// byte count (!W).  One lane.
template <bool W>
__device__ uint32_t op_out(const PatchJsonIn& I, const JsonPools& P, const pt_log_desc& L, uint32_t log, bool is_mark, uint32_t j, uint8_t* d,
                           unsigned long long* miss) {
    uint32_t n = 0;
    if (!is_mark) {
        const uint64_t r = L.insdel_off + j;
        const pt_patch_rec pr = I.recs[r];
        const uint32_t payload = I.insdel[r].payload, idx = pr.index & 0x7FFFFFFFu;
        if (PT_PAYLOAD_KIND(payload) == PT_KIND_DELETE) {
            if (!(pr.index >> 31)) return PTJ_LIT(W, d, "[]");
            n += PTJ_LIT(W, d, "[{\"action\":\"delete\",\"count\":1,\"index\":");
            n += put_dec<W>(d + n, idx);
            n += PTJ_LIT(W, d + n, ",\"path\":[\"text\"]}]");
            return n;
        }
        n += PTJ_LIT(W, d, "[{\"action\":\"insert\",\"index\":");
        n += put_dec<W>(d + n, idx);
        n += PTJ_LIT(W, d + n, ",\"marks\":{");
        bool sep = false;
        if (pr.flags & PT_SPAN_COMMENT) {
            n += PTJ_LIT(W, d + n, "\"comment\":[");
            const uint64_t s0 = I.seg[r], s1 = I.seg[r + 1];
            for (uint64_t q = s0; q < s1; q++) {
                if (q > s0) n += PTJ_LIT(W, d + n, ",");
                n += pool_frag<W>(P.com, P.coff, P.ncom, I.items[q].x, 2, d + n, miss, log);
            }
            n += PTJ_LIT(W, d + n, "]");
            sep = true;
        }
        if (pr.flags & PT_SPAN_EM) {
            if (sep) n += PTJ_LIT(W, d + n, ",");
            n += PTJ_LIT(W, d + n, "\"em\":{\"active\":true}");
            sep = true;
        }
        if (pr.flags & PT_SPAN_LINK) {
            if (sep) n += PTJ_LIT(W, d + n, ",");
            n += PTJ_LIT(W, d + n, "\"link\":");
            n += pool_frag<W>(P.link, P.loff, P.nlink, pr.link_attr, 1, d + n, miss, log);
            sep = true;
        }
        if (pr.flags & PT_SPAN_STRONG) {
            if (sep) n += PTJ_LIT(W, d + n, ",");
            n += PTJ_LIT(W, d + n, "\"strong\":{\"active\":true}");
        }
        n += PTJ_LIT(W, d + n, "},\"path\":[\"text\"],\"values\":[\"");
        // every value is a string of its own: surrogate halves pair only inside it
        n += elem_out<W>(make_elem<W>(PT_PAYLOAD_TOKEN(payload), P, miss, log), kNoUnit, kNoUnit, d + n);
        n += PTJ_LIT(W, d + n, "\"]}]");
        return n;
    }
    const uint64_t k = L.mark_off + j, o = I.n_insdel + k;
    const uint32_t kind = I.marks[k].kind, attr = I.marks[k].attr, type = (kind >> 1) & 3u;
    const bool add = !(kind & 1u), with_attrs = add && (type == PT_MARK_COMMENT || type == PT_MARK_LINK);
    const uint64_t s0 = I.seg[o], s1 = I.seg[o + 1];
    n += PTJ_LIT(W, d, "[");
    for (uint64_t q = s0; q < s1; q++) {
        const uint2 ab = I.items[q];
        if (q > s0) n += PTJ_LIT(W, d + n, ",");
        n += add ? PTJ_LIT(W, d + n, "{\"action\":\"addMark\",") : PTJ_LIT(W, d + n, "{\"action\":\"removeMark\",");
        if (with_attrs) {
            n += PTJ_LIT(W, d + n, "\"attrs\":");
            n += type == PT_MARK_LINK ? pool_frag<W>(P.link, P.loff, P.nlink, attr, 1, d + n, miss, log)
                                      : pool_frag<W>(P.com, P.coff, P.ncom, attr, 2, d + n, miss, log);
            n += PTJ_LIT(W, d + n, ",");
        }
        n += PTJ_LIT(W, d + n, "\"endIndex\":");
        n += put_dec<W>(d + n, ab.y);
        n += PTJ_LIT(W, d + n, ",\"markType\":\"");
        switch (type) {
            case PT_MARK_STRONG: n += PTJ_LIT(W, d + n, "strong"); break;
            case PT_MARK_EM: n += PTJ_LIT(W, d + n, "em"); break;
            case PT_MARK_COMMENT: n += PTJ_LIT(W, d + n, "comment"); break;
            default: n += PTJ_LIT(W, d + n, "link"); break;
        }
        n += PTJ_LIT(W, d + n, "\",\"path\":[\"text\"],\"startIndex\":");
        n += put_dec<W>(d + n, ab.x);
        n += PTJ_LIT(W, d + n, "}");
    }
    n += PTJ_LIT(W, d + n, "]");
    return n;
}

// Log `log`'s patch JSON at d (W) or its byte count (!W).  Warp-collective; every lane returns the same count.
// Op order: mark record k sits at position arrival_k + k, so it comes before ins/del record arrival_k; a trip's lanes learn
// which of their positions hold mark ops from one OR-reduction of the 32 next marks' positions.  The trips start at the patch
// window's first position, with the records before it counted by the patch kernel's own rule (patch_window.cuh).
template <bool W>
__device__ uint64_t render_patch_log(const PatchJsonIn& I, const JsonPools& P, uint32_t log, uint8_t* d, unsigned long long* miss, uint32_t lane) {
    const pt_log_desc L = I.desc[log];
    const uint32_t n = L.n_insdel, m = L.n_mark, total = n + m, w0 = I.first_op[log];
    uint64_t pos = 0;
    PTR_LIT(W, d, pos, "[", lane);
    uint32_t mi = ptw::marks_before(I.marks + L.mark_off, n, m, w0, lane), ri = w0 - mi;   // ins/del and mark records before this trip
    for (uint32_t base = w0; base < total; base += 32) {
        uint32_t bit = 0;
        if (mi + lane < m) {
            const uint32_t p = min(I.marks[L.mark_off + mi + lane].arrival, n) + mi + lane;
            if (p >= base && p < base + 32) bit = 1u << (p - base);
        }
        const uint32_t mk = __reduce_or_sync(kFull, bit), below = __popc(mk & ((1u << lane) - 1u));
        const bool is_mark = (mk >> lane) & 1u;
        const uint32_t j = is_mark ? mi + below : ri + lane - below, p = base + lane;
        const bool live = p < total && j < (is_mark ? m : n);
        const uint32_t c = live ? (p != w0 ? 1u : 0u) + op_out<false>(I, P, L, log, is_mark, j, nullptr, miss) : 0u;
        const uint32_t incl = warp_incl_scan(c, lane);
        if (W && live) {
            uint8_t* o = d + pos + incl - c;
            if (p != w0) *o++ = ',';
            op_out<true>(I, P, L, log, is_mark, j, o, nullptr);
        }
        pos += __shfl_sync(kFull, incl, 31);
        mi += __popc(mk); ri += 32u - __popc(mk);
    }
    PTR_LIT(W, d, pos, "]", lane);
    return pos;
}

__device__ __forceinline__ bool patch_log_renders(const PatchJsonIn& I, uint32_t li) { return I.res[li].status == PT_LOG_OK && I.pstatus[li] == 0; }

// One warp per log, grid-stride.
__global__ void patches_json_size_kernel(const PatchJsonIn I, uint32_t n_logs, JsonPools P, unsigned long long* __restrict__ sizes,
                                         unsigned long long* __restrict__ miss) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        const uint64_t s = patch_log_renders(I, li) ? render_patch_log<false>(I, P, li, nullptr, miss, lane) : 0;
        if (lane == 0) sizes[li] = s;
    }
}

__global__ void patches_json_write_kernel(const PatchJsonIn I, uint32_t n_logs, JsonPools P, const unsigned long long* __restrict__ off,
                                          uint8_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        if (!patch_log_renders(I, li)) continue;
        const uint64_t end = render_patch_log<true>(I, P, li, out + off[li], nullptr, lane);
#ifdef PT_RENDER_CHECK
        assert(end == off[li + 1] - off[li]);      // the write pass ends exactly where the size pass said
#else
        (void)end;
#endif
    }
}

}  // namespace ptr
