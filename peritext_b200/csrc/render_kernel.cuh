// render_kernel.cuh — pt_batch_render_json: every merged document's FormatSpanWithText[] (reference src/peritext.ts:35-38,
// 337-455) as UTF-8 JSON text, written on the device from the capacity-layout outputs the merge left behind.
//
// Output of a log that merged (DESIGN.md §4.6 has the full contract):
//   [{"marks":{"comment":[C,...],"em":{"active":true},"link":L,"strong":{"active":true}},"text":T},...]
// keys sorted, only the marks present; T is the span's text as JSON.stringify writes a string (well-formed form: escapes
// \" \\ \b \t \n \f \r, \u00xx below U+0020, lone surrogates \udxxx, everything else raw UTF-8; a high surrogate followed by
// a low one in the same span is one 4-byte character even across elements); C / L are the caller's pool fragments, copied
// verbatim except that an encoded lone surrogate (ED A0..BF xx) becomes \udxxx.  A failed log renders as zero bytes.
//
// Two passes with one decomposition: json_size_kernel computes each log's exact byte count, an exclusive scan gives the
// offsets, json_write_kernel writes.  Both run render_log<W>: one warp per log, spans in order, a span's elements 32 per
// trip (one per lane).  Everything that decides a byte count is shared between the passes (unit_out, frag_out, emit_lit
// take a write-or-count flag; the write pass counts each element with the same call before it writes it), so the passes
// cannot disagree.  Build with -DPT_RENDER_CHECK (make RENDER_CHECK=1) to assert that on the device.
#pragma once
#include <cassert>
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace ptr {

struct JsonPools {                 // device copies of pt_json_pools
    const uint8_t* val; const uint64_t* voff; uint64_t nval;
    const uint8_t* link; const uint64_t* loff; uint64_t nlink;
    const uint8_t* com; const uint64_t* coff; uint64_t ncom;
};

constexpr uint32_t kFull = 0xffffffffu;
constexpr uint32_t kNoUnit = 0xffffffffu;        // "no neighbouring unit" (span start / end); neither surrogate half

__device__ __forceinline__ bool is_hi(uint32_t u) { return (u & 0xFC00u) == 0xD800u; }
__device__ __forceinline__ bool is_lo(uint32_t u) { return (u & 0xFC00u) == 0xDC00u; }

template <bool W> __device__ __forceinline__ uint32_t put_u_escape(uint8_t* d, uint32_t u) {   // \uxxxx, lowercase hex
    if (W) {
        const char* hx = "0123456789abcdef";
        d[0] = '\\'; d[1] = 'u'; d[2] = hx[(u >> 12) & 15]; d[3] = hx[(u >> 8) & 15]; d[4] = hx[(u >> 4) & 15]; d[5] = hx[u & 15];
    }
    return 6;
}

// Bytes of UTF-16 unit u of a span's text, given the units just before (p) and after (n) it in the same span.  A paired
// high surrogate writes the 4-byte character and its low half writes nothing.
template <bool W> __device__ __forceinline__ uint32_t unit_out(uint32_t u, uint32_t p, uint32_t n, uint8_t* d) {
    if (u < 0x80u) {
        uint8_t e = 0;
        switch (u) {
            case '"': e = '"'; break; case '\\': e = '\\'; break; case 8: e = 'b'; break; case 9: e = 't'; break;
            case 10: e = 'n'; break; case 12: e = 'f'; break; case 13: e = 'r'; break; default: break;
        }
        if (e) { if (W) { d[0] = '\\'; d[1] = e; } return 2; }
        if (u < 0x20u) return put_u_escape<W>(d, u);
        if (W) d[0] = (uint8_t)u;
        return 1;
    }
    if (u < 0x800u) { if (W) { d[0] = (uint8_t)(0xC0u | (u >> 6)); d[1] = (uint8_t)(0x80u | (u & 0x3Fu)); } return 2; }
    if (is_hi(u)) {
        if (!is_lo(n)) return put_u_escape<W>(d, u);
        const uint32_t c = 0x10000u + ((u - 0xD800u) << 10) + (n - 0xDC00u);
        if (W) { d[0] = (uint8_t)(0xF0u | (c >> 18)); d[1] = (uint8_t)(0x80u | ((c >> 12) & 0x3Fu)); d[2] = (uint8_t)(0x80u | ((c >> 6) & 0x3Fu)); d[3] = (uint8_t)(0x80u | (c & 0x3Fu)); }
        return 4;
    }
    if (is_lo(u)) return is_hi(p) ? 0u : put_u_escape<W>(d, u);
    if (W) { d[0] = (uint8_t)(0xE0u | (u >> 12)); d[1] = (uint8_t)(0x80u | ((u >> 6) & 0x3Fu)); d[2] = (uint8_t)(0x80u | (u & 0x3Fu)); }
    return 3;
}

// One element's value as UTF-16 units: a code point token gives 1 or 2 units, a pooled value its units from the pool.
struct Elem {
    uint32_t n = 0, u0 = kNoUnit, u1 = kNoUnit;
    const uint8_t* p = nullptr;
    __device__ __forceinline__ uint32_t unit(uint32_t j) const { return p ? (uint32_t)p[2 * j] | ((uint32_t)p[2 * j + 1] << 8) : (j ? u1 : u0); }
    __device__ __forceinline__ uint32_t first() const { return n ? unit(0) : kNoUnit; }
    __device__ __forceinline__ uint32_t last() const { return n ? unit(n - 1) : kNoUnit; }
};

// Missing pool entries are recorded as one 64-bit key (atomicMin: the lowest log, then kind value < link < comment, then
// the lowest index) and render as nothing.
__device__ __forceinline__ void note_missing(unsigned long long* miss, uint32_t log, uint32_t kind, uint32_t idx) {
    atomicMin(miss, ((unsigned long long)log << 34) | ((unsigned long long)kind << 32) | idx);
}

template <bool W>
__device__ __forceinline__ Elem make_elem(uint32_t tok, const JsonPools& P, unsigned long long* miss, uint32_t log) {
    Elem e;
    const uint32_t v = tok & (PT_TOKEN_POOLED - 1u);
    if (tok & PT_TOKEN_POOLED) {
        if (v >= P.nval) { if (!W) note_missing(miss, log, 0, v); return e; }
        const uint64_t a = P.voff[v], b = P.voff[v + 1];
        e.n = (uint32_t)((b - a) >> 1); e.p = P.val + a;
    } else if (v >= 0x10000u) {
        e.n = 2; e.u0 = 0xD800u + ((v - 0x10000u) >> 10); e.u1 = 0xDC00u + ((v - 0x10000u) & 0x3FFu);
    } else {
        e.n = 1; e.u0 = v;
    }
    return e;
}

template <bool W> __device__ __forceinline__ uint32_t elem_out(const Elem& e, uint32_t prev, uint32_t next, uint8_t* d) {
    uint32_t bytes = 0, p = prev, u = e.first();
    for (uint32_t j = 0; j < e.n; j++) {
        const uint32_t n = j + 1 < e.n ? e.unit(j + 1) : next;
        bytes += unit_out<W>(u, p, n, d + bytes);
        p = u; u = n;
    }
    return bytes;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t x, uint32_t lane) {
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(kFull, x, o); if (lane >= (uint32_t)o) x += y; }
    return x;
}

// Literal bytes, copied by the lanes.
template <bool W> __device__ __forceinline__ void emit_lit(uint8_t* d, uint64_t& pos, const char* s, uint32_t len, uint32_t lane) {
    if (W) for (uint32_t k = lane; k < len; k += 32) d[pos + k] = (uint8_t)s[k];
    pos += len;
}
#define PTR_LIT(W, d, pos, s, lane) emit_lit<W>(d, pos, s, (uint32_t)(sizeof(s) - 1), lane)

// The one rule for pool fragments: byte k of f[0, len) is written verbatim (1 byte), except that the 3-byte encoding of a
// lone surrogate becomes \udxxx: its lead byte writes the 6-byte escape of unit *cu, its two continuation bytes nothing.
__device__ __forceinline__ uint32_t frag_byte(const uint8_t* f, uint64_t k, uint64_t len, uint32_t& cu) {
    const uint8_t x = f[k];
    if (x == 0xEDu && k + 2 < len && (f[k + 1] & 0xE0u) == 0xA0u) { cu = 0xD000u | ((f[k + 1] & 0x3Fu) << 6) | (f[k + 2] & 0x3Fu); return 6; }
    const bool cont = (k >= 1 && f[k - 1] == 0xEDu && (x & 0xE0u) == 0xA0u && k + 1 < len) ||
                      (k >= 2 && f[k - 2] == 0xEDu && (f[k - 1] & 0xE0u) == 0xA0u);
    return cont ? 0u : 1u;
}
template <bool W> __device__ __forceinline__ void frag_put(const uint8_t* f, uint64_t k, uint32_t c, uint32_t cu, uint8_t* o) {
    if (W && c) { if (c == 6) put_u_escape<true>(o, cu); else o[0] = f[k]; }
}

// A pool fragment, 32 bytes per trip (warp-collective).
template <bool W> __device__ __forceinline__ void frag_out(const uint8_t* f, uint64_t len, uint8_t* d, uint64_t& pos, uint32_t lane) {
    for (uint64_t b = 0; b < len; b += 32) {
        const uint64_t k = b + lane;
        uint32_t c = 0, cu = 0;
        if (k < len) c = frag_byte(f, k, len, cu);
        const uint32_t incl = warp_incl_scan(c, lane);
        frag_put<W>(f, k, c, cu, d + pos + incl - c);
        pos += __shfl_sync(kFull, incl, 31);
    }
}

// A pool fragment copied by one lane; returns its byte count.
template <bool W> __device__ __forceinline__ uint32_t frag_copy(const uint8_t* f, uint64_t len, uint8_t* d) {
    uint32_t n = 0;
    for (uint64_t k = 0; k < len; k++) { uint32_t cu = 0; const uint32_t c = frag_byte(f, k, len, cu); frag_put<W>(f, k, c, cu, d + n); n += c; }
    return n;
}

// Log `log`'s JSON at d (W) or its byte count (!W).  Warp-collective; every lane returns the same count.
template <bool W>
__device__ uint64_t render_log(uint32_t log, const pt_log_result& R, const pt_span* sp, const uint32_t* tok, const uint32_t* cpool,
                               const JsonPools& P, uint8_t* d, unsigned long long* miss, uint32_t lane) {
    uint64_t pos = 0;
    PTR_LIT(W, d, pos, "[", lane);
    const uint32_t ns = R.n_spans, nv = R.n_visible;
    for (uint32_t j = 0; j < ns; j++) {
        const pt_span S = sp[j];
        const uint32_t a = S.start, e = j + 1 < ns ? sp[j + 1].start : nv;
        if (j) PTR_LIT(W, d, pos, ",", lane);
        PTR_LIT(W, d, pos, "{\"marks\":{", lane);
        bool sep = false;
        if (S.flags & PT_SPAN_COMMENT) {
            PTR_LIT(W, d, pos, "\"comment\":[", lane);
            const uint32_t nc = PT_SPAN_NCOMMENTS(S.flags);
            for (uint32_t c = 0; c < nc; c++) {
                const uint32_t r = cpool[S.comment_off + c];
                if (c) PTR_LIT(W, d, pos, ",", lane);
                if (r >= P.ncom) { if (!W && lane == 0) note_missing(miss, log, 2, r); continue; }
                frag_out<W>(P.com + P.coff[r], P.coff[r + 1] - P.coff[r], d, pos, lane);
            }
            PTR_LIT(W, d, pos, "]", lane);
            sep = true;
        }
        if (S.flags & PT_SPAN_EM) {
            if (sep) PTR_LIT(W, d, pos, ",", lane);
            PTR_LIT(W, d, pos, "\"em\":{\"active\":true}", lane);
            sep = true;
        }
        if (S.flags & PT_SPAN_LINK) {
            if (sep) PTR_LIT(W, d, pos, ",", lane);
            PTR_LIT(W, d, pos, "\"link\":", lane);
            const uint32_t r = S.link_attr;
            if (r >= P.nlink) { if (!W && lane == 0) note_missing(miss, log, 1, r); }
            else frag_out<W>(P.link + P.loff[r], P.loff[r + 1] - P.loff[r], d, pos, lane);
            sep = true;
        }
        if (S.flags & PT_SPAN_STRONG) {
            if (sep) PTR_LIT(W, d, pos, ",", lane);
            PTR_LIT(W, d, pos, "\"strong\":{\"active\":true}", lane);
        }
        PTR_LIT(W, d, pos, "},\"text\":\"", lane);
        // The span's elements, 32 per trip.  Pairing at element boundaries needs the last unit of the nearest non-empty
        // element before each lane's and the first unit of the nearest one after it (empty values "" are skipped, as
        // concatenation skips them): inside the trip from the ballot of non-empty lanes, across trips from `carry` (the
        // span's last unit so far) and the next trip's elements, which are loaded one trip ahead.
        uint32_t carry = kNoUnit;
        uint32_t la_at = a, la_unit = kNoUnit;     // cached scan past an all-empty next trip: first non-empty element >= la_at
        Elem cur = a + lane < e ? make_elem<W>(tok[a + lane], P, miss, log) : Elem();
        for (uint32_t b = a; b < e; b += 32) {
            const uint32_t nb = b + 32;
            const Elem nxt = nb + lane < e ? make_elem<W>(tok[nb + lane], P, miss, log) : Elem();
            const uint32_t ne = __ballot_sync(kFull, cur.n != 0), ne_next = __ballot_sync(kFull, nxt.n != 0);
            const uint32_t first = cur.first(), last = cur.last();
            uint32_t ahead = kNoUnit;                                // first unit after this trip, within the span
            if (ne_next) {
                ahead = __shfl_sync(kFull, nxt.first(), __ffs(ne_next) - 1);
            } else if (nb + 32 < e) {
                if (nb + 32 > la_at) {                               // scan on; each element is looked at once per span
                    la_at = e; la_unit = kNoUnit;
                    for (uint32_t q = nb + 32; q < e; q += 32) {
                        const Elem x = q + lane < e ? make_elem<W>(tok[q + lane], P, miss, log) : Elem();
                        const uint32_t m = __ballot_sync(kFull, x.n != 0);
                        if (m) { la_at = q + __ffs(m) - 1; la_unit = __shfl_sync(kFull, x.first(), __ffs(m) - 1); break; }
                    }
                }
                ahead = la_unit;
            }
            const uint32_t lower = ne & ((1u << lane) - 1u), higher = ne & ~((2u << lane) - 1u);
            uint32_t prev = __shfl_sync(kFull, last, lower ? 31 - __clz(lower) : lane);
            uint32_t next = __shfl_sync(kFull, first, higher ? __ffs(higher) - 1 : lane);
            if (!lower) prev = carry;
            if (!higher) next = ahead;
            if (ne) carry = __shfl_sync(kFull, last, 31 - __clz(ne));
            // per-element byte counts -> warp-exclusive scan -> each lane writes its element at its position
            const uint32_t c = elem_out<false>(cur, prev, next, nullptr);
            const uint32_t incl = warp_incl_scan(c, lane);
            if (W) elem_out<true>(cur, prev, next, d + pos + incl - c);
            pos += __shfl_sync(kFull, incl, 31);
            cur = nxt;
        }
        PTR_LIT(W, d, pos, "\"}", lane);
    }
    PTR_LIT(W, d, pos, "]", lane);
    return pos;
}

// One warp per log, grid-stride.  res / text_off / span_off / text / spans / cpool are the merge's capacity-layout outputs.
__global__ void json_size_kernel(const pt_log_result* __restrict__ res, uint32_t n, const uint64_t* __restrict__ text_off,
                                 const uint64_t* __restrict__ span_off, const uint32_t* __restrict__ text, const pt_span* __restrict__ spans,
                                 const uint32_t* __restrict__ cpool, JsonPools P, unsigned long long* __restrict__ sizes,
                                 unsigned long long* __restrict__ miss) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n; li += nwarps) {
        const pt_log_result R = res[li];
        const uint64_t s = R.status == PT_LOG_OK ? render_log<false>(li, R, spans + span_off[li], text + text_off[li], cpool, P, nullptr, miss, lane) : 0;
        if (lane == 0) sizes[li] = s;
    }
}

__global__ void json_write_kernel(const pt_log_result* __restrict__ res, uint32_t n, const uint64_t* __restrict__ text_off,
                                  const uint64_t* __restrict__ span_off, const uint32_t* __restrict__ text, const pt_span* __restrict__ spans,
                                  const uint32_t* __restrict__ cpool, JsonPools P, const unsigned long long* __restrict__ off,
                                  uint8_t* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n; li += nwarps) {
        const pt_log_result R = res[li];
        if (R.status != PT_LOG_OK) continue;
        const uint64_t end = render_log<true>(li, R, spans + span_off[li], text + text_off[li], cpool, P, out + off[li], nullptr, lane);
#ifdef PT_RENDER_CHECK
        assert(end == off[li + 1] - off[li]);      // the write pass ends exactly where the size pass said
#else
        (void)end;
#endif
    }
}

}  // namespace ptr
