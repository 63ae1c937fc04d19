// plan.cpp — routes every log of a batch to a kernel and sizes what the launches need (plan.h).
#include "plan.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <numeric>

namespace ptp {

RouteConfig RouteConfig::from_env() {
    RouteConfig c;
    if (const char* f = getenv("PT_WARP_FORCE")) c.force = atoi(f) != 0;
    if (const char* t = getenv("PT_TEAM")) c.team_on = atoi(t) != 0;
    if (const char* pw = getenv("PT_PATCH_WARP")) c.patch_warp_on = atoi(pw) != 0;
    if (const char* w = getenv("PT_WARP")) {
        unsigned long a, wp, sl, ct;
        if (sscanf(w, "%lu:%lu:%lu:%lu", &a, &wp, &sl, &ct) == 4) {
            if (sl < 256) sl *= 1024;
            sl &= ~(unsigned long)15;
            if ((wp == 2 || wp == 4 || wp == 8) && sl * wp <= 227 * 1024) c.warp = BinCfg{(uint32_t)a, (int)wp * 32, (uint32_t)sl, (int)ct};
        } else if (atoi(w) == 0) {
            c.warp_on = false; c.team_on = false;
        }
    }
    return c;
}

Route route_of(const pt_log_desc& L, const RouteConfig& cfg, bool emit_sequence) {
    const uint64_t n = L.n_insdel, m = L.n_mark, R = L.n_actors ? L.n_actors : 1, recs = n + m, KS = (uint64_t)L.max_ctr * R;
    const bool key16 = !emit_sequence && KS < 0xFFFFull;     // the warp and team kernels: 16-bit keys, no sequence output
    // short logs: one warp per log.  Footprint estimate: id table (packed3: three actors, 2 bits per key; compact: >= 3
    // actors, one slot per counter + overflow) + bitmaps + run-tree temporaries for ~ n/3 runs; a low guess only costs a
    // device-side deferral
    // (<= 255 actors: a log with more actors goes to the CTA kernel, the route tests/test_gpu_merge_copy.py pins)
    if (cfg.warp_on && key16 && R <= 255 && recs <= cfg.warp.max_recs) {
        const bool packed3 = R == 3 && n <= 1022, compact = R >= 3 && R <= 30 && n <= 2046;
        const uint64_t idbytes = packed3 ? 4ull * L.max_ctr : compact ? 2ull * L.max_ctr + 512 : 2 * KS;
        // packed3: per-word state 16 B per 32 records, ~14 B per run for ~ n/4 runs, key bitmap + prefix
        const uint64_t rest = packed3 ? n / 2 + 32 + 14 * (n / 4) + (KS / 32 + 2) * 6 + 512 : n / 2 + 16 * n / 3 + 1024;
        if (cfg.force || idbytes + rest <= cfg.warp.smem) return packed3 ? kPacked3 : compact ? kCompact : kDirect;
    }
    // medium logs without mark ops: a team of 8 warps per log (team_kernel.cuh)
    if (cfg.team_on && key16 && m == 0 && n < 0xFFFFu && (3 * n) / 4 + 2 * KS + 2 * n + 1024 <= kTeamSmem) return kTeam;
    // the CTA bins: by record count, then by the typical shared-memory need (runs ~ n/6, segments ~ min(2m, n/2)): id table
    // + bitmaps / run offsets (~1.4 B per record) + the larger of the run-tree temporaries (~5 B per record for typing-heavy
    // logs) and the mark tables (per-op arrays + ~18 B per elementary segment); a wrong guess only costs a device-side deferral
    int bin = 1;
    while (bin < kNumBins - 1 && recs > kCtaBins[bin].max_recs) bin++;
    const uint64_t I = (n < 32000 && m < 32000) ? 2 : 4, seg = std::min<uint64_t>(2 * m + 2, n / 2 + 2);
    const uint64_t typical = KS * I + (14 * n) / 10 + std::max<uint64_t>(5 * n, m ? m * (6 * I + 13) + 18 * seg : 0) + 2048;
    while (bin < kNumBins - 1 && typical > kCtaBins[bin].smem) bin++;
    return Route(kCta1 + bin - 1);
}

static size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }

// An upper bound on the sum of every Arena::alloc in merge_one_log with M <= N <= n, S <= 2m+2, nvis <= n, Mc <= m,
// nspans <= 2m+1 (released arrays are counted too).
size_t arena_worst_bytes(uint64_t n, uint64_t m, uint64_t KS) {
    const size_t I = (n < 32000 && m < 32000) ? 2 : 4;
    size_t b = 0;
    auto A = [&](uint64_t count, size_t sz) { b += al16((size_t)count * sz); };
    const uint64_t NWr = (n + 31) / 32 + 1;
    A(KS, I); A(NWr, 4); A(NWr, 4); A(NWr, 4); A(NWr, I); A(NWr, I);               // T InsBits HeadBits VisBits HeadPre VisPre
    A(NWr * 32 + 32, 1); A(NWr * 32 + 32, 1);                                      // Other Del
    A(2 * n + 3, 8); A((2 * n + 9) / 8 + 3, 8); A((2 * n + 9) / 8 + 3, 8);         // Node Sub Sub2
    A(n + 1, I); A(n + 2, 4); A(n + 2, 4); A(n + 1, I); A(n + 1, 4); A(n + 2, I);  // RunHead PosBase VisBase Prun Key GrpOff
    A(n + 1, I); A(n + 1, I); A(n + 1, I);                                         // Unsorted Sorted SPos
    A(n / 33 + 2, I); A(KS / 32 + 2, 4); A(KS / 32 + 2, I);                        // BigList GBits GPre
    if (m) {
        const uint64_t KW = KS / 32 + 2, S = 2 * m + 2, Mc = m, nsp = 2 * m + 1, NWp = (n + 32) / 32 + 1;
        A(KW + 1, 4); A(KW + 1, I); for (int k = 0; k < 6; k++) A(m + 1, I);       // KBits KPre ByRank MRank IvA IvB IvVA IvVB
        A(m + 1, 1); A(m + 1, 4); A(m + 1, 4);                                     // MKind MAttr CompactC
        A(NWp + 1, 4); A(NWp + 1, I);                                              // BndBits SegPre
        A(2 * S + 2, 4); A(S + 1, 4); A(S + 1, 4); A(S + 2, 4);                    // Tree SegFlags SegLink CDiff
        A(n / 32 + 3, 4); A(Mc + 1, 4); A(Mc + 1, I); A(Mc + 1, I); A(Mc + 1, I);  // CHead CId CK CG0 CGn
        A(2 * Mc + 1, I); A(2 * Mc + 1, I);                                        // PcA PcB
        A(4 * Mc + 8, 4); A(4 * Mc + 9, 4); A(4 * Mc + 9, I); A(Mc + 1, I);        // HTab HCnt HOff CSlot
        A(n + 1, I); A(n / 32 + 2, 4); A(n / 32 + 2, I);                           // VisSeg HeadB HeadP
        A(nsp + 1, I); A(nsp + 1, 4); A(nsp + 1, 4); A(nsp + 1, 4);                // SpanStart SpanCC SpanCO SpanCur
    }
    return b + 256;
}

const char* make_plan(const pt_packed_ops& ops, const pt_limits& limits, int num_sms, Plan& plan) {
    Plan p;
    p.cfg = RouteConfig::from_env();
    const uint32_t nl = ops.n_logs;
    const bool emit_sequence = limits.flags & PT_FLAG_EMIT_SEQUENCE, emit_patches = limits.flags & PT_FLAG_EMIT_PATCHES;
    const bool large = emit_patches && (limits.flags & PT_FLAG_EMIT_LARGE_PATCHES);
    std::vector<uint8_t> route(nl);
    p.text_off.resize(nl); p.span_off.resize(nl);
    uint64_t ncomment_bound = 0, patch_need = 4096;
    for (uint32_t i = 0; i < nl; i++) {
        const pt_log_desc& L = ops.logs[i];
        if (L.insdel_off + L.n_insdel > ops.n_insdel_total || L.mark_off + L.n_mark > ops.n_mark_total) return "log descriptor out of range";
        p.text_off[i] = p.n_text; p.span_off[i] = p.n_span;
        p.n_text += L.n_insdel;
        p.n_span += std::min<uint64_t>(L.n_insdel, 2ull * L.n_mark + 1);
        ncomment_bound += L.n_mark;
        route[i] = route_of(L, p.cfg, emit_sequence);
        p.n_route[route[i]]++;
        const uint64_t KS = (uint64_t)L.max_ctr * (L.n_actors ? L.n_actors : 1);
        if (KS > 0x7FFFFFFFull) return "max_ctr * n_actors too large; re-rank counters densely on the host";
        // only a log whose worst-case working set exceeds the largest shared-memory budget can ever spill to the global slab
        const size_t worst = arena_worst_bytes(L.n_insdel, L.n_mark, KS);
        if (worst > kCtaBins[kNumBins - 1].smem) { p.slab_bytes = std::max(p.slab_bytes, worst); p.n_spill++; }
        if (emit_patches) {   // the patch kernel's footprint; logs above the 200 KB cap are left to the host
            const uint64_t need = ((KS * 2 + 15) & ~15ull) + 3 * (((uint64_t)L.n_insdel * 2 + 15) & ~15ull) + (((uint64_t)L.n_insdel * 4 + 15) & ~15ull) +
                                  6 * (((uint64_t)L.n_mark * 4 + 15) & ~15ull) + (((uint64_t)L.n_mark * 2 + 15) & ~15ull) + 256;
            if (need <= 200 * 1024) patch_need = std::max(patch_need, need);
            if (large && (!p.cfg.patch_warp_on || KS >= 0xFFFFull || need > 200 * 1024)) {
                p.large_cand.push_back(i);
                p.large_bytes = std::max<uint64_t>(p.large_bytes, large_patch_bytes(L.n_insdel, L.n_mark, KS, L.n_insdel));
            }
        }
    }
    if (emit_patches) p.patch_smem = (uint32_t)((patch_need + 1023) & ~1023ull);   // one warp per CTA: the largest footprint
    p.large_slots = (uint32_t)std::min<size_t>(p.large_cand.size(), (size_t)num_sms * kLargeCtasPerSm);
    // default pool: 4 entries per mark op (+slack) fits the generated workloads (c3, the densest, needs < 2); a batch that needs
    // more reports its exact demand and merges again (BatchEngine.run), so the pool need not be sized for the worst case
    p.pool_cap = limits.comment_pool_entries ? limits.comment_pool_entries : 4ull * ncomment_bound + 1024;
    // spill slab: one slot per CTA that can ever spill = min(logs that can spill, CTAs of the last bin); a batch with one huge
    // log does not multiply its worst case by the whole grid
    p.slab_slots = (uint32_t)std::min<size_t>(p.n_spill, (size_t)num_sms * kCtaBins[kNumBins - 1].ctas_per_sm);
    p.order.resize(nl);
    std::iota(p.order.begin(), p.order.end(), 0u);
    std::stable_sort(p.order.begin(), p.order.end(), [&](uint32_t x, uint32_t y) {
        if (route[x] != route[y]) return route[x] < route[y];
        return (uint64_t)ops.logs[x].n_insdel + ops.logs[x].n_mark > (uint64_t)ops.logs[y].n_insdel + ops.logs[y].n_mark; });
    for (int r = 0; r < kNumRoutes; r++) p.bin_first[route_bin(r) + 1] += p.n_route[r];
    for (int k = 0; k < kNumBins; k++) p.bin_first[k + 1] += p.bin_first[k];
    plan = std::move(p);
    return nullptr;
}

}  // namespace ptp
