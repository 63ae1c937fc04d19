// plan.h — the host-side plan of a batch: which kernel merges each log, in what order, and what the launches need.
// Plain C++ with no CUDA.  engine.cu launches only from a Plan; tests/test_gpu_routes.py::expected_route restates route_of.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/peritext_b200.h"

namespace ptp {

constexpr int kNumBins = 5;
struct BinCfg { uint32_t max_recs; int block; uint32_t smem; int ctas_per_sm; };
// shared memory per SM: 228 KB, 1 KB reserved per resident CTA, 227 KB max per CTA.
// Bin 0 is the WARP-PER-LOG kernel (warp_kernel.cuh): block = warps per CTA * 32, smem = bytes PER WARP; a log it cannot
// finish is deferred on the device to bin 1.  Its geometry can be set per batch (RouteConfig).
// Bins 1..4 are the CTA-per-log kernel (merge_kernel.cuh).
constexpr BinCfg kWarpBin = {2048u, 8 * 32, 7136u, 4};
constexpr BinCfg kCtaBins[kNumBins] = {
    {0u, 0, 0u, 0},                        // bin 0: RouteConfig::warp
    {1536u, 128, 31u * 1024u, 7},
    {4096u, 256, 74u * 1024u, 3},
    {12288u, 512, 112u * 1024u, 2},
    {0xFFFFFFFFu, 1024, 226u * 1024u, 1},
};
constexpr int kTeamWarps = 8;                 // team kernel (team_kernel.cuh): 8 warps per log, 4 logs per SM
constexpr uint32_t kTeamSmem = 55u * 1024u;

// Which kernels a batch may use, read from the environment by every plan (tests compare the kernels on one batch):
//   PT_WARP=0                  the CTA-per-log kernels only (no warp, no team kernel)
//   PT_WARP=max:warps:slice:ctas   the warp bin's geometry: at most `max` records, `warps` per CTA (2, 4 or 8), `slice`
//                              shared-memory bytes per warp (KB, or bytes when >= 256), `ctas` per SM; any other form
//                              leaves the default bin
//   PT_WARP_FORCE=1            send a log to the warp kernel without the host's footprint estimate (device-side deferral)
//   PT_TEAM=0                  no team kernel
//   PT_PATCH_WARP=0            with PT_FLAG_EMIT_LARGE_PATCHES: no patch_logs_kernel; every log is a candidate of
//                              patch_large_kernel (tests reach the large kernel with small logs; the probe times it on them)
struct RouteConfig {
    BinCfg warp = kWarpBin;
    bool warp_on = true, team_on = true, force = false, patch_warp_on = true;
    static RouteConfig from_env();
};

#ifdef __CUDACC__
#define PTP_HD __host__ __device__
#else
#define PTP_HD
#endif
// The global scratch slot of one patch_large_kernel log (patch_large_kernel.cuh): byte offsets of its tables, 16-aligned.
// The host sizes a slot with N = n (N, the log's element count, is at most n); the kernel lays it out with the real N.
struct LargeLayout {
    uint64_t T, PosOf, TIns, TDel, Ps, Pe, PeRaw, MKey, MInf, MAttr, MArr, CIdx, Pres, Vis, PresPre, VisPre, SBits, SPre, Bnd, FirstDef, Tree, CSort, bytes;
    uint32_t NW, SW, P2, P2c;   // bitmap words over positions / over slots; leaves per mark-type tree; comment sort length
};
PTP_HD inline uint64_t large_take(uint64_t& at, uint64_t bytes) { const uint64_t o = at; at += (bytes + 15) & ~15ull; return o; }
PTP_HD inline LargeLayout large_layout(uint64_t n, uint64_t m, uint64_t KS, uint64_t N) {
    LargeLayout g{};
    uint64_t at = 0;
    g.NW = (uint32_t)(N >> 5) + 1; g.SW = (uint32_t)((2 * N) >> 5) + 1;
    g.P2 = 1; while (g.P2 < 2 * m + 1) g.P2 <<= 1;
    g.P2c = 1; while (g.P2c < m) g.P2c <<= 1;
    g.T = large_take(at, 4 * KS); g.PosOf = large_take(at, 4 * n); g.TIns = large_take(at, 4 * N); g.TDel = large_take(at, 4 * N);
    g.Ps = large_take(at, 4 * m); g.Pe = large_take(at, 4 * m); g.PeRaw = large_take(at, 4 * m); g.MKey = large_take(at, 4 * m);
    g.MInf = large_take(at, 4 * m); g.MAttr = large_take(at, 4 * m); g.MArr = large_take(at, 4 * m); g.CIdx = large_take(at, 4 * m);
    g.Pres = large_take(at, 4ull * g.NW); g.Vis = large_take(at, 4ull * g.NW); g.PresPre = large_take(at, 4ull * (g.NW + 1)); g.VisPre = large_take(at, 4ull * (g.NW + 1));
    g.SBits = large_take(at, 4ull * g.SW); g.SPre = large_take(at, 4ull * (g.SW + 1));
    g.Bnd = large_take(at, 4 * (2 * m + 2)); g.FirstDef = large_take(at, 4 * (2 * m + 2));
    g.Tree = large_take(at, 8ull * 4 * 2 * g.P2); g.CSort = large_take(at, 8ull * g.P2c);
    g.bytes = at;
    return g;
}
PTP_HD inline uint64_t large_patch_bytes(uint64_t n, uint64_t m, uint64_t KS, uint64_t N) { return large_layout(n, m, KS, N).bytes; }
constexpr uint32_t kLargeCtasPerSm = 1;       // patch_large_kernel: 512 threads, one resident CTA per SM

// Where a log is merged.  Bin 0's list holds, in this order, the warp kernel's three id-table launches and the team kernel.
enum Route : uint8_t { kPacked3, kCompact, kDirect, kTeam, kCta1, kCta2, kCta3, kCta4, kNumRoutes };
constexpr int route_bin(int r) { return r < kCta1 ? 0 : r - kCta1 + 1; }
Route route_of(const pt_log_desc& L, const RouteConfig& cfg, bool emit_sequence);

// Worst-case arena bytes of one CTA-per-log merge (merge_kernel.cuh).
size_t arena_worst_bytes(uint64_t n, uint64_t m, uint64_t KS);

struct Plan {
    RouteConfig cfg;                          // the geometry the batch is launched with
    std::vector<uint32_t> order;              // log indices by route, each route's logs largest first
    uint32_t bin_first[kNumBins + 1] = {};    // bin k's logs are order[bin_first[k], bin_first[k + 1])
    uint32_t n_route[kNumRoutes] = {};
    std::vector<uint64_t> text_off, span_off; // per-log output capacity: n_insdel tokens, min(n_insdel, 2 n_mark + 1) spans
    uint64_t n_text = 0, n_span = 0;
    uint64_t pool_cap = 0;                    // comment-pool entries
    uint32_t n_spill = 0, slab_slots = 0;     // logs that can spill to the global slab / slab slots to allocate
    size_t slab_bytes = 0;                    // per slot
    uint32_t patch_smem = 0;                  // patch kernel's shared memory (PT_FLAG_EMIT_PATCHES)
    // PT_FLAG_EMIT_LARGE_PATCHES: the logs patch_logs_kernel can decline besides failed merges (key space >= 0xFFFF, or a
    // host footprint estimate above its 200 KB cap; every log with PT_PATCH_WARP=0), the scratch bytes of one slot (the
    // largest candidate) and the slots (one per resident CTA of patch_large_kernel, at most one per candidate)
    std::vector<uint32_t> large_cand;
    uint64_t large_bytes = 0;
    uint32_t large_slots = 0;
};

// Plans the batch into `plan`; returns nullptr, or what is wrong with the descriptors (then `plan` is unchanged).
const char* make_plan(const pt_packed_ops& ops, const pt_limits& limits, int num_sms, Plan& plan);

}  // namespace ptp
