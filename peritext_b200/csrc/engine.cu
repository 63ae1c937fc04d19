// engine.cu — C-ABI of the batch CRDT-merge engine (include/peritext_b200.h) over the sm_90a kernels.
//
// Host responsibilities (all per batch, none per op): plan the batch (plan.h: each log's kernel and bin, the order of
// the persistent-CTA work queues, output capacities), launch from the plan, and move results.  There is NO CPU
// fallback: without a CUDA device every entry point fails.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "merge_kernel.cuh"
#include "warp_kernel.cuh"
#include "patch_kernel.cuh"
#include "patch_large_kernel.cuh"
#include "team_kernel.cuh"
#include "render_kernel.cuh"
#include "patch_json_kernel.cuh"
#include "append_kernel.cuh"
#include "change_kernel.cuh"
#include "exchange_kernel.cuh"
#include "changes_json_kernel.cuh"
#include "upload_kernel.cuh"
#include "scan_kernel.cuh"
#include "admit_kernel.cuh"
#include "query_kernel.cuh"
#include "sync_kernel.cuh"
#include "checkout_kernel.cuh"
#include "attribute_kernel.cuh"
#include "restore_kernel.cuh"
#include "plan.h"

namespace {

thread_local std::string g_last_error;

#define PT_CUDA(call)                                                                                   \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) {                                                                       \
            g_last_error = std::string(#call) + ": " + cudaGetErrorString(e__);                        \
            return PT_ERR_CUDA;                                                                         \
        }                                                                                               \
    } while (0)

// Device memory, or pinned host memory, that grows on demand and is freed with its owner.
template <bool kPinned>
struct Buf {
    void* p = nullptr; size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    void release() { if (p) { if (kPinned) cudaFreeHost(p); else cudaFree(p); } p = nullptr; cap = 0; }
    void swap(Buf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
    int reserve(size_t bytes) {
        if (bytes <= cap) return PT_OK;
        release();
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = kPinned ? cudaMallocHost(&p, want) : cudaMalloc(&p, want);
        if (e != cudaSuccess) { g_last_error = std::string(kPinned ? "cudaMallocHost: " : "cudaMalloc: ") + cudaGetErrorString(e); return PT_ERR_NOMEM; }
        cap = want; return PT_OK;
    }
};
using DevBuf = Buf<false>;
using HostBuf = Buf<true>;

using ptp::kNumBins;
using ptp::kCtaBins;

// Room for n elements of T, at least one: a batch without logs or records still gets valid pointers.
template <class T, bool kPinned>
int reserve_n(Buf<kPinned>& buf, uint64_t n) { return buf.reserve(std::max<uint64_t>(1, n) * sizeof(T)); }

// One JSON render's buffers: per-log sizes, scan, offsets, missing-entry key and output on the device; the view's offsets
// and bytes and the read-back of the total in pinned memory.
struct JsonBufs {
    DevBuf size, bsum, off, miss, bytes;
    HostBuf hoff, hbytes, hmisc;
};

// The device counter block of a batch, zeroed before every merge; the kernels get pointers to its fields.
struct DevCounters {
    unsigned long long stats[3];          // BatchParams::stats: logs finished shared-only, on the spill path, deferred
    unsigned long long comment_used;      // comment-pool cursor: counts past the capacity, so it ends as the batch's demand
    unsigned long long patch_items;       // patch-item cursor, likewise
    uint32_t slab[2];                     // next free spill-slab slot: the last bin's own launch, its retry launch
    uint32_t packed3, compact, direct, team;   // work-queue heads of bin 0's launches
    uint32_t head[kNumBins];              // work-queue heads of the CTA bins' own lists ([0] unused)
    uint32_t retry_head[kNumBins];        // work-queue heads of the CTA bins' retry launches ([0] unused)
    uint32_t deferred[kNumBins];          // logs deferred into bin k, appended to list k of d_retry ([0] unused)
};

}  // namespace

struct pt_batch {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 0;
    pt_limits limits{};
    // batch
    bool have_batch = false, merged = false;
    bool patch_pool_changed = false;   // pt_batch_set_patch_pool replaced the item pool after the last merge
    bool patch_window_changed = false; // pt_batch_set_patch_window changed the window after the last merge
    uint32_t n_logs = 0;
    uint64_t n_insdel = 0, n_mark = 0;
    std::vector<pt_log_desc> h_desc;
    ptp::Plan plan;
    // device
    DevBuf d_runs, d_tokens, d_run_off, d_tok_off, d_cins, d_cmarks;
    DevBuf d_desc, d_insdel, d_marks, d_order, d_counters, d_results, d_text_off, d_span_off, d_text, d_spans, d_pool, d_slab, d_retry, d_seq;
    DevBuf d_bsum, d_ctoff, d_csoff, d_ctext, d_cspans;   // download path: packed outputs + their offsets ([n_logs + 1])
    DevBuf d_cdesc, d_changes, d_deps, d_admit;           // admission pre-pass (optional change table)
    std::vector<pt_change_desc> h_cdesc;                 // its descriptors, and its totals
    uint64_t n_changes = 0, n_deps = 0;
    DevBuf d_patch_recs, d_patch_items, d_patch_status;   // PT_FLAG_EMIT_PATCHES
    DevBuf d_patch_first;                                 // [n_logs] the patch window's first list op per log (0: whole log)
    DevBuf d_large_cand, d_large_scratch;                 // PT_FLAG_EMIT_LARGE_PATCHES: candidate logs, scratch slots
    HostBuf h_patch_recs, h_patch_items, h_patch_status, h_patch_misc, h_patch_first;
    DevBuf d_jval, d_jvoff, d_jlink, d_jloff, d_jcom, d_jcoff;          // both JSON renders: the caller's pools
    JsonBufs spans_json, patches_json;                                  // each render's own scratch and view
    JsonBufs changes_json;                                              // pt_batch_render_changes_json: its own scratch and view
    HostBuf h_cj_status;                                                //   and its per-request status
    DevBuf d_picnt, d_piseg, d_pibsum, d_pitmp, d_pisorted;             // pt_batch_render_patches_json: the ordered patch items
    uint64_t patch_cap = 0;
    bool have_changes = false;
    uint32_t adm_maxR = 1;
    const pt_insdel_rec* dp_insdel = nullptr;
    const pt_mark_rec* dp_marks = nullptr;
    DevBuf d_key_insdel, d_key_marks;     // the warp kernel's key-record copy of the records (derive_key_records); empty when
                                          // no log is on a warp route
    // pinned host
    HostBuf h_stage, h_results, h_text, h_spans, h_pool, h_misc, h_seq, h_ctoff, h_csoff;
    HostBuf h_chg_status, h_chg_desc, h_chg_insdel, h_chg_marks;   // the view of the last pt_batch_change
    HostBuf h_xch_totals, h_xch_status, h_xch_off, h_xch_delivered, h_xch_desc;   // the view of the last pt_batch_exchange
    // pt_batch_upload_actors: each log's actor ids in the PT_POOL_ACTORS layout, and per log its first id and first byte
    // ([n_logs + 1]) and whether its counters were re-ranked densely
    bool have_actors = false;
    DevBuf d_anames, d_aoff, d_afirst;
    std::vector<uint64_t> h_afirst, h_abyte;
    std::vector<char> h_adense;
    HostBuf h_act_data, h_act_off, h_act_first;                          // the view of pt_batch_download_actors
    HostBuf h_syn_totals, h_syn_status, h_syn_off, h_syn_aoff, h_syn_amap;   // the view of the last pt_batch_sync_pairs
    HostBuf h_add_totals, h_add_rank, h_add_aoff, h_add_amap;               // the view of the last pt_batch_add_actors
    HostBuf h_clk_off, h_clk_seq, h_clk_status;                             // the view of the last pt_batch_download_clocks
    HostBuf h_attr_status, h_attr_off, h_attr_runs;                         // the view of the last pt_batch_attribute
    HostBuf h_rst_status, h_rst_ops, h_rst_seq;                             // the view of the last pt_batch_restore
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaStream_t side = nullptr, launch_stream = nullptr;   // side: the CTA-per-log bins' own launches run beside the warp / team kernels
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    uint64_t launches = 0;
    cudaGraphExec_t graph_exec = nullptr;   // the merge sequence of the current batch, captured once
    bool graph_ok = false, graph_tried = false;
    uint32_t merges_since_upload = 0;
    bool dl_begun = false;
    uint32_t kernels_per_merge = 0;
    uint64_t pool_used_host = 0;
};

namespace {

DevCounters* counters(const pt_batch* b) { return (DevCounters*)b->d_counters.p; }

// The launch sequence, or a pointer or capacity baked into it, changed: capture it again at the next repeated merge.
void drop_graph(pt_batch* b) {
    if (b->graph_exec) cudaGraphExecDestroy(b->graph_exec);
    b->graph_exec = nullptr; b->graph_ok = false; b->graph_tried = false; b->merges_since_upload = 0;
}

// Every kernel launch is followed by PT_CUDA(launched(b)): the launch's error, else one more in pt_batch_launch_count.
cudaError_t launched(pt_batch* b) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) b->launches++;
    return e;
}

// reserve_n, then (n > 0) the copy of n elements from the host on the batch's stream.
template <class T>
int upload_n(pt_batch* b, DevBuf& buf, const T* src, uint64_t n) {
    int rc;
    if ((rc = reserve_n<T>(buf, n))) return rc;
    if (n) PT_CUDA(cudaMemcpyAsync(buf.p, src, n * sizeof(T), cudaMemcpyHostToDevice, b->stream));
    return PT_OK;
}

// CTAs of `threads` threads for a grid-stride loop over n_items items of `lanes` threads (a warp): at most 16 per SM.
uint32_t warp_grid(const pt_batch* b, uint64_t n_items, uint32_t threads, uint32_t lanes = 32) {
    return (uint32_t)std::min<uint64_t>((n_items * lanes + threads - 1) / threads, (uint64_t)b->num_sms * 16);
}

// One warp per item (n_items > 0), and an item with many records shared by up to 64 warps, one per slice of 8 K records
// (gridDim.y): a few huge items (c5) must not leave the copy to a handful of warps.  most: the largest item's records.
dim3 slice_grid(const pt_batch* b, uint64_t n_items, uint64_t most, uint32_t threads) {
    const uint32_t slices = (uint32_t)std::clamp<uint64_t>(most / 8192, 1, 64);
    return dim3(std::min<uint32_t>(warp_grid(b, n_items, threads), (uint32_t)b->num_sms * 16 / slices), slices);
}

// admit_kernel and exchange_select_kernel keep two words per actor for each warp in shared memory, at most kAdmitMaxBytes.
constexpr size_t kAdmitMaxBytes = 200 * 1024;
size_t actor_table_bytes(uint32_t maxR) { return (size_t)2 * maxR * 4; }

// Their launch shape (warps per CTA, shared bytes): 4 warps while the tables fit the default 48 KB, else one warp.
std::pair<uint32_t, size_t> actor_shape(uint32_t maxR) {
    const size_t per_warp = actor_table_bytes(maxR);
    const uint32_t wpb = per_warp * 4 <= 48 * 1024 ? 4u : 1u;
    return {wpb, per_warp * wpb};
}

// One warp per item over n_items items of a kernel with those tables, on the batch's stream: the launch's error, else PT_OK.
template <class... Params, class... Args>
int launch_actor_kernel(pt_batch* b, void (*kernel)(Params...), uint64_t n_items, Args... args) {
    const auto [wpb, smem] = actor_shape(b->adm_maxR);
    if (smem > 48 * 1024) PT_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<warp_grid(b, n_items, wpb * 32), wpb * 32, smem, b->stream>>>(args...);
    PT_CUDA(launched(b));
    return PT_OK;
}

// The scan triple over n per-log counts of src (scan_kernel.cuh): block sums into bsum, their scan, then each log's
// exclusive offset in off0 (channel a) and off1 (channel c; may be null), the totals at [n].
template <class Src>
int scan_offsets(pt_batch* b, Src src, uint32_t n, DevBuf& bsum_buf, unsigned long long* off0, unsigned long long* off1) {
    const uint32_t nb = (n + pts::kScanBlock - 1) / pts::kScanBlock;
    int rc;
    if ((rc = reserve_n<unsigned long long>(bsum_buf, 2 * nb + 2))) return rc;
    unsigned long long* bsum = (unsigned long long*)bsum_buf.p;
    pts::out_block_sums_kernel<<<nb, pts::kScanBlock, 0, b->stream>>>(src, n, bsum);
    PT_CUDA(launched(b));
    pts::out_scan_blocks_kernel<<<1, 1024, 0, b->stream>>>(bsum, nb);
    PT_CUDA(launched(b));
    pts::out_offsets_kernel<<<nb, pts::kScanBlock, 0, b->stream>>>(src, n, bsum, nb, off0, off1);
    PT_CUDA(launched(b));
    return PT_OK;
}

int alloc_and_upload_plan(pt_batch* b) {
    int rc;
    const size_t n = b->n_logs;
    const ptp::Plan& pl = b->plan;
    if ((rc = reserve_n<pt_log_desc>(b->d_desc, n))) return rc;
    if ((rc = reserve_n<uint32_t>(b->d_order, n))) return rc;
    if ((rc = b->d_counters.reserve(sizeof(DevCounters)))) return rc;
    if ((rc = reserve_n<pt_log_result>(b->d_results, n))) return rc;
    if ((rc = reserve_n<uint64_t>(b->d_text_off, n))) return rc;
    if ((rc = reserve_n<uint64_t>(b->d_span_off, n))) return rc;
    if ((rc = reserve_n<uint32_t>(b->d_text, pl.n_text))) return rc;
    if ((b->limits.flags & PT_FLAG_EMIT_SEQUENCE) && (rc = reserve_n<uint32_t>(b->d_seq, pl.n_text))) return rc;
    if ((rc = reserve_n<pt_span>(b->d_spans, pl.n_span))) return rc;
    if ((rc = reserve_n<uint32_t>(b->d_pool, pl.pool_cap))) return rc;
    if ((rc = reserve_n<uint32_t>(b->d_retry, n * kNumBins + 4))) return rc;
    if (b->limits.flags & PT_FLAG_EMIT_PATCHES) {
        b->patch_cap = b->limits.patch_pool_items ? b->limits.patch_pool_items : 4ull * (b->n_insdel + b->n_mark) + 1024;
        if ((rc = reserve_n<pt_patch_rec>(b->d_patch_recs, b->n_insdel))) return rc;
        if ((rc = reserve_n<pt_patch_item>(b->d_patch_items, b->patch_cap))) return rc;
        if ((rc = reserve_n<uint32_t>(b->d_patch_status, n))) return rc;
        if ((rc = reserve_n<uint32_t>(b->d_patch_first, n))) return rc;
        PT_CUDA(cudaMemsetAsync(b->d_patch_first.p, 0, n * 4, b->stream));   // every upload / append: whole logs
        b->patch_window_changed = false;
        if (!pl.large_cand.empty()) {
            if ((rc = b->d_large_cand.reserve(pl.large_cand.size() * 4))) return rc;
            if ((rc = b->d_large_scratch.reserve((size_t)pl.large_slots * pl.large_bytes))) return rc;
        }
    }
    if ((rc = b->d_slab.reserve(std::max<size_t>((size_t)pl.slab_slots * pl.slab_bytes, 16)))) return rc;
    // stage the small host-derived arrays through pinned memory
    size_t stage = n * (sizeof(pt_log_desc) + 4 + 8 + 8) + pl.large_cand.size() * 4 + 64;
    if ((rc = b->h_stage.reserve(stage))) return rc;
    char* s = (char*)b->h_stage.p;
    if (n) {
        memcpy(s, b->h_desc.data(), n * sizeof(pt_log_desc));
        PT_CUDA(cudaMemcpyAsync(b->d_desc.p, s, n * sizeof(pt_log_desc), cudaMemcpyHostToDevice, b->stream)); s += n * sizeof(pt_log_desc);
        memcpy(s, pl.order.data(), n * 4);
        PT_CUDA(cudaMemcpyAsync(b->d_order.p, s, n * 4, cudaMemcpyHostToDevice, b->stream)); s += n * 4;
        memcpy(s, pl.text_off.data(), n * 8);
        PT_CUDA(cudaMemcpyAsync(b->d_text_off.p, s, n * 8, cudaMemcpyHostToDevice, b->stream)); s += n * 8;
        memcpy(s, pl.span_off.data(), n * 8);
        PT_CUDA(cudaMemcpyAsync(b->d_span_off.p, s, n * 8, cudaMemcpyHostToDevice, b->stream)); s += n * 8;
    }
    if ((b->limits.flags & PT_FLAG_EMIT_PATCHES) && !pl.large_cand.empty()) {
        memcpy(s, pl.large_cand.data(), pl.large_cand.size() * 4);
        PT_CUDA(cudaMemcpyAsync(b->d_large_cand.p, s, pl.large_cand.size() * 4, cudaMemcpyHostToDevice, b->stream));
    }
    return PT_OK;
}

// Bin k's own list (retry = false), or the logs deferred into it (retry = true: list k of d_retry, its length on the device).
template <int BLOCK>
int launch_bin_t(pt_batch* b, int k, ptk::BatchParams P, bool retry) {
    const ptp::BinCfg& cfg = kCtaBins[k];
    uint32_t cnt = retry ? b->n_logs : b->plan.bin_first[k + 1] - b->plan.bin_first[k];
    uint32_t grid = (uint32_t)std::min<size_t>(cnt, (size_t)b->num_sms * cfg.ctas_per_sm);
    DevCounters* c = counters(b);
    uint32_t* lists = (uint32_t*)b->d_retry.p;
    if (retry) {
        P.order = lists + (size_t)k * b->n_logs; P.n_work = 0; P.n_work_dev = &c->deferred[k];
        P.work_counter = &c->retry_head[k];
    } else {
        P.order = (const uint32_t*)b->d_order.p + b->plan.bin_first[k]; P.n_work = cnt; P.n_work_dev = nullptr;
        P.work_counter = &c->head[k];
    }
    const bool last = k == kNumBins - 1;
    P.slab_bytes = last ? b->plan.slab_bytes : 0;
    P.slab_counter = &c->slab[retry ? 1 : 0];   // the two launches of the last bin run one after the other: each counts its slots from zero
    P.retry_list = last ? nullptr : lists + (size_t)(k + 1) * b->n_logs;
    P.retry_count = last ? nullptr : &c->deferred[k + 1];
    P.smem_arena_bytes = cfg.smem;
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_kernel<BLOCK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smem));
    ptk::merge_logs_kernel<BLOCK><<<grid, BLOCK, cfg.smem, b->launch_stream>>>(P);
    PT_CUDA(launched(b));
    return PT_OK;
}
// cnt logs of bin 0's list from position first, on one id-table form of the warp kernel
template <int WARPS, int IDM>
int launch_warp_range(pt_batch* b, ptk::BatchParams P, uint32_t first, uint32_t cnt, uint32_t* head) {
    if (!cnt) return PT_OK;
    const ptp::BinCfg& cfg = b->plan.cfg.warp;
    const uint32_t per_cta = WARPS * ptk::kWarpGrab;
    const uint32_t grid = (uint32_t)std::min<size_t>((cnt + per_cta - 1) / per_cta, (size_t)b->num_sms * cfg.ctas_per_sm);
    P.order = (const uint32_t*)b->d_order.p + b->plan.bin_first[0] + first; P.n_work = cnt; P.n_work_dev = nullptr;
    P.work_counter = head;
    P.slab_bytes = 0;
    P.retry_list = (uint32_t*)b->d_retry.p + (size_t)1 * b->n_logs;   // deferrals go to the first CTA-per-log bin
    P.retry_count = &counters(b)->deferred[1];
    P.smem_arena_bytes = cfg.smem;                       // per warp
    const int smem = (int)(cfg.smem * WARPS);
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_warp_kernel<WARPS, IDM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ptk::merge_logs_warp_kernel<WARPS, IDM><<<grid, WARPS * 32, smem, b->launch_stream>>>(P);
    PT_CUDA(launched(b));
    return PT_OK;
}
int launch_team_range(pt_batch* b, ptk::BatchParams P, uint32_t first, uint32_t cnt) {
    if (!cnt) return PT_OK;
    const uint32_t grid = (uint32_t)std::min<size_t>(cnt, (size_t)b->num_sms * 4);
    P.order = (const uint32_t*)b->d_order.p + b->plan.bin_first[0] + first; P.n_work = cnt; P.n_work_dev = nullptr;
    P.work_counter = &counters(b)->team;
    P.slab_bytes = 0;
    P.retry_list = (uint32_t*)b->d_retry.p + (size_t)3 * b->n_logs;   // a log that does not fit goes to the 512-thread CTA bin (and on from there)
    P.retry_count = &counters(b)->deferred[3];
    P.smem_arena_bytes = ptp::kTeamSmem;
    PT_CUDA(cudaFuncSetAttribute(ptk::merge_logs_team_kernel<ptp::kTeamWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ptp::kTeamSmem));
    ptk::merge_logs_team_kernel<ptp::kTeamWarps><<<grid, ptp::kTeamWarps * 32, ptp::kTeamSmem, b->launch_stream>>>(P);
    PT_CUDA(launched(b));
    return PT_OK;
}
// bin 0's list, in route order: the warp kernel with the packed3, compact and direct id tables, then the team kernel
template <int WARPS>
int launch_warp_bin_t(pt_batch* b, const ptk::BatchParams& P) {
    const uint32_t np = b->plan.n_route[ptp::kPacked3], nc = b->plan.n_route[ptp::kCompact], nd = b->plan.n_route[ptp::kDirect];
    DevCounters* c = counters(b);
    int rc;
    if ((rc = launch_warp_range<WARPS, ptk::kIdPacked3>(b, P, 0, np, &c->packed3))) return rc;
    if ((rc = launch_warp_range<WARPS, ptk::kIdCompact>(b, P, np, nc, &c->compact))) return rc;
    if ((rc = launch_warp_range<WARPS, ptk::kIdDirect>(b, P, np + nc, nd, &c->direct))) return rc;
    return launch_team_range(b, P, np + nc + nd, b->plan.n_route[ptp::kTeam]);
}
int launch_bin(pt_batch* b, int k, const ptk::BatchParams& P, bool retry) {
    if (!retry && b->plan.bin_first[k + 1] == b->plan.bin_first[k]) return PT_OK;
    if (k == 0) {
        switch (b->plan.cfg.warp.block / 32) {      // RouteConfig accepts 2, 4 or 8 warps per CTA
            case 2: return launch_warp_bin_t<2>(b, P);
            case 4: return launch_warp_bin_t<4>(b, P);
            default: return launch_warp_bin_t<8>(b, P);
        }
    }
    switch (k) {
        case 1: return launch_bin_t<kCtaBins[1].block>(b, k, P, retry);
        case 2: return launch_bin_t<kCtaBins[2].block>(b, k, P, retry);
        case 3: return launch_bin_t<kCtaBins[3].block>(b, k, P, retry);
        default: return launch_bin_t<kCtaBins[4].block>(b, k, P, retry);
    }
}

// Makes `plan` (made by ptp::make_plan from `ops`) the handle's batch: its shape, descriptors, per-log arrays and output
// buffers (own_records: the engine keeps its own copy of the records and allocates for them).  Every upload and
// pt_batch_append end their planning here.
int install_plan(pt_batch* b, const pt_packed_ops& ops, ptp::Plan&& plan, bool own_records) {
    b->n_logs = ops.n_logs; b->n_insdel = ops.n_insdel_total; b->n_mark = ops.n_mark_total;
    b->h_desc.assign(ops.logs, ops.logs + ops.n_logs);
    b->plan = std::move(plan);
    int rc;
    if ((rc = alloc_and_upload_plan(b))) return rc;
    if (own_records) {
        if ((rc = reserve_n<pt_insdel_rec>(b->d_insdel, b->n_insdel))) return rc;
        if ((rc = reserve_n<pt_mark_rec>(b->d_marks, b->n_mark))) return rc;
    }
    return PT_OK;
}

// Shared start of every upload: the staging buffer and the device arrays of the previous batch are reused, so wait for
// it; then plan the new batch and allocate for it.
int begin_upload(pt_batch* b, const pt_packed_ops& ops, bool own_records) {
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->have_batch = false; b->merged = false; b->dl_begun = false; b->have_changes = false; b->have_actors = false;
    drop_graph(b);
    ptp::Plan plan;
    if (const char* err = ptp::make_plan(ops, b->limits, b->num_sms, plan)) { g_last_error = err; return PT_ERR_INVALID; }
    return install_plan(b, ops, std::move(plan), own_records);
}

// The warp kernel's key-record copy of the records the merge reads (upload_kernel.cuh), derived on the batch's stream wherever
// those records change: at every upload and when pt_batch_append swaps in the spliced records.  A batch without a log on a
// warp route keeps no copy.
int derive_key_records(pt_batch* b) {
    const uint32_t* nr = b->plan.n_route;
    if (!(nr[ptp::kPacked3] + nr[ptp::kCompact] + nr[ptp::kDirect])) { b->d_key_insdel.release(); b->d_key_marks.release(); return PT_OK; }
    int rc;
    // 32 mark records of slack past the end: the warp kernel's mark pass loads one trip (32 records) ahead without a bounds clamp
    if ((rc = reserve_n<uint32_t>(b->d_key_insdel, b->n_insdel)) || (rc = reserve_n<uint2>(b->d_key_marks, b->n_mark + 32))) return rc;
    const uint32_t threads = 256;      // one warp per log
    if (b->n_logs) {
        ptu::derive_key_records_kernel<<<warp_grid(b, b->n_logs, threads), threads, 0, b->stream>>>(
            (const pt_log_desc*)b->d_desc.p, b->dp_insdel, b->dp_marks, (uint32_t*)b->d_key_insdel.p, (uint2*)b->d_key_marks.p, b->n_logs);
        PT_CUDA(launched(b));
    }
    return PT_OK;
}

// Shared finish: the records the merge reads and their key-record copy, and a wait for the copies when one of the caller's
// sources (pointer, bytes read) is pageable, because such a buffer may be freed on return (pinned ones stay asynchronous).
int finish_upload(pt_batch* b, const void* insdel, const void* marks, std::initializer_list<std::pair<const void*, uint64_t>> sources) {
    bool pageable = false;
    for (const auto& s : sources) {
        if (!s.second) continue;
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, s.first) != cudaSuccess) { cudaGetLastError(); pageable = true; }
        else if (a.type != cudaMemoryTypeHost) pageable = true;
    }
    b->dp_insdel = (const pt_insdel_rec*)insdel; b->dp_marks = (const pt_mark_rec*)marks;
    int rc;
    if ((rc = derive_key_records(b))) return rc;
    if (pageable) PT_CUDA(cudaStreamSynchronize(b->stream));
    b->have_batch = true;
    return PT_OK;
}

// pt_batch_query_elements / pt_batch_find_elements: n queries up, one warp per query, n answers back.
template <class Q, class A, class Launch>
int run_queries(pt_batch* b, const char* fn, const char* verb, const Q* queries, uint32_t n, A* out, Launch launch) {
    if (!b || (n && (!queries || !out))) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = std::string(verb) + " before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = "the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    if (!n) return PT_OK;
    PT_CUDA(cudaSetDevice(b->device));
    DevBuf dq, da;
    int rc;
    if ((rc = dq.reserve((size_t)n * sizeof(Q))) || (rc = da.reserve((size_t)n * sizeof(A)))) return rc;
    cudaError_t e = cudaMemcpyAsync(dq.p, queries, (size_t)n * sizeof(Q), cudaMemcpyHostToDevice, b->stream);
    if (e == cudaSuccess) {
        launch(warp_grid(b, n, 128), 128u, (const Q*)dq.p, (A*)da.p);
        e = launched(b);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, da.p, (size_t)n * sizeof(A), cudaMemcpyDeviceToHost, b->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->stream);
    if (e != cudaSuccess) { g_last_error = std::string(fn) + ": " + cudaGetErrorString(e); return PT_ERR_CUDA; }
    return PT_OK;
}

// The caller's pools of both JSON renders: checked on the host, then (for a batch with logs) copied into the handle's device
// buffers and described for the kernels in *P.
int load_json_pools(pt_batch* b, const pt_json_pools* pools, const char* fn, ptr::JsonPools* P) {
    struct Pool { const uint8_t* data; const uint64_t* off; uint64_t count; DevBuf* dd; DevBuf* doff; const char* name; };
    const Pool ps[3] = {{pools->values, pools->values_off, pools->n_values, &b->d_jval, &b->d_jvoff, "values"},
                        {pools->links, pools->links_off, pools->n_links, &b->d_jlink, &b->d_jloff, "links"},
                        {pools->comments, pools->comments_off, pools->n_comments, &b->d_jcom, &b->d_jcoff, "comments"}};
    for (const Pool& p : ps) {
        if (p.count && (!p.data || !p.off)) { g_last_error = std::string(fn) + ": null " + p.name + " pool with a nonzero count"; return PT_ERR_INVALID; }
        for (uint64_t k = 0; k < p.count; k++)
            if (p.off[k + 1] < p.off[k]) { g_last_error = std::string(fn) + ": " + p.name + " offsets decrease"; return PT_ERR_INVALID; }
    }
    PT_CUDA(cudaSetDevice(b->device));
    if (!b->n_logs) return PT_OK;
    const uint8_t** pdata[3] = {&P->val, &P->link, &P->com};
    const uint64_t** poff[3] = {&P->voff, &P->loff, &P->coff};
    uint64_t* pcount[3] = {&P->nval, &P->nlink, &P->ncom};
    int rc;
    for (int k = 0; k < 3; k++) {
        const Pool& p = ps[k];
        const uint64_t lo = p.count ? p.off[0] : 0, hi = p.count ? p.off[p.count] : 0;     // entries address data[lo, hi)
        if ((rc = reserve_n<uint8_t>(*p.dd, hi))) return rc;
        if (hi > lo) PT_CUDA(cudaMemcpyAsync((uint8_t*)p.dd->p + lo, p.data + lo, hi - lo, cudaMemcpyHostToDevice, b->stream));
        if ((rc = upload_n(b, *p.doff, p.off, p.count ? p.count + 1 : 0))) return rc;
        *pdata[k] = (const uint8_t*)p.dd->p; *poff[k] = (const uint64_t*)p.doff->p; *pcount[k] = p.count;
    }
    return PT_OK;
}

// Both renders after their pools are loaded: size pass (size(grid, threads, sizes, miss)), scan of the sizes through the
// download path's scan kernels, read-back of the total and the missing-entry key (one sync), an output of exactly that size,
// write pass (write(grid, threads, off, bytes)), copy back into J's pinned view.
template <class Size, class Write>
int render_passes(pt_batch* b, const char* fn, JsonBufs& J, Size size, Write write, pt_json_view* out) {
    int rc;
    const uint32_t n = b->n_logs;
    if ((rc = J.hoff.reserve(((size_t)n + 1) * 8)) || (rc = J.hbytes.reserve(1)) || (rc = J.hmisc.reserve(16))) return rc;
    uint64_t* hoff = (uint64_t*)J.hoff.p;
    if (!n) {
        hoff[0] = 0;
        *out = pt_json_view{0, hoff, (const char*)J.hbytes.p, 0};
        return PT_OK;
    }
    if ((rc = J.size.reserve((size_t)n * 8)) || (rc = J.off.reserve(((size_t)n + 1) * 8)) || (rc = J.miss.reserve(8))) return rc;
    unsigned long long *sizes = (unsigned long long*)J.size.p, *doff = (unsigned long long*)J.off.p, *miss = (unsigned long long*)J.miss.p;
    const uint32_t threads = 128, grid = warp_grid(b, n, threads);
    PT_CUDA(cudaMemsetAsync(miss, 0xFF, 8, b->stream));
    size(grid, threads, sizes, miss);
    PT_CUDA(launched(b));
    if ((rc = scan_offsets(b, pts::PlainCounts{sizes}, n, J.bsum, doff, nullptr))) return rc;
    uint64_t* hm = (uint64_t*)J.hmisc.p;
    PT_CUDA(cudaMemcpyAsync(hm, doff + n, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(hm + 1, miss, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t total = hm[0], key = hm[1];
    if (key != ~0ull) {
        static const char* kinds[3] = {"value", "link", "comment"};
        g_last_error = std::string(fn) + ": log " + std::to_string(key >> 34) + " names " + kinds[(key >> 32) & 3] + " pool entry " +
                       std::to_string(key & 0xFFFFFFFFull) + ", which the caller's pools do not hold";
        return PT_ERR_INVALID;
    }
    if ((rc = reserve_n<uint8_t>(J.bytes, total)) || (rc = reserve_n<uint8_t>(J.hbytes, total))) return rc;
    write(grid, threads, (const unsigned long long*)doff, (uint8_t*)J.bytes.p);
    PT_CUDA(launched(b));
    PT_CUDA(cudaMemcpyAsync(hoff, doff, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    if (total) PT_CUDA(cudaMemcpyAsync(J.hbytes.p, J.bytes.p, total, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    *out = pt_json_view{n, hoff, (const char*)J.hbytes.p, total};
    return PT_OK;
}

}  // namespace

extern "C" {

int pt_batch_create(int device, const pt_limits* limits, void* cuda_stream, pt_batch** out) {
    if (!out) return PT_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0 || device < 0 || device >= count) {
        g_last_error = e != cudaSuccess ? cudaGetErrorString(e) : "no such CUDA device (this engine has no CPU fallback)";
        return PT_ERR_NO_DEVICE;
    }
    PT_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    PT_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) { g_last_error = "device is not sm_90-class (kernels are built for sm_90a only)"; return PT_ERR_NO_DEVICE; }
    pt_batch* b = new pt_batch();
    b->device = device; b->stream = (cudaStream_t)cuda_stream; b->num_sms = prop.multiProcessorCount;
    if (limits) b->limits = *limits;
    if (b->limits.flags & PT_FLAG_EMIT_LARGE_PATCHES) b->limits.flags |= PT_FLAG_EMIT_PATCHES;
    if (b->limits.flags & PT_FLAG_EMIT_PATCHES) b->limits.flags |= PT_FLAG_EMIT_SEQUENCE;
    if (cudaEventCreate(&b->ev0) != cudaSuccess || cudaEventCreate(&b->ev1) != cudaSuccess) { delete b; g_last_error = "cudaEventCreate failed"; return PT_ERR_CUDA; }
    if (b->stream != nullptr) {          // fork / join needs a real stream (not the legacy default stream)
        if (cudaStreamCreateWithFlags(&b->side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&b->ev_join, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); b->side = nullptr; }
    }
    b->launch_stream = b->stream;
    *out = b;
    return PT_OK;
}

int pt_batch_upload(pt_batch* b, const pt_packed_ops* ops) {
    if (!b || !ops || (ops->n_logs && !ops->logs)) return PT_ERR_INVALID;
    int rc = begin_upload(b, *ops, true);
    if (rc) return rc;
    if (b->n_insdel) PT_CUDA(cudaMemcpyAsync(b->d_insdel.p, ops->insdel, b->n_insdel * sizeof(pt_insdel_rec), cudaMemcpyHostToDevice, b->stream));
    if (b->n_mark) PT_CUDA(cudaMemcpyAsync(b->d_marks.p, ops->marks, b->n_mark * sizeof(pt_mark_rec), cudaMemcpyHostToDevice, b->stream));
    return finish_upload(b, b->d_insdel.p, b->d_marks.p, {{ops->insdel, b->n_insdel}, {ops->marks, b->n_mark}});
}

// The run table as expand_runs_kernel reads it: each log's runs expand to exactly its descriptor's n_insdel records and
// consume exactly its slice of the token stream, so the expansion stays inside the log's records (make_plan checks the
// descriptors themselves).  Returns the problem, or null.
static const char* check_run_table(const pt_packed_runs& rr) {
    const uint32_t nl = rr.n_logs;
    if (!nl) return nullptr;
    if (rr.run_off[0] != 0 || rr.tok_off[0] != 0) return "run table: run_off[0] and tok_off[0] must be 0";
    for (uint32_t i = 0; i < nl; i++)
        if (rr.run_off[i + 1] < rr.run_off[i] || rr.tok_off[i + 1] < rr.tok_off[i]) return "run table: run_off / tok_off decrease";
    if ((rr.run_off[nl] && !rr.runs) || (rr.tok_off[nl] && !rr.tokens) || (rr.n_mark_total && !rr.marks)) return "run table: null array with a nonzero count";
    for (uint32_t i = 0; i < nl; i++) {
        uint64_t recs = 0, toks = 0;
        for (uint64_t r = rr.run_off[i]; r < rr.run_off[i + 1]; r++) {
            const uint32_t cnt = rr.runs[r].kind_count & 0x3FFFFFFFu, kind = rr.runs[r].kind_count >> 30;   // a 2-bit kind is always <= 3
            if (!cnt) return "run table: a run with count 0";
            recs += cnt;
            if (kind == PT_KIND_INSERT) toks += cnt;
        }
        if (recs != rr.logs[i].n_insdel) return "run table: a log's run counts do not sum to its n_insdel";
        if (toks != rr.tok_off[i + 1] - rr.tok_off[i]) return "run table: a log's insert runs do not match its token count";
    }
    return nullptr;
}

int pt_batch_upload_runs(pt_batch* b, const pt_packed_runs* rr) {
    if (!b || !rr || (rr->n_logs && (!rr->logs || !rr->run_off || !rr->tok_off))) return PT_ERR_INVALID;
    if (const char* err = check_run_table(*rr)) { g_last_error = err; return PT_ERR_INVALID; }
    int rc = begin_upload(b, pt_packed_ops{rr->n_logs, rr->logs, nullptr, rr->n_insdel_total, nullptr, rr->n_mark_total}, true);
    if (rc) return rc;
    const size_t nl = rr->n_logs;
    const uint64_t n_runs = nl ? rr->run_off[nl] : 0, n_tok = nl ? rr->tok_off[nl] : 0;
    if ((rc = upload_n(b, b->d_run_off, rr->run_off, nl ? nl + 1 : 0)) || (rc = upload_n(b, b->d_tok_off, rr->tok_off, nl ? nl + 1 : 0)) ||
        (rc = upload_n(b, b->d_runs, rr->runs, n_runs)) || (rc = upload_n(b, b->d_tokens, rr->tokens, n_tok))) return rc;
    if (b->n_mark) PT_CUDA(cudaMemcpyAsync(b->d_marks.p, rr->marks, b->n_mark * sizeof(pt_mark_rec), cudaMemcpyHostToDevice, b->stream));
    if (nl) {
        const uint32_t threads = 128;
        ptu::expand_runs_kernel<<<warp_grid(b, nl, threads), threads, 0, b->stream>>>(
            (const pt_log_desc*)b->d_desc.p, (const unsigned long long*)b->d_run_off.p, (const unsigned long long*)b->d_tok_off.p,
            (const pt_run_rec*)b->d_runs.p, (const uint32_t*)b->d_tokens.p, (pt_insdel_rec*)b->d_insdel.p, (uint32_t)nl);
        PT_CUDA(launched(b));
    }
    return finish_upload(b, b->d_insdel.p, b->d_marks.p, {{rr->runs, n_runs}, {rr->tokens, n_tok}, {rr->marks, b->n_mark}, {rr->run_off, nl}, {rr->tok_off, nl}});
}

int pt_compress_runs(const pt_packed_ops* ops, uint64_t* run_off, uint64_t* tok_off, pt_run_rec* runs, uint32_t* tokens,
                     uint64_t* n_runs_out, uint64_t* n_tokens_out) {
    if (!ops || !run_off || !tok_off) return PT_ERR_INVALID;
    uint64_t nr = 0, nt = 0;
    for (uint32_t li = 0; li < ops->n_logs; li++) {
        const pt_log_desc& L = ops->logs[li];
        const pt_insdel_rec* r = ops->insdel + L.insdel_off;
        run_off[li] = nr; tok_off[li] = nt;
        uint32_t i = 0;
        while (i < L.n_insdel) {
            const uint32_t kind = PT_PAYLOAD_KIND(r[i].payload);
            uint32_t j = i + 1;
            if (kind == PT_KIND_INSERT) {
                while (j < L.n_insdel && PT_PAYLOAD_KIND(r[j].payload) == PT_KIND_INSERT && r[j].actor == r[i].actor && r[j].ctr == r[j - 1].ctr + 1 &&
                       r[j].ref_ctr == r[j - 1].ctr && r[j].ref_actor == r[j - 1].actor && (j - i) < 0x3FFFFFFFu) j++;
            } else if (kind == PT_KIND_DELETE) {
                while (j < L.n_insdel && PT_PAYLOAD_KIND(r[j].payload) == PT_KIND_DELETE && r[j].actor == r[i].actor && r[j].ctr == r[j - 1].ctr + 1 &&
                       r[j].ref_ctr == r[j - 1].ref_ctr + 1 && r[j].ref_actor == r[i].ref_actor && (j - i) < 0x3FFFFFFFu) j++;
            }
            if (runs) { pt_run_rec q; q.ctr0 = r[i].ctr; q.ref_ctr = r[i].ref_ctr; q.actor = r[i].actor; q.ref_actor = r[i].ref_actor; q.kind_count = (kind << 30) | (j - i); runs[nr] = q; }
            if (kind == PT_KIND_INSERT) { if (tokens) for (uint32_t k = i; k < j; k++) tokens[nt + (k - i)] = PT_PAYLOAD_TOKEN(r[k].payload); nt += j - i; }
            nr++;
            i = j;
        }
    }
    run_off[ops->n_logs] = nr; tok_off[ops->n_logs] = nt;
    if (n_runs_out) *n_runs_out = nr;
    if (n_tokens_out) *n_tokens_out = nt;
    return PT_OK;
}
int pt_batch_adopt_device(pt_batch* b, const pt_packed_ops* ops) {
    if (!b || !ops || (ops->n_logs && !ops->logs)) return PT_ERR_INVALID;
    int rc = begin_upload(b, *ops, false);
    if (rc) return rc;
    return finish_upload(b, ops->insdel, ops->marks, {});
}

int pt_compact_ops(const pt_packed_ops* ops, pt_insdel_c8* io, pt_mark_c16* mo, int threads) {
    if (!ops || (ops->n_insdel_total && !io) || (ops->n_mark_total && !mo)) return PT_ERR_INVALID;
    for (uint32_t i = 0; i < ops->n_logs; i++) {
        const pt_log_desc& L = ops->logs[i];
        if (L.max_ctr >= 65536u || L.n_insdel >= 65536u || L.n_actors > 16u) { g_last_error = "log not representable in the compact wire format"; return PT_ERR_INVALID; }
    }
    // Every field is checked against its compact width: a record that names a counter or actor outside the log's bounds
    // (a faulty log) would otherwise be truncated into a valid-looking one and merge where the plain form reports it.
    static const char* const kField[] = {"value token", "insert/delete ctr", "insert/delete ref_ctr", "insert/delete actor",
                                          "insert/delete ref_actor", "mark ctr", "mark start_ctr", "mark end_ctr", "mark arrival",
                                          "mark actor", "mark start_actor", "mark end_actor", "mark kind", "mark bounds"};
    int T = threads > 0 ? threads : (int)std::max(1u, std::thread::hardware_concurrency());
    std::atomic<uint32_t> bad{0};      // bit f: some record's field kField[f] does not fit
    auto work = [&](int t) {
        // OR of every record's value per field: a field fits iff its OR does (widths are powers of two)
        uint32_t o_val = 0, o_ctr = 0, o_ref = 0, o_act = 0, o_ref_act = 0;
        const uint64_t n = ops->n_insdel_total, a = n * t / T, b2 = n * (t + 1) / T;
        for (uint64_t k = a; k < b2; k++) {
            const pt_insdel_rec& r = ops->insdel[k];
            const uint32_t tok = PT_PAYLOAD_TOKEN(r.payload), val = tok & (PT_TOKEN_POOLED - 1);
            o_val |= val; o_ctr |= r.ctr; o_ref |= r.ref_ctr; o_act |= r.actor; o_ref_act |= r.ref_actor;
            pt_insdel_c8 o; o.ctr = (uint16_t)r.ctr; o.ref_ctr = (uint16_t)r.ref_ctr;
            o.w = (r.actor & 0xFu) | ((r.ref_actor & 0xFu) << 4) | (PT_PAYLOAD_KIND(r.payload) << 8) | (((tok & PT_TOKEN_POOLED ? 0x200000u : 0u) | (val & 0x1FFFFFu)) << 10);
            io[k] = o;
        }
        uint32_t m_ctr = 0, m_start = 0, m_end = 0, m_arr = 0, m_act = 0, m_sact = 0, m_eact = 0, m_kind = 0, m_bounds = 0;
        const uint64_t m = ops->n_mark_total, c = m * t / T, d = m * (t + 1) / T;
        for (uint64_t k = c; k < d; k++) {
            const pt_mark_rec& r = ops->marks[k];
            m_ctr |= r.ctr; m_start |= r.start_ctr; m_end |= r.end_ctr; m_arr |= r.arrival;
            m_act |= r.actor; m_sact |= r.start_actor; m_eact |= r.end_actor; m_kind |= r.kind; m_bounds |= r.bounds;
            pt_mark_c16 o; o.ctr = (uint16_t)r.ctr; o.start_ctr = (uint16_t)r.start_ctr; o.end_ctr = (uint16_t)r.end_ctr; o.arrival = (uint16_t)r.arrival; o.attr = r.attr;
            o.w = (r.actor & 0xFu) | ((r.start_actor & 0xFu) << 4) | ((r.end_actor & 0xFu) << 8) | ((r.kind & 7u) << 12) | ((r.bounds & 0xFu) << 15);
            mo[k] = o;
        }
        const uint32_t mask = (o_val >= 0x200000u) | (o_ctr >= 65536u) << 1 | (o_ref >= 65536u) << 2 | (o_act >= 16u) << 3 | (o_ref_act >= 16u) << 4 |
                              (m_ctr >= 65536u) << 5 | (m_start >= 65536u) << 6 | (m_end >= 65536u) << 7 | (m_arr >= 65536u) << 8 |
                              (m_act >= 16u) << 9 | (m_sact >= 16u) << 10 | (m_eact >= 16u) << 11 | (m_kind >= 8u) << 12 | (m_bounds >= 16u) << 13;
        if (mask) bad.fetch_or(mask);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    if (const uint32_t m = bad.load()) {
        std::string names;
        for (uint32_t f = 0; f < sizeof(kField) / sizeof(kField[0]); f++)
            if (m >> f & 1u) names += (names.empty() ? "" : ", ") + std::string(kField[f]);
        g_last_error = "not representable in the compact wire format: " + names;
        return PT_ERR_INVALID;
    }
    return PT_OK;
}

int pt_batch_upload_compact(pt_batch* b, const pt_packed_compact* cc) {
    if (!b || !cc || (cc->n_logs && !cc->logs)) return PT_ERR_INVALID;
    int rc = begin_upload(b, pt_packed_ops{cc->n_logs, cc->logs, nullptr, cc->n_insdel_total, nullptr, cc->n_mark_total}, true);
    if (rc) return rc;
    const uint32_t threads = 256;      // one thread per record
    if ((rc = upload_n(b, b->d_cins, cc->insdel, b->n_insdel))) return rc;
    if (b->n_insdel) {
        ptu::expand_insdel_c8_kernel<<<warp_grid(b, b->n_insdel, threads, 1), threads, 0, b->stream>>>(
            (const pt_insdel_c8*)b->d_cins.p, (pt_insdel_rec*)b->d_insdel.p, b->n_insdel);
        PT_CUDA(launched(b));
    }
    if ((rc = upload_n(b, b->d_cmarks, cc->marks, b->n_mark))) return rc;
    if (b->n_mark) {
        ptu::expand_mark_c16_kernel<<<warp_grid(b, b->n_mark, threads, 1), threads, 0, b->stream>>>(
            (const pt_mark_c16*)b->d_cmarks.p, (pt_mark_rec*)b->d_marks.p, b->n_mark);
        PT_CUDA(launched(b));
    }
    return finish_upload(b, b->d_insdel.p, b->d_marks.p, {{cc->insdel, b->n_insdel}, {cc->marks, b->n_mark}});
}

int pt_batch_upload_changes(pt_batch* b, const pt_change_table* t) {
    if (!b || !t) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_upload_changes before pt_batch_upload"; return PT_ERR_STATE; }
    if (t->n_logs != b->n_logs || (t->n_logs && !t->logs)) { g_last_error = "change table does not match the batch"; return PT_ERR_INVALID; }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    uint32_t maxR = 1;
    for (uint32_t i = 0; i < b->n_logs; i++) {
        const pt_change_desc& D = t->logs[i];
        if (D.change_off + D.n_changes > t->n_changes_total || D.dep_off + D.n_deps > t->n_deps_total) { g_last_error = "change descriptor out of range"; return PT_ERR_INVALID; }
        maxR = std::max<uint32_t>(maxR, b->h_desc[i].n_actors);
    }
    if (actor_table_bytes(maxR) > kAdmitMaxBytes) { g_last_error = "more than 25600 actors in one log: not supported by the admission pre-pass"; return PT_ERR_INVALID; }
    int rc;
    const size_t n = b->n_logs;
    if ((rc = upload_n(b, b->d_cdesc, t->logs, n)) || (rc = upload_n(b, b->d_changes, t->changes, t->n_changes_total)) ||
        (rc = upload_n(b, b->d_deps, t->deps, t->n_deps_total)) || (rc = reserve_n<uint32_t>(b->d_admit, n))) return rc;
    PT_CUDA(cudaStreamSynchronize(b->stream));            // the caller's arrays may be freed on return
    b->h_cdesc.assign(t->logs, t->logs + n); b->n_changes = t->n_changes_total; b->n_deps = t->n_deps_total;
    b->adm_maxR = maxR; b->have_changes = true;
    drop_graph(b);                                       // the launch sequence changes
    return PT_OK;
}

static std::string at(uint32_t log) { return "log " + std::to_string(log) + ": "; }   // an error's prefix

// A counter map c[0, nc): entry 0 (HEAD) maps to 0 and the mapped entries (all but 0xFFFFFFFF) strictly increase.  Returns
// the problem, or null; bound gets the image of the last mapped entry at or below `upto`.
static const char* check_ctr_map(const uint32_t* c, uint64_t nc, uint64_t upto, uint32_t& bound) {
    if (nc && c[0] != 0) return "ctr_map[0] is not 0";
    uint32_t last = 0;
    bound = 0;
    for (uint64_t k = 1; k < nc; k++) {
        if (c[k] == 0xFFFFFFFFu) continue;
        if (c[k] <= last) return "the counter map is not strictly increasing";
        last = c[k];
        if (k <= upto) bound = c[k];
    }
    return nullptr;
}

// Host checks of a delta and its remap against the resident batch (include/peritext_b200.h, pt_batch_append); on success
// nd / ncd hold the descriptors of the concatenated batch and its change table.  Returns the problem, or an empty string.
static std::string check_append(const pt_batch* b, const pt_packed_ops& delta, bool delta_on_device, const pt_append_remap& R, const pt_change_table* dch,
                                std::vector<pt_log_desc>& nd, std::vector<pt_change_desc>& ncd, uint32_t& maxR) {
    const uint32_t n = b->n_logs;
    if (delta.n_logs != n) return "the delta has " + std::to_string(delta.n_logs) + " logs and the batch " + std::to_string(n);
    if ((dch != nullptr) != b->have_changes)
        return b->have_changes ? "the batch has a change table and the delta none" : "the delta has a change table and the batch none";
    if ((delta.n_insdel_total && !delta.insdel) || (delta.n_mark_total && !delta.marks)) return "null delta records with a nonzero count";
    if ((R.actor_off && R.actor_off[n] > R.actor_off[0] && !R.actor_map) || (R.ctr_off && R.ctr_off[n] > R.ctr_off[0] && !R.ctr_map) ||
        (R.n_comment_map && !R.comment_map)) return "null map with a nonzero length";
    for (uint64_t k = 1; R.comment_map && k < R.n_comment_map; k++)
        if (R.comment_map[k] <= R.comment_map[k - 1]) return "comment_map is not strictly increasing";
    nd.resize(n);
    uint64_t io = 0, mo = 0;
    maxR = 1;
    for (uint32_t i = 0; i < n; i++) {
        const pt_log_desc &O = b->h_desc[i], &D = delta.logs[i];
        if (D.insdel_off + D.n_insdel > delta.n_insdel_total || D.mark_off + D.n_mark > delta.n_mark_total) return at(i) + "delta descriptor out of range";
        if ((uint64_t)O.n_insdel + D.n_insdel > 0xFFFFFFFFull || (uint64_t)O.n_mark + D.n_mark > 0xFFFFFFFFull) return at(i) + "more than 2^32 - 1 records";
        const uint64_t na = R.actor_off ? R.actor_off[i + 1] - R.actor_off[i] : 0, nc = R.ctr_off ? R.ctr_off[i + 1] - R.ctr_off[i] : 0;
        if (R.actor_off && R.actor_off[i + 1] < R.actor_off[i]) return "actor_off decreases";
        if (R.ctr_off && R.ctr_off[i + 1] < R.ctr_off[i]) return "ctr_off decreases";
        if (na) {
            const uint16_t* a = R.actor_map + R.actor_off[i];
            if (na != O.n_actors) return at(i) + "the actor map has " + std::to_string(na) + " entries and the log had " + std::to_string(O.n_actors) + " actors";
            for (uint64_t k = 1; k < na; k++) if (a[k] <= a[k - 1]) return at(i) + "the actor map is not strictly increasing";
            if (a[na - 1] >= D.n_actors) return at(i) + "the actor map names a rank >= the new n_actors";
        } else if (O.n_actors > D.n_actors) {
            return at(i) + "the new n_actors is below the old (identity actor map)";
        }
        if (nc) {
            if (nc <= (uint64_t)O.max_ctr) return at(i) + "the counter map has " + std::to_string(nc) + " entries and the log's old max_ctr is " + std::to_string(O.max_ctr);
            uint32_t bound;                       // the image of the old max_ctr
            if (const char* e = check_ctr_map(R.ctr_map + R.ctr_off[i], nc, O.max_ctr, bound)) return at(i) + e;
            if (bound > D.max_ctr) return at(i) + "the counter map sends the old max_ctr past the new max_ctr";
        } else if (O.max_ctr > D.max_ctr) {
            return at(i) + "the new max_ctr is below the old (identity counter map)";
        }
        for (uint32_t k = 0; !delta_on_device && k < D.n_mark; k++) {     // device records (pt_batch_change) carry their arrival by construction
            const uint32_t a = delta.marks[D.mark_off + k].arrival;
            if (a < O.n_insdel || a > (uint64_t)O.n_insdel + D.n_insdel) return at(i) + "delta mark " + std::to_string(k) + " has arrival " + std::to_string(a) +
                                                                                 " outside [" + std::to_string(O.n_insdel) + ", " + std::to_string((uint64_t)O.n_insdel + D.n_insdel) + "]";
        }
        nd[i] = pt_log_desc{io, mo, O.n_insdel + D.n_insdel, O.n_mark + D.n_mark, D.n_actors, D.max_ctr};
        io += nd[i].n_insdel; mo += nd[i].n_mark;
        maxR = std::max<uint32_t>(maxR, D.n_actors);
    }
    if (dch) {
        if (dch->n_logs != n || (n && !dch->logs)) return "the delta's change table does not match the batch";
        if ((dch->n_changes_total && !dch->changes) || (dch->n_deps_total && !dch->deps)) return "null delta change records with a nonzero count";
        if (actor_table_bytes(maxR) > kAdmitMaxBytes) return "more than 25600 actors in one log: not supported by the admission pre-pass";
        ncd.resize(n);
        uint64_t co = 0, po = 0;
        for (uint32_t i = 0; i < n; i++) {
            const pt_change_desc &O = b->h_cdesc[i], &D = dch->logs[i];
            if (D.change_off + D.n_changes > dch->n_changes_total || D.dep_off + D.n_deps > dch->n_deps_total) return at(i) + "delta change descriptor out of range";
            if ((uint64_t)O.n_changes + D.n_changes > 0xFFFFFFFFull || (uint64_t)O.n_deps + D.n_deps > 0xFFFFFFFFull) return at(i) + "more than 2^32 - 1 changes or deps";
            ncd[i] = pt_change_desc{co, po, O.n_changes + D.n_changes, O.n_deps + D.n_deps};
            co += ncd[i].n_changes; po += ncd[i].n_deps;
        }
    }
    return std::string();
}

// The splice of pt_batch_append and pt_batch_select_logs once their host checks pass: new log i (nd[i], ncd[i]) is the resident
// log from[i] (from == nullptr: log i; PT_SELECT_ADDED: none) with its ids through R's maps, followed by delta log i's records,
// and likewise for the change table.  `delta`'s records are host memory, or device memory the caller keeps alive
// (delta_on_device); so are the change and dep records of `dch` (table_on_device).  The delta's descriptors, the remap, `from`
// and the change table's descriptors are host memory.  keep_actors: the actor tables still describe the new logs.
static int splice(pt_batch* b, const char* fn, std::vector<pt_log_desc>&& nd, std::vector<pt_change_desc>&& ncd, uint32_t maxR,
                  const pt_packed_ops* delta, bool delta_on_device, const pt_append_remap& R, const uint32_t* from,
                  const pt_change_table* dch, bool table_on_device, bool keep_actors) {
    const uint32_t n = (uint32_t)nd.size();
    const uint64_t n_ins = n ? nd[n - 1].insdel_off + nd[n - 1].n_insdel : 0, n_mk = n ? nd[n - 1].mark_off + nd[n - 1].n_mark : 0;
    const pt_packed_ops ops{n, nd.data(), nullptr, n_ins, nullptr, n_mk};
    ptp::Plan plan;
    if (const char* e = ptp::make_plan(ops, b->limits, b->num_sms, plan)) { g_last_error = std::string(fn) + e; return PT_ERR_INVALID; }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // the merge and downloads of the resident batch are done
    // The delta and the remap go to the device; the splice writes NEW buffers, so the resident batch stays intact until the
    // device has accepted every record.
    int rc;
    DevBuf ndesc, nins, nmarks, ncdesc, nch, ndp;              // the new batch's descriptors, records and change table
    DevBuf ddesc, dins, dmarks, dcdesc, dchg, ddep, amap[5], abad, dfrom;   // the delta, its remap, the index, the refusal flag: freed on return
    if ((rc = upload_n(b, ddesc, delta->logs, n)) || (rc = upload_n(b, ndesc, nd.data(), n)) || (rc = abad.reserve(4)) ||
        (rc = reserve_n<pt_insdel_rec>(nins, n_ins)) || (rc = reserve_n<pt_mark_rec>(nmarks, n_mk))) return rc;
    if (from && (rc = upload_n(b, dfrom, from, n))) return rc;
    const uint32_t* d_from = from ? (const uint32_t*)dfrom.p : nullptr;
    const pt_insdel_rec* d_dins = delta->insdel;
    const pt_mark_rec* d_dmarks = delta->marks;
    if (!delta_on_device) {
        if ((rc = upload_n(b, dins, delta->insdel, delta->n_insdel_total)) || (rc = upload_n(b, dmarks, delta->marks, delta->n_mark_total))) return rc;
        d_dins = (const pt_insdel_rec*)dins.p; d_dmarks = (const pt_mark_rec*)dmarks.p;
    }
    pta::Remap DR{};
    const void* hsrc[5] = {R.actor_off, R.actor_map, R.ctr_off, R.ctr_map, R.comment_map};
    const size_t hbytes[5] = {R.actor_off ? ((size_t)n + 1) * 8 : 0, R.actor_off ? (size_t)R.actor_off[n] * 2 : 0,
                              R.ctr_off ? ((size_t)n + 1) * 8 : 0, R.ctr_off ? (size_t)R.ctr_off[n] * 4 : 0, R.comment_map ? (size_t)R.n_comment_map * 4 : 0};
    const void* dptr[5] = {};
    for (int k = 0; k < 5; k++) {
        if (!hsrc[k]) continue;
        if ((rc = amap[k].reserve(std::max<size_t>(16, hbytes[k])))) return rc;
        if (hbytes[k]) PT_CUDA(cudaMemcpyAsync(amap[k].p, hsrc[k], hbytes[k], cudaMemcpyHostToDevice, b->stream));
        dptr[k] = amap[k].p;
    }
    DR.actor_off = (const unsigned long long*)dptr[0]; DR.actor_map = (const uint16_t*)dptr[1];
    DR.ctr_off = (const unsigned long long*)dptr[2]; DR.ctr_map = (const uint32_t*)dptr[3];
    DR.comment_map = (const uint32_t*)dptr[4]; DR.n_comment = R.comment_map ? R.n_comment_map : 0;
    PT_CUDA(cudaMemsetAsync(abad.p, 0, 4, b->stream));
    const uint32_t threads = 128;
    if (n) {
        uint64_t most = 0;
        for (uint32_t i = 0; i < n; i++) most = std::max<uint64_t>(most, (uint64_t)nd[i].n_insdel + 2ull * nd[i].n_mark);
        pta::splice_records_kernel<<<slice_grid(b, n, most, threads), threads, 0, b->stream>>>(
            (const pt_log_desc*)b->d_desc.p, (const pt_log_desc*)ndesc.p, (const pt_log_desc*)ddesc.p, d_from, n, DR, b->dp_insdel, b->dp_marks,
            d_dins, d_dmarks, (pt_insdel_rec*)nins.p, (pt_mark_rec*)nmarks.p, (uint32_t*)abad.p);
        PT_CUDA(launched(b));
    }
    uint64_t n_ch = 0, n_dp = 0;
    if (dch) {
        n_ch = n ? ncd[n - 1].change_off + ncd[n - 1].n_changes : 0; n_dp = n ? ncd[n - 1].dep_off + ncd[n - 1].n_deps : 0;
        if ((rc = upload_n(b, dcdesc, dch->logs, n)) || (rc = upload_n(b, ncdesc, ncd.data(), n)) ||
            (rc = reserve_n<pt_change_rec>(nch, n_ch)) || (rc = reserve_n<pt_dep_rec>(ndp, n_dp))) return rc;
        const pt_change_rec* d_dchg = dch->changes;
        const pt_dep_rec* d_ddep = dch->deps;
        if (!table_on_device) {
            if ((rc = upload_n(b, dchg, dch->changes, dch->n_changes_total)) || (rc = upload_n(b, ddep, dch->deps, dch->n_deps_total))) return rc;
            d_dchg = (const pt_change_rec*)dchg.p; d_ddep = (const pt_dep_rec*)ddep.p;
        }
        if (n) {
            pta::splice_changes_kernel<<<warp_grid(b, n, threads), threads, 0, b->stream>>>(
                (const pt_change_desc*)b->d_cdesc.p, (const pt_change_desc*)ncdesc.p, (const pt_change_desc*)dcdesc.p, d_from, n, DR,
                (const pt_change_rec*)b->d_changes.p, (const pt_dep_rec*)b->d_deps.p, d_dchg, d_ddep, (pt_change_rec*)nch.p, (pt_dep_rec*)ndp.p);
            PT_CUDA(launched(b));
        }
        if ((rc = reserve_n<uint32_t>(b->d_admit, n))) return rc;
    }
    uint32_t bad = 0;
    PT_CUDA(cudaMemcpyAsync(&bad, abad.p, 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // also: the caller's arrays may be freed on return
    if (bad) { g_last_error = std::string(fn) + "a resident comment rank is outside comment_map or maps to 0xFFFFFFFF"; return PT_ERR_INVALID; }
    // Accepted: the new records and change table replace the old ones (freed with the locals), and the batch is re-planned.
    b->have_actors = b->have_actors && keep_actors;
    b->have_batch = false; b->merged = false; b->dl_begun = false;
    drop_graph(b);
    b->d_insdel.swap(nins); b->d_marks.swap(nmarks);
    if (dch) {
        b->d_cdesc.swap(ncdesc); b->d_changes.swap(nch); b->d_deps.swap(ndp);
        b->h_cdesc = std::move(ncd); b->n_changes = n_ch; b->n_deps = n_dp; b->adm_maxR = maxR;
    }
    if ((rc = install_plan(b, ops, std::move(plan), true))) return rc;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->dp_insdel = (const pt_insdel_rec*)b->d_insdel.p; b->dp_marks = (const pt_mark_rec*)b->d_marks.p;
    if ((rc = derive_key_records(b))) return rc;
    b->have_batch = true;
    return PT_OK;
}

// pt_batch_append after its host checks, and the append of pt_batch_change and pt_batch_exchange (`fn` prefixes the error text).
static int splice_append(pt_batch* b, const char* fn, const pt_packed_ops* delta, bool delta_on_device, const pt_append_remap& R,
                         const pt_change_table* dch, bool table_on_device) {
    std::vector<pt_log_desc> nd;
    std::vector<pt_change_desc> ncd;
    uint32_t maxR = 1;
    const std::string err = check_append(b, *delta, delta_on_device, R, dch, nd, ncd, maxR);
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    // The actor tables stay only while no log's actor set can have changed: no actor or counter map, every n_actors kept.
    const uint32_t n = b->n_logs;
    bool keep_actors = !(R.actor_off && R.actor_off[n] > R.actor_off[0]) && !(R.ctr_off && R.ctr_off[n] > R.ctr_off[0]);
    for (uint32_t i = 0; keep_actors && i < n; i++) keep_actors = nd[i].n_actors == b->h_desc[i].n_actors;
    return splice(b, fn, std::move(nd), std::move(ncd), maxR, delta, delta_on_device, R, nullptr, dch, table_on_device, keep_actors);
}

int pt_batch_append(pt_batch* b, const pt_packed_ops* delta, const pt_append_remap* remap, const pt_change_table* dch) {
    if (!b || !delta || (delta->n_logs && !delta->logs)) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_append before pt_batch_upload"; return PT_ERR_STATE; }
    return splice_append(b, "pt_batch_append: ", delta, false, remap ? *remap : pt_append_remap{}, dch, false);
}

// pt_batch_change's host checks of the InputOperations (include/peritext_b200.h).  On success dd holds the delta layout for
// every log succeeding (records in log order, the new max_ctr), new_elems each log's insert values and work the logs with a
// change.  Returns the problem, or an empty string.
static std::string check_change(const pt_batch* b, const pt_change_input& in, std::vector<pt_log_desc>& dd, std::vector<uint32_t>& new_elems,
                                std::vector<uint32_t>& work) {
    const uint32_t n = b->n_logs;
    if (in.n_logs != n) return "the input has " + std::to_string(in.n_logs) + " logs and the batch " + std::to_string(n);
    if (!n) return std::string();
    if (!in.actor || !in.input_off) return "null actor or input_off";
    if (in.input_off[0] != 0) return "input_off[0] is not 0";
    if ((in.input_off[n] && !in.ops) || (in.n_tokens && !in.tokens)) return "null ops or tokens with a nonzero count";
    dd.resize(n); new_elems.assign(n, 0);
    uint64_t io = 0, mo = 0;
    for (uint32_t i = 0; i < n; i++) {
        const pt_log_desc& L = b->h_desc[i];
        const uint64_t lo = in.input_off[i], hi = in.input_off[i + 1];
        if (hi < lo) return "input_off decreases at log " + std::to_string(i);
        dd[i] = pt_log_desc{io, mo, 0, 0, L.n_actors, L.max_ctr};
        const uint32_t A = in.actor[i];
        if (A == PT_CHANGE_NO_ACTOR) {
            if (hi > lo) return at(i) + "InputOperations without an actor";
            continue;
        }
        if (A >= L.n_actors) return at(i) + "actor rank " + std::to_string(A) + " >= the log's " + std::to_string(L.n_actors) + " actors";
        uint64_t next = (uint64_t)L.max_ctr + 1, last = L.max_ctr, nid = 0, nmk = 0, nel = 0;
        for (uint64_t k = lo; k < hi; k++) {
            const pt_input_op& op = in.ops[k];
            const std::string here = at(i) + "InputOperation " + std::to_string(k - lo) + ": ";
            uint64_t gen = 0;
            if (op.action == PT_INPUT_INSERT) {
                if (op.arg < 0) return here + "a negative number of values";
                gen = (uint64_t)op.arg;
                if (op.tok_off > in.n_tokens || gen > in.n_tokens - op.tok_off) return here + "tokens out of range";
                for (uint64_t j = 0; j < gen; j++) {
                    const uint32_t t = in.tokens[op.tok_off + j];
                    const bool ok = (t & PT_TOKEN_POOLED) ? (t >> 30) == 0 && (t & (PT_TOKEN_POOLED - 1)) < in.n_values : t <= 0x10FFFFu;
                    if (!ok) return here + "token " + std::to_string(j) + " (" + std::to_string(t) + ") out of range";
                }
                nid += gen; nel += gen;
            } else if (op.action == PT_INPUT_DELETE) {
                gen = op.arg > 0 ? (uint64_t)op.arg : 0;
                nid += gen;
            } else if (op.action == PT_INPUT_ADD_MARK || op.action == PT_INPUT_REMOVE_MARK) {
                if (op.mark_type > PT_MARK_LINK) return here + "unknown mark type " + std::to_string(op.mark_type);
                const bool ok = op.mark_type == PT_MARK_LINK ? op.attr < in.n_links : op.mark_type == PT_MARK_COMMENT ? op.attr < in.n_comments : op.attr == PT_ATTR_NONE;
                if (!ok) return here + "attr " + std::to_string(op.attr) + " out of range";
                gen = 1; nmk++;
            } else {
                return here + "unknown action " + std::to_string(op.action);
            }
            if (op.first_ctr < next)
                return here + "first_ctr " + std::to_string(op.first_ctr) + " is below " + std::to_string(next) + " (the log's max_ctr + 1, or the previous InputOperation's next counter)";
            if (op.first_ctr + gen - (gen ? 1 : 0) > 0xFFFFFFFFull) return here + "counters past 2^32 - 1";
            next = op.first_ctr + gen;
            if (gen) last = op.first_ctr + gen - 1;
        }
        if (last * std::max<uint32_t>(1, L.n_actors) > 0x7FFFFFFFull) return at(i) + "max_ctr x n_actors would reach 2^31";
        if (L.n_insdel + nid > 0xFFFFFFFFull || L.n_mark + nmk > 0xFFFFFFFFull) return at(i) + "more than 2^32 - 1 records";
        dd[i].n_insdel = (uint32_t)nid; dd[i].n_mark = (uint32_t)nmk; dd[i].max_ctr = (uint32_t)last;
        new_elems[i] = (uint32_t)std::min<uint64_t>(nel, 0xFFFFFFFFu);
        work.push_back(i);
        io += nid; mo += nmk;
    }
    return std::string();
}

int pt_batch_change(pt_batch* b, const pt_change_input* in, const pt_change_table* changes, pt_change_view* out) {
    if (!b || !in || !out) return PT_ERR_INVALID;
    if (!b->have_batch || !b->merged) { g_last_error = "pt_batch_change: no completed merge since the last upload, append or change"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = "pt_batch_change: the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    const uint32_t n = b->n_logs;
    std::string err;
    if ((changes != nullptr) != b->have_changes)
        err = b->have_changes ? "the batch has a change table and the change none" : "the change has a change table and the batch none";
    else if (changes && (changes->n_logs != n || (n && !changes->logs)))
        err = "the change table does not match the batch";
    std::vector<pt_log_desc> dd;
    std::vector<uint32_t> new_elems, work;
    if (err.empty()) err = check_change(b, *in, dd, new_elems, work);
    if (!err.empty()) { g_last_error = "pt_batch_change: " + err; return PT_ERR_INVALID; }
    const uint64_t n_ins = n ? dd[n - 1].insdel_off + dd[n - 1].n_insdel : 0, n_mk = n ? dd[n - 1].mark_off + dd[n - 1].n_mark : 0;
    std::vector<unsigned long long> soff(n, 0);
    uint64_t n_scratch = 0;
    for (uint32_t i : work) {                          // a slot holds the log's elements and its new ones, 16-byte aligned
        soff[i] = n_scratch;
        n_scratch += ((uint64_t)b->h_desc[i].n_insdel + new_elems[i] + 3) & ~3ull;
    }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // the merge is complete
    int rc;
    DevBuf dwork, dactor, dioff, dops, dtok, ddelta, dnel, dsoff, dscr, dst, dgi, dgm;   // freed on return
    const uint64_t n_ops = n ? in->input_off[n] : 0;
    if ((rc = upload_n(b, dwork, work.data(), work.size())) || (rc = upload_n(b, dactor, in->actor, n)) ||
        (rc = upload_n(b, dioff, in->input_off, n ? n + 1 : 0)) || (rc = upload_n(b, ddelta, dd.data(), n)) ||
        (rc = upload_n(b, dnel, new_elems.data(), n)) || (rc = upload_n(b, dsoff, soff.data(), n)) || (rc = reserve_n<pt_change_status>(dst, n)))
        return rc;
    if (n) PT_CUDA(cudaMemsetAsync(dst.p, 0, (size_t)n * sizeof(pt_change_status), b->stream));   // logs without a change: OK
    if ((rc = upload_n(b, dops, in->ops, n_ops)) || (rc = upload_n(b, dtok, in->tokens, in->n_tokens)) ||
        (rc = dscr.reserve(std::max<uint64_t>(4, n_scratch) * 4)) || (rc = reserve_n<pt_insdel_rec>(dgi, n_ins)) || (rc = reserve_n<pt_mark_rec>(dgm, n_mk)))
        return rc;
    if (!work.empty()) {
        ptc::ChangeParams P{};
        P.work = (const uint32_t*)dwork.p; P.n_work = (uint32_t)work.size();
        P.desc = (const pt_log_desc*)b->d_desc.p; P.insdel = b->dp_insdel; P.results = (const pt_log_result*)b->d_results.p;
        P.seq_off = (const uint64_t*)b->d_text_off.p; P.seq = (const uint32_t*)b->d_seq.p;
        P.actor = (const uint32_t*)dactor.p; P.input_off = (const unsigned long long*)dioff.p; P.ops = (const pt_input_op*)dops.p;
        P.tokens = (const uint32_t*)dtok.p; P.delta = (const pt_log_desc*)ddelta.p; P.new_elems = (const uint32_t*)dnel.p;
        P.scratch_off = (const unsigned long long*)dsoff.p; P.scratch = (uint32_t*)dscr.p;
        P.out_insdel = (pt_insdel_rec*)dgi.p; P.out_marks = (pt_mark_rec*)dgm.p; P.status = (pt_change_status*)dst.p;
        ptc::change_resolve_kernel<<<warp_grid(b, work.size(), 128), 128, 0, b->stream>>>(P);
        PT_CUDA(launched(b));
    }
    // the status of every log (the logs without a change are OK) and the generated records, into the view's pinned buffers
    if ((rc = reserve_n<pt_change_status>(b->h_chg_status, n)) || (rc = reserve_n<pt_log_desc>(b->h_chg_desc, n)) ||
        (rc = reserve_n<pt_insdel_rec>(b->h_chg_insdel, n_ins)) || (rc = reserve_n<pt_mark_rec>(b->h_chg_marks, n_mk)))
        return rc;
    pt_change_status* st = (pt_change_status*)b->h_chg_status.p;
    if (n) PT_CUDA(cudaMemcpyAsync(st, dst.p, (size_t)n * sizeof(pt_change_status), cudaMemcpyDeviceToHost, b->stream));
    if (n_ins) PT_CUDA(cudaMemcpyAsync(b->h_chg_insdel.p, dgi.p, n_ins * sizeof(pt_insdel_rec), cudaMemcpyDeviceToHost, b->stream));
    if (n_mk) PT_CUDA(cudaMemcpyAsync(b->h_chg_marks.p, dgm.p, n_mk * sizeof(pt_mark_rec), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    for (uint32_t i = 0; i < n; i++) if (st[i].status == PT_CHANGE_OK) st[i].input = 0xFFFFFFFFu;
    for (uint32_t i : work)
        if (st[i].status == ptc::kRefuseMergeStatus || st[i].status == ptc::kRefuseElements) {
            g_last_error = "pt_batch_change: log " + std::to_string(i) + (st[i].status == ptc::kRefuseMergeStatus ? ": its merge status is not PT_LOG_OK"
                                                                                                                  : ": the change would bring it to 2^22 elements or more");
            return PT_ERR_INVALID;
        }
    // a log whose change failed appends nothing: no records, its old max_ctr, no change record
    std::vector<pt_change_desc> cdesc;
    pt_change_table ct{};
    if (changes) { cdesc.assign(changes->logs, changes->logs + n); ct = *changes; ct.logs = cdesc.data(); }
    for (uint32_t i : work)
        if (st[i].status != PT_CHANGE_OK) {
            dd[i].n_insdel = 0; dd[i].n_mark = 0; dd[i].max_ctr = b->h_desc[i].max_ctr;
            if (changes) { cdesc[i].n_changes = 0; cdesc[i].n_deps = 0; }
        }
    memcpy(b->h_chg_desc.p, dd.data(), (size_t)n * sizeof(pt_log_desc));
    const pt_packed_ops delta{n, dd.data(), (const pt_insdel_rec*)dgi.p, n_ins, (const pt_mark_rec*)dgm.p, n_mk};
    if ((rc = splice_append(b, "pt_batch_change: ", &delta, true, pt_append_remap{}, changes ? &ct : nullptr, false))) return rc;
    out->n_logs = n;
    out->status = st;
    out->delta = pt_packed_ops{n, (const pt_log_desc*)b->h_chg_desc.p, (const pt_insdel_rec*)b->h_chg_insdel.p, n_ins, (const pt_mark_rec*)b->h_chg_marks.p, n_mk};
    return PT_OK;
}

// pt_batch_exchange's host checks of the pairs and their maps (include/peritext_b200.h).  On success slot_off holds each
// pair's scratch slot (exclusive scan of its src's n_changes).  Returns the problem, or an empty string.
static std::string pair_at(uint32_t p) { return "pair " + std::to_string(p) + ": "; }   // an error's prefix

// The rules every pair of pt_batch_exchange and pt_batch_sync_pairs follows: both logs in the batch, src != dst, no dst named
// twice (is_dst: the dsts of the earlier pairs).  Returns the problem, or an empty string.
static std::string check_pair(const pt_batch* b, uint32_t p, pt_exchange_pair pr, std::vector<char>& is_dst) {
    const uint32_t n = b->n_logs, src = pr.src, dst = pr.dst;
    if (src >= n || dst >= n) return pair_at(p) + "log " + std::to_string(src >= n ? src : dst) + " is outside the batch's " + std::to_string(n) + " logs";
    if (src == dst) return pair_at(p) + "src and dst are both log " + std::to_string(src);
    if (is_dst[dst]) return pair_at(p) + "log " + std::to_string(dst) + " is the dst of an earlier pair";
    is_dst[dst] = 1;
    return std::string();
}

static std::string check_exchange(const pt_batch* b, const pt_exchange_input& in, std::vector<unsigned long long>& slot_off) {
    const uint32_t n = b->n_logs, np = in.n_pairs;
    auto at = pair_at;
    if (!in.pairs || !in.actor_off) return "null pairs or actor_off";
    if (in.actor_off[np] > in.actor_off[0] && !in.actor_map) return "null actor_map with a nonzero length";
    if (in.ctr_off && in.ctr_off[np] > in.ctr_off[0] && !in.ctr_map) return "null ctr_map with a nonzero length";
    std::vector<char> is_dst(n, 0);
    slot_off.assign((size_t)np + 1, 0);
    for (uint32_t p = 0; p < np; p++) {
        const uint32_t src = in.pairs[p].src, dst = in.pairs[p].dst;
        std::string e = check_pair(b, p, in.pairs[p], is_dst);
        if (!e.empty()) return e;
        if (in.actor_off[p + 1] < in.actor_off[p]) return "actor_off decreases";
        const uint64_t na = in.actor_off[p + 1] - in.actor_off[p];
        if (na != b->h_desc[src].n_actors)
            return at(p) + "the actor map has " + std::to_string(na) + " entries and log " + std::to_string(src) + " has " + std::to_string(b->h_desc[src].n_actors) + " actors";
        const uint16_t* a = in.actor_map + in.actor_off[p];
        int64_t last = -1;
        for (uint64_t k = 0; k < na; k++) {
            if (a[k] == 0xFFFFu) continue;
            if ((int64_t)a[k] <= last) return at(p) + "the actor map is not strictly increasing";
            if (a[k] >= b->h_desc[dst].n_actors) return at(p) + "the actor map names a rank >= log " + std::to_string(dst) + "'s n_actors";
            last = a[k];
        }
        if (in.ctr_off) {
            if (in.ctr_off[p + 1] < in.ctr_off[p]) return "ctr_off decreases";
            const uint64_t nc = in.ctr_off[p + 1] - in.ctr_off[p];
            if (nc > 0xFFFFFFFFull) return at(p) + "the counter map has more than 2^32 - 1 entries";
            uint32_t bound;
            if (const char* e = check_ctr_map(in.ctr_map + in.ctr_off[p], nc, 0, bound)) return at(p) + e;
        }
        slot_off[p + 1] = slot_off[p] + b->h_cdesc[src].n_changes;
    }
    return std::string();
}

static int exchange_core(pt_batch* b, const char* fn, const pt_exchange_pair* pairs, uint32_t np, const std::vector<unsigned long long>& slot_off,
                         const unsigned long long* actor_off, const uint16_t* actor_map, const unsigned long long* ctr_off, const uint32_t* ctr_map,
                         pt_exchange_view* out);

// The pinned buffers of an exchange view for np pairs.
static int reserve_exchange_view(pt_batch* b, uint32_t np) {
    int rc;
    if ((rc = reserve_n<ptct::PairTotals>(b->h_xch_totals, np)) || (rc = reserve_n<uint32_t>(b->h_xch_status, np)) ||
        (rc = reserve_n<uint64_t>(b->h_xch_off, (uint64_t)np + 1)) || (rc = reserve_n<pt_log_desc>(b->h_xch_desc, b->n_logs))) return rc;
    return PT_OK;
}

// The exchange view of no pairs, in the reserved buffers: every log's delta empty, with its n_actors and max_ctr.
static int empty_exchange_view(pt_batch* b, pt_exchange_view* out) {
    int rc;
    if ((rc = b->h_xch_delivered.reserve(4))) return rc;
    pt_log_desc* dd = (pt_log_desc*)b->h_xch_desc.p;
    for (uint32_t i = 0; i < b->n_logs; i++) dd[i] = pt_log_desc{0, 0, 0, 0, b->h_desc[i].n_actors, b->h_desc[i].max_ctr};
    ((uint64_t*)b->h_xch_off.p)[0] = 0;
    *out = pt_exchange_view{0, (const uint32_t*)b->h_xch_status.p, (const uint64_t*)b->h_xch_off.p, (const uint32_t*)b->h_xch_delivered.p, dd};
    return PT_OK;
}

// The changes a select kernel (exchange_select_kernel, checkout_select_kernel) delivered, as one delta: the pairs' records,
// change records and deps back to back in pair order.
struct Delta {
    std::vector<ptct::PairBase> base;          // [np] where pair p's start
    std::vector<unsigned long long> dlv_off;   // [np + 1] exclusive scan of the pairs' delivered changes
    uint64_t n_ins = 0, n_mk = 0, n_ch = 0, n_dp = 0;
    DevBuf insdel, marks, changes, deps, d_dlv_off, d_base;
};

// Lays out the delta of the pairs' totals tot (host; a pair that is not OK has zero counts) and gathers it with
// exchange_gather_kernel: P holds the pairs and their maps, the select's scratch and totals (device), and the pairs' dsts index
// dst_desc.  delivered (may be null) gets each delivered change's index in its src's table.
static int gather_delta(pt_batch* b, ptx::ExchangeParams& P, const ptct::PairTotals* tot, const pt_log_desc* dst_desc, DevBuf* delivered, Delta& D) {
    const uint32_t np = P.n_pairs;
    D.base.resize(np);
    D.dlv_off.assign((size_t)np + 1, 0);
    uint64_t most = 0;                         // the largest pair's records: an upper bound of its longest change
    for (uint32_t p = 0; p < np; p++) {
        D.base[p] = ptct::PairBase{D.n_ins, D.n_mk, D.n_ch, D.n_dp};
        D.n_ins += tot[p].n_insdel; D.n_mk += tot[p].n_mark; D.n_ch += tot[p].n_changes; D.n_dp += tot[p].n_deps;
        D.dlv_off[p + 1] = D.n_ch;
        most = std::max<uint64_t>(most, (uint64_t)tot[p].n_insdel + 2ull * tot[p].n_mark);
    }
    int rc;
    if ((rc = reserve_n<pt_insdel_rec>(D.insdel, D.n_ins)) || (rc = reserve_n<pt_mark_rec>(D.marks, D.n_mk)) ||
        (rc = reserve_n<pt_change_rec>(D.changes, D.n_ch)) || (rc = reserve_n<pt_dep_rec>(D.deps, D.n_dp)) ||
        (delivered && (rc = reserve_n<uint32_t>(*delivered, D.n_ch)))) return rc;
    if (!D.n_ch) return PT_OK;
    if ((rc = upload_n(b, D.d_dlv_off, D.dlv_off.data(), (uint64_t)np + 1)) || (rc = upload_n(b, D.d_base, D.base.data(), np))) return rc;
    P.desc = (const pt_log_desc*)b->d_desc.p; P.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    P.changes = (const pt_change_rec*)b->d_changes.p; P.deps = (const pt_dep_rec*)b->d_deps.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.dlv_off = (const unsigned long long*)D.d_dlv_off.p; P.n_dlv = D.n_ch; P.base = (const ptct::PairBase*)D.d_base.p; P.dst_desc = dst_desc;
    P.out_insdel = (pt_insdel_rec*)D.insdel.p; P.out_marks = (pt_mark_rec*)D.marks.p; P.out_changes = (pt_change_rec*)D.changes.p; P.out_deps = (pt_dep_rec*)D.deps.p;
    P.out_delivered = delivered ? (uint32_t*)delivered->p : nullptr;
    ptx::exchange_gather_kernel<<<slice_grid(b, D.n_ch, most, 128), 128, 0, b->stream>>>(P);   // one warp per delivered change
    PT_CUDA(launched(b));
    return PT_OK;
}

int pt_batch_exchange(pt_batch* b, const pt_exchange_input* in, pt_exchange_view* out) {
    if (!b || !in || !out) { g_last_error = "pt_batch_exchange: null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_exchange before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = "pt_batch_exchange: the handle has no change table"; return PT_ERR_STATE; }
    const uint32_t np = in->n_pairs;
    int rc;
    if ((rc = reserve_exchange_view(b, np))) return rc;
    if (!np) {
        PT_CUDA(cudaSetDevice(b->device));
        PT_CUDA(cudaStreamSynchronize(b->stream));          // the pinned view buffers may still be the target of an earlier copy
        return empty_exchange_view(b, out);
    }
    std::vector<unsigned long long> slot_off;
    std::string err = check_exchange(b, *in, slot_off);
    if (!err.empty()) { g_last_error = "pt_batch_exchange: " + err; return PT_ERR_INVALID; }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    DevBuf daoff, damap, dcoff, dcmap;                          // the maps: freed on return
    const uint64_t n_amap = in->actor_off[np], n_cmap = in->ctr_off ? in->ctr_off[np] : 0;
    if ((rc = upload_n(b, daoff, in->actor_off, (uint64_t)np + 1)) || (rc = upload_n(b, damap, in->actor_map, n_amap))) return rc;
    if (in->ctr_off && ((rc = upload_n(b, dcoff, in->ctr_off, (uint64_t)np + 1)) || (rc = upload_n(b, dcmap, in->ctr_map, n_cmap)))) return rc;
    return exchange_core(b, "pt_batch_exchange: ", in->pairs, np, slot_off, (const unsigned long long*)daoff.p, (const uint16_t*)damap.p,
                         in->ctr_off ? (const unsigned long long*)dcoff.p : nullptr, (const uint32_t*)dcmap.p, out);
}

// pt_batch_exchange after its host checks (pt_batch_sync_pairs after deriving its maps): the pairs (host memory) and their maps
// (device memory; ctr_off null = identity), the scratch slots of check_exchange.  Writes the view into the h_xch_* buffers.
static int exchange_core(pt_batch* b, const char* fn, const pt_exchange_pair* pairs, uint32_t np, const std::vector<unsigned long long>& slot_off,
                         const unsigned long long* actor_off, const uint16_t* actor_map, const unsigned long long* ctr_off, const uint32_t* ctr_map,
                         pt_exchange_view* out) {
    const uint32_t n = b->n_logs;
    int rc;
    ptct::PairTotals* tot = (ptct::PairTotals*)b->h_xch_totals.p;
    uint32_t* status = (uint32_t*)b->h_xch_status.p;
    uint64_t* doff = (uint64_t*)b->h_xch_off.p;
    pt_log_desc* dd = (pt_log_desc*)b->h_xch_desc.p;
    const uint64_t n_slot = slot_off[np];
    // the pairs and the select kernel's scratch: freed on return
    DevBuf dpairs, dslot, dqueue, dpos, ddlv, dtot, dgx;
    if ((rc = upload_n(b, dpairs, pairs, np)) || (rc = upload_n(b, dslot, slot_off.data(), (uint64_t)np + 1)) ||
        (rc = reserve_n<uint32_t>(dqueue, n_slot)) || (rc = reserve_n<uint32_t>(dpos, n_slot)) ||
        (rc = reserve_n<ptct::Delivered>(ddlv, n_slot)) || (rc = reserve_n<ptct::PairTotals>(dtot, np))) return rc;
    ptx::ExchangeParams P{};
    P.pairs = (const pt_exchange_pair*)dpairs.p; P.n_pairs = np; P.maxR = b->adm_maxR;
    P.actor_off = actor_off; P.actor_map = actor_map;
    P.ctr_off = ctr_off; P.ctr_map = ctr_map;
    P.desc = (const pt_log_desc*)b->d_desc.p; P.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    P.changes = (const pt_change_rec*)b->d_changes.p; P.deps = (const pt_dep_rec*)b->d_deps.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.slot_off = (const unsigned long long*)dslot.p; P.queue = (uint32_t*)dqueue.p; P.pos = (uint32_t*)dpos.p; P.dlv = (ptct::Delivered*)ddlv.p;
    P.totals = (ptct::PairTotals*)dtot.p;
    if ((rc = launch_actor_kernel(b, ptx::exchange_select_kernel, np, P))) return rc;
    PT_CUDA(cudaMemcpyAsync(tot, dtot.p, (size_t)np * sizeof(ptct::PairTotals), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    Delta D;
    if ((rc = gather_delta(b, P, tot, P.desc, &dgx, D)) || (rc = reserve_n<uint32_t>(b->h_xch_delivered, D.n_ch))) return rc;
    uint32_t* delivered = (uint32_t*)b->h_xch_delivered.p;
    if (D.n_ch) {
        PT_CUDA(cudaMemcpyAsync(tot, dtot.p, (size_t)np * sizeof(ptct::PairTotals), cudaMemcpyDeviceToHost, b->stream));   // status and max_ctr
        PT_CUDA(cudaMemcpyAsync(delivered, dgx.p, D.n_ch * 4, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    // the delta per log; a pair that found an id without an image delivers nothing: its records are never spliced
    std::vector<pt_change_desc> cdesc(n, pt_change_desc{0, 0, 0, 0});
    for (uint32_t i = 0; i < n; i++) dd[i] = pt_log_desc{0, 0, 0, 0, b->h_desc[i].n_actors, b->h_desc[i].max_ctr};
    doff[0] = 0;
    for (uint32_t p = 0; p < np; p++) {
        status[p] = tot[p].status;
        const uint32_t dst = pairs[p].dst, cnt = status[p] == PT_EXCHANGE_OK ? tot[p].n_changes : 0u;
        if (cnt) {
            dd[dst] = pt_log_desc{D.base[p].insdel, D.base[p].mark, tot[p].n_insdel, tot[p].n_mark, b->h_desc[dst].n_actors, std::max(b->h_desc[dst].max_ctr, tot[p].max_ctr)};
            cdesc[dst] = pt_change_desc{D.base[p].change, D.base[p].dep, tot[p].n_changes, tot[p].n_deps};
            if (doff[p] != D.dlv_off[p]) memmove(delivered + doff[p], delivered + D.dlv_off[p], (size_t)cnt * 4);
        }
        doff[p + 1] = doff[p] + cnt;
    }
    const pt_packed_ops delta{n, dd, (const pt_insdel_rec*)D.insdel.p, D.n_ins, (const pt_mark_rec*)D.marks.p, D.n_mk};
    const pt_change_table ct{n, cdesc.data(), (const pt_change_rec*)D.changes.p, D.n_ch, (const pt_dep_rec*)D.deps.p, D.n_dp};
    if ((rc = splice_append(b, fn, &delta, true, pt_append_remap{}, &ct, true))) return rc;
    *out = pt_exchange_view{np, status, doff, delivered, dd};
    return PT_OK;
}

// UTF-16 code-unit order of two UTF-16LE strings (JS string order): <0, 0, >0.
static int js_cmp_host(const uint8_t* a, uint64_t na, const uint8_t* b, uint64_t nb) {
    for (uint64_t i = 0; i + 1 < std::min(na, nb); i += 2) {
        const uint32_t x = a[i] | (uint32_t)a[i + 1] << 8, y = b[i] | (uint32_t)b[i + 1] << 8;
        if (x != y) return x < y ? -1 : 1;
    }
    return na < nb ? -1 : na > nb ? 1 : 0;
}

// pt_batch_upload_actors' host checks (include/peritext_b200.h) of tables for the n logs `desc`.  Returns the problem, or an
// empty string.
static std::string check_actor_tables(const pt_log_desc* desc, uint32_t n, const pt_actor_tables& t) {
    if (t.n_logs != n) return "the tables have " + std::to_string(t.n_logs) + " logs and the batch " + std::to_string(n);
    if (!t.per_log_first || !t.off) return "null per_log_first or off";
    if (t.count && t.off[t.count] > t.off[0] && !t.data) return "null data with a nonzero length";
    if (t.per_log_first[0] != 0 || t.per_log_first[n] != t.count) return "per_log_first does not run from 0 to count";
    for (uint64_t k = 0; k < t.count; k++) if (t.off[k + 1] < t.off[k]) return "the byte offsets decrease at id " + std::to_string(k);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t lo = t.per_log_first[i], hi = t.per_log_first[i + 1];
        if (hi < lo || hi > t.count) return at(i) + "per_log_first decreases or passes count";
        const uint64_t cnt = hi - lo, R = desc[i].n_actors;
        if (cnt != R && !(cnt == 0 && R == 1)) return at(i) + std::to_string(cnt) + " actor ids and n_actors " + std::to_string(R);
        for (uint64_t k = lo; k < hi; k++) {
            if ((t.off[k + 1] - t.off[k]) & 1) return at(i) + "actor " + std::to_string(k - lo) + " has an odd byte length";
            if (k > lo && js_cmp_host(t.data + t.off[k - 1], t.off[k] - t.off[k - 1], t.data + t.off[k], t.off[k + 1] - t.off[k]) >= 0)
                return at(i) + "actor " + std::to_string(k - lo) + " does not sort after actor " + std::to_string(k - lo - 1) + " (UTF-16 code-unit order)";
        }
        if (t.counters_first && t.counters_first[i + 1] < t.counters_first[i]) return at(i) + "counters_first decreases";
    }
    return std::string();
}

int pt_batch_upload_actors(pt_batch* b, const pt_actor_tables* t) {
    if (!b || !t) { g_last_error = "pt_batch_upload_actors: null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_upload_actors before pt_batch_upload"; return PT_ERR_STATE; }
    const std::string err = check_actor_tables(b->h_desc.data(), b->n_logs, *t);
    if (!err.empty()) { g_last_error = "pt_batch_upload_actors: " + err; return PT_ERR_INVALID; }
    const uint32_t n = b->n_logs;
    const uint64_t lo = t->count ? t->off[0] : 0, bytes = t->count ? t->off[t->count] - lo : 0;
    std::vector<uint64_t> off(t->count + 1), abyte(n + 1);
    for (uint64_t k = 0; k <= t->count; k++) off[k] = t->count ? t->off[k] - lo : 0;
    for (uint32_t i = 0; i <= n; i++) abyte[i] = off[t->per_log_first[i]];
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    int rc;
    if ((rc = upload_n(b, b->d_anames, bytes ? t->data + lo : nullptr, bytes)) || (rc = upload_n(b, b->d_aoff, off.data(), off.size())) ||
        (rc = upload_n(b, b->d_afirst, t->per_log_first, (uint64_t)n + 1))) { b->have_actors = false; return rc; }
    PT_CUDA(cudaStreamSynchronize(b->stream));            // the caller's arrays may be freed on return
    b->h_afirst.assign(t->per_log_first, t->per_log_first + n + 1);
    b->h_abyte = std::move(abyte);
    b->h_adense.assign(n, 0);
    for (uint32_t i = 0; t->counters_first && i < n; i++) b->h_adense[i] = t->counters_first[i + 1] > t->counters_first[i];
    b->have_actors = true;
    return PT_OK;
}

int pt_batch_download_actors(pt_batch* b, pt_actor_tables* out) {
    if (!b || !out) { g_last_error = "pt_batch_download_actors: null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch || !b->have_actors) { g_last_error = "pt_batch_download_actors: the handle has no actor tables"; return PT_ERR_STATE; }
    const uint32_t n = b->n_logs;
    const uint64_t count = b->h_afirst[n], bytes = b->h_abyte[n];
    int rc;
    if ((rc = reserve_n<uint8_t>(b->h_act_data, bytes)) || (rc = reserve_n<uint64_t>(b->h_act_off, count + 1)) ||
        (rc = reserve_n<uint64_t>(b->h_act_first, (uint64_t)n + 1))) return rc;
    PT_CUDA(cudaSetDevice(b->device));
    if (bytes) PT_CUDA(cudaMemcpyAsync(b->h_act_data.p, b->d_anames.p, bytes, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(b->h_act_off.p, b->d_aoff.p, (count + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    memcpy(b->h_act_first.p, b->h_afirst.data(), ((size_t)n + 1) * 8);
    *out = pt_actor_tables{n, (const uint8_t*)b->h_act_data.p, (const uint64_t*)b->h_act_off.p, count, (const uint64_t*)b->h_act_first.p, nullptr};
    return PT_OK;
}

// Grows every log i with grow[i] != ~0 by the n_new names of slot grow[i] (tot[slot]: n_new, new_bytes, moves), which are the
// ids new_id[new_off[slot] ..] of the pool (new_data, new_byte_off), in JS order, none in the log's table: the merge kernel
// writes the grown tables and the old -> new rank maps of the logs whose ranks move; when a rank moves or an n_actors grows,
// one splice of an empty delta with those maps applies it (identity counters).  Then the grown tables replace the old.  The
// per-log maps go to haoff ([n_logs + 1]) / hamap.
static int grow_tables(pt_batch* b, const char* fn, const std::vector<uint32_t>& grow, const pty::SyncTotals* tot, uint32_t n_slots,
                       const uint8_t* new_data, const unsigned long long* new_byte_off, const unsigned long long* new_off, const unsigned long long* new_id,
                       HostBuf& haoff, HostBuf& hamap, bool* spliced = nullptr) {
    const uint32_t n = b->n_logs;
    int rc;
    if ((rc = reserve_n<uint64_t>(haoff, (uint64_t)n + 1))) return rc;
    uint64_t* aoff = (uint64_t*)haoff.p;
    std::vector<uint32_t> n_new(n_slots, 0);
    for (uint32_t g = 0; g < n_slots; g++) n_new[g] = tot[g].n_new;
    std::vector<unsigned long long> map_off(n, ~0ull), new_first((size_t)n + 1, 0), new_byte((size_t)n + 1, 0);
    std::vector<uint32_t> new_actors(n);
    bool grows = false, splice = false;
    uint64_t n_map = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t g = grow[i];
        const uint64_t cnt = b->h_afirst[i + 1] - b->h_afirst[i] + (g == 0xFFFFFFFFu ? 0 : n_new[g]);
        new_first[i + 1] = new_first[i] + cnt;
        new_byte[i + 1] = new_byte[i] + (b->h_abyte[i + 1] - b->h_abyte[i]) + (g == 0xFFFFFFFFu ? 0 : tot[g].new_bytes);
        new_actors[i] = (uint32_t)std::max<uint64_t>(std::max<uint64_t>(1, cnt), b->h_desc[i].n_actors);
        if (cnt > 0xFFFF) { g_last_error = std::string(fn) + at(i) + "more than 65535 actors"; return PT_ERR_INVALID; }
        if (g == 0xFFFFFFFFu) continue;
        grows = true;
        if (tot[g].moves) { map_off[i] = n_map; n_map += b->h_desc[i].n_actors; }
        splice = splice || tot[g].moves || new_actors[i] != b->h_desc[i].n_actors;
    }
    DevBuf nnames, noff, nfirst, nbyte, dgrow, dnn, dmoff, dmap, dsrc;   // the grown tables (swapped in once accepted) and scratch
    if (grows) {
        if ((rc = reserve_n<uint8_t>(nnames, new_byte[n])) || (rc = reserve_n<unsigned long long>(noff, new_first[n] + 1)) ||
            (rc = upload_n(b, nfirst, new_first.data(), (uint64_t)n + 1)) || (rc = upload_n(b, nbyte, new_byte.data(), n)) ||
            (rc = upload_n(b, dgrow, grow.data(), n)) || (rc = upload_n(b, dnn, n_new.data(), n_slots)) || (rc = upload_n(b, dmoff, map_off.data(), n)) ||
            (rc = reserve_n<uint16_t>(dmap, n_map)) || (rc = reserve_n<const uint8_t*>(dsrc, new_first[n]))) return rc;
        PT_CUDA(cudaMemsetAsync(noff.p, 0, 8, b->stream));
        pty::MergeParams M{};
        M.n_logs = n;
        M.old_t = pty::Tables{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
        M.data = (uint8_t*)nnames.p; M.off = (unsigned long long*)noff.p; M.first = (const unsigned long long*)nfirst.p;
        M.byte_base = (const unsigned long long*)nbyte.p; M.grow = (const uint32_t*)dgrow.p;
        M.new_data = new_data; M.new_byte_off = new_byte_off; M.new_off = new_off; M.new_id = new_id; M.n_new = (const uint32_t*)dnn.p;
        M.map_off = (const unsigned long long*)dmoff.p; M.map = (uint16_t*)dmap.p; M.src_at = (const uint8_t**)dsrc.p;
        pty::actor_merge_kernel<<<warp_grid(b, n, 128), 128, 0, b->stream>>>(M);
        PT_CUDA(launched(b));
    }
    if ((rc = reserve_n<uint16_t>(hamap, n_map))) return rc;
    aoff[0] = 0;
    for (uint32_t i = 0; i < n; i++) aoff[i + 1] = aoff[i] + (map_off[i] == ~0ull ? 0 : b->h_desc[i].n_actors);
    if (n_map) PT_CUDA(cudaMemcpyAsync(hamap.p, dmap.p, n_map * 2, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    if (spliced) *spliced = splice;
    if (splice) {
        std::vector<pt_log_desc> dd(n);
        for (uint32_t i = 0; i < n; i++) dd[i] = pt_log_desc{0, 0, 0, 0, new_actors[i], b->h_desc[i].max_ctr};
        std::vector<pt_change_desc> cd(n, pt_change_desc{0, 0, 0, 0});
        const pt_packed_ops delta{n, dd.data(), nullptr, 0, nullptr, 0};
        const pt_change_table ct{n, cd.data(), nullptr, 0, nullptr, 0};
        const pt_append_remap R{n_map ? aoff : nullptr, (const uint16_t*)hamap.p, nullptr, nullptr, nullptr, 0};
        if ((rc = splice_append(b, fn, &delta, true, R, b->have_changes ? &ct : nullptr, false))) return rc;
    }
    if (grows) {
        b->d_anames.swap(nnames); b->d_aoff.swap(noff); b->d_afirst.swap(nfirst);
        b->h_afirst.assign(new_first.begin(), new_first.end()); b->h_abyte.assign(new_byte.begin(), new_byte.end());
        b->have_actors = true;
    }
    return PT_OK;
}

int pt_batch_sync_pairs(pt_batch* b, const pt_exchange_pair* pairs, uint32_t np, pt_sync_view* out) {
    const char* fn = "pt_batch_sync_pairs: ";
    if (!b || !out || (np && !pairs)) { g_last_error = std::string(fn) + "null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_sync_pairs before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = std::string(fn) + "the handle has no change table"; return PT_ERR_STATE; }
    if (!b->have_actors) { g_last_error = std::string(fn) + "the handle has no actor tables"; return PT_ERR_STATE; }
    const uint32_t n = b->n_logs;
    int rc;
    if ((rc = reserve_exchange_view(b, np)) || (rc = reserve_n<uint32_t>(b->h_syn_status, np)) || (rc = reserve_n<uint64_t>(b->h_syn_off, (uint64_t)np + 1)) ||
        (rc = reserve_n<uint64_t>(b->h_syn_aoff, (uint64_t)n + 1)) || (rc = reserve_n<pty::SyncTotals>(b->h_syn_totals, np))) return rc;
    uint32_t* status = (uint32_t*)b->h_syn_status.p;
    uint64_t* soff = (uint64_t*)b->h_syn_off.p;
    pty::SyncTotals* tot = (pty::SyncTotals*)b->h_syn_totals.p;
    std::vector<char> is_dst(n, 0);
    for (uint32_t p = 0; p < np; p++) {
        const std::string e = check_pair(b, p, pairs[p], is_dst);
        if (!e.empty()) { g_last_error = fn + e; return PT_ERR_INVALID; }
    }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // the pinned view buffers may still be the target of an earlier copy
    // ---- derive: a pair with a densely ranked log is DENSE outright; the others go to the derive kernel ----
    std::vector<uint32_t> live;
    std::vector<pt_exchange_pair> lp;
    std::vector<unsigned long long> slot_off(1, 0), new_off(1, 0);
    for (uint32_t p = 0; p < np; p++) {
        status[p] = PT_EXCHANGE_DENSE;
        if (b->h_adense[pairs[p].src] || b->h_adense[pairs[p].dst]) continue;
        live.push_back(p); lp.push_back(pairs[p]);
        slot_off.push_back(slot_off.back() + b->h_cdesc[pairs[p].src].n_changes);
        new_off.push_back(new_off.back() + (b->h_afirst[pairs[p].src + 1] - b->h_afirst[pairs[p].src]));
    }
    const uint32_t nl = (uint32_t)live.size();
    const pty::Tables T0{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
    DevBuf dlp, dslot, dpos, dnoff, dnew, dtot;                 // freed on return
    if (nl) {
        if ((rc = upload_n(b, dlp, lp.data(), nl)) || (rc = upload_n(b, dslot, slot_off.data(), (uint64_t)nl + 1)) ||
            (rc = upload_n(b, dnoff, new_off.data(), (uint64_t)nl + 1)) || (rc = reserve_n<uint32_t>(dpos, slot_off[nl])) ||
            (rc = reserve_n<unsigned long long>(dnew, new_off[nl])) || (rc = reserve_n<pty::SyncTotals>(dtot, nl))) return rc;
        pty::DeriveParams D{};
        D.pairs = (const pt_exchange_pair*)dlp.p; D.n_pairs = nl; D.maxR = b->adm_maxR; D.T = T0;
        D.desc = (const pt_log_desc*)b->d_desc.p; D.cdesc = (const pt_change_desc*)b->d_cdesc.p;
        D.changes = (const pt_change_rec*)b->d_changes.p; D.deps = (const pt_dep_rec*)b->d_deps.p; D.insdel = b->dp_insdel; D.marks = b->dp_marks;
        D.slot_off = (const unsigned long long*)dslot.p; D.pos = (uint32_t*)dpos.p;
        D.new_off = (const unsigned long long*)dnoff.p; D.new_id = (unsigned long long*)dnew.p; D.totals = (pty::SyncTotals*)dtot.p;
        if ((rc = launch_actor_kernel(b, pty::sync_derive_kernel, nl, D))) return rc;
        PT_CUDA(cudaMemcpyAsync(tot, dtot.p, (size_t)nl * sizeof(pty::SyncTotals), cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    // ---- growth and pre-append ----
    std::vector<uint32_t> grow(n, 0xFFFFFFFFu);
    for (uint32_t k = 0; k < nl; k++) {
        if (tot[k].verdict == pty::kDeriveDense) continue;
        status[live[k]] = PT_EXCHANGE_OK;
        if (tot[k].verdict == pty::kDeriveGrow && tot[k].n_new) grow[lp[k].dst] = k;
    }
    if ((rc = grow_tables(b, fn, grow, tot, nl, T0.data, T0.off, (const unsigned long long*)dnoff.p, (const unsigned long long*)dnew.p,
                          b->h_syn_aoff, b->h_syn_amap))) return rc;
    // ---- the exchange of the pairs that are not DENSE, with the maps of the grown tables ----
    std::vector<pt_exchange_pair> xp;
    std::vector<unsigned long long> xslot(1, 0), xaoff(1, 0);
    for (uint32_t p = 0; p < np; p++) {
        if (status[p] == PT_EXCHANGE_DENSE) continue;
        xp.push_back(pairs[p]);
        xslot.push_back(xslot.back() + b->h_cdesc[pairs[p].src].n_changes);
        xaoff.push_back(xaoff.back() + b->h_desc[pairs[p].src].n_actors);
    }
    const uint32_t nx = (uint32_t)xp.size();
    pt_exchange_view xv{};
    if (nx) {
        DevBuf dxp, dxaoff, dxmap;
        if ((rc = upload_n(b, dxp, xp.data(), nx)) || (rc = upload_n(b, dxaoff, xaoff.data(), (uint64_t)nx + 1)) || (rc = reserve_n<uint16_t>(dxmap, xaoff[nx]))) return rc;
        const pty::Tables T{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
        pty::sync_maps_kernel<<<warp_grid(b, nx, 128), 128, 0, b->stream>>>((const pt_exchange_pair*)dxp.p, nx, T, (const pt_log_desc*)b->d_desc.p,
                                                                            (const unsigned long long*)dxaoff.p, (uint16_t*)dxmap.p);
        PT_CUDA(launched(b));
        if ((rc = exchange_core(b, fn, xp.data(), nx, xslot, (const unsigned long long*)dxaoff.p, (const uint16_t*)dxmap.p, nullptr, nullptr, &xv))) return rc;
    } else if ((rc = empty_exchange_view(b, &xv))) return rc;
    // the view: the exchange's, with the DENSE pairs (nothing delivered) in their places
    soff[0] = 0;
    for (uint32_t p = 0, x = 0; p < np; p++) {
        if (status[p] == PT_EXCHANGE_DENSE) { soff[p + 1] = soff[p]; continue; }
        status[p] = xv.status[x];
        soff[p + 1] = soff[p] + (xv.delivered_off[x + 1] - xv.delivered_off[x]);
        x++;
    }
    *out = pt_sync_view{np, status, soff, xv.delivered, xv.delta, (const uint64_t*)b->h_syn_aoff.p, (const uint16_t*)b->h_syn_amap.p};
    return PT_OK;
}

int pt_batch_add_actors(pt_batch* b, const pt_actor_input* in, pt_actor_view* out) {
    const char* fn = "pt_batch_add_actors: ";
    if (!b || !in || !out) { g_last_error = std::string(fn) + "null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_add_actors before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_actors) { g_last_error = std::string(fn) + "the handle has no actor tables"; return PT_ERR_STATE; }
    const uint32_t n = b->n_logs;
    std::string err;
    if (in->n_logs != n) err = "the input has " + std::to_string(in->n_logs) + " logs and the batch " + std::to_string(n);
    else if (!in->per_log_first || (in->count && !in->off)) err = "null per_log_first or off";
    else if (in->count && in->off[in->count] > in->off[0] && !in->data) err = "null data with a nonzero length";
    else if (in->per_log_first[0] != 0 || in->per_log_first[n] != in->count) err = "per_log_first does not run from 0 to count";
    for (uint32_t i = 0; err.empty() && i < n; i++) {
        if (in->per_log_first[i + 1] < in->per_log_first[i] || in->per_log_first[i + 1] > in->count) err = at(i) + "per_log_first decreases or passes count";
        for (uint64_t k = in->per_log_first[i]; err.empty() && k < in->per_log_first[i + 1]; k++) {
            if (in->off[k + 1] < in->off[k]) err = "the byte offsets decrease at id " + std::to_string(k);
            else if ((in->off[k + 1] - in->off[k]) & 1) err = at(i) + "id " + std::to_string(k - in->per_log_first[i]) + " has an odd byte length";
        }
    }
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    const uint64_t count = in->count, lo = count ? in->off[0] : 0, bytes = count ? in->off[count] - lo : 0;
    int rc;
    if ((rc = reserve_n<uint16_t>(b->h_add_rank, count)) || (rc = reserve_n<pty::SyncTotals>(b->h_add_totals, n))) return rc;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // the pinned view buffers may still be the target of an earlier copy
    std::vector<unsigned long long> off(count + 1);
    for (uint64_t k = 0; k <= count; k++) off[k] = count ? in->off[k] - lo : 0;
    DevBuf ddata, doff, dfirst, dfresh, dnew, dtot, drank;      // freed on return
    if ((rc = upload_n(b, ddata, bytes ? in->data + lo : nullptr, bytes)) || (rc = upload_n(b, doff, off.data(), count + 1)) ||
        (rc = upload_n(b, dfirst, in->per_log_first, (uint64_t)n + 1)) || (rc = reserve_n<uint32_t>(dfresh, count)) ||
        (rc = reserve_n<unsigned long long>(dnew, count)) || (rc = reserve_n<pty::SyncTotals>(dtot, n)) || (rc = reserve_n<uint16_t>(drank, count))) return rc;
    pty::SyncTotals* tot = (pty::SyncTotals*)b->h_add_totals.p;
    std::vector<uint32_t> grow(n, 0xFFFFFFFFu);
    bool spliced = false;
    if (count) {
        pty::AddParams A{};
        A.n_logs = n; A.T = pty::Tables{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
        A.data = (const uint8_t*)ddata.p; A.off = (const unsigned long long*)doff.p; A.first = (const unsigned long long*)dfirst.p;
        A.fresh = (uint32_t*)dfresh.p; A.new_id = (unsigned long long*)dnew.p; A.totals = (pty::SyncTotals*)dtot.p;
        pty::add_select_kernel<<<warp_grid(b, n, 128), 128, 0, b->stream>>>(A);
        PT_CUDA(launched(b));
        PT_CUDA(cudaMemcpyAsync(tot, dtot.p, (size_t)n * sizeof(pty::SyncTotals), cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
        for (uint32_t i = 0; i < n; i++) if (tot[i].n_new) grow[i] = i;
    } else {
        for (uint32_t i = 0; i < n; i++) tot[i] = pty::SyncTotals{};
    }
    if ((rc = grow_tables(b, fn, grow, tot, n, (const uint8_t*)ddata.p, (const unsigned long long*)doff.p, (const unsigned long long*)dfirst.p,
                          (const unsigned long long*)dnew.p, b->h_add_aoff, b->h_add_amap, &spliced))) return rc;
    if (count) {
        const pty::Tables T{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
        pty::add_ranks_kernel<<<warp_grid(b, n, 128), 128, 0, b->stream>>>(n, T, (const uint8_t*)ddata.p, (const unsigned long long*)doff.p,
                                                                           (const unsigned long long*)dfirst.p, (uint16_t*)drank.p);
        PT_CUDA(launched(b));
        PT_CUDA(cudaMemcpyAsync(b->h_add_rank.p, drank.p, count * 2, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    *out = pt_actor_view{n, count, (const uint16_t*)b->h_add_rank.p, (const uint64_t*)b->h_add_aoff.p, (const uint16_t*)b->h_add_amap.p, spliced ? 1u : 0u};
    return PT_OK;
}

// pt_batch_select_logs' host checks (include/peritext_b200.h).  On success nd / dd / ncd / dcd hold the new batch's
// descriptors and the per-new-log delta descriptors of the splice (an added log's records, empty for a kept one) and
// add_idx[i] the added log new log i is (or ~0u).  Returns the problem, or an empty string.
static std::string check_select(const pt_batch* b, const uint32_t* from, uint32_t n, const pt_packed_ops* added, const pt_change_table* ach,
                                const pt_actor_tables* aact, const uint32_t* comment_map, uint64_t n_comment_map,
                                std::vector<pt_log_desc>& nd, std::vector<pt_log_desc>& dd, std::vector<pt_change_desc>& ncd,
                                std::vector<pt_change_desc>& dcd, std::vector<uint32_t>& add_idx, uint32_t& maxR) {
    if (n && !from) return "null from with n_logs > 0";
    const uint32_t na = added ? added->n_logs : 0;
    if (added && na && !added->logs) return "null added descriptors with a nonzero n_logs";
    add_idx.assign(n, ~0u);
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (from[i] == PT_SELECT_ADDED) { add_idx[i] = k++; continue; }
        if (from[i] >= b->n_logs) return "from[" + std::to_string(i) + "] = " + std::to_string(from[i]) + " names no resident log (the batch has " + std::to_string(b->n_logs) + ")";
    }
    if (k != na) return std::to_string(k) + " entries are PT_SELECT_ADDED and added has " + std::to_string(na) + " logs";
    if (!na && (ach || aact)) return "added change or actor tables without added logs";
    if (na && (ach != nullptr) != b->have_changes)
        return b->have_changes ? "the batch has a change table and the added logs none" : "the added logs have a change table and the batch none";
    if (na && (aact != nullptr) != b->have_actors)
        return b->have_actors ? "the batch has actor tables and the added logs none" : "the added logs have actor tables and the batch none";
    if (na && ((added->n_insdel_total && !added->insdel) || (added->n_mark_total && !added->marks))) return "null added records with a nonzero count";
    if (n_comment_map && !comment_map) return "null comment_map with a nonzero length";
    uint64_t last = 0;
    bool any = false;
    for (uint64_t c = 0; comment_map && c < n_comment_map; c++) {
        if (comment_map[c] == 0xFFFFFFFFu) continue;
        if (any && comment_map[c] <= last) return "comment_map is not strictly increasing at entry " + std::to_string(c);
        last = comment_map[c]; any = true;
    }
    for (uint32_t j = 0; j < na; j++) {
        const pt_log_desc& A = added->logs[j];
        if (A.insdel_off + A.n_insdel > added->n_insdel_total || A.mark_off + A.n_mark > added->n_mark_total) return "added log " + std::to_string(j) + ": descriptor out of range";
    }
    if (ach) {
        if (ach->n_logs != na || !ach->logs) return "the added change table does not match the added logs";
        if ((ach->n_changes_total && !ach->changes) || (ach->n_deps_total && !ach->deps)) return "null added change records with a nonzero count";
        for (uint32_t j = 0; j < na; j++) {
            const pt_change_desc& D = ach->logs[j];
            if (D.change_off + D.n_changes > ach->n_changes_total || D.dep_off + D.n_deps > ach->n_deps_total) return "added log " + std::to_string(j) + ": change descriptor out of range";
        }
    }
    if (aact) {
        const std::string e = check_actor_tables(added->logs, na, *aact);
        if (!e.empty()) return "added actor tables: " + e;
    }
    nd.resize(n); dd.assign(n, pt_log_desc{}); ncd.clear(); dcd.clear();
    if (b->have_changes) { ncd.resize(n); dcd.assign(n, pt_change_desc{}); }
    uint64_t io = 0, mo = 0, co = 0, po = 0;
    maxR = 1;
    for (uint32_t i = 0; i < n; i++) {
        const bool add = add_idx[i] != ~0u;
        const pt_log_desc S = add ? added->logs[add_idx[i]] : b->h_desc[from[i]];
        if (add) dd[i] = pt_log_desc{S.insdel_off, S.mark_off, S.n_insdel, S.n_mark, S.n_actors, S.max_ctr};
        nd[i] = pt_log_desc{io, mo, S.n_insdel, S.n_mark, S.n_actors, S.max_ctr};
        io += S.n_insdel; mo += S.n_mark;
        maxR = std::max<uint32_t>(maxR, S.n_actors);
        if (!b->have_changes) continue;
        const pt_change_desc C = add ? ach->logs[add_idx[i]] : b->h_cdesc[from[i]];
        if (add) dcd[i] = C;
        ncd[i] = pt_change_desc{co, po, C.n_changes, C.n_deps};
        co += C.n_changes; po += C.n_deps;
    }
    if (b->have_changes && actor_table_bytes(maxR) > kAdmitMaxBytes) return "more than 25600 actors in one log: not supported by the admission pre-pass";
    return std::string();
}

// New actor tables for the n logs of a select or a checkout: new log i takes resident log from[i]'s table, or (from[i] ==
// PT_SELECT_ADDED) added log add_idx[i]'s of `added`.  They are gathered into buffers of their own, which replace the handle's
// (install_actor_tables) once the splice is accepted.
struct NewActorTables {
    DevBuf names, off, first, byte, from, adata, aoff, afirst;   // the tables, and the gather's inputs
    std::vector<unsigned long long> h_first, h_byte;
    std::vector<char> dense;
};

static int gather_actor_tables(pt_batch* b, const uint32_t* from, uint32_t n, const pt_actor_tables* added, const std::vector<uint32_t>& add_idx,
                               NewActorTables& T) {
    int rc;
    const uint64_t lo = added && added->count ? added->off[0] : 0;
    const uint64_t abytes = added && added->count ? added->off[added->count] - lo : 0, acount = added ? added->count : 0;
    std::vector<unsigned long long> add_first(n, 0), add_off(acount + 1, 0);
    for (uint64_t k = 0; k <= acount && added; k++) add_off[k] = acount ? added->off[k] - lo : 0;
    T.h_first.assign((size_t)n + 1, 0); T.h_byte.assign((size_t)n + 1, 0); T.dense.assign(n, 0);
    for (uint32_t i = 0; i < n; i++) {
        uint64_t cnt, bytes;
        if (add_idx[i] != ~0u) {
            const uint64_t* pf = added->per_log_first + add_idx[i];
            add_first[i] = pf[0]; cnt = pf[1] - pf[0]; bytes = add_off[pf[1]] - add_off[pf[0]];
            T.dense[i] = added->counters_first && added->counters_first[add_idx[i] + 1] > added->counters_first[add_idx[i]];
        } else {
            const uint32_t s = from[i];
            cnt = b->h_afirst[s + 1] - b->h_afirst[s]; bytes = b->h_abyte[s + 1] - b->h_abyte[s];
            T.dense[i] = b->h_adense[s];
        }
        T.h_first[i + 1] = T.h_first[i] + cnt; T.h_byte[i + 1] = T.h_byte[i] + bytes;
    }
    if ((rc = reserve_n<uint8_t>(T.names, T.h_byte[n])) || (rc = reserve_n<unsigned long long>(T.off, T.h_first[n] + 1)) ||
        (rc = upload_n(b, T.first, T.h_first.data(), (uint64_t)n + 1)) || (rc = upload_n(b, T.byte, T.h_byte.data(), (uint64_t)n + 1)) ||
        (rc = upload_n(b, T.from, from, n)) || (rc = upload_n(b, T.adata, abytes ? added->data + lo : nullptr, abytes)) ||
        (rc = upload_n(b, T.aoff, add_off.data(), acount + 1)) || (rc = upload_n(b, T.afirst, add_first.data(), n))) return rc;
    PT_CUDA(cudaMemsetAsync(T.off.p, 0, 8, b->stream));
    if (n) {
        pty::GatherParams G{};
        G.n_logs = n; G.from = (const uint32_t*)T.from.p;
        G.old_t = pty::Tables{(const uint8_t*)b->d_anames.p, (const unsigned long long*)b->d_aoff.p, (const unsigned long long*)b->d_afirst.p};
        G.add_data = (const uint8_t*)T.adata.p; G.add_off = (const unsigned long long*)T.aoff.p; G.add_first = (const unsigned long long*)T.afirst.p;
        G.data = (uint8_t*)T.names.p; G.off = (unsigned long long*)T.off.p;
        G.first = (const unsigned long long*)T.first.p; G.byte_base = (const unsigned long long*)T.byte.p;
        pty::actor_gather_kernel<<<warp_grid(b, n, 128), 128, 0, b->stream>>>(G);
        PT_CUDA(launched(b));
    }
    return PT_OK;
}

static void install_actor_tables(pt_batch* b, NewActorTables& T) {
    b->d_anames.swap(T.names); b->d_aoff.swap(T.off); b->d_afirst.swap(T.first);
    b->h_afirst.assign(T.h_first.begin(), T.h_first.end()); b->h_abyte.assign(T.h_byte.begin(), T.h_byte.end());
    b->h_adense = std::move(T.dense);
}

int pt_batch_select_logs(pt_batch* b, const uint32_t* from, uint32_t n, const pt_packed_ops* added, const pt_change_table* added_changes,
                         const pt_actor_tables* added_actors, const uint32_t* comment_map, uint64_t n_comment_map) {
    const char* fn = "pt_batch_select_logs: ";
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_select_logs before pt_batch_upload"; return PT_ERR_STATE; }
    std::vector<pt_log_desc> nd, dd;
    std::vector<pt_change_desc> ncd, dcd;
    std::vector<uint32_t> add_idx;
    uint32_t maxR = 1;
    const std::string err = check_select(b, from, n, added, added_changes, added_actors, comment_map, n_comment_map, nd, dd, ncd, dcd, add_idx, maxR);
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    // the splice's delta: the added logs' records, described per new log
    const pt_packed_ops delta{n, dd.data(), added ? added->insdel : nullptr, added ? added->n_insdel_total : 0, added ? added->marks : nullptr,
                              added ? added->n_mark_total : 0};
    const pt_change_table dch{n, dcd.data(), added_changes ? added_changes->changes : nullptr, added_changes ? added_changes->n_changes_total : 0,
                              added_changes ? added_changes->deps : nullptr, added_changes ? added_changes->n_deps_total : 0};
    const pt_append_remap R{nullptr, nullptr, nullptr, nullptr, comment_map, comment_map ? n_comment_map : 0};
    PT_CUDA(cudaSetDevice(b->device));
    // The actor tables are gathered first, into new buffers that replace the old ones once the splice is accepted.
    int rc;
    NewActorTables T;
    if (b->have_actors && (rc = gather_actor_tables(b, from, n, added_actors, add_idx, T))) return rc;
    if ((rc = splice(b, fn, std::move(nd), std::move(ncd), maxR, &delta, false, R, from, b->have_changes ? &dch : nullptr, false, true))) return rc;
    if (b->have_actors) install_actor_tables(b, T);
    return PT_OK;
}

// The request checks of pt_batch_checkout and pt_batch_attribute: logs inside the batch and, with clock_off, their clocks.
// Returns the problem, or an empty string.
static std::string check_clock_requests(const pt_batch* b, const uint32_t* logs, uint32_t n, const uint64_t* clock_off, const pt_clock_entry* clock) {
    if (clock_off && clock_off[0] != 0) return "clock_off[0] is not 0";
    std::vector<uint32_t> seen;                           // seen[a] = k + 1: request k names actor a
    for (uint32_t k = 0; k < n; k++) {
        const std::string here = "request " + std::to_string(k) + ": ";
        if (logs[k] >= b->n_logs) return here + "log " + std::to_string(logs[k]) + " is outside the batch's " + std::to_string(b->n_logs) + " logs";
        if (!clock_off) continue;
        if (clock_off[k + 1] < clock_off[k]) return "clock_off decreases at request " + std::to_string(k);
        if (clock_off[k + 1] > clock_off[k] && !clock) return "null clock with a nonzero length";
        const uint32_t R = b->h_desc[logs[k]].n_actors;
        if (seen.size() < R) seen.resize(R, 0);
        for (uint64_t e = clock_off[k]; e < clock_off[k + 1]; e++) {
            const uint32_t a = clock[e].actor;
            if (a >= R) return here + "clock actor " + std::to_string(a) + " >= log " + std::to_string(logs[k]) + "'s " + std::to_string(R) + " actors";
            if (seen[a] == k + 1) return here + "actor " + std::to_string(a) + " is named twice";
            seen[a] = k + 1;
        }
    }
    return std::string();
}

// pt_batch_checkout's host checks (include/peritext_b200.h).  Returns the problem, or an empty string.
static std::string check_checkout(const pt_batch* b, const uint32_t* logs, uint32_t n, const uint32_t* n_changes, const uint64_t* clock_off,
                                  const pt_clock_entry* clock, const uint32_t* status_out) {
    if (!logs || !status_out) return "null logs or status_out";
    if ((n_changes != nullptr) == (clock_off != nullptr)) return "exactly one of n_changes (prefix mode) and clock_off (clock mode) must be given";
    if ((uint64_t)b->n_logs + n > 0xFFFFFFFFull) return "the batch would have more than 2^32 - 1 logs";
    return check_clock_requests(b, logs, n, clock_off, clock);
}

int pt_batch_checkout(pt_batch* b, const uint32_t* logs, uint32_t n, const uint32_t* n_changes, const uint64_t* clock_off,
                      const pt_clock_entry* clock, uint32_t* status_out) {
    const char* fn = "pt_batch_checkout: ";
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_checkout before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = std::string(fn) + "the handle has no change table"; return PT_ERR_STATE; }
    if (!n) return PT_OK;
    const std::string err = check_checkout(b, logs, n, n_changes, clock_off, clock, status_out);
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    const uint32_t n0 = b->n_logs, nn = n0 + n;
    std::vector<unsigned long long> slot_off((size_t)n + 1, 0);
    for (uint32_t k = 0; k < n; k++) slot_off[k + 1] = slot_off[k] + b->h_cdesc[logs[k]].n_changes;
    const uint64_t n_slot = slot_off[n];
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    int rc;
    // ---- select: which changes each request covers, its status and its records' places ----
    DevBuf dlogs, dnch, dcoff, dclk, dslot, dpos, dcov, ddlv, dtot;   // freed on return
    if ((rc = upload_n(b, dlogs, logs, n)) || (rc = upload_n(b, dslot, slot_off.data(), (uint64_t)n + 1)) ||
        (rc = reserve_n<uint32_t>(dpos, n_slot)) || (rc = reserve_n<uint32_t>(dcov, n_slot)) ||
        (rc = reserve_n<ptct::Delivered>(ddlv, n_slot)) || (rc = reserve_n<ptct::PairTotals>(dtot, n))) return rc;
    if (n_changes && (rc = upload_n(b, dnch, n_changes, n))) return rc;
    if (clock_off && ((rc = upload_n(b, dcoff, clock_off, (uint64_t)n + 1)) || (rc = upload_n(b, dclk, clock, clock_off[n])))) return rc;
    ptck::CheckoutParams C{};
    C.logs = (const uint32_t*)dlogs.p; C.n = n; C.maxR = b->adm_maxR;
    C.n_changes = n_changes ? (const uint32_t*)dnch.p : nullptr;
    C.clock_off = (const unsigned long long*)dcoff.p; C.clock = (const pt_clock_entry*)dclk.p;
    C.desc = (const pt_log_desc*)b->d_desc.p; C.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    C.changes = (const pt_change_rec*)b->d_changes.p; C.deps = (const pt_dep_rec*)b->d_deps.p; C.marks = b->dp_marks;
    C.slot_off = (const unsigned long long*)dslot.p; C.pos = (uint32_t*)dpos.p; C.cov = (uint32_t*)dcov.p; C.dlv = (ptct::Delivered*)ddlv.p;
    C.totals = (ptct::PairTotals*)dtot.p;
    if ((rc = launch_actor_kernel(b, ptck::checkout_select_kernel, n, C))) return rc;
    std::vector<ptct::PairTotals> tot(n);
    PT_CUDA(cudaMemcpyAsync(tot.data(), dtot.p, (size_t)n * sizeof(ptct::PairTotals), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    // ---- gather: the covered changes' records, change and dep records into the delta, identity maps, arrivals from 0 ----
    std::vector<pt_exchange_pair> pairs(n);
    for (uint32_t k = 0; k < n; k++) pairs[k] = pt_exchange_pair{logs[k], k};
    DevBuf dpairs, dempty;
    if ((rc = upload_n(b, dpairs, pairs.data(), n)) || (rc = reserve_n<pt_log_desc>(dempty, n))) return rc;
    PT_CUDA(cudaMemsetAsync(dempty.p, 0, (size_t)n * sizeof(pt_log_desc), b->stream));
    ptx::ExchangeParams P{};
    P.pairs = (const pt_exchange_pair*)dpairs.p; P.n_pairs = n;
    P.slot_off = (const unsigned long long*)dslot.p; P.dlv = (ptct::Delivered*)ddlv.p; P.totals = (ptct::PairTotals*)dtot.p;
    Delta D;
    if ((rc = gather_delta(b, P, tot.data(), (const pt_log_desc*)dempty.p, nullptr, D))) return rc;
    // ---- the new batch: the resident logs, then one log per request (a request that is not OK has zero totals) ----
    std::vector<uint32_t> from(nn), tables_from(nn);
    std::vector<pt_log_desc> nd(nn), dd(nn, pt_log_desc{});
    std::vector<pt_change_desc> ncd(nn), dcd(nn, pt_change_desc{});
    uint64_t io = 0, mo = 0, co = 0, po = 0;
    for (uint32_t i = 0; i < nn; i++) {
        const bool old = i < n0;
        const uint32_t s = old ? i : logs[i - n0];
        const pt_log_desc S = b->h_desc[s];
        const pt_change_desc CS = b->h_cdesc[s];
        from[i] = old ? i : PT_SELECT_ADDED; tables_from[i] = s;
        pt_log_desc L = S;
        pt_change_desc LC = CS;
        if (!old) {
            const uint32_t k = i - n0;
            const ptct::PairTotals& t = tot[k];
            const ptct::PairBase& B = D.base[k];
            status_out[k] = t.status;
            L = pt_log_desc{B.insdel, B.mark, t.n_insdel, t.n_mark, S.n_actors, S.max_ctr};
            LC = pt_change_desc{B.change, B.dep, t.n_changes, t.n_deps};
            dd[i] = L; dcd[i] = LC;
        }
        nd[i] = pt_log_desc{io, mo, L.n_insdel, L.n_mark, L.n_actors, L.max_ctr};
        ncd[i] = pt_change_desc{co, po, LC.n_changes, LC.n_deps};
        io += L.n_insdel; mo += L.n_mark; co += LC.n_changes; po += LC.n_deps;
    }
    // ---- splice: the delta as added logs behind the kept ones, and the sources' actor tables ----
    const pt_packed_ops delta{nn, dd.data(), (const pt_insdel_rec*)D.insdel.p, D.n_ins, (const pt_mark_rec*)D.marks.p, D.n_mk};
    const pt_change_table dch{nn, dcd.data(), (const pt_change_rec*)D.changes.p, D.n_ch, (const pt_dep_rec*)D.deps.p, D.n_dp};
    NewActorTables T;
    if (b->have_actors && (rc = gather_actor_tables(b, tables_from.data(), nn, nullptr, std::vector<uint32_t>(nn, ~0u), T))) return rc;
    if ((rc = splice(b, fn, std::move(nd), std::move(ncd), b->adm_maxR, &delta, true, pt_append_remap{}, from.data(), &dch, true, true))) return rc;
    if (b->have_actors) install_actor_tables(b, T);
    return PT_OK;
}

int pt_batch_download_clocks(pt_batch* b, const uint64_t** off, const uint32_t** seq, const uint32_t** status) {
    if (!b || !off || !seq || !status) { g_last_error = "pt_batch_download_clocks: null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_download_clocks before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = "pt_batch_download_clocks: the handle has no change table"; return PT_ERR_STATE; }
    const uint32_t n = b->n_logs;
    int rc;
    if ((rc = reserve_n<uint64_t>(b->h_clk_off, (uint64_t)n + 1)) || (rc = reserve_n<uint32_t>(b->h_clk_status, n))) return rc;
    uint64_t* hoff = (uint64_t*)b->h_clk_off.p;
    hoff[0] = 0;
    for (uint32_t i = 0; i < n; i++) hoff[i + 1] = hoff[i] + b->h_desc[i].n_actors;
    if ((rc = reserve_n<uint32_t>(b->h_clk_seq, hoff[n]))) return rc;
    PT_CUDA(cudaSetDevice(b->device));
    if (n) {
        DevBuf doff, dseq, dst;                              // freed on return
        if ((rc = upload_n(b, doff, hoff, (uint64_t)n + 1)) || (rc = reserve_n<uint32_t>(dseq, hoff[n])) || (rc = reserve_n<uint32_t>(dst, n))) return rc;
        ptck::clocks_kernel<<<warp_grid(b, n, 128), 128, 0, b->stream>>>((const pt_change_desc*)b->d_cdesc.p, (const pt_change_rec*)b->d_changes.p,
                                                                         (const pt_log_desc*)b->d_desc.p, n, (const unsigned long long*)doff.p,
                                                                         (uint32_t*)dseq.p, (uint32_t*)dst.p);
        PT_CUDA(launched(b));
        if (hoff[n]) PT_CUDA(cudaMemcpyAsync(b->h_clk_seq.p, dseq.p, hoff[n] * 4, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->h_clk_status.p, dst.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    *off = hoff; *seq = (const uint32_t*)b->h_clk_seq.p; *status = (const uint32_t*)b->h_clk_status.p;
    return PT_OK;
}

int pt_batch_download_descs(pt_batch* b, const pt_log_desc** out) {
    if (!b || !out) { g_last_error = "pt_batch_download_descs: null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = "pt_batch_download_descs before pt_batch_upload"; return PT_ERR_STATE; }
    *out = b->h_desc.data();
    return PT_OK;
}

static int enqueue_merge(pt_batch* b) {
    DevCounters* c = counters(b);
    PT_CUDA(cudaMemsetAsync(c, 0, sizeof(DevCounters), b->stream));   // stats, cursors and queue heads in one shot
    ptk::BatchParams P{};
    P.desc = (const pt_log_desc*)b->d_desc.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.key_insdel = (const uint32_t*)b->d_key_insdel.p; P.key_marks = (const uint2*)b->d_key_marks.p;
    P.results = (pt_log_result*)b->d_results.p;
    P.text_off = (const uint64_t*)b->d_text_off.p; P.span_off = (const uint64_t*)b->d_span_off.p;
    P.text = (uint32_t*)b->d_text.p; P.spans = (pt_span*)b->d_spans.p;
    P.comment_pool = (uint32_t*)b->d_pool.p; P.comment_used = &c->comment_used; P.comment_cap = b->plan.pool_cap;
    P.slab = (char*)b->d_slab.p;
    P.slab_counter = c->slab; P.slab_slots = b->plan.slab_slots;
    P.seq = (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) ? (uint32_t*)b->d_seq.p : nullptr;
    P.stats = c->stats;
    P.admit = nullptr;
    int rc;
    if (b->have_changes && b->n_logs) {
        if ((rc = launch_actor_kernel(b, ptadm::admit_kernel, b->n_logs,     // admission pre-pass
                                      (const pt_change_desc*)b->d_cdesc.p, (const pt_change_rec*)b->d_changes.p, (const pt_dep_rec*)b->d_deps.p,
                                      (const pt_log_desc*)b->d_desc.p, b->n_logs, b->adm_maxR, (uint32_t*)b->d_admit.p, (pt_log_result*)b->d_results.p)))
            return rc;
        P.admit = (const uint32_t*)b->d_admit.p;
    }
    { const char* e = getenv("PT_PREFETCH"); P.prefetch_next = e ? (uint32_t)atoi(e) : 0u; }
    { const char* e = getenv("PT_WARP_FLAGS"); P.warp_flags = e ? (uint32_t)atoi(e) : 0x704u; }   // default: phase-aligned rounds (bit 2), the in-log phase barriers 2-4 skipped (bits 8-10: measured), no extra L2 prefetch
    { const char* e = getenv("PT_TMA"); P.use_tma = e ? (uint32_t)atoi(e) : 1u; }
    // ascending bins; a log whose working set does not fit bin k's shared memory is deferred (on the device) to bin k+1;
    // only the last bin can spill to the global slab
    // The CTA-per-log bins' own lists do not depend on the warp / team kernels: when both exist they are launched on a side
    // stream (fork / join, also inside the captured graph) and fill the SMs the warp kernel's tail leaves idle.  The deferral
    // launches come after the join, in ascending bin order.
    const uint32_t* bin_first = b->plan.bin_first;
    const bool have0 = bin_first[1] > bin_first[0], haveBlocks = bin_first[kNumBins] > bin_first[1];
    const bool fork = have0 && haveBlocks && b->side != nullptr;
    if (fork) {
        PT_CUDA(cudaEventRecord(b->ev_fork, b->stream));
        PT_CUDA(cudaStreamWaitEvent(b->side, b->ev_fork, 0));
        b->launch_stream = b->side;
        for (int k = 1; k < kNumBins; k++) if ((rc = launch_bin(b, k, P, false))) { b->launch_stream = b->stream; return rc; }
        PT_CUDA(cudaEventRecord(b->ev_join, b->side));
        b->launch_stream = b->stream;
        if ((rc = launch_bin(b, 0, P, false))) return rc;
        PT_CUDA(cudaStreamWaitEvent(b->stream, b->ev_join, 0));
        for (int k = 1; k < kNumBins; k++) if ((rc = launch_bin(b, k, P, true))) return rc;
    } else {
        bool lower = false;
        for (int k = 0; k < kNumBins; k++) {
            if ((rc = launch_bin(b, k, P, false))) return rc;
            if (k > 0 && lower && (rc = launch_bin(b, k, P, true))) return rc;
            lower = lower || bin_first[k + 1] > bin_first[k];
        }
    }
    if ((b->limits.flags & PT_FLAG_EMIT_PATCHES) && b->n_logs) {
        ptk::PatchParams Q{};
        Q.desc = P.desc; Q.insdel = P.insdel; Q.marks = P.marks; Q.results = P.results; Q.text_off = P.text_off; Q.seq = P.seq;
        Q.first_op = (const uint32_t*)b->d_patch_first.p;
        Q.n_logs = b->n_logs; Q.smem_bytes = b->plan.patch_smem;
        Q.recs = (pt_patch_rec*)b->d_patch_recs.p; Q.items = (pt_patch_item*)b->d_patch_items.p;
        Q.item_cursor = &c->patch_items; Q.item_cap = b->patch_cap;
        Q.status = (uint32_t*)b->d_patch_status.p;
        const bool large = (b->limits.flags & PT_FLAG_EMIT_LARGE_PATCHES) && !b->plan.large_cand.empty();
        const bool warp = !(b->limits.flags & PT_FLAG_EMIT_LARGE_PATCHES) || b->plan.cfg.patch_warp_on;
        if (warp) {
            PT_CUDA(cudaFuncSetAttribute(ptk::patch_logs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b->plan.patch_smem));
            const uint32_t per_sm = std::clamp<uint32_t>((227u * 1024u) / (b->plan.patch_smem + 1024u), 1, 32);
            const uint32_t grid = (uint32_t)std::min<uint64_t>(b->n_logs, (uint64_t)b->num_sms * per_sm);
            ptk::patch_logs_kernel<<<grid, 32, b->plan.patch_smem, b->stream>>>(Q);
            PT_CUDA(launched(b));
        }
        if (large) {   // the logs the warp kernel declined (or, with PT_PATCH_WARP=0, every log)
            ptk::LargePatchParams G{};
            G.desc = Q.desc; G.insdel = Q.insdel; G.marks = Q.marks; G.results = Q.results; G.text_off = Q.text_off; G.seq = Q.seq;
            G.first_op = Q.first_op;
            G.cand = (const uint32_t*)b->d_large_cand.p; G.n_cand = (uint32_t)b->plan.large_cand.size(); G.after_warp = warp;
            G.scratch = (char*)b->d_large_scratch.p; G.slot_bytes = b->plan.large_bytes;
            G.recs = Q.recs; G.items = Q.items; G.item_cursor = Q.item_cursor; G.item_cap = Q.item_cap; G.status = Q.status;
            ptk::patch_large_kernel<<<b->plan.large_slots, ptk::kLargeThreads, 0, b->stream>>>(G);
            PT_CUDA(launched(b));
        }
    }
    return PT_OK;
}

int pt_batch_merge(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_merge before pt_batch_upload"; return PT_ERR_STATE; }
    PT_CUDA(cudaSetDevice(b->device));
    // The launch sequence of a batch is fixed: capture it once into a CUDA graph (not possible on the legacy default
    // stream, where the launches are simply enqueued directly).
    if (!b->graph_tried && b->merges_since_upload >= 1) {   // a batch merged more than once: replay its launch sequence as a graph
        b->graph_tried = true;
        if (b->stream != nullptr) {
            const uint64_t l0 = b->launches;
            if (cudaStreamBeginCapture(b->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
                int rc = enqueue_merge(b);
                cudaGraph_t g = nullptr;
                cudaError_t e = cudaStreamEndCapture(b->stream, &g);
                if (rc == PT_OK && e == cudaSuccess && g && cudaGraphInstantiate(&b->graph_exec, g, 0) == cudaSuccess) {
                    b->graph_ok = true; b->kernels_per_merge = (uint32_t)(b->launches - l0);
                }
                if (g) cudaGraphDestroy(g);
                b->launches = l0;
            }
            cudaGetLastError();
        }
    }
    PT_CUDA(cudaEventRecord(b->ev0, b->stream));
    if (b->graph_ok) {
        PT_CUDA(cudaGraphLaunch(b->graph_exec, b->stream));
        b->launches += b->kernels_per_merge;
    } else {
        int rc = enqueue_merge(b);
        if (rc) return rc;
    }
    PT_CUDA(cudaEventRecord(b->ev1, b->stream));
    b->merged = true; b->merges_since_upload++; b->dl_begun = false; b->patch_pool_changed = false; b->patch_window_changed = false;
    return PT_OK;
}

int pt_batch_sync(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    return PT_OK;
}

float pt_batch_last_merge_ms(pt_batch* b) {
    if (!b || !b->merged) return -1.f;
    if (cudaEventSynchronize(b->ev1) != cudaSuccess) return -1.f;
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, b->ev0, b->ev1) != cudaSuccess) return -1.f;
    return ms;
}

int pt_batch_download_results(pt_batch* b, pt_log_result* out, uint32_t n_logs) {
    if (!b || (!out && n_logs)) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    if (n_logs > b->n_logs) return PT_ERR_INVALID;
    int rc;
    if ((rc = reserve_n<pt_log_result>(b->h_results, b->n_logs))) return rc;
    if (n_logs) PT_CUDA(cudaMemcpyAsync(b->h_results.p, b->d_results.p, (size_t)n_logs * sizeof(pt_log_result), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    if (n_logs) memcpy(out, b->h_results.p, (size_t)n_logs * sizeof(pt_log_result));
    return PT_OK;
}

// Pack the outputs on the device (see the compaction kernels above) and enqueue the device -> host copies of the per-log
// headers, the packed offsets and the comment-pool cursor (asynchronous, pinned destinations); pt_batch_download then
// waits, learns the packed sizes and copies exactly the used tokens / spans / comment ids.  Lets a caller overlap one
// handle's download with another handle's upload / merge.
int pt_batch_download_begin(pt_batch* b) {
    if (!b) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    int rc;
    const size_t n = b->n_logs;
    if ((rc = reserve_n<pt_log_result>(b->h_results, n))) return rc;
    if ((rc = b->h_ctoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->h_csoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->h_misc.reserve(16))) return rc;
    if ((rc = b->d_ctoff.reserve((n + 1) * 8))) return rc;
    if ((rc = b->d_csoff.reserve((n + 1) * 8))) return rc;
    // packed outputs can never exceed the capacities; sized once per batch
    if ((rc = reserve_n<uint32_t>(b->d_ctext, b->plan.n_text))) return rc;
    if ((rc = reserve_n<pt_span>(b->d_cspans, b->plan.n_span))) return rc;
    PT_CUDA(cudaMemcpyAsync(b->h_misc.p, &counters(b)->comment_used, 8, cudaMemcpyDeviceToHost, b->stream));   // pool cursor = the batch's demand
    if (n) {
        const pt_log_result* res = (const pt_log_result*)b->d_results.p;
        unsigned long long *toff = (unsigned long long*)b->d_ctoff.p, *soff = (unsigned long long*)b->d_csoff.p;
        if ((rc = scan_offsets(b, pts::MergedCounts{res}, (uint32_t)n, b->d_bsum, toff, soff))) return rc;
        pts::out_gather_kernel<<<warp_grid(b, n, 256), 256, 0, b->stream>>>(res, (uint32_t)n, (const uint64_t*)b->d_text_off.p, (const uint64_t*)b->d_span_off.p,
                                                                       toff, soff, (const uint32_t*)b->d_text.p, (const pt_span*)b->d_spans.p,
                                                                       (uint32_t*)b->d_ctext.p, (pt_span*)b->d_cspans.p);
        PT_CUDA(launched(b));
        PT_CUDA(cudaMemcpyAsync(b->h_results.p, b->d_results.p, n * sizeof(pt_log_result), cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->h_ctoff.p, b->d_ctoff.p, (n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(b->h_csoff.p, b->d_csoff.p, (n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    } else {
        ((uint64_t*)b->h_ctoff.p)[0] = 0; ((uint64_t*)b->h_csoff.p)[0] = 0;
    }
    if (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) {
        if ((rc = reserve_n<uint32_t>(b->h_seq, b->plan.n_text))) return rc;
        if (b->plan.n_text) PT_CUDA(cudaMemcpyAsync(b->h_seq.p, b->d_seq.p, b->plan.n_text * 4, cudaMemcpyDeviceToHost, b->stream));
    }
    b->dl_begun = true;
    return PT_OK;
}

int pt_batch_download(pt_batch* b, pt_spans_view* out) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    int rc;
    if (!b->dl_begun && (rc = pt_batch_download_begin(b))) return rc;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const bool want_seq = (b->limits.flags & PT_FLAG_EMIT_SEQUENCE) != 0;
    const size_t n = b->n_logs;
    const uint64_t demand = *(unsigned long long*)b->h_misc.p;
    const uint64_t used = std::min<uint64_t>(demand, b->plan.pool_cap);
    const uint64_t n_ctext = ((const uint64_t*)b->h_ctoff.p)[n], n_cspan = ((const uint64_t*)b->h_csoff.p)[n];
    b->pool_used_host = used;
    if ((rc = reserve_n<uint32_t>(b->h_pool, used))) return rc;
    if ((rc = reserve_n<uint32_t>(b->h_text, n_ctext))) return rc;
    if ((rc = reserve_n<pt_span>(b->h_spans, n_cspan))) return rc;
    if (n_ctext) PT_CUDA(cudaMemcpyAsync(b->h_text.p, b->d_ctext.p, n_ctext * 4, cudaMemcpyDeviceToHost, b->stream));
    if (n_cspan) PT_CUDA(cudaMemcpyAsync(b->h_spans.p, b->d_cspans.p, n_cspan * sizeof(pt_span), cudaMemcpyDeviceToHost, b->stream));
    if (used) PT_CUDA(cudaMemcpyAsync(b->h_pool.p, b->d_pool.p, used * 4, cudaMemcpyDeviceToHost, b->stream));
    if (n_ctext || n_cspan || used) PT_CUDA(cudaStreamSynchronize(b->stream));
    out->n_logs = b->n_logs;
    out->results = (const pt_log_result*)b->h_results.p;
    out->text_off = (const uint64_t*)b->h_ctoff.p;
    out->span_off = (const uint64_t*)b->h_csoff.p;
    out->text = (const uint32_t*)b->h_text.p;
    out->spans = (const pt_span*)b->h_spans.p;
    out->comment_pool = (const uint32_t*)b->h_pool.p;
    out->comment_pool_used = used;
    out->seq = want_seq ? (const uint32_t*)b->h_seq.p : nullptr;
    out->seq_off = want_seq ? b->plan.text_off.data() : nullptr;
    out->comment_pool_needed = demand;                  // the cursor counts past the capacity
    return PT_OK;
}

int pt_batch_download_patches(pt_batch* b, pt_patch_view* out) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "download before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_PATCHES)) { g_last_error = "the handle was created without PT_FLAG_EMIT_PATCHES"; return PT_ERR_STATE; }
    if (b->patch_window_changed) { g_last_error = "pt_batch_download_patches: the patch window was set after the last merge; merge again"; return PT_ERR_STATE; }
    int rc;
    if ((rc = b->h_patch_misc.reserve(16))) return rc;
    if ((rc = reserve_n<pt_patch_rec>(b->h_patch_recs, b->n_insdel))) return rc;
    if ((rc = reserve_n<uint32_t>(b->h_patch_status, b->n_logs))) return rc;
    PT_CUDA(cudaMemcpyAsync(b->h_patch_misc.p, &counters(b)->patch_items, 8, cudaMemcpyDeviceToHost, b->stream));
    if (b->n_insdel) PT_CUDA(cudaMemcpyAsync(b->h_patch_recs.p, b->d_patch_recs.p, b->n_insdel * sizeof(pt_patch_rec), cudaMemcpyDeviceToHost, b->stream));
    if (b->n_logs) PT_CUDA(cudaMemcpyAsync(b->h_patch_status.p, b->d_patch_status.p, (size_t)b->n_logs * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t demand = *(unsigned long long*)b->h_patch_misc.p, used = std::min<uint64_t>(demand, b->patch_cap);
    if ((rc = reserve_n<pt_patch_item>(b->h_patch_items, used))) return rc;
    if (used) { PT_CUDA(cudaMemcpyAsync(b->h_patch_items.p, b->d_patch_items.p, used * sizeof(pt_patch_item), cudaMemcpyDeviceToHost, b->stream)); PT_CUDA(cudaStreamSynchronize(b->stream)); }
    out->recs = (const pt_patch_rec*)b->h_patch_recs.p; out->items = (const pt_patch_item*)b->h_patch_items.p;
    out->n_items = used; out->n_items_needed = demand; out->status = (const uint32_t*)b->h_patch_status.p;
    return PT_OK;
}

int pt_batch_set_patch_pool(pt_batch* b, uint64_t items) {
    if (!b || items > 0xFFFFFFFFull) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->limits.patch_pool_items = (uint32_t)items;
    if (b->have_batch && items && (b->limits.flags & PT_FLAG_EMIT_PATCHES)) {
        b->patch_cap = items;
        b->patch_pool_changed = b->merged;
        int rc;
        if ((rc = b->d_patch_items.reserve(b->patch_cap * sizeof(pt_patch_item)))) return rc;
        drop_graph(b);                                   // the item pool pointer / capacity are baked in
    }
    return PT_OK;
}

// The window lives in d_patch_first, allocated with the batch, so the captured merge graph reads whichever window is set.
int pt_batch_set_patch_window(pt_batch* b, const uint32_t* first_op, uint32_t n_logs) {
    static const char* fn = "pt_batch_set_patch_window";
    if (!b) return PT_ERR_INVALID;
    if (!(b->limits.flags & PT_FLAG_EMIT_PATCHES)) { g_last_error = std::string(fn) + ": the handle was created without PT_FLAG_EMIT_PATCHES"; return PT_ERR_STATE; }
    if (!b->have_batch) { g_last_error = std::string(fn) + " before pt_batch_upload"; return PT_ERR_STATE; }
    if (n_logs != b->n_logs) {
        g_last_error = std::string(fn) + ": n_logs is " + std::to_string(n_logs) + ", the batch has " + std::to_string(b->n_logs);
        return PT_ERR_INVALID;
    }
    if (first_op) {
        for (uint32_t i = 0; i < n_logs; i++) {
            const uint64_t ops = (uint64_t)b->h_desc[i].n_insdel + b->h_desc[i].n_mark;
            if (first_op[i] > ops) {
                g_last_error = std::string(fn) + ": log " + std::to_string(i) + ": first_op " + std::to_string(first_op[i]) + " > its " +
                               std::to_string(ops) + " list ops";
                return PT_ERR_INVALID;
            }
        }
    }
    if (!n_logs) return PT_OK;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));           // the staging buffer of an earlier call may still be in flight
    if (first_op) {
        int rc;
        if ((rc = b->h_patch_first.reserve((size_t)n_logs * 4))) return rc;
        memcpy(b->h_patch_first.p, first_op, (size_t)n_logs * 4);
        PT_CUDA(cudaMemcpyAsync(b->d_patch_first.p, b->h_patch_first.p, (size_t)n_logs * 4, cudaMemcpyHostToDevice, b->stream));
    } else {
        PT_CUDA(cudaMemsetAsync(b->d_patch_first.p, 0, (size_t)n_logs * 4, b->stream));
    }
    b->patch_window_changed = b->merged;
    return PT_OK;
}

int pt_batch_query_elements(pt_batch* b, const pt_elem_query* queries, uint32_t n, uint32_t* out) {
    return run_queries(b, "pt_batch_query_elements", "query", queries, n, out, [&](uint32_t grid, uint32_t threads, const pt_elem_query* dq, uint32_t* da) {
        ptq::query_elements_kernel<<<grid, threads, 0, b->stream>>>(dq, n, (const pt_log_result*)b->d_results.p, (const uint64_t*)b->d_text_off.p,
                                                                   (const uint32_t*)b->d_seq.p, b->n_logs, da);
    });
}

int pt_batch_find_elements(pt_batch* b, const pt_elem_ref* refs, uint32_t n, pt_elem_pos* out) {
    return run_queries(b, "pt_batch_find_elements", "find", refs, n, out, [&](uint32_t grid, uint32_t threads, const pt_elem_ref* dq, pt_elem_pos* da) {
        ptq::find_elements_kernel<<<grid, threads, 0, b->stream>>>(dq, n, (const pt_log_desc*)b->d_desc.p, b->dp_insdel, (const pt_log_result*)b->d_results.p,
                                                                  (const uint64_t*)b->d_text_off.p, (const uint32_t*)b->d_seq.p, b->n_logs, da);
    });
}

int pt_batch_attribute(pt_batch* b, const uint32_t* logs, uint32_t n, const uint64_t* clock_off, const pt_clock_entry* clock, pt_attr_view* out) {
    const char* fn = "pt_batch_attribute: ";
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_attribute before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = std::string(fn) + "the handle has no change table"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = std::string(fn) + "the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    if (!b->merged) { g_last_error = "attribute before merge"; return PT_ERR_STATE; }
    if (!out || (n && !logs)) { g_last_error = std::string(fn) + "null logs or out"; return PT_ERR_INVALID; }
    const std::string err = check_clock_requests(b, logs, n, clock_off, clock);
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    int rc;
    if ((rc = reserve_n<uint32_t>(b->h_attr_status, n)) || (rc = reserve_n<uint64_t>(b->h_attr_off, (uint64_t)n + 1)) ||
        (rc = reserve_n<pt_attr_run>(b->h_attr_runs, 0))) return rc;
    uint64_t* hoff = (uint64_t*)b->h_attr_off.p;
    hoff[0] = 0;
    if (!n) { *out = pt_attr_view{0, (const uint32_t*)b->h_attr_status.p, hoff, (const pt_attr_run*)b->h_attr_runs.p, 0}; return PT_OK; }
    std::vector<unsigned long long> chg_slot((size_t)n + 1, 0), rec_slot((size_t)n + 1, 0);
    for (uint32_t k = 0; k < n; k++) {
        chg_slot[k + 1] = chg_slot[k] + b->h_cdesc[logs[k]].n_changes;
        rec_slot[k + 1] = rec_slot[k] + b->h_desc[logs[k]].n_insdel;
    }
    const uint64_t nc = chg_slot[n], nr = rec_slot[n];
    PT_CUDA(cudaSetDevice(b->device));
    // ---- resolve: each request's table checks, each record's change, each element's attributed delete ----
    DevBuf dlogs, dcoff, dclk, dcs, drs, dfirst, dcov, dchg, ddchg, ddcov, ddkey, dtab, dst, dcnt, dbsum, doff, druns;   // freed on return
    if ((rc = upload_n(b, dlogs, logs, n)) || (rc = upload_n(b, dcs, chg_slot.data(), (uint64_t)n + 1)) ||
        (rc = upload_n(b, drs, rec_slot.data(), (uint64_t)n + 1)) || (rc = reserve_n<uint32_t>(dfirst, nc)) || (rc = reserve_n<uint32_t>(dcov, nc)) ||
        (rc = reserve_n<uint32_t>(dchg, nr)) || (rc = reserve_n<uint32_t>(ddchg, nr)) || (rc = reserve_n<uint32_t>(ddcov, nr)) ||
        (rc = reserve_n<unsigned long long>(ddkey, nr)) || (rc = reserve_n<uint32_t>(dtab, 2 * nr)) || (rc = reserve_n<uint32_t>(dst, n)) ||
        (rc = reserve_n<unsigned long long>(dcnt, n)) || (rc = reserve_n<unsigned long long>(doff, (uint64_t)n + 1))) return rc;
    if (clock_off && ((rc = upload_n(b, dcoff, clock_off, (uint64_t)n + 1)) || (rc = upload_n(b, dclk, clock, clock_off[n])))) return rc;
    pta::AttrParams P{};
    P.logs = (const uint32_t*)dlogs.p; P.n = n; P.maxR = b->adm_maxR;
    P.clock_off = clock_off ? (const unsigned long long*)dcoff.p : nullptr; P.clock = clock_off ? (const pt_clock_entry*)dclk.p : nullptr;
    P.desc = (const pt_log_desc*)b->d_desc.p; P.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    P.changes = (const pt_change_rec*)b->d_changes.p; P.deps = (const pt_dep_rec*)b->d_deps.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.res = (const pt_log_result*)b->d_results.p; P.seq_off = (const uint64_t*)b->d_text_off.p; P.seq = (const uint32_t*)b->d_seq.p;
    P.chg_slot = (const unsigned long long*)dcs.p; P.rec_slot = (const unsigned long long*)drs.p;
    P.first = (uint32_t*)dfirst.p; P.cov = (uint32_t*)dcov.p;
    P.chg = (uint32_t*)dchg.p; P.dchg = (uint32_t*)ddchg.p; P.dcov = (uint32_t*)ddcov.p; P.dkey = (unsigned long long*)ddkey.p; P.table = (uint32_t*)dtab.p;
    P.status = (uint32_t*)dst.p; P.count = (unsigned long long*)dcnt.p; P.off = (const unsigned long long*)doff.p;
    if ((rc = launch_actor_kernel(b, pta::attribute_resolve_kernel, n, P))) return rc;
    // ---- count, scan, one total back, write ----
    const uint32_t threads = 128, grid = warp_grid(b, n, threads);
    pta::attribute_runs_kernel<false><<<grid, threads, 0, b->stream>>>(P);
    PT_CUDA(launched(b));
    if ((rc = scan_offsets(b, pts::PlainCounts{P.count}, n, dbsum, (unsigned long long*)doff.p, nullptr))) return rc;
    PT_CUDA(cudaMemcpyAsync(hoff, doff.p, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(b->h_attr_status.p, dst.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t total = hoff[n];
    if ((rc = reserve_n<pt_attr_run>(druns, total)) || (rc = reserve_n<pt_attr_run>(b->h_attr_runs, total))) return rc;
    if (total) {
        P.runs = (pt_attr_run*)druns.p;
        pta::attribute_runs_kernel<true><<<grid, threads, 0, b->stream>>>(P);
        PT_CUDA(launched(b));
        PT_CUDA(cudaMemcpyAsync(b->h_attr_runs.p, druns.p, total * sizeof(pt_attr_run), cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
    }
    *out = pt_attr_view{n, (const uint32_t*)b->h_attr_status.p, hoff, (const pt_attr_run*)b->h_attr_runs.p, total};
    return PT_OK;
}

// pt_batch_restore's host checks of the requests (include/peritext_b200.h).  Returns the problem, or an empty string.
static std::string check_restore(const pt_batch* b, const pt_restore_request* req, uint32_t n) {
    std::vector<char> target(b->n_logs, 0);
    for (uint32_t k = 0; k < n; k++) {
        const pt_restore_request& q = req[k];
        const std::string here = "request " + std::to_string(k) + ": ";
        if (q.log >= b->n_logs || q.version >= b->n_logs)
            return here + "log " + std::to_string(q.log >= b->n_logs ? q.log : q.version) + " is outside the batch's " + std::to_string(b->n_logs) + " logs";
        if (target[q.log]) return here + "log " + std::to_string(q.log) + " is the log of an earlier request";
        target[q.log] = 1;
        const pt_log_desc& L = b->h_desc[q.log];
        if (q.actor >= L.n_actors) return here + "actor rank " + std::to_string(q.actor) + " >= the log's " + std::to_string(L.n_actors) + " actors";
        if (q.first_ctr <= L.max_ctr) return here + "first_ctr " + std::to_string(q.first_ctr) + " is not above the log's max_ctr " + std::to_string(L.max_ctr);
    }
    return std::string();
}

int pt_batch_restore(pt_batch* b, const pt_restore_request* req, uint32_t n, uint32_t mode, pt_restore_view* out) {
    const char* fn = "pt_batch_restore: ";
    if (!b) return PT_ERR_INVALID;
    if (!b->have_batch) { g_last_error = "pt_batch_restore before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = std::string(fn) + "the handle has no change table"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_SEQUENCE)) { g_last_error = std::string(fn) + "the handle was created without PT_FLAG_EMIT_SEQUENCE"; return PT_ERR_STATE; }
    if (!b->merged) { g_last_error = std::string(fn) + "no completed merge since the last call that changed the batch"; return PT_ERR_STATE; }
    if (!out || (n && !req)) { g_last_error = std::string(fn) + "null requests or out"; return PT_ERR_INVALID; }
    if (mode != PT_RESTORE_TEXT && mode != PT_RESTORE_MARKS) { g_last_error = std::string(fn) + "mode " + std::to_string(mode) + " is not exactly one of PT_RESTORE_TEXT, PT_RESTORE_MARKS"; return PT_ERR_INVALID; }
    const std::string err = check_restore(b, req, n);
    if (!err.empty()) { g_last_error = fn + err; return PT_ERR_INVALID; }
    int rc;
    if ((rc = reserve_n<uint32_t>(b->h_rst_status, n)) || (rc = reserve_n<uint32_t>(b->h_rst_ops, n)) || (rc = reserve_n<uint32_t>(b->h_rst_seq, n))) return rc;
    uint32_t *hst = (uint32_t*)b->h_rst_status.p, *hops = (uint32_t*)b->h_rst_ops.p, *hseq = (uint32_t*)b->h_rst_seq.p;
    *out = pt_restore_view{n, hst, hops, hseq};
    if (!n) return PT_OK;
    const bool marks = mode == PT_RESTORE_MARKS;
    std::vector<unsigned long long> slot((size_t)n + 1, 0), vis((size_t)n + 1, 0), open((size_t)n + 1, 0);
    for (uint32_t k = 0; k < n; k++) {
        slot[k + 1] = slot[k] + b->h_cdesc[req[k].log].n_changes;
        vis[k + 1] = vis[k] + (marks ? b->h_desc[req[k].log].n_insdel : 0);   // n_visible <= n_insdel
        open[k + 1] = open[k] + (marks ? 2ull * ((uint64_t)b->h_desc[req[k].log].n_mark + b->h_desc[req[k].version].n_mark) : 0);
    }
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));              // the merge is complete; the view's buffers are free
    // ---- count: statuses, ops, deps, seq and element totals back to the host ----
    DevBuf dreq, dslot, dpos, dvoff, dvis, dooff, dopen, dst, dops, ddeps, dseq, delems, ddesc, dcdesc, dins, dmk, dch, ddp;   // freed on return
    if ((rc = upload_n(b, dreq, req, n)) || (rc = upload_n(b, dslot, slot.data(), (uint64_t)n + 1)) || (rc = reserve_n<uint32_t>(dpos, slot[n])) ||
        (rc = reserve_n<uint32_t>(dst, n)) || (rc = reserve_n<uint32_t>(dops, n)) || (rc = reserve_n<uint32_t>(ddeps, n)) ||
        (rc = reserve_n<uint32_t>(dseq, n)) || (rc = reserve_n<uint32_t>(delems, n)) || (rc = upload_n(b, dvoff, vis.data(), (uint64_t)n + 1)) ||
        (rc = reserve_n<uint32_t>(dvis, vis[n])) || (rc = upload_n(b, dooff, open.data(), (uint64_t)n + 1)) || (rc = reserve_n<uint4>(dopen, open[n]))) return rc;
    ptrs::RestoreParams P{};
    P.req = (const pt_restore_request*)dreq.p; P.n = n; P.maxR = b->adm_maxR;
    P.desc = (const pt_log_desc*)b->d_desc.p; P.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    P.changes = (const pt_change_rec*)b->d_changes.p; P.deps = (const pt_dep_rec*)b->d_deps.p;
    P.insdel = b->dp_insdel; P.marks = b->dp_marks;
    P.res = (const pt_log_result*)b->d_results.p; P.seq_off = (const uint64_t*)b->d_text_off.p; P.seq = (const uint32_t*)b->d_seq.p;
    P.mode = mode;
    P.text_off = (const uint64_t*)b->d_text_off.p; P.text = (const uint32_t*)b->d_text.p;
    P.span_off = (const uint64_t*)b->d_span_off.p; P.spans = (const pt_span*)b->d_spans.p; P.cpool = (const uint32_t*)b->d_pool.p;
    P.slot_off = (const unsigned long long*)dslot.p; P.pos = (uint32_t*)dpos.p;
    P.vis_off = (const unsigned long long*)dvoff.p; P.vis = (uint32_t*)dvis.p; P.open_off = (const unsigned long long*)dooff.p; P.open = (uint4*)dopen.p;
    P.status = (uint32_t*)dst.p; P.n_ops = (uint32_t*)dops.p; P.n_deps = (uint32_t*)ddeps.p; P.seq_out = (uint32_t*)dseq.p; P.elems = (uint32_t*)delems.p;
    if ((rc = launch_actor_kernel(b, ptrs::restore_kernel<false>, n, P))) return rc;
    std::vector<uint32_t> nd(n), el(n);
    PT_CUDA(cudaMemcpyAsync(hst, dst.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(hops, dops.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(hseq, dseq.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(nd.data(), ddeps.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(el.data(), delems.p, (size_t)n * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    // ---- the limits that depend on the counts, and the delta's layout: records, one change record and its deps per log ----
    const uint32_t nl = b->n_logs;
    std::vector<pt_log_desc> dd(nl);
    std::vector<pt_change_desc> cd(nl, pt_change_desc{0, 0, 0, 0});
    for (uint32_t i = 0; i < nl; i++) dd[i] = pt_log_desc{0, 0, 0, 0, b->h_desc[i].n_actors, b->h_desc[i].max_ctr};
    for (uint32_t k = 0; k < n; k++) {
        if (!hops[k]) continue;
        const pt_restore_request& q = req[k];
        const std::string here = std::string(fn) + "request " + std::to_string(k) + ": ";
        const uint64_t last = (uint64_t)q.first_ctr + hops[k] - 1;
        if (last > 0xFFFFFFFFull) { g_last_error = here + "counters past 2^32 - 1"; return PT_ERR_INVALID; }
        if (last * std::max<uint32_t>(1, b->h_desc[q.log].n_actors) > 0x7FFFFFFFull) { g_last_error = here + "max_ctr x n_actors would reach 2^31"; return PT_ERR_INVALID; }
        if (el[k] >= (1u << 22)) { g_last_error = here + "the change would bring the log to 2^22 elements or more"; return PT_ERR_INVALID; }
        (marks ? dd[q.log].n_mark : dd[q.log].n_insdel) = hops[k];
        dd[q.log].max_ctr = (uint32_t)last;
        cd[q.log].n_changes = 1; cd[q.log].n_deps = nd[k];
    }
    uint64_t n_ins = 0, n_mk = 0, n_ch = 0, n_dp = 0;
    for (uint32_t i = 0; i < nl; i++) {
        dd[i].insdel_off = n_ins; dd[i].mark_off = n_mk; cd[i].change_off = n_ch; cd[i].dep_off = n_dp;
        n_ins += dd[i].n_insdel; n_mk += dd[i].n_mark; n_ch += cd[i].n_changes; n_dp += cd[i].n_deps;
    }
    // ---- write, then pt_batch_append's splice with the delta and its change table on the device ----
    if ((rc = upload_n(b, ddesc, dd.data(), nl)) || (rc = upload_n(b, dcdesc, cd.data(), nl)) || (rc = reserve_n<pt_insdel_rec>(dins, n_ins)) ||
        (rc = reserve_n<pt_mark_rec>(dmk, n_mk)) || (rc = reserve_n<pt_change_rec>(dch, n_ch)) || (rc = reserve_n<pt_dep_rec>(ddp, n_dp))) return rc;
    if (n_ch) {
        P.delta = (const pt_log_desc*)ddesc.p; P.delta_cdesc = (const pt_change_desc*)dcdesc.p;
        P.out_insdel = (pt_insdel_rec*)dins.p; P.out_marks = (pt_mark_rec*)dmk.p; P.out_changes = (pt_change_rec*)dch.p; P.out_deps = (pt_dep_rec*)ddp.p;
        if ((rc = launch_actor_kernel(b, ptrs::restore_kernel<true>, n, P))) return rc;
    }
    const pt_packed_ops delta{nl, dd.data(), (const pt_insdel_rec*)dins.p, n_ins, (const pt_mark_rec*)dmk.p, n_mk};
    const pt_change_table ct{nl, cd.data(), (const pt_change_rec*)dch.p, n_ch, (const pt_dep_rec*)ddp.p, n_dp};
    return splice_append(b, fn, &delta, true, pt_append_remap{}, &ct, true);
}

// JSON render of the spans (render_kernel.cuh).
int pt_batch_render_json(pt_batch* b, const pt_json_pools* pools, pt_json_view* out) {
    if (!b || !pools || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "render before merge"; return PT_ERR_STATE; }
    ptr::JsonPools P{};
    int rc;
    if ((rc = load_json_pools(b, pools, "pt_batch_render_json", &P))) return rc;
    const pt_log_result* res = (const pt_log_result*)b->d_results.p;
    const uint64_t *toff = (const uint64_t*)b->d_text_off.p, *soff = (const uint64_t*)b->d_span_off.p;
    const uint32_t* text = (const uint32_t*)b->d_text.p;
    const pt_span* spans = (const pt_span*)b->d_spans.p;
    const uint32_t* cpool = (const uint32_t*)b->d_pool.p;
    const uint32_t n = b->n_logs;
    return render_passes(b, "pt_batch_render_json", b->spans_json,
        [&](uint32_t grid, uint32_t threads, unsigned long long* sizes, unsigned long long* miss) {
            ptr::json_size_kernel<<<grid, threads, 0, b->stream>>>(res, n, toff, soff, text, spans, cpool, P, sizes, miss);
        },
        [&](uint32_t grid, uint32_t threads, const unsigned long long* off, uint8_t* bytes) {
            ptr::json_write_kernel<<<grid, threads, 0, b->stream>>>(res, n, toff, soff, text, spans, cpool, P, off, bytes);
        }, out);
}

// JSON render of the Patch stream (patch_json_kernel.cuh): check the item demand, order the item pool by owner and key
// (count, scan, scatter, rank), then the same passes as the span render.
int pt_batch_render_patches_json(pt_batch* b, const pt_json_pools* pools, pt_json_view* out) {
    static const char* fn = "pt_batch_render_patches_json";
    if (!b || !pools || !out) return PT_ERR_INVALID;
    if (!b->merged) { g_last_error = "render before merge"; return PT_ERR_STATE; }
    if (!(b->limits.flags & PT_FLAG_EMIT_PATCHES)) { g_last_error = "the handle was created without PT_FLAG_EMIT_PATCHES"; return PT_ERR_STATE; }
    if (b->patch_pool_changed) { g_last_error = std::string(fn) + ": the patch pool was replaced after the last merge; merge again"; return PT_ERR_STATE; }
    if (b->patch_window_changed) { g_last_error = std::string(fn) + ": the patch window was set after the last merge; merge again"; return PT_ERR_STATE; }
    ptr::JsonPools P{};
    int rc;
    if ((rc = load_json_pools(b, pools, fn, &P))) return rc;
    const uint32_t n = b->n_logs;
    ptr::PatchJsonIn I{};
    if (n) {
        if ((rc = b->h_patch_misc.reserve(16))) return rc;
        PT_CUDA(cudaMemcpyAsync(b->h_patch_misc.p, &counters(b)->patch_items, 8, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
        const uint64_t items = *(unsigned long long*)b->h_patch_misc.p, owners = b->n_insdel + b->n_mark;
        if (items > b->patch_cap) {
            g_last_error = std::string(fn) + ": the last merge needs " + std::to_string(items) + " patch items and the pool holds " +
                           std::to_string(b->patch_cap) + "; call pt_batch_set_patch_pool(" + std::to_string(items) + ") and merge again";
            return PT_ERR_STATE;
        }
        if (owners >= 0xFFFFFFFFull) { g_last_error = std::string(fn) + ": more than 2^32 - 2 op records"; return PT_ERR_INVALID; }
        const uint32_t no = (uint32_t)owners;
        if ((rc = reserve_n<uint64_t>(b->d_picnt, owners)) || (rc = b->d_piseg.reserve((owners + 1) * 8)) ||
            (rc = reserve_n<pt_patch_item>(b->d_pitmp, items)) || (rc = reserve_n<uint2>(b->d_pisorted, items))) return rc;
        unsigned long long *cnt = (unsigned long long*)b->d_picnt.p, *seg = (unsigned long long*)b->d_piseg.p;
        const pt_log_desc* desc = (const pt_log_desc*)b->d_desc.p;
        const pt_patch_item* pool = (const pt_patch_item*)b->d_patch_items.p;
        pt_patch_item* tmp = (pt_patch_item*)b->d_pitmp.p;
        uint2* sorted = (uint2*)b->d_pisorted.p;
        if (no) {
            const uint32_t threads = 256, grid = warp_grid(b, items, threads, 1);     // one thread per item
            PT_CUDA(cudaMemsetAsync(cnt, 0, owners * 8, b->stream));
            if (items) {
                ptr::pitem_count_kernel<<<grid, threads, 0, b->stream>>>(pool, items, desc, b->n_insdel, cnt);
                PT_CUDA(launched(b));
            }
            if ((rc = scan_offsets(b, pts::PlainCounts{cnt}, no, b->d_pibsum, seg, nullptr))) return rc;
            if (items) {
                ptr::pitem_scatter_kernel<<<grid, threads, 0, b->stream>>>(pool, items, desc, b->n_insdel, cnt, seg, tmp);
                PT_CUDA(launched(b));
                ptr::pitem_rank_kernel<<<grid, threads, 0, b->stream>>>(tmp, items, desc, b->n_insdel, seg, sorted);
                PT_CUDA(launched(b));
            }
        } else {
            PT_CUDA(cudaMemsetAsync(seg, 0, 8, b->stream));
        }
        I.desc = desc; I.insdel = b->dp_insdel; I.marks = b->dp_marks; I.res = (const pt_log_result*)b->d_results.p;
        I.recs = (const pt_patch_rec*)b->d_patch_recs.p; I.pstatus = (const uint32_t*)b->d_patch_status.p;
        I.seg = seg; I.items = sorted; I.n_insdel = b->n_insdel; I.first_op = (const uint32_t*)b->d_patch_first.p;
    }
    return render_passes(b, fn, b->patches_json,
        [&](uint32_t grid, uint32_t threads, unsigned long long* sizes, unsigned long long* miss) {
            ptr::patches_json_size_kernel<<<grid, threads, 0, b->stream>>>(I, n, P, sizes, miss);
        },
        [&](uint32_t grid, uint32_t threads, const unsigned long long* off, uint8_t* bytes) {
            ptr::patches_json_write_kernel<<<grid, threads, 0, b->stream>>>(I, n, P, off, bytes);
        }, out);
}

// pt_batch_render_changes_json's host checks of the requests, the string pools and the extras (include/peritext_b200.h).  On
// success slot_off holds each request's scratch slot (exclusive scan of its log's n_changes).  Returns the problem, or "".
static std::string check_changes_json(const pt_batch* b, const pt_changes_json_input& in, std::vector<unsigned long long>& slot_off) {
    const uint32_t n = b->n_logs, nr = in.n_requests;
    auto req = [](uint32_t r) { return "request " + std::to_string(r) + ": "; };
    if (!in.requests) return "null requests";
    if (in.n_clock && !in.clock) return "null clock with a nonzero n_clock";
    if (!in.actors_first || !in.actors_off || !in.counters_first || !in.list_ids_off) return "null actor, counter or list-id pool";
    if (in.n_extras && !in.extras) return "null extras with a nonzero n_extras";
    if (in.n_extra_ops && (!in.extra_ops || !in.extra_ops_off)) return "null extra-ops pool with a nonzero count";
    for (uint32_t i = 0; i < n; i++) {
        if (in.actors_first[i + 1] < in.actors_first[i] || in.counters_first[i + 1] < in.counters_first[i] || in.list_ids_off[i + 1] < in.list_ids_off[i])
            return at(i) + "a pool's per-log offsets decrease";
        if ((in.list_ids_off[i + 1] - in.list_ids_off[i]) & 1) return at(i) + "the list id is not UTF-16LE (odd byte count)";
    }
    if (in.actors_first[0] != 0 || in.counters_first[0] != 0) return "the actor and counter ranges must start at entry 0";
    if (in.counters_first[n] && !in.counters) return "null counter pool with a nonzero count";
    if (in.actors_first[n] && !in.actors) return "null actor pool with a nonzero count";
    for (uint64_t k = 0; k < in.actors_first[n]; k++)
        if (in.actors_off[k + 1] < in.actors_off[k] || ((in.actors_off[k + 1] - in.actors_off[k]) & 1)) return "actor pool entry " + std::to_string(k) + " is not UTF-16LE";
    for (uint64_t k = 0; k < in.n_extra_ops; k++)
        if (in.extra_ops_off[k + 1] < in.extra_ops_off[k]) return "extra-ops offsets decrease";
    slot_off.assign((size_t)nr + 1, 0);
    for (uint32_t r = 0; r < nr; r++) {
        const pt_changes_request& q = in.requests[r];
        if (q.log >= n) return req(r) + "log " + std::to_string(q.log) + " is outside the batch's " + std::to_string(n) + " logs";
        if (q.mode != PT_CHANGES_RANGE && q.mode != PT_CHANGES_MISSING) return req(r) + "unknown mode " + std::to_string(q.mode);
        if (q.mode == PT_CHANGES_MISSING) {
            if (q.clock_off > in.n_clock || q.n_clock > in.n_clock - q.clock_off) return req(r) + "the clock range is outside the clock array";
            for (uint32_t k = 0; k < q.n_clock; k++)
                if (in.clock[q.clock_off + k].actor >= b->h_desc[q.log].n_actors)
                    return req(r) + "clock entry " + std::to_string(k) + " names actor " + std::to_string(in.clock[q.clock_off + k].actor) + " and log " +
                           std::to_string(q.log) + " has " + std::to_string(b->h_desc[q.log].n_actors) + " actors";
        }
        slot_off[r + 1] = slot_off[r] + b->h_cdesc[q.log].n_changes;
    }
    for (uint64_t e = 0; e < in.n_extras; e++) {
        const pt_change_extra& x = in.extras[e];
        const std::string ex = "extra " + std::to_string(e) + ": ";
        if (x.log >= n || x.change >= b->h_cdesc[x.log].n_changes) return ex + "log " + std::to_string(x.log) + " has no change " + std::to_string(x.change);
        if (x.op != PT_EXTRA_NONE && x.op >= in.n_extra_ops) return ex + "op " + std::to_string(x.op) + " is outside the extra-ops pool";
        if (e == 0) continue;
        const pt_change_extra& p = in.extras[e - 1];
        if (p.log > x.log || (p.log == x.log && p.change > x.change)) return ex + "the extras are not sorted by (log, change, pos)";
        if (p.log == x.log && p.change == x.change) {
            if (p.pos >= x.pos) return ex + "the extras are not sorted by (log, change, pos)";
            if (p.start_op != x.start_op) return ex + "a different start_op than the change's other extras";
            if (p.op == PT_EXTRA_NONE || x.op == PT_EXTRA_NONE) return ex + "a PT_EXTRA_NONE entry beside another entry of the change";
        }
    }
    return std::string();
}

// JSON render of Change objects (changes_json_kernel.cuh): select, then the item passes.
int pt_batch_render_changes_json(pt_batch* b, const pt_changes_json_input* in, pt_changes_json_view* out) {
    static const char* fn = "pt_batch_render_changes_json";
    if (!b || !in || !out) { g_last_error = std::string(fn) + ": null argument"; return PT_ERR_INVALID; }
    if (!b->have_batch) { g_last_error = std::string(fn) + " before pt_batch_upload"; return PT_ERR_STATE; }
    if (!b->have_changes) { g_last_error = std::string(fn) + ": the handle has no change table"; return PT_ERR_STATE; }
    const uint32_t nr = in->n_requests, n = b->n_logs;
    JsonBufs& J = b->changes_json;
    int rc;
    if ((rc = J.hoff.reserve(((size_t)nr + 1) * 8)) || (rc = J.hbytes.reserve(1)) || (rc = J.hmisc.reserve(32)) ||
        (rc = reserve_n<uint32_t>(b->h_cj_status, nr))) return rc;
    uint64_t* hoff = (uint64_t*)J.hoff.p;
    uint32_t* hstatus = (uint32_t*)b->h_cj_status.p;
    if (!nr) {
        PT_CUDA(cudaSetDevice(b->device));
        PT_CUDA(cudaStreamSynchronize(b->stream));          // the pinned view buffers may still be the target of an earlier copy
        hoff[0] = 0;
        *out = pt_changes_json_view{0, hoff, (const char*)J.hbytes.p, 0, hstatus};
        return PT_OK;
    }
    std::vector<unsigned long long> slot_off;
    std::string err = check_changes_json(b, *in, slot_off);
    if (!err.empty()) { g_last_error = std::string(fn) + ": " + err; return PT_ERR_INVALID; }
    ptr::JsonPools P{};
    if ((rc = load_json_pools(b, &in->pools, fn, &P))) return rc;
    PT_CUDA(cudaStreamSynchronize(b->stream));
    // the requests, the string pools, the extras and the select kernel's scratch: freed on return
    DevBuf dreq, dclock, dact, dactoff, dactfirst, dctr, dctrfirst, dlid, dlidoff, dx, dxops, dxoff, dslot, dpos, dsel, dnsel, dstat, ditems, dbad,
           ditemoff, dbsum, dsizes, dboff, doff, dmiss, dbytes;
    const uint64_t n_slot = slot_off[nr], n_act = in->actors_first[n], n_ctr = in->counters_first[n];
    const uint64_t act_bytes = n_act ? in->actors_off[n_act] : 0, lid_bytes = in->list_ids_off[n], xop_bytes = in->n_extra_ops ? in->extra_ops_off[in->n_extra_ops] : 0;
    if ((rc = upload_n(b, dreq, in->requests, nr)) || (rc = upload_n(b, dclock, in->clock, in->n_clock)) ||
        (rc = upload_n(b, dact, in->actors, act_bytes)) || (rc = upload_n(b, dactoff, in->actors_off, n_act + 1)) ||
        (rc = upload_n(b, dactfirst, in->actors_first, (uint64_t)n + 1)) || (rc = upload_n(b, dctr, in->counters, n_ctr)) ||
        (rc = upload_n(b, dctrfirst, in->counters_first, (uint64_t)n + 1)) || (rc = upload_n(b, dlid, in->list_ids, lid_bytes)) ||
        (rc = upload_n(b, dlidoff, in->list_ids_off, (uint64_t)n + 1)) || (rc = upload_n(b, dx, in->extras, in->n_extras)) ||
        (rc = upload_n(b, dxops, in->extra_ops, xop_bytes)) || (rc = upload_n(b, dxoff, in->extra_ops_off, in->n_extra_ops ? in->n_extra_ops + 1 : 0)) ||
        (rc = upload_n(b, dslot, slot_off.data(), (uint64_t)nr + 1)) || (rc = reserve_n<uint32_t>(dpos, n_slot)) ||
        (rc = reserve_n<ptcj::Sel>(dsel, n_slot)) || (rc = reserve_n<uint32_t>(dnsel, nr)) || (rc = reserve_n<uint32_t>(dstat, nr)) ||
        (rc = reserve_n<unsigned long long>(ditems, nr)) || (rc = reserve_n<unsigned long long>(dbad, 2)) ||
        (rc = reserve_n<unsigned long long>(ditemoff, (uint64_t)nr + 1)) || (rc = reserve_n<unsigned long long>(dmiss, 2)) ||
        (rc = reserve_n<unsigned long long>(doff, (uint64_t)nr + 1))) return rc;
    ptcj::ChangesParams C{};
    C.req = (const pt_changes_request*)dreq.p; C.n_req = nr; C.maxR = b->adm_maxR; C.clock = (const pt_clock_entry*)dclock.p;
    C.desc = (const pt_log_desc*)b->d_desc.p; C.cdesc = (const pt_change_desc*)b->d_cdesc.p;
    C.changes = (const pt_change_rec*)b->d_changes.p; C.deps = (const pt_dep_rec*)b->d_deps.p;
    C.insdel = b->dp_insdel; C.marks = b->dp_marks;
    C.slot_off = (const unsigned long long*)dslot.p; C.pos = (uint32_t*)dpos.p; C.sel = (ptcj::Sel*)dsel.p;
    C.n_sel = (uint32_t*)dnsel.p; C.status = (uint32_t*)dstat.p; C.items = (unsigned long long*)ditems.p;
    C.extras = (const pt_change_extra*)dx.p; C.n_extras = in->n_extras; C.bad = (unsigned long long*)dbad.p;
    C.item_off = (const unsigned long long*)ditemoff.p;
    C.actors = (const uint8_t*)dact.p; C.actors_off = (const unsigned long long*)dactoff.p; C.actors_first = (const unsigned long long*)dactfirst.p;
    C.counters = (const unsigned long long*)dctr.p; C.counters_first = (const unsigned long long*)dctrfirst.p;
    C.list_ids = (const uint8_t*)dlid.p; C.list_ids_off = (const unsigned long long*)dlidoff.p;
    C.xops = (const uint8_t*)dxops.p; C.xops_off = (const unsigned long long*)dxoff.p;
    unsigned long long* bad = (unsigned long long*)dbad.p;
    unsigned long long* miss = (unsigned long long*)dmiss.p;
    PT_CUDA(cudaMemsetAsync(bad, 0xFF, 16, b->stream));
    if ((rc = launch_actor_kernel(b, ptcj::changes_select_kernel, nr, C))) return rc;
    if ((rc = scan_offsets(b, pts::PlainCounts{C.items}, nr, dbsum, (unsigned long long*)ditemoff.p, nullptr))) return rc;
    // read-back 1: the item count and the select kernel's findings
    uint64_t* hm = (uint64_t*)J.hmisc.p;
    PT_CUDA(cudaMemcpyAsync(hm, (unsigned long long*)ditemoff.p + nr, 8, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaMemcpyAsync(hm + 1, bad, 16, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    const uint64_t n_items = hm[0];
    for (int k = 0; k < 2; k++)
        if (hm[1 + k] != ~0ull) {
            g_last_error = std::string(fn) + ": log " + std::to_string(hm[1 + k] >> 32) + " change " + std::to_string(hm[1 + k] & 0xFFFFFFFFull) +
                           (k == 0 ? " has neither list ops nor extras, so nothing gives its startOp" : ": its extras' positions lie past the change's ops");
            return PT_ERR_INVALID;
        }
    if (n_items >= 0xFFFFFFFFull) { g_last_error = std::string(fn) + ": more than 2^32 - 2 work items"; return PT_ERR_INVALID; }
    C.n_items = n_items;
    uint64_t total = 0;
    if (n_items) {
        if ((rc = reserve_n<unsigned long long>(dsizes, n_items)) || (rc = reserve_n<unsigned long long>(dboff, n_items + 1))) return rc;
        unsigned long long *sizes = (unsigned long long*)dsizes.p, *boff = (unsigned long long*)dboff.p;
        const uint32_t threads = 128, grid = warp_grid(b, n_items, threads);
        PT_CUDA(cudaMemsetAsync(miss, 0xFF, 16, b->stream));
        ptcj::changes_json_size_kernel<<<grid, threads, 0, b->stream>>>(C, P, sizes, miss, miss + 1);
        PT_CUDA(launched(b));
        if ((rc = scan_offsets(b, pts::PlainCounts{sizes}, (uint32_t)n_items, dbsum, boff, nullptr))) return rc;
        ptcj::changes_offsets_kernel<<<warp_grid(b, (uint64_t)nr + 1, 256, 1), 256, 0, b->stream>>>(C.item_off, boff, nr, (unsigned long long*)doff.p);
        PT_CUDA(launched(b));
        // read-back 2: the byte total and the missing pool entries
        PT_CUDA(cudaMemcpyAsync(hm, boff + n_items, 8, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaMemcpyAsync(hm + 1, miss, 16, cudaMemcpyDeviceToHost, b->stream));
        PT_CUDA(cudaStreamSynchronize(b->stream));
        total = hm[0];
        if (hm[1] != ~0ull) {
            static const char* kinds[3] = {"value", "link", "comment"};
            g_last_error = std::string(fn) + ": log " + std::to_string(hm[1] >> 34) + " names " + kinds[(hm[1] >> 32) & 3] + " pool entry " +
                           std::to_string(hm[1] & 0xFFFFFFFFull) + ", which the caller's pools do not hold";
            return PT_ERR_INVALID;
        }
        if (hm[2] != ~0ull) {
            g_last_error = std::string(fn) + ": log " + std::to_string(hm[2] >> 34) + " names " + ((hm[2] >> 32) & 3 ? "counter" : "actor") + " " +
                           std::to_string(hm[2] & 0xFFFFFFFFull) + ", which the caller's " + ((hm[2] >> 32) & 3 ? "counter" : "actor") + " pool does not hold";
            return PT_ERR_INVALID;
        }
        if ((rc = reserve_n<uint8_t>(J.bytes, total)) || (rc = reserve_n<uint8_t>(J.hbytes, total))) return rc;
        ptcj::changes_json_write_kernel<<<grid, threads, 0, b->stream>>>(C, P, boff, (uint8_t*)J.bytes.p);
        PT_CUDA(launched(b));
        PT_CUDA(cudaMemcpyAsync(hoff, doff.p, ((size_t)nr + 1) * 8, cudaMemcpyDeviceToHost, b->stream));
        if (total) PT_CUDA(cudaMemcpyAsync(J.hbytes.p, J.bytes.p, total, cudaMemcpyDeviceToHost, b->stream));
    } else {
        memset(hoff, 0, ((size_t)nr + 1) * 8);              // every request failed: zero bytes each
    }
    PT_CUDA(cudaMemcpyAsync(hstatus, dstat.p, (size_t)nr * 4, cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    *out = pt_changes_json_view{nr, hoff, (const char*)J.hbytes.p, total, hstatus};
    return PT_OK;
}

int pt_batch_device_results(pt_batch* b, void** dev_ptr, uint32_t* n_logs) {
    if (!b || !dev_ptr) return PT_ERR_INVALID;
    if (!b->have_batch) return PT_ERR_STATE;
    *dev_ptr = b->d_results.p;
    if (n_logs) *n_logs = b->n_logs;
    return PT_OK;
}

uint64_t pt_batch_launch_count(const pt_batch* b) { return b ? b->launches : 0; }

int pt_batch_stats(pt_batch* b, uint64_t out[4]) {
    if (!b || !out) return PT_ERR_INVALID;
    if (!b->merged) return PT_ERR_STATE;
    DevCounters h;
    PT_CUDA(cudaMemcpyAsync(&h, b->d_counters.p, sizeof(h), cudaMemcpyDeviceToHost, b->stream));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    for (int i = 0; i < 3; i++) out[i] = h.stats[i];
    out[3] = h.comment_used;                             // comment-pool entries the batch needs
    return PT_OK;
}

#ifdef PT_PHASE_CLOCKS
// Profiling build only (make PHASE_CLOCKS=1): the warp kernel's per-phase cycle sums on the current device, summed over
// its warps since the last reset: out[0..8] = log start, A+B, C, D, E, F, G, I, round wait; out[9] = logs merged.
int pt_phase_clocks(uint64_t out[ptk::kNumPhases + 1], int reset) {
    if (!out) return PT_ERR_INVALID;
    PT_CUDA(cudaDeviceSynchronize());
    PT_CUDA(cudaMemcpyFromSymbol(out, ptk::ptk_phase_clk, sizeof(ptk::ptk_phase_clk)));
    if (reset) {
        static const unsigned long long zero[ptk::kNumPhases + 1] = {};
        PT_CUDA(cudaMemcpyToSymbol(ptk::ptk_phase_clk, zero, sizeof(zero)));
    }
    return PT_OK;
}
#endif

int pt_batch_set_comment_pool(pt_batch* b, uint64_t entries) {
    if (!b) return PT_ERR_INVALID;
    PT_CUDA(cudaSetDevice(b->device));
    PT_CUDA(cudaStreamSynchronize(b->stream));
    b->limits.comment_pool_entries = entries;
    if (b->have_batch && entries) {
        b->plan.pool_cap = entries;
        int rc;
        if ((rc = reserve_n<uint32_t>(b->d_pool, b->plan.pool_cap))) return rc;
        drop_graph(b);                                   // the pool pointer / capacity are baked in
    }
    return PT_OK;
}

void pt_batch_destroy(pt_batch* b) {
    if (!b) return;
    cudaSetDevice(b->device);
    cudaStreamSynchronize(b->stream);
    if (b->side) cudaStreamDestroy(b->side);
    if (b->ev_fork) cudaEventDestroy(b->ev_fork);
    if (b->ev_join) cudaEventDestroy(b->ev_join);
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    drop_graph(b);
    delete b;
}

const char* pt_strerror(int status) {
    switch (status) {
        case PT_OK: return "ok";
        case PT_ERR_INVALID: return "invalid argument";
        case PT_ERR_CUDA: return "CUDA runtime error";
        case PT_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (no CPU fallback)";
        case PT_ERR_STATE: return "call out of order";
        case PT_ERR_NOMEM: return "out of memory";
        default: return "unknown status";
    }
}
const char* pt_last_error(void) { return g_last_error.c_str(); }
const char* pt_version(void) { return "peritext_b200 0.1 (sm_90a)"; }

}  // extern "C"
