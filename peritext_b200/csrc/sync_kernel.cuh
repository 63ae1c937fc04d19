// sync_kernel.cuh — the device side of pt_batch_sync_pairs (include/peritext_b200.h): the exchange maps and the actor growth of
// pt_batch_exchange derived from the handle's actor tables (pt_batch_upload_actors) instead of the caller's.
//
// Actor tables: per log, its actor ids in rank order as UTF-16LE strings (the PT_POOL_ACTORS layout: bytes, absolute byte
// offsets [count + 1], per-log first id [n_logs + 1]).  Ranks follow JS string order (UTF-16 code units), so a name is found
// by bisection (js_cmp) and two tables join by name without a hash.
//
// sync_derive_kernel: one warp per pair.  Shared memory per warp, two words per src/dst rank (actor_shape's budget):
//   1. clocks: ptct::count_clock over dst's change table by dst rank into A, ptct::source_clock over src's by src rank into B
//      (with the list-op positions); a table that fails the checks leaves the pair to the exchange, which reports BAD_TABLE.
//   2. have: B[r] = A[dst rank of src rank r's name] (0 without one): dst's clock keyed by actor NAME.  A becomes a bitmap over
//      src ranks.
//   3. missing set: src's changes with seq > B[actor].  Each marks its actor and its deps' actors in the bitmap; its records
//      (ptct::change_records; records that do not fit leave the pair to the exchange too) are read by the whole warp,
//      marking the actor of every id whose counter is non-zero, and giving the top opId counter and the op count.
//   4. growth: the marked src names dst lacks, compacted in rank (= name) order into the pair's slot; their count and bytes,
//      whether the first sorts before dst's last name (dst's ranks move), and the DENSE test of the grown dst.
// actor_merge_kernel: one warp per log.  Each output id gets its new rank (old rank + the new names before it, or index among
// the new names + the old names before it), its length and source into scratch; a warp scan turns the lengths into the new
// table's byte offsets; then each lane copies one id.  A log that moves writes its old -> new rank map.
// sync_maps_kernel: one warp per pair, src rank -> dst rank of the same name in the grown tables (0xFFFF without one).
// add_select_kernel (pt_batch_add_actors): one warp per log sorts and deduplicates the caller's ids for it by counting, per id,
// the distinct ids before it (O(m^2) compares: a log names few ids per call, and a long list is slower but exact), and keeps the
// ones the table lacks; actor_merge_kernel then merges them in.  add_ranks_kernel: each given id's rank in the grown table.
// actor_gather_kernel (pt_batch_select_logs): one warp per new log copies its ids' bytes and rebased offsets from the old
// tables or the added ones.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"
#include "change_table.cuh"

namespace pty {

// JS string order (compareOpIds / Array.sort's default) of two UTF-16LE strings of byte lengths na, nb: code unit by code
// unit, then the shorter first.  Returns <0, 0, >0.
__device__ __forceinline__ int js_cmp(const uint8_t* a, uint32_t na, const uint8_t* b, uint32_t nb) {
    const uint32_t n = min(na, nb) >> 1;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t x = a[2 * i] | (uint32_t)a[2 * i + 1] << 8, y = b[2 * i] | (uint32_t)b[2 * i + 1] << 8;
        if (x != y) return x < y ? -1 : 1;
    }
    return na < nb ? -1 : na > nb ? 1 : 0;
}

struct Tables {
    const uint8_t* data; const unsigned long long* off; const unsigned long long* first;   // first: [n_logs + 1]
    __device__ __forceinline__ uint32_t count(uint32_t log) const { return (uint32_t)(first[log + 1] - first[log]); }
    __device__ __forceinline__ const uint8_t* name(uint32_t log, uint32_t r, uint32_t& len) const {
        const unsigned long long k = first[log] + r, o = off[k];
        len = (uint32_t)(off[k + 1] - o);
        return data + o;
    }
    // the number of log's names that sort before s (bisection); *found: one of them equals s
    __device__ __forceinline__ uint32_t lower_bound(uint32_t log, const uint8_t* s, uint32_t ns, bool* found) const {
        uint32_t lo = 0, hi = count(log);
        while (lo < hi) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            uint32_t len;
            const uint8_t* x = name(log, mid, len);
            if (js_cmp(x, len, s, ns) < 0) lo = mid + 1; else hi = mid;
        }
        if (found) {
            uint32_t len = 0;
            const uint8_t* x = lo < count(log) ? name(log, lo, len) : nullptr;
            *found = x && js_cmp(x, len, s, ns) == 0;
        }
        return lo;
    }
};

enum : uint32_t { kDeriveGrow = 0, kDeriveSkip = 1, kDeriveDense = PT_EXCHANGE_DENSE };

struct SyncTotals {           // 32 B per pair
    uint32_t verdict;         // kDeriveGrow, kDeriveSkip (tables the exchange refuses), kDeriveDense
    uint32_t n_new;           // src names dst lacks
    uint32_t moves;           // 1: the first new name sorts before dst's last, so dst's ranks move
    uint32_t top;             // the largest opId counter of the missing records
    unsigned long long new_bytes, n_ops;   // the new names' bytes; the missing records
};

struct DeriveParams {
    const pt_exchange_pair* pairs; uint32_t n_pairs; uint32_t maxR;
    Tables T;
    const pt_log_desc* desc; const pt_change_desc* cdesc; const pt_change_rec* changes; const pt_dep_rec* deps;
    const pt_insdel_rec* insdel; const pt_mark_rec* marks;
    const unsigned long long* slot_off;   // [n_pairs + 1] src's n_changes: the list-op positions
    uint32_t* pos;
    const unsigned long long* new_off;    // [n_pairs + 1] src's name count: the new names, as ids of the tables
    unsigned long long* new_id;
    SyncTotals* totals;
};

// A record id naming a rank >= R is not marked: it has no name to add.  (packing.sync_maps raises on such a record; here the
// exchange that follows finds no image for it and reports the pair PT_EXCHANGE_UNMAPPED, so both refuse the pair.)
__device__ __forceinline__ void mark_actor(uint32_t* bits, uint32_t a, uint32_t R) { if (a < R) atomicOr(&bits[a >> 5], 1u << (a & 31)); }

__global__ void sync_derive_kernel(DeriveParams P) {
    extern __shared__ uint32_t syn_smem[];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t* A = syn_smem + (size_t)wib * 2 * P.maxR;     // dst's clock by dst rank, then the bitmap over src ranks
    uint32_t* B = A + P.maxR;                               // src's clock by src rank, then dst's clock by src rank (name)
    for (uint32_t p = blockIdx.x * wpb + wib; p < P.n_pairs; p += gridDim.x * wpb) {
        const pt_exchange_pair pr = P.pairs[p];
        const pt_log_desc S = P.desc[pr.src], D = P.desc[pr.dst];
        const pt_change_desc CS = P.cdesc[pr.src], CD = P.cdesc[pr.dst];
        const uint32_t Rs = S.n_actors, Rd = D.n_actors, Ns = P.T.count(pr.src), Nd = P.T.count(pr.dst);
        for (uint32_t a = lane; a < Rd; a += 32) A[a] = 0;
        for (uint32_t a = lane; a < Rs; a += 32) B[a] = 0;
        __syncwarp();
        const pt_change_rec* c0 = P.changes + CS.change_off;
        const pt_dep_rec* d0 = P.deps + CS.dep_off;
        uint32_t* pos = P.pos + P.slot_off[p];
        bool ok = ptct::count_clock(P.changes + CD.change_off, CD.n_changes, CD.n_deps, Rd, A, nullptr, nullptr, lane) &&
                  ptct::source_clock(c0, CS, S, B, pos, lane);
        // ---- 2: dst's clock by src rank, through the names ----
        if (ok) {
            for (uint32_t r = lane; r < Rs; r += 32) {
                uint32_t have = 0;
                if (r < Ns) {
                    uint32_t len;
                    const uint8_t* s = P.T.name(pr.src, r, len);
                    bool found;
                    const uint32_t j = P.T.lower_bound(pr.dst, s, len, &found);
                    if (found && j < Rd) have = A[j];
                }
                B[r] = have;
            }
            __syncwarp();
            for (uint32_t w = lane; w < (Rs + 31) / 32; w += 32) A[w] = 0;
            __syncwarp();
        }
        // ---- 3: the missing set's named actors, top counter and records ----
        uint32_t top = 0;
        unsigned long long n_ops = 0;
        bool any = false, bad = false;
        const pt_insdel_rec* ins = P.insdel + S.insdel_off;
        const pt_mark_rec* mk = P.marks + S.mark_off;
        for (uint32_t base = 0; ok && base < CS.n_changes; base += 32) {
            const uint32_t k = base + lane;
            uint4 r = make_uint4(0, 0, 0, 0);
            if (k < CS.n_changes) r = __ldg(reinterpret_cast<const uint4*>(c0 + k));
            const bool miss = k < CS.n_changes && r.x > B[r.y & 0xFFFFu];
            ptct::Records x{};
            if (miss) {
                mark_actor(A, r.y & 0xFFFFu, Rs);
                for (uint32_t d = 0; d < (r.y >> 16); d++) {
                    const uint32_t da = d0[r.z + d].actor;
                    if (da >= Rs) bad = true; else mark_actor(A, da, Rs);
                }
                x = ptct::change_records(mk, S, pos[k], r.w);
                if (!x.fits) bad = true;
            }
            if (__any_sync(0xffffffffu, bad)) { ok = false; break; }
            // the whole warp reads each missing change's records in turn
            for (uint32_t todo = __ballot_sync(0xffffffffu, miss); todo; todo &= todo - 1) {
                const uint32_t src = __ffs(todo) - 1;
                const uint32_t il = __shfl_sync(0xffffffffu, x.ins_lo, src), in_ = __shfl_sync(0xffffffffu, x.n_insdel, src);
                const uint32_t ml = __shfl_sync(0xffffffffu, x.mk_lo, src), mn = __shfl_sync(0xffffffffu, x.n_mark, src);
                any = true;
                n_ops += (unsigned long long)in_ + mn;
                for (uint32_t i = lane; i < in_; i += 32) {
                    const pt_insdel_rec q = ins[il + i];
                    if (q.ctr) mark_actor(A, q.actor, Rs);
                    if (q.ref_ctr) mark_actor(A, q.ref_actor, Rs);
                    top = max(top, q.ctr);
                }
                for (uint32_t i = lane; i < mn; i += 32) {
                    const pt_mark_rec q = mk[ml + i];
                    if (q.ctr) mark_actor(A, q.actor, Rs);
                    if (q.start_ctr) mark_actor(A, q.start_actor, Rs);
                    if (q.end_ctr) mark_actor(A, q.end_actor, Rs);
                    top = max(top, q.ctr);
                }
            }
        }
        for (int o = 16; o > 0; o >>= 1) top = max(top, __shfl_xor_sync(0xffffffffu, top, o));
        __syncwarp();
        // ---- 4: the names dst lacks, in src rank order ----
        SyncTotals t{ok ? kDeriveGrow : kDeriveSkip, 0u, 0u, top, 0ull, n_ops};
        if (ok && any &&
            (unsigned long long)max(D.max_ctr, top) > 2ull * ((unsigned long long)D.n_insdel + D.n_mark + n_ops) + 16ull)   // packing._wants_dense
            t.verdict = kDeriveDense;
        if (t.verdict == kDeriveGrow && any) {
            unsigned long long* out = P.new_id + P.new_off[p];
            unsigned long long bytes = 0;
            uint32_t first_new = 0xFFFFFFFFu;
            for (uint32_t rb = 0; rb < Ns; rb += 32) {
                const uint32_t r = rb + lane;
                bool add = false;
                uint32_t len = 0;
                if (r < Ns && (A[r >> 5] >> (r & 31) & 1u)) {
                    const uint8_t* s = P.T.name(pr.src, r, len);
                    bool found;
                    P.T.lower_bound(pr.dst, s, len, &found);
                    add = !found;
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, add);
                if (add) { out[t.n_new + __popc(bal & lt)] = P.T.first[pr.src] + r; bytes += len; }
                if (bal && first_new == 0xFFFFFFFFu) first_new = rb + __ffs(bal) - 1;
                t.n_new += __popc(bal);
            }
            for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
            t.new_bytes = bytes;
            if (t.n_new && Nd && lane == 0) {
                uint32_t la, lb;
                const uint8_t* a = P.T.name(pr.src, first_new, la);
                const uint8_t* b = P.T.name(pr.dst, Nd - 1, lb);
                t.moves = js_cmp(a, la, b, lb) < 0;
            }
        }
        if (lane == 0) P.totals[p] = t;
        __syncwarp();
    }
}

struct MergeParams {
    uint32_t n_logs;
    Tables old_t;
    uint8_t* data; unsigned long long* off; const unsigned long long* first;   // the new tables; off[0] is set by the host
    const unsigned long long* byte_base;     // [n_logs] where log i's bytes start in data
    const uint32_t* grow;                    // [n_logs] log i's slot of new names, or 0xFFFFFFFF: none
    // the new names: slot g holds n_new[g] ids new_id[new_off[g] ..], in JS order, of the pool (new_data, new_byte_off)
    const uint8_t* new_data; const unsigned long long* new_byte_off;
    const unsigned long long* new_off; const unsigned long long* new_id; const uint32_t* n_new;
    const unsigned long long* map_off;       // [n_logs] where log i's old -> new rank map goes, or ~0ull: its ranks stay
    uint16_t* map;
    const uint8_t** src_at;                  // [new id count] scratch: each new id's bytes
};

__global__ void actor_merge_kernel(MergeParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < P.n_logs; i += nwarps) {
        const uint32_t m = P.old_t.count(i), g = P.grow[i];
        const uint32_t q = g == 0xFFFFFFFFu ? 0u : P.n_new[g];
        const unsigned long long* nid = g == 0xFFFFFFFFu ? nullptr : P.new_id + P.new_off[g];
        auto new_name = [&](uint32_t k, uint32_t& len) {
            const unsigned long long x = nid[k], o = P.new_byte_off[x];
            len = (uint32_t)(P.new_byte_off[x + 1] - o);
            return P.new_data + o;
        };
        const unsigned long long f = P.first[i];
        // each output id: its rank, length (into off[f + rank + 1]) and source bytes
        for (uint32_t r = lane; r < m + q; r += 32) {
            uint32_t len, t;
            const uint8_t* s;
            if (r < m) {
                s = P.old_t.name(i, r, len);
                uint32_t lo = 0, hi = q;                      // the new names that sort before old name r
                while (lo < hi) {
                    const uint32_t mid = lo + ((hi - lo) >> 1);
                    uint32_t l2;
                    const uint8_t* x = new_name(mid, l2);
                    if (js_cmp(x, l2, s, len) < 0) lo = mid + 1; else hi = mid;
                }
                t = r + lo;
                if (P.map_off[i] != ~0ull) P.map[P.map_off[i] + r] = (uint16_t)t;
            } else {
                s = new_name(r - m, len);
                t = (r - m) + P.old_t.lower_bound(i, s, len, nullptr);
            }
            P.off[f + t + 1] = len;
            P.src_at[f + t] = s;
        }
        __syncwarp();
        // lengths -> byte offsets
        unsigned long long run = P.byte_base[i];
        for (uint32_t rb = 0; rb < m + q; rb += 32) {
            const uint32_t r = rb + lane;
            const unsigned long long len = r < m + q ? P.off[f + r + 1] : 0ull;
            unsigned long long s = len;
            for (int d = 1; d < 32; d <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, s, d); if (lane >= (uint32_t)d) s += y; }
            if (r < m + q) P.off[f + r + 1] = run + s;
            run += __shfl_sync(0xffffffffu, s, 31);
        }
        __syncwarp();
        for (uint32_t r = lane; r < m + q; r += 32) {
            const unsigned long long lo = r ? P.off[f + r] : P.byte_base[i], hi = P.off[f + r + 1];
            const uint8_t* s = P.src_at[f + r];
            for (unsigned long long b = lo; b < hi; b++) P.data[b] = s[b - lo];
        }
    }
}

// pt_batch_select_logs: new log i's table is resident log from[i]'s, or (PT_SELECT_ADDED) the ids of the added tables from
// id add_first[i] on.  The host knows every log's id and byte counts, so first / byte_base (the new layout) come from it.
struct GatherParams {
    uint32_t n_logs;
    const uint32_t* from;
    Tables old_t;
    const uint8_t* add_data; const unsigned long long* add_off; const unsigned long long* add_first;   // add_first: [n_logs]
    uint8_t* data; unsigned long long* off;                      // the new tables; off[0] is set by the host
    const unsigned long long* first; const unsigned long long* byte_base;   // [n_logs + 1] each
};

__global__ void actor_gather_kernel(GatherParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < P.n_logs; i += nwarps) {
        const uint32_t s = P.from[i];
        const bool added = s == PT_SELECT_ADDED;
        const uint8_t* src = added ? P.add_data : P.old_t.data;
        const unsigned long long* so = (added ? P.add_off : P.old_t.off) + (added ? P.add_first[i] : P.old_t.first[s]);
        const unsigned long long f = P.first[i], cnt = P.first[i + 1] - f, b0 = so[0], nb = P.byte_base[i];
        for (unsigned long long r = lane; r < cnt; r += 32) P.off[f + r + 1] = so[r + 1] - b0 + nb;
        for (unsigned long long k = lane; k < P.byte_base[i + 1] - nb; k += 32) P.data[nb + k] = src[b0 + k];
    }
}

// pair p's actor map, src rank -> dst rank of the same name in the (grown) tables T: exactly src's n_actors entries
__global__ void sync_maps_kernel(const pt_exchange_pair* pairs, uint32_t n_pairs, Tables T, const pt_log_desc* desc,
                                 const unsigned long long* actor_off, uint16_t* actor_map) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t p = warp; p < n_pairs; p += nwarps) {
        const pt_exchange_pair pr = pairs[p];
        const uint32_t Rs = desc[pr.src].n_actors, Ns = T.count(pr.src);
        uint16_t* out = actor_map + actor_off[p];
        for (uint32_t r = lane; r < Rs; r += 32) {
            uint32_t img = 0xFFFFu;
            if (r < Ns) {
                uint32_t len;
                const uint8_t* s = T.name(pr.src, r, len);
                bool found;
                const uint32_t j = T.lower_bound(pr.dst, s, len, &found);
                if (found) img = j;
            }
            out[r] = (uint16_t)img;
        }
    }
}

// pt_batch_add_actors' ids: pool (data, byte offsets), log i's ids are first[i] .. first[i + 1], in any order.
struct AddParams {
    uint32_t n_logs;
    Tables T;                                 // the tables before the call
    const uint8_t* data; const unsigned long long* off; const unsigned long long* first;
    uint32_t* fresh;                          // [count] scratch: 1 = the first copy of an id the table lacks
    unsigned long long* new_id;               // [count] log i's new ids at first[i] .., in JS order
    SyncTotals* totals;                       // [n_logs] n_new, new_bytes, moves
};

__global__ void add_select_kernel(AddParams P) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    auto id = [&](unsigned long long k, uint32_t& len) { const unsigned long long o = P.off[k]; len = (uint32_t)(P.off[k + 1] - o); return P.data + o; };
    for (uint32_t i = warp; i < P.n_logs; i += nwarps) {
        const unsigned long long lo = P.first[i], hi = P.first[i + 1];
        for (unsigned long long k = lo + lane; k < hi; k += 32) {
            uint32_t len, l2;
            const uint8_t* s = id(k, len);
            bool fresh = true;
            for (unsigned long long j = lo; fresh && j < k; j++) { const uint8_t* x = id(j, l2); fresh = js_cmp(x, l2, s, len) != 0; }
            bool found = false;
            if (fresh) P.T.lower_bound(i, s, len, &found);
            P.fresh[k] = fresh && !found;
        }
        __syncwarp();
        uint32_t n_new = 0;
        unsigned long long bytes = 0;
        for (unsigned long long kb = lo; kb < hi; kb += 32) {
            const unsigned long long k = kb + lane;
            const bool mine = k < hi && P.fresh[k];
            if (mine) {
                uint32_t len, l2;
                const uint8_t* s = id(k, len);
                uint32_t before = 0;                  // the fresh ids that sort before it: its place among them
                for (unsigned long long j = lo; j < hi; j++) {
                    if (!P.fresh[j]) continue;
                    const uint8_t* x = id(j, l2);
                    before += js_cmp(x, l2, s, len) < 0;
                }
                P.new_id[lo + before] = k;
                bytes += len;
            }
            n_new += __popc(__ballot_sync(0xffffffffu, mine));
        }
        for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
        __syncwarp();
        if (lane == 0) {
            SyncTotals t{kDeriveGrow, n_new, 0u, 0u, bytes, 0ull};
            const uint32_t m = P.T.count(i);
            if (n_new && m) {
                uint32_t la, lb;
                const uint8_t* a = id(P.new_id[lo], la);
                const uint8_t* b = P.T.name(i, m - 1, lb);
                t.moves = js_cmp(a, la, b, lb) < 0;
            }
            P.totals[i] = t;
        }
        __syncwarp();
    }
}

// each given id's rank in log i's table T (the grown one)
__global__ void add_ranks_kernel(uint32_t n_logs, Tables T, const uint8_t* data, const unsigned long long* off, const unsigned long long* first, uint16_t* rank) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n_logs; i += nwarps)
        for (unsigned long long k = first[i] + lane; k < first[i + 1]; k += 32)
            rank[k] = (uint16_t)T.lower_bound(i, data + off[k], (uint32_t)(off[k + 1] - off[k]), nullptr);
}

}  // namespace pty
