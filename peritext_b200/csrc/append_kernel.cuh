// append_kernel.cuh — the device splice of pt_batch_append (include/peritext_b200.h).
//
// splice_records_kernel: one warp per log, grid-stride over the logs in x; a log with many records is shared by the
// gridDim.y warps of its slices (slice y takes every gridDim.y-th run of 32 records).  The log's old records are read from
// the resident batch with coalesced 16-byte loads, go through the log's id maps (actor rank, counter, and the batch's comment rank), and are written
// at the log's place in the new record buffers; the log's delta records follow them verbatim.  A 32-byte mark record is two
// 16-byte words, so lane pairs hold one mark: the even lane maps the opId and the counters of the boundaries, the odd lane
// the boundary actors and the attr, with the fields it needs from its partner by one shuffle.  A log whose maps are all
// identity is a straight copy.  splice_changes_kernel does the same for the change and dep tables (actor ranks only; the
// delta changes' dep_off moves past the log's old deps).
//
// Both kernels also run pt_batch_select_logs: `from` names the resident log each new log copies (nullptr: log i itself, as in
// an append; PT_SELECT_ADDED: none, so the log's records are all the delta's).  A select passes only the comment map.
#pragma once
#include <cstdint>

#include "../../include/peritext_b200.h"

namespace pta {

// The device copy of a pt_append_remap; a null map is the identity.
struct Remap {
    const unsigned long long* actor_off; const uint16_t* actor_map;
    const unsigned long long* ctr_off;  const uint32_t* ctr_map;
    const uint32_t* comment_map; unsigned long long n_comment;
};

// One log's maps: na / nc = 0 is the identity.  A value outside the domain becomes the all-ones value of its field, so a
// faulty record stays faulty.
struct LogMaps {
    const uint16_t* a; uint32_t na;
    const uint32_t* c; uint32_t nc;
    __device__ __forceinline__ uint32_t actor(uint32_t x) const { return na ? (x < na ? (uint32_t)__ldg(a + x) : 0xFFFFu) : x; }
    __device__ __forceinline__ uint32_t ctr(uint32_t x) const { return nc ? (x < nc ? __ldg(c + x) : 0xFFFFFFFFu) : x; }
    // the actor of an id whose (old) counter is ctr: counter 0 is HEAD / a text boundary and names no actor
    __device__ __forceinline__ uint32_t id_actor(uint32_t ctr_old, uint32_t x) const { return ctr_old ? actor(x) : x; }
};

__device__ __forceinline__ LogMaps log_maps(const Remap& R, uint32_t li) {
    LogMaps m{nullptr, 0u, nullptr, 0u};
    if (R.actor_off) { const unsigned long long o = R.actor_off[li]; m.a = R.actor_map + o; m.na = (uint32_t)(R.actor_off[li + 1] - o); }
    if (R.ctr_off) { const unsigned long long o = R.ctr_off[li]; m.c = R.ctr_map + o; m.nc = (uint32_t)(R.ctr_off[li + 1] - o); }
    return m;
}

// The resident descriptor new log li copies: its own, log from[li]'s, or an empty one for an added log.
template <class Desc>
__device__ __forceinline__ Desc source_desc(const Desc* __restrict__ old, const uint32_t* __restrict__ from, uint32_t li) {
    const uint32_t s = from ? __ldg(from + li) : li;
    return s == PT_SELECT_ADDED ? Desc{} : old[s];
}

__global__ void splice_records_kernel(const pt_log_desc* __restrict__ old_desc, const pt_log_desc* __restrict__ new_desc,
                                      const pt_log_desc* __restrict__ delta_desc, const uint32_t* __restrict__ from, uint32_t n_logs, Remap R,
                                      const pt_insdel_rec* __restrict__ old_ins, const pt_mark_rec* __restrict__ old_marks,
                                      const pt_insdel_rec* __restrict__ delta_ins, const pt_mark_rec* __restrict__ delta_marks,
                                      pt_insdel_rec* __restrict__ new_ins, pt_mark_rec* __restrict__ new_marks, uint32_t* __restrict__ bad) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t first = blockIdx.y * 32u + lane, step = gridDim.y * 32u;     // this warp's slice of each log
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        const pt_log_desc O = source_desc(old_desc, from, li), N = new_desc[li], D = delta_desc[li];
        const LogMaps m = log_maps(R, li);
        const bool ident = !m.na && !m.nc && !R.comment_map;       // warp-uniform
        // ins/del records: {ctr, ref_ctr, actor | ref_actor << 16, payload}
        const uint4* is = reinterpret_cast<const uint4*>(old_ins + O.insdel_off);
        uint4* id = reinterpret_cast<uint4*>(new_ins + N.insdel_off);
        for (uint32_t k = first; k < O.n_insdel; k += step) {
            uint4 r = __ldg(is + k);
            if (!ident) {
                const uint32_t a = m.id_actor(r.x, r.z & 0xFFFFu), ra = m.id_actor(r.y, r.z >> 16);
                r.x = m.ctr(r.x); r.y = m.ctr(r.y); r.z = (a & 0xFFFFu) | (ra << 16);
            }
            id[k] = r;
        }
        const uint4* dis = reinterpret_cast<const uint4*>(delta_ins + D.insdel_off);
        for (uint32_t k = first; k < D.n_insdel; k += step) id[O.n_insdel + k] = __ldg(dis + k);
        // mark records, two words each: A = {ctr, actor | kind << 16 | bounds << 24, start_ctr, end_ctr},
        // B = {start_actor | end_actor << 16, attr, arrival, reserved}
        const uint4* ms = reinterpret_cast<const uint4*>(old_marks + O.mark_off);
        uint4* md = reinterpret_cast<uint4*>(new_marks + N.mark_off);
        const uint32_t nq = 2u * O.n_mark;
        if (ident) {
            for (uint32_t k = first; k < nq; k += step) md[k] = __ldg(ms + k);
        } else {
            for (uint32_t base = first - lane; base < nq; base += step) {       // 32-aligned: a mark's two words share a trip
                const uint32_t k = base + lane;
                const bool valid = k < nq;
                uint4 q = valid ? __ldg(ms + k) : make_uint4(0, 0, 0, 0);
                const uint32_t py = __shfl_xor_sync(0xffffffffu, q.y, 1), pz = __shfl_xor_sync(0xffffffffu, q.z, 1),
                               pw = __shfl_xor_sync(0xffffffffu, q.w, 1);
                if (!valid) continue;
                if (!(lane & 1u)) {
                    const uint32_t a = m.id_actor(q.x, q.y & 0xFFFFu);
                    q.x = m.ctr(q.x); q.y = (q.y & 0xFFFF0000u) | (a & 0xFFFFu); q.z = m.ctr(q.z); q.w = m.ctr(q.w);
                } else {
                    const uint32_t sa = m.id_actor(pz, q.x & 0xFFFFu), ea = m.id_actor(pw, q.x >> 16);
                    q.x = (sa & 0xFFFFu) | (ea << 16);
                    if (R.comment_map && ((py >> 17) & 3u) == PT_MARK_COMMENT && q.y != PT_ATTR_NONE) {
                        q.y = q.y < R.n_comment ? __ldg(R.comment_map + q.y) : PT_ATTR_NONE;
                        if (q.y == PT_ATTR_NONE) atomicOr(bad, 1u);   // refused: the new buffers are not used
                    }
                }
                md[k] = q;
            }
        }
        const uint4* dms = reinterpret_cast<const uint4*>(delta_marks + D.mark_off);
        for (uint32_t k = first; k < 2u * D.n_mark; k += step) md[nq + k] = __ldg(dms + k);
    }
}

// Change table splice: per log, the old change records (actor mapped), the delta's (dep_off rebased past the log's old
// deps), the old dep records (actor mapped), the delta's.
__global__ void splice_changes_kernel(const pt_change_desc* __restrict__ old_cd, const pt_change_desc* __restrict__ new_cd,
                                      const pt_change_desc* __restrict__ delta_cd, const uint32_t* __restrict__ from, uint32_t n_logs, Remap R,
                                      const pt_change_rec* __restrict__ old_ch, const pt_dep_rec* __restrict__ old_dp,
                                      const pt_change_rec* __restrict__ delta_ch, const pt_dep_rec* __restrict__ delta_dp,
                                      pt_change_rec* __restrict__ new_ch, pt_dep_rec* __restrict__ new_dp) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t li = warp; li < n_logs; li += nwarps) {
        const pt_change_desc O = source_desc(old_cd, from, li), N = new_cd[li], D = delta_cd[li];
        const LogMaps m = log_maps(R, li);
        // change records: {seq, actor | n_deps << 16, dep_off, n_ops}
        const uint4* cs = reinterpret_cast<const uint4*>(old_ch + O.change_off);
        uint4* cd = reinterpret_cast<uint4*>(new_ch + N.change_off);
        for (uint32_t k = lane; k < O.n_changes; k += 32) {
            uint4 r = __ldg(cs + k);
            r.y = (r.y & 0xFFFF0000u) | (m.actor(r.y & 0xFFFFu) & 0xFFFFu);
            cd[k] = r;
        }
        const uint4* dcs = reinterpret_cast<const uint4*>(delta_ch + D.change_off);
        for (uint32_t k = lane; k < D.n_changes; k += 32) {
            uint4 r = __ldg(dcs + k);
            r.z += O.n_deps;
            cd[O.n_changes + k] = r;
        }
        // dep records: {seq, actor | reserved << 16}
        const uint2* ps = reinterpret_cast<const uint2*>(old_dp + O.dep_off);
        uint2* pd = reinterpret_cast<uint2*>(new_dp + N.dep_off);
        for (uint32_t k = lane; k < O.n_deps; k += 32) {
            uint2 r = __ldg(ps + k);
            r.y = (r.y & 0xFFFF0000u) | (m.actor(r.y & 0xFFFFu) & 0xFFFFu);
            pd[k] = r;
        }
        const uint2* dps = reinterpret_cast<const uint2*>(delta_dp + D.dep_off);
        for (uint32_t k = lane; k < D.n_deps; k += 32) pd[O.n_deps + k] = __ldg(dps + k);
    }
}

}  // namespace pta
