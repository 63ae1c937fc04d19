// warp_kernel.cuh — op-log apply + flatten for SHORT logs: ONE WARP materialises one log (sm_90a).
//
// Same closed form as merge_kernel.cuh (SURVEY.md §9.2; reference src/micromerge.ts:534-724, src/peritext.ts:154-455),
// re-cut for logs of up to a few thousand records (BASELINE.json configs[3]: 100K docs x 1K ops x 3 replicas):
//   * no block barriers: every scan is a shuffle scan, every reduction a redux.sync, phases are separated by __syncwarp;
//     several warps of a CTA work on different logs, each in its own slice of dynamic shared memory
//   * 16-bit everything (record indices, opId keys K = (ctr-1)*R + actor, Euler nodes = next:16 | visible weight:16)
//   * sibling order without sorting groups: run heads are ranked by K with a key-space bitmap (unique keys: counting sort),
//     then threaded in ASCENDING K with __match_any_sync — the previously threaded sibling of the same parent is the next
//     sibling in the reference's descending order (src/micromerge.ts:628-635), the last one threaded is the first child
//   * marks are resolved in VISIBLE space: a mark op covers visible element v iff vis(start slot) <= v < vis(end slot); ops
//     that cover no visible element (most of them in fuzz-shaped logs, where nearly everything is a tombstone) are dropped
//     right after their two boundary lookups; spans come from the few survivors by stabbing the elementary segments
//   * comment ops fold in ARRIVAL order (src/peritext.ts:314-322 has no opId comparison; quirk Q4)
// A log that does not fit the warp's slice, or whose surviving mark set is too large for the stabbing loops, is DEFERRED on
// the device to the block kernel's bins (merge_kernel.cuh) — results are identical either way.
#pragma once
#include "merge_kernel.cuh"
#include "upload_kernel.cuh"

namespace ptk {

constexpr uint32_t kFull = 0xffffffffu;
constexpr uint32_t kNone16 = 0xFFFFu;
constexpr uint32_t kWarpGrab = 4;            // logs taken from the work queue per atomic
constexpr uint32_t kMaxSegSurvivorWork = 1536;   // ceil(S/32) * nS above this: defer to the block kernel's segment trees
constexpr uint32_t kMaxCommentSurvivors = 48;    // the comment loops are quadratic in the surviving comment ops

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(kFull, v, o); if (lane >= (uint32_t)o) v += y; }
    return v;
}

// per-warp bump allocator over the warp's slice of dynamic shared memory (offsets from the __shared__ symbol: LDS/STS)
struct WArena {
    uint32_t base, used, cap;
    // bump; the caller checks fits() once per group of allocations, BEFORE touching any of them
    template <class T> __device__ __forceinline__ T* alloc(uint32_t count) {
        const uint32_t off = used;
        used += (uint32_t)((count * sizeof(T) + 15u) & ~15u);
        return reinterpret_cast<T*>(ptk_smem + base + off);
    }
    __device__ __forceinline__ bool fits() const { return used <= cap; }
};

// Phase alignment of the warps of one CTA (optional).  The kernel's code is far larger than the instruction caches
// (L0 ~6 KB per scheduler, L1.5 32 KB per SM), and warps that drift apart each stream their own part of it from L2; named
// barriers at a few phase boundaries keep the warps of a CTA in the same code region.  A warp that leaves a log early
// (error status, deferral, no work) ARRIVES at the remaining barriers without waiting, so nobody waits for it.
constexpr uint32_t kFirstPhaseBar = 2, kLastPhaseBar = 5;      // barrier 1 = start of a round (work loop)
__device__ __noinline__ void phase_arrive_rest(uint32_t next, uint32_t nthreads, uint32_t skip) {
    for (; next <= kLastPhaseBar; next++)
        if (!((skip >> (next - kFirstPhaseBar)) & 1u)) asm volatile("barrier.arrive %0, %1;" ::"r"(next), "r"(nthreads) : "memory");
}
struct PhaseSync {
    uint32_t on, nthreads, next, skip;      // skip: bit k set = phase barrier kFirstPhaseBar + k is not used (tuning)
    __device__ __forceinline__ void pass() {
        if (on && !((skip >> (next - kFirstPhaseBar)) & 1u)) asm volatile("barrier.sync %0, %1;" ::"r"(next), "r"(nthreads) : "memory");
        next++;
    }
    __device__ __forceinline__ void leave() {
        if (on && next <= kLastPhaseBar) phase_arrive_rest(next, nthreads, skip);
        next = kLastPhaseBar + 1;
    }
};

template <class T>
__device__ __forceinline__ void wfill(T* p, uint32_t count, T v, uint32_t lane) {   // allocations are padded to 16 B
    const uint32_t nvec = (uint32_t)((count * sizeof(T) + 15u) >> 4);
    uint32_t w;
    if (sizeof(T) == 1) w = 0x01010101u * (uint32_t)(uint8_t)v;
    else if (sizeof(T) == 2) w = 0x00010001u * (uint32_t)(uint16_t)v;
    else w = (uint32_t)v;
    const uint4 q = make_uint4(w, w, w, w);
    uint4* d = reinterpret_cast<uint4*>(p);
#pragma unroll 1
    for (uint32_t i = lane; i < nvec; i += 32) d[i] = q;
}

// Per-phase cycle profile (build with `make PHASE_CLOCKS=1`; tools/phase_profile.py reads it through pt_phase_clocks).
// Every warp sums clock64() deltas per phase in registers and adds them to ptk_phase_clk when it exits; the default build
// contains none of it.
#ifdef PT_PHASE_CLOCKS
enum : int { kPhStart, kPhAB, kPhC, kPhD, kPhE, kPhF, kPhG, kPhI, kPhRound, kNumPhases };
__device__ unsigned long long ptk_phase_clk[kNumPhases + 1];   // cycles per phase summed over warps, then the logs merged
struct PhaseClock {
    long long t;
    unsigned long long c[kNumPhases], logs;
    __device__ __forceinline__ void mark(int k) { const long long now = clock64(); c[k] += (unsigned long long)(now - t); t = now; }
};
#define PT_PHASE(k) pclk.mark(k)
#define PT_PHASE_PARAM , PhaseClock& pclk
#define PT_PHASE_ARG , pclk
#else
#define PT_PHASE(k) ((void)0)
#define PT_PHASE_PARAM
#define PT_PHASE_ARG
#endif

// id-table forms of the warp kernel (one kernel instantiation each; the host sorts the logs into the launches)
constexpr int kIdDirect = 0, kIdCompact = 1, kIdPacked3 = 2;

// returns 0: done (result header written), 1: defer to the block kernel.  IDM selects the id-table form (below).
template <int IDM>
__device__ __forceinline__ int warp_merge_one_log(const BatchParams& P, const uint32_t li, const uint32_t slice_base, const uint32_t slice_bytes, const uint32_t li_next, PhaseSync ps PT_PHASE_PARAM) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t lt = (1u << lane) - 1u;

    // descriptor: all lanes read the same 32 bytes (one broadcast transaction)
    const uint4 dsc0 = __ldg(reinterpret_cast<const uint4*>(P.desc + li)), dsc1 = __ldg(reinterpret_cast<const uint4*>(P.desc + li) + 1);
    const unsigned long long insdel_off = (unsigned long long)dsc0.x | ((unsigned long long)dsc0.y << 32);
    const unsigned long long mark_off = (unsigned long long)dsc0.z | ((unsigned long long)dsc0.w << 32);
    const uint32_t n = dsc1.x, m = dsc1.y, R = dsc1.z ? dsc1.z : 1u, C = dsc1.w;
    const unsigned long long KS64 = (unsigned long long)C * R;
    // 16-bit keys / indices only, and arrivals that fit the 11-bit field of the key records (the host routes no other log here
    // at the default max_recs)
    if (KS64 >= 0xFFFFull || n >= 0xFFFFu || m >= 0xFFFFu || (m && n > 2047u)) { ps.leave(); return 1; }
    const uint32_t KS = (uint32_t)KS64;
    // the record streams are read from the key-record copy (upload_kernel.cuh: ins own:16 | ref:16, marks {own | start << 16,
    // end | arrival << 16 | kind << 27 | start bound << 30 | end bound << 31}, keys K = (ctr-1)*R + actor, kS0 / kS1 above every
    // key); phase F reads the full ins/del records for the payloads of visible elements, and G's link and comment survivors
    // their attrs from the full mark records
    constexpr uint32_t kS0 = ptu::kKeyS0, kS1 = ptu::kKeyS1;
    const uint32_t* __restrict__ ins = P.key_insdel + insdel_off;
    const uint2* __restrict__ mk = P.key_marks + mark_off;
    const pt_insdel_rec* __restrict__ full_ins = P.insdel + insdel_off;
    uint32_t* text_out = P.text + P.text_off[li];
    pt_log_result* res = P.results + li;

    if ((P.warp_flags & 1u) && m) {       // this log's mark records are needed late: pull them into L2 now
        const char* p0 = reinterpret_cast<const char*>(mk);
        const uint32_t lines = (m * 8u + 127u) >> 7;
        for (uint32_t l = lane; l < lines; l += 32) prefetch_l2(p0 + ((size_t)l << 7));
    }

    WArena A; A.base = slice_base; A.used = 0; A.cap = slice_bytes;
    uint32_t st = 0;                                           // lane-local failures, bit (1 << code); the checkpoints report the highest code
    auto fail = [&](uint32_t code) { st |= 1u << code; };
    // a duplicate insert opId sets bit 0 (no status has code 0): it is reported as PT_LOG_BAD_OPID only when the record pass
    // found no other failure — the block and team kernels count duplicates only after their record pass (DESIGN.md §2)
    auto failDup = [&]() { st |= 1u; };
    auto bail = [&](uint32_t code) { if (lane == 0) { pt_log_result r{}; r.status = code; *res = r; } };

    // ---- id table: opId -> insert record index ------------------------------------------------------------------------------
    // direct : T[K(ctr, actor)], 2 bytes per key of the key space C*R (what merge_kernel.cuh does).
    // compact: with >= 3 actors most of that space is empty (c4: 250 inserts in 2200 keys), and shared memory per warp is what
    //          bounds the number of resident warps.  T[ctr-1] = actor:5 | index:11 of ONE insert with that counter; the few
    //          inserts that share a counter with an earlier one (concurrent edits) go to a small open-addressing overflow
    //          table OV (key:16 | index:16, linear probing).  More than kOvMax of those: the log is deferred.
    // packed3: exactly 3 actors and <= 1022 records (c4's shape: three concurrent replicas): one 32-bit word per COUNTER holds
    //          the three actors' record indices + 1 in 10-bit fields.  An insert is ONE atomicOr (the old value tells a
    //          duplicate opId), a lookup one LDS + shift + mask; no overflow table, nothing to probe.
    constexpr bool compact = IDM == kIdCompact, packed = IDM == kIdPacked3;
    if (compact && !(R >= 3u && R <= 30u && n <= 2046u)) { ps.leave(); return 1; }     // (the host only sends such logs to this launch)
    if (packed && !(R == 3u && n <= 1022u)) { ps.leave(); return 1; }
    constexpr uint32_t kOvSlots = 128, kOvMax = 96, kOvEmpty = 0xFFFFFFFFu;
    const uint32_t NWr = (n + 31) / 32 + 1;                    // bit words over record indices (+1 zero pad word)
    // layout: the arrays at FIXED offsets first (their addresses are one add away from the slice base)
    uint32_t* OV = A.alloc<uint32_t>(compact ? kOvSlots : 0u);
    // per 32-record word: x = insert bits, y = chain-link bits (after C: run-head bits), z = visible bits (after C),
    // w = run heads before the word | visible elements before the word << 16 (after C)
    uint4* WI = A.alloc<uint4>(NWr);
    uint16_t* T = A.alloc<uint16_t>(packed ? 2u * C : compact ? C : KS);
    uint32_t* T32 = reinterpret_cast<uint32_t*>(T);              // packed3 view
    // key-space bitmap of the opIds seen: A+B sets every insert key, G every mark key, so G's duplicate-opId test is the old
    // bit of its one atomicOr (no id-table lookup)
    const uint32_t KW = (KS + 31) / 32;
    uint32_t* KSeen = A.alloc<uint32_t>(KW + 1);
    if (!A.fits()) { ps.leave(); return 1; }
    if (packed) wfill<uint32_t>(T32, C, 0u, lane);
    else wfill<uint16_t>(T, compact ? C : KS, (uint16_t)kNone16, lane);
    if (compact) wfill<uint32_t>(OV, kOvSlots, kOvEmpty, lane);
    wfill<uint32_t>(KSeen, KW + 1, 0u, lane);
    // during A+B the z / w fields of WI collect the "element has a child that is not its log successor" and tombstone bits (atomicOr)
    wfill<uint32_t>(reinterpret_cast<uint32_t*>(WI), 4 * NWr, 0u, lane);
    __syncwarp();
    auto ovHash = [&](uint32_t key) -> uint32_t { return ((key * 40503u) >> 7) & (kOvSlots - 1u); };
    // key -> (ctr - 1, actor).  packed3: key / 3 as a multiply-high, exact for 16-bit keys.  compact: key / R with the log's
    // reciprocal ceil(2^32 / R), exact for 16-bit keys (the error is below (R-1) * 2^16 / 2^32 < 1 / R)
    const uint32_t invR = compact ? 0xFFFFFFFFu / R + 1u : 0u;
    auto ctrOf = [&](uint32_t key) -> uint32_t { return packed ? (key * 0xAAABu) >> 17 : __umulhi(key, invR); };
    // index of the insert record with opId key `key`; if there is none, kNone16 (packed3: 0xFFFFFFFF); the key must be valid (< kS0)
    auto lookup = [&](uint32_t key) -> uint32_t {
        if (!packed && !compact) return T[key];
        const uint32_t c = ctrOf(key), actor = key - c * (packed ? 3u : R);
        if (packed) return ((T32[c] >> (10u * actor)) & 1023u) - 1u;    // field 0 (none): 0xFFFFFFFF, above every index
        const uint32_t e = T[c];
        if (e == kNone16) return kNone16;                      // no insert with this counter at all
        if ((e >> 11) == actor) return e & 0x7FFu;
        for (uint32_t h = ovHash(key);; h = (h + 1u) & (kOvSlots - 1u)) {
            const uint32_t v = OV[h];
            if (v == kOvEmpty) return kNone16;
            if ((v >> 16) == key) return v & 0xFFFFu;
        }
    };

    // ---- A+B: one pass over the ins/del records, 32 per trip (128 B), two trips in flight -----------------------------------
    // A: id table, insert bits, chain-link bits (reference element == the insert at record i-1: compare with the left
    //    neighbour's key, no lookup).  B: parents of non-chain inserts ("has another child" bits) and deletes (tombstones, OR).
    //    A referenced element must have arrived EARLIER in the log (src/micromerge.ts:752 throws otherwise).
    uint32_t nOv = 0;
    {
        uint32_t carryK = 0xFFFFFFFFu;                         // key of the last record of the previous trip if it is an insert
        // records past the end are loaded from a clamped index and ignored (every use is guarded by i < n)
        const uint32_t nm1 = n ? n - 1u : 0u;
        uint32_t ra = 0;
        if (n) ra = __ldg(ins + min(lane, nm1));
        // the whole stream past the first two trips (a c4 log's is ~2 KB) goes to L2 up front: DRAM latency under load is longer
        // than two trips
        const char* insb = reinterpret_cast<const char*>(ins);
        const uint32_t insBytes = n * 4u;
        for (uint32_t o = 256u + lane * 128u; o < insBytes; o += 32u * 128u) prefetch_l2(insb + o);
        PT_PHASE(kPhStart);
#pragma unroll 2
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t rc = __ldg(ins + min(i + 32u, nm1));         // one trip ahead (the lines are in L2 by now); unrolled by 2: no moves
            const uint32_t own = ra & 0xFFFFu, rkey = ra >> 16;
            // straight-line form: predicates instead of nested branches.  own == kS1: a bad kind (rkey == kS1) or a bad opId;
            // own == kS0: a delete; else an insert with key own.  rkey: kS0 = the head, kS1 = out of range, else a key
            const bool inb = i < n;
            const bool valid = inb && own != kS1;
            if (inb && !valid) fail(rkey == kS1 ? PT_LOG_BAD_KIND : PT_LOG_BAD_OPID);
            const uint32_t key = own;
            const bool isIns = valid && own != kS0;
            bool toOv = false, wrote = false;
            uint32_t mine = 0;
            if (isIns) {
                atomicOr(&KSeen[key >> 5], 1u << (key & 31));
                if (packed) {
                    const uint32_t c = ctrOf(key), sh = 10u * (key - 3u * c);
                    if ((atomicOr(&T32[c], (i + 1u) << sh) >> sh) & 1023u) failDup();   // two inserts with one opId
                } else if (!compact) {
                    if (T[key] != kNone16) failDup();                  // two inserts with one opId (earlier trip)
                    T[key] = (uint16_t)i;
                } else {
                    const uint32_t c = ctrOf(key), actor = key - c * R;
                    mine = (actor << 11) | i;
                    const uint32_t e = T[c];
                    if (e == kNone16) { T[c] = (uint16_t)mine; wrote = true; }
                    else if ((e >> 11) == actor) failDup();
                    else toOv = true;
                }
            }
            const uint32_t myK = isIns ? key : 0xFFFFFFFFu;
            uint32_t prevK = __shfl_up_sync(kFull, myK, 1);
            if (lane == 0) prevK = carryK;
            carryK = __shfl_sync(kFull, myK, 31);
            const bool refOk = rkey < kS0;
            bool cand = isIns && refOk && rkey == prevK;           // typing-chain link: the reference element is record i-1
            if (cand && rkey >= key) { fail(PT_LOG_CYCLE); cand = false; }
            const uint32_t insW = __ballot_sync(kFull, isIns), candW = __ballot_sync(kFull, cand);
            if (lane == 0) *reinterpret_cast<uint2*>(&WI[base >> 5]) = make_uint2(insW, candW);
            __syncwarp();                                          // the trip's ids are in T
            if (IDM == kIdDirect) {
                if (isIns && T[key] != (uint16_t)i) failDup();               // two inserts with one opId (same trip)
            } else if (compact) {
                if (wrote) {                                       // same counter twice in one trip: one lane owns the slot
                    const uint32_t e2 = T[ctrOf(key)];
                    if (e2 != mine) { if ((e2 >> 11) == (mine >> 11)) failDup(); else toOv = true; }
                }
                const uint32_t ovW = __ballot_sync(kFull, toOv);
                if (ovW) {
                    nOv += __popc(ovW);
                    if (toOv && nOv <= kOvMax) {
                        const uint32_t val = (key << 16) | i;
                        for (uint32_t h = ovHash(key);; h = (h + 1u) & (kOvSlots - 1u)) {
                            const uint32_t old = atomicCAS(&OV[h], kOvEmpty, val);
                            if (old == kOvEmpty) break;
                            if ((old >> 16) == key) { failDup(); break; }
                        }
                    }
                    __syncwarp();
                }
            }
            {   // B: the reference element of a non-chain record (rkey == kS0: an insert at the head of the list)
                const bool need = valid && !cand, hasRef = rkey != kS0;
                uint32_t j = kNone16;
                if (need && refOk) j = lookup(rkey);
                const bool found = j != kNone16 && j < i;              // must have arrived earlier
                const bool cyc = isIns && rkey >= key;
                if (need) {
                    if (hasRef ? !found : !isIns) fail(PT_LOG_ELEM_NOT_FOUND);
                    else if (hasRef && cyc) fail(PT_LOG_CYCLE);
                }
                if (need && found && !cyc) atomicOr(reinterpret_cast<uint32_t*>(&WI[j >> 5]) + (isIns ? 2u : 3u), 1u << (j & 31));   // deletes: OR, idempotent (micromerge.ts:689)
            }
            ra = rc;
        }
    }
    __syncwarp();
    ps.pass();                                                     // (2) end of the record pass
    if (compact && nOv > kOvMax) { ps.leave(); return 1; }                                    // too many concurrent-counter inserts for the compact table
    st = __reduce_or_sync(kFull, st);
    if (st) { bail(st > 1u ? 31u - __clz(st) : PT_LOG_BAD_OPID); ps.leave(); return 0; }
    PT_PHASE(kPhAB);

    // ---- C: runs, bit-parallel: head = insert & (!chain-link | predecessor has another child); visible = insert & !deleted
    uint32_t M, nvis, N = 0;
    {
        uint32_t carryH = 0, carryV = 0, otherCarry = 0;
        for (uint32_t wb = 0; wb < NWr; wb += 32) {
            const uint32_t w = wb + lane;
            uint32_t insW = 0, candW = 0, otherW = 0, delW = 0;
            if (w < NWr) { const uint4 q = WI[w]; insW = q.x; candW = q.y; otherW = q.z; delW = q.w; }
            const uint32_t up = __shfl_up_sync(kFull, otherW, 1);
            const uint32_t prevBit = lane ? (up >> 31) : otherCarry;
            otherCarry = __shfl_sync(kFull, otherW, 31) >> 31;
            const uint32_t head = insW & (~candW | ((otherW << 1) | prevBit));
            const uint32_t vis = insW & ~delW;
            const uint32_t pc = __popc(head) | (__popc(vis) << 16);
            const uint32_t inc = warp_incl_scan(pc, lane), ex = inc - pc, tot = __shfl_sync(kFull, inc, 31);
            if (w < NWr) WI[w] = make_uint4(insW, head, vis, (carryH + (ex & 0xFFFFu)) | ((carryV + (ex >> 16)) << 16));
            // phase D reads every run head's record again: the 128-byte lines (32 records) that hold heads go to L2 now, all at once
            if (head) prefetch_l2(ins + w * 32u);
            carryH += tot & 0xFFFFu; carryV += tot >> 16;
            N += __reduce_add_sync(kFull, (uint32_t)__popc(insW));
        }
        M = carryH; nvis = carryV;
    }
    __syncwarp();
    PT_PHASE(kPhC);

    auto runOf = [&](uint32_t i) -> uint32_t {
        const uint4 q = WI[i >> 5];
        return (q.w & 0xFFFFu) + __popc(q.y & (0xFFFFFFFFu >> (31 - (i & 31)))) - 1u;
    };
    auto visBefore = [&](uint32_t i) -> uint32_t {
        const uint4 q = WI[i >> 5];
        return (q.w >> 16) + __popc(q.z & ((1u << (i & 31)) - 1u));
    };

    if ((P.warp_flags & 2u) && li_next != 0xFFFFFFFFu && lane == 0) prefetch_l2(P.desc + li_next);   // read in phase F
    // ---- D: run tree; E: Euler tour + splitter list ranking of the VISIBLE weights ------------------------------------------
    const uint32_t E = 2 * (M + 1), END = (E + 7u) & ~7u;          // END: terminator id, a multiple of 8 like every splitter node
    if (END + 1 >= 0xFFFFu) { ps.leave(); return 1; }
    uint16_t* VisBase = A.alloc<uint16_t>(M + 1);                  // vis(i) = VisBase[run(i)] + visBefore(i)   (mod 2^16)
    const uint32_t markD = A.used;
    {
        // Euler tour nodes: enter(r) = r, exit(r) = (M+1) + r, r in 0..M (M = HEAD).  One 32-bit word per node: low half =
        // successor (later: owner splitter), high half = visible weight of the node (later: weight prefix inside the owner's
        // sublist); exits weigh 0.  Splitter ids: k < SPEND: node 8k; SPEND: the terminator; SPEND + 1: the tour's first node.
        const uint32_t SPEND = END >> 3, nSp = SPEND + 2;
        uint32_t* Node = A.alloc<uint32_t>(E);
        uint16_t* N16 = reinterpret_cast<uint16_t*>(Node);         // N16[2x] = successor of x, N16[2x + 1] = weight of x
        // run head record index, then visBefore(head); it lives in VisBase, which the last loop of E writes over it entry by
        // entry (D's footprint bounds the runs a slice holds)
        uint16_t* HV = VisBase;
        uint16_t* Prun = A.alloc<uint16_t>(M + 1);
        uint16_t* RKey = A.alloc<uint16_t>(M + 2);                 // key of the run head; dead after the ranking, then:
        uint16_t* Last = RKey;                                     // last threaded child of run q (q = M: HEAD)
        // ByG[pos] (run with the pos-th smallest head key) lives in the weight halves of the exit nodes until the tour is threaded
        auto ByG = [&](uint32_t pos) -> uint16_t& { return N16[2 * ((M + 1) + pos) + 1]; };
        // key bitmap + prefix (ranking of the head keys); dead after the ranking, then the splitter summaries live there
        const uint32_t uBytes = max((uint32_t)(((KW + 1) * 4 + 15) & ~15u) + (uint32_t)(((KW + 1) * 2 + 15) & ~15u), 2u * (uint32_t)((nSp * 4 + 15) & ~15u));
        char* U = A.alloc<char>(uBytes);
        if (!A.fits()) { ps.leave(); return 1; }
        uint32_t* KBits = reinterpret_cast<uint32_t*>(U);
        uint16_t* KPre = reinterpret_cast<uint16_t*>(U + (((KW + 1) * 4 + 15) & ~15u));
        uint32_t* Sub = reinterpret_cast<uint32_t*>(U);
        uint32_t* Sub2 = reinterpret_cast<uint32_t*>(U + ((nSp * 4 + 15) & ~15u));
#pragma unroll 1
        for (uint32_t wb = 0; wb < NWr; wb += 32) {                // compact the run heads (one bit word per lane)
            const uint32_t w = wb + lane;
            if (w < NWr) {
                const uint4 q = WI[w];
                uint32_t hb = q.y, rid = q.w & 0xFFFFu;
                while (hb) { const uint32_t b = __ffs(hb) - 1; hb &= hb - 1; HV[rid++] = (uint16_t)(w * 32 + b); }
            }
        }
        wfill<uint32_t>(KBits, KW + 1, 0u, lane);
        __syncwarp();
#pragma unroll 1
        for (uint32_t rb = 0; rb < M; rb += 32) {                  // one lane per run: extent, parent run, visible weight, key bit
            const uint32_t r = rb + lane;
            if (r < M) {
                const uint32_t i = HV[r], w = i >> 5, b = i & 31;
                const uint32_t rec = __ldg(ins + i);               // issued before the run-end scan: its latency overlaps the scan
                const uint4 q0 = WI[w];
                uint32_t stop = (q0.y | ~q0.x) & ~(0xFFFFFFFFu >> (31 - b));
                uint32_t ww = w;
                while (!stop) { ww++; const uint2 q1 = *reinterpret_cast<const uint2*>(&WI[ww]); stop = q1.y | ~q1.x; }   // pad word: insert bits == 0 -> stops
                const uint32_t end = ww * 32 + (__ffs(stop) - 1);
                const uint32_t key = rec & 0xFFFFu, rkey = rec >> 16;   // a run head is a valid insert: rkey is kS0 or a key
                const uint32_t p = rkey == kS0 ? n : lookup(rkey);
                const uint32_t q = p == n ? M : runOf(p);
                const uint32_t hv = visBefore(i);
                N16[2 * r + 1] = (uint16_t)(visBefore(end) - hv);
                HV[r] = (uint16_t)hv;
                Prun[r] = (uint16_t)q; RKey[r] = (uint16_t)key;
                atomicOr(&KBits[key >> 5], 1u << (key & 31));
            }
        }
        __syncwarp();
        {
            uint32_t carry = 0;
#pragma unroll 1
            for (uint32_t wb = 0; wb < KW; wb += 32) {
                const uint32_t w = wb + lane;
                const uint32_t cnt = w < KW ? __popc(KBits[w]) : 0u;
                const uint32_t inc = warp_incl_scan(cnt, lane);
                if (w < KW) KPre[w] = (uint16_t)(carry + inc - cnt);
                carry += __shfl_sync(kFull, inc, 31);
            }
        }
        __syncwarp();
#pragma unroll 1
        for (uint32_t rb = 0; rb < M; rb += 32) {                  // rank of the run head's key among all run heads (unique keys)
            const uint32_t r = rb + lane;
            if (r < M) {
                const uint32_t key = RKey[r];
                ByG((uint32_t)KPre[key >> 5] + __popc(KBits[key >> 5] & ((1u << (key & 31)) - 1u))) = (uint16_t)r;
            }
        }
        __syncwarp();
        ps.pass();                                                 // (3) run heads ranked
        wfill<uint16_t>(Last, M + 2, (uint16_t)kNone16, lane);     // RKey, KBits, KPre are dead from here
        __syncwarp();
        // thread the runs in ASCENDING key order: among the children of one parent, the previously threaded one is the
        // NEXT sibling in descending-opId order (src/micromerge.ts:628-635), the last one threaded is the FIRST child
#pragma unroll 1
        for (uint32_t cb = 0; cb < M; cb += 32) {
            const uint32_t pos = cb + lane;
            const bool valid = pos < M;
            const uint32_t r = valid ? (uint32_t)ByG(pos) : 0u;
            const uint32_t q = valid ? (uint32_t)Prun[r] : (0x10000u + lane);
            // siblings inside this chunk of 32: MATCH.ANY over the parents (measured: cheaper than any probe that would avoid it)
            uint32_t mask = 1u << lane;
            const uint32_t pm = __ballot_sync(kFull, valid);
            if (valid) mask = __match_any_sync(pm, q);
            const uint32_t lower = mask & lt;
            const uint32_t src = lower ? (31u - __clz(lower)) : lane;
            const uint32_t rs = __shfl_sync(kFull, r, src);
            uint32_t ns = kNone16;
            if (valid) ns = lower ? rs : (uint32_t)Last[q];
            __syncwarp();
            if (valid) {
                N16[2 * ((M + 1) + r)] = (uint16_t)(ns != kNone16 ? ns : (M + 1) + q);   // exit(r): next sibling, else exit(parent)
                if (((mask >> lane) >> 1) == 0) Last[q] = (uint16_t)r;              // highest lane of its group
            }
            __syncwarp();
        }
        PT_PHASE(kPhD);
#pragma unroll 1
        for (uint32_t rb = 0; rb <= M; rb += 32) {                 // enter(r): first child, else exit(r)
            const uint32_t r = rb + lane;
            if (r <= M) { const uint32_t f = Last[r]; N16[2 * r] = (uint16_t)(f != kNone16 ? f : (M + 1) + r); if (r < M) N16[2 * ((M + 1) + r) + 1] = 0; }   // exits weigh 0 (ByG is dead)
        }
        if (lane == 0) { N16[2 * M + 1] = 0; Node[(M + 1) + M] = END; }
        __syncwarp();
        // splitter list ranking: every 8th node id (and the tour's first node) walks its sublist once; only the splitter
        // summaries are ranked by pointer jumping; suffix(x) = suffix(owner sublist) - prefix(x)
        // (no node's successor is the tour's first node, and END is a multiple of 8: a sublist ends where the successor id is)
        const uint32_t headNode = M;
#pragma unroll 1
        for (uint32_t kb = 0; kb < nSp; kb += 32) {
            const uint32_t k = kb + lane;
            if (k < nSp) {
                uint32_t cur = k < SPEND ? 8 * k : headNode, acc = 0, nx = END;
                const bool valid = k < SPEND ? cur < E : (k > SPEND && (headNode & 7u) != 0);
                if (valid) {
                    for (;;) {
                        const uint32_t a = Node[cur];
                        nx = a & 0xFFFFu;
                        Node[cur] = k | (acc << 16);               // owner | weight prefix before this node
                        acc += a >> 16;
                        if ((nx & 7u) == 0) break;
                        cur = nx;
                    }
                }
                Sub[k] = (acc << 16) | (nx >> 3);                  // invalid / terminator entries: weight 0, successor SPEND
            }
        }
        __syncwarp();
        {
            uint32_t *cur = Sub, *nxt2 = Sub2;
            for (uint32_t span = 1; span < nSp + 1; span <<= 1) {
#pragma unroll 1
                for (uint32_t x = lane; x < nSp; x += 32) {
                    const uint32_t a = cur[x], b = cur[a & 0xFFFFu];
                    nxt2[x] = ((a & 0xFFFF0000u) + (b & 0xFFFF0000u)) | (b & 0xFFFFu);
                }
                __syncwarp();
                uint32_t* t = cur; cur = nxt2; nxt2 = t;
            }
            Sub = cur;
        }
#pragma unroll 1
        for (uint32_t rb = 0; rb < M; rb += 32) {
            const uint32_t r = rb + lane;
            if (r < M) {
                const uint32_t a = Node[r];
                const uint32_t suf = (Sub[a & 0xFFFFu] >> 16) - (a >> 16);          // visible elements from run r to the end
                VisBase[r] = (uint16_t)((nvis - suf) - (uint32_t)HV[r]);
            }
        }
        __syncwarp();
    }
    A.used = markD;                                                // release the run-tree temporaries
    ps.pass();                                                     // (4) sequence ranked
    PT_PHASE(kPhE);

    // ---- F: per-element visible rank table + text out (visible index = prefix count of non-deleted elements,
    // micromerge.ts:747-750).  EV[i] = visible elements before insert record i in the sequence | visible << 15: every mark
    // boundary below is then one table read instead of run / prefix arithmetic.
    uint16_t* EV = A.alloc<uint16_t>(n + 1);
    if (!A.fits() || nvis >= 0x8000u) { ps.leave(); return 1; }
    if (lane == 0) EV[n] = 0;                                      // what G reads for a boundary that has no insert record
    unsigned long long d0 = 0, d1 = 0;
#pragma unroll 1
    for (uint32_t w = 0; w + 1 < NWr; w++) {
        const uint4 q = WI[w];                                     // uniform: one broadcast LDS.128
        const uint32_t ib = q.x;
        if (!ib) continue;
        const uint32_t hbits = q.y, vbits = q.z, hp = q.w & 0xFFFFu, vp = q.w >> 16;
        if ((ib >> lane) & 1u) {
            const uint32_t i = w * 32 + lane;
            const uint32_t run = hp + __popc(hbits & (0xFFFFFFFFu >> (31 - lane))) - 1u;
            const uint32_t vr = ((uint32_t)VisBase[run] + vp + __popc(vbits & lt)) & 0xFFFFu;
            const uint32_t isv = (vbits >> lane) & 1u;
            EV[i] = (uint16_t)(vr | (isv << 15));
            if (isv) {
                const uint32_t tok = PT_PAYLOAD_TOKEN(__ldg(&full_ins[i].payload));
                text_out[vr] = tok;
                digest_add(d0, d1, pt_term_text(vr, tok));
            }
        }
    }
    __syncwarp();

    uint32_t nspans = 0;
    if ((P.warp_flags & 2u) && li_next != 0xFFFFFFFFu) {        // the next log's ins/del records -> L2 while this one does its marks
        const uint4 q0 = __ldg(reinterpret_cast<const uint4*>(P.desc + li_next)), q1 = __ldg(reinterpret_cast<const uint4*>(P.desc + li_next) + 1);
        const char* p0 = reinterpret_cast<const char*>(P.key_insdel + ((unsigned long long)q0.x | ((unsigned long long)q0.y << 32)));
        const uint32_t lines = (q1.x * 4u + 127u) >> 7;
        for (uint32_t l = lane; l < lines; l += 32) prefetch_l2(p0 + ((size_t)l << 7));
    }

    // the first 24 trips (6 KB) of mark records -> L2 now, just before G: prefetched right after C, most lines were evicted from
    // L2 (thousands of logs in flight stream through it) before G read them (DESIGN.md §4.1)
    if (m) {
        const uint32_t pfb = min(m * 8u, 6u * 1024u);
        for (uint32_t o = lane * 128u; o < pfb; o += 32u * 128u) prefetch_l2(reinterpret_cast<const char*>(mk) + o);
    }
    PT_PHASE(kPhF);
    uint32_t nS = 0, nC = 0;
    uint4* Sv = nullptr;                                           // survivors: {va | vb << 16, priority:16 | kind << 16, attr, k}
    uint16_t* CIdx = nullptr;                                      // surviving comment ops (indices into Sv), arrival order
    if (m) {
        // ---- G: mark ops -> visible intervals [va, vb); only ops that cover a visible element survive ---------------------
        CIdx = A.alloc<uint16_t>(kMaxCommentSurvivors + 32);
        if (!A.fits()) { ps.leave(); return 1; }
        const uint32_t room = A.cap - A.used, svStart = A.used;
        uint32_t capS = room > 256u ? (room - 256u) / 16u : 0u;
        if (capS > m) capS = m;
        Sv = A.alloc<uint4>(capS + 1);
        if (!A.fits()) { ps.leave(); return 1; }
        const uint32_t ksMax = KS ? KS - 1u : 0u;                  // boundary keys are clamped to a valid slot for the lookups
        // one trip of 32 marks; `tail`: the last, partial trip (the full trips need no bounds test).  Straight-line form: both
        // boundary chains (lookup, then EV read) are issued unconditionally, on keys clamped to a valid slot and on EV's entry n
        // for "no insert record", so they overlap; the hit rules are selects after the loads.  A boundary element must exist AND
        // have arrived before the mark op: the reference's walk never matches anything else (peritext.ts:236-241) — a missing
        // start is a no-op, a missing end never ends
        auto markTrip = [&](const uint2 a, const uint32_t kb, const bool tail) {
            const uint32_t k = kb + lane;
            // own / start / end == kS1: the id is out of range (a start or end also when its bound is above PT_BOUND_AFTER)
            const uint32_t key = a.x & 0xFFFFu, skey = a.x >> 16, ekey = a.y & 0xFFFFu, arrival = (a.y >> 16) & 0x7FFu;
            const uint32_t kind = (a.y >> 27) & 7u, sb = (a.y >> 30) & 1u, eb = a.y >> 31;
            const uint32_t type = (kind >> 1) & 3u;
            const bool inb = !tail || k < m;
            const uint32_t js = lookup(min(skey, ksMax)), je = lookup(min(ekey, ksMax));
            const uint32_t es = EV[min(js, n)], ee = EV[min(je, n)];
            // st is 0 here (A+B's failures returned): any bit set in the pass is a bad opId
            if (inb) {                                             // out of range, or an insert's or an earlier mark's opId
                if (key == kS1) st |= 1u;
                else { const uint32_t bit = 1u << (key & 31); st |= atomicOr(&KSeen[key >> 5], bit) & bit; }
            }
            // a missing boundary's index is above every arrival (11 bits).  A bad own id fails the log: its survivors are unused
            const bool sHit = inb && skey != kS1 && js < arrival;
            // same slot: the start branch wins and the op never ends (quirk Q2)
            const bool eHit = ekey != kS1 && je < arrival && !(je == js && eb == sb);
            const uint32_t va = (es & 0x7FFFu) + (sb & (es >> 15));
            const uint32_t vb = eHit ? (ee & 0x7FFFu) + (eb & (ee >> 15)) : nvis;
            const bool surv = sHit && va < vb;
            const uint32_t bal = __ballot_sync(kFull, surv);
            if (surv) {
                const uint32_t idx = nS + __popc(bal & lt);
                // priority: LWW types compare opIds (peritext.ts:304-313) = keys; comments fold in arrival order (Q4)
                if (idx < capS) Sv[idx] = make_uint4(va | (vb << 16), (type == PT_MARK_COMMENT ? k : key) | (kind << 16), PT_ATTR_NONE, k);
                // the attr that the batch after the loop loads: its line goes to L2 now, off the end of the pass
                if (type == PT_MARK_LINK || type == PT_MARK_COMMENT) prefetch_l2(&P.marks[(mk + k) - P.key_marks].attr);
            }
            nS += __popc(bal);
        };
        // the key-record copy has 32 records of slack past its end: the one-ahead loads need no clamp
        uint2 a = __ldg(mk + lane);
        const uint32_t mkBytes = m * 8u, mFull = m & ~31u;
#pragma unroll 2
        for (uint32_t kb = 0; kb < mFull; kb += 32) {
            if ((kb & 511u) == 0u) {                               // every 16th trip: the 32 lines of trips t+24 .. t+39 (256 B per trip)
                const uint32_t po = (kb + 768u) * 8u + lane * 128u;
                if (po < mkBytes) prefetch_l2(reinterpret_cast<const char*>(mk) + po);
            }
            const uint2 b = __ldg(mk + (kb + 32u + lane));         // one trip ahead (L2 hits); unrolled by 2: no moves
            markTrip(a, kb, false);
            a = b;
        }
        if (mFull < m) markTrip(a, mFull, true);
        __syncwarp();
        if (__reduce_or_sync(kFull, st)) { bail(PT_LOG_BAD_OPID); ps.leave(); return 0; }
        if (nS > capS) { ps.leave(); return 1; }
        A.used = svStart + ((nS * 16u + 15u) & ~15u);               // keep only the survivors
        // the attrs of the link and comment survivors (phase I reads no other) from the full records, all loads in flight at
        // once; the comment survivors in arrival order (Sv's order) go to CIdx
        const pt_mark_rec* __restrict__ full_mk = P.marks + (mk - P.key_marks);
#pragma unroll 1
        for (uint32_t s0 = 0; s0 < nS; s0 += 32) {
            const uint32_t s = s0 + lane;
            uint32_t t = 0;
            if (s < nS) {
                const uint4 sv = Sv[s];
                t = (sv.y >> 17) & 3u;
                if (t == PT_MARK_LINK || t == PT_MARK_COMMENT) Sv[s].z = __ldg(&full_mk[sv.w].attr);
            }
            const bool isC = s < nS && t == PT_MARK_COMMENT;
            const uint32_t balC = __ballot_sync(kFull, isC);
            if (isC) { const uint32_t ci = nC + __popc(balC & lt); if (ci <= kMaxCommentSurvivors) CIdx[ci] = (uint16_t)s; }
            nC += __popc(balC);
        }
        __syncwarp();
    }

    ps.pass();                                                     // (5) marks resolved
    PT_PHASE(kPhG);
    unsigned long long pool_base = 0;
    pt_span* span_out = P.spans + P.span_off[li];               // derived here, not at the log's start: A+B to G need the registers
    if (nvis == 0) nspans = 0;
    else if (nS == 0) {
        // no mark op touches a visible element: one span {} (peritext.ts:392)
        if (lane == 0) {
            pt_span s; s.start = 0; s.flags = 0; s.link_attr = PT_ATTR_NONE; s.comment_off = 0;
            span_out[0] = s;
            digest_add(d0, d1, pt_term_span(0, 0, 0, PT_ATTR_NONE));
        }
        nspans = 1;
    } else {
        // ---- I: elementary segments of the visible text -> marks per segment -> spans ---------------------------------------
        if (nC > kMaxCommentSurvivors) { ps.leave(); return 1; }
        if (nvis <= 32u && nC <= 32u) {
            // ---- I (short text): at most 32 visible characters: one lane per visible POSITION instead of elementary segments — no
            // boundary bitmap, no segment arrays.  Marks / link / comment-id set per position; a span starts where any of them
            // differs from the position before (same result as the segment form below: nothing changes inside a segment).
            const uint32_t x = lane;
            uint32_t w0 = 0, w1 = 0, w2 = 0, flags = 0, link = PT_ATTR_NONE;
#pragma unroll 1
            for (uint32_t j = 0; j < nS; j++) {
                const uint4 sv = Sv[j];                              // one broadcast LDS.128
                const uint32_t ab = sv.x, pk = sv.y;
                const bool cover = x >= (ab & 0xFFFFu) && x < (ab >> 16);
                const uint32_t t = (pk >> 17) & 3u, val = (((pk & 0xFFFFu) << 16) | j) + 1u;
                if (cover) {
                    if (t == PT_MARK_STRONG) w0 = max(w0, val);
                    else if (t == PT_MARK_EM) w1 = max(w1, val);
                    else if (t == PT_MARK_LINK) w2 = max(w2, val);
                    else flags |= PT_SPAN_COMMENT;                   // `comment` key present iff any comment op covers (quirk Q3)
                }
            }
            // LWW winners (peritext.ts:304-313): the max-opId covering op of the type; present iff it is an addMark
            if (w0 && !((Sv[(w0 - 1u) & 0xFFFFu].y >> 16) & 1u)) flags |= PT_SPAN_STRONG;
            if (w1 && !((Sv[(w1 - 1u) & 0xFFFFu].y >> 16) & 1u)) flags |= PT_SPAN_EM;
            if (w2) { const uint32_t j2 = (w2 - 1u) & 0xFFFFu; if (!((Sv[j2].y >> 16) & 1u)) { flags |= PT_SPAN_LINK; link = Sv[j2].z; } }
            // comment ids present at x: ids whose last-arrived covering op is an add (peritext.ts:314-322); the set is a bit mask
            // over the surviving comment ops, an id being named by the FIRST surviving op that carries it
            uint32_t cmask = 0;
            if (nC) {
                uint32_t canon = lane;
                if (lane < nC) {
                    const uint32_t id = Sv[CIdx[lane]].z;
                    for (uint32_t c0 = 0; c0 < lane; c0++) if (Sv[CIdx[c0]].z == id) { canon = c0; break; }
                }
#pragma unroll 1
                for (uint32_t cj = 0; cj < nC; cj++) {
                    const uint4 s1 = Sv[CIdx[cj]];                   // uniform
                    const uint32_t rep = __shfl_sync(kFull, canon, cj);
                    const bool cov = x >= (s1.x & 0xFFFFu) && x < (s1.x >> 16);
                    if (!__any_sync(kFull, cov)) continue;
                    bool later = false;
                    for (uint32_t c2 = cj + 1; c2 < nC; c2++) {
                        const uint4 s2 = Sv[CIdx[c2]];
                        if (s2.z != s1.z) continue;                  // uniform
                        if (x >= (s2.x & 0xFFFFu) && x < (s2.x >> 16)) later = true;
                    }
                    if (cov && !later && !((s1.y >> 16) & 1u)) cmask |= 1u << rep;
                }
            }
            const uint32_t pf = __shfl_up_sync(kFull, flags, 1), pl = __shfl_up_sync(kFull, link, 1), pm = __shfl_up_sync(kFull, cmask, 1);
            const bool head = x < nvis && (x == 0 || ((flags ^ pf) & 0xFu) != 0 || link != pl || cmask != pm);
            const uint32_t hb = __ballot_sync(kFull, head);
            const uint32_t cnt = head ? (uint32_t)__popc(cmask) : 0u;
            const uint32_t inc = warp_incl_scan(cnt, lane), off = inc - cnt, totalC = __shfl_sync(kFull, inc, 31);
            nspans = __popc(hb);
            if (totalC) {
                uint32_t pst = 0;
                if (lane == 0) pool_base = pool_reserve(P, totalC, pst);
                pst = __shfl_sync(kFull, pst, 0);
                if (pst) { bail(pst); ps.leave(); return 0; }
                pool_base = __shfl_sync(kFull, pool_base, 0);
            }
            if (head) {
                const uint32_t jo = __popc(hb & lt);
                uint32_t* pool = P.comment_pool + pool_base;
                uint32_t filled = 0;
                for (uint32_t mm = cmask; mm; mm &= mm - 1u) {       // ascending id order (sortBy, peritext.ts:318); the lists are short
                    const uint32_t id = Sv[CIdx[__ffs(mm) - 1]].z;
                    uint32_t y = filled;
                    while (y > 0 && pool[off + y - 1] > id) { pool[off + y] = pool[off + y - 1]; y--; }
                    pool[off + y] = id; filled++;
                }
                pt_span sp; sp.start = x; sp.flags = (flags & 0xFu) | (cnt << 8); sp.link_attr = link;
                sp.comment_off = cnt ? (uint32_t)(pool_base + off) : 0u;
                span_out[jo] = sp;
                for (uint32_t y = 0; y < cnt; y++) digest_add(d0, d1, pt_term_comment(jo, y, pool[off + y]));
                digest_add(d0, d1, pt_term_span(jo, sp.start, sp.flags, sp.link_attr));
            }
        } else {
        const uint32_t BW = nvis / 32 + 1;
        uint32_t* Bnd = A.alloc<uint32_t>(BW + 1);
        uint16_t* BPre = A.alloc<uint16_t>(BW + 1);
        if (!A.fits()) { ps.leave(); return 1; }
        wfill<uint32_t>(Bnd, BW + 1, 0u, lane);
        __syncwarp();
#pragma unroll 1
        for (uint32_t s = lane; s < nS; s += 32) {
            const uint32_t ab = Sv[s].x, va = ab & 0xFFFFu, vb = ab >> 16;
            atomicOr(&Bnd[va >> 5], 1u << (va & 31));
            if (vb < nvis) atomicOr(&Bnd[vb >> 5], 1u << (vb & 31));
        }
        __syncwarp();
        uint32_t nB = 0;
#pragma unroll 1
        for (uint32_t wb = 0; wb < BW; wb += 32) {
            const uint32_t w = wb + lane;
            const uint32_t cnt = w < BW ? __popc(Bnd[w]) : 0u;
            const uint32_t inc = warp_incl_scan(cnt, lane);
            if (w < BW) BPre[w] = (uint16_t)(nB + inc - cnt);
            nB += __shfl_sync(kFull, inc, 31);
        }
        const uint32_t S = nB + 1;                                   // segment s >= 1 starts at the s-th boundary; segment 0 = [0, first)
        if (((S + 31) / 32) * nS > kMaxSegSurvivorWork) { ps.leave(); return 1; }
        uint16_t* SegStart = A.alloc<uint16_t>(S + 1);
        uint32_t* SegFlags = A.alloc<uint32_t>(S + 1);               // bits3:0 span flags, bit4 comment set differs from x-1, bit5 head
        uint32_t* SegLink = A.alloc<uint32_t>(S + 1);
        uint16_t* SegCnt = A.alloc<uint16_t>(S + 1);                 // comment ids of the span starting here
        uint16_t* SegOut = A.alloc<uint16_t>(S + 1);                 // span index
        uint32_t* SegCOff = A.alloc<uint32_t>(S + 1);                // offset of its comment list in the log's pool reservation
        if (!A.fits()) { ps.leave(); return 1; }
        __syncwarp();
#pragma unroll 1
        for (uint32_t wb = 0; wb < BW; wb += 32) {
            const uint32_t w = wb + lane;
            if (w < BW) {
                uint32_t bb = Bnd[w], id = (uint32_t)BPre[w] + 1u;
                while (bb) { const uint32_t b = __ffs(bb) - 1; bb &= bb - 1; SegStart[id++] = (uint16_t)(w * 32 + b); }
            }
        }
        if (lane == 0) SegStart[0] = 0;
        const bool seg0_empty = (Bnd[0] & 1u) != 0;                  // position 0 is itself a boundary
        __syncwarp();
        // pass 1: marks of every segment = stabbing query over the survivors (uniform loop, broadcast reads)
#pragma unroll 1
        for (uint32_t sb = 0; sb < S; sb += 32) {
            const uint32_t s = sb + lane;
            const uint32_t x = s < S ? (uint32_t)SegStart[s] : 0u;
            uint32_t w0 = 0, w1 = 0, w2 = 0, flags = 0, link = PT_ATTR_NONE;
#pragma unroll 1
            for (uint32_t j = 0; j < nS; j++) {
                const uint4 sv = Sv[j];                              // one broadcast LDS.128
                const uint32_t ab = sv.x, pk = sv.y;
                const bool cover = x >= (ab & 0xFFFFu) && x < (ab >> 16);
                const uint32_t t = (pk >> 17) & 3u, val = (((pk & 0xFFFFu) << 16) | j) + 1u;
                if (cover) {
                    if (t == PT_MARK_STRONG) w0 = max(w0, val);
                    else if (t == PT_MARK_EM) w1 = max(w1, val);
                    else if (t == PT_MARK_LINK) w2 = max(w2, val);
                    else flags |= PT_SPAN_COMMENT;                   // `comment` key present iff any comment op covers (quirk Q3)
                }
            }
            // LWW winners (peritext.ts:304-313): the max-opId covering op of the type; present iff it is an addMark
            if (w0 && !((Sv[(w0 - 1u) & 0xFFFFu].y >> 16) & 1u)) flags |= PT_SPAN_STRONG;
            if (w1 && !((Sv[(w1 - 1u) & 0xFFFFu].y >> 16) & 1u)) flags |= PT_SPAN_EM;
            if (w2) { const uint32_t j2 = (w2 - 1u) & 0xFFFFu; if (!((Sv[j2].y >> 16) & 1u)) { flags |= PT_SPAN_LINK; link = Sv[j2].z; } }
            // comment ids differ between x-1 and x?  only ids with a boundary exactly at x can change; presence of an id =
            // "its last-arrived covering op is an add" (peritext.ts:314-322)
            if (nC) {
                const bool live = s >= 1 && s < S && x > 0;
                bool cd = false;
                for (uint32_t cj = 0; cj < nC; cj++) {
                    const uint32_t j = CIdx[cj], ab = Sv[j].x;
                    const bool touch = live && ((ab & 0xFFFFu) == x || (ab >> 16) == x);
                    if (!__any_sync(kFull, touch)) continue;
                    const uint32_t id = Sv[j].z;
                    bool pPrev = false, pCur = false;
                    for (uint32_t c2 = 0; c2 < nC; c2++) {
                        const uint32_t j2 = CIdx[c2];
                        const uint4 s2 = Sv[j2];
                        if (s2.z != id) continue;                    // uniform
                        const uint32_t a2 = s2.x & 0xFFFFu, b2 = s2.x >> 16;
                        const bool add2 = !((s2.y >> 16) & 1u);
                        if (x - 1u >= a2 && x - 1u < b2) pPrev = add2;
                        if (x >= a2 && x < b2) pCur = add2;
                    }
                    if (touch && pPrev != pCur) cd = true;
                }
                if (cd) flags |= 16u;
            }
            if (s < S) { SegFlags[s] = flags; SegLink[s] = link; }
        }
        __syncwarp();
        // pass 2: span heads, span indices, comment counts
        uint32_t totalC = 0;
#pragma unroll 1
        for (uint32_t sb = 0; sb < S; sb += 32) {
            const uint32_t s = sb + lane;
            bool head = false;
            uint32_t cnt = 0;
            const uint32_t x = s < S ? (uint32_t)SegStart[s] : 0u;
            if (s < S) {
                const uint32_t f = SegFlags[s];
                if (s == 0) head = !seg0_empty;
                else if (x == 0) head = true;
                else head = ((f ^ SegFlags[s - 1]) & 0xFu) != 0 || SegLink[s] != SegLink[s - 1] || (f & 16u);
            }
            if (nC) {
                for (uint32_t cj = 0; cj < nC; cj++) {               // members: ids whose last-arrived covering op is an add
                    const uint32_t j = CIdx[cj], ab = Sv[j].x, id = Sv[j].z;
                    const bool cov = head && x >= (ab & 0xFFFFu) && x < (ab >> 16);
                    if (!__any_sync(kFull, cov)) continue;
                    bool later = false;
                    for (uint32_t c2 = cj + 1; c2 < nC; c2++) {
                        const uint32_t j2 = CIdx[c2];
                        if (Sv[j2].z != id) continue;
                        const uint32_t ab2 = Sv[j2].x;
                        if (x >= (ab2 & 0xFFFFu) && x < (ab2 >> 16)) later = true;
                    }
                    if (cov && !later && !((Sv[j].y >> 16) & 1u)) cnt++;
                }
            }
            const uint32_t hb = __ballot_sync(kFull, head);
            const uint32_t inc = warp_incl_scan(cnt, lane);
            __syncwarp();                                            // every lane has read its left neighbour's flags
            if (s < S) {
                SegFlags[s] = (SegFlags[s] & 0x1Fu) | (head ? 32u : 0u);
                SegCnt[s] = (uint16_t)cnt;
                SegOut[s] = (uint16_t)(nspans + __popc(hb & lt));
                SegCOff[s] = totalC + inc - cnt;
            }
            nspans += __popc(hb);
            totalC += __shfl_sync(kFull, inc, 31);
            __syncwarp();
        }
        if (totalC) {
            uint32_t pst = 0;
            if (lane == 0) pool_base = pool_reserve(P, totalC, pst);
            pst = __shfl_sync(kFull, pst, 0);
            if (pst) { bail(pst); ps.leave(); return 0; }
            pool_base = __shfl_sync(kFull, pool_base, 0);
        }
        __syncwarp();
        // pass 3: span records, comment lists (ascending id, sortBy peritext.ts:318), digest
        uint32_t* pool = P.comment_pool + pool_base;
#pragma unroll 1
        for (uint32_t sb = 0; sb < S; sb += 32) {
            const uint32_t s = sb + lane;
            const bool head = s < S && (SegFlags[s] & 32u);
            const uint32_t x = s < S ? (uint32_t)SegStart[s] : 0u;
            const uint32_t cnt = head ? (uint32_t)SegCnt[s] : 0u, off = head ? SegCOff[s] : 0u;
            if (nC && __any_sync(kFull, cnt != 0)) {
                uint32_t filled = 0;
                for (uint32_t cj = 0; cj < nC; cj++) {
                    const uint32_t j = CIdx[cj], ab = Sv[j].x, id = Sv[j].z;
                    const bool cov = cnt != 0 && x >= (ab & 0xFFFFu) && x < (ab >> 16);
                    if (!__any_sync(kFull, cov)) continue;
                    bool later = false;
                    for (uint32_t c2 = cj + 1; c2 < nC; c2++) {
                        const uint32_t j2 = CIdx[c2];
                        if (Sv[j2].z != id) continue;
                        const uint32_t ab2 = Sv[j2].x;
                        if (x >= (ab2 & 0xFFFFu) && x < (ab2 >> 16)) later = true;
                    }
                    if (cov && !later && !((Sv[j].y >> 16) & 1u)) {  // insert in ascending id order (lists are short)
                        uint32_t y = filled;
                        while (y > 0 && pool[off + y - 1] > id) { pool[off + y] = pool[off + y - 1]; y--; }
                        pool[off + y] = id; filled++;
                    }
                }
            }
            if (head) {
                const uint32_t jo = SegOut[s];
                pt_span sp; sp.start = x; sp.flags = (SegFlags[s] & 0xFu) | (cnt << 8); sp.link_attr = SegLink[s];
                sp.comment_off = cnt ? (uint32_t)(pool_base + off) : 0u;
                span_out[jo] = sp;
                for (uint32_t y = 0; y < cnt; y++) digest_add(d0, d1, pt_term_comment(jo, y, pool[off + y]));
                digest_add(d0, d1, pt_term_span(jo, sp.start, sp.flags, sp.link_attr));
            }
        }
        }   // segment form
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(kFull, d0, o); d1 ^= __shfl_xor_sync(kFull, d1, o); }
    if (lane == 0) {
        pt_log_result r;
        r.status = PT_LOG_OK; r.n_elems = N; r.n_visible = nvis; r.n_spans = nspans;
        const uint64_t t = pt_term_counts(nvis, nspans);
        r.digest[0] = d0 + t; r.digest[1] = d1 ^ pt_term_hi(t);
        *res = r;
    }
    PT_PHASE(kPhI);
#ifdef PT_PHASE_CLOCKS
    pclk.logs++;
#endif
    ps.leave();
    return 0;
}

// Persistent warps: every warp pulls logs (largest first) from the bin's work queue.  Two modes:
//   free  : each warp takes kWarpGrab logs per atomic and runs on its own;
//   phased: (warp_flags bit 2, the default) the CTA takes one log per warp per ROUND: its warps start a round together (consecutive
//           logs of the size-sorted queue are nearly the same size, so they also finish together) and share the instruction caches;
//           the named barriers at the phase boundaries INSIDE a log are optional (bits 8-11 skip them; default: only the last one).
template <int WARPS, int IDM>
__global__ void __launch_bounds__(WARPS * 32, (32 / WARPS) > 0 ? (32 / WARPS) : 1) merge_logs_warp_kernel(const BatchParams P) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t n_work = P.n_work;
    const uint32_t slice = P.smem_arena_bytes;
    uint32_t base = warp * slice;
    asm volatile("" : "+r"(base));         // opaque: keep it in a register instead of re-deriving it from threadIdx at every shared-memory access
    uint32_t done = 0, deferred = 0;
    const bool phased = (P.warp_flags & 4u) != 0;
    __shared__ uint32_t s_base[2], s_nxt[2];
    PhaseSync ps; ps.on = phased ? 1u : 0u; ps.nthreads = WARPS * 32; ps.next = kFirstPhaseBar; ps.skip = (P.warp_flags >> 8) & 0xFu;
    uint32_t nextb = 0, nextb2 = 0, par = 0;   // phased: the CTA's next two rounds (held by thread 0)
    uint32_t w = 0, wend = 0, wn = 0;      // free: this warp's current grab [w, wend) and the next one
#ifdef PT_PHASE_CLOCKS
    PhaseClock pclk{};
    pclk.t = clock64();
#endif
    if (phased) { if (threadIdx.x == 0) { nextb = atomicAdd(P.work_counter, (uint32_t)WARPS); nextb2 = atomicAdd(P.work_counter, (uint32_t)WARPS); } }
    else {
        if (lane == 0) { w = atomicAdd(P.work_counter, kWarpGrab); wn = atomicAdd(P.work_counter, kWarpGrab); }
        w = __shfl_sync(kFull, w, 0); wn = __shfl_sync(kFull, wn, 0);
        wend = min(w + kWarpGrab, n_work);
    }
    for (;;) {
        uint32_t x, xn = 0xFFFFFFFFu;
        if (phased) {
            // the round after this one is known too (fetched a round ago): its logs' records can be on their way to L2
            if (threadIdx.x == 0) { s_base[par] = nextb; s_nxt[par] = nextb2; nextb = nextb2; nextb2 = atomicAdd(P.work_counter, (uint32_t)WARPS); }
            asm volatile("barrier.sync 1, %0;" ::"r"((uint32_t)(WARPS * 32)) : "memory");
            const uint32_t b0 = s_base[par], bn = s_nxt[par];
            par ^= 1u;
            if (b0 >= n_work) break;
            x = b0 + warp;
            xn = bn + warp;
            ps.next = kFirstPhaseBar;
        } else {
            if (w >= wend) {
                w = wn;
                if (w >= n_work) break;
                if (lane == 0) wn = atomicAdd(P.work_counter, kWarpGrab);
                wn = __shfl_sync(kFull, wn, 0);
                wend = min(w + kWarpGrab, n_work);
            }
            x = w++;
            xn = w < wend ? w : wn;
        }
        PT_PHASE(kPhRound);
        if (x < n_work) {
            const uint32_t li = P.order[x];
            if (P.admit && P.admit[li]) { ps.leave(); continue; }      // rejected by the admission pre-pass
            const uint32_t li_next = ((P.warp_flags & 2u) && xn < n_work) ? P.order[xn] : 0xFFFFFFFFu;
            const int rc = warp_merge_one_log<IDM>(P, li, base, slice, li_next, ps PT_PHASE_ARG);   // the host put the log in the right launch
            __syncwarp();
            if (rc) { if (lane == 0) P.retry_list[atomicAdd(P.retry_count, 1u)] = li; deferred++; } else done++;
        } else ps.leave();
    }
    if (lane == 0) {
        if (done) atomicAdd(&P.stats[0], (unsigned long long)done);
        if (deferred) atomicAdd(&P.stats[2], (unsigned long long)deferred);
#ifdef PT_PHASE_CLOCKS
        for (int k = 0; k < kNumPhases; k++) atomicAdd(&ptk_phase_clk[k], pclk.c[k]);
        atomicAdd(&ptk_phase_clk[kNumPhases], pclk.logs);
#endif
    }
}

}  // namespace ptk
