/* peritext_b200.h — C-ABI of the H100 batch CRDT-merge engine (libperitext_b200.so).
 *
 * Drop-in boundary for ONE hot path of inkandswitch/peritext: replaying op logs and flattening the
 * documents to formatted spans, i.e. what the reference does in
 *     Micromerge.applyChange -> applyOp          (reference src/micromerge.ts:499-608)
 *     applyListInsert / applyListUpdate           (src/micromerge.ts:614-724)
 *     applyAddRemoveMark                          (src/peritext.ts:154-249)
 *     getTextWithFormatting / addCharactersToSpans(src/peritext.ts:337-455)
 * for MANY (document, replica) op logs at once.  The reference has no FFI seam (it is pure TypeScript);
 * these entry points are what an N-API addon behind a `Micromerge` facade binds (see INTEGRATION.md).
 *
 * Conventions: plain C types only, no C++/torch types; every function returns a pt_status code (never
 * throws); device work is enqueued on the CUDA stream handle given at create time; host buffers passed
 * in are owned by the caller.  PAGEABLE input buffers may be freed as soon as the call returns (the call
 * waits for the copy); buffers in PINNED (page-locked) memory are read asynchronously by the copy engine and
 * must stay valid until the next synchronising call on the handle (pt_batch_sync, pt_batch_download*,
 * pt_batch_last_merge_ms, the next pt_batch_upload*).
 */
#ifndef PERITEXT_B200_H
#define PERITEXT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Packed op records (host and device layout are identical; little endian).
 *
 * One LOG = the ops one replica applied to one text list, in that replica's arrival order
 * (the concatenation of `change.ops` over its applyChange calls, src/micromerge.ts:513).
 * opIds "ctr@actor" (src/micromerge.ts:488) are packed as (ctr, actor_rank) where actor_rank is the rank
 * of the actorId among the log's actors in JS string order (UTF-16 code units), so that
 * compareOpIds (src/micromerge.ts:812-827) == compare (ctr, actor_rank) lexicographically.
 * ---------------------------------------------------------------------------------------------- */

/* Insert (`action:"set", insert:true`, src/micromerge.ts:150-160) or delete (`action:"del"`, :162-168). 16 B. */
typedef struct pt_insdel_rec {
    uint32_t ctr;       /* opId counter (>=1)                                                     */
    uint32_t ref_ctr;   /* insert: reference elemId counter, 0 = HEAD; delete: target elemId ctr */
    uint16_t actor;     /* opId actor rank                                                        */
    uint16_t ref_actor; /* reference / target elemId actor rank                                   */
    uint32_t payload;   /* bits31:30 kind (PT_KIND_*); insert: bit29 = value-pool flag, bits28:0 =
                           Unicode code point (single-character value) or value-pool index        */
} pt_insdel_rec;

#define PT_KIND_INSERT 0u
#define PT_KIND_DELETE 1u
#define PT_PAYLOAD_KIND(p) ((uint32_t)(p) >> 30)
#define PT_PAYLOAD_TOKEN(p) ((uint32_t)(p) & 0x3FFFFFFFu)
#define PT_TOKEN_POOLED 0x20000000u

/* addMark / removeMark (src/peritext.ts:25-65). 32 B. */
typedef struct pt_mark_rec {
    uint32_t ctr;         /* opId counter                                                         */
    uint16_t actor;       /* opId actor rank                                                      */
    uint8_t  kind;        /* bit0: 0 addMark, 1 removeMark; bits2:1 mark type (PT_MARK_*)          */
    uint8_t  bounds;      /* bits1:0 start boundary type, bits3:2 end boundary type (PT_BOUND_*)   */
    uint32_t start_ctr;   /* start.elemId counter (before/after only)                              */
    uint32_t end_ctr;     /* end.elemId counter (before/after only)                                */
    uint16_t start_actor; /* start.elemId actor rank                                               */
    uint16_t end_actor;   /* end.elemId actor rank                                                 */
    uint32_t attr;        /* link: interned url id; comment: comment-id rank (JS string order of
                             the id, per batch); PT_ATTR_NONE otherwise                           */
    uint32_t arrival;     /* number of ins/del records of this log that arrived before this op   */
    uint32_t reserved;    /* 0                                                                     */
} pt_mark_rec;

/* Mark types in ALL_MARKS order (src/schema.ts:125). strong/em: inclusive, single; comment:
 * non-inclusive, allowMultiple; link: non-inclusive, single (src/schema.ts:45-96). */
#define PT_MARK_STRONG 0u
#define PT_MARK_EM 1u
#define PT_MARK_COMMENT 2u
#define PT_MARK_LINK 3u
#define PT_BOUND_BEFORE 0u
#define PT_BOUND_AFTER 1u
#define PT_BOUND_START_OF_TEXT 2u
#define PT_BOUND_END_OF_TEXT 3u
#define PT_ATTR_NONE 0xFFFFFFFFu

/* Per-log descriptor. 32 B. */
typedef struct pt_log_desc {
    uint64_t insdel_off; /* first pt_insdel_rec of the log in the batch's insdel array            */
    uint64_t mark_off;   /* first pt_mark_rec of the log in the batch's mark array                */
    uint32_t n_insdel;
    uint32_t n_mark;
    uint32_t n_actors;   /* actor ranks are < n_actors                                             */
    uint32_t max_ctr;    /* every ctr in the log is in [1, max_ctr]                                */
} pt_log_desc;

/* ------------------------------------------------------------------------------------------------
 * Run-compressed wire format (optional, for the host -> device leg).  The ops of one Change are
 * consecutive (`opId = ++maxOp`, src/micromerge.ts:487) and a typed run chains every insert to the
 * previous one (`elemId = result`, :351-359), so the ins/del stream compresses to RUNS:
 *   insert run: `count` inserts with opIds (ctr0 + k, actor); the first references (ref_ctr, ref_actor),
 *               each following one references its predecessor; values = `count` tokens of the token stream
 *   delete run: `count` deletes with opIds (ctr0 + k, actor) of the elements (ref_ctr + k, ref_actor)
 * pt_batch_upload_runs expands runs to pt_insdel_rec on the device; results are identical.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_run_rec {
    uint32_t ctr0;
    uint32_t ref_ctr;
    uint16_t actor;
    uint16_t ref_actor;
    uint32_t kind_count; /* bits31:30 kind (PT_KIND_*), bits29:0 count (>= 1) */
} pt_run_rec;

typedef struct pt_packed_runs {
    uint32_t n_logs;
    const pt_log_desc* logs;      /* [n_logs] — the EXPANDED layout (insdel_off / n_insdel count records)      */
    const uint64_t* run_off;      /* [n_logs + 1] first run of each log                                         */
    const uint64_t* tok_off;      /* [n_logs + 1] first insert token of each log                                */
    const pt_run_rec* runs;       /* [run_off[n_logs]]                                                          */
    const uint32_t* tokens;       /* [tok_off[n_logs]] PT_PAYLOAD_TOKEN values of the inserts, in record order  */
    const pt_mark_rec* marks;     /* [n_mark_total] (not compressed)                                            */
    uint64_t n_insdel_total;      /* expanded record count                                                      */
    uint64_t n_mark_total;
} pt_packed_runs;

/* ------------------------------------------------------------------------------------------------
 * Change table (optional): what Micromerge.applyChange checks BEFORE it applies a change
 * (src/micromerge.ts:499-511): seq == clock[actor] + 1, and every deps[a] <= clock[a] (a missing or
 * zero clock entry fails).  One pt_change_rec per Change the replica applied, in arrival order; the
 * admission pre-pass (pt_batch_upload_changes) validates every log on the device and reports the
 * first rejected change as the log's status instead of throwing mid-batch; such a log is not merged.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_change_rec {   /* 16 B */
    uint32_t seq;     /* change.seq                                                                */
    uint16_t actor;   /* change.actor, rank among the log's actors (same ranks as the op records)  */
    uint16_t n_deps;  /* entries of change.deps                                                    */
    uint32_t dep_off; /* first pt_dep_rec of the change, relative to the log's dep_off             */
    uint32_t n_ops;   /* ops of the change that target the log's text list (informational)         */
} pt_change_rec;
typedef struct pt_dep_rec {      /* 8 B */
    uint32_t seq;
    uint16_t actor;
    uint16_t reserved;
} pt_dep_rec;
typedef struct pt_change_desc {  /* 24 B */
    uint64_t change_off;
    uint64_t dep_off;
    uint32_t n_changes;
    uint32_t n_deps;
} pt_change_desc;
typedef struct pt_change_table {
    uint32_t n_logs;              /* must equal the uploaded batch's n_logs */
    const pt_change_desc* logs;
    const pt_change_rec* changes;
    uint64_t n_changes_total;
    const pt_dep_rec* deps;
    uint64_t n_deps_total;
} pt_change_table;

/* ------------------------------------------------------------------------------------------------
 * Compact wire format (optional, for the host -> device leg): the same records in half the bytes.
 * Usable for a log with max_ctr < 65536, n_insdel < 65536 and n_actors <= 16 (any document the
 * benchmark shapes produce); value tokens must fit 22 bits (any Unicode code point, or a value-pool
 * index < 2^21).  Every record field must fit its compact width on its own, whatever the descriptor
 * says: ctr, ref_ctr, start_ctr, end_ctr and arrival < 65536; actor, ref_actor, start_actor and
 * end_actor < 16; mark kind < 8 and bounds < 16.  pt_compact_ops refuses a batch with any other
 * record (naming the field), so a faulty record is never truncated into a valid one.  Records keep their positions (the descriptors are those of the expanded layout);
 * pt_batch_upload_compact expands them to pt_insdel_rec / pt_mark_rec on the device, elementwise.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_insdel_c8 {   /* 8 B */
    uint16_t ctr, ref_ctr;
    uint32_t w;                 /* bits3:0 actor, 7:4 ref_actor, 9:8 kind, 31:10 token (bit21 of the token = value-pool flag) */
} pt_insdel_c8;
typedef struct pt_mark_c16 {    /* 16 B */
    uint16_t ctr, start_ctr, end_ctr, arrival;
    uint32_t attr;
    uint32_t w;                 /* bits3:0 actor, 7:4 start_actor, 11:8 end_actor, 14:12 kind, 18:15 bounds */
} pt_mark_c16;
typedef struct pt_packed_compact {
    uint32_t n_logs;
    const pt_log_desc* logs;       /* the EXPANDED layout */
    const pt_insdel_c8* insdel;    /* [n_insdel_total] */
    uint64_t n_insdel_total;
    const pt_mark_c16* marks;      /* [n_mark_total] */
    uint64_t n_mark_total;
} pt_packed_compact;

/* A host-side batch of logs (SoA). */
typedef struct pt_packed_ops {
    uint32_t n_logs;
    const pt_log_desc* logs;     /* [n_logs]                 */
    const pt_insdel_rec* insdel; /* [sum n_insdel]           */
    uint64_t n_insdel_total;
    const pt_mark_rec* marks;    /* [sum n_mark]             */
    uint64_t n_mark_total;
} pt_packed_ops;

/* ------------------------------------------------------------------------------------------------
 * Results
 * ---------------------------------------------------------------------------------------------- */

/* Per-log status; each maps to a reference throw site. */
#define PT_LOG_OK 0u
#define PT_LOG_ELEM_NOT_FOUND 1u /* "List element not found" src/micromerge.ts:752                 */
#define PT_LOG_BAD_OPID 2u       /* ctr/actor outside the descriptor's bounds, or duplicate opId   */
#define PT_LOG_BAD_KIND 3u       /* record kind not insert/delete                                  */
#define PT_LOG_OVERFLOW 4u       /* an engine capacity (comment pool / scratch) was exceeded       */
#define PT_LOG_CYCLE 5u          /* reference elemId does not causally precede the insert (a peer chose a startOp below
                                    an element it references: the reference would still merge it; this engine's
                                    closed form needs Lamport counters, src/micromerge.ts:487,511)                */
#define PT_LOG_SEQ_GAP 6u        /* admission: "Expected sequence number ..." src/micromerge.ts:501-504; n_elems =
                                    index of the rejected change in the log                                        */
#define PT_LOG_MISSING_DEP 7u    /* admission: "Missing dependency ..." src/micromerge.ts:505-509; n_elems = index of
                                    the rejected change                                                            */

/* Per-log result header. 32 B. */
typedef struct pt_log_result {
    uint32_t status;    /* PT_LOG_*                                                                */
    uint32_t n_elems;   /* list elements incl. tombstones (metadata.length)                        */
    uint32_t n_visible; /* visible elements (text.length, src/micromerge.ts:657)                   */
    uint32_t n_spans;   /* FormatSpanWithText count (src/peritext.ts:361)                          */
    uint64_t digest[2]; /* 128-bit digest of (text tokens, spans, marks) — convergence check       */
} pt_log_result;

/* One formatted span (src/peritext.ts:35-38). 16 B. Text of span j = tokens [start_j, start_{j+1}). */
typedef struct pt_span {
    uint32_t start;       /* index of the span's first visible element                             */
    uint32_t flags;       /* bit0 strong, bit1 em, bit2 link present, bit3 `comment` key present;
                             bits31:8 number of comment ids                                        */
    uint32_t link_attr;   /* url id if bit2, else PT_ATTR_NONE                                     */
    uint32_t comment_off; /* first comment id of the span in the comment pool (ascending ids)      */
} pt_span;

#define PT_SPAN_STRONG 1u
#define PT_SPAN_EM 2u
#define PT_SPAN_LINK 4u
#define PT_SPAN_COMMENT 8u
#define PT_SPAN_NCOMMENTS(f) ((uint32_t)(f) >> 8)

/* Host view of a merged batch; pointers are engine-owned pinned host memory, valid until the next
 * pt_batch_upload/pt_batch_destroy on the handle. The outputs are PACKED on the device before the copy: log i's
 * tokens are text[text_off[i] .. text_off[i+1]), its spans spans[span_off[i] .. span_off[i+1]). */
typedef struct pt_spans_view {
    uint32_t n_logs;
    const pt_log_result* results; /* [n_logs]                                                      */
    const uint64_t* text_off;     /* [n_logs + 1] packed offsets (exclusive scan of n_visible)      */
    const uint64_t* span_off;     /* [n_logs + 1] packed offsets (exclusive scan of n_spans)        */
    const uint32_t* text;         /* visible element value tokens (PT_PAYLOAD_TOKEN)               */
    const pt_span* spans;
    const uint32_t* comment_pool;
    uint64_t comment_pool_used;
    const uint32_t* seq;          /* NULL unless PT_FLAG_EMIT_SEQUENCE: per log (offset seq_off[i], n_elems entries) the element
                                     sequence incl. tombstones (the reference's `metadata` array, src/micromerge.ts:255):
                                     bits29:0 = index of the element's insert record in the log's ins/del records,
                                     bit30 = the element's markOpsAfter slot is defined (src/micromerge.ts:784),
                                     bit31 = deleted                                                                  */
    const uint64_t* seq_off;      /* [n_logs] offsets into seq (capacity layout: running sum of n_insdel); NULL without seq */
    uint64_t comment_pool_needed; /* comment-pool entries the whole batch needs; > the pool's capacity iff some logs
                                     reported PT_LOG_OVERFLOW: call pt_batch_set_comment_pool(needed) and merge again  */
} pt_spans_view;

/* Engine limits / tuning. Zero-initialise for defaults. */
typedef struct pt_limits {
    uint64_t comment_pool_entries; /* 0: 4 x number of mark ops in the batch (+slack)             */
    uint32_t flags;                /* PT_FLAG_*                                                     */
    uint32_t patch_pool_items;     /* 0: 4 x number of op records in the batch (+slack)            */
    uint32_t reserved[4];
} pt_limits;
#define PT_FLAG_EMIT_SEQUENCE 1u   /* also emit the element sequence (needed by op generation / cursors on the host) */
#define PT_FLAG_EMIT_PATCHES 2u    /* also derive the Patch stream of every op on the device (implies EMIT_SEQUENCE) */
/* Also derive on the device the Patch stream of the logs the warp patch kernel declines (max_ctr x n_actors >= 0xFFFF, or
 * tables above its 200 KB of shared memory), with a CTA-per-log arrival sweep (implies EMIT_PATCHES).  Then a log's patch
 * status is 1 only if its merge failed (admission-rejected logs included); its records, items and item demand are what
 * the warp kernel's contract below defines, window and pool rules included.  Cost: one more launch per merge when the
 * batch has such logs, and a global scratch slab of min(such logs, SMs) slots, each sized by the largest such log
 * (4 B per key of max_ctr x n_actors + ~13 B per ins/del record + 64 x next_pow2(2 n_mark + 1) B of mark trees + ~56 B
 * per mark op, i.e. 180-320 B per mark op; the exact formula is ptp::large_layout in csrc/plan.h); pt_batch_upload /
 * pt_batch_append fail with PT_ERR_NOMEM if it cannot be allocated. */
#define PT_FLAG_EMIT_LARGE_PATCHES 4u

/* ------------------------------------------------------------------------------------------------
 * Patch stream (PT_FLAG_EMIT_PATCHES): what Micromerge.applyChange returns for every op of a log, given the
 * log's arrival order (src/micromerge.ts:659-671, 689-703; src/peritext.ts:175-220, 251-281).
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_patch_rec {   /* one per ins/del record, at the record's offset. 16 B */
    uint32_t index;     /* bits30:0: Patch.index (visible elements left of the op's element at apply time);
                           bit31: the op emits a patch (inserts always; a delete only if it is the element's first) */
    uint32_t flags;     /* insert: the `marks` of the patch = marks inherited from the left neighbour at apply time
                           (getActiveMarksAtIndex, src/peritext.ts:328): PT_SPAN_* bits, bits31:8 number of comment ids  */
    uint32_t link_attr; /* url id if PT_SPAN_LINK                                                                 */
    uint32_t reserved;
} pt_patch_rec;
typedef struct pt_patch_item {  /* pool entry, any order. 16 B */
    uint32_t log;       /* log index                                                                             */
    uint32_t tag;       /* bit31 set: mark patch of mark record (tag & 0x7FFFFFFF): a = startIndex, b = endIndex;
                           bit31 clear: comment id `a` in the `marks` of the insert patch of ins/del record `tag`       */
    uint32_t a, b;
} pt_patch_item;
typedef struct pt_patch_view {
    const pt_patch_rec* recs;      /* [n_insdel_total]                                                            */
    const pt_patch_item* items;    /* [n_items]                                                                   */
    uint64_t n_items;
    uint64_t n_items_needed;       /* > the pool's capacity: call pt_batch_set_patch_pool(needed) and merge again */
    const uint32_t* status;        /* [n_logs] 0: computed; 1: not computed (log too large for the device patch kernel or
                                      merge failed; with PT_FLAG_EMIT_LARGE_PATCHES merge failed only) — derive on the host */
} pt_patch_view;

typedef enum pt_status {
    PT_OK = 0,
    PT_ERR_INVALID = 1,   /* bad argument                                                          */
    PT_ERR_CUDA = 2,      /* CUDA runtime error (see pt_last_error)                                */
    PT_ERR_NO_DEVICE = 3, /* no usable sm_90 device                                                */
    PT_ERR_STATE = 4,     /* call out of order (e.g. merge before upload)                          */
    PT_ERR_NOMEM = 5
} pt_status;

typedef struct pt_batch pt_batch; /* opaque; one per (GPU, batch); not thread-safe per handle */

/* Create an engine handle on CUDA device `device`; work is enqueued on `cuda_stream`
 * (a cudaStream_t / CUstream passed as void*, NULL = legacy default stream). */
int pt_batch_create(int device, const pt_limits* limits, void* cuda_stream, pt_batch** out);

/* Copy a packed batch host -> device (asynchronous on the handle's stream for pinned inputs, see the buffer
 * rule above; the descriptors are staged through engine-owned pinned memory). Waits for the handle's previous
 * work first. Replaces any previous batch.
 * This is the H2D leg of Micromerge.applyChange's input (src/micromerge.ts:499). */
int pt_batch_upload(pt_batch*, const pt_packed_ops* host_ops);

/* Same as pt_batch_upload for the run-compressed form: copies runs / tokens / marks host -> device and expands the runs
 * to pt_insdel_rec records on the device (one small kernel).  Typically 2-3x fewer bytes over PCIe.  The run table is
 * checked on the host first (PT_ERR_INVALID, nothing copied): run_off / tok_off start at 0 and never decrease, every count
 * is >= 1, and per log the counts sum to n_insdel and the insert counts to the log's token span. */
int pt_batch_upload_runs(pt_batch*, const pt_packed_runs* host_runs);

/* Host helper: compress a packed batch into runs.  Call once with runs == NULL / tokens == NULL to get the counts
 * (*n_runs, *n_tokens), then with buffers of that size; run_off / tok_off need n_logs + 1 entries. */
int pt_compress_runs(const pt_packed_ops* ops, uint64_t* run_off, uint64_t* tok_off, pt_run_rec* runs, uint32_t* tokens,
                     uint64_t* n_runs, uint64_t* n_tokens);

/* Attach the change table of the uploaded batch (host arrays, copied): the next pt_batch_merge first runs the
 * admission pre-pass on the device; logs with a sequence gap / missing dependency get PT_LOG_SEQ_GAP /
 * PT_LOG_MISSING_DEP and are skipped by the merge (the reference throws before mutating, src/micromerge.ts:501-509).
 * Call after pt_batch_upload*; a new upload drops the table. */
int pt_batch_upload_changes(pt_batch*, const pt_change_table* host_changes);

/* Host helper (multithreaded): convert a packed batch to the compact wire format into caller-provided arrays of
 * n_insdel_total / n_mark_total entries.  PT_ERR_INVALID (nothing useful written) if some log or record is not
 * representable (the rules above the compact records). */
int pt_compact_ops(const pt_packed_ops* ops, pt_insdel_c8* insdel_out, pt_mark_c16* marks_out, int threads /* 0 = all cores */);

/* Same as pt_batch_upload for the compact form: half the bytes over PCIe, expanded on the device (two elementwise kernels). */
int pt_batch_upload_compact(pt_batch*, const pt_packed_compact* host_compact);

/* Adopt a batch that is ALREADY RESIDENT in device memory (pointers are device pointers owned by the
 * caller, e.g. torch tensors); only the descriptors are read on the host.  The records are also read at adopt time, on
 * the handle's stream, to derive the warp kernel's half-width copy of them: after an in-place change to the adopted
 * arrays, adopt them again before the next merge. */
int pt_batch_adopt_device(pt_batch*, const pt_packed_ops* host_desc_device_arrays);

/* ------------------------------------------------------------------------------------------------
 * Append: extend every log of the resident batch with new records on the device, so that a re-merge after a few new
 * changes (Micromerge.applyChange on a document that already exists, src/micromerge.ts:499) uploads only what is new.
 * After a successful append the handle holds exactly the batch an upload of the concatenated logs would hold: logs
 * contiguous and in order, each with its old records first and then its delta records; the same descriptors, plan and
 * change table.
 *
 * Three packed id spaces carry an ORDER, and new changes can move every existing id in them: the per-log actor rank
 * (a new actor that sorts before the old ones), the per-log dense counter rank (where the packer re-ranked sparse
 * counters; a log can also switch between dense and plain counters as it grows) and the per-batch comment rank.  The
 * remap says how the resident records' ids move; value-pool indices and link attr ids carry no order and never move.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_append_remap {      /* NULL pointer = identity everywhere */
    const uint64_t* actor_off;        /* [n_logs + 1] or NULL: log i's map is actor_map[actor_off[i] .. actor_off[i+1]),
                                         old rank -> new rank; empty = identity, else exactly the log's old n_actors
                                         entries, strictly increasing                                                   */
    const uint16_t* actor_map;
    const uint64_t* ctr_off;          /* [n_logs + 1] or NULL: log i's map is ctr_map[ctr_off[i] .. ctr_off[i+1]), old
                                         ctr -> new ctr; empty = identity, else at least old max_ctr + 1 entries (more
                                         where a record names a counter past max_ctr, e.g. a mark boundary on an element
                                         inserted later), entry 0 = 0 (HEAD), strictly increasing over the entries that are not
                                         0xFFFFFFFF; 0xFFFFFFFF marks an old counter that no record of the log names
                                         (a plain log turning dense: the dense ranks leave no room for unused values)   */
    const uint32_t* ctr_map;
    const uint32_t* comment_map;      /* old comment rank -> new rank, n_comment_map entries, strictly increasing;
                                         NULL = identity                                                                */
    uint64_t n_comment_map;
} pt_append_remap;

/* Append `delta` to the resident batch.  The delta has the batch's n_logs; descriptor i indexes the delta's own arrays and
 * counts only log i's NEW records (zero is allowed); its n_actors / max_ctr are the log's values AFTER the append.  Delta
 * records are already in the new id space.  A delta mark's arrival counts the ins/del records of the whole log, so it lies
 * in [old n_insdel, old n_insdel + delta n_insdel].  delta_changes is the change table of the new changes (NULL iff the
 * handle has no change table); a delta change record's dep_off is relative to its delta log's deps (the engine rebases it).
 * Resident records: actor ranks go through the log's actor map, counters (ctr, ref_ctr, start_ctr, end_ctr) through its
 * counter map, and the attr of a comment mark through the comment map.  An id whose counter is 0 (HEAD, start / end of
 * text) keeps its actor field.  A resident value outside its map's domain (actor >= old n_actors, ctr > old max_ctr) or
 * mapped to 0xFFFFFFFF becomes 0xFFFF / 0xFFFFFFFF, so a faulty log still fails at merge; identity maps copy verbatim.  The
 * change table is concatenated per log, and the old change and dep records' actor ranks go through the actor maps.
 * Refused before anything changes (PT_ERR_INVALID, pt_last_error names the problem): n_logs differs; a map has the wrong
 * length or is not strictly increasing; ctr_map[0] != 0; a mapped old bound (identity included; for the counter map, the
 * image of the old max_ctr) exceeds the new n_actors / max_ctr; a delta descriptor or arrival is out of range; a log would exceed 2^32 - 1 records; a change table on one side
 * only.  No batch: PT_ERR_STATE.  The device refuses too: a resident comment rank (other than PT_ATTR_NONE) outside
 * comment_map, or mapped to 0xFFFFFFFF, gives PT_ERR_INVALID with the batch untouched, because the splice writes new record buffers and only a
 * successful one replaces the old.
 * On success: the batch is re-planned like an upload (routes, capacities and the patch kernel's shared memory can change),
 * there is no merge (views of the last merge are invalid, as after an upload), comment-pool and patch-pool settings persist
 * as across uploads, and the records are engine-owned, also after pt_batch_adopt_device (whose arrays it only reads).
 * Synchronises; the caller's arrays may be freed on return.
 * Device: one warp per log (up to 64 for a log with many records) copies the old records with coalesced 16-byte accesses,
 * applying the log's maps (a log with identity maps is a straight copy), then the delta records; a second warp-per-log
 * kernel splices the change and dep tables.  Peak device memory during the call: old + delta + new records (and change
 * tables).  The delta, remap and change-table copies on the device are freed on return; the handle keeps only the new
 * batch. */
int pt_batch_append(pt_batch*, const pt_packed_ops* delta, const pt_append_remap* remap, const pt_change_table* delta_changes);

/* ------------------------------------------------------------------------------------------------
 * Local changes: Micromerge.change (src/micromerge.ts:308-441, changeMark src/peritext.ts:458-501) for many documents at
 * once.  Each log's InputOperations are resolved on the device against the document of the last merge, in order, each
 * generated op applied before the next (so an index refers to the document after the earlier InputOperations of the same
 * change), and the generated records are appended to the resident batch without leaving the device.
 * ---------------------------------------------------------------------------------------------- */
#define PT_INPUT_INSERT 0u
#define PT_INPUT_DELETE 1u
#define PT_INPUT_ADD_MARK 2u
#define PT_INPUT_REMOVE_MARK 3u
typedef struct pt_input_op {   /* one InputOperation on the log's text list. 32 B */
    uint8_t  action;     /* PT_INPUT_*                                                                                */
    uint8_t  mark_type;  /* marks: PT_MARK_*; 0 otherwise                                                             */
    uint16_t reserved0;  /* 0                                                                                         */
    int32_t  index;      /* insert / delete: index; marks: startIndex (negative: out of bounds, as in the reference)  */
    int32_t  arg;        /* insert: number of values (>= 0); delete: count (<= 0 generates nothing); marks: endIndex    */
    uint32_t attr;       /* marks: as pt_mark_rec.attr (link url id < n_links, comment rank < n_comments; PT_ATTR_NONE
                            for strong / em); PT_ATTR_NONE otherwise                                                  */
    uint32_t first_ctr;  /* packed counter of the first op the record generates; op j gets first_ctr + j (makeNewOp,
                            src/micromerge.ts:483-493).  A record that generates no op still needs a value > the log's
                            max_ctr and >= the previous record's next counter                                         */
    uint32_t reserved1;  /* 0                                                                                         */
    uint64_t tok_off;    /* insert: its `arg` value tokens are tokens[tok_off ..] (PT_PAYLOAD_TOKEN values: a code point
                            <= 0x10FFFF, or PT_TOKEN_POOLED | value-pool index < n_values)                             */
} pt_input_op;
#define PT_CHANGE_NO_ACTOR 0xFFFFFFFFu
typedef struct pt_change_input {
    uint32_t n_logs;             /* must equal the batch's n_logs                                                       */
    const uint32_t* actor;       /* [n_logs] the acting actor's rank in the log, or PT_CHANGE_NO_ACTOR: no change        */
    const uint64_t* input_off;   /* [n_logs + 1] log i's InputOperations are ops[input_off[i] .. input_off[i+1]), in the
                                    change's order (a log without an actor must have none)                              */
    const pt_input_op* ops;
    const uint32_t* tokens;      /* [n_tokens] */
    uint64_t n_tokens;
    uint32_t n_values, n_links, n_comments;   /* the pools the tokens and attrs index (bounds of the checks above)     */
    uint32_t reserved;
} pt_change_input;
#define PT_CHANGE_OK 0u
#define PT_CHANGE_OUT_OF_BOUNDS 1u   /* "List index out of bounds" (src/micromerge.ts:804): the log appends nothing */
typedef struct pt_change_status { uint32_t status; uint32_t input; } pt_change_status;   /* 8 B; input: the failing
                                                    InputOperation relative to the log's first, 0xFFFFFFFF when OK */
typedef struct pt_change_view {
    uint32_t n_logs;
    const pt_change_status* status;   /* [n_logs]                                                                     */
    pt_packed_ops delta;              /* the generated records: descriptor i = log i's new records (n_insdel = n_mark = 0
                                         for a failed log or one without a change), with the log's n_actors and new max_ctr */
} pt_change_view;

/* Generate every log's local change from its InputOperations on the device and append the generated records to the resident
 * batch.  Per InputOperation, against the document of the last merge with the earlier generated ops applied (exactly the list
 * ops of Micromerge.change):
 *   insert      reference = HEAD if index == 0, else the (index - 1)-th visible element with lookAfterTombstones (the last
 *               following tombstone whose markOpsAfter slot is defined, src/micromerge.ts:775-797), evaluated before the values,
 *               so a zero-value insert out of bounds still fails; value j references value j - 1 and lands right after it
 *   delete      `arg` times: the index-th visible element, which is deleted before the next
 *   add/remove  start = before(elem[startIndex]); end = endOfText for strong / em when endIndex >= the visible length, else
 *   Mark        before(elem[endIndex]); for comment / link after(elem[endIndex - 1]), which defines that element's after slot
 *               for the InputOperations that follow; arrival = the log's ins/del records before the mark
 * Generated records: ins/del op j of a record has ctr first_ctr + j and the actor's rank; insert references, delete targets and
 * mark boundaries are the resolved elements' packed opIds.  A log whose change hits "List index out of bounds" appends
 * nothing (status PT_CHANGE_OUT_OF_BOUNDS, `input` names the failing InputOperation) and the other logs proceed; the
 * reference instead bumps seq and keeps the ops it generated before the throw.
 * `changes` is the change table of the new changes (one pt_change_rec per log that has a change, as for pt_batch_append;
 * NULL iff the handle has no change table); the records of failed logs are dropped.  A new actor or comment id shifts packed
 * ranks: introduce it first with a pt_batch_append of an empty delta and its remap, then call this with the new ranks.
 * Refused before anything changes:
 *   PT_ERR_STATE    no completed merge since the last upload, append, change or select; a handle without PT_FLAG_EMIT_SEQUENCE
 *   PT_ERR_INVALID  (pt_last_error names the first offender) n_logs differs; input_off not increasing from 0 or past the ops; a log
 *                   with inputs and no actor; an actor rank >= the log's n_actors; a log with a change whose merge status is not
 *                   PT_LOG_OK; an unknown action or mark type; first_ctr not above the log's max_ctr, or below the previous
 *                   record's next counter, or a counter past 2^32 - 1; an attr or a token out of range; a log that would hold
 *                   2^22 elements or more, or whose max_ctr x n_actors would reach 2^31; a change table on one side only
 * On success the handle holds exactly the batch pt_batch_append of the view's delta with identity maps would give (the same
 * re-plan; no merge, so views of the last merge are invalid; the patch window is reset; pools persist).  A following merge
 * under pt_batch_set_patch_window(first_op = old n_insdel + n_mark) gives the Patch stream change() returns.
 * The view is engine-owned pinned memory, valid until the next upload, append, change or destroy.  Synchronises; the caller's
 * arrays may be freed on return.
 * Device: one warp per log with InputOperations copies the log's element sequence into a scratch slot (n_elems + its insert
 * values words) and resolves the InputOperations in order: ballot / popcount selection of the k-th visible element (O(N) per
 * InputOperation, the reference's own cost), one warp-cooperative splice per insert, the deleted bit per delete, the
 * after-slot bit per `after` end; it writes the records into the delta as it goes.  The delta goes through pt_batch_append's
 * splice on the device. */
int pt_batch_change(pt_batch*, const pt_change_input* in, const pt_change_table* changes, pt_change_view* out);

/* ------------------------------------------------------------------------------------------------
 * Sync between logs of the batch: getMissingChanges(source, target) followed by applyChanges(target, missing) (reference
 * test/merge.ts:4-38, called both ways per step at test/fuzz.ts:198-199), for many (source, target) pairs of resident logs at
 * once.  A document's replicas are logs of one batch; the changes one of them generated (pt_batch_change) or received
 * (pt_batch_append) reach another without leaving the device.  Needs a change table whose n_ops counts each change's list ops.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_exchange_pair { uint32_t src, dst; } pt_exchange_pair;
typedef struct pt_exchange_input {
    uint32_t n_pairs;
    const pt_exchange_pair* pairs;   /* deliver to log dst what it is missing from log src                                   */
    const uint64_t* actor_off;       /* [n_pairs + 1]; pair p's map is actor_map[actor_off[p] .. actor_off[p+1])              */
    const uint16_t* actor_map;       /* src actor rank -> dst actor rank, exactly src's n_actors entries; 0xFFFF = the actor has
                                        no rank in dst                                                                        */
    const uint64_t* ctr_off;         /* [n_pairs + 1] or NULL = identity for every pair                                       */
    const uint32_t* ctr_map;         /* src packed counter -> dst packed counter (needed only where the packer re-ranked sparse
                                        counters in either log); empty range = identity; entry 0 = 0; 0xFFFFFFFF = no image in
                                        dst; a counter past the map has no image                                              */
} pt_exchange_input;

#define PT_EXCHANGE_OK 0u
#define PT_EXCHANGE_BAD_TABLE 1u  /* src's or dst's change table is not seq-contiguous per actor, names an actor >= n_actors or
                                     deps outside the log's, or src's n_ops do not sum to its n_insdel + n_mark (or its mark
                                     arrivals do not fit those positions)                                                      */
#define PT_EXCHANGE_STUCK 2u      /* a pass over the queue admitted nothing: a missing change depends on a change neither log
                                     holds                                                                                     */
#define PT_EXCHANGE_UNMAPPED 3u   /* a missing change, one of its deps or one of its records names an actor or counter without
                                     an image in dst                                                                           */
typedef struct pt_exchange_view {
    uint32_t n_pairs;
    const uint32_t* status;        /* [n_pairs] PT_EXCHANGE_*; a pair that is not OK delivers nothing                          */
    const uint64_t* delivered_off; /* [n_pairs + 1]                                                                            */
    const uint32_t* delivered;     /* pair p: delivered[delivered_off[p] .. delivered_off[p+1]) = indices into src's change
                                      table, in delivery order                                                                 */
    const pt_log_desc* delta;      /* [n_logs] per log the records it received (n_insdel, n_mark; offsets into the engine's
                                      delta, not meaningful to the caller), its n_actors and its new max_ctr                   */
} pt_exchange_view;

/* For every pair, deliver to log dst the changes it is missing from log src, in the order the reference's sync applies them.
 * All pairs read the batch as it is BEFORE the call, so {A->B, B->A} in one call is the reference's two-way sync (what A lacks
 * from B cannot include what B just received from A: those are A's own), and {A->B, B->C} does not forward A's changes to C.
 * Per pair:
 *   1. clocks   clock[a] = the number of changes by actor a in the log's change table, for src and for dst.  While counting,
 *               every change of both logs must have seq == count + 1 (PT_EXCHANGE_BAD_TABLE otherwise).  No merge is needed:
 *               in a sync loop the call follows pt_batch_change, which leaves the batch unmerged.
 *   2. missing  getMissingChanges order (test/merge.ts:25-38): src's actors in the order src first saw them (the insertion
 *               order of source.clock), and for each the changes with seq > clock_dst[map(actor)], ascending; an actor without
 *               a rank in dst has clock 0.
 *   3. order    the order applyChanges admits them (test/merge.ts:4-23): the queue front is delivered if seq == clock + 1 and
 *               every dep <= clock (src/micromerge.ts:501-509; a zero clock entry fails), else it moves to the back.  That is
 *               repeated in-order passes over the remaining queue.  The reference gives up after 10 001 iterations; the engine
 *               has no such cap: it ends a pair with PT_EXCHANGE_STUCK after a full pass that delivers nothing, and otherwise
 *               delivers however many passes it takes.
 *   4. records  change c of src holds the list ops at positions [P_c, P_c + n_ops_c), P_c = the sum of the earlier n_ops (the
 *               positions of pt_batch_set_patch_window).  The delivered changes' ins/del records are concatenated in delivery
 *               order, and so are their mark records.  Actor fields go through the actor map and counters (ctr, ref_ctr,
 *               start_ctr, end_ctr) through the counter map; an id whose counter is 0 keeps its actor field, as in
 *               pt_batch_append.  Value tokens, link ids and comment ranks are per batch and are copied.  A mark's arrival
 *               becomes dst's old n_insdel + the delivered ins/del records before it.  Change records keep seq and n_ops; their
 *               actor and their deps' actors go through the actor map.
 *   5. splice   the delta is appended with identity maps: the handle then holds exactly what pt_batch_append of that delta would
 *               give (re-planned; no merge, so views of the last merge are invalid; the patch window is reset; pools persist).
 *               pt_batch_set_patch_window(first_op = old n_insdel + n_mark) then gives the Patches applyChanges returned.
 * A pair whose status is not PT_EXCHANGE_OK delivers nothing and does not fail the call; the other pairs proceed.  A new actor,
 * or a counter that moves dst's packed ranks, is introduced first by a pt_batch_append of an empty delta with its remap, as for
 * pt_batch_change; without that the pair reports PT_EXCHANGE_UNMAPPED.
 * Refused with nothing changed:
 *   PT_ERR_STATE    no batch, or a handle without a change table
 *   PT_ERR_INVALID  (pt_last_error names the first offender) null arguments; src or dst >= n_logs; src == dst; a dst named
 *                   twice; an actor map whose length is not src's n_actors, whose mapped entries are not strictly increasing or
 *                   name a rank >= dst's n_actors; a counter map whose entry 0 is not 0 or whose mapped entries are not strictly
 *                   increasing; a log that would exceed 2^32 - 1 records, and whatever pt_batch_append refuses for the resulting
 *                   batch (the same messages)
 * n_pairs == 0: PT_OK, nothing launched, nothing changed.  Synchronises; the caller's arrays may be freed on return.  The view
 * is engine-owned pinned memory, valid until the next upload, append, change, exchange or destroy.
 * Device: a select kernel, one warp per pair (clocks in shared memory; the queue, 32 candidates per trip, in a scratch slot),
 * the per-pair totals back to the host (32 B per pair), a gather kernel, one warp per delivered change (up to 64 for a long
 * one) with 16-byte coalesced copies, then pt_batch_append's splice with the delta records and the delta change table both
 * on the device: no record and no change record crosses PCIe; besides the totals only the view's delivered indices come back.
 * Peak device memory: old + delta + new records and change tables, plus 40 B of scratch per change of every pair's src. */
int pt_batch_exchange(pt_batch*, const pt_exchange_input* in, pt_exchange_view* out);

/* ------------------------------------------------------------------------------------------------
 * Actor tables: each log's actor ids on the device, so that a sync step derives pt_batch_exchange's maps and its pre-append
 * there (pt_batch_sync_pairs) and the caller needs no host copy of the records.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_actor_tables {
    uint32_t n_logs;
    const uint8_t* data; const uint64_t* off; uint64_t count;   /* PT_POOL_ACTORS: UTF-16LE ids, byte offsets [count + 1]       */
    const uint64_t* per_log_first;                              /* [n_logs + 1] log i's ids are per_log_first[i] .. [i + 1]     */
    const uint64_t* counters_first;                             /* [n_logs + 1] PT_POOL_COUNTERS ranges, or NULL: a non-empty
                                                                   range marks a log whose counters were re-ranked densely      */
} pt_actor_tables;

/* Attach the batch's per-log actor ids: pt_ingest_pool's PT_POOL_ACTORS (and PT_POOL_COUNTERS' per-log ranges) or
 * packing.string_pools pass straight through.  Of counters_first the handle keeps one bit per log.
 * Refused with PT_ERR_INVALID, pt_last_error naming the first bad log: n_logs differs; per_log_first does not run from 0 to
 * count or decreases; a log's count is not its n_actors (0 is allowed only when n_actors == 1); an id of odd byte length; ids
 * not strictly increasing in UTF-16 code-unit order (JS string order, compareOpIds).  No batch: PT_ERR_STATE.
 * Lifetime: every upload form and pt_batch_adopt_device drop the tables (as they drop the change table); pt_batch_change and
 * pt_batch_exchange keep them; pt_batch_select_logs gathers them with their logs; pt_batch_append keeps them only when its remap has no actor map, no counter map and no log's
 * n_actors changes (a comment-only remap keeps them).  Synchronises; the caller's arrays may be freed on return. */
int pt_batch_upload_actors(pt_batch*, const pt_actor_tables* tables);

/* The current tables in the PT_POOL_ACTORS layout (counters_first = NULL): the `actors` pool pt_batch_render_changes_json
 * takes.  No tables: PT_ERR_STATE.  Synchronises.  The view is engine-owned pinned memory, valid until the next call of it,
 * upload or destroy. */
int pt_batch_download_actors(pt_batch*, pt_actor_tables* out);

/* Introduce actor ids per log, in any order (duplicates and ids the log knows allowed): the acting actor before its first
 * pt_batch_change on a replica, for example.  Each log's table becomes the sorted union and its n_actors max(1, count).
 * Where a rank moves or an n_actors grows, the records, change records and dep records go through pt_batch_append's splice
 * with the derived actor maps (an empty delta, counters untouched): the handle then holds exactly what pt_batch_append of
 * packing.add_actors' delta and remap gives, with no merge (the patch window is reset, pools persist).  Otherwise the batch
 * and its last merge are untouched.  View (engine-owned pinned memory, valid until the next call of it, upload or destroy):
 * the rank of every given id after the call, and the per-log old -> new actor maps (empty range: unchanged), so the caller
 * can move its own rank-indexed data.  Refused: no batch or no actor tables (PT_ERR_STATE); n_logs differs, per_log_first
 * not from 0 to count or decreasing, an id of odd byte length, a log that would have more than 65535 actors, and what
 * pt_batch_append refuses (PT_ERR_INVALID, nothing changed).  Synchronises; the caller's arrays may be freed on return.
 * Device: one warp per log sorts and deduplicates its ids by counting (O(m^2) compares for a log given m ids), the merge
 * kernel of pt_batch_sync_pairs writes the grown tables, then the splice and a rank kernel. */
typedef struct pt_actor_input {
    uint32_t n_logs;
    const uint8_t* data; const uint64_t* off; uint64_t count;   /* UTF-16LE ids, byte offsets [count + 1]                         */
    const uint64_t* per_log_first;                              /* [n_logs + 1] log i's ids are per_log_first[i] .. [i + 1]       */
} pt_actor_input;
typedef struct pt_actor_view {
    uint32_t n_logs; uint64_t count;
    const uint16_t* rank;          /* [count] each given id's rank in its log after the call                                  */
    const uint64_t* actor_off;     /* [n_logs + 1] per-log old -> new actor rank maps; empty range: unchanged                 */
    const uint16_t* actor_map;
    uint32_t spliced;              /* 1: the splice ran (the batch needs a merge, the patch window was reset)                 */
} pt_actor_view;
int pt_batch_add_actors(pt_batch*, const pt_actor_input* in, pt_actor_view* out);

#define PT_EXCHANGE_DENSE 4u      /* pt_batch_sync_pairs only: src or dst is densely ranked, or dst would be once grown; the
                                     pair delivers nothing and dst does not grow (exchange it with caller maps instead)        */
typedef struct pt_sync_view {
    uint32_t n_pairs;
    const uint32_t* status;        /* [n_pairs] PT_EXCHANGE_*, PT_EXCHANGE_DENSE included                                     */
    const uint64_t* delivered_off; /* [n_pairs + 1]  as pt_exchange_view                                                       */
    const uint32_t* delivered;
    const pt_log_desc* delta;      /* [n_logs]                                                                                 */
    const uint64_t* actor_off;     /* [n_logs + 1] the pre-append's per-log old -> new actor rank maps (empty range: unchanged) */
    const uint16_t* actor_map;
} pt_sync_view;

/* pt_batch_exchange with its maps and its pre-append derived on the device from the actor tables (pt_batch_upload_actors).
 * (Named pt_batch_sync_pairs because pt_batch_sync already names the stream synchronisation above.)  The caller sends only
 * the pairs.  The pair rules, the refusals of the pairs and "every pair reads the batch as it is before
 * the call" are pt_batch_exchange's.  Per pair:
 *   1. missing  src's changes whose seq exceeds dst's count of the same actor ID (the two tables joined by name).
 *   2. named    the src actors those changes name: the change actor, dep actors, and the actor of every ins/del and mark
 *               record id whose counter is non-zero; and the top opId counter and the op count of their records.
 *   3. growth   dst's table becomes the sorted union (packing._grown_ids).  If src or dst is densely ranked, or the grown dst
 *               would be (packing._wants_dense of max(dst max_ctr, top) and dst's ops + the missing ops), the pair is
 *               PT_EXCHANGE_DENSE: it delivers nothing and dst does not grow.
 *   4. pre      if a dst's ranks move or its n_actors grows, one pt_batch_append splice of an empty delta applies every pair's
 *               growth (derived before any is applied, so {A->B, B->A} sees both logs grown), identity counters.
 *   5. maps     src rank -> dst rank of the same name in the grown tables (0xFFFF for a rank without a name or an image);
 *               identity counter maps.
 *   6. exchange pt_batch_exchange's select, gather and splice with those maps; STUCK / BAD_TABLE / UNMAPPED as there.
 * Afterwards the handle and the tables equal packing.sync_maps' exchange_maps of the pairs that are not DENSE, then
 * apply_append of its pre-append, then apply_exchange.  A refusal of the delivery's splice after a pre-append leaves the
 * pre-append applied.
 * Refused: PT_ERR_STATE without a batch, change table or actor tables; PT_ERR_INVALID for null arguments, the pair rules of
 * pt_batch_exchange, a log that would have more than 65535 actors, and what pt_batch_append refuses.
 * n_pairs == 0: PT_OK, nothing launched.  Synchronises.  The view is engine-owned pinned memory, valid until the next
 * upload, append, change, exchange, sync or destroy.
 * Device: a derive kernel (one warp per pair; clocks, the name join and a bitmap over src ranks in shared memory, the missing
 * records read by the whole warp), a merge kernel (one warp per log) writing the grown tables and the rank maps, the splice,
 * a map kernel (one warp per pair), then pt_batch_exchange's kernels.  Besides the pairs, 32 B per pair and the moved logs'
 * rank maps cross PCIe. */
int pt_batch_sync_pairs(pt_batch*, const pt_exchange_pair* pairs, uint32_t n_pairs, pt_sync_view* out);

/* ------------------------------------------------------------------------------------------------
 * Select: change WHICH logs the resident batch holds, on the device.  A server that opens and closes documents, or a sync
 * session in which a new replica joins (a fresh Micromerge that applies the initial change, then syncs), keeps every log that
 * stays resident, including what pt_batch_change, pt_batch_exchange and pt_batch_sync_pairs wrote there, and uploads only the
 * logs it adds.
 * ---------------------------------------------------------------------------------------------- */
#define PT_SELECT_ADDED 0xFFFFFFFFu
/* New log i = resident log from[i], or, where from[i] == PT_SELECT_ADDED, the next log of `added` (in order).  `from` may drop
 * logs, reorder them and name one log several times (a fork: a replica with the same state and arrival order).
 * A kept log keeps its records, descriptor fields, change and dep records and actor table; only the comment ranks of its
 * comment marks move, through comment_map (old rank -> new rank, n_comment_map entries; NULL = identity).  The mapped entries
 * (all but 0xFFFFFFFF) strictly increase; 0xFFFFFFFF drops a rank that no kept log names, so retiring documents can shrink the
 * batch-wide comment order.  An added log's records, change table (added_changes, dep_off relative to the log's deps, as for
 * an upload) and actor ids (added_actors, pt_batch_upload_actors' layout and rules) are in the new id space and are copied
 * verbatim: value-pool indices and link ids carry no order and never move, and counters and actor ranks are per log.
 * added is NULL or has 0 logs iff no entry is PT_SELECT_ADDED; then added_changes and added_actors are NULL.  Otherwise
 * added_changes is NULL iff the handle has no change table, and added_actors NULL iff it has no actor tables.
 * On success the handle holds exactly what pt_batch_upload of the selected batch, pt_batch_upload_changes of its change table
 * and pt_batch_upload_actors of its actor tables would hold: the batch is re-planned and its key records derived again, there
 * is no merge (views of the last merge are invalid), the patch window is reset, and comment-pool and patch-pool settings
 * persist.  n_logs == 0 is accepted, as by pt_batch_upload.
 * Refused with nothing changed:
 *   PT_ERR_STATE    no batch
 *   PT_ERR_INVALID  (pt_last_error names the first offender) from[i] >= the old n_logs and not PT_SELECT_ADDED; the number of
 *                   PT_SELECT_ADDED entries is not added->n_logs; an added descriptor or change descriptor out of range; a
 *                   change table or actor tables on one side only, or added actor tables that pt_batch_upload_actors refuses;
 *                   comment_map not strictly increasing over its mapped entries; a new batch that an upload refuses (make_plan)
 * The device refuses too: a kept comment mark whose rank is outside comment_map or maps to 0xFFFFFFFF gives PT_ERR_INVALID with
 * the batch untouched, because the splice writes new buffers and only a successful one replaces the old.
 * Synchronises; the caller's arrays may be freed on return.
 * Device: pt_batch_append's splice with a gather index (one warp per new log, up to 64 for a log with many records, 16-byte
 * coalesced copies; a log without a comment map is a straight copy) and a warp-per-log gather of the actor tables.  Peak
 * device memory: old + added + new records (and change and actor tables). */
int pt_batch_select_logs(pt_batch*, const uint32_t* from, uint32_t n_logs,
                         const pt_packed_ops* added,            /* NULL iff no entry is PT_SELECT_ADDED           */
                         const pt_change_table* added_changes,  /* NULL iff the handle has no change table          */
                         const pt_actor_tables* added_actors,   /* NULL iff the handle has no actor tables          */
                         const uint32_t* comment_map, uint64_t n_comment_map);   /* NULL = identity              */

/* ------------------------------------------------------------------------------------------------
 * Checkout: an EARLIER version of a resident log as a new log, on the device.  A history slider, "what does peer P see" (the
 * version named by P's vector clock, getMissingChanges' input, reference test/merge.ts:25-38) and the last clock two diverged
 * replicas shared are all a version: what a fresh Micromerge holds after applyChange of exactly the changes it covers.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_clock_entry { uint32_t actor; uint32_t seq; } pt_clock_entry;   /* actor rank in the request's log */
#define PT_CHECKOUT_OK 0u
#define PT_CHECKOUT_BAD_TABLE 1u   /* the source's change table fails pt_batch_exchange's BAD_TABLE rules for a src: not
                                      seq-contiguous per actor, an actor >= n_actors, deps outside the log's, n_ops that do not
                                      sum to its n_insdel + n_mark, or mark arrivals that do not fit those positions          */
#define PT_CHECKOUT_UNKNOWN 2u     /* clock mode: clock[a] > the log's number of changes by a (the version holds changes this
                                      log does not)                                                                          */
#define PT_CHECKOUT_NOT_CLOSED 3u  /* a fresh replica applying the covered changes in table order would reject one           */
/* Request k adds new log old n_logs + k, holding log logs[k] at a version:
 *   covered   prefix mode (n_changes non-NULL): the first min(n_changes[k], table size) changes of the log's table.  Clock mode
 *             (clock_off non-NULL): the changes with seq <= clock[actor], request k's clock being the entries
 *             clock[clock_off[k] .. clock_off[k+1]) (actor ranks of log logs[k]); an absent actor counts as 0 and a seq of 0 is
 *             allowed.  In a seq-contiguous table prefix j is the clock mode of the prefix's per-actor counts.
 *   records   the covered changes' ins/del records, concatenated in table order, then their mark records likewise; record
 *             ranges come from the list-op positions (pt_batch_exchange step 4).  A mark's arrival is the number of covered
 *             ins/del records before it.  Change records keep seq and n_ops; dep_off is rebased and the deps are copied.
 *   ids       the source's: actor ranks, counters, comment ranks, value and link ids, and the descriptor's n_actors and
 *             max_ctr.  With actor tables attached the new log gets the source's table and its dense-counter bit.
 *   status    status_out[k] = PT_CHECKOUT_*.  NOT_CLOSED is applyChange's check (src/micromerge.ts:505-509) in table order: a
 *             covered change c fails it when a dep (a, d) of c has fewer than max(d, 1) covered changes by a before c, so a
 *             zero clock entry fails and a source that admission rejected is reported as such.  A request that is not OK still
 *             adds its log, with no records and no changes, so the indices stay stable.
 * Several requests may name one log.  Afterwards the handle holds exactly what pt_batch_select_logs(from = [0 .. n_logs)
 * followed by PT_SELECT_ADDED x n, added = the new logs) would hold: the batch is re-planned and its key records derived again,
 * there is no merge (views of the last merge are invalid), the patch window is reset, pool settings persist, and a later
 * pt_batch_select_logs([0 .. old n_logs)) retires the checkouts.  No merge is needed before the call.
 * Refused with nothing changed:
 *   PT_ERR_STATE    no batch, or a handle without a change table
 *   PT_ERR_INVALID  (pt_last_error names the first offender) null arguments; a log >= n_logs; both modes or neither; clock_off
 *                   not non-decreasing from 0; a clock actor >= the log's n_actors; an actor named twice in one request; what
 *                   an upload refuses for the resulting batch (make_plan)
 * n == 0: PT_OK, nothing launched, nothing changed.  Synchronises; the caller's arrays may be freed on return.
 * Device: a select kernel, one warp per request (the clocks in shared memory, then one pass over the table and an in-order
 * pass that checks closure and places the covered changes' records, 32 changes per trip), the per-request totals back to the
 * host (32 B per request), pt_batch_exchange's gather kernel with identity maps into empty logs, then pt_batch_select_logs'
 * splice and actor-table gather.  No record and no change record crosses PCIe: only the requests, the totals and the
 * statuses.  Peak device memory: old + delta + new records and change tables, plus 40 B of scratch per change of every
 * request's source. */
int pt_batch_checkout(pt_batch*, const uint32_t* logs, uint32_t n,
                      const uint32_t* n_changes,      /* [n] prefix mode, or NULL                                           */
                      const uint64_t* clock_off,      /* [n + 1] clock mode, or NULL; exactly one of the two is non-NULL       */
                      const pt_clock_entry* clock,    /* request k's clock = clock[clock_off[k] .. clock_off[k+1])             */
                      uint32_t* status_out);          /* [n] caller-owned, PT_CHECKOUT_*                                       */

/* Every log's clock: seq[off[i] + a] = the number of changes by actor rank a in log i's change table (Micromerge.clock by
 * rank), off = the exclusive scan of n_actors ([n_logs + 1]).  status[i] is PT_CHECKOUT_BAD_TABLE where the table fails
 * pt_batch_exchange's clock checks (not seq-contiguous per actor, an actor >= n_actors, deps outside the log's); that log's
 * entries are 0.  This names the version a log holds now, also after pt_batch_change, pt_batch_exchange or
 * pt_batch_sync_pairs, so that it can be checked out later.  No batch or no change table: PT_ERR_STATE; null arguments:
 * PT_ERR_INVALID.  Synchronises.  The view is engine-owned pinned memory, valid until the next call of it, upload or
 * destroy.  Device: one warp per log counting its table (ptct::count_clock) into the output. */
int pt_batch_download_clocks(pt_batch*, const uint64_t** off, const uint32_t** seq, const uint32_t** status);

/* The handle's per-log descriptors ([n_logs]; offsets into the engine's records): the shape of the resident batch after calls
 * that build logs on the device, such as pt_batch_checkout, whose record counts the caller does not know.  No batch:
 * PT_ERR_STATE; null out: PT_ERR_INVALID.  The view is engine-owned host memory, valid until the next call that changes the
 * batch (upload, append, change, exchange, sync, select, checkout) or destroy.  No device work. */
int pt_batch_download_descs(pt_batch*, const pt_log_desc** out);

/* Enqueue the merge: op-log apply + flatten for every log of the batch (the replacement for the
 * applyOp loop src/micromerge.ts:513 and getTextWithFormatting src/peritext.ts:337). Asynchronous. */
int pt_batch_merge(pt_batch*);

/* Block until the handle's stream is idle. */
int pt_batch_sync(pt_batch*);

/* Enqueue the device -> host copies of the result arrays without waiting (pinned destinations); a following
 * pt_batch_download only waits.  Lets a caller overlap this handle's download with other handles' work. */
int pt_batch_download_begin(pt_batch*);

/* Copy results device -> host (pinned) and return a view. Synchronises the stream. */
int pt_batch_download(pt_batch*, pt_spans_view* out);

/* PT_FLAG_EMIT_PATCHES: copy the Patch stream of the last merge device -> host and return a view (engine-owned pinned
 * memory, valid until the next upload / destroy). Synchronises. */
int pt_batch_download_patches(pt_batch*, pt_patch_view* out);
int pt_batch_set_patch_pool(pt_batch*, uint64_t items);

/* PT_FLAG_EMIT_PATCHES: restrict the Patch stream of the following merges to a suffix of every log's list ops — what an editor
 * that has seen the first changes needs from Micromerge.applyChange for the rest (src/micromerge.ts:499-514).
 * first_op[i] is the position of log i's first op inside the window, in the list-op order of pt_batch_render_patches_json:
 * ins/del record j is at j + #{k : min(arrival_k, n) <= j}, mark record k at min(arrival_k, n) + k.  0 is the whole log,
 * n_insdel + n_mark an empty window; first_op == NULL sets every log to 0.  After a pt_batch_append, first_op[i] = the log's
 * old n_insdel + old n_mark gives exactly the new changes' ops.  With a change table whose n_ops counts the log's list ops,
 * change c starts at the sum of n_ops over the log's earlier changes.
 * A merge under a window computes what the whole-log merge computes for the ops inside it: their pt_patch_rec records are
 * identical, the records before the window are {0, 0, PT_ATTR_NONE, 0}, and the item pool holds only the items of ops inside
 * the window (n_items_needed is the window's demand, and a pool of that size is enough).  The patch status and its limits
 * are those of the whole log.  pt_batch_render_patches_json renders each log as "[" + the inner arrays of the ops at positions
 * >= first_op[i] + "]": the whole-log bytes with the first first_op[i] inner arrays removed.
 * Cost: the per-op loops of the patch kernel are O(window x log) per log instead of O(log^2); the tables still cover the
 * whole log (linear), and the merge itself is unchanged.
 * The window persists across merges; every upload form and pt_batch_append reset it to whole logs.  Setting it after a merge
 * makes the patch outputs of that merge stale: pt_batch_download_patches and pt_batch_render_patches_json return PT_ERR_STATE
 * until the next merge.  Refused with nothing changed: n_logs other than the batch's, or a first_op[i] > n_insdel + n_mark
 * (PT_ERR_INVALID, pt_last_error names the first such log); no batch, or a handle without PT_FLAG_EMIT_PATCHES (PT_ERR_STATE).
 * n_logs == 0: PT_OK.  Synchronises; first_op may be freed on return. */
int pt_batch_set_patch_window(pt_batch*, const uint32_t* first_op /* [n_logs] or NULL = whole logs */, uint32_t n_logs);

/* Batched index -> element resolution on the materialised documents (PT_FLAG_EMIT_SEQUENCE, after a merge): what
 * op generation and cursors need (getListElementId, src/micromerge.ts:762-805; getCursor :465).  Query k asks log
 * `log` for its `index`-th visible element; with PT_QUERY_LOOK_AFTER_TOMBSTONES the answer moves to the LAST following
 * tombstone whose markOpsAfter slot is defined (:775-797, the rule Micromerge.change uses for insert positions).
 * Answers: index of the element's insert record in the log's ins/del records, PT_ELEM_NOT_FOUND if the index is out of
 * bounds ("List index out of bounds", :804).  One warp per query on the device; synchronises. */
typedef struct pt_elem_query { uint32_t log; uint32_t index; uint32_t flags; uint32_t reserved; } pt_elem_query;
#define PT_QUERY_LOOK_AFTER_TOMBSTONES 1u
#define PT_ELEM_NOT_FOUND 0xFFFFFFFFu
int pt_batch_query_elements(pt_batch*, const pt_elem_query* queries, uint32_t n, uint32_t* record_index_out);

/* Batched elemId -> position resolution, the inverse of the query above: findListElement (src/micromerge.ts:731-755) on the
 * materialised documents, whose `.visible` is resolveCursor's answer (:475-477).  Same preconditions as
 * pt_batch_query_elements (PT_FLAG_EMIT_SEQUENCE and a completed merge, else PT_ERR_STATE); synchronises.
 * Query k names the element of log `log` whose insert op has the opId (ctr, actor) in the PACKED id space (actor rank; the
 * dense counter rank where the packer re-ranked sparse counters).  An opId that no INSERT record of the log carries is not
 * found: opIds of delete and mark ops (not list elements), ctr 0 (HEAD), ctr > max_ctr, actor >= n_actors.  Not found means
 * index = record = PT_ELEM_NOT_FOUND and visible = 0; a log index >= n_logs or a log whose status is not PT_LOG_OK also sets
 * PT_ELEM_LOG_FAILED (the reference would have thrown before such a document existed).
 * One warp per query on the device: a coalesced scan of the log's ins/del records for the insert, then of its element
 * sequence for the position, counting the visible elements before it. */
typedef struct pt_elem_ref { uint32_t log; uint32_t ctr; uint16_t actor; uint16_t reserved0; uint32_t reserved1; } pt_elem_ref;   /* 16 B */
typedef struct pt_elem_pos {
    uint32_t index;    /* position in the element sequence incl. tombstones (the reference's metadata index)           */
    uint32_t visible;  /* non-deleted elements before it (resolveCursor's answer)                                     */
    uint32_t record;   /* its insert record in the log's ins/del records (what pt_batch_query_elements returns)       */
    uint32_t flags;    /* PT_ELEM_DELETED, PT_ELEM_AFTER_DEFINED (the sequence's bit 30), PT_ELEM_LOG_FAILED          */
} pt_elem_pos;     /* 16 B */
#define PT_ELEM_DELETED 1u
#define PT_ELEM_AFTER_DEFINED 2u
#define PT_ELEM_LOG_FAILED 4u
int pt_batch_find_elements(pt_batch*, const pt_elem_ref* refs, uint32_t n, pt_elem_pos* out);

/* ------------------------------------------------------------------------------------------------
 * Attribution: which change inserted, and which change deleted, every element of a merged log, and what changed since a
 * version.  Blame ("written by"), highlighting what collaborators changed while one was away (the reference's essay demo does
 * it for live patches, src/essay-demo.ts:47-75) and showing deleted text in a review view all read it.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_attr_run {   /* 32 B: a maximal run of consecutive elements (element-sequence order, tombstones included) with
                                  equal (ins_actor, ins_seq, del_actor, del_seq, flags) */
    uint32_t elem;       /* index of its first element in the element sequence (the reference's metadata index)          */
    uint32_t visible;    /* visible elements before it (resolveCursor's answer for its first element)                    */
    uint32_t n;          /* elements in the run; all visible iff del_seq == 0                                            */
    uint32_t flags;      /* PT_ATTR_INSERTED_SINCE, PT_ATTR_DELETED_SINCE (clock requests only, else 0)                   */
    uint32_t ins_seq;    /* Change.seq of the change whose op inserted the elements                                      */
    uint32_t del_seq;    /* 0: not deleted; else Change.seq of the change holding the elements' attributed delete        */
    uint16_t ins_actor;  /* that change's actor rank in the log                                                          */
    uint16_t del_actor;  /* the deleting change's actor rank (0 when del_seq == 0)                                       */
    uint32_t reserved;   /* 0 */
} pt_attr_run;
#define PT_ATTR_INSERTED_SINCE 1u   /* the inserting change is not covered by the request's clock                       */
#define PT_ATTR_DELETED_SINCE 2u    /* deleted now, and no delete of the element is in a covered change                 */
#define PT_ATTR_OK 0u
#define PT_ATTR_LOG_FAILED 1u       /* the log's merge status is not PT_LOG_OK (admission-rejected logs included)       */
#define PT_ATTR_BAD_TABLE 2u        /* the table fails pt_batch_exchange's BAD_TABLE rules for a src (as PT_CHECKOUT_BAD_TABLE) */
typedef struct pt_attr_view {
    uint32_t n;
    const uint32_t* status;         /* [n] PT_ATTR_*; a request that is not OK has no runs                              */
    const uint64_t* off;            /* [n + 1] request k's runs are runs[off[k] .. off[k+1])                            */
    const pt_attr_run* runs; uint64_t n_runs;
} pt_attr_view;
/* Request k attributes every element of log logs[k] in the element sequence of the last merge:
 *   insert    the element's insert record lies at list-op position p (pt_batch_set_patch_window's order); its change is the c
 *             with P_c <= p < P_c + n_ops_c, P_c = the sum of the earlier n_ops.  ins_actor / ins_seq are c's.  In Change terms:
 *             the change whose actor is the elemId's actor and whose [startOp, startOp + ops.length) holds its counter.
 *   delete    of the delete records that target the element, the one with the smallest opId in compareOpIds order (packed
 *             (ctr, actor rank) order, src/micromerge.ts:812-827) is attributed, and its change gives del_actor / del_seq.  The
 *             first delete by arrival would depend on the replica; the smallest opId makes converged replicas give identical
 *             runs once actor ranks are mapped to ids.
 *   clock     (clock_off non-NULL) request k's clock = clock[clock_off[k] .. clock_off[k+1]) (actor ranks of log logs[k]); a
 *             change is covered iff seq <= clock[actor], an absent actor counting as 0 (pt_batch_checkout's clock mode; no
 *             closure check).  INSERTED_SINCE: the inserting change is not covered.  DELETED_SINCE: the element is deleted and
 *             none of its deletes is covered (a concurrent uncovered delete can have a smaller opId than a covered one).  An
 *             element was visible at the clock's version iff !INSERTED_SINCE && (del_seq == 0 || DELETED_SINCE).
 *   status    PT_ATTR_LOG_FAILED before PT_ATTR_BAD_TABLE; a request that is not OK has no runs.
 * Several requests may name one log.  A log without elements has no runs.
 * Refused with nothing changed:
 *   PT_ERR_STATE    no batch, no change table, a handle without PT_FLAG_EMIT_SEQUENCE, or no completed merge since the last call
 *                   that changed the batch (pt_batch_find_elements' rules)
 *   PT_ERR_INVALID  (pt_last_error names the first offender) null arguments; a log >= n_logs; clock_off not non-decreasing from 0;
 *                   a clock actor >= the log's n_actors; an actor named twice in one request (pt_batch_checkout's clock rules)
 * n == 0: PT_OK with an empty view, nothing launched.  Synchronises.  The view is engine-owned pinned memory, valid until the
 * next pt_batch_attribute, upload or destroy; every other view stays valid.
 * Device: a resolve kernel, one warp per request (the clocks in shared memory; ptct::count_clock and ptw::marks_before_lane give
 * each change's first ins/del record; each record finds its change by bisection over those, 32 records per trip; each delete
 * finds its target through an open-addressing opId table over the log's inserts and takes part in an atomicMin of its opId,
 * and a second pass lets the winner write its change), then a count pass and a write pass over the element sequence (one warp
 * per request, 32 words per trip, one function for both), with the runs sized exactly by the exclusive scan of the counts in
 * between.  Only the requests, the total, the statuses, the offsets and the runs cross PCIe.  Cost per request:
 * O(n_changes + n_insdel x (log n_changes + probes) + n_elems).  Peak scratch: 28 B per ins/del record (the opId table at half
 * load is 8 of them) and 8 B per change of every request's log (a log named twice counts twice), plus 32 B per run. */
int pt_batch_attribute(pt_batch*, const uint32_t* logs, uint32_t n,
                       const uint64_t* clock_off,     /* [n + 1] or NULL: no clock, flags are 0                           */
                       const pt_clock_entry* clock,   /* request k's clock = clock[clock_off[k] .. clock_off[k+1])         */
                       pt_attr_view* out);

/* ------------------------------------------------------------------------------------------------
 * Restore: make a resident log's visible text equal to an earlier version's, as a NEW local change.  In a CRDT a restore
 * cannot truncate the log (peers already hold the later changes): it is a change an actor makes on top of the current
 * document, which reaches peers through the normal sync (pt_batch_exchange / pt_batch_sync_pairs) like any other edit.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_restore_request {  /* 16 B */
    uint32_t log;        /* the log that gets the new change                                                           */
    uint32_t version;    /* a resident log in log's id space holding the target version (a pt_batch_checkout of log, or a
                            pt_batch_select_logs fork of one)                                                           */
    uint32_t actor;      /* the acting actor's rank in log (introduce a new actor first, as for pt_batch_change)         */
    uint32_t first_ctr;  /* packed counter of the first generated op; op j gets first_ctr + j; must exceed log's max_ctr  */
} pt_restore_request;
#define PT_RESTORE_TEXT 1u          /* make log's visible text equal to version's                                        */
#define PT_RESTORE_MARKS 2u         /* make log's formatting equal to version's (the visible texts must already be equal)  */
#define PT_RESTORE_OK 0u
#define PT_RESTORE_LOG_FAILED 1u    /* log's or version's merge status is not PT_LOG_OK                                  */
#define PT_RESTORE_BAD_TABLE 2u     /* log's change table fails the change-table rules for a src (as PT_CHECKOUT_BAD_TABLE) */
#define PT_RESTORE_FOREIGN 3u       /* TEXT: an element of version has no element of the same packed opId, in order, in log */
#define PT_RESTORE_TEXT_DIFFERS 4u  /* MARKS: the two visible token sequences differ                                     */
typedef struct pt_restore_view {
    uint32_t n;
    const uint32_t* status;   /* [n] PT_RESTORE_*; a request that is not OK appends nothing                              */
    const uint32_t* n_ops;    /* [n] list ops of the appended change; 0 = nothing to do, no change appended              */
    const uint32_t* seq;      /* [n] the appended change's seq (0 when none)                                             */
} pt_restore_view;
/* Request k appends to log req[k].log one change by actor req[k].actor that makes its visible text (mode PT_RESTORE_TEXT) or
 * its formatting (PT_RESTORE_MARKS) equal to that of log req[k].version, both as of the last merge.  mode is exactly one of the
 * two.  The full restore is TEXT, merge, MARKS, merge: MARKS compares the formatting the restored text inherits, and only a
 * merge computes it.  TEXT:
 *   join      log's element sequence is walked in order and merge-joined with version's by packed opId (ctr, actor of each
 *             element's insert record): a log element matches when its opId is that of the next unmatched version element.  A
 *             pt_batch_checkout keeps its source's packed ids and RGA never reorders elements, so a version of the log is a
 *             subsequence of it; if the walk ends with version elements unmatched the status is FOREIGN.
 *   classes   visible now and visible in version: keep; visible now, deleted in or absent from version: delete; deleted now,
 *             visible in version: restore; deleted now and not visible in version: nothing (stays a tombstone).
 *   runs      maximal sequences of one action in element order ("nothing" does not break a run, a kept element does).  With v
 *             the visible index in the document as changed by the earlier InputOperations of the same change, a delete run of
 *             k elements is {delete, index v, count k} and a restore run {insert, index v, values = its elements' value
 *             tokens}, then v += k.  The change is by definition Micromerge.change of exactly these InputOperations (reference
 *             src/micromerge.ts:308-441), lookAfterTombstones included: the inserted values are NEW elements (RGA cannot
 *             revive a tombstone).
 *   records   op j has ctr first_ctr + j and the actor's rank; a delete targets its element; an insert's first value
 *             references HEAD at v == 0, else the last tombstone with a defined after slot (the sequence's bit 30) that follows
 *             the (v - 1)-th visible element before the next element visible at that moment, else that element (elements this
 *             change deleted count as tombstones); each further value references the one before.  These are the records
 *             pt_batch_change generates from the same InputOperations with first_ctr advanced per op.
 *   change    seq = the log's number of changes by actor + 1; deps = every actor with a nonzero count in the log's clock, in
 *             the order the table first shows them (the key order of the reference's Object.assign({}, this.clock); the
 *             acting actor is included iff it has earlier changes), each with that count; n_ops = the generated ops.  A
 *             request with nothing to do appends no change and leaves seq unchanged (the reference's change([]) would still
 *             bump its seq).
 *   status    LOG_FAILED before BAD_TABLE before FOREIGN / TEXT_DIFFERS; a request that is not OK appends nothing.
 * MARKS (the change record and statuses as above; FOREIGN does not occur):
 *   compare   the visible token sequences must be equal (else TEXT_DIFFERS).  At every visible position compare strong, em, the
 *             link attr and the set of comment ranks (PT_SPAN_COMMENT with no ids, quirk Q3, is not compared: no op can remove
 *             the empty `comment` key).
 *   ops       one per maximal range of positions differing the same way: strong / em addMark where only version has it,
 *             removeMark where only log has it; link addMark with version's attr where version's link is present and differs,
 *             removeMark (no attrs, attr PT_ATTR_NONE) where it is absent; comment, per rank, addMark where only version has it,
 *             removeMark where only log has it (attr = the rank).  Ordered by startIndex, then mark type in ALL_MARKS order, then
 *             comment rank.  Boundaries are pt_batch_change's for mark InputOperations: start before(elem[start]); end
 *             endOfText for strong / em ending at the visible length, else before(elem[end]); after(elem[end - 1]) for comment
 *             and link.  Op j has ctr first_ctr + j; every mark arrives after all of log's ins/del records.
 * Preconditions: pt_batch_find_elements' (PT_FLAG_EMIT_SEQUENCE and a completed merge since the last call that changed the
 * batch), and a change table.  All requests read the batch as it is before the call.
 * Refused with nothing changed:
 *   PT_ERR_STATE    no batch, no change table, a handle without PT_FLAG_EMIT_SEQUENCE, or no completed merge since the last call
 *                   that changed the batch
 *   PT_ERR_INVALID  (pt_last_error names the first offender) null arguments; mode not exactly one flag; a log or version
 *                   >= n_logs; a log named twice; an actor >= the log's n_actors; first_ctr <= the log's max_ctr, or a counter past
 *                   2^32 - 1; a log that would hold 2^22 elements or more, or whose max_ctr x n_actors would reach 2^31; whatever
 *                   pt_batch_append refuses for the resulting batch.  The count pass runs before the splice, so the limits that
 *                   depend on the generated counts are refused with nothing changed too.
 * n == 0: PT_OK, nothing launched.  On success the handle holds exactly what pt_batch_append of the generated delta (identity
 * maps) would give: re-planned, no merge, the patch window reset, pools persisting; pt_batch_set_patch_window(first_op = old
 * n_insdel + n_mark) then gives the Patches change() returned.  Synchronises; req may be freed on return.  The view is
 * engine-owned pinned memory, valid until the next pt_batch_restore or destroy.
 * Device: restore_kernel<false> (count) and <true> (write), one warp per request, through one function: the log's clock in
 * shared memory (ptct::source_clock, then ptct::first_shown for the deps), then TEXT's element walk, 32 elements of the log
 * per trip, the version cursor advanced by ballot / popcount over a 32-element window of version's sequence, or MARKS' walk: a
 * warp-built visible -> record table of log, then one lane merging the two span lists with the open ranges (comment ranks in
 * scratch).  The records go straight into the delta that pt_batch_append's splice reads on the device.  Only the requests, the
 * per-request counts and the view cross PCIe.  Cost per request: TEXT O(n_changes + n_elems(log) + n_elems(version)); MARKS
 * O(n_changes + n_elems(log) + n_visible + (n_spans(log) + n_spans(version)) x the comment ids per span).  Scratch: 4 B per change
 * of each request's log; MARKS also 4 B per ins/del record of log and 32 B per mark record of log and version. */
int pt_batch_restore(pt_batch*, const pt_restore_request* req, uint32_t n, uint32_t mode, pt_restore_view* out);

/* getTextWithFormatting's return value (FormatSpanWithText[], src/peritext.ts:35-38, 337-455) of every merged log as UTF-8
 * JSON text, rendered on the device.  Log i's text is bytes[off[i] .. off[i+1]):
 *   [{"marks":M,"text":T},...]      one object per span, keys sorted; no visible text gives []
 *   M = {"comment":[C,...],"em":{"active":true},"link":L,"strong":{"active":true}}, only the marks present ({} for none);
 *       the comment list follows the span's comment pool order (ascending rank = sortBy id), and is [] for a span whose
 *       PT_SPAN_COMMENT is set with zero ids (quirk Q3)
 *   T = the span's text (the concatenation of its element values, in UTF-16 code units) as JSON.stringify writes a string:
 *       \" \\ \b \t \n \f \r, \u00xx (lowercase) for the other units below U+0020, raw UTF-8 for everything else (U+007F,
 *       U+2028, U+2029, / included); a high surrogate immediately followed by a low surrogate in the same span is one 4-byte
 *       character, also when the halves come from different elements; any other surrogate unit is \udxxx (lowercase)
 *   C, L = the fragments of the caller's pools for the comment rank / link attr id, copied verbatim, except that the 3-byte
 *       encoding of a lone surrogate (ED A0..BF xx) becomes \udxxx; so the output is always valid UTF-8
 * A log whose status is not PT_LOG_OK renders as zero bytes; a log that merged is at least "[]".
 * Pools: data + byte offsets [count + 1] each, the layouts of pt_ingest_pool's kinds PT_POOL_VALUES (UTF-16LE values),
 * PT_POOL_LINK_ATTRS and PT_POOL_COMMENT_ATTRS (canonical JSON), so a C caller passes those three straight through.  A pool
 * with count 0 may have null pointers.
 * Preconditions of pt_batch_download (a completed merge, else PT_ERR_STATE); PT_FLAG_EMIT_SEQUENCE is not needed.  Null pools
 * or out: PT_ERR_INVALID.  A log that merged and names a value index, link id or comment rank >= its pool's count:
 * PT_ERR_INVALID, pt_last_error names the first such entry (lowest log, then value / link / comment, then lowest index), no
 * view.  n_logs == 0: PT_OK with off[0] = 0, nothing launched.
 * Synchronises.  The view is engine-owned pinned memory, valid until the next render, upload or destroy on the handle; the
 * pt_spans_view / pt_patch_view of the same merge stay valid and unchanged, and rendering again gives identical bytes.
 * Device: a size pass and a write pass, one warp per log, 32 elements of a span per trip. */
typedef struct pt_json_pools {          /* layouts = pt_ingest_pool's kinds 0, 1, 3: data + byte offsets [count + 1] */
    const uint8_t* values;   const uint64_t* values_off;   uint64_t n_values;    /* UTF-16LE element values (PT_POOL_VALUES)   */
    const uint8_t* links;    const uint64_t* links_off;    uint64_t n_links;     /* JSON fragment per link attr id              */
    const uint8_t* comments; const uint64_t* comments_off; uint64_t n_comments;  /* JSON fragment per comment rank              */
} pt_json_pools;
typedef struct pt_json_view { uint32_t n_logs; const uint64_t* off; /* [n_logs + 1] */ const char* bytes; uint64_t n_bytes; } pt_json_view;
int pt_batch_render_json(pt_batch*, const pt_json_pools*, pt_json_view* out);

/* PT_FLAG_EMIT_PATCHES: the Patch[] return values of Micromerge.applyChange (src/micromerge.ts:25-31, 659-703;
 * src/peritext.ts:175-281) of every log of the last merge as UTF-8 JSON text, rendered on the device from the patch stream
 * (pt_patch_view).  Log i's text is bytes[off[i] .. off[i+1]).  A log whose merge status is PT_LOG_OK and whose patch status
 * is 0 renders as one array with one inner array per list op of the log, in arrival order (mark record k comes right before
 * ins/del record arrival_k), holding the patches that op's applyChange returned; keys sorted; a log without list ops is []:
 *   insert     [{"action":"insert","index":I,"marks":M,"path":["text"],"values":[V]}]
 *              I = index & 0x7FFFFFFF; M = the marks object of pt_batch_render_json built from the record's flags /
 *              link_attr and its comment ids (ascending rank); V = the element's value alone as JSON.stringify writes a string
 *              (the span render's rules; surrogate halves pair only inside one value)
 *   delete     [{"action":"delete","count":1,"index":I,"path":["text"]}] if bit 31 of index is set, else []
 *   mark op    [{"action":A,"attrs":F,"endIndex":b,"markType":T,"path":["text"],"startIndex":a},...] its mark patches in
 *              ascending startIndex; A addMark / removeMark; T strong / em / comment / link; "attrs" only for addMark of a link
 *              (links pool fragment of attr) or a comment (comments pool fragment of the rank); no patches gives []
 * A log whose merge status is not 0 or whose patch status is 1 renders as zero bytes (pt_log_result.status /
 * pt_patch_view.status say why).  The ROOT makeList patch is not part of the output.  Where ops naming one comment id carry
 * different attrs objects, F and C are the first-seen attrs of the id (the span render's corner).
 * Pools and missing-entry errors as pt_batch_render_json.  Null arguments: PT_ERR_INVALID.  No completed merge, a handle
 * created without PT_FLAG_EMIT_PATCHES, or an item demand of the last merge above the patch pool's capacity (pt_last_error
 * gives the needed count: pt_batch_set_patch_pool and merge again), or a pt_batch_set_patch_pool or pt_batch_set_patch_window
 * since the last merge: PT_ERR_STATE.  n_logs == 0: PT_OK with off[0] = 0.  Under a patch window (pt_batch_set_patch_window)
 * each log renders only the inner arrays of the window's ops.
 * Synchronises.  The view is engine-owned pinned memory of its own, valid until the next pt_batch_render_patches_json,
 * upload or destroy; a pt_batch_render_json view, the pt_spans_view and the pt_patch_view stay valid and unchanged.  The bytes
 * do not depend on the order of the item pool.
 * Device: the item pool ordered by owner and key (count, scan, scatter, rank), then a size pass and a write pass, one warp
 * per log and one lane per op. */
int pt_batch_render_patches_json(pt_batch*, const pt_json_pools*, pt_json_view* out);

/* ------------------------------------------------------------------------------------------------
 * Changes as JSON: the reference's Change objects (src/micromerge.ts:60-71; "can be JSON-encoded to send to another node",
 * :304-307) of resident logs, rendered on the device from the change table and the records, so a batch can serve a peer
 * what it is missing (getMissingChanges, reference test/merge.ts:25-38) or save a document's history.
 *
 * The records hold only the ops that target the log's text list.  The other ops of a change (the ROOT makeList, ops on other
 * objects) and each change's startOp come from an optional side table, the EXTRAS, built where those ops are still visible
 * (pt_ingest_change_extras, packing.change_extras / input_extras).  Without extras the call renders the list-op projection
 * of every change: its list ops only, and startOp = the original counter of its first list op.
 * ---------------------------------------------------------------------------------------------- */
#define PT_EXTRA_NONE 0xFFFFFFFFFFFFFFFFull
typedef struct pt_change_extra {   /* 32 B; sorted by (log, change, pos) */
    uint32_t log;
    uint32_t change;    /* index in the log's change table                                                               */
    uint32_t pos;       /* index in change.ops                                                                           */
    uint32_t reserved;  /* 0                                                                                             */
    uint64_t start_op;  /* change.startOp; every entry of one change has the same value                                  */
    uint64_t op;        /* the op's canonical JSON: entry `op` of the extra-ops pool; PT_EXTRA_NONE: no op, the entry only
                           supplies startOp (then it is the change's only entry and pos is 0)                            */
} pt_change_extra;

#define PT_CHANGES_RANGE 0u     /* changes [first, first + count) of the log's table, clipped at its end                  */
#define PT_CHANGES_MISSING 1u   /* the changes not covered by the request's clock, in getMissingChanges order            */
typedef struct pt_changes_request {   /* 32 B */
    uint32_t log, mode, first, count;
    uint64_t clock_off;                /* MISSING: the peer's clock is clock[clock_off .. clock_off + n_clock)             */
    uint32_t n_clock, reserved;
} pt_changes_request;
typedef struct pt_changes_json_input {
    uint32_t n_requests, reserved;
    const pt_changes_request* requests;
    const pt_clock_entry* clock; uint64_t n_clock;
    pt_json_pools pools;                                       /* as pt_batch_render_json takes them                  */
    const uint8_t* actors; const uint64_t* actors_off;         /* PT_POOL_ACTORS: UTF-16LE ids, byte offsets [count + 1] */
    const uint64_t* actors_first;                              /* [n_logs + 1] log i's actor rank r is entry first[i] + r */
    const uint64_t* counters; const uint64_t* counters_first;  /* PT_POOL_COUNTERS as u64 entries, [n_logs + 1] ranges;
                                                                  an empty range: the log's counters are the original ones */
    const uint8_t* list_ids; const uint64_t* list_ids_off;     /* PT_POOL_LIST_IDS: one UTF-16LE id per log, [n_logs + 1] */
    const pt_change_extra* extras; uint64_t n_extras;          /* NULL / 0: the list-op projection                     */
    const uint8_t* extra_ops; const uint64_t* extra_ops_off; uint64_t n_extra_ops;   /* PT_POOL_EXTRA_OPS               */
} pt_changes_json_input;
#define PT_CHANGES_OK 0u
#define PT_CHANGES_BAD_TABLE 1u  /* MISSING on a table that is not seq-contiguous per actor, or any mode where the table's n_ops
                                    do not sum to the log's n_insdel + n_mark or a change's deps (dep_off + n_deps) leave the
                                    log's dep records                                                                        */
typedef struct pt_changes_json_view {
    uint32_t n_requests;
    const uint64_t* off;        /* [n_requests + 1] request r's text is bytes[off[r] .. off[r+1])                                */
    const char* bytes; uint64_t n_bytes;
    const uint32_t* status;     /* [n_requests] PT_CHANGES_*; a request that is not OK renders zero bytes                        */
} pt_changes_json_view;

/* Render each request's changes of a resident log as the UTF-8 JSON text of a Change[]: "[" + changes joined by "," + "]".
 *   change    {"actor":A,"deps":{...},"ops":[...],"seq":S,"startOp":N}  top-level keys sorted; deps in the table's stored order
 *   insert    {"action":"set","elemId":E,"insert":true,"obj":L,"opId":O,"value":V}
 *   delete    {"action":"del","elemId":E,"obj":L,"opId":O}
 *   mark      {"action":"addMark|removeMark",["attrs":F,]"end":B,"markType":T,"obj":L,"opId":O,"start":B}
 *   boundary  {"elemId":E,"type":"before|after"} or {"type":"startOfText|endOfText"}
 * opIds and elemIds are "ctr@actor" with the original counter (through the counter pool) in decimal; HEAD is "_head" (the form
 * of the oracle and of packing.change_dicts, not the reference's Symbol-dropping JSON.stringify).  Actor ids, L (the log's list
 * id) and V (the element's value alone) follow the span render's JSON.stringify string rules.  "attrs" is present exactly when
 * the mark record's attr is not PT_ATTR_NONE: the links pool fragment, or the comments pool fragment of the rank, which is the
 * first-seen attrs object of the comment id (the renders' corner); strong / em {"active":true} attrs are dropped by the packers
 * and do not come back.  Ops: extra entry e sits at index e.pos of change.ops, the list ops fill the other indices in arrival
 * order (mark record k before ins/del record arrival_k); startOp is the extras' start_op, else the original counter of the
 * change's first list op.  pt_ingest_parse of a rendered log rebuilds the batch's records, change table and pools exactly.
 * Requests:
 *   RANGE    changes [first, first + count) of the log's table, clipped at its end (count 0 or first past the end: "[]")
 *   MISSING  the changes whose seq exceeds the clock's entry for their actor (an absent actor counts as 0), actors in the order
 *            the log's table first shows them, then ascending seq: getMissingChanges with that clock (pt_batch_exchange step 2)
 * Per request status: PT_CHANGES_BAD_TABLE (see above) renders zero bytes; the other requests proceed.  A table that admission
 * rejected still renders when it is seq-gapped or misses a dependency, since RANGE does not need causal order.
 * Refused, no view (pt_last_error names the first offender):
 *   PT_ERR_STATE    no batch, or a handle without a change table
 *   PT_ERR_INVALID  null arguments; a request's log >= n_logs, unknown mode, or clock range outside the clock array; a clock
 *                   actor >= the log's n_actors; extras out of order, naming a log or change outside the batch, with different
 *                   start_op in one change, a NONE entry beside another entry, an op outside the extra-ops pool, or a pos past
 *                   the change's ops; a pool entry the output needs and the pools do not hold (actor, counter, value, link,
 *                   comment); a selected change with neither list ops nor extras (it has no startOp)
 * n_requests == 0: PT_OK, nothing launched.  Needs no merge and works on logs whose merge failed.  Every other view of the handle
 * stays valid and unchanged.  Synchronises.  The view is engine-owned pinned memory of its own, valid until the next
 * pt_batch_render_changes_json, upload or destroy.
 * Device: a select kernel, one warp per request (the list-op positions, for MISSING the peer's clock in shared memory and the
 * queue as pt_batch_exchange builds it); the selected changes cut into work items of at most 1024 list ops; a size pass, a scan
 * and a write pass, one warp per item and one lane per op.  Two read-backs: the item count and the byte total. */
int pt_batch_render_changes_json(pt_batch*, const pt_changes_json_input* in, pt_changes_json_view* out);

/* Copy only the per-log result headers (status, counts, digest). Synchronises the stream. */
int pt_batch_download_results(pt_batch*, pt_log_result* out, uint32_t n_logs);

/* Device pointer to the per-log result headers ([n_logs] pt_log_result) — for the multi-GPU digest
 * all-gather without a host round trip. */
int pt_batch_device_results(pt_batch*, void** dev_ptr, uint32_t* n_logs);

/* Number of kernel launches the handle has enqueued so far (bench `gpu_launches`). */
uint64_t pt_batch_launch_count(const pt_batch*);

/* Diagnostics of the last merge: out[0] = logs materialised entirely in shared memory, out[1] = logs that were
 * restarted on the spill-capable path (working set larger than the bin's shared-memory budget), out[2] = logs deferred on
 * the device to a kernel variant with a larger budget, out[3] = comment-pool entries the batch needs. Synchronises. */
int pt_batch_stats(pt_batch*, uint64_t out[4]);

/* Resize the comment pool (entries of 4 bytes) of the current batch and of later uploads.  Logs that find the pool full
 * report PT_LOG_OVERFLOW (which ones depends on scheduling); pt_spans_view.comment_pool_needed / pt_batch_stats out[3]
 * give the batch's exact demand, so ONE re-merge after pt_batch_set_comment_pool(needed) always succeeds and is
 * deterministic.  Synchronises. */
int pt_batch_set_comment_pool(pt_batch*, uint64_t entries);

/* Time of the last pt_batch_merge on the device, in milliseconds (CUDA events recorded on the
 * handle's stream around the launches); <0 if not available. Synchronises. */
float pt_batch_last_merge_ms(pt_batch*);

void pt_batch_destroy(pt_batch*);

/* ------------------------------------------------------------------------------------------------
 * Native wire-format ingest (host, multithreaded): JSON text of the reference's Change objects
 * (src/micromerge.ts:60-71; the `queues` of the traces/ files) -> packed batch + change table + string pools.
 * logs_json[i] = UTF-8 JSON array of the Change objects replica i applied, in arrival order.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pt_ingest pt_ingest;
#define PT_POOL_VALUES 0        /* multi-character element values, UTF-16LE; token = PT_TOKEN_POOLED | index          */
#define PT_POOL_LINK_ATTRS 1    /* link attrs as canonical JSON (UTF-8); pt_mark_rec.attr = index                      */
#define PT_POOL_COMMENT_IDS 2   /* comment ids, UTF-16LE, in rank order (JS string order); pt_mark_rec.attr = rank     */
#define PT_POOL_COMMENT_ATTRS 3 /* the first-seen attrs object of each comment id as canonical JSON, same order        */
#define PT_POOL_ACTORS 4        /* actor ids UTF-16LE, rank order per log; per_log_first[i] .. per_log_first[i+1]       */
#define PT_POOL_COUNTERS 5      /* dense counter rank -> original counter (u64 each) of logs whose counters were
                                   re-ranked; empty range otherwise; per_log_first as above                            */
#define PT_POOL_LIST_IDS 6      /* each log's text-list object id, UTF-16LE, one entry per log (empty: no list)        */
#define PT_POOL_EXTRA_OPS 7     /* the canonical JSON (UTF-8) of every op that does not target its log's text list, in
                                   the order of the extras (pt_change_extra.op indexes it)                             */
int pt_ingest_create(pt_ingest** out);
int pt_ingest_parse(pt_ingest*, const char* const* logs_json, const uint64_t* lens, uint32_t n_logs, int threads /* 0 = all cores */);
/* Views into the parsed batch (valid until the next pt_ingest_parse / pt_ingest_destroy). */
int pt_ingest_packed(pt_ingest*, pt_packed_ops* ops, pt_change_table* changes);
int pt_ingest_pool(pt_ingest*, int kind, const uint8_t** data, const uint64_t** offsets /* [count + 1] */, uint64_t* count,
                   const uint64_t** per_log_first /* may be NULL */);
/* The extras of the parsed batch (pt_batch_render_changes_json): per change, in order, one entry per op that does not target
 * the log's text list, and a PT_EXTRA_NONE entry for a change that has no such op but has no list op either, or whose startOp
 * is not the counter of its first list op.  Sorted by (log, change, pos). */
int pt_ingest_change_extras(pt_ingest*, const pt_change_extra** out, uint64_t* n);
const char* pt_ingest_error(pt_ingest*);
void pt_ingest_destroy(pt_ingest*);

const char* pt_strerror(int status);
const char* pt_last_error(void); /* thread-local detail string of the last failing call */
const char* pt_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PERITEXT_B200_H */
