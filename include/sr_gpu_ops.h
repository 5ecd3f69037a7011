/*
 * sr_gpu_ops.h -- C-ABI of the H100-native StarRocks BE hot path
 * (columnar Chunk scan -> predicate/filter -> hash-join build+probe -> hash aggregate,
 *  plus the hash-partition step of ExchangeSink).
 *
 * This is the drop-in boundary: plain C structs, opaque handles, int32 status codes,
 * no exceptions and no torch / C++ types in any signature.  The C++ adapters in
 * starrocks_b200/host/ (GpuScanOperator, GpuHashJoinBuild/ProbeOperator,
 * GpuAggregateBlockingSink/SourceOperator) are thin shims over these calls and keep the
 * reference's pipeline::Operator / OperatorFactory virtual interface
 * (be/src/exec/pipeline/operator.h:44-352, :354-456; source_operator.h:37-189).
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * StarRocks source tree).
 *
 * Conventions
 *  - every function returning int32_t returns SR_OK (0) or a negative sr_status; the message
 *    is available from sr_last_error(ctx).
 *  - a sr_chunk_view mirrors column::Chunk (be/src/column/chunk.h:52): equal-length columns
 *    addressed by slot id.  `mem` says whether the column pointers are host or device
 *    addresses.  Host chunks are copied H2D by the callee on the context's stream; device
 *    chunks are consumed in place (zero copy) and must stay valid until sr_ctx_sync().
 *  - all work is enqueued on the context's CUDA stream; calls return without synchronising
 *    unless documented ("_sync" or a pull that hands back host memory).
 *  - build row indexes are 1-based; 0 means "no row" (the reference reserves build row 0 as a
 *    sentinel, be/src/exec/join/join_hash_table.cpp:712-752).
 */
#ifndef SR_GPU_OPS_H
#define SR_GPU_OPS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SR_ABI_VERSION 1

/* ---------------------------------------------------------------------------------------
 * status codes (negative = error).  Mirrors the Status codes the adapters translate to
 * (be/src/base/status.h): InvalidArgument, NotSupported, MemoryLimitExceeded, InternalError.
 * ------------------------------------------------------------------------------------- */
typedef enum sr_status {
    SR_OK = 0,
    SR_ERR_INVALID_ARGUMENT = -1,
    SR_ERR_NOT_SUPPORTED = -2,
    SR_ERR_OUT_OF_MEMORY = -3,
    SR_ERR_CUDA = -4,
    SR_ERR_STATE = -5, /* call made in the wrong phase (e.g. probe before build_finish)          */
    SR_ERR_NO_DEVICE = -6
} sr_status;

/* ---------------------------------------------------------------------------------------
 * logical types -- subset of be/src/types/logical_type.h used by the hot path.
 * Physical layout = FixedLengthColumnBase<T> (be/src/column/fixed_length_column_base.h:49):
 * a contiguous array of T.  DATE = int32 julian day (types/date_value.h:120), DATETIME =
 * int64 (types/timestamp_value.h:165), DECIMAL32/64/128 = DecimalV3<int32/int64/int128>.
 * ------------------------------------------------------------------------------------- */
typedef enum sr_type {
    SR_TYPE_BOOLEAN = 1,  /* uint8  */
    SR_TYPE_TINYINT = 2,  /* int8   */
    SR_TYPE_SMALLINT = 3, /* int16  */
    SR_TYPE_INT = 4,      /* int32  */
    SR_TYPE_BIGINT = 5,   /* int64  */
    SR_TYPE_LARGEINT = 6, /* int128 */
    SR_TYPE_FLOAT = 7,
    SR_TYPE_DOUBLE = 8,
    SR_TYPE_DATE = 9,       /* int32 */
    SR_TYPE_DATETIME = 10,  /* int64 */
    SR_TYPE_DECIMAL32 = 11, /* int32 */
    SR_TYPE_DECIMAL64 = 12, /* int64 */
    SR_TYPE_DECIMAL128 = 13 /* int128 */
} sr_type;

/* byte width of one value of the type (0 for an unknown type). */
int32_t sr_type_width(int32_t type);

/* Where a caller's buffer lives: every `mem`, `sel_mem`, `out_mem`, `dst_mem`, `src_mem` argument and sr_chunk_view.mem.
 * SR_MEM_HOST: pageable or pinned host memory, copied with H2D / D2H copies on the context's stream.
 * SR_MEM_DEVICE: device pointers, read and written in place.
 * SR_MEM_HOST_PINNED: page-locked host memory mapped into the device address space (cudaHostAlloc /
 *   cudaHostRegister, e.g. a registered ColumnAllocator pool).
 * One rule for all entry points:
 *  1. An unknown kind is refused with SR_ERR_INVALID_ARGUMENT before any copy, allocation or launch.
 *  2. Only sr_fragment_push (the fact columns), sr_fragment_push_chunks (the chunks' columns) and sr_pages_decode /
 *     sr_null_maps_decode (the pages) read SR_MEM_HOST_PINNED buffers IN PLACE over PCIe: the fragment fetches a column
 *     only for the 32-byte sectors holding rows that survived the earlier joins, so far fewer bytes cross the bus than a
 *     full H2D copy; sr_fragment_push_chunks reads every column the fragment needs in full, once, with device loads.
 *     These three resolve a buffer read in place through the library's registry of the ranges made by sr_host_alloc and
 *     sr_host_register first (no driver call); a pointer outside it costs one driver lookup per allocation and call.
 *     Memory that is not page-locked and mapped is refused with SR_ERR_INVALID_ARGUMENT.  Every other entry point treats
 *     SR_MEM_HOST_PINNED exactly like SR_MEM_HOST, for inputs and for outputs.
 *  3. A call that writes its result into host memory (either host kind) synchronises before it returns; a result
 *     handed back in host memory (sr_chunk_out.mem) is reported as SR_MEM_HOST.
 *  4. Host inputs: a call waits for the copies of its host inputs before it returns, so that the caller may free or
 *     reuse them, except sr_fragment_push, sr_fragment_push_chunks, sr_agg_push and sr_agg_push_selective on a dense or
 *     single-state table,
 *     sr_scan_evaluate with a device selection, sr_xchg_hash with device outputs and sr_chunk_serialize into device
 *     memory.  After one of these a page-locked input (pageable memory may be reused at once), and after any call a
 *     buffer read in place, must stay valid and unmodified until the next synchronising call on the context
 *     (sr_ctx_sync, sr_agg_sink_finish, sr_fragment_rows_passed, or any call that waits). */
typedef enum sr_mem { SR_MEM_HOST = 0, SR_MEM_DEVICE = 1, SR_MEM_HOST_PINNED = 2 } sr_mem;

/* mirrors FixedLengthColumn / NullableColumn raw buffers (be/src/column/nullable_column.h:32:
 * data column + uint8 null column, 1 = null). nulls == NULL means "not nullable / no nulls".
 * Alignment: a column the kernels read in place (SR_MEM_DEVICE, and SR_MEM_HOST_PINNED where it is read in place) must be
 * naturally aligned: `data` a multiple of the value width, of 8 bytes for 16-byte values (so row k of a larger column
 * qualifies).  Such a column that is not is refused with SR_ERR_INVALID_ARGUMENT before any launch.  SR_MEM_HOST columns
 * are copied and may have any alignment. */
typedef struct sr_col_view {
    const void* data;
    const uint8_t* nulls;
    int32_t type;    /* sr_type */
    int32_t slot_id; /* SlotId the column is registered under in the Chunk */
} sr_col_view;

/* mirrors column::Chunk (be/src/column/chunk.h:52-354).
 * Every entry point that takes one refuses, with SR_ERR_INVALID_ARGUMENT before any allocation, copy or launch: an
 * unknown mem kind, num_rows < 0, num_cols < 0, cols == NULL with num_cols > 0, and, in a column it reads, an unknown
 * type, data == NULL with num_rows > 0 or a column read in place that is not naturally aligned (see sr_col_view). */
typedef struct sr_chunk_view {
    const sr_col_view* cols;
    int32_t num_cols;
    int32_t mem; /* sr_mem: where the column pointers live */
    int64_t num_rows;
} sr_chunk_view;

/* Output chunk.  Buffers are owned by the producing handle and stay valid until the next
 * pull / release on the same handle (same contract as a ChunkPtr the operator keeps alive). */
typedef struct sr_col_out {
    void* data;
    uint8_t* nulls; /* NULL when the column has no null column */
    int32_t type;
    int32_t slot_id;
} sr_col_out;

#define SR_MAX_OUT_COLS 32

typedef struct sr_chunk_out {
    sr_col_out cols[SR_MAX_OUT_COLS];
    int32_t num_cols;
    int32_t mem; /* sr_mem of the buffers handed back */
    int64_t num_rows;
} sr_chunk_out;

/* ---------------------------------------------------------------------------------------
 * context: one per GPU (one per BE process per device); owns the stream and the device
 * memory the operators allocate.  Plays the part of RuntimeState + MemTracker for the GPU
 * side (be/src/exec/pipeline/operator.h:157,350).
 * ------------------------------------------------------------------------------------- */
typedef struct sr_ctx sr_ctx;

/* device: CUDA ordinal.  stream: a cudaStream_t to enqueue on, or NULL to create one. */
sr_ctx* sr_ctx_create(int32_t device, void* cuda_stream);
void sr_ctx_destroy(sr_ctx* ctx);
/* cudaStreamSynchronize on the context's stream; surfaces any asynchronous kernel error. */
int32_t sr_ctx_sync(sr_ctx* ctx);
/* last error message recorded on this context (never NULL). With ctx == NULL: the message
 * of the last failed create call on this thread. */
const char* sr_last_error(sr_ctx* ctx);
/* sr_status of the last failure recorded on this context -- needed after a *_create call
 * returned NULL (the status cannot travel in the return value there). */
int32_t sr_last_error_code(sr_ctx* ctx);
int32_t sr_abi_version(void);
/* number of kernels this library has launched on the context since creation
 * (bench.py reports it as gpu_launches). */
int64_t sr_ctx_kernel_launches(sr_ctx* ctx);
/* bytes of device memory currently held by the context's handles. */
int64_t sr_ctx_device_bytes(sr_ctx* ctx);
void* sr_ctx_stream(sr_ctx* ctx);

/* ---------------------------------------------------------------------------------------
 * scan predicates -- the pushed-down / non-pushdown `col OP const` conjuncts.
 * Replaces ColumnPredicate::evaluate / evaluate_and (be/src/storage/column_predicate.h:128-149,
 * column_operator_predicate.h:41-111) and the AND-merge of ChunkPredicateEvaluator::
 * eval_conjuncts (be/src/exprs/chunk_predicate_evaluator.cpp:84-149).
 * A NULL input never passes (count_true_with_notnull semantics), except IS_NULL.
 * ------------------------------------------------------------------------------------- */
typedef enum sr_pred_op {
    SR_PRED_EQ = 1,
    SR_PRED_NE = 2,
    SR_PRED_LT = 3,
    SR_PRED_LE = 4,
    SR_PRED_GT = 5,
    SR_PRED_GE = 6,
    SR_PRED_BETWEEN = 7, /* lo <= v <= hi */
    SR_PRED_IN = 8,
    SR_PRED_NOT_IN = 9,
    SR_PRED_IS_NULL = 10,
    SR_PRED_IS_NOT_NULL = 11
} sr_pred_op;

#define SR_MAX_IN_LIST 16

typedef struct sr_pred {
    int32_t slot_id;
    int32_t op; /* sr_pred_op */
    /* integer / date / decimal columns compare against ilo (and ihi for BETWEEN);
     * FLOAT / DOUBLE columns compare against dlo (and dhi). */
    int64_t ilo, ihi;
    double dlo, dhi;
    int64_t in_list[SR_MAX_IN_LIST]; /* IN / NOT_IN on integer-class columns */
    int32_t in_count;
    int32_t reserved;
} sr_pred;

/* ---------------------------------------------------------------------------------------
 * expressions -- postfix programs over slots; the subset of the vectorized Expr tree the
 * path needs (be/src/exprs/binary_predicate.cpp:134-143, compound_predicate.cpp,
 * arithmetic_expr.cpp, column_ref.h).  Integer-class operands are computed in int64 with
 * two's-complement wrap (the FE casts INT operands of + - * to BIGINT); FLOAT/DOUBLE in
 * double.  Comparison / AND / OR / NOT follow SQL three-valued logic.
 * ------------------------------------------------------------------------------------- */
typedef enum sr_expr_op {
    SR_EX_COL = 1,    /* push slot value                          */
    SR_EX_ICONST = 2, /* push ival                                */
    SR_EX_DCONST = 3, /* push dval                                */
    SR_EX_ADD = 4,
    SR_EX_SUB = 5,
    SR_EX_MUL = 6,
    SR_EX_TO_DOUBLE = 7, /* cast top of stack to double            */
    SR_EX_EQ = 8,
    SR_EX_NE = 9,
    SR_EX_LT = 10,
    SR_EX_LE = 11,
    SR_EX_GT = 12,
    SR_EX_GE = 13,
    SR_EX_AND = 14,
    SR_EX_OR = 15,
    SR_EX_NOT = 16,
    SR_EX_IS_NULL = 17,
    SR_EX_DIV = 18 /* double division only (ints are cast first) */
} sr_expr_op;

typedef struct sr_expr_node {
    int32_t op; /* sr_expr_op */
    int32_t slot_id;
    int64_t ival;
    double dval;
} sr_expr_node;

#define SR_MAX_EXPR_NODES 24
#define SR_EXPR_STACK 8

typedef struct sr_expr {
    sr_expr_node nodes[SR_MAX_EXPR_NODES];
    int32_t num_nodes;
    int32_t reserved;
} sr_expr;

/* ---------------------------------------------------------------------------------------
 * scan + filter.  Replaces OlapChunkSource::_read_chunk_from_storage's filter step
 * (be/src/exec/pipeline/scan/olap_chunk_source.cpp:676-722): predicate evaluation into a
 * uint8 selection vector, then Chunk::filter -> Column::filter_range order-preserving
 * compaction (be/src/column/chunk.cpp:362-372, column_filter_range.cpp:39-148).
 * The GPU ScanOperator batches many <=4096-row chunks per push.
 * ------------------------------------------------------------------------------------- */
typedef struct sr_scan_desc {
    const sr_pred* preds; /* conjuncts in ColumnPredicate form */
    int32_t num_preds;
    int32_t num_filter_exprs;
    const sr_expr* filter_exprs; /* generic boolean conjuncts (ChunkPredicateEvaluator) */
    const int32_t* out_slots;    /* slots to emit (in this order) */
    int32_t num_out_slots;
    int32_t reserved;
} sr_scan_desc;

typedef struct sr_scan sr_scan;

/* ScanOperator / ChunkSource::prepare with the conjuncts of the scan node (scan_operator.cpp:69-112). */
sr_scan* sr_scan_create(sr_ctx* ctx, const sr_scan_desc* desc);
void sr_scan_destroy(sr_scan* scan);
/* OlapChunkSource::_read_chunk_from_storage, the part behind the segment iterator (olap_chunk_source.cpp:676-722);
 * the adapter's ScanOperator::pull_chunk (scan_operator.cpp:286-309) hands its result on.
 * filter one batch.  `out` receives DEVICE buffers (owned by the scan handle, valid until the
 * next push) holding the surviving rows in input order; out->num_rows is filled after an
 * internal sync on the tiny row counter. */
int32_t sr_scan_filter(sr_scan* scan, const sr_chunk_view* in, sr_chunk_out* out);
/* evaluate only: write the uint8 selection vector (1 = row passes) to `selection` in sel_mem (sr_mem rules: a host
 * selection is complete on return) -- the ColumnPredicate::evaluate contract. */
int32_t sr_scan_evaluate(sr_scan* scan, const sr_chunk_view* in, uint8_t* selection, int32_t sel_mem);

/* ---------------------------------------------------------------------------------------
 * hash join.  One sr_join is shared by the build operator and the N probe operators, like
 * HashJoiner (be/src/exec/hash_joiner.h:191-330).
 *   append_build  <- HashJoiner::append_chunk_to_ht / JoinHashTable::append_chunk
 *                    (hash_joiner.cpp:213-223, join_hash_table.cpp:712-752)
 *   build_finish  <- HashJoiner::build_ht / JoinHashTable::build (join_hash_table.cpp:633-685,
 *                    selector :161-350, construct_hash_table join_hash_map_method.hpp)
 *   probe         <- JoinHashTable::probe / JoinHashMap::probe (join_hash_map.hpp:63-134,
 *                    _probe_from_ht :718-795, _probe_output/_build_output :163-269)
 * ------------------------------------------------------------------------------------- */
typedef enum sr_join_type {
    SR_JOIN_INNER = 0,
    SR_JOIN_LEFT_OUTER = 1,
    SR_JOIN_LEFT_SEMI = 2,
    SR_JOIN_LEFT_ANTI = 3,
    /* Joins that emit build rows after the probe phase (HashJoiner's POST_PROBE phase, exec/hash_joiner.h:161-188,314-329;
     * JoinHashMap::probe_remain / _search_ht_remain, join_hash_map.hpp:136-143,420-457).  Every probe marks the build rows
     * it matched (HashTableProbeState::build_match_index); after the last probe sr_join_probe_remain emits, in build
     * order, the rows that were never matched (RIGHT OUTER, FULL OUTER, RIGHT ANTI; build rows with a NULL key never
     * match) or that were matched (RIGHT SEMI).  Probe-phase output: RIGHT OUTER = INNER, FULL OUTER = LEFT OUTER, RIGHT
     * SEMI / ANTI nothing.  (The reference emits RIGHT SEMI rows during the probe, at their first match,
     * join_hash_map.hpp:1405-1440; here they come out of the remain call in build order -- the same rows.) */
    SR_JOIN_RIGHT_OUTER = 4,
    SR_JOIN_RIGHT_SEMI = 5,
    SR_JOIN_RIGHT_ANTI = 6,
    SR_JOIN_FULL_OUTER = 7
} sr_join_type;

/* table layout chosen at build_finish; mirrors JoinHashMapMethodType
 * (be/src/exec/join/join_hash_map_method_fwd.h) for the families the GPU path implements. */
typedef enum sr_join_method {
    SR_JOIN_METHOD_NONE = 0,
    SR_JOIN_METHOD_DIRECT_MAPPING = 1,       /* <= 16-bit keys: first[key - type_min]           */
    SR_JOIN_METHOD_RANGE_DIRECT_MAPPING = 2, /* first[key - min_value]                          */
    SR_JOIN_METHOD_LINEAR_CHAINED = 3        /* open addressing, chain of equal keys in next[]  */
} sr_join_method;

#define SR_MAX_JOIN_KEYS 4
#define SR_MAX_JOIN_OUT 16

typedef struct sr_join_desc {
    int32_t join_type; /* sr_join_type */
    int32_t num_keys;  /* 1..SR_MAX_JOIN_KEYS; the packed key must fit 16 bytes (<= 8: SERIALIZED_FIXED_SIZE_INT / BIGINT, 9..16:
                        * SERIALIZED_FIXED_SIZE_LARGEINT, join_hash_table.cpp:221-250) */
    int32_t build_key_slots[SR_MAX_JOIN_KEYS];
    int32_t probe_key_slots[SR_MAX_JOIN_KEYS];
    int32_t key_types[SR_MAX_JOIN_KEYS]; /* sr_type, integer class */
    /* columns of the build / probe side that appear in the join's output chunk */
    int32_t num_build_out;
    int32_t build_out_slots[SR_MAX_JOIN_OUT];
    int32_t num_probe_out;
    int32_t probe_out_slots[SR_MAX_JOIN_OUT];
    /* session switch enable_hash_join_range_direct_mapping_opt (join_hash_table.cpp:259) */
    int32_t enable_range_direct_mapping;
    int32_t reserved;
    /* sr_type of every build_out_slot (0 = take it from the appended chunks).  The reference knows the build side's
     * schema from the plan (HashJoinerParam::_build_row_descriptor, exec/hash_joiner.h:66-133) even when no build chunk
     * ever arrives -- a dimension scan that filters everything out; with the types declared here such a join probes to
     * zero rows (INNER / SEMI) or to NULL-padded rows (LEFT OUTER) instead of failing. */
    int32_t build_out_types[SR_MAX_JOIN_OUT];
    /* sr_type of every probe_out_slot (0 = take it from the probed chunks): sr_join_probe_remain pads the probe columns
     * of RIGHT / FULL OUTER rows with NULLs and needs their types even when no probe chunk ever arrived */
    int32_t probe_out_types[SR_MAX_JOIN_OUT];
    /* other-join conjunct (HashJoiner::_other_join_conjunct_ctxs, exec/hash_joiner.h:314-329; applied by
     * JoinHashMap / HashJoinProber after the key match, hash_joiner.cpp `_process_other_conjunct`,
     * `_process_outer_join_with_other_conjunct`, `_process_semi_join_with_other_conjunct`, ...): a boolean expression over
     * slots of the PROBE chunk and of the BUILD chunk (slot ids of the two sides are distinct, as in the output chunk).
     * num_nodes = 0: none.  A key-matched pair only counts when the conjunct is true (NULL = false): INNER / RIGHT OUTER
     * emit the passing pairs, LEFT / FULL OUTER pad probe rows without a passing pair, LEFT SEMI / ANTI test "some pair
     * passes", RIGHT / FULL joins mark build rows by passing pairs only.  Output keeps probe order. */
    sr_expr other_conjunct;
} sr_join_desc;

typedef struct sr_join sr_join;

typedef struct sr_join_info {
    int32_t method;         /* sr_join_method */
    int32_t has_duplicates; /* 1 when some build key occurs more than once */
    int64_t build_rows;     /* rows appended (excluding the sentinel row 0) */
    int64_t bucket_size;    /* entries of first[] */
    int64_t min_value, max_value;
} sr_join_info;

/* HashJoiner::prepare_builder / prepare_prober + _init_hash_table_param (be/src/exec/hash_joiner.cpp:115-211). */
sr_join* sr_join_create(sr_ctx* ctx, const sr_join_desc* desc);
void sr_join_destroy(sr_join* join);
/* HashJoinBuildOperator::push_chunk -> HashJoiner::append_chunk_to_ht (hash_join_build_operator.cpp:41-43,
 * hash_joiner.cpp:213-223). */
int32_t sr_join_append_build(sr_join* join, const sr_chunk_view* chunk);
/* HashJoinBuildOperator::set_finishing -> HashJoiner::build_ht (hash_join_build_operator.cpp:86-220, hash_joiner.cpp:248-262):
 * chooses the hash-map method and builds first[] / next[]. */
int32_t sr_join_build_finish(sr_join* join);
/* HashJoinProbeOperator::is_ready (hash_join_probe_operator.cpp:75-77): probers wait for HashJoinPhase::PROBE. */
int32_t sr_join_is_build_done(const sr_join* join);
int32_t sr_join_get_info(const sr_join* join, sr_join_info* info);
/* copy first[] / next[] back to the host (test / debug aid; sizes from sr_join_get_info:
 * bucket_size and build_rows + 1). Only for the *_MAPPING methods is first[] comparable with
 * the reference layout. */
int32_t sr_join_copy_table(sr_join* join, uint32_t* first_host, uint32_t* next_host);

/* HashJoinProbeOperator::push_chunk + pull_chunk -> HashJoiner::push_chunk / _pull_probe_output_chunk
 * (hash_join_probe_operator.cpp:79-88, hash_joiner.cpp:288-330) -> JoinHashTable::probe (join_hash_table.cpp:695-702).
 * Probe one batch (any number of rows).  Output rows keep probe order; matches of one probe
 * row are adjacent.  `out` holds DEVICE buffers owned by the join handle (per prober_id),
 * valid until the next probe with the same prober_id.  Also exposes the
 * (probe_index, build_index) pairs of HashTableProbeState
 * (be/src/exec/join/join_hash_table_descriptor.h:207-330). */
int32_t sr_join_probe(sr_join* join, int32_t prober_id, const sr_chunk_view* probe, sr_chunk_out* out);
/* POST_PROBE phase of SR_JOIN_RIGHT_* / SR_JOIN_FULL_OUTER (see sr_join_type): call once, after every prober's last
 * sr_join_probe has returned (the reference lets the last HashJoinProbeOperator to finish do this, hash_joiner.cpp:315-327).
 * All rows come in one chunk -- probe_out columns first (all NULL; absent for RIGHT SEMI / ANTI), then the build_out columns --
 * in DEVICE buffers owned by the join (valid until the next call on this join); the adapter slices it into chunk_size pieces. */
int32_t sr_join_probe_remain(sr_join* join, sr_chunk_out* out);
/* device pointers to the index pairs of the last probe of prober_id (num = out->num_rows). */
int32_t sr_join_probe_indexes(sr_join* join, int32_t prober_id, const uint32_t** probe_index_dev,
                              const uint32_t** build_index_dev);

/* K5: JoinKeyHash / calc_bucket_num (be/src/exec/join/join_hash_map_helper.h:35-54,79-84)
 * on the device, exposed so the multiplicative hash can be pinned against the reference's
 * golden vectors.  keys: `n` values of key_type in `mem`; buckets: n uint32 in `mem` (sr_mem rules: host buckets are
 * complete on return; device keys and buckets must be naturally aligned). */
int32_t sr_join_key_hash(sr_ctx* ctx, const void* keys, int32_t key_type, int64_t n, uint32_t log_bucket_size,
                         uint32_t* buckets, int32_t mem);

/* ---------------------------------------------------------------------------------------
 * runtime filter (SURVEY.md 8f-1): what HashJoinBuildOperator::set_finishing publishes to the scans of the probe side
 * (hash_join_build_operator.cpp:100-215) -- min/max + has_null (MinMaxRuntimeFilter, be/src/runtime/runtime_filter.h:584)
 * and a split-block bloom filter with the reference's exact layout and hashing (SimdBlockFilter, runtime_filter.h:79-240:
 * 32-byte buckets of 8 words, bucket = hash & mask, bit i = (uint32(hash >> log_buckets) * SALT[i]) >> 27;
 * hash = phmap_mix<8>(std::hash(value)), runtime_filter.h:1270-1276).  The directory bytes equal the reference's
 * `_directory`, so a filter built here can be merged with / shipped to CPU BEs and vice versa.
 * Integer-class single-column keys (width <= 8).
 * ------------------------------------------------------------------------------------- */
typedef struct sr_rf sr_rf;
typedef struct sr_rf_info {
    int64_t min_value, max_value; /* min > max: no non-NULL key was inserted */
    int64_t num_inserted;         /* non-NULL keys */
    int32_t has_null;             /* a NULL key was inserted (null-safe joins) */
    int32_t log_num_buckets;      /* directory = 2^log_num_buckets buckets of 32 bytes; 0: no bloom part */
    int32_t key_type;
    int32_t num_in_values;        /* runtime IN filter: distinct keys held (exact membership); -1: no IN part (more than
                                   * SR_RF_IN_FILTER_ROW_LIMIT rows were inserted) */
} sr_rf_info;
/* HashJoiner::runtime_in_filter_row_limit / max_pushdown_conditions_per_column (hash_joiner.h:270, hash_joiner.cpp:563-575):
 * membership filters (with_bloom != 0) over at most this many build rows also carry their distinct keys; membership is
 * then tested exactly */
#define SR_RF_IN_FILTER_ROW_LIMIT 1024
/* Build from key number `key_index` of a finished join build side.  with_bloom = 0 builds the min/max part only.
 * insert_nulls != 0 records NULL build keys (has_null) -- the reference does so for null-safe equal joins. */
sr_rf* sr_join_build_runtime_filter(sr_join* join, int32_t key_index, int32_t with_bloom, int32_t insert_nulls);
/* Build from a column of a chunk (the general RuntimeFilterBuilder path); expected_rows sizes the bloom directory
 * exactly like SimdBlockFilter::init(expected_rows). */
sr_rf* sr_rf_create(sr_ctx* ctx, int32_t key_type, int64_t expected_rows, int32_t with_bloom);
int32_t sr_rf_insert(sr_rf* rf, const sr_chunk_view* in, int32_t slot_id, int32_t insert_nulls);
/* the IN part: copy the sorted distinct keys out (returns their number, or -1 when the filter has no IN part); merge the keys
 * of a partial filter in (n = -1: the partial filter has no IN part, so the merged one has none either) */
int32_t sr_rf_copy_in_values(sr_rf* rf, int64_t* values_host, int32_t capacity);
int32_t sr_rf_merge_in_values(sr_rf* rf, const int64_t* values_host, int32_t n);
void sr_rf_destroy(sr_rf* rf);
int32_t sr_rf_get_info(sr_rf* rf, sr_rf_info* info);
/* bloom directory: copy out (bytes = 32 << log_num_buckets) / merge another filter in: OR of the directories
 * (SimdBlockFilter::merge; `mem` says where `directory` lives; NULL when `other` has no bloom part) and union of
 * min/max/has_null/num_inserted taken from `other` -- the wire-compatible parts of serialize / merge.  A SR_MEM_DEVICE
 * directory is read in place and must be 4-byte aligned, else SR_ERR_INVALID_ARGUMENT. */
int32_t sr_rf_copy_directory(sr_rf* rf, void* dst, int64_t bytes, int32_t mem);
int32_t sr_rf_merge_directory(sr_rf* rf, const void* directory, int64_t bytes, int32_t mem, const sr_rf_info* other);
/* RuntimeFilter::evaluate on one column of a chunk: selection[i] = has_null for NULL rows, else min <= v <= max and
 * bloom test.  merge_and != 0: rows already 0 in `selection` stay 0 (the merged-selection use of the probe collector). */
int32_t sr_rf_evaluate(sr_rf* rf, const sr_chunk_view* in, int32_t slot_id, uint8_t* selection, int32_t sel_mem, int32_t merge_and);
/* Attach the filter to a scan: rows of `probe_slot` that fail it are dropped by sr_scan_filter / sr_scan_evaluate after
 * the conjuncts (the ScanOperator side of runtime filters, scan_operator.h:212-225).  At most SR_MAX_SCAN_RFS per scan;
 * the filter must outlive the scan. */
#define SR_MAX_SCAN_RFS 4
/* Use of runtime filter `index` (order of sr_scan_add_runtime_filter) by sr_scan_filter so far.  Like
 * RuntimeFilterProbeCollector (runtime_filter_probe.cpp:203-262,408-480) the scan measures every filter's selectivity (rows
 * passed / rows tested) and stops evaluating a filter that lets more than half of its rows through for the next 31 batches,
 * then samples it again.  adaptive = 0 in sr_scan_set_rf_adaptive evaluates every filter on every batch. */
typedef struct sr_scan_rf_stats {
    int64_t rows_tested, rows_passed; /* over the batches that evaluated the filter */
    int64_t batches_skipped;          /* batches on which it was switched off */
    double last_selectivity;
} sr_scan_rf_stats;
int32_t sr_scan_add_runtime_filter(sr_scan* scan, sr_rf* rf, int32_t probe_slot);
int32_t sr_scan_get_rf_stats(sr_scan* scan, int32_t index, sr_scan_rf_stats* stats);
int32_t sr_scan_set_rf_adaptive(sr_scan* scan, int32_t adaptive);

/* ---------------------------------------------------------------------------------------
 * hash aggregate.  One sr_agg is shared by the sink and source operators, like Aggregator
 * (be/src/exec/aggregator.h:253-637).
 *   push         <- AggregateBlockingSinkOperator::push_chunk: evaluate_groupby_exprs,
 *                   build_hash_map, compute_batch_agg_states
 *                   (aggregate_blocking_sink_operator.cpp:101-138, aggregator.cpp:907-929,
 *                   1616-1640) or compute_single_agg_state when there is no GROUP BY (:882-905)
 *   sink_finish  <- set_finishing / sink_complete (:56-89)
 *   pull         <- AggregateBlockingSourceOperator::pull_chunk -> convert_hash_map_to_chunk
 *                   (aggregate_blocking_source_operator.cpp:46-72, aggregator.cpp:1696-1791)
 * Functions: be/src/exprs/agg/{sum,count,avg,maxmin}.h with the nullable wrapper semantics
 * of nullable_aggregate.h (NULL inputs are skipped; result NULL when no non-null input).
 * ------------------------------------------------------------------------------------- */
typedef enum sr_agg_fn_kind {
    SR_AGG_SUM = 1,
    SR_AGG_COUNT = 2,      /* COUNT(expr): non-null inputs */
    SR_AGG_COUNT_STAR = 3, /* COUNT(*) */
    SR_AGG_AVG = 4,
    SR_AGG_MIN = 5,
    SR_AGG_MAX = 6,
    /* merge phase of AVG over (sum, count) state columns: `input` = the DOUBLE sum state, `reserved` = slot id of the
     * BIGINT count state (see sr_agg_two_phase_descs); result = total sum / total count, NULL when the count is 0 */
    SR_AGG_AVG_MERGE = 7,
    /* COUNT(DISTINCT col): `input` must be a single column reference of an integer-class type (<= 8 bytes; group keys +
     * value + null flags <= 16 bytes).  Reference: DistinctAggregateFunction / multi_distinct_count,
     * be/src/exprs/agg/distinct.h:48-300 -- a hash set per group state.  Here ONE second-level hash set keyed
     * (group keys, value) for the whole operator, folded into the group states at sink_finish.  NULL values are not
     * counted; the result is BIGINT, never NULL.  Single-phase only (sr_agg_merge / *_states / two_phase_descs and
     * the fused fragment answer SR_ERR_NOT_SUPPORTED: shuffle on the distinct column's group instead). */
    SR_AGG_COUNT_DISTINCT = 8
} sr_agg_fn_kind;

typedef struct sr_agg_fn {
    int32_t kind;       /* sr_agg_fn_kind */
    int32_t input_type; /* sr_type of the argument (decides the result type, sum.h:24-34) */
    int32_t out_slot;   /* slot id of the result column */
    int32_t reserved;   /* SR_AGG_AVG_MERGE: slot id of the count state column; otherwise 0 */
    sr_expr input; /* argument expression over the input chunk's slots (ignored for COUNT_STAR) */
} sr_agg_fn;

#define SR_MAX_GROUP_KEYS 4
#define SR_MAX_AGG_FNS 8

typedef struct sr_agg_desc {
    int32_t num_group_keys; /* 0 = no GROUP BY (single state) */
    int32_t group_slots[SR_MAX_GROUP_KEYS];
    int32_t group_types[SR_MAX_GROUP_KEYS];
    /* optional value ranges of the group-by columns (the FE passes group-by min/max statistics
     * for the compressed-key variants, aggregator.cpp:1516-1566).  has_ranges != 0 and a small
     * product of ranges selects the dense, shared-memory accumulated table. */
    int32_t has_ranges;
    int32_t group_nullable[SR_MAX_GROUP_KEYS];
    int64_t group_min[SR_MAX_GROUP_KEYS];
    int64_t group_max[SR_MAX_GROUP_KEYS];
    int32_t num_fns;
    int32_t reserved;
    sr_agg_fn fns[SR_MAX_AGG_FNS];
    /* expected number of distinct groups (0 = unknown): initial capacity of the hash table */
    int64_t expected_groups;
} sr_agg_desc;

typedef struct sr_agg sr_agg;

/* Aggregator::prepare: hash-map variant and function states from the plan node (be/src/exec/aggregator.cpp:411-570). */
sr_agg* sr_agg_create(sr_ctx* ctx, const sr_agg_desc* desc);
void sr_agg_destroy(sr_agg* agg);
/* AggregateBlockingSinkOperator::push_chunk (aggregate_blocking_sink_operator.cpp:101-138): evaluate_groupby_exprs +
 * evaluate_agg_fn_exprs + build_hash_map + compute_batch_agg_states (aggregator.cpp:1044,1376,1616,907), or
 * compute_single_agg_state (:882) without group keys. */
int32_t sr_agg_push(sr_agg* agg, const sr_chunk_view* chunk);
/* AggregateBlockingSinkOperator::set_finishing (aggregate_blocking_sink_operator.cpp:56-89): input done, the hash-map
 * iterator is positioned for the source. */
int32_t sr_agg_sink_finish(sr_agg* agg);
/* number of result rows (groups); valid after sink_finish (synchronises on a counter). */
int64_t sr_agg_num_groups(sr_agg* agg);
/* AggregateBlockingSourceOperator::pull_chunk (aggregate_blocking_source_operator.cpp:47-72) ->
 * Aggregator::convert_hash_map_to_chunk / convert_to_chunk_no_groupby (aggregator.cpp:1696-1791, 997-1042).
 * Emit up to max_rows groups starting at the handle's cursor: key columns (group_slots order)
 * then one result column per function.  out_mem selects host buffers (page-locked, owned by the handle, complete on
 * return; out->mem = SR_MEM_HOST for either host kind) or device buffers.  Returns SR_OK with out->num_rows == 0 at
 * end of stream. */
int32_t sr_agg_pull(sr_agg* agg, int64_t max_rows, int32_t out_mem, sr_chunk_out* out);
/* Operator::reset_state (be/src/exec/pipeline/operator.h:143): clear every group and state so
 * the handle can aggregate a new stream; keeps the compiled plan and the table capacity. */
int32_t sr_agg_reset(sr_agg* agg);
/* merge the (already finished) states of `other` into `agg` -- the final phase of a two-phase
 * distributed aggregate (AggregateFunction::merge, be/src/exprs/agg/aggregate.h:365-445).
 * Both handles must have been created from the same desc on the same context. */
int32_t sr_agg_merge(sr_agg* agg, sr_agg* other);

/* ---------------------------------------------------------------------------------------
 * two-phase / streaming aggregation (SURVEY.md 8f-2): AggregateStreamingSinkOperator
 * (be/src/exec/pipeline/aggregate/aggregate_streaming_sink_operator.cpp:80-372) is the FIRST phase of a distributed
 * aggregate: it pre-aggregates what it can and hands rows on in the INTERMEDIATE format (group-by columns + one state per
 * function, AggregateFunction::convert_to_serialize_format / serialize_to_column), which the second phase merges
 * (AggregateFunction::merge).  Here the intermediate format is a plain chunk:
 *      SUM -> its running sum (result type, NULL while no non-NULL input was seen)      slot out_slot
 *      COUNT / COUNT(*) -> BIGINT count                                                  slot out_slot
 *      MIN / MAX -> the value (input type, nullable)                                     slot out_slot
 *      AVG -> DOUBLE sum (slot out_slot) + BIGINT count (slot SR_AGG_STATE_SLOT(out_slot))
 * sr_agg_two_phase_descs derives, from the single-phase desc of a query, the desc of the first phase (AVG split into
 * SUM(double) + COUNT; its sr_agg_pull output IS the intermediate chunk) and of the merge phase (SUM of sums / counts,
 * MIN of MINs, SR_AGG_AVG_MERGE), whose result equals the single-phase result.  SR_ERR_NOT_SUPPORTED when a state would be
 * 128 bits wide (decimal / LARGEINT sums) or the first phase would need more than SR_MAX_AGG_FNS functions.
 * sr_agg_convert_to_states is the pass-through leg (Aggregator::output_chunk_by_streaming, aggregator.cpp:1071-1120): the
 * rows of `chunk` become intermediate rows one to one (no hash table involved); `agg` must be a first-phase handle; the
 * output columns are device buffers owned by the handle, valid until its next call.
 * The adaptive choice between the two legs (the AUTO state machine) lives in the operator:
 * starrocks_b200/host/gpu/gpu_operators.h GpuAggregateStreamingSinkOperator.
 * ------------------------------------------------------------------------------------- */
#define SR_AGG_STATE_SLOT(out_slot) ((out_slot) | 0x40000000)
int32_t sr_agg_two_phase_descs(const sr_agg_desc* desc, sr_agg_desc* phase1, sr_agg_desc* phase2);
/* groups in the table right now (before sink_finish; synchronises on a counter): what the AUTO mode compares with the rows
 * it has fed to decide whether pre-aggregation still pays (Aggregator::should_expand_preagg_hash_tables,
 * aggregator.cpp:1241-1290).  0 for dense tables and aggregates without GROUP BY (bounded: always worth keeping);
 * negative = sr_status. */
int64_t sr_agg_current_groups(sr_agg* agg);
int32_t sr_agg_convert_to_states(sr_agg* agg, const sr_chunk_view* chunk, sr_chunk_out* out);
/* SELECTIVE_PREAGG leg (AggregateStreamingSinkOperator::_push_chunk_by_selective_preaggregation,
 * aggregate_streaming_sink_operator.cpp:173-210: build_hash_map_with_selection, compute_batch_agg_states_with_selection,
 * output_chunk_by_streaming_with_selection): rows whose group is already in the table are aggregated into it; the others
 * create no group and come back in `out` as intermediate rows (the format of sr_agg_convert_to_states), in input order.
 * `out` is owned by the aggregate (valid until its next call).  A hash-table aggregate refuses a batch of 0x7FFFFFF0 rows
 * or more with SR_ERR_NOT_SUPPORTED once the chunk is staged, before the conversion to intermediate rows allocates or
 * launches anything. */
int32_t sr_agg_push_selective(sr_agg* agg, const sr_chunk_view* chunk, sr_chunk_out* out);

/* Element-wise mergeable view of a DENSE aggregate table (group-by columns with declared ranges, or no
 * GROUP BY): one array per state component, every array indexed by the same slot number on every
 * instance created from the same desc.  Partial states of fragment instances on several GPUs are then
 * merged IN PLACE by an all-reduce per array (reduce = SR_STATE_SUM / MIN / MAX over int64 or double
 * elements) -- SURVEY.md 8e "ncclAllReduce on a dense slot array when the group domain is tiny and
 * enumerable" -- instead of the gather + sr_agg_merge exchange; afterwards every instance holds the
 * final state and any of them can be pulled.  Call between the last push and the first pull.  The arrays
 * are written by work queued on the context's stream: run the collective on that stream (or sr_ctx_sync
 * first).  All instances must have been fed the same chunk schema (same column nullability), so that they
 * expose the same list of arrays.  SR_ERR_NOT_SUPPORTED for hash tables and for 128-bit sums (carry is not
 * element-wise). */
typedef enum sr_state_reduce { SR_STATE_SUM = 0, SR_STATE_MIN = 1, SR_STATE_MAX = 2 } sr_state_reduce;
typedef struct sr_agg_state_array {
    void* data;        /* device pointer */
    int64_t count;     /* elements */
    int32_t elem_type; /* SR_TYPE_BIGINT or SR_TYPE_DOUBLE */
    int32_t reduce;    /* sr_state_reduce */
} sr_agg_state_array;
#define SR_MAX_STATE_ARRAYS (1 + 3 * SR_MAX_AGG_FNS)
int32_t sr_agg_dense_state(sr_agg* agg, sr_agg_state_array* arrays, int32_t max_arrays, int32_t* num_arrays);

/* ---------------------------------------------------------------------------------------
 * fused pipeline fragment:  scan -> filter -> [hash-join probe]* -> hash aggregate in ONE
 * pass over the fact columns (no intermediate Chunk materialisation).  This is what the GPU
 * ScanOperator runs when the downstream operators of its pipeline are GPU join probes and a
 * GPU aggregate sink (SURVEY.md section 7 "keep the API, change the cadence").
 * The joins must be built (sr_join_build_finish) INNER, LEFT_SEMI, LEFT_ANTI or LEFT_OUTER joins
 * on one key column; only INNER and LEFT_SEMI joins may carry an other-join conjunct.  Otherwise
 * SR_ERR_NOT_SUPPORTED is returned and the caller runs the per-operator path.
 * An other-join conjunct computes what sr_join_probe does with it (NULL counts as false): an INNER
 * join emits a combination only when the conjunct is TRUE for it, a LEFT_SEMI join passes a row
 * once when the conjunct is TRUE for some build row with its key.  It may read fact columns and
 * any column of its own join's build chunks (not only payloads), resolved fact first; over a build
 * side that never received a chunk a build column's type comes from build_out_types
 * (SR_ERR_STATE when it is not declared), and such a join passes nothing.  The first push refuses,
 * before any launch: a slot that is a column of another fragment join -- its payload, a column its
 * conjunct reads, or any column of its build chunks, so two conjuncts may not read one slot id
 * from their own build sides -- (SR_ERR_NOT_SUPPORTED); a slot on neither side or a double-valued
 * conjunct (SR_ERR_INVALID_ARGUMENT); more than SR_MAX_VALUES distinct columns in the fragment
 * (SR_ERR_NOT_SUPPORTED).  A conjunct always runs the selection-vector passes (mode_hint 1 then
 * runs mode 2), and its final pass evaluates it (k_frag_gather_agg) one thread per surviving row;
 * rows_passed counts the combinations that pass it.
 * Speed: fuse a conjunct join that most rows never reach (measured on an H100: the TPC-DS Q94
 * body's LEFT SEMI self join, 2.5-2.8 ms fused against 8.9-12.1 ms per operator).  Keep per
 * operator an expanding INNER conjunct join with long chains that most rows reach (the Q95
 * ws_wh self join, 15.7 entries per chain, every row surviving: 1023 ms fused against 176 ms):
 * the final pass walks each row's chain serially, and the per-operator probe is faster there.  Duplicate build keys are allowed (INNER and
 * LEFT_OUTER joins emit one combination per matching build row).  Payloads are allowed on INNER
 * and LEFT_OUTER joins only (SR_ERR_INVALID_ARGUMENT otherwise); a LEFT_OUTER payload is
 * nullable for the aggregate: a probe row without a build row reads NULL.  A build side that
 * never received a chunk takes a payload's type from sr_join_desc.build_out_types, as
 * sr_join_probe does, and reads it as NULL (SR_ERR_STATE when the type is not declared).
 * LEFT_ANTI is not null-aware: a row passes when its key is NULL or no build row has it.
 * ------------------------------------------------------------------------------------- */
#define SR_MAX_FRAG_JOINS 6
#define SR_MAX_FRAG_PAYLOAD 2

typedef struct sr_frag_join {
    sr_join* join;          /* built table (shared, not owned) */
    int32_t probe_key_slot; /* fact column holding the probe key */
    int32_t num_payload;    /* build columns carried downstream (<= SR_MAX_FRAG_PAYLOAD) */
    int32_t payload_build_slots[SR_MAX_FRAG_PAYLOAD];
} sr_frag_join;

typedef struct sr_fragment_desc {
    sr_scan_desc scan; /* preds / filter_exprs on fact columns; out_slots ignored.  They name fact slots only: one that
                        * names a join's payload slot makes the first sr_fragment_push fail with SR_ERR_NOT_SUPPORTED */
    int32_t num_joins;
    /* execution mode: 0 = decide from the pass rates sampled on the first batch, 1 = single fused kernel
     * (warp-queue cascade), 2 = selection-vector passes (stream -> gather -> aggregate).  Both modes give
     * identical results; the knob exists for tests and experiments.  A one-to-many INNER / LEFT_OUTER join or an
     * other-join conjunct always runs mode 2, whatever the hint. */
    int32_t mode_hint;
    sr_frag_join joins[SR_MAX_FRAG_JOINS]; /* hint order; the fragment reorders by measured pass rate */
    sr_agg_desc agg; /* group keys / fn inputs may reference fact slots and payload slots */
} sr_fragment_desc;

typedef struct sr_fragment sr_fragment;

sr_fragment* sr_fragment_create(sr_ctx* ctx, const sr_fragment_desc* desc);
void sr_fragment_destroy(sr_fragment* frag);
/* what PipelineDriver::process (pipeline_driver.cpp:270-500) does for one morsel of the probe-side pipeline: scan filter,
 * every HashJoinProbeOperator in turn, AggregateBlockingSinkOperator::push_chunk -- with no chunk materialised in between.
 * consume one batch of fact rows (one morsel: any number of rows). */
int32_t sr_fragment_push(sr_fragment* frag, const sr_chunk_view* fact);
/* The rows of chunks[0], chunks[1], ... in that order, pushed as one batch: same result, rows_passed and plan as
 * sr_fragment_push of their concatenation -- the form a scan that hands out chunks of at most chunk_size rows, each in
 * its own column buffers, pushes without first copying them into one batch on the host.
 *  - Every chunk carries the same set of (slot_id, type); the column order may differ.  Each chunk's own `mem` is
 *    honoured: SR_MEM_DEVICE and SR_MEM_HOST_PINNED columns are gathered into one device batch by one kernel launch
 *    (pinned columns are read over PCIe, in full); SR_MEM_HOST columns are copied H2D straight to their place in that
 *    batch, which is correct but slow: one small copy per chunk column.  Only the slots the fragment reads are moved.
 *  - A column is nullable in the batch when any chunk of the call has nulls != NULL for it; the chunks without a null
 *    column contribute zeros.  When no chunk has one, the batch column has none either, so the NOT NULL kernel paths
 *    stay eligible exactly as for a contiguous push.
 *  - Refused with SR_ERR_INVALID_ARGUMENT before any allocation, copy or launch: num_chunks < 0, chunks == NULL with
 *    num_chunks > 0, an unknown mem kind, chunks of different schemas, negative rows, data == NULL with rows > 0, a device
 *    or pinned column that is not naturally aligned (see sr_col_view), pinned memory that is not page-locked and mapped.
 *    A total of 0xFFFFFFF0 rows or more: SR_ERR_NOT_SUPPORTED, before any column is looked at.
 *  - Zero chunks, or only empty ones, behave like a zero-row sr_fragment_push (the first push still plans).
 *  - sr_mem rules 2 and 4: the call only queues work; pinned and device chunk buffers must stay valid and unchanged until
 *    an event recorded after the call has completed, or until the next synchronising call. */
int32_t sr_fragment_push_chunks(sr_fragment* frag, const sr_chunk_view* chunks, int32_t num_chunks);
/* the aggregate the fragment feeds (owned by the fragment): finish / pull / merge through
 * the sr_agg_* calls. */
sr_agg* sr_fragment_agg(sr_fragment* frag);
/* the plan the fragment chose on its first batch: probe order (indexes into desc->joins), the
 * pass rate each join measured on the sample, shared memory per CTA and the persistent grid. */
typedef struct sr_fragment_plan {
    int32_t num_joins;
    int32_t order[SR_MAX_FRAG_JOINS];
    int32_t bitmap_in_smem[SR_MAX_FRAG_JOINS]; /* per probe position */
    double pass_rate[SR_MAX_FRAG_JOINS];       /* per desc->joins index */
    int32_t smem_bytes;
    int32_t grid;
    int32_t block;
    int32_t agg_in_smem;
    int32_t mode;             /* 1 = fused cascade kernel, 2 = selection-vector passes */
    int32_t num_stream_joins; /* mode 2: joins tested by the streaming pass */
    int32_t num_gather_passes;
    int32_t final_pass; /* mode 2: the final pass of the last push, SR_FINAL_PASS_* */
    double pred_rate; /* fraction of sampled rows passing the scan conjuncts */
} sr_fragment_plan;
#define SR_FINAL_PASS_NONE 0    /* no push yet, or the fused cascade kernel */
#define SR_FINAL_PASS_GENERIC 1 /* k_frag_gather_agg<EXPAND = false>: any join, aggregate and expression */
#define SR_FINAL_PASS_EXPAND 2  /* k_frag_gather_agg<EXPAND = true>: one-to-many joins */
#define SR_FINAL_PASS_DENSE 3   /* k_frag_final_dense: slot-digit directories, batched rows, dense shared-memory aggregate */
int32_t sr_fragment_get_plan(sr_fragment* frag, sr_fragment_plan* plan);
/* device time of the passes of the LAST push in selection-vector mode (CUDA events on the context's
 * stream; synchronises): ms[0] = streaming pass, ms[1] = gather-join passes, ms[2] = final pass.
 * Returns SR_ERR_STATE when the last push did not run in that mode. */
int32_t sr_fragment_last_pass_ms(sr_fragment* frag, float ms[3]);
/* reset_state for the whole fragment: clears its aggregate and the rows_passed counter. */
int32_t sr_fragment_reset(sr_fragment* frag);
/* rows that survived scan predicates and all joins so far (synchronises). */
int64_t sr_fragment_rows_passed(sr_fragment* frag);

/* ---------------------------------------------------------------------------------------
 * exchange: hash-partition a chunk's rows to `num_channels` destinations.
 * Replaces ExchangeSinkOperator::push_chunk's hash + shuffle + row-index counting sort
 * (be/src/exec/pipeline/exchange/exchange_sink_operator.cpp:586-637), Shuffler::
 * exchange_shuffle (shuffler.h:72-89) and Column::fnv_hash / crc32_hash
 * (be/src/column/column_hash/column_hash.cpp:138-300, base/hash/hash_util.hpp:127-134,
 * 242-244).  The transport itself (NCCL all-to-all in place of brpc transmit_chunk) is
 * driven by the host with the per-channel counts this call produces.
 * ------------------------------------------------------------------------------------- */
/* SR_HASH_XXH3: the exchange hash of exchange_hash_function_version = 1 (exchange_sink_operator.cpp:597-601): every
 * partition column feeds XXH3_64bits_withSeed(value bytes, width, seed = the row's 32-bit hash so far) truncated to 32 bits,
 * starting from HashUtil::XXH3_SEED_32 (ColumnHashVisitor<XXHash3>, column_hash.cpp:64-68). */
typedef enum sr_hash_fn { SR_HASH_FNV = 0, SR_HASH_CRC32 = 1, SR_HASH_XXH3 = 2 } sr_hash_fn;
typedef enum sr_reduce_op { SR_REDUCE_MULHI = 0 /* ReduceOp */, SR_REDUCE_MODULO = 1 /* ModuloOp */ } sr_reduce_op;

#define SR_MAX_PART_KEYS 4

typedef struct sr_part_desc {
    int32_t hash_fn;   /* sr_hash_fn: FNV (or XXH3, hash function version 1) for HASH_PARTITIONED, CRC32 for BUCKET_SHUFFLE */
    int32_t reduce_op; /* sr_reduce_op */
    int32_t num_channels;
    int32_t num_part_slots;
    int32_t part_slots[SR_MAX_PART_KEYS];
} sr_part_desc;

typedef struct sr_xchg sr_xchg;

/* ExchangeSinkOperator::prepare with the partition exprs of the TDataStreamSink (exchange_sink_operator.cpp:395-483). */
sr_xchg* sr_xchg_create(sr_ctx* ctx, const sr_part_desc* desc);
void sr_xchg_destroy(sr_xchg* x);
/* ExchangeSinkOperator::push_chunk, the HASH_PARTITIONED / BUCKET_SHUFFLE branch (exchange_sink_operator.cpp:586-637):
 * hash of the partition columns, Shuffler::exchange_shuffle (shuffler.h:72-89), per-channel row index lists.
 * Partition one batch.  out: DEVICE buffers, all columns of `in` reordered so that the rows
 * of channel c occupy [offsets[c], offsets[c+1]) in input order (stable, like the reference's
 * counting sort).  channel_offsets_host: num_channels + 1 int64 written on return (syncs).  A batch of zero rows gives
 * zero-row columns whose `data` may be NULL; a nullable input column still gets a non-NULL (empty) `nulls`, so every
 * batch's output, and every channel's ChunkPB, has the same null columns. */
int32_t sr_xchg_partition(sr_xchg* x, const sr_chunk_view* in, sr_chunk_out* out, int64_t* channel_offsets_host);
/* hash values + channel ids only (arrays of num_rows uint32 in `mem`; sr_mem rules: host arrays are complete on return). */
int32_t sr_xchg_hash(sr_xchg* x, const sr_chunk_view* in, uint32_t* hash_values, uint32_t* channel_ids, int32_t mem);

/* ---------------------------------------------------------------------------------------
 * Segment data pages decoded on the device (SURVEY.md 8f-4) -- the column a scan would otherwise get from the CPU page
 * decoders.  Replaces, for 4- and 8-byte integer-class columns (INT, BIGINT, DATE, DATETIME, DECIMAL32/64):
 *   FrameOfReferencePageDecoder::next_batch  be/src/storage/rowset/frame_of_reference_page.h:113-222
 *       (ForDecoder, be/src/util/frame_of_reference_coding.cpp:246-352)
 *   PlainPageDecoder::next_batch             be/src/storage/rowset/plain_page.h:135-260
 * and, for every fixed-width type (widths 1, 2, 4, 8 and 16: BOOLEAN ... LARGEINT, FLOAT, DOUBLE, DECIMAL128 -- the decode
 * moves bytes and does no arithmetic), the default encoding of those columns:
 *   BitShufflePageDecoder::next_batch        be/src/storage/rowset/bitshuffle_page.h (bitshuffle + LZ4 blocks)
 * For every encoding `out` must be aligned to the value width (8 bytes for 16-byte values), as any device column is
 * (sr_col_view): SR_ERR_INVALID_ARGUMENT before anything is copied or launched otherwise.
 * `pages`: the BODIES of consecutive data pages of one column (after the page's checksum handling of page_io.cpp, without
 * the null map a nullable column's page ends with: sr_null_maps_decode), all in `mem`: SR_MEM_DEVICE, SR_MEM_HOST_PINNED (page-locked mapped memory, e.g. a registered page cache:
 * read in place over PCIe, the decode is the transfer) or SR_MEM_HOST (pageable: staged page by page).  The values of page
 * k follow those of page k - 1 in `out` (device memory, room for out_capacity values); *out_rows receives the total.
 * And, for TYPE_INT only, the data pages of a dictionary-encoded (DICT_ENCODING: CHAR / VARCHAR) column, decoded
 * straight into ids -- the low-cardinality global dictionary's scan step (GlobalDictCodeColumnIterator):
 *   BinaryDictPageDecoder::next_batch        be/src/storage/rowset/binary_dict_page.{h,cpp}
 *   A data page is a 4-byte little-endian mode word (EncodingTypePB) and, with mode 5 (DICT_ENCODING), a BIT_SHUFFLE page
 *   of int32 codes.  Code k is stored as values[k] of the last sr_page_decoder_set_dict (SR_ERR_STATE when there is
 *   none); a code >= num_words is a corrupt page.  Mode 2 (PLAIN_ENCODING: the dictionary overflowed and the column
 *   fell back to plain string pages) gives SR_ERR_NOT_SUPPORTED when no page of the call is malformed.
 * SR_ERR_INVALID_ARGUMENT for a page that is not well formed (sizes, frame table, bit widths, the bitshuffle header, block
 * chain or LZ4 streams, the dictionary mode word or codes).  Asynchronous on the context stream except for one small
 * read-back of the per-page counts and, for FOR, BIT_SHUFFLE, DICT and RLE, one of the error flag at the end.
 * And, for BOOLEAN only, RLE pages (the default encoding of BOOLEAN columns):
 *   RlePageDecoder::next_batch               be/src/storage/rowset/rle_page.h (RlePageBuilder::finish writes the page)
 *   A page is a little-endian uint32 value count, then an RleEncoder stream (be/src/util/rle_encoding.h) at bit width 1:
 *   runs, each a ULEB128 header of at most 5 bytes h -- h & 1: (h >> 1) groups of 8 bit-packed values, one byte each, least
 *   significant bit first; else (h >> 1) copies of the value in the next byte.  The decode stops at the count: values
 *   and bytes past it are never read.  A header longer than 5 bytes or cut off, a run of length 0, a repeated value other
 *   than 0 / 1, values up to the count past the page's end, or a stream that ends before the count is a malformed page.
 * Other types with SR_PAGE_RLE, and plain-mode string pages, are not covered: SR_ERR_NOT_SUPPORTED. */
typedef enum sr_page_encoding {
    SR_PAGE_PLAIN = 0,      /* EncodingTypePB::PLAIN_ENCODING */
    SR_PAGE_FOR = 1,        /* EncodingTypePB::FOR_ENCODING */
    SR_PAGE_BITSHUFFLE = 2, /* EncodingTypePB::BIT_SHUFFLE */
    SR_PAGE_DICT = 3,       /* EncodingTypePB::DICT_ENCODING */
    SR_PAGE_RLE = 4         /* EncodingTypePB::RLE (SR_TYPE_BOOLEAN) */
} sr_page_encoding;

typedef struct sr_page_view {
    const void* data;
    int64_t size;
} sr_page_view;

typedef struct sr_page_decoder sr_page_decoder;
sr_page_decoder* sr_page_decoder_create(sr_ctx* ctx);
void sr_page_decoder_destroy(sr_page_decoder* dec);
int32_t sr_pages_decode(sr_page_decoder* dec, int32_t encoding, int32_t type, const sr_page_view* pages, int32_t num_pages, int32_t mem, void* out,
                        int64_t out_capacity, int64_t* out_rows);
/* The code -> value table of SR_PAGE_DICT pages (BinaryDictPageDecoder::set_dict_decoder): values[k] is what code k
 * decodes to -- for a low-cardinality column, the segment's local -> global id table (the global id of word k of the
 * segment's dictionary page, 0 for an empty word the global dictionary lacks: build_code_convert_map).  `values` (num_words
 * int32 in `mem`: SR_MEM_HOST, SR_MEM_HOST_PINNED or SR_MEM_DEVICE) is copied into the decoder; the caller may free it
 * when the call returns (it synchronises the context stream).  A later call replaces the table: one table per segment, so
 * a caller decoding several segments into one column sets each segment's table and advances `out`. */
int32_t sr_page_decoder_set_dict(sr_page_decoder* dec, const int32_t* values, int64_t num_words, int32_t mem);

/* The null maps of a nullable column's data pages (page format 2: a page stores a value for every row, NULL rows included,
 * and its body is `values | null map`, DataPageFooterPB.nullmap_size giving the map's length) decoded on the device into
 * the uint8 null column (1 = NULL) that goes with the values sr_pages_decode makes of the same pages:
 *   ParsedPage / PageDecoder null handling   be/src/storage/rowset/parsed_page.cpp, page_io.cpp
 * One view per data page, in page order: the map's bytes and the page's num_values (footer).  size == 0: the page holds
 * no NULL (the writer omits the map) and its rows get 0.  Page k's flags follow page k - 1's in out_nulls (device memory,
 * room for out_capacity flags, any alignment), as sr_pages_decode places the values.
 *   SR_NULL_BITSHUFFLE (NullEncodingPB::BITSHUFFLE_NULL): bitshuffle::compress_lz4 of the flags zero-padded to
 *     ALIGN_UP(num_rows, 8), 1-byte elements -- the block chain of a BIT_SHUFFLE page without its 16-byte header, ending
 *     exactly at `size`.
 *   SR_NULL_RLE (NullEncodingPB::RLE_NULL): the RleEncoder stream at bit width 1 described at SR_PAGE_RLE, num_rows values.
 * *out_rows: the rows of all pages; *out_null_count: the nonzero flags among them -- 0 lets the caller pass the batch with
 * nulls = NULL (sr_col_view), which keeps the scan and fragment kernels on their paths for columns without NULLs.
 * SR_ERR_NOT_SUPPORTED for another encoding; SR_ERR_INVALID_ARGUMENT for a negative size or row count, a row count past
 * 2^32 - 1, missing data or more rows than out_capacity (before anything is copied or launched), and for a malformed map
 * (after the read-back; nothing is written past the pages' rows).  Asynchronous on the context stream except for that one
 * read-back of the error flag and the count. */
typedef enum sr_null_encoding {
    SR_NULL_BITSHUFFLE = 0, /* NullEncodingPB::BITSHUFFLE_NULL */
    SR_NULL_RLE = 1         /* NullEncodingPB::RLE_NULL */
} sr_null_encoding;

typedef struct sr_null_map_view {
    const void* data; /* the map's bytes in `mem` (sr_pages_decode's memory kinds) */
    int64_t size;     /* DataPageFooterPB.nullmap_size; 0: no NULL in the page */
    int64_t num_rows; /* the page's num_values */
} sr_null_map_view;

int32_t sr_null_maps_decode(sr_page_decoder* dec, int32_t null_encoding, const sr_null_map_view* maps, int32_t num_pages, int32_t mem, uint8_t* out_nulls,
                            int64_t out_capacity, int64_t* out_rows, int64_t* out_null_count);

/* ---------------------------------------------------------------------------------------
 * exchange wire format (SURVEY.md 8f-3): the bytes of ChunkPB.data as ProtobufChunkSerde::serialize_without_meta writes
 * them (be/src/serde/protobuf_serde.cpp:88-140) with encode level 0 and no compression:
 *      fixed32 version = 1 | fixed32 num_rows | columns in chunk order
 *      FixedLengthColumn<T>:  fixed32 byte size | raw little-endian values      (column_array_serde.cpp:214-255)
 *      NullableColumn:        the null column (a uint8 FixedLengthColumn) | the data column          (:759-782)
 * so a channel slice produced by sr_xchg_partition can be handed to the unchanged brpc sender (ExchangeSinkOperator::
 * Channel::send_one_chunk, exchange_sink_operator.cpp) and a ChunkPB received from a CPU BE can be consumed on the device.
 * The protobuf envelope itself (slot_id_map, is_nulls, is_consts, serialized_size, uncompressed_size, compress_type) stays
 * host code; sr_chunk_pb_meta carries what it needs.  Fixed-length and nullable fixed-length columns; the integer
 * (streamvbyte) encodings of encode_level > 0 and var-length columns are not produced.
 * ------------------------------------------------------------------------------------- */
typedef struct sr_chunk_pb_meta {
    int64_t serialized_size; /* bytes of ChunkPB.data = ChunkPB.serialized_size = uncompressed_size (no padding at level 0) */
    int64_t num_rows;
    int32_t num_cols;
    int32_t reserved;
    int32_t slot_ids[SR_MAX_OUT_COLS];  /* slot_id_map: slot id -> column index, in column order */
    int32_t types[SR_MAX_OUT_COLS];     /* sr_type of every column (the receiver knows it from its RowDescriptor) */
    uint8_t is_nulls[SR_MAX_OUT_COLS];  /* ChunkPB.is_nulls */
    uint8_t is_consts[SR_MAX_OUT_COLS]; /* ChunkPB.is_consts: always 0 here */
} sr_chunk_pb_meta;
/* bytes rows [row_begin, row_end) of `chunk` serialize to */
int64_t sr_chunk_serialized_size(const sr_chunk_view* chunk, int64_t row_begin, int64_t row_end);
/* Serialize rows [row_begin, row_end) of `chunk` (host or device columns) into dst (dst_mem: host memory -- a page-locked
 * buffer makes it one DMA per column -- or SR_MEM_DEVICE); dst_capacity >= sr_chunk_serialized_size.  Queued on the context's
 * stream; synchronises when dst is host memory. */
int32_t sr_chunk_serialize(sr_ctx* ctx, const sr_chunk_view* chunk, int64_t row_begin, int64_t row_end, void* dst, int64_t dst_capacity,
                           int32_t dst_mem, sr_chunk_pb_meta* meta);
/* Parse ChunkPB.data (src in src_mem) described by `meta` (num_cols, slot_ids, types, is_nulls) into device columns owned by
 * `handle` (valid until its next deserialize / destroy); checks version, sizes and bounds like the reference's
 * deserialize (SR_ERR_INVALID_ARGUMENT on a malformed payload).  The payload must be exactly the columns `meta` describes:
 * bytes == meta->serialized_size, header num_rows == meta->num_rows and no bytes after the last column, else
 * SR_ERR_INVALID_ARGUMENT.  A const column (meta->is_consts[k] != 0) gives SR_ERR_NOT_SUPPORTED.  A refused payload
 * leaves no copy queued. */
typedef struct sr_serde sr_serde;
sr_serde* sr_serde_create(sr_ctx* ctx);
void sr_serde_destroy(sr_serde* handle);
int32_t sr_chunk_deserialize(sr_serde* handle, const void* src, int64_t bytes, int32_t src_mem, const sr_chunk_pb_meta* meta, sr_chunk_out* out);

/* ---------------------------------------------------------------------------------------
 * K11: Column::append_selective gather (be/src/column/fixed_length_column_base.cpp:54):
 * dst[j] = src[index[j]] for one column; all pointers in `mem` (SR_MEM_DEVICE only) and naturally aligned (see
 * sr_col_view), else SR_ERR_INVALID_ARGUMENT.
 * ------------------------------------------------------------------------------------- */
int32_t sr_gather(sr_ctx* ctx, const void* src, int32_t type, const uint32_t* index, int64_t n, void* dst,
                  int32_t mem);

/* sizeof() of the ABI structs as compiled into the library, so a foreign-language binding can
 * verify its own struct layouts at load time.  which: 0 sr_col_view, 1 sr_chunk_view,
 * 2 sr_chunk_out, 3 sr_pred, 4 sr_expr, 5 sr_scan_desc, 6 sr_join_desc, 7 sr_join_info,
 * 8 sr_agg_fn, 9 sr_agg_desc, 10 sr_frag_join, 11 sr_fragment_desc, 12 sr_part_desc, 13 sr_agg_state_array,
 * 14 sr_fragment_plan, 15 sr_rf_info, 16 sr_null_map_view.
 * returns -1 for an unknown index. */
int32_t sr_abi_sizeof(int32_t which);

/* plumbing aid: synchronous copy on the context's stream. kind: 0 = host->device,
 * 1 = device->host, 2 = device->device.  Lets hosts without a CUDA runtime binding of their
 * own (the ctypes tests, a JNI shim) read the device buffers handed back in sr_chunk_out. */
int32_t sr_memcpy(sr_ctx* ctx, void* dst, const void* src, int64_t bytes, int32_t kind);

/* ---------------------------------------------------------------------------------------
 * plumbing for asynchronous adapters.  Operator::push_chunk must not block (be/src/exec/pipeline/operator.h:100-118: the
 * driver polls need_input / has_output / pending_finish instead), so an adapter hands a batch of page-locked columns to
 * the library, records an event behind the work it queued and re-uses the batch only once the event has completed.
 *   sr_host_alloc / sr_host_free: page-locked, device-mapped host memory (what a cudaHostRegister-ed ColumnAllocator
 *     pool would provide, be/src/common/memory/column_allocator.h:23-54); valid as SR_MEM_HOST_PINNED columns.
 *   sr_event_*: a marker on the context's stream.  record: after everything queued so far; query: 1 = reached,
 *     0 = still pending (never blocks), < 0 = sr_status; sync: block until reached.
 * ------------------------------------------------------------------------------------- */
int32_t sr_host_alloc(sr_ctx* ctx, int64_t bytes, void** ptr);
int32_t sr_host_free(sr_ctx* ctx, void* ptr);
/* Page-lock and map caller memory (cudaHostRegister, mapped | portable): the hook for a pinned ColumnAllocator pool,
 * whose buffers are then valid as SR_MEM_HOST_PINNED columns.  Refused (SR_ERR_INVALID_ARGUMENT): bytes <= 0, a range
 * overlapping one already registered or allocated by sr_host_alloc.  sr_host_unregister takes the pointer passed to
 * sr_host_register and refuses any other; the GPU must no longer read the range (sync or an event first). */
int32_t sr_host_register(sr_ctx* ctx, void* ptr, int64_t bytes);
int32_t sr_host_unregister(sr_ctx* ctx, void* ptr);
/* 1 if [ptr, ptr + bytes) lies inside one range from sr_host_alloc or sr_host_register, 0 if not.  A host lookup in the
 * library's registry (process-wide, like the portable allocations it records): no driver call, no context lock. */
int32_t sr_host_is_mapped(sr_ctx* ctx, const void* ptr, int64_t bytes);
typedef struct sr_event sr_event;
sr_event* sr_event_create(sr_ctx* ctx);
void sr_event_destroy(sr_event* ev);
int32_t sr_event_record(sr_event* ev);
int32_t sr_event_query(sr_event* ev);
int32_t sr_event_sync(sr_event* ev);

/* measurement aid: read-only 128-bit-load bandwidth kernel over `bytes` of device memory
 * (SURVEY.md section 8d "measure the achievable peak"); returns the xor checksum through
 * *checksum_host after syncing. */
int32_t sr_bandwidth_probe(sr_ctx* ctx, const void* dev_ptr, int64_t bytes, uint64_t* checksum_host);
/* write `bytes` of zeros to a scratch buffer larger than L2 (flushes L2 between timed steps) */
int32_t sr_flush_l2(sr_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* SR_GPU_OPS_H */
