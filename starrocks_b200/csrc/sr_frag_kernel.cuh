// sr_frag_kernel.cuh -- device code of the fused fragment (see sr_frag.cuh for the design notes).
#pragma once

#include "sr_agg.cuh"

namespace srd {

struct FragJoinDev {
    JoinDev j;
    int32_t key_value_id;
    int32_t smem_off; // word offset of the bitmap copy in dynamic shared memory, -1 = global
    int32_t bitmap_words;
    int32_t use_bitmap; // range-mapped table: test the bitmap; otherwise probe the hash table
    int32_t need_head;  // a payload column of this join is read downstream
    int32_t idx32;      // bitmap join whose [min, max] fits int32: 32-bit index arithmetic is exact
    int32_t expand;     // INNER / LEFT OUTER join whose build side has duplicate keys: a probe row is emitted once per chain entry
    int32_t kind;       // FRAG_FILTER, FRAG_ANTI or FRAG_OUTER
};

// What a fragment join does to a probe row.  FILTER (INNER, LEFT SEMI): the row passes when a build row has its key (a
// NULL key never matches).  ANTI (LEFT ANTI): the inverted test -- the row passes when its key is NULL or no build row
// has it.  OUTER (LEFT OUTER): never drops a row; a row without a build row reads NULL payloads (build row 0, the
// sentinel).  Outer joins are placed after every filtering join and are only ever looked up, in a final pass.
constexpr int32_t FRAG_FILTER = 0;
constexpr int32_t FRAG_ANTI = 1;
constexpr int32_t FRAG_OUTER = 2;

// whether a tested row passes a filtering or anti join: `nul` its key is NULL, `hit` a build row has the key
__device__ __forceinline__ bool frag_join_pass(int32_t kind, bool nul, bool hit) {
    return kind == FRAG_ANTI ? (nul || !hit) : (!nul && hit);
}

struct FragDev {
    int32_t num_preds, num_exprs, num_joins;
    // the second join's key column is streamed together with the first one (its sectors would
    // nearly all be fetched anyway) and travels through queue 0 with the row id
    int32_t eager1;
    int32_t num_filter_joins; // joins [0, num_filter_joins) filter (FILTER / ANTI), the outer joins follow them
    int32_t pad;
    CPred preds[8];
    CExpr exprs[4];
    FragJoinDev joins[SR_MAX_FRAG_JOINS];
    unsigned long long* rows_passed;
    // other-join conjuncts of INNER / LEFT SEMI joins, by probe position: bit j of conj_mask says conj[j] is join j's.  Only
    // the final pass reads them (k_frag_gather_agg<..., CONJ = true>)
    int32_t conj_mask;
    int32_t pad2;
    CExpr conj[SR_MAX_FRAG_JOINS];
};

// k_frag_sample's counters: [j] rows passing join j, [SAMPLE_ALL_PREDS] rows passing every scan conjunct,
// [SAMPLE_PREDS_UPTO + p] rows passing conjuncts 0..p
constexpr int SAMPLE_ALL_PREDS = SR_MAX_FRAG_JOINS;
constexpr int SAMPLE_PREDS_UPTO = 16;
constexpr int SAMPLE_COUNTERS = SAMPLE_PREDS_UPTO + 8;
static_assert(SAMPLE_ALL_PREDS < SAMPLE_PREDS_UPTO, "sample counter layout");

// kernel prologues: copy `count` descriptors into shared memory, block-cooperatively (the caller synchronises)
template <typename T>
__device__ __forceinline__ void smem_copy(T* dst, const T* src, int count) {
    for (int i = threadIdx.x; i < (int)(sizeof(T) / 4) * count; i += blockDim.x) ((uint32_t*)dst)[i] = ((const uint32_t*)src)[i];
}

// copy the bitmaps of joins [0, nj) that the plan put in shared memory (smem_off >= 0); GUARD: plus one zero word behind
// each copy (stream_test_reg clamps an out-of-range key onto it)
template <bool GUARD>
__device__ __forceinline__ void smem_stage_bitmaps(uint32_t* smem, const FragJoinDev* joins, int nj) {
    for (int j = 0; j < nj; j++) {
        const FragJoinDev& fj = joins[j];
        if (fj.smem_off < 0) continue;
        if (GUARD)
            for (int w = threadIdx.x; w <= fj.bitmap_words; w += blockDim.x) smem[fj.smem_off + w] = w < fj.bitmap_words ? fj.j.bitmap[w] : 0u;
        else
            for (int w = threadIdx.x; w < fj.bitmap_words; w += blockDim.x) smem[fj.smem_off + w] = fj.j.bitmap[w];
    }
}

// the tile shape of the cascade (k_fragment) and of the streaming passes (k_frag_stream, k_frag_stream_tests)
constexpr int FRAG_BLOCK = 512;
constexpr int FRAG_WARPS = FRAG_BLOCK / 32;
constexpr int FRAG_ROWS = 4;   // consecutive rows per thread and group (one 128-bit load of an int32 column)
constexpr int FRAG_GROUPS = 2; // independent groups per thread and tile (memory-level parallelism)
constexpr int FRAG_TILE = FRAG_BLOCK * FRAG_ROWS * FRAG_GROUPS;

// the first row of each of the calling thread's groups in `tile`, and which of their rows lie below n
__device__ __forceinline__ void frag_tile_rows(int64_t tile, int64_t n, int64_t (&row0)[FRAG_GROUPS], uint32_t (&alive)[FRAG_GROUPS]) {
#pragma unroll
    for (int g = 0; g < FRAG_GROUPS; g++) {
        row0[g] = tile * FRAG_TILE + (int64_t)g * (FRAG_BLOCK * FRAG_ROWS) + (int64_t)threadIdx.x * FRAG_ROWS;
        alive[g] = 0;
#pragma unroll
        for (int r = 0; r < FRAG_ROWS; r++)
            if (row0[g] + r < n) alive[g] |= 1u << r;
    }
}

constexpr int FRAG_QCAP = 64; // queue capacity per warp and stage: < 32 pending + <= 32 appended
// dynamic shared memory per warp for the cascade: SR_MAX_FRAG_JOINS row queues, the key lane of
// queue 0, and the fill counts
constexpr int FRAG_WARP_QWORDS = (SR_MAX_FRAG_JOINS + 1) * FRAG_QCAP + 8;

struct FragLoader {
    const VTab& vt;
    int64_t row;
    uint32_t bidx[SR_MAX_FRAG_JOINS];
    // optional: one fact value that travelled with the row id in the selection vector (the key of a streamed join
    // whose build row the final pass looks up) -- saves the final pass one random sector read per row
    int32_t carry_id;  // value id, -1 = none
    int32_t carry_val; // non-NULL by construction: the row passed that join
    __device__ __forceinline__ bool load(int id, int64_t& bits) const {
        if (id == carry_id) {
            bits = (int64_t)carry_val;
            return false;
        }
        const VDesc& d = vt.v[id];
        if (d.src < 0) {
            if (vt.plain32) { // non-nullable int32-class fact columns only (warp-uniform)
                bits = (int64_t)ldg_stream_s32((const int32_t*)d.data + row);
                return false;
            }
            const bool nul = d.nulls != nullptr && d.nulls[row] != 0;
            bits = is_float_class(d.type) ? __double_as_longlong(load_double(d.data, d.type, row)) : load_int(d.data, d.type, row);
            return nul;
        }
        // build row 0 is the sentinel: a LEFT OUTER join without a matching build row reads NULL payloads
        const int64_t r = bidx[d.src];
        const bool nul = r == 0 || (d.nulls != nullptr && d.nulls[r] != 0);
        if (is_float_class(d.type))
            bits = __double_as_longlong(d.type == SR_TYPE_FLOAT ? (double)__ldg((const float*)d.data + r) : __ldg((const double*)d.data + r));
        else
            bits = load_int_cached(d.data, d.type, r);
        return nul;
    }
};

// one fact value for each alive row of a 4-row group (warp-uniform descriptor)
__device__ __forceinline__ void load_rows4(const VDesc& d, int64_t row0, uint32_t alive, int64_t vals[FRAG_ROWS], uint32_t& nullmask) {
    nullmask = 0;
    const int w = type_width(d.type);
    const bool isf = is_float_class(d.type);
    if (w == 4 && !isf) {
        if (alive == 0xF && (((uintptr_t)d.data) & 15) == 0) {
            const int4 v = ldg_stream_v4((const int32_t*)d.data + row0); // row0 % 4 == 0
            vals[0] = v.x;
            vals[1] = v.y;
            vals[2] = v.z;
            vals[3] = v.w;
        } else {
#pragma unroll
            for (int r = 0; r < FRAG_ROWS; r++) vals[r] = ldg_stream_s32_pred((const int32_t*)d.data + row0 + r, (alive >> r) & 1u);
        }
    } else if (w == 8 && !isf) {
#pragma unroll
        for (int r = 0; r < FRAG_ROWS; r++) vals[r] = ldg_stream_s64_pred((const int64_t*)d.data + row0 + r, (alive >> r) & 1u);
    } else {
#pragma unroll
        for (int r = 0; r < FRAG_ROWS; r++)
            if (alive & (1u << r)) vals[r] = isf ? __double_as_longlong(load_double(d.data, d.type, row0 + r)) : load_int(d.data, d.type, row0 + r);
    }
    if (d.nulls) {
#pragma unroll
        for (int r = 0; r < FRAG_ROWS; r++)
            if ((alive & (1u << r)) && d.nulls[row0 + r]) nullmask |= 1u << r;
    }
}

// whether a build row has the (non-NULL) key: the range-mapped bitmap, or the hash table's first[].  STAGED: the kernel
// copied the bitmaps with smem_off >= 0 to `smem` (smem_stage_bitmaps); otherwise every bitmap is read from global memory
template <bool STAGED>
__device__ __forceinline__ bool frag_join_hit(const FragJoinDev& fj, const uint32_t* smem, int64_t key) {
    if (fj.use_bitmap) {
        if (key < fj.j.min_value || key > fj.j.max_value) return false;
        const uint64_t idx = (uint64_t)(key - fj.j.min_value);
        const uint32_t word = STAGED && fj.smem_off >= 0 ? smem[fj.smem_off + (idx >> 5)] : __ldg(fj.j.bitmap + (idx >> 5));
        return (word >> (idx & 31)) & 1u;
    }
    return join_lookup(fj.j, key) != 0;
}

// whether a row passes filtering or anti join fj: `nul` its key is NULL
template <bool STAGED>
__device__ __forceinline__ bool frag_join_row(const FragJoinDev& fj, const uint32_t* smem, int64_t key, bool nul) {
    return frag_join_pass(fj.kind, nul, !nul && frag_join_hit<STAGED>(fj, smem, key));
}

// the rows of a 4-row group (`alive` bits, keys `vals`, NULL keys `nullmask`) that pass filtering or anti join fj,
// tested row by row against the staged bitmaps
template <typename K>
__device__ __forceinline__ uint32_t frag_join_group(const FragJoinDev& fj, const uint32_t* smem, const K (&vals)[FRAG_ROWS], uint32_t nullmask, uint32_t alive) {
    // NULL keys never match (join_hash_table.cpp:166-170): they fail a filtering join and pass an anti join
    const uint32_t tested = alive & ~nullmask;
    if (fj.kind != FRAG_ANTI) alive = tested;
#pragma unroll
    for (int r = 0; r < FRAG_ROWS; r++)
        if ((tested & (1u << r)) && !frag_join_pass(fj.kind, false, frag_join_hit<true>(fj, smem, (int64_t)vals[r]))) alive &= ~(1u << r);
    return alive;
}

// a tile's filter: the scan conjuncts (ColumnPredicate form, `preds` the shared copies; warp-uniform loop, the loads of
// both groups first), then the generic boolean conjuncts row by row.  Clears the alive bits of the rows that fail.  vals /
// nullmask: the caller's load registers, which its join test reuses (separate arrays cost the streaming pass spills)
__device__ __forceinline__ void frag_tile_filter(const FragDev& fd, const CPred* preds, const VTab& vt, const int64_t (&row0)[FRAG_GROUPS], uint32_t (&alive)[FRAG_GROUPS],
                                                 int64_t (&vals)[FRAG_GROUPS][FRAG_ROWS], uint32_t (&nullmask)[FRAG_GROUPS]) {
#pragma unroll 1
    for (int p = 0; p < fd.num_preds; p++) {
        const VDesc& d = vt.v[preds[p].value_id];
#pragma unroll
        for (int g = 0; g < FRAG_GROUPS; g++) load_rows4(d, row0[g], alive[g], vals[g], nullmask[g]);
#pragma unroll
        for (int g = 0; g < FRAG_GROUPS; g++)
#pragma unroll
            for (int r = 0; r < FRAG_ROWS; r++)
                if ((alive[g] & (1u << r)) && !eval_pred(preds[p], vals[g][r], (nullmask[g] >> r) & 1u)) alive[g] &= ~(1u << r);
    }
#pragma unroll 1
    for (int e = 0; e < fd.num_exprs; e++) {
#pragma unroll 1
        for (int g = 0; g < FRAG_GROUPS; g++)
#pragma unroll 1
            for (int r = 0; r < FRAG_ROWS; r++) {
                if (alive[g] & (1u << r)) {
                    ChunkLoader ld{vt, row0[g] + r};
                    int64_t bits;
                    const bool nul = eval_expr(fd.exprs[e], ld, bits);
                    if (nul || bits == 0) alive[g] &= ~(1u << r);
                }
            }
    }
}

// The joins of one row that reached a final pass, in probe order: the filtering and anti joins of [first_test, S) are
// tested (frag_join_pass), and every join whose payload is read downstream or whose chain expands (need_head) is looked
// up -- an outer join only that way: it never fails the row, and a NULL key or a key without a build row leaves build
// row 0, whose payloads read NULL.  Fills ld.bidx with the build rows found and, when `head` is given, head[j] with the
// same chain heads (0 for a join not looked up).  Returns whether the row passed.  `joins` and `S` are read through
// references: the cascade keeps them in its per-warp state in local memory, and re-reading them there per join keeps
// copies out of k_fragment's registers (capped at 64, already spilling) across the walk.
__device__ __forceinline__ bool frag_final_joins(const FragJoinDev* const& joins, const int& S, int first_test, FragLoader& ld, uint32_t* head) {
    bool ok = true;
#pragma unroll 1
    for (int j = 0; j < S && ok; j++) {
        if (head) head[j] = 0;
        const bool test = j >= first_test && joins[j].kind != FRAG_OUTER;
        if (!test && !joins[j].need_head) continue;
        int64_t key;
        const bool nul = ld.load(joins[j].key_value_id, key);
        if (joins[j].need_head || !joins[j].use_bitmap) {
            const uint32_t h = nul ? 0u : join_lookup(joins[j].j, key);
            ld.bidx[j] = h;
            if (head) head[j] = h;
            if (test && !frag_join_pass(joins[j].kind, nul, h != 0)) ok = false;
        } else if (!frag_join_row<false>(joins[j], nullptr, key, nul)) {
            ok = false;
        }
    }
    return ok;
}

// everything a warp needs to run the cascade (kept in registers / shared memory)
struct Cascade {
    const VTab& vt;
    const AggDev& ad;
    const AccPtrs& acc;
    const FragJoinDev* joins; // shared-memory copies
    const uint32_t* smem;     // dynamic shared memory base (bitmaps)
    uint32_t* q;              // this warp's queues: [SR_MAX_FRAG_JOINS][FRAG_QCAP] rows, then [FRAG_QCAP] keys of queue 0
    uint32_t* qc;             // this warp's fill counts
    int S, NQ;
    int eager1;
    int shared_acc; // the accumulators live in shared memory
    uint32_t lane;
    unsigned long long passed;
    uint32_t* fail_rows; // hash aggregate: the rows a full slice refuses (they applied nothing), counted at fail_count
    unsigned long long* fail_count;

    __device__ __forceinline__ void set_count(int k, uint32_t v) {
        if (lane == 0) qc[k] = v;
        __syncwarp();
    }
    // append the rows of lanes with `keep` to queue k (caller guarantees qc[k] < 32 beforehand)
    __device__ __forceinline__ void append(int k, uint32_t row32, bool keep) {
        const uint32_t m = __ballot_sync(SR_FULL_MASK, keep);
        if (m == 0) return;
        const uint32_t cnt = qc[k];
        if (keep) q[k * FRAG_QCAP + cnt + __popc(m & lanemask_lt())] = row32;
        __syncwarp();
        set_count(k, cnt + __popc(m));
    }
    // queue 0 with the eagerly loaded key of the second join riding along
    __device__ __forceinline__ void append0_key(uint32_t row32, int32_t key1, bool keep) {
        const uint32_t m = __ballot_sync(SR_FULL_MASK, keep);
        if (m == 0) return;
        const uint32_t cnt = qc[0];
        if (keep) {
            const uint32_t pos = cnt + __popc(m & lanemask_lt());
            q[pos] = row32;
            q[SR_MAX_FRAG_JOINS * FRAG_QCAP + pos] = (uint32_t)key1;
        }
        __syncwarp();
        set_count(0, cnt + __popc(m));
    }
    // last queue: build-row lookups, group slot, aggregate update; one row per lane
    __device__ __forceinline__ void consume_final(uint32_t row32, bool valid) {
        if (valid) {
            FragLoader ld{vt, (int64_t)row32, {0, 0, 0, 0, 0, 0}, -1, 0};
            frag_final_joins(joins, S, S, ld, nullptr); // the queue stages tested every join: lookups only
            const long long slot = agg_find_slot(ad, ld);
            if (slot >= 0) {
                if (shared_acc)
                    agg_apply_row<true>(ad, acc, slot, ld);
                else
                    agg_apply_row<false>(ad, acc, slot, ld);
            } else if (!ad.dense) {
                fail_rows[atomicAdd(fail_count, 1ull)] = row32;
                return; // counted in rows_passed when it is run again
            }
            passed++;
        }
    }
    // queue k < NQ-1: probe join k+1 for up to 32 queued rows, survivors go to queue k+1
    __device__ __forceinline__ void consume_join(int k, uint32_t row32, int32_t carried_key, bool valid) {
        const FragJoinDev& fj = joins[k + 1];
        bool pass = false;
        if (valid) {
            if (k == 0 && eager1) { // the eagerly streamed key column is never nullable
                pass = frag_join_row<true>(fj, smem, (int64_t)carried_key, false);
            } else {
                const VDesc& d = vt.v[fj.key_value_id];
                const int64_t key = load_int(d.data, d.type, (int64_t)row32);
                const bool nul = d.nulls != nullptr && d.nulls[row32] != 0;
                pass = frag_join_row<true>(fj, smem, key, nul);
            }
        }
        append(k + 1, row32, pass);
    }
    // take the last `take` rows of queue k and run its consumer
    __device__ __noinline__ void drain(int k, uint32_t take) {
        const uint32_t base = qc[k] - take;
        const bool valid = lane < take;
        const uint32_t row32 = valid ? q[k * FRAG_QCAP + base + lane] : 0u;
        const int32_t key = (valid && k == 0 && eager1) ? (int32_t)q[SR_MAX_FRAG_JOINS * FRAG_QCAP + base + lane] : 0;
        __syncwarp();
        set_count(k, base);
        if (k == NQ - 1)
            consume_final(row32, valid);
        else
            consume_join(k, row32, key, valid);
    }
    // forward sweep: every queue >= kstart that holds a full batch runs once.  Restores the
    // invariant "every queue holds < 32 rows" when at most queue kstart was over.
    __device__ __forceinline__ void pump_full(int kstart) {
#pragma unroll 1
        for (int k = kstart; k < NQ; k++)
            if (qc[k] >= 32) drain(k, 32);
    }
    __device__ __forceinline__ void flush() {
#pragma unroll 1
        for (int k = 0; k < NQ; k++) {
            while (qc[k] > 0) {
                const uint32_t c = qc[k];
                drain(k, c >= 32 ? 32u : c);
                pump_full(k + 1);
            }
        }
    }
};

template <bool SMEM_AGG>
__global__ void __launch_bounds__(FRAG_BLOCK, 2) k_fragment(const FragDev* __restrict__ fdp, const AggDev* __restrict__ adp, const __grid_constant__ VTab vt, int64_t n,
                                                             int32_t queue_word_off, uint32_t* __restrict__ fail_rows, unsigned long long* __restrict__ fail_count) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ FragJoinDev s_joins[SR_MAX_FRAG_JOINS];
    __shared__ CPred s_preds[8];
    const FragDev& fd = *fdp;
    const AggDev& ad = *adp;
    const int S = fd.num_joins;
    // the filtering joins are the queue stages; the outer joins behind them are looked up by consume_final only
    const int SF = fd.num_filter_joins;
    // descriptors + bitmaps of the leading joins into shared memory
    smem_copy(s_joins, fd.joins, S);
    smem_copy(s_preds, fd.preds, fd.num_preds);
    smem_stage_bitmaps<false>(smem, fd.joins, S);
    AccPtrs acc;
    if (SMEM_AGG) {
        acc_ptrs_at(ad, (long long*)smem, ad.cap, acc);
        acc_smem_init(ad, acc);
    } else {
        acc_ptrs_global(ad, acc);
    }
    const int warp = threadIdx.x >> 5;
    uint32_t* const wq = smem + queue_word_off + warp * FRAG_WARP_QWORDS;
    if (lane_id() < 8) wq[(SR_MAX_FRAG_JOINS + 1) * FRAG_QCAP + lane_id()] = 0;
    __syncthreads();

    // streamed (prefetched) columns: join 0's key and, when eager, join 1's key.  The fast path needs
    // int32-class, 16-byte aligned, non-nullable key columns and no scan conjuncts ahead of the joins.
    bool fast0 = false, fast1 = false;
    const int32_t* key0 = nullptr;
    const int32_t* key1 = nullptr;
    if (SF > 0 && fd.num_preds == 0 && fd.num_exprs == 0) {
        const VDesc& d0 = vt.v[s_joins[0].key_value_id];
        fast0 = type_width(d0.type) == 4 && !is_float_class(d0.type) && d0.nulls == nullptr && (((uintptr_t)d0.data) & 15) == 0;
        key0 = (const int32_t*)d0.data;
        if (fast0 && fd.eager1 && SF > 1) {
            const VDesc& d1 = vt.v[s_joins[1].key_value_id];
            fast1 = type_width(d1.type) == 4 && !is_float_class(d1.type) && d1.nulls == nullptr && (((uintptr_t)d1.data) & 15) == 0;
            key1 = (const int32_t*)d1.data;
        }
    }

    // queue k feeds join k+1 (k+1 < SF) or the aggregate (the last queue)
    Cascade cs{vt, ad, acc, s_joins, smem, wq, wq + (SR_MAX_FRAG_JOINS + 1) * FRAG_QCAP, S, SF > 1 ? SF : 1, fast1 ? 1 : 0, SMEM_AGG ? 1 : 0, lane_id(), 0ull, fail_rows, fail_count};

    const int64_t num_tiles = (n + FRAG_TILE - 1) / FRAG_TILE;
    const int64_t full_tiles = n / FRAG_TILE; // tiles [0, full_tiles) have every row in range
    int4 pk0[FRAG_GROUPS], pk1[FRAG_GROUPS];
#pragma unroll
    for (int g = 0; g < FRAG_GROUPS; g++) pk0[g] = pk1[g] = make_int4(0, 0, 0, 0);
    auto prefetch = [&](int64_t tile) {
        if (fast0 && tile < full_tiles) {
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) {
                const int64_t r0 = tile * FRAG_TILE + (int64_t)g * (FRAG_BLOCK * FRAG_ROWS) + (int64_t)threadIdx.x * FRAG_ROWS;
                pk0[g] = ldg_stream_v4(key0 + r0);
                if (fast1) pk1[g] = ldg_stream_v4(key1 + r0);
            }
        }
    };
    prefetch(blockIdx.x);

    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int64_t row0[FRAG_GROUPS];
        uint32_t alive[FRAG_GROUPS];
        int32_t k1v[FRAG_GROUPS][FRAG_ROWS]; // eager second key
        frag_tile_rows(tile, n, row0, alive);
        const bool streamed = fast0 && tile < full_tiles;
        if (streamed) {
            // keys of this tile were requested one iteration ago: test them, then request the next tile's
            // (the requests stay in flight while this tile's survivors run through the cascade)
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) {
                const int32_t kv[FRAG_ROWS] = {pk0[g].x, pk0[g].y, pk0[g].z, pk0[g].w};
                k1v[g][0] = pk1[g].x;
                k1v[g][1] = pk1[g].y;
                k1v[g][2] = pk1[g].z;
                k1v[g][3] = pk1[g].w;
                alive[g] = frag_join_group(s_joins[0], smem, kv, 0u, alive[g]);
            }
            prefetch(tile + gridDim.x);
        } else {
            int64_t vals[FRAG_GROUPS][FRAG_ROWS];
            uint32_t nullmask[FRAG_GROUPS];
            frag_tile_filter(fd, s_preds, vt, row0, alive, vals, nullmask);
            // ---- first join on its key column ----
            if (SF > 0) {
                const VDesc& d = vt.v[s_joins[0].key_value_id];
#pragma unroll
                for (int g = 0; g < FRAG_GROUPS; g++) load_rows4(d, row0[g], alive[g], vals[g], nullmask[g]);
#pragma unroll
                for (int g = 0; g < FRAG_GROUPS; g++) alive[g] = frag_join_group(s_joins[0], smem, vals[g], nullmask[g], alive[g]);
                if (fast1) { // tail tile of a streamed run: the consumer of queue 0 expects the key to ride along
#pragma unroll
                    for (int g = 0; g < FRAG_GROUPS; g++)
#pragma unroll
                        for (int r = 0; r < FRAG_ROWS; r++) k1v[g][r] = ldg_stream_s32_pred(key1 + row0[g] + r, (alive[g] >> r) & 1u);
                }
            }
        }
        __syncwarp();
        // ---- append survivors to queue 0 and pump the cascade ----
        // (one call site: the loop is kept rolled so the live state is saved around a single call)
        static_assert(FRAG_GROUPS == 2, "the append loop packs two groups of alive bits");
        const uint32_t alive_all = alive[0] | (alive[1] << FRAG_ROWS);
        if (__ballot_sync(SR_FULL_MASK, alive_all != 0)) {
#pragma unroll 1
            for (int i = 0; i < FRAG_GROUPS * FRAG_ROWS; i++) {
                const int64_t rbase = i < FRAG_ROWS ? row0[0] : row0[1];
                const uint32_t row32 = (uint32_t)(rbase + (i & (FRAG_ROWS - 1)));
                const bool keep = (alive_all >> i) & 1u;
                if (fast1) {
                    int32_t kk = 0;
#pragma unroll
                    for (int q = 0; q < FRAG_GROUPS * FRAG_ROWS; q++)
                        if (q == i) kk = k1v[q / FRAG_ROWS][q % FRAG_ROWS];
                    cs.append0_key(row32, kk, keep);
                } else {
                    cs.append(0, row32, keep);
                }
                if (cs.qc[0] >= 32) cs.pump_full(0);
            }
        }
    }
    cs.flush();
    if (SMEM_AGG) {
        __syncthreads();
        acc_smem_flush(ad, acc);
    }
    const unsigned long long passed = warp_sum(cs.passed);
    if (lane_id() == 0 && passed) atomicAdd(fd.rows_passed, passed);
}

// adaptive join ordering: independent pass counts of each join on a sample of rows.  A join's other-join conjunct is not
// evaluated here, so its sampled pass rate is that of the key test alone: an overestimate, which orders the join later than
// it might go and sizes a hash aggregate's table for more survivors than arrive (the safe side)
__global__ void __launch_bounds__(256) k_frag_sample(const FragDev* __restrict__ fdp, const __grid_constant__ VTab vt, int64_t n,
                                                      unsigned long long* __restrict__ counts) {
    const FragDev& fd = *fdp;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        ChunkLoader ld{vt, row};
        {
            // rows passing every scan conjunct -> counts[SAMPLE_ALL_PREDS]
            bool pass = true;
            for (int p = 0; p < fd.num_preds; p++) {
                if (pass) {
                    int64_t bits;
                    const bool nul = ld.load(fd.preds[p].value_id, bits);
                    pass = eval_pred(fd.preds[p], bits, nul);
                }
                // rows passing conjuncts 0..p -> counts[SAMPLE_PREDS_UPTO + p] (how many rows reach the next streamed column)
                const uint32_t mp = __ballot_sync(__activemask(), pass);
                if (pass && (mp & lanemask_lt()) == 0) atomicAdd(&counts[SAMPLE_PREDS_UPTO + p], (unsigned long long)__popc(mp));
            }
            for (int e = 0; e < fd.num_exprs && pass; e++) {
                int64_t bits;
                const bool nul = eval_expr(fd.exprs[e], ld, bits);
                pass = !nul && bits != 0;
            }
            const uint32_t m = __ballot_sync(__activemask(), pass);
            if (pass && (m & lanemask_lt()) == 0) atomicAdd(&counts[SAMPLE_ALL_PREDS], (unsigned long long)__popc(m));
        }
        // rows each join lets through: an outer join all of them
        for (int j = 0; j < fd.num_joins; j++) {
            const FragJoinDev& fj = fd.joins[j];
            int64_t key;
            const bool nul = ld.load(fj.key_value_id, key);
            const bool pass = fj.kind == FRAG_OUTER || frag_join_row<false>(fj, nullptr, key, nul);
            const uint32_t m = __ballot_sync(__activemask(), pass);
            if (pass && (m & lanemask_lt()) == 0) atomicAdd(&counts[j], (unsigned long long)__popc(m));
        }
    }
}

} // namespace srd
