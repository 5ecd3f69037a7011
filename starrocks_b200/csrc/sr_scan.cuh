// sr_scan.cuh -- scan predicates -> uint8 selection vector -> order-preserving compaction.
// Replaces K1-K4 of SURVEY.md section 2b:
//   ColumnPredicate::evaluate/evaluate_and   be/src/storage/column_operator_predicate.h:41-111
//   ChunkPredicateEvaluator::eval_conjuncts  be/src/exprs/chunk_predicate_evaluator.cpp:84-149
//   Chunk::filter / t_filter_range<T>        be/src/column/chunk.cpp:362, column_filter_range.cpp:39-148
// HBM-bound streaming kernels: coalesced 4/8-byte loads per lane, selection kept as bytes (the
// reference's Filter), block counts + one scan, then a scatter that keeps input order.
#pragma once

#include "sr_rf.cuh"

namespace srd {

struct ChunkLoader {
    const VTab& vt;
    int64_t row;
    __device__ __forceinline__ bool load(int id, int64_t& bits) const {
        const VDesc& d = vt.v[id];
        if (vt.plain32) { // every column of this batch is a non-nullable int32-class column (warp-uniform)
            bits = (int64_t)ldg_stream_s32((const int32_t*)d.data + row);
            return false;
        }
        const bool nul = d.nulls != nullptr && d.nulls[row] != 0;
        bits = is_float_class(d.type) ? __double_as_longlong(load_double(d.data, d.type, row)) : load_int(d.data, d.type, row);
        return nul;
    }
};

struct ScanProg {
    CPred preds[16];
    int32_t num_preds;
    int32_t num_exprs;
    CExpr exprs[8];
};

// single-block exclusive scan of `n` uint32 counts into uint64 offsets; total -> *total.  The scan is 64-bit inside each
// 1024-count step as well: 1024 counts can sum past 2^32 (the probe blocks of a join with long chains), and a total that
// wrapped would let the host size the output too small instead of refusing it.
__global__ void __launch_bounds__(1024) k_scan_counts(const uint32_t* __restrict__ counts, int64_t n, uint64_t* __restrict__ offsets,
                                                       uint64_t* __restrict__ total) {
    __shared__ unsigned long long s_scan[1024 / 32 + 1];
    __shared__ uint64_t s_running;
    if (threadIdx.x == 0) s_running = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t i = base + threadIdx.x;
        const uint32_t v = i < n ? counts[i] : 0;
        unsigned long long tot;
        const unsigned long long ex = block_excl_scan64<1024>(v, s_scan, &tot);
        const uint64_t run = s_running;
        if (i < n) offsets[i] = run + ex;
        __syncthreads();
        if (threadIdx.x == 0) s_running = run + tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_running;
}

struct CompactCol {
    const void* src;
    void* dst;
    int32_t width;
    int32_t vec16; // width 16 with src and dst 16-byte aligned: one int4 per value
};
// a 16-byte value that need only be 8-byte aligned: copied as two 8-byte words
struct Words16 {
    unsigned long long lo, hi;
};
struct CompactArgs {
    CompactCol c[2 * SR_MAX_OUT_COLS];
    int32_t n;
};

// ---- warp-tile scan: 8 consecutive rows per lane, 256 rows per warp -----------------------------------------------
// k_scan_mask    conjuncts -> one selection BYTE PER LANE (bit r = row r of the lane's 8 rows survives), the tile's
//                survivor count, and (optionally) the reference-style uint8-per-row Filter
// k_scan_lvl1    first level of the exclusive scan of the tile counts (1024 tiles per block)
// k_scan_compact order-preserving compaction of every output column in ONE pass: a warp's survivors land in one
//                contiguous output run (tile offset + lane prefix + rank inside the lane)
// FAST form of the conjuncts: lo <= v <= lo + span on non-nullable int32-class columns (EQ / LT / LE / GT / GE /
// BETWEEN all reduce to it); the first column is read with two 128-bit loads per lane, the later ones only for the
// rows still alive (predicated loads).
constexpr int SCANW_ROWS = 8;
constexpr int SCANW_TILE = 32 * SCANW_ROWS;
constexpr int SCANW_BLOCK = 256;
#define SR_MAX_SCAN_RANGE_TESTS 8

struct RangeTest {
    int32_t value_id;
    uint32_t lo, span;
};
struct ScanTests {
    int32_t num_tests; // 0: generic evaluation
    int32_t vec0;      // the first column may be read with 128-bit loads (16-byte aligned)
    RangeTest t[SR_MAX_SCAN_RANGE_TESTS];
    // runtime filters attached to the scan (sr_scan_add_runtime_filter): applied to the rows the conjuncts keep
    int32_t num_rfs;
    int32_t pad;
    RfDev rfs[SR_MAX_SCAN_RFS];
    // per filter: rows tested / rows passed in this batch (nullptr: not counted) -- what RuntimeFilterProbeCollector::
    // update_selectivity measures (runtime_filter_probe.cpp:408-480)
    unsigned long long* rf_stats;
    int32_t rf_stat_index[SR_MAX_SCAN_RFS]; // slot of filter f in rf_stats (the scan's own numbering)
};

template <bool FAST, bool RF>
__global__ void __launch_bounds__(SCANW_BLOCK) k_scan_mask(const ScanProg* __restrict__ prog, const __grid_constant__ ScanTests st, const __grid_constant__ VTab vt,
                                                            int64_t n, uint8_t* __restrict__ mask_bits, uint32_t* __restrict__ tile_counts,
                                                            uint8_t* __restrict__ sel_bytes) {
    const int64_t ntiles = (n + SCANW_TILE - 1) / SCANW_TILE;
    const int64_t warps = (int64_t)gridDim.x * (SCANW_BLOCK / 32);
    const uint32_t lane = lane_id();
    for (int64_t tile = (int64_t)blockIdx.x * (SCANW_BLOCK / 32) + (threadIdx.x >> 5); tile < ntiles; tile += warps) {
        const int64_t base = tile * SCANW_TILE + (int64_t)lane * SCANW_ROWS;
        uint32_t m = 0;
#pragma unroll
        for (int r = 0; r < SCANW_ROWS; r++)
            if (base + r < n) m |= 1u << r;
        if (FAST) {
            const bool full = m == 0xFFu;
#pragma unroll 1
            for (int t = 0; t < st.num_tests; t++) {
                const RangeTest& rt = st.t[t];
                const int32_t* col = (const int32_t*)vt.v[rt.value_id].data;
                int32_t k[SCANW_ROWS];
                if (t == 0 && st.vec0 && full) {
                    uint32_t w[8];
                    ldg_stream_u32x8(col + base, w); // the lane's 8 consecutive rows = one 32-byte sector = one 256-bit load
#pragma unroll
                    for (int r = 0; r < SCANW_ROWS; r++) k[r] = (int32_t)w[r];
                } else {
#pragma unroll
                    for (int r = 0; r < SCANW_ROWS; r++) k[r] = ldg_stream_s32_pred(col + base + r, (m >> r) & 1u);
                }
                uint32_t pass = 0;
#pragma unroll
                for (int r = 0; r < SCANW_ROWS; r++) pass |= ((uint32_t)k[r] - rt.lo <= rt.span ? 1u : 0u) << r;
                m &= pass;
            }
        } else {
#pragma unroll 1
            for (int r = 0; r < SCANW_ROWS; r++) {
                if (!((m >> r) & 1u)) continue;
                ChunkLoader ld{vt, base + r};
                bool pass = true;
                for (int p = 0; p < prog->num_preds && pass; p++) {
                    int64_t bits;
                    const bool nul = ld.load(prog->preds[p].value_id, bits);
                    pass = eval_pred(prog->preds[p], bits, nul);
                }
                for (int e = 0; e < prog->num_exprs && pass; e++) {
                    int64_t bits;
                    const bool nul = eval_expr(prog->exprs[e], ld, bits);
                    pass = !nul && bits != 0;
                }
                if (!pass) m &= ~(1u << r);
            }
        }
        if (RF) {
            // RuntimeFilterProbeCollector::evaluate: every filter ANDs into the selection; a NULL probe value passes
            // only a filter that saw a NULL build key.  Only surviving rows pay the bucket read (one 32-byte sector).
#pragma unroll 1
            for (int f = 0; f < st.num_rfs && (st.rf_stats ? __any_sync(SR_FULL_MASK, m != 0) : m != 0); f++) {
                const RfDev& rf = st.rfs[f];
                uint32_t nulls = 0;
                long long v[SCANW_ROWS];
                const int32_t* c32 = (const int32_t*)vt.v[rf.value_id].data;
                if (vt.plain32 && m == 0xFFu && (((uintptr_t)c32) & 31) == 0) { // whole tile alive: one 256-bit load
                    uint32_t w[8];
                    ldg_stream_u32x8(c32 + base, w);
#pragma unroll
                    for (int r = 0; r < SCANW_ROWS; r++) v[r] = (int32_t)w[r];
                } else {
#pragma unroll
                    for (int r = 0; r < SCANW_ROWS; r++) {
                        int64_t bits = 0;
                        if ((m >> r) & 1u) nulls |= (ChunkLoader{vt, base + r}.load(rf.value_id, bits) ? 1u : 0u) << r;
                        v[r] = bits;
                    }
                }
                static_assert(SCANW_ROWS == 8, "two half-tiles of four rows");
                const long long va[4] = {v[0], v[1], v[2], v[3]}, vb[4] = {v[4], v[5], v[6], v[7]};
                const uint32_t test = m & ~nulls;
                const uint32_t pass = rf_test_rows<4>(rf, va, test & 15u) | (rf_test_rows<4>(rf, vb, test >> 4) << 4);
                if (st.rf_stats) { // one pair of atomics per warp, tile and filter
                    const uint32_t tested = warp_sum((uint32_t)__popc(m)), passed = warp_sum((uint32_t)__popc(pass | (rf.has_null ? m & nulls : 0u)));
                    if (lane == 0 && tested) {
                        atomicAdd(st.rf_stats + 2 * st.rf_stat_index[f], (unsigned long long)tested);
                        atomicAdd(st.rf_stats + 2 * st.rf_stat_index[f] + 1, (unsigned long long)passed);
                    }
                }
                m = pass | (rf.has_null ? m & nulls : 0u);
            }
        }
        if (mask_bits) mask_bits[tile * 32 + lane] = (uint8_t)m;
        if (sel_bytes) {
#pragma unroll
            for (int r = 0; r < SCANW_ROWS; r++)
                if (base + r < n) sel_bytes[base + r] = (uint8_t)((m >> r) & 1u);
        }
        if (tile_counts) {
            const uint32_t c = warp_sum((uint32_t)__popc(m));
            if (lane == 0) tile_counts[tile] = c;
        }
    }
}

// exclusive scan inside blocks of 1024 counts; block_sums[b] = total of block b.  SAT_SUM: the total is summed in 64 bits
// and stored saturated at 0xFFFFFFFF, so that counts passing 2^32 in one block cannot wrap to a small total (scan_counts:
// the host refuses such an output, and the wrapped offsets inside the block are never used)
template <bool SAT_SUM>
__global__ void __launch_bounds__(1024) k_scan_lvl1(const uint32_t* __restrict__ counts, int64_t n, uint32_t* __restrict__ local_excl, uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t s_scan[1024 / 32 + 1];
    __shared__ unsigned long long s_sum;
    const int64_t i = (int64_t)blockIdx.x * 1024 + threadIdx.x;
    const uint32_t v = i < n ? counts[i] : 0;
    if (SAT_SUM && threadIdx.x == 0) s_sum = 0;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<1024>(v, s_scan, &tot); // (synchronises the block: s_sum is initialised)
    if (i < n) local_excl[i] = ex;
    if (SAT_SUM) {
        const unsigned long long ws = warp_sum((unsigned long long)v);
        if (lane_id() == 0) atomicAdd(&s_sum, ws);
        __syncthreads();
        if (threadIdx.x == 0) block_sums[blockIdx.x] = s_sum > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)s_sum;
    } else if (threadIdx.x == 0) {
        block_sums[blockIdx.x] = tot;
    }
}

// offsets[i] = base of i's 1024-block + position inside the block (second half of the two-level scan)
__global__ void __launch_bounds__(1024) k_scan_add_base(const uint32_t* __restrict__ local_excl, const uint64_t* __restrict__ block_offsets, int64_t n,
                                                         uint64_t* __restrict__ offsets) {
    const int64_t i = (int64_t)blockIdx.x * 1024 + threadIdx.x;
    if (i < n) offsets[i] = block_offsets[blockIdx.x] + local_excl[i];
}

template <typename T>
__device__ __forceinline__ void compact_rows(const void* __restrict__ src, void* __restrict__ dst, int64_t base, uint32_t m, uint64_t out_pos) {
    const T* s = (const T*)src + base;
    T* d = (T*)dst + out_pos;
    uint32_t q = 0;
#pragma unroll
    for (int r = 0; r < SCANW_ROWS; r++)
        if ((m >> r) & 1u) d[q++] = s[r];
}
// dense tile, 4-byte column: the lane's 8 consecutive values by two 128-bit loads instead of up to 8 scalar ones
__device__ __forceinline__ void compact_rows_vec32(const void* __restrict__ src, void* __restrict__ dst, int64_t base, uint32_t m, uint64_t out_pos) {
    uint32_t v[SCANW_ROWS];
    ldg_stream_u32x8((const uint32_t*)src + base, v);
    uint32_t* d = (uint32_t*)dst + out_pos;
    uint32_t q = 0;
#pragma unroll
    for (int r = 0; r < SCANW_ROWS; r++)
        if ((m >> r) & 1u) d[q++] = v[r];
}

// survivors of a tile staged in shared memory (in order), then written by consecutive lanes: the direct form above lets
// every lane store to its own run of the output, i.e. up to 32 partially written sectors per store instruction, which is
// what bounds the dense-pass case
template <typename T>
__device__ __forceinline__ void compact_rows_staged(const void* __restrict__ src, void* __restrict__ dst, int64_t base, uint32_t m, bool vec, T* __restrict__ stage,
                                                    uint32_t my_off, uint32_t tile_total, uint64_t tile_out) {
    const T* s = (const T*)src + base;
    uint32_t q = my_off;
    if (sizeof(T) == 4 && vec) {
        uint32_t v[SCANW_ROWS];
        ldg_stream_u32x8(s, v);
#pragma unroll
        for (int r = 0; r < SCANW_ROWS; r++)
            if ((m >> r) & 1u) ((uint32_t*)stage)[q++] = v[r];
    } else {
#pragma unroll
        for (int r = 0; r < SCANW_ROWS; r++)
            if ((m >> r) & 1u) stage[q++] = s[r];
    }
    __syncwarp();
    T* d = (T*)dst + tile_out;
    for (uint32_t i = lane_id(); i < tile_total; i += 32) d[i] = stage[i];
    __syncwarp();
}

// STAGED: instantiated with the staging buffer; the host picks it when at least 1/8 of the rows survive (the buffer's
// 16 KB per CTA and the extra registers cost the sparse case its latency hiding)
template <bool STAGED>
__global__ void __launch_bounds__(SCANW_BLOCK) k_scan_compact(const uint8_t* __restrict__ mask_bits, const uint32_t* __restrict__ local_excl,
                                                               const uint64_t* __restrict__ block_offsets, CompactArgs args, int64_t n) {
    __shared__ unsigned long long s_stage[STAGED ? SCANW_BLOCK / 32 : 1][STAGED ? SCANW_TILE : 1];
    const int64_t ntiles = (n + SCANW_TILE - 1) / SCANW_TILE;
    const int64_t warps = (int64_t)gridDim.x * (SCANW_BLOCK / 32);
    const uint32_t lane = lane_id();
    for (int64_t tile = (int64_t)blockIdx.x * (SCANW_BLOCK / 32) + (threadIdx.x >> 5); tile < ntiles; tile += warps) {
        const uint32_t m = mask_bits[tile * 32 + lane];
        const uint32_t cnt = __popc(m);
        const uint32_t incl = warp_incl_scan(cnt);
        const uint32_t tile_total = __shfl_sync(SR_FULL_MASK, incl, 31);
        if (tile_total == 0) continue;
        const int64_t base = tile * SCANW_TILE + (int64_t)lane * SCANW_ROWS;
        const uint64_t out_pos = block_offsets[tile >> 10] + local_excl[tile] + (incl - cnt);
        // a tile where a quarter of the rows survive touches nearly every sector anyway: vector loads (warp-uniform)
        const bool dense = tile_total >= SCANW_TILE / 4 && (tile + 1) * SCANW_TILE <= n;
        const bool staged = STAGED && tile_total >= 32;
        if (staged) { // enough survivors to fill whole sectors: stage and write coalesced (all lanes take part)
            unsigned long long* stage = s_stage[threadIdx.x >> 5];
            const uint64_t tile_out = block_offsets[tile >> 10] + local_excl[tile];
            bool all_staged = true;
#pragma unroll 1
            for (int c = 0; c < args.n; c++) {
                const CompactCol col = args.c[c];
                if (col.width == 4)
                    compact_rows_staged<uint32_t>(col.src, col.dst, base, m, dense && (((uintptr_t)col.src) & 31) == 0, (uint32_t*)stage, incl - cnt, tile_total, tile_out);
                else if (col.width == 8)
                    compact_rows_staged<unsigned long long>(col.src, col.dst, base, m, false, stage, incl - cnt, tile_total, tile_out);
                else if (col.width == 1)
                    compact_rows_staged<uint8_t>(col.src, col.dst, base, m, false, (uint8_t*)stage, incl - cnt, tile_total, tile_out);
                else
                    all_staged = false;
            }
            if (all_staged) continue;
        }
        if (cnt == 0) continue;
#pragma unroll 1
        for (int c = 0; c < args.n; c++) {
            const CompactCol col = args.c[c];
            if (staged && (col.width == 4 || col.width == 8 || col.width == 1)) continue; // written by the staged path
            switch (col.width) {
            case 1:
                compact_rows<uint8_t>(col.src, col.dst, base, m, out_pos);
                break;
            case 2:
                compact_rows<uint16_t>(col.src, col.dst, base, m, out_pos);
                break;
            case 4:
                if (dense && (((uintptr_t)col.src) & 31) == 0)
                    compact_rows_vec32(col.src, col.dst, base, m, out_pos);
                else
                    compact_rows<uint32_t>(col.src, col.dst, base, m, out_pos);
                break;
            case 8:
                compact_rows<uint64_t>(col.src, col.dst, base, m, out_pos);
                break;
            default:
                if (col.vec16)
                    compact_rows<int4>(col.src, col.dst, base, m, out_pos);
                else
                    compact_rows<Words16>(col.src, col.dst, base, m, out_pos);
                break;
            }
        }
    }
}

template <typename T>
__device__ __forceinline__ void copy_elem(const void* src, void* dst, int64_t s, int64_t d) {
    ((T*)dst)[d] = ((const T*)src)[s];
}

// K11: dst[j] = src[index[j]] (Column::append_selective); index 0 of a build column is the
// sentinel row.  null_out (optional): 1 when index == 0 (outer join miss) or src null.
struct GatherArgs {
    GatherCol c[SR_MAX_OUT_COLS];
    int32_t n;
};

__global__ void __launch_bounds__(256) k_gather(const uint32_t* __restrict__ index, int64_t n, GatherArgs args) {
    const GatherCol col = args.c[blockIdx.y];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = index[i];
        switch (col.width) {
        case 1:
            copy_elem<uint8_t>(col.src, col.dst, s, i);
            break;
        case 2:
            copy_elem<uint16_t>(col.src, col.dst, s, i);
            break;
        case 4:
            copy_elem<uint32_t>(col.src, col.dst, s, i);
            break;
        case 8:
            copy_elem<uint64_t>(col.src, col.dst, s, i);
            break;
        default: // 16-byte values need only be 8-byte aligned
            if (col.vec16) {
                copy_elem<int4>(col.src, col.dst, s, i);
            } else {
                copy_elem<uint64_t>(col.src, col.dst, 2 * s, 2 * i);
                copy_elem<uint64_t>(col.src, col.dst, 2 * s + 1, 2 * i + 1);
            }
            break;
        }
        if (col.dst_nulls) {
            uint8_t nu = col.src_nulls ? col.src_nulls[s] : 0;
            if (col.zero_is_null && s == 0) nu = 1;
            col.dst_nulls[i] = nu;
        }
    }
}

} // namespace srd

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
// Exclusive scan of n uint32 counts into uint64 offsets, total -> ctx->dscratch[0].  Small inputs: one block walks
// the array (k_scan_counts); large inputs: 1024-entry blocks in parallel, a scan of the block sums, a fix-up pass
// (a single block walks 1024 entries at a time, far too slow for the ~780 K tiles of a 200 M-row probe).
// With `total`, the total is also read back to the host: one synchronisation, which also covers whatever the caller
// enqueued before.
struct ScanScratch {
    DevBuf local, sums, bases;
};
static int32_t scan_counts(sr_ctx* ctx, ScanScratch* sc, const uint32_t* counts, int64_t n, uint64_t* offsets, int64_t* total = nullptr) {
    if (n <= 16 * 1024) {
        srd::k_scan_counts<<<1, 1024, 0, ctx->stream>>>(counts, n, offsets, ctx->dscratch);
        SR_LAUNCH_CHECK(ctx);
    } else {
        const int64_t nblk = (n + 1023) / 1024;
        SR_TRY(sc->local.reserve(ctx, sizeof(uint32_t) * (size_t)n));
        SR_TRY(sc->sums.reserve(ctx, sizeof(uint32_t) * (size_t)nblk));
        SR_TRY(sc->bases.reserve(ctx, sizeof(uint64_t) * (size_t)nblk));
        srd::k_scan_lvl1<true><<<(int)nblk, 1024, 0, ctx->stream>>>(counts, n, sc->local.as<uint32_t>(), sc->sums.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
        srd::k_scan_counts<<<1, 1024, 0, ctx->stream>>>(sc->sums.as<uint32_t>(), nblk, sc->bases.as<uint64_t>(), ctx->dscratch);
        SR_LAUNCH_CHECK(ctx);
        srd::k_scan_add_base<<<(int)nblk, 1024, 0, ctx->stream>>>(sc->local.as<uint32_t>(), sc->bases.as<uint64_t>(), n, offsets);
        SR_LAUNCH_CHECK(ctx);
    }
    if (total) {
        SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned, ctx->dscratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *total = (int64_t)ctx->pinned[0];
    }
    return SR_OK;
}

// K11 over ga.n columns (n > 0, ga.n > 0): dst rows [0, n) from src rows index[0, n)
static int32_t launch_gather(sr_ctx* ctx, const uint32_t* index, int64_t n, srd::GatherArgs& ga) {
    for (int k = 0; k < ga.n; k++) {
        srd::GatherCol& g = ga.c[k];
        g.vec16 = g.width == 16 && (((uintptr_t)g.src | (uintptr_t)g.dst) & 15) == 0 ? 1 : 0;
    }
    srd::k_gather<<<dim3(std::min(grid_for(n, 256), ctx->num_sms * 16), ga.n), 256, 0, ctx->stream>>>(index, n, ga);
    SR_LAUNCH_CHECK(ctx);
    return SR_OK;
}

struct sr_scan {
    sr_ctx* ctx = nullptr;
    std::vector<sr_pred> preds;
    std::vector<sr_expr> exprs;
    std::vector<int32_t> out_slots;
    // compiled against the first chunk's slot types
    bool compiled = false;
    VReg reg;
    DevBuf prog;
    Staged staged;
    DevBuf sel;
    // warp-tile scan (k_scan_mask / k_scan_lvl1 / k_scan_compact)
    DevBuf mask_bits, tile_counts, local_excl, block_sums, block_offsets;
    srd::ScanTests tests; // range form of the conjuncts (num_tests == 0: generic evaluation)
    std::vector<std::pair<sr_rf*, int32_t>> rfs; // runtime filters (filter, probe slot)
    std::vector<int32_t> rf_value_ids;
    // adaptive use of the filters (RuntimeFilterProbeCollector::do_evaluate / update_selectivity, runtime_filter_probe.cpp:
    // 203-262,408-480): a filter that let more than half of the rows it tested through is not evaluated for the next 31
    // batches, then sampled again; the reference does the same per 32 chunks
    struct RfUse {
        unsigned long long tested = 0, passed = 0; // totals over all batches that evaluated it
        double last_selectivity = 0.0;
        int skip_batches = 0;
        int64_t batches_skipped = 0;
    };
    std::vector<RfUse> rf_use;
    DevBuf rf_stats; // 2 counters per filter, cleared per batch
    bool rf_adaptive = true;
    ColBufs out_cols; // one per out slot
};

static int32_t staged_slot_type(void* user, int32_t slot) {
    const Staged* st = (const Staged*)user;
    const int k = st->find(slot);
    return k < 0 ? 0 : st->cols[k].type;
}

static int32_t scan_compile(sr_scan* s) {
    sr_ctx* ctx = s->ctx;
    if (s->preds.size() > 16 || s->exprs.size() > 8) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many scan conjuncts");
    std::vector<uint8_t> hostbuf(sizeof(srd::ScanProg), 0);
    srd::ScanProg* hp = (srd::ScanProg*)hostbuf.data();
    s->reg = VReg();
    for (size_t k = 0; k < s->preds.size(); k++) SR_TRY(compile_pred(ctx, &s->preds[k], &s->reg, staged_slot_type, &s->staged, &hp->preds[k]));
    for (size_t k = 0; k < s->exprs.size(); k++) {
        SR_TRY(compile_expr(ctx, &s->exprs[k], &s->reg, staged_slot_type, &s->staged, &hp->exprs[k]));
        if (hp->exprs[k].result_is_double) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "filter expression %zu is not boolean", k);
    }
    hp->num_preds = (int32_t)s->preds.size();
    hp->num_exprs = (int32_t)s->exprs.size();
    // range form: every conjunct is EQ / LT / LE / GT / GE / BETWEEN with integer bounds on an int32-class column
    memset(&s->tests, 0, sizeof(s->tests));
    {
        bool ok = s->exprs.empty() && !s->preds.empty() && s->preds.size() <= SR_MAX_SCAN_RANGE_TESTS;
        for (size_t k = 0; k < s->preds.size() && ok; k++) {
            const srd::CPred& cp = hp->preds[k];
            long long lo, hi;
            const int32_t t = s->reg.types[cp.value_id];
            ok = pred_int32_range(cp, &lo, &hi) && srd::type_width(t) == 4 && !srd::is_float_class(t);
            if (!ok) break;
            s->tests.t[k] = srd::RangeTest{cp.value_id, (uint32_t)(int32_t)lo, (uint32_t)(hi - lo)};
        }
        s->tests.num_tests = ok ? (int32_t)s->preds.size() : 0;
    }
    s->rf_value_ids.clear();
    for (auto& rf : s->rfs) {
        const int32_t t = staged_slot_type(&s->staged, rf.second);
        if (t == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "runtime filter probes unknown slot %d", rf.second);
        if (srd::type_width(t) > 8 || srd::is_float_class(t)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "runtime filter on slot %d: integer-class columns only", rf.second);
        const int id = s->reg.add(rf.second, t);
        if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
        s->rf_value_ids.push_back(id);
    }
    SR_TRY(s->prog.reserve(ctx, sizeof(srd::ScanProg)));
    SR_CUDA(ctx, cudaMemcpyAsync(s->prog.p, hp, sizeof(srd::ScanProg), cudaMemcpyHostToDevice, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // hostbuf goes out of scope
    s->compiled = true;
    return SR_OK;
}

// runs predicate evaluation; leaves selection bytes in s->sel (device) and, when
// want_counts, tile counts/offsets + the total in ctx->pinned[0] (after a sync)
static int32_t scan_select(sr_scan* s, const sr_chunk_view* in, bool want_counts, int64_t* total_out) {
    sr_ctx* ctx = s->ctx;
    SR_TRY(s->staged.stage(ctx, in));
    if (!s->compiled) SR_TRY(scan_compile(s));
    VTab vt;
    SR_TRY(bind_vtab(ctx, s->reg, s->staged, &vt));
    const int64_t n = in->num_rows;
    const int64_t tiles = (n + srd::SCANW_TILE - 1) / srd::SCANW_TILE;
    const int64_t nblk = (tiles + 1023) / 1024;
    if (!want_counts) SR_TRY(s->sel.reserve(ctx, (size_t)std::max<int64_t>(n, 1)));
    if (want_counts) {
        SR_TRY(s->mask_bits.reserve(ctx, (size_t)std::max<int64_t>(tiles, 1) * 32));
        SR_TRY(s->tile_counts.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(tiles, 1)));
        SR_TRY(s->local_excl.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(tiles, 1)));
        SR_TRY(s->block_sums.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(nblk, 1)));
        SR_TRY(s->block_offsets.reserve(ctx, sizeof(uint64_t) * (size_t)std::max<int64_t>(nblk, 1)));
    }
    // the fast (range) form needs plain columns in THIS batch: not nullable; vector loads on the first one if aligned
    srd::ScanTests tests = s->tests;
    for (int t = 0; t < tests.num_tests; t++)
        if (vt.v[tests.t[t].value_id].nulls != nullptr) tests.num_tests = 0;
    tests.vec0 = tests.num_tests > 0 && (((uintptr_t)vt.v[tests.t[0].value_id].data) & 31) == 0 ? 1 : 0;
    tests.num_rfs = 0;
    tests.rf_stats = nullptr;
    if (s->rf_use.size() != s->rfs.size()) s->rf_use.assign(s->rfs.size(), sr_scan::RfUse());
    const bool count_rf = want_counts && s->rf_adaptive && !s->rfs.empty(); // the compacting call synchronises anyway: read the counters with it
    if (count_rf) {
        SR_TRY(s->rf_stats.reserve(ctx, sizeof(unsigned long long) * 2 * SR_MAX_SCAN_RFS));
        SR_CUDA(ctx, cudaMemsetAsync(s->rf_stats.p, 0, sizeof(unsigned long long) * 2 * SR_MAX_SCAN_RFS, ctx->stream));
        tests.rf_stats = s->rf_stats.as<unsigned long long>();
    }
    for (size_t f = 0; f < s->rfs.size(); f++) {
        if (count_rf && s->rf_use[f].skip_batches > 0) { // unselective at its last sample: skipped for now
            s->rf_use[f].skip_batches--;
            s->rf_use[f].batches_skipped++;
            continue;
        }
        const int k = tests.num_rfs++;
        SR_TRY(rf_device_desc(s->rfs[f].first, &tests.rfs[k])); // reads min/max once the build side is complete
        tests.rfs[k].value_id = s->rf_value_ids[f];
        tests.rf_stat_index[k] = (int32_t)f;
    }
    if (n > 0) {
        const int grid = (int)std::min<int64_t>((tiles + srd::SCANW_BLOCK / 32 - 1) / (srd::SCANW_BLOCK / 32), (int64_t)ctx->num_sms * 8);
        uint8_t* mask = want_counts ? s->mask_bits.as<uint8_t>() : nullptr;
        uint32_t* counts = want_counts ? s->tile_counts.as<uint32_t>() : nullptr;
        uint8_t* bytes = want_counts ? nullptr : s->sel.as<uint8_t>();
        const srd::ScanProg* prog = (const srd::ScanProg*)s->prog.p;
        if (tests.num_rfs > 0) {
            if (tests.num_tests > 0)
                srd::k_scan_mask<true, true><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(prog, tests, vt, n, mask, counts, bytes);
            else
                srd::k_scan_mask<false, true><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(prog, tests, vt, n, mask, counts, bytes);
        } else if (tests.num_tests > 0) {
            srd::k_scan_mask<true, false><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(prog, tests, vt, n, mask, counts, bytes);
        } else {
            srd::k_scan_mask<false, false><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(prog, tests, vt, n, mask, counts, bytes);
        }
        SR_LAUNCH_CHECK(ctx);
    }
    if (want_counts) {
        if (n > 0) {
            srd::k_scan_lvl1<false><<<(int)nblk, 1024, 0, ctx->stream>>>(s->tile_counts.as<uint32_t>(), tiles, s->local_excl.as<uint32_t>(), s->block_sums.as<uint32_t>());
            SR_LAUNCH_CHECK(ctx);
            srd::k_scan_counts<<<1, 1024, 0, ctx->stream>>>(s->block_sums.as<uint32_t>(), nblk, s->block_offsets.as<uint64_t>(), ctx->dscratch);
            SR_LAUNCH_CHECK(ctx);
            SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned, ctx->dscratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
            if (count_rf) SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned + 8, s->rf_stats.p, sizeof(unsigned long long) * 2 * SR_MAX_SCAN_RFS, cudaMemcpyDeviceToHost, ctx->stream));
            SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            *total_out = (int64_t)ctx->pinned[0];
            if (count_rf) {
                for (size_t f = 0; f < s->rfs.size(); f++) {
                    const unsigned long long tested = ctx->pinned[8 + 2 * f], passed = ctx->pinned[8 + 2 * f + 1];
                    if (tested == 0) continue;
                    sr_scan::RfUse& u = s->rf_use[f];
                    u.tested += tested;
                    u.passed += passed;
                    u.last_selectivity = (double)passed / (double)tested;
                    if (u.last_selectivity > 0.5) u.skip_batches = 31; // "useful filter": selectivity <= 0.5 (runtime_filter_probe.cpp:449)
                }
            }
        } else {
            *total_out = 0;
        }
    }
    return SR_OK;
}
