// sr_frag_pass.cuh -- the SELECTIVE mode of the fused fragment: a short pipeline of passes connected by
// device-resident selection vectors (the GPU form of the reference's Filter / selection vector,
// be/src/column/chunk.cpp:362 and storage late materialisation):
//
//   pass S  k_frag_stream       streams the scan-predicate columns and the key columns of the leading joins
//                               (128-bit loads, next tile prefetched), tests their bitmaps, appends the
//                               surviving row ids to a selection vector (warp-aggregated atomicAdd);
//   pass G  k_frag_gather_join  one per remaining selective join: lane-per-row gather of the key for the
//                               selected rows only (late materialisation at DRAM-sector granularity),
//                               bitmap / hash test, appends survivors to the next selection vector;
//   pass F  k_frag_gather_agg   remaining non-selective joins inline, build-row lookups, payload gathers,
//                               group slot, aggregate update in shared-memory accumulators.
//
// Every pass runs with full warps; the selection vectors are tiny next to the fact columns (4 B per
// surviving row), and no pass waits on the host: a pass reads its input length from the counter the
// previous pass bumped (same stream).  Row order inside a selection vector is not kept -- the consumer
// is an aggregate.
#pragma once

#include "sr_frag_kernel.cuh"

namespace srd {

// one test of the streaming pass in "fast" form (k_frag_stream_tests)
struct StreamTest {
    int32_t kind;     // 0: scan predicate as a range, lo <= v <= lo + span; 1: streamed join `join`
    int32_t value_id; // the int32-class column it reads
    int32_t join;
    uint32_t lo, span;
};
#define SR_MAX_STREAM_TESTS 6

// How k_frag_stream_tests runs one of its two vector-column tests, planned on the host (frag_plan_stream_tests) and read from the kernel
// parameter: nothing of it occupies a register of the issue-bound, register-capped kernel, and nothing is re-read from
// shared memory per tile.  kind: 0 = range conjunct, 1 = bitmap in shared memory at word smem_off (int32 index arithmetic,
// zero GUARD bit at index span + 1: an out-of-range key is clamped onto it, so the test needs neither a predicate nor a
// select), 2 = bitmap in global memory at bm (predicated word fetches, issued back to back), 3 = anything else (falls back
// to stream_test).  lo / span: the range, or the join table's [min, min + span].  inv (kinds 1 and 2): all ones for an anti
// join, whose test is the inverted bitmap test -- one 3-input logic op, (hits ^ inv) & alive; an out-of-range key reads a
// clear bit and so passes it.
struct VecTest {
    uint32_t kind;
    uint32_t lo, span;
    int32_t smem_off;
    const uint32_t* bm;
    uint32_t inv;
    uint32_t pad;
};

struct PassDev {
    int32_t num_tests; // > 0: the streaming pass can run as k_frag_stream_tests (subject to the batch's nullability)
    int32_t num_vec;   // its first num_vec (1 or 2) tests read their column with prefetched 128-bit loads
    VecTest vec[2];    // tests 0 and (num_vec > 1 ? 1 : 0) in the form k_frag_stream_tests runs them
    StreamTest tests[SR_MAX_STREAM_TESTS];
    int32_t num_stream_joins; // joins [0, num_stream_joins) are tested by the streaming pass
    int32_t final_first_join; // joins [final_first_join, S) are tested inline by the final pass
    // fact columns the final pass reads (k_frag_final_dense loads all of them for a batch of rows before anything
    // depends on them)
    int8_t final_vals[8];  // value ids, -1 = unused
    int8_t num_final_vals; // how many the final pass needs (may exceed 8: then only the generic final pass applies)
    // the int32 key of one streamed join whose build row the final pass needs travels in the upper half of the
    // selection-vector entries, so the final pass does not gather it from the fact table again
    int8_t carry_join;     // index of that join among the streamed joins, -1 = none
    int8_t carry_value_id; // its key's value id
    int8_t pad[2];
};

// selection-vector entry: row id (low 32 bits) + carried key (high 32 bits)
typedef unsigned long long SelEntry;
__device__ __forceinline__ uint32_t sel_row(SelEntry e) { return (uint32_t)e; }
__device__ __forceinline__ int32_t sel_carry(SelEntry e) { return (int32_t)(e >> 32); }
__device__ __forceinline__ SelEntry sel_make(uint32_t row, int32_t carry) { return (SelEntry)row | ((SelEntry)(uint32_t)carry << 32); }

#define SR_FINAL_PREFETCH 8

// bitmap word of a row that is still alive (alive_bit != 0) and whose index lies in the table's range; 0 otherwise.  The
// predicate is formed inside the asm block from the raw operands: handing a C++ bool in costs a select to 0 / 1 and a
// compare back (ncu: 6.6 instructions per row on this line of the issue-bound streaming pass)
__device__ __forceinline__ uint32_t ldg_bitmap_word(const uint32_t* bm, uint32_t idx, uint32_t span, uint32_t alive_bit) {
    uint32_t r;
    asm volatile(
            "{ .reg .pred q;\n"
            "  setp.le.u32 q, %2, %3;\n"
            "  setp.ne.and.u32 q, %4, 0, q;\n"
            "  mov.u32 %0, 0;\n"
            "  @q ld.global.nc.u32 %0, [%1]; }"
            : "=r"(r)
            : "l"(bm + (idx >> 5)), "r"(idx), "r"(span), "r"(alive_bit));
    return r;
}

__device__ __forceinline__ uint32_t ldg_u32_pred(const uint32_t* p, bool pred) {
    uint32_t r;
    asm volatile(
            "{ .reg .pred q; setp.ne.u32 q, %2, 0; mov.u32 %0, 0;\n"
            "  @q ld.global.nc.u32 %0, [%1]; }"
            : "=r"(r)
            : "l"(p), "r"((uint32_t)pred));
    return r;
}

// Test N keys (bit i of `alive` says whether key i is still wanted) against one join and clear the bits of
// the misses.  For bitmap joins the N word fetches are issued back to back (predicated, branch-free) so a
// thread pays one L2 round trip for its whole group instead of one per row.
template <int N, typename K>
__device__ __forceinline__ uint32_t join_test_batch(const FragJoinDev& fj, const uint32_t* smem, const K (&keys)[N], uint32_t alive) {
    if (sizeof(K) == 4 && fj.use_bitmap && fj.idx32) {
        // int32 keys against a table whose [min, max] fits int32: one unsigned subtract + compare does the
        // range check, and the whole test stays in 32-bit arithmetic (the stream kernel is issue bound)
        const uint32_t umin = (uint32_t)(int32_t)fj.j.min_value;
        const uint32_t span = (uint32_t)(fj.j.max_value - fj.j.min_value);
        uint32_t out = 0;
        if (fj.smem_off >= 0) {
            const uint32_t* bm = smem + fj.smem_off;
#pragma unroll
            for (int i = 0; i < N; i++) {
                const uint32_t idx = (uint32_t)keys[i] - umin;
                const bool p = ((alive >> i) & 1u) && idx <= span;
                const uint32_t word = p ? bm[idx >> 5] : 0u;
                // rotate bit (idx mod 32) of the word to position i, then one 3-input logic op merges it into `out`
                out |= __funnelshift_r(word, word, idx - (uint32_t)i) & (1u << i);
            }
        } else {
            uint32_t words[N];
#pragma unroll
            for (int i = 0; i < N; i++) {
                const uint32_t idx = (uint32_t)keys[i] - umin;
                const bool p = ((alive >> i) & 1u) && idx <= span;
                words[i] = ldg_u32_pred(fj.j.bitmap + (idx >> 5), p);
            }
#pragma unroll
            for (int i = 0; i < N; i++) {
                const uint32_t idx = (uint32_t)keys[i] - umin;
                out |= __funnelshift_r(words[i], words[i], idx - (uint32_t)i) & (1u << i);
            }
        }
        return out;
    }
    if (fj.use_bitmap) {
        const int64_t mn = fj.j.min_value, mx = fj.j.max_value;
        uint32_t words[N];
        uint32_t want = 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const bool p = ((alive >> i) & 1u) && keys[i] >= mn && keys[i] <= mx;
            const uint64_t idx = (uint64_t)(keys[i] - mn);
            want |= (p ? 1u : 0u) << i;
            if (fj.smem_off >= 0)
                words[i] = p ? smem[fj.smem_off + (idx >> 5)] : 0u;
            else
                words[i] = ldg_u32_pred(fj.j.bitmap + (idx >> 5), p);
        }
        uint32_t out = 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint64_t idx = (uint64_t)(keys[i] - mn);
            out |= (((want >> i) & 1u) & (words[i] >> (idx & 31))) << i;
        }
        return out;
    }
    uint32_t out = alive;
#pragma unroll
    for (int i = 0; i < N; i++)
        if (((alive >> i) & 1u) && join_lookup(fj.j, keys[i]) == 0) out &= ~(1u << i);
    return out;
}

constexpr int STREAM_MAX_JOINS = 2;

// Selection vectors are written through a per-warp chunk allocator: a warp takes SEL_CHUNK entries at a
// time from the global counter (one same-address atomic per ~SEL_CHUNK survivors instead of one per
// tile -- same-address atomics serialise in L2) and pads what it leaves unused with SEL_INVALID, which
// the consuming pass skips.  The counter therefore counts allocated entries, valid or not.
#define SEL_INVALID 0xFFFFFFFFu
constexpr uint32_t SEL_CHUNK = 256;

struct WarpSelWriter {
    SelEntry* __restrict__ out;
    unsigned long long* __restrict__ counter;
    unsigned long long pos, end; // warp-uniform
    __device__ __forceinline__ void init(SelEntry* o, unsigned long long* c) {
        out = o;
        counter = c;
        pos = end = 0;
    }
    // reserve `total` (<= SEL_CHUNK, warp-uniform) entries, returns the start index
    __device__ __forceinline__ unsigned long long reserve(uint32_t total) {
        if (pos + total > end) {
            for (unsigned long long i = pos + lane_id(); i < end; i += 32) out[i] = SEL_INVALID;
            unsigned long long base = 0;
            if (lane_id() == 0) base = atomicAdd(counter, (unsigned long long)SEL_CHUNK);
            pos = __shfl_sync(SR_FULL_MASK, base, 0);
            end = pos + SEL_CHUNK;
        }
        const unsigned long long p = pos;
        pos += total;
        return p;
    }
    __device__ __forceinline__ void finish() {
        for (unsigned long long i = pos + lane_id(); i < end; i += 32) out[i] = SEL_INVALID;
        pos = end;
    }
};

// append the rows flagged in `alive` (bit i -> row base_i + (i & 3)) with their carried keys (key_at(i), i not a
// compile-time constant) to the selection vector
template <bool CARRY, typename KeyAt>
__device__ __forceinline__ void warp_append_rows(uint32_t alive_all, int64_t row0_g0, int64_t row0_g1, KeyAt key_at, WarpSelWriter& w) {
    const uint32_t cnt = __popc(alive_all);
    const uint32_t incl = warp_incl_scan(cnt);
    const uint32_t total = __shfl_sync(SR_FULL_MASK, incl, 31);
    if (total == 0) return;
    SelEntry* __restrict__ sel_out = w.out + (w.reserve(total) + incl - cnt);
    // few rows survive (a lane holds 0..2 of its 8): walk the set bits instead of testing all eight
    const uint32_t r0 = (uint32_t)row0_g0, r1 = (uint32_t)row0_g1 - FRAG_ROWS;
    uint32_t m = alive_all, pos = 0;
    while (m) {
        const uint32_t i = (uint32_t)__ffs((int)m) - 1u;
        m &= m - 1u;
        const uint32_t row = (i < FRAG_ROWS ? r0 : r1) + i;
        sel_out[pos++] = CARRY ? sel_make(row, key_at(i)) : (SelEntry)row;
    }
}

// CARRY: the key of streamed join pd.carry_join rides in the upper half of the entries, so the final pass does not
// gather it from the fact table again (one random 32-byte sector per surviving row from HBM, ~2.5 ns of bus time per
// sector from pinned host memory).  (Re-reading the key for the survivors in this pass instead puts an L2 round trip
// on every tile's critical path.)
template <bool CARRY>
__global__ void __launch_bounds__(FRAG_BLOCK, 2) k_frag_stream(const FragDev* __restrict__ fdp, PassDev pd, const __grid_constant__ VTab vt, int64_t n,
                                                               SelEntry* __restrict__ sel_out, unsigned long long* __restrict__ counter) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ FragJoinDev s_joins[STREAM_MAX_JOINS];
    __shared__ CPred s_preds[8];
    const FragDev& fd = *fdp;
    const int SJ = pd.num_stream_joins;
    smem_copy(s_joins, fd.joins, SJ);
    smem_copy(s_preds, fd.preds, fd.num_preds);
    smem_stage_bitmaps<false>(smem, fd.joins, SJ);
    __syncthreads();

    // (the common shapes -- range conjuncts and joins on plain int32 columns -- run in k_frag_stream_tests below;
    // this kernel is the general form: any predicate, generic filter expressions, nullable / wide key columns)
    const int64_t num_tiles = (n + FRAG_TILE - 1) / FRAG_TILE;
    const int64_t full_tiles = n / FRAG_TILE;
    // Each CTA streams a CONTIGUOUS run of tiles (not a grid-stride walk): the rows a warp appends to one
    // selection-vector chunk then come from a narrow band of the table (~25 tiles) instead of being spread over
    // the whole batch, so the later gather passes touch neighbouring sectors / pages back to back.
    const int64_t tiles_per_cta = (num_tiles + gridDim.x - 1) / gridDim.x;
    const int64_t tile_begin = (int64_t)blockIdx.x * tiles_per_cta;
    const int64_t tile_end = tile_begin + tiles_per_cta < num_tiles ? tile_begin + tiles_per_cta : num_tiles;
    WarpSelWriter writer;
    writer.init(sel_out, counter);

    for (int64_t tile = tile_begin; tile < tile_end; tile++) {
        int64_t row0[FRAG_GROUPS];
        uint32_t alive[FRAG_GROUPS];
#pragma unroll
        for (int g = 0; g < FRAG_GROUPS; g++) {
            row0[g] = tile * FRAG_TILE + (int64_t)g * (FRAG_BLOCK * FRAG_ROWS) + (int64_t)threadIdx.x * FRAG_ROWS;
            alive[g] = 0xFu;
        }
        if (tile >= full_tiles) frag_tile_rows(tile, n, row0, alive); // only the last tile can be ragged
        int32_t carry[FRAG_GROUPS * FRAG_ROWS];
        if (CARRY) {
#pragma unroll
            for (int i = 0; i < FRAG_GROUPS * FRAG_ROWS; i++) carry[i] = 0;
        }
        int64_t vals[FRAG_GROUPS][FRAG_ROWS];
        uint32_t nullmask[FRAG_GROUPS];
        frag_tile_filter(fd, s_preds, vt, row0, alive, vals, nullmask);
#pragma unroll 1
        for (int j = 0; j < SJ; j++) {
            const VDesc& d = vt.v[s_joins[j].key_value_id];
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) load_rows4(d, row0[g], alive[g], vals[g], nullmask[g]);
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) alive[g] = frag_join_group(s_joins[j], smem, vals[g], nullmask[g], alive[g]);
            if (CARRY && j == pd.carry_join) {
#pragma unroll
                for (int g = 0; g < FRAG_GROUPS; g++)
#pragma unroll
                    for (int r = 0; r < FRAG_ROWS; r++) carry[g * FRAG_ROWS + r] = (int32_t)vals[g][r];
            }
        }
        static_assert(FRAG_GROUPS == 2, "two groups of alive bits are packed into one word");
        auto key_at = [&](uint32_t i) { // a select chain: indexing the register array with i would put it in local memory
            int32_t v = carry[0];
#pragma unroll
            for (int k = 1; k < FRAG_GROUPS * FRAG_ROWS; k++) v = i == (uint32_t)k ? carry[k] : v;
            return v;
        };
        warp_append_rows<CARRY>(alive[0] | (alive[1] << FRAG_ROWS), row0[0], row0[1], key_at, writer);
    }
    writer.finish();
}

// Streaming pass over a list of TESTS (PassDev::tests): scan predicates in range form (lo <= v <= lo + span on an
// int32-class column: EQ / LT / LE / GT / GE / BETWEEN all reduce to one unsigned subtract + compare) followed by the
// streamed joins.  The columns of the first one or two tests are read with 128-bit loads prefetched a tile ahead (most
// of their sectors are needed anyway); every later test loads its column only for the rows still alive (predicated
// loads, issued back to back).  The host picks this kernel when every test column is int32-class and not nullable
// (frag_push); anything else takes the generic path of k_frag_stream.  (Staging the vector columns in shared memory with
// cp.async.bulk instead buys nothing: the pass is issue bound, and every key then costs a shared-memory load as well.)
template <int N>
__device__ __forceinline__ uint32_t stream_test(const StreamTest& st, const FragJoinDev* s_joins, const uint32_t* smem, const int32_t (&k)[N], uint32_t alive) {
    if (st.kind == 0) {
        uint32_t out = 0;
#pragma unroll
        for (int i = 0; i < N; i++) out |= ((uint32_t)k[i] - st.lo <= st.span ? 1u : 0u) << i;
        return out & alive;
    }
    const FragJoinDev& fj = s_joins[st.join];
    const uint32_t inv = fj.kind == FRAG_ANTI ? ~0u : 0u; // the hits are a subset of `alive`
    return (join_test_batch<N>(fj, smem, k, alive) ^ inv) & alive;
}

// one of the two vector-column tests of k_frag_stream_tests in the form the host planned (VecTest); sbm = smem +
// t.smem_off
template <int N>
__device__ __forceinline__ uint32_t stream_test_reg(const VecTest& t, const uint32_t* sbm, const StreamTest& st, const FragJoinDev* s_joins, const uint32_t* smem,
                                                    const int32_t (&k)[N], uint32_t alive) {
    uint32_t out = 0;
    if (t.kind == 1) {
        const uint32_t guard = t.span + 1u;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint32_t idx = min((uint32_t)k[i] - t.lo, guard);
            const uint32_t word = sbm[idx >> 5];
            out |= __funnelshift_r(word, word, idx - (uint32_t)i) & (1u << i);
        }
        return (out ^ t.inv) & alive;
    }
    if (t.kind == 2) {
        uint32_t words[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint32_t idx = (uint32_t)k[i] - t.lo;
            words[i] = ldg_bitmap_word(t.bm, idx, t.span, alive & (1u << i));
        }
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint32_t idx = (uint32_t)k[i] - t.lo;
            out |= __funnelshift_r(words[i], words[i], idx - (uint32_t)i) & (1u << i);
        }
        return (out ^ t.inv) & alive;
    }
    if (t.kind == 0) {
#pragma unroll
        for (int i = 0; i < N; i++) out |= ((uint32_t)k[i] - t.lo <= t.span ? 1u : 0u) << i;
        return out & alive;
    }
    return stream_test<N>(st, s_joins, smem, k, alive);
}

// CARRY: the carried keys wait for the append in a per-thread STASH in shared memory (16 KB per CTA), not in registers.
// At two 512-thread CTAs per SM the kernel has 64 registers, and eight more live from the carried test to the append
// spilled: the spill stores of the prefetched vectors then waited on their loads on every tile.  Two 128-bit shared stores
// per tile instead, and a shared load per surviving row.
template <bool CARRY>
__global__ void __launch_bounds__(FRAG_BLOCK, 2) k_frag_stream_tests(const FragDev* __restrict__ fdp, const __grid_constant__ PassDev pd, const __grid_constant__ VTab vt, int64_t n,
                                                                     SelEntry* __restrict__ sel_out, unsigned long long* __restrict__ counter) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ FragJoinDev s_joins[STREAM_MAX_JOINS];
    __shared__ StreamTest s_tests[SR_MAX_STREAM_TESTS];
    __shared__ int4 s_carry[CARRY ? FRAG_GROUPS * FRAG_BLOCK : 1]; // [group][thread]: the keys of the thread's 4 rows
    const FragDev& fd = *fdp;
    const int SJ = pd.num_stream_joins;
    const int NT = pd.num_tests;
    const int NV = pd.num_vec;
    smem_copy(s_joins, fd.joins, SJ);
    smem_copy(s_tests, pd.tests, NT);
    smem_stage_bitmaps<true>(smem, fd.joins, SJ); // + the zero guard words (frag_plan_stream_smem reserves them)
    __syncthreads();
    const VecTest& t0 = pd.vec[0];
    const VecTest& t1 = pd.vec[1];
    const uint32_t* sbm0 = smem + (t0.kind == 1 ? t0.smem_off : 0);
    const uint32_t* sbm1 = smem + (t1.kind == 1 ? t1.smem_off : 0);
    const bool carry0 = CARRY && s_tests[0].kind == 1 && s_tests[0].join == pd.carry_join;
    const bool carry1 = CARRY && NV > 1 && s_tests[1].kind == 1 && s_tests[1].join == pd.carry_join;
    const int32_t* col0 = (const int32_t*)vt.v[pd.tests[0].value_id].data;
    const int32_t* col1 = NV > 1 ? (const int32_t*)vt.v[pd.tests[1].value_id].data : nullptr;
    const int64_t num_tiles = (n + FRAG_TILE - 1) / FRAG_TILE;
    const int64_t full_tiles = n / FRAG_TILE;
    const int64_t tiles_per_cta = (num_tiles + gridDim.x - 1) / gridDim.x;
    const int64_t tile_begin = (int64_t)blockIdx.x * tiles_per_cta;
    const int64_t tile_end = tile_begin + tiles_per_cta < num_tiles ? tile_begin + tiles_per_cta : num_tiles;
    const int64_t prefetch_end = tile_end < full_tiles ? tile_end : full_tiles;
    int4 pk[2][FRAG_GROUPS];
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
        for (int g = 0; g < FRAG_GROUPS; g++) pk[j][g] = make_int4(0, 0, 0, 0);
    auto prefetch = [&](int64_t tile) {
        if (tile < prefetch_end) {
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) {
                const int64_t r0 = tile * FRAG_TILE + (int64_t)g * (FRAG_BLOCK * FRAG_ROWS) + (int64_t)threadIdx.x * FRAG_ROWS;
                pk[0][g] = ldg_stream_v4(col0 + r0);
                if (col1) pk[1][g] = ldg_stream_v4(col1 + r0);
            }
        }
    };
    prefetch(tile_begin);
    WarpSelWriter writer;
    writer.init(sel_out, counter);
    static_assert(FRAG_GROUPS == 2 && FRAG_ROWS == 4, "8 rows per thread and tile");
    for (int64_t tile = tile_begin; tile < tile_end; tile++) {
        int64_t row0[FRAG_GROUPS];
#pragma unroll
        for (int g = 0; g < FRAG_GROUPS; g++)
            row0[g] = tile * FRAG_TILE + (int64_t)g * (FRAG_BLOCK * FRAG_ROWS) + (int64_t)threadIdx.x * FRAG_ROWS;
        uint32_t a8 = 0xFFu;
        int first_pred = 0; // tests [first_pred, NT) load their column for the live rows only
        if (tile < full_tiles) {
#pragma unroll
            for (int g = 0; g < FRAG_GROUPS; g++) {
                if (carry0) s_carry[g * FRAG_BLOCK + threadIdx.x] = pk[0][g];
                if (carry1) s_carry[g * FRAG_BLOCK + threadIdx.x] = pk[1][g];
            }
            const int32_t k0[8] = {pk[0][0].x, pk[0][0].y, pk[0][0].z, pk[0][0].w, pk[0][1].x, pk[0][1].y, pk[0][1].z, pk[0][1].w};
            const int32_t k1[8] = {pk[1][0].x, pk[1][0].y, pk[1][0].z, pk[1][0].w, pk[1][1].x, pk[1][1].y, pk[1][1].z, pk[1][1].w};
            prefetch(tile + 1); // the next tile's vector columns stay in flight while this tile is tested
            a8 = stream_test_reg<8>(t0, sbm0, s_tests[0], s_joins, smem, k0, 0xFFu);
            if (NV > 1) a8 = stream_test_reg<8>(t1, sbm1, s_tests[1], s_joins, smem, k1, a8);
            first_pred = NV;
        } else { // the ragged last tile: every test through predicated loads
            a8 = 0;
#pragma unroll
            for (int i = 0; i < 8; i++)
                if (row0[i >> 2] + (i & 3) < n) a8 |= 1u << i;
        }
#pragma unroll 1
        for (int t = first_pred; t < NT; t++) {
            const StreamTest& st = s_tests[t];
            const int32_t* col = (const int32_t*)vt.v[st.value_id].data;
            int32_t kk[8];
#pragma unroll
            for (int i = 0; i < 8; i++) kk[i] = ldg_stream_s32_pred(col + row0[i >> 2] + (i & 3), (a8 >> i) & 1u);
            a8 = stream_test<8>(st, s_joins, smem, kk, a8);
            if (CARRY && st.kind == 1 && st.join == pd.carry_join) {
#pragma unroll
                for (int g = 0; g < FRAG_GROUPS; g++) s_carry[g * FRAG_BLOCK + threadIdx.x] = make_int4(kk[4 * g], kk[4 * g + 1], kk[4 * g + 2], kk[4 * g + 3]);
            }
        }
        const int32_t* stash = (const int32_t*)s_carry + FRAG_ROWS * threadIdx.x;
        warp_append_rows<CARRY>(a8, row0[0], row0[1], [&](uint32_t i) { return stash[(i >> 2) * (FRAG_ROWS * FRAG_BLOCK) + (i & 3)]; }, writer);
    }
    writer.finish();
}

constexpr int GATHER_BLOCK = 256;

// the contiguous run [begin, end) of a selection vector of n entries that the calling warp owns (a multiple
// of 32 entries, so every warp-wide read of the vector is one aligned 128-byte line)
__device__ __forceinline__ void warp_sel_range(unsigned long long n, unsigned long long& begin, unsigned long long& end) {
    const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x >> 5);
    const unsigned long long me = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    unsigned long long per = (n + warps - 1) / warps;
    per = (per + 31) & ~31ull;
    begin = me * per;
    end = begin + per < n ? begin + per : n;
    if (begin > n) begin = n;
}

// one selective join on the selected rows: sel_in[0, *n_in) -> sel_out (appended at *counter_out)
__global__ void __launch_bounds__(GATHER_BLOCK) k_frag_gather_join(const FragDev* __restrict__ fdp, int32_t j, const __grid_constant__ VTab vt,
                                                                    const SelEntry* __restrict__ sel_in, const unsigned long long* __restrict__ n_in_ptr,
                                                                    SelEntry* __restrict__ sel_out, unsigned long long* __restrict__ counter_out) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ FragJoinDev s_join;
    smem_copy(&s_join, &fdp->joins[j], 1);
    __syncthreads();
    const unsigned long long n_in = *n_in_ptr;
    const FragJoinDev& fj = s_join;
    const VDesc& d = vt.v[fj.key_value_id];
    WarpSelWriter writer;
    writer.init(sel_out, counter_out);
    // each warp walks its own contiguous run of the input vector (whole chunks of one producer warp), so what
    // it appends keeps the producer's locality
    unsigned long long w_begin, w_end;
    warp_sel_range(n_in, w_begin, w_end);
    for (unsigned long long i0 = w_begin; i0 < w_end; i0 += 32) {
        const unsigned long long i = i0 + lane_id();
        bool hit = false;
        SelEntry entry = (SelEntry)SEL_INVALID;
        if (i < n_in) entry = sel_in[i];
        const uint32_t row = sel_row(entry);
        if (row != SEL_INVALID) {
            // (an L2::evict_first policy on this single-use load, and on the final pass's fact loads, to keep bitmaps and
            // directories resident changed neither pass on H100: 0.569 / 0.752 ms against 0.569 / 0.748 ms)
            const int64_t key = load_int(d.data, d.type, (int64_t)row);
            const bool nul = d.nulls != nullptr && d.nulls[row] != 0;
            hit = frag_join_row<false>(fj, nullptr, key, nul); // global bitmap copy: L1/L2 resident
        }
        const uint32_t m = __ballot_sync(SR_FULL_MASK, hit);
        if (m) {
            const unsigned long long base = writer.reserve(__popc(m));
            if (hit) sel_out[base + __popc(m & lanemask_lt())] = entry; // the carried key travels along
        }
    }
    writer.finish();
}

// the final pass is a chain of dependent gathers per row: latency bound, so resident warps matter more than spills.
// Five CTAs per SM (48 registers) balance resident warps against spills.
constexpr int GATHER_AGG_MIN_BLOCKS = 5;
// (The CONJ instantiations spill 72-504 B under this cap.  Three CTAs per SM remove every spill but made the Q95 ws_wh
// leg slower on H100, 1229 against 1023 ms: tools/frag_conjuncts.py, DESIGN.md section 6.)

// the first entry of join j's build chain, from ld.bidx[j] on, that makes the join's other-join conjunct TRUE (NULL counts
// as false).  Leaves ld.bidx[j] on it and returns whether there is one.
__device__ __forceinline__ bool frag_conj_seek(const FragDev& fd, const FragJoinDev& fj, int j, FragLoader& ld) {
#pragma unroll 1
    for (uint32_t b = ld.bidx[j]; b != 0; b = fj.j.has_dup ? __ldg(fj.j.next + b) : 0u) {
        ld.bidx[j] = b;
        int64_t bits;
        if (!eval_expr(fd.conj[j], ld, bits) && bits != 0) return true;
    }
    return false;
}

// The other-join conjuncts of a row that passed frag_final_joins.  A LEFT SEMI join passes the row when some entry of its
// chain makes its conjunct TRUE; an INNER join with unique keys when its one build row does; an expanding INNER join when
// some entry does, and that first entry becomes the head its odometer starts from and returns to (frag_next_combination
// then skips the entries that fail).  Each conjunct reads only fact values and its own join's build row, so the passing
// combinations are exactly the product of each join's passing entries.
template <bool EXPAND>
__device__ __forceinline__ bool frag_final_conjuncts(const FragDev& fd, const FragJoinDev* joins, int S, FragLoader& ld, uint32_t* head) {
    const int32_t mask = fd.conj_mask;
#pragma unroll 1
    for (int j = 0; j < S; j++) {
        if (!((mask >> j) & 1)) continue;
        if (!frag_conj_seek(fd, joins[j], j, ld)) return false;
        if (EXPAND) head[j] = ld.bidx[j];
    }
    return true;
}

// the next combination of chain entries of a row's expanding joins, like an odometer: advance the last expanding join,
// carry into the one before it when its chain ends.  False when every chain is back at its head.  CONJ: a join with an
// other-join conjunct advances to its next entry that makes the conjunct TRUE.
template <bool CONJ>
__device__ __forceinline__ bool frag_next_combination(const FragDev& fd, const FragJoinDev* joins, int S, FragLoader& ld, const uint32_t* head) {
#pragma unroll 1
    for (int j = S - 1; j >= 0; j--) {
        if (!joins[j].expand) continue;
        const uint32_t nx = __ldg(joins[j].j.next + ld.bidx[j]);
        if (CONJ && ((fd.conj_mask >> j) & 1)) {
            ld.bidx[j] = nx;
            if (frag_conj_seek(fd, joins[j], j, ld)) return true;
        } else if (nx) {
            ld.bidx[j] = nx;
            return true;
        }
        ld.bidx[j] = head[j];
    }
    return false;
}

// final pass: remaining joins inline, payload lookups, aggregate update.  SINGLE: no GROUP BY (its register state
// would only cost the grouped instantiations spills).
// EXPAND: some joins have duplicate build keys (reference: JoinHashMap::_probe_from_ht one-to-many walk,
// be/src/exec/join/join_hash_map.hpp:718-795 -- every probe row is emitted once per entry of the build chain of its
// key).  The probe output is never materialised: the thread that owns a surviving fact row walks the chains of its
// expanding joins like an odometer (last join fastest) and applies the aggregate once per combination, reading the
// payload columns at the current chain entries, into global accumulators.
// CONJ: some join has an other-join conjunct (frag_final_conjuncts); only the combinations that pass them are applied and
// counted, by both walks of the hash-table path.
template <bool SMEM_AGG, bool SINGLE, bool EXPAND, bool CONJ>
__global__ void __launch_bounds__(GATHER_BLOCK, GATHER_AGG_MIN_BLOCKS) k_frag_gather_agg(const FragDev* __restrict__ fdp, const AggDev* __restrict__ adp, const __grid_constant__ PassDev pd,
                                                                   const __grid_constant__ VTab vt, const SelEntry* __restrict__ sel_in,
                                                                   const unsigned long long* __restrict__ n_in_ptr, SelEntry* __restrict__ fail_list,
                                                                   unsigned long long* __restrict__ fail_count) {
    static_assert(!(SMEM_AGG && EXPAND), "the expanding form accumulates in global memory");
    // Hash aggregate tables are sized from the SAMPLED survivor estimate, not for the worst case "every row is a new
    // group" (a 65 M-row batch would allocate and clear a 13 GB table for 0.2 M groups).  A row the table cannot admit
    // (admission limit) is appended to fail_list; the host grows the table and runs this kernel again over that list.
    // A row is applied with all its combinations or not at all: with one combination its slot is found and applied in
    // one step; with EXPAND a first walk only finds / inserts the group slots, so a refused row has applied nothing.
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ FragJoinDev s_joins[SR_MAX_FRAG_JOINS];
    const FragDev& fd = *fdp;
    const AggDev& ad = *adp;
    const int S = fd.num_joins;
    const bool hash_table = !SINGLE && !ad.dense && ad.num_keys > 0;
    unsigned long long known_groups = hash_table && fail_list ? *(volatile unsigned long long*)ad.ngroups : 0ull;
    smem_copy(s_joins, fd.joins, S);
    AccPtrs acc;
    if (SMEM_AGG) {
        acc_ptrs_at(ad, (long long*)smem, ad.cap, acc);
        acc_smem_init(ad, acc);
    } else {
        acc_ptrs_global(ad, acc);
    }
    __syncthreads(); // s_joins and the shared accumulators are filled cooperatively: no warp may run ahead of that
    // Not done: requesting the NEXT row's fact sectors with prefetch.global.L2 while the current row walks its dependent
    // chain.  For HBM-resident input the prefetch fetches whole 128-byte lines where the loads need one 32-byte sector
    // (4x the DRAM traffic of a pass that is bound by random-sector throughput, not latency); mapped host memory is not
    // kept in L2, so for host-resident input the prefetch only doubles the PCIe requests.
    const unsigned long long n_in = *n_in_ptr;
    unsigned long long passed = 0;
    SingleAcc sacc;
    if (SINGLE) single_acc_init(ad, sacc);
    unsigned long long w_begin, w_end;
    warp_sel_range(n_in, w_begin, w_end);
    for (unsigned long long i = w_begin + lane_id(); i < w_end; i += 32) {
        const SelEntry entry = sel_in[i];
        const uint32_t row = sel_row(entry);
        if (row == SEL_INVALID) continue;
        // (a variant that fetches every fact value of the row in one burst before the dependent lookups costs more
        // issue slots and registers than the latency it hides)
        FragLoader ld{vt, (int64_t)row, {0, 0, 0, 0, 0, 0}, pd.carry_join >= 0 ? (int32_t)pd.carry_value_id : -1, sel_carry(entry)};
        uint32_t head[EXPAND ? SR_MAX_FRAG_JOINS : 1];
        if (!frag_final_joins(s_joins, S, pd.final_first_join, ld, EXPAND ? head : nullptr)) continue;
        if (CONJ && !frag_final_conjuncts<EXPAND>(fd, s_joins, S, ld, head)) continue;
        auto hash_slot = [&]() {
            HKey key;
            agg_pack_key(ad, ld, key);
            bool inserted;
            const long long slot = agg_find_slot_key(ad, key, inserted, known_groups);
            agg_count_new_groups(ad, inserted, known_groups);
            return slot;
        };
        if (EXPAND && hash_table) {
            // a first walk only finds / inserts the group slots of every combination (the second finds the same slots:
            // tables never shrink in between)
            bool refused = false;
            do {
                refused = hash_slot() < 0;
            } while (!refused && frag_next_combination<CONJ>(fd, s_joins, S, ld, head));
            if (refused) {
                if (fail_list) fail_list[atomicAdd(fail_count, 1ull)] = entry;
                continue;
            }
#pragma unroll 1
            for (int j = 0; j < S; j++) ld.bidx[j] = head[j]; // the odometer ends on the heads anyway; keeps the second walk independent of that
        }
        while (true) {
            if (SINGLE) { // no GROUP BY: the state lives in the thread, not behind an atomic
                single_acc_row(ad, sacc, ld);
            } else if (hash_table) {
                const long long slot = hash_slot();
                if (slot < 0) {
                    if (fail_list) fail_list[atomicAdd(fail_count, 1ull)] = entry; // retried after the table has grown
                    break;
                }
                agg_apply_row<SMEM_AGG>(ad, acc, slot, ld);
            } else {
                const long long slot = agg_find_slot(ad, ld);
                if (slot >= 0) agg_apply_row<SMEM_AGG>(ad, acc, slot, ld);
            }
            passed++;
            if (!EXPAND || !frag_next_combination<CONJ>(fd, s_joins, S, ld, head)) break;
        }
    }
    __syncwarp();
    if (SINGLE) single_acc_flush(ad, sacc);
    if (SMEM_AGG) {
        __syncthreads();
        acc_smem_flush(ad, acc);
    }
    passed = warp_sum(passed);
    if (lane_id() == 0 && passed) atomicAdd(fd.rows_passed, passed);
}

// ---- the final pass in batched form for dense star-join aggregates (k_frag_final_dense) ----
// A SLOT-DIGIT DIRECTORY replaces the two dependent lookups first[key - min] -> payload[b] of a join whose payload
// columns are only dense group keys: digit[key - min] is that join's share of the group slot, sum of idx_k * stride_k
// over the group keys that are its payloads (idx_k as agg_find_slot computes it).  Two values are reserved: MISS (no
// build row: the row fails the join; a LEFT OUTER join's directory holds its all-NULL digit there instead) and BAD (a
// payload outside the declared range, or NULL where the key is not nullable: the row passes, flags[1] is set, nothing
// is aggregated -- what agg_find_slot does).  2 bytes per key of the range, half of first[].
#define SR_DIGIT_MISS 0xFFFFu
#define SR_DIGIT_BAD 0xFFFEu

// one group key a directory folds in: a payload column of the join, read at the build row
struct DigitKey {
    const void* data;
    const uint8_t* nulls;
    int32_t type;
    int32_t nullable;
    long long min, extent, stride;
};
struct DigitPlan {
    int32_t num_keys;
    uint32_t miss; // the digit of a key without a build row: SR_DIGIT_MISS, or a LEFT OUTER join's all-NULL digit
    DigitKey k[SR_MAX_GROUP_KEYS];
};

__global__ void __launch_bounds__(256) k_frag_build_digits(const uint32_t* __restrict__ first, int64_t n, const __grid_constant__ DigitPlan dp,
                                                           uint16_t* __restrict__ digit) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = first[i];
        if (b == 0) {
            digit[i] = (uint16_t)dp.miss;
            continue;
        }
        long long slot = 0;
        bool bad = false;
#pragma unroll
        for (int k = 0; k < SR_MAX_GROUP_KEYS; k++) {
            if (k < dp.num_keys) {
                const DigitKey& d = dp.k[k];
                long long idx = 0;
                if (d.nulls != nullptr && d.nulls[b] != 0) {
                    bad |= !d.nullable;
                } else {
                    const int64_t v = load_int(d.data, d.type, b);
                    const unsigned long long off = (unsigned long long)v - (unsigned long long)d.min; // as agg_find_slot
                    bad |= off >= (unsigned long long)(d.extent - d.nullable);
                    idx = (long long)off + d.nullable;
                }
                slot += idx * d.stride;
            }
        }
        digit[i] = (uint16_t)(bad ? SR_DIGIT_BAD : (uint32_t)slot);
    }
}

constexpr int FINAL_MAX_VALS = 6;  // fact columns loaded per row
constexpr int FINAL_MAX_LOOK = 2;  // joins looked up through a directory
constexpr int FINAL_MAX_TEST = 2;  // joins only tested (bitmap)
constexpr int FINAL_MAX_FKEYS = 2; // group keys that are fact columns
constexpr int FINAL_MAX_FNS = 4;   // aggregate functions other than COUNT(*)
// R = 4 rows per lane and batch, three CTAs of 256 threads per SM: 66 registers, no spills (sm_90a).  Four CTAs cap the
// registers at 64 and spill.
constexpr int FINAL_ROWS = 4;
constexpr int FINAL_MIN_BLOCKS = 3;

// Everything k_frag_final_dense reads, in one kernel parameter (the constant bank): no shared descriptor copies, no
// per-row descriptor loads.  `val` fields index the fact values of `cols`.
struct FinalDense {
    int32_t num_vals, carry_val; // carry_val: index of the value the selection-vector entries carry, -1 = none
    const int32_t* cols[FINAL_MAX_VALS];
    int32_t num_look, num_test, num_fkeys, num_fns;
    struct Look {
        const uint16_t* digit;
        uint32_t lo, span; // directory index = key - lo, valid when <= span
        int32_t val;
        uint32_t miss; // the digit of a key outside the directory: SR_DIGIT_MISS, or a LEFT OUTER join's all-NULL digit
    } look[FINAL_MAX_LOOK];
    struct Test {
        const uint32_t* bitmap;
        uint32_t lo, span;
        int32_t val;
        uint32_t inv; // 1 for an anti join: the row passes on a clear bit
    } test[FINAL_MAX_TEST];
    struct FKey {
        long long lo;     // dense_min
        long long span;   // non-NULL values of the declared range
        uint32_t base;    // 1 when the key is nullable (index 0 is NULL)
        uint32_t stride;
        int32_t val, pad;
    } fkey[FINAL_MAX_FKEYS];
    struct Fn {
        long long* gacc; // global acc0
        int32_t mode;
        int32_t val;      // -1 for COUNT (a plain fact column is never NULL)
        int32_t smem_off; // long-long offset of its accumulators in shared memory
        int32_t pad;
    } fn[FINAL_MAX_FNS];
    int32_t cap, pad;
    long long* gcnt;
    int32_t* flags;
    unsigned long long* rows_passed;
};

// v[idx] for a warp-uniform idx without indexing the register array (a select chain, no local memory)
__device__ __forceinline__ int32_t final_pick(const int32_t (&v)[FINAL_MAX_VALS], int32_t idx) {
    int32_t x = 0;
#pragma unroll
    for (int k = 0; k < FINAL_MAX_VALS; k++)
        if (k == idx) x = v[k];
    return x;
}

__device__ __forceinline__ uint32_t ldg_u16_pred(const uint16_t* p, bool pred, uint32_t other) {
    uint16_t r;
    asm volatile(
            "{ .reg .pred q; setp.ne.u32 q, %2, 0; mov.u16 %0, %3;\n"
            "  @q ld.global.nc.u16 %0, [%1]; }"
            : "=h"(r)
            : "l"(p), "r"((uint32_t)pred), "h"((uint16_t)other));
    return r;
}

// Final pass for the shape of a star join into a dense shared-memory aggregate: every join the pass looks up has a
// slot-digit directory, every other join it handles is a bitmap test, every aggregate input is one plain int32 fact
// column in an integer mode.  A warp takes 32 x R consecutive selection-vector entries per iteration (lane l: entries
// base + l + 32 r, so each read of the vector is coalesced) and runs them in three phases: (1) every fact load of the
// R rows, (2) every directory load and bitmap test, (3) the shared-memory updates.  Against k_frag_gather_agg a row
// waits on two round trips instead of ~8 in a row, and R rows overlap theirs.
template <int R>
__global__ void __launch_bounds__(GATHER_BLOCK, FINAL_MIN_BLOCKS) k_frag_final_dense(const __grid_constant__ FinalDense fp, const SelEntry* __restrict__ sel_in,
                                                                                        const unsigned long long* __restrict__ n_in_ptr) {
    extern __shared__ __align__(16) uint32_t smem[];
    long long* const acc = (long long*)smem;
    const int cap = fp.cap;
    for (int i = threadIdx.x; i < cap; i += blockDim.x) {
        acc[i] = 0;
#pragma unroll
        for (int f = 0; f < FINAL_MAX_FNS; f++)
            if (f < fp.num_fns) acc[fp.fn[f].smem_off + i] = acc_init_value(fp.fn[f].mode);
    }
    __syncthreads();
    const unsigned long long n_in = *n_in_ptr;
    unsigned long long w_begin, w_end;
    warp_sel_range(n_in, w_begin, w_end);
    uint32_t passed = 0;
    bool any_bad = false;
    for (unsigned long long i0 = w_begin + lane_id(); i0 < w_end; i0 += 32 * R) {
        uint32_t row[R];
        int32_t carry[R];
        uint32_t live = 0;
#pragma unroll
        for (int r = 0; r < R; r++) {
            const unsigned long long i = i0 + 32 * r;
            const SelEntry e = i < w_end ? sel_in[i] : (SelEntry)SEL_INVALID;
            row[r] = sel_row(e);
            carry[r] = sel_carry(e);
            live |= (row[r] != SEL_INVALID ? 1u : 0u) << r;
        }
        // phase 1: every fact value of every row
        int32_t v[R][FINAL_MAX_VALS];
#pragma unroll
        for (int k = 0; k < FINAL_MAX_VALS; k++) {
#pragma unroll
            for (int r = 0; r < R; r++) {
                v[r][k] = 0;
                if (k < fp.num_vals) v[r][k] = k == fp.carry_val ? carry[r] : ldg_stream_s32_pred(fp.cols[k] + row[r], (live >> r) & 1u);
            }
        }
        // phase 2: directory words and bitmap words
        uint32_t dg[R][FINAL_MAX_LOOK];
        uint32_t tw[R][FINAL_MAX_TEST];
#pragma unroll
        for (int L = 0; L < FINAL_MAX_LOOK; L++) {
#pragma unroll
            for (int r = 0; r < R; r++) {
                dg[r][L] = 0;
                if (L < fp.num_look) {
                    const uint32_t idx = (uint32_t)final_pick(v[r], fp.look[L].val) - fp.look[L].lo;
                    dg[r][L] = ldg_u16_pred(fp.look[L].digit + idx, ((live >> r) & 1u) && idx <= fp.look[L].span, fp.look[L].miss);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < FINAL_MAX_TEST; t++) {
#pragma unroll
            for (int r = 0; r < R; r++) {
                tw[r][t] = 0;
                if (t < fp.num_test) {
                    const uint32_t idx = (uint32_t)final_pick(v[r], fp.test[t].val) - fp.test[t].lo;
                    tw[r][t] = ldg_u32_pred(fp.test[t].bitmap + (idx >> 5), ((live >> r) & 1u) && idx <= fp.test[t].span);
                    tw[r][t] = ((tw[r][t] >> (idx & 31)) & 1u) ^ fp.test[t].inv;
                }
            }
        }
        // phase 3: join verdicts, group slot, shared-memory update
#pragma unroll
        for (int r = 0; r < R; r++) {
            bool ok = (live >> r) & 1u;
            bool bad = false;
            uint32_t slot = 0;
#pragma unroll
            for (int L = 0; L < FINAL_MAX_LOOK; L++) {
                if (L < fp.num_look) {
                    ok &= dg[r][L] != SR_DIGIT_MISS;
                    bad |= dg[r][L] == SR_DIGIT_BAD;
                    slot += dg[r][L];
                }
            }
#pragma unroll
            for (int t = 0; t < FINAL_MAX_TEST; t++)
                if (t < fp.num_test) ok &= tw[r][t] != 0;
#pragma unroll
            for (int k = 0; k < FINAL_MAX_FKEYS; k++) {
                if (k < fp.num_fkeys) {
                    const long long idx = (long long)final_pick(v[r], fp.fkey[k].val) - fp.fkey[k].lo;
                    bad |= (unsigned long long)idx >= (unsigned long long)fp.fkey[k].span;
                    slot += ((uint32_t)idx + fp.fkey[k].base) * fp.fkey[k].stride;
                }
            }
            if (!ok) continue;
            passed++;
            if (bad) {
                any_bad = true;
                continue;
            }
            smem_add_u64(acc + slot, 1ull);
#pragma unroll
            for (int f = 0; f < FINAL_MAX_FNS; f++)
                if (f < fp.num_fns) acc_apply_shared(fp.fn[f].mode, acc + fp.fn[f].smem_off, nullptr, slot, (long long)final_pick(v[r], fp.fn[f].val));
        }
    }
    if (any_bad) fp.flags[1] = 1;
    __syncthreads();
    for (int i = threadIdx.x; i < cap; i += blockDim.x) {
        const long long c = acc[i];
        if (c == 0) continue;
        atomicAdd((unsigned long long*)fp.gcnt + i, (unsigned long long)c);
#pragma unroll
        for (int f = 0; f < FINAL_MAX_FNS; f++)
            if (f < fp.num_fns) acc_merge(fp.fn[f].mode, fp.fn[f].gacc, nullptr, i, acc[fp.fn[f].smem_off + i], 0);
    }
    const unsigned long long total = warp_sum((unsigned long long)passed);
    if (lane_id() == 0 && total) atomicAdd(fp.rows_passed, total);
}

} // namespace srd
