// sr_device.cuh -- device-side building blocks shared by all kernels of libsr_gpu.so:
// typed column loads, the reference's hash functions, the compiled expression interpreter,
// block scan / ordered compaction helpers.  sm_90a only.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sr_gpu_ops.h"

#define SR_WARP 32
#define SR_FULL_MASK 0xffffffffu

namespace srd {

// ---------------------------------------------------------------------------------------
// device column descriptor (mirror of sr_col_view with the width resolved)
// ---------------------------------------------------------------------------------------
struct DCol {
    const void* data;
    const uint8_t* nulls;
    int32_t type;
    int32_t width;
};

__host__ __device__ inline int type_width(int32_t t) {
    switch (t) {
    case SR_TYPE_BOOLEAN:
    case SR_TYPE_TINYINT:
        return 1;
    case SR_TYPE_SMALLINT:
        return 2;
    case SR_TYPE_INT:
    case SR_TYPE_FLOAT:
    case SR_TYPE_DATE:
    case SR_TYPE_DECIMAL32:
        return 4;
    case SR_TYPE_BIGINT:
    case SR_TYPE_DOUBLE:
    case SR_TYPE_DATETIME:
    case SR_TYPE_DECIMAL64:
        return 8;
    case SR_TYPE_LARGEINT:
    case SR_TYPE_DECIMAL128:
        return 16;
    default:
        return 0;
    }
}
__host__ __device__ inline bool is_float_class(int32_t t) {
    return t == SR_TYPE_FLOAT || t == SR_TYPE_DOUBLE;
}
__host__ __device__ inline bool is_decimal(int32_t t) {
    return t == SR_TYPE_DECIMAL32 || t == SR_TYPE_DECIMAL64 || t == SR_TYPE_DECIMAL128;
}

// streaming loads: fact columns are read once -> bypass L1 allocation, keep L1/L2 for tables
#ifndef SR_LD_HINT
#define SR_LD_HINT ".L1::no_allocate"
#endif
__device__ __forceinline__ int4 ldg_stream_v4(const void* p) {
    int4 r;
    asm volatile("ld.global.nc" SR_LD_HINT ".v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
// a whole 32-byte sector per lane: sm_90 has no 256-bit load, so two 128-bit loads issued back to back (both halves are
// in flight before either is used).  p must be 32-byte aligned.
__device__ __forceinline__ void ldg_nc_u32x8(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
                 : "l"(p));
}
__device__ __forceinline__ void ldg_stream_u32x8(const void* p, uint32_t (&w)[8]) {
    asm volatile("ld.global.nc" SR_LD_HINT ".v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc" SR_LD_HINT ".v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
                 : "l"(p));
}
__device__ __forceinline__ int32_t ldg_stream_s32(const void* p) {
    int32_t r;
    asm volatile("ld.global.nc" SR_LD_HINT ".s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ int64_t ldg_stream_s64(const void* p) {
    int64_t r;
    asm volatile("ld.global.nc" SR_LD_HINT ".s64 %0, [%1];" : "=l"(r) : "l"(p));
    return r;
}
// predicated streaming loads: no branch, so the loads of a group issue back to back
__device__ __forceinline__ int32_t ldg_stream_s32_pred(const void* p, bool pred) {
    int32_t r;
    asm volatile(
            "{ .reg .pred q; setp.ne.u32 q, %2, 0; mov.s32 %0, 0;\n"
            "  @q ld.global.nc" SR_LD_HINT ".s32 %0, [%1]; }"
            : "=r"(r)
            : "l"(p), "r"((uint32_t)pred));
    return r;
}
__device__ __forceinline__ int64_t ldg_stream_s64_pred(const void* p, bool pred) {
    int64_t r;
    asm volatile(
            "{ .reg .pred q; setp.ne.u32 q, %2, 0; mov.s64 %0, 0;\n"
            "  @q ld.global.nc.L1::no_allocate.s64 %0, [%1]; }"
            : "=l"(r)
            : "l"(p), "r"((uint32_t)pred));
    return r;
}

// request a line into L2 without waiting for it (no destination register, no scoreboard)
__device__ __forceinline__ void prefetch_l2(const void* p) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// value of integer-class column at row i, sign/zero extended to int64 (truncating int128)
__device__ __forceinline__ int64_t load_int(const void* data, int32_t type, int64_t i) {
    switch (type) {
    case SR_TYPE_BOOLEAN:
        return ((const uint8_t*)data)[i];
    case SR_TYPE_TINYINT:
        return ((const int8_t*)data)[i];
    case SR_TYPE_SMALLINT:
        return ((const int16_t*)data)[i];
    case SR_TYPE_INT:
    case SR_TYPE_DATE:
    case SR_TYPE_DECIMAL32:
        return ldg_stream_s32((const int32_t*)data + i);
    case SR_TYPE_BIGINT:
    case SR_TYPE_DATETIME:
    case SR_TYPE_DECIMAL64:
        return ldg_stream_s64((const int64_t*)data + i);
    case SR_TYPE_LARGEINT:
    case SR_TYPE_DECIMAL128:
        return ((const int64_t*)data)[2 * i];
    default:
        return 0;
    }
}
__device__ __forceinline__ double load_double(const void* data, int32_t type, int64_t i) {
    if (type == SR_TYPE_FLOAT) return (double)((const float*)data)[i];
    if (type == SR_TYPE_DOUBLE) return ((const double*)data)[i];
    return (double)load_int(data, type, i);
}
// cached variants for build-side / table data (reused across probes)
__device__ __forceinline__ int64_t load_int_cached(const void* data, int32_t type, int64_t i) {
    switch (type_width(type)) {
    case 1:
        return type == SR_TYPE_BOOLEAN ? (int64_t)((const uint8_t*)data)[i] : (int64_t)((const int8_t*)data)[i];
    case 2:
        return ((const int16_t*)data)[i];
    case 4:
        return __ldg((const int32_t*)data + i);
    case 8:
        return __ldg((const long long*)data + i);
    case 16:
        return __ldg((const long long*)data + 2 * i);
    default:
        return 0;
    }
}

// ---------------------------------------------------------------------------------------
// hash functions of the reference
// ---------------------------------------------------------------------------------------
// JoinKeyHash<T,4> / <T,8>: be/src/exec/join/join_hash_map_helper.h:35-54
__host__ __device__ __forceinline__ uint32_t join_key_hash32(uint32_t v, uint32_t log_buckets) {
    v ^= v >> (32 - log_buckets);
    return (v * 2654435761u) >> (32 - log_buckets);
}
__host__ __device__ __forceinline__ uint32_t join_key_hash64(uint64_t v, uint32_t log_buckets) {
    v ^= v >> (64 - log_buckets);
    return (uint32_t)((v * 11400714819323198485ull) >> (64 - log_buckets));
}
// HashUtil::fnv_hash over the little-endian bytes of one value: hash_util.hpp:127-134
__device__ __forceinline__ uint32_t fnv_hash_bytes(uint64_t lo, uint64_t hi, int width, uint32_t h) {
#pragma unroll 1
    for (int b = 0; b < width; b++) {
        const uint32_t byte = (uint32_t)((b < 8 ? (lo >> (8 * b)) : (hi >> (8 * (b - 8)))) & 0xFF);
        h = (byte ^ h) * 0x01000193u;
    }
    return h;
}
// zlib crc32 (HashUtil::zlib_crc_hash), bitwise: polynomial 0xEDB88320, pre/post inverted
__device__ __forceinline__ uint32_t zlib_crc32_bytes(uint64_t lo, uint64_t hi, int width, uint32_t seed) {
    uint32_t c = seed ^ 0xFFFFFFFFu;
#pragma unroll 1
    for (int b = 0; b < width; b++) {
        const uint32_t byte = (uint32_t)((b < 8 ? (lo >> (8 * b)) : (hi >> (8 * (b - 8)))) & 0xFF);
        c ^= byte;
#pragma unroll
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : (c >> 1);
    }
    return c ^ 0xFFFFFFFFu;
}
// HashUtil::xx_hash3_64 = XXH3_64bits_withSeed (be/src/base/hash/xxhash.h) of one fixed-width value of 1..16 bytes held in
// (lo, hi): XXH3_len_1to3_64b / XXH3_len_4to8_64b / XXH3_len_9to16_64b with the default secret.  The secret words are the
// little-endian reads of kSecret at the offsets the three routines use.
__device__ __forceinline__ uint64_t xxh3_64_value(uint64_t lo, uint64_t hi, int width, uint64_t seed) {
    if (width <= 2) { // (width 3 does not occur: fixed-width types are 1, 2, 4, 8, 16 bytes)
        const uint32_t b0 = (uint32_t)lo & 0xFFu, bm = (uint32_t)(lo >> (8 * (width >> 1))) & 0xFFu, bl = (uint32_t)(lo >> (8 * (width - 1))) & 0xFFu;
        const uint32_t combined = (b0 << 16) | (bm << 24) | bl | ((uint32_t)width << 8);
        uint64_t h = (uint64_t)combined ^ ((uint64_t)(0x396cfeb8u ^ 0xbe4ba423u) + seed); // secret[0..3] ^ secret[4..7]
        h ^= h >> 33;
        h *= 0xC2B2AE3D27D4EB4Full;
        h ^= h >> 29;
        h *= 0x165667B19E3779F9ull;
        return h ^ (h >> 32);
    }
    if (width <= 8) {
        seed ^= (uint64_t)__byte_perm((uint32_t)seed, 0, 0x0123) << 32;
        const uint32_t in1 = (uint32_t)lo, in2 = (uint32_t)(lo >> (8 * (width - 4)));
        uint64_t h = ((uint64_t)in2 + ((uint64_t)in1 << 32)) ^ ((0x1cad21f72c81017cull ^ 0xdb979083e96dd4deull) - seed); // secret[8..15] ^ secret[16..23]
        h ^= ((h << 49) | (h >> 15)) ^ ((h << 24) | (h >> 40));
        h *= 0x9FB21C651E98DF25ull;
        h ^= (h >> 35) + (uint64_t)width;
        h *= 0x9FB21C651E98DF25ull;
        return h ^ (h >> 28);
    }
    const uint64_t l = lo ^ ((0x1f67b3b7a4a44072ull ^ 0x78e5c0cc4ee679cbull) + seed); // secret[24..31] ^ secret[32..39]
    const uint64_t r = hi ^ ((0x2172ffcc7dd05a82ull ^ 0x8e2443f7744608b8ull) - seed); // secret[40..47] ^ secret[48..55]   (width 16: the last 8 bytes)
    const uint64_t sw = ((uint64_t)__byte_perm((uint32_t)l, 0, 0x0123) << 32) | (uint64_t)__byte_perm((uint32_t)(l >> 32), 0, 0x0123);
    uint64_t h = (uint64_t)width + sw + r + ((l * r) ^ __umul64hi(l, r));
    h ^= h >> 37;
    h *= 0x165667919E3779F9ull;
    return h ^ (h >> 32);
}
// ReduceOp: hash_util.hpp:242-244
__host__ __device__ __forceinline__ uint32_t reduce_op(uint32_t l, uint32_t r) {
    return (uint32_t)(((uint64_t)l * (uint64_t)r) >> 32);
}
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

// ---------------------------------------------------------------------------------------
// compiled expressions.  The host resolves slots to "value ids" and types statically
// (sr_host.cuh: compile_expr) so the device never inspects sr_type at run time.
// ---------------------------------------------------------------------------------------
enum COp : int32_t {
    C_LOAD_I = 1, // push integer-class value `arg`
    C_LOAD_D,     // push double-class value `arg`
    C_ICONST,
    C_DCONST,
    C_ADD_I,
    C_SUB_I,
    C_MUL_I,
    C_ADD_D,
    C_SUB_D,
    C_MUL_D,
    C_DIV_D,
    C_I2D,  // convert top of stack
    C_I2D2, // convert second of stack
    C_EQ_I,
    C_NE_I,
    C_LT_I,
    C_LE_I,
    C_GT_I,
    C_GE_I,
    C_EQ_D,
    C_NE_D,
    C_LT_D,
    C_LE_D,
    C_GT_D,
    C_GE_D,
    C_AND,
    C_OR,
    C_NOT,
    C_IS_NULL
};

struct CNode {
    int32_t op;
    int32_t arg; // value id for C_LOAD_*
    union {
        int64_t i;
        double d;
    } c;
};

// shapes the host recognises at compile time so the common aggregate inputs (a, a op b, a op const with + - *) skip
// the stack interpreter, whose dynamically indexed stack lives in local memory
enum CExprForm { F_GENERIC = 0, F_COL = 1, F_BIN_CC = 2, F_BIN_CK = 3 };

struct CExpr {
    CNode nodes[SR_MAX_EXPR_NODES];
    int32_t num_nodes;
    int32_t result_is_double;
    int32_t form; // CExprForm
    int32_t pad;
};

__host__ __device__ inline bool cexpr_is_simple_arith(int op) {
    return op == C_ADD_I || op == C_SUB_I || op == C_MUL_I || op == C_ADD_D || op == C_SUB_D || op == C_MUL_D;
}
__device__ __forceinline__ int64_t cexpr_simple_arith(int op, int64_t a, int64_t b) {
    if (op == C_MUL_I) return (int64_t)((uint64_t)a * (uint64_t)b);
    if (op == C_SUB_I) return (int64_t)((uint64_t)a - (uint64_t)b);
    if (op == C_ADD_I) return (int64_t)((uint64_t)a + (uint64_t)b);
    const double x = __longlong_as_double(a), y = __longlong_as_double(b);
    return __double_as_longlong(op == C_MUL_D ? x * y : op == C_SUB_D ? x - y : x + y);
}

// Loader concept: struct with
//   __device__ bool load(int value_id, int64_t& bits)   -> returns is_null; bits = int64 or
//   double bit pattern according to the static type of the value.
template <typename Loader>
__device__ __forceinline__ bool eval_expr(const CExpr& e, Loader& ld, int64_t& out_bits) {
    if (e.form == F_COL) return ld.load(e.nodes[0].arg, out_bits);
    if (e.form == F_BIN_CC || e.form == F_BIN_CK) {
        int64_t a, b = e.nodes[1].c.i;
        bool nul = ld.load(e.nodes[0].arg, a);
        if (e.form == F_BIN_CC) nul |= ld.load(e.nodes[1].arg, b);
        out_bits = cexpr_simple_arith(e.nodes[2].op, a, b);
        return nul;
    }
    int64_t st[SR_EXPR_STACK];
    bool nu[SR_EXPR_STACK];
    int sp = 0;
#pragma unroll 1
    for (int k = 0; k < e.num_nodes; k++) {
        const CNode nd = e.nodes[k];
        switch (nd.op) {
        case C_LOAD_I:
        case C_LOAD_D: {
            int64_t b;
            nu[sp] = ld.load(nd.arg, b);
            st[sp] = b;
            sp++;
            break;
        }
        case C_ICONST:
        case C_DCONST:
            st[sp] = nd.c.i;
            nu[sp] = false;
            sp++;
            break;
        case C_I2D:
            st[sp - 1] = __double_as_longlong((double)st[sp - 1]);
            break;
        case C_I2D2:
            st[sp - 2] = __double_as_longlong((double)st[sp - 2]);
            break;
        case C_NOT:
            st[sp - 1] = st[sp - 1] ? 0 : 1;
            break;
        case C_IS_NULL:
            st[sp - 1] = nu[sp - 1] ? 1 : 0;
            nu[sp - 1] = false;
            break;
        case C_AND:
        case C_OR: {
            // SQL three-valued logic
            const bool an = nu[sp - 2], bn = nu[sp - 1];
            const bool av = !an && st[sp - 2] != 0, bv = !bn && st[sp - 1] != 0;
            bool rv, rn;
            if (nd.op == C_AND) {
                const bool af = !an && !av, bf = !bn && !bv;
                rv = !(af || bf) && !(an || bn);
                rn = !(af || bf) && (an || bn);
            } else {
                rv = av || bv;
                rn = !rv && (an || bn);
            }
            sp--;
            st[sp - 1] = rv ? 1 : 0;
            nu[sp - 1] = rn;
            break;
        }
        default: {
            const int64_t a = st[sp - 2], b = st[sp - 1];
            const double x = __longlong_as_double(a), y = __longlong_as_double(b);
            int64_t r = 0;
            switch (nd.op) {
            case C_ADD_I:
                r = (int64_t)((uint64_t)a + (uint64_t)b);
                break;
            case C_SUB_I:
                r = (int64_t)((uint64_t)a - (uint64_t)b);
                break;
            case C_MUL_I:
                r = (int64_t)((uint64_t)a * (uint64_t)b);
                break;
            case C_ADD_D:
                r = __double_as_longlong(x + y);
                break;
            case C_SUB_D:
                r = __double_as_longlong(x - y);
                break;
            case C_MUL_D:
                r = __double_as_longlong(x * y);
                break;
            case C_DIV_D:
                r = __double_as_longlong(x / y);
                break;
            case C_EQ_I:
                r = a == b;
                break;
            case C_NE_I:
                r = a != b;
                break;
            case C_LT_I:
                r = a < b;
                break;
            case C_LE_I:
                r = a <= b;
                break;
            case C_GT_I:
                r = a > b;
                break;
            case C_GE_I:
                r = a >= b;
                break;
            case C_EQ_D:
                r = x == y;
                break;
            case C_NE_D:
                r = x != y;
                break;
            case C_LT_D:
                r = x < y;
                break;
            case C_LE_D:
                r = x <= y;
                break;
            case C_GT_D:
                r = x > y;
                break;
            case C_GE_D:
                r = x >= y;
                break;
            }
            sp--;
            st[sp - 1] = r;
            // a zero divisor yields NULL (ArithmeticRightZeroCheck, be/src/exprs/arithmetic_operation.h:638), DOUBLE included
            nu[sp - 1] = nu[sp - 1] || nu[sp] || (nd.op == C_DIV_D && y == 0.0);
            break;
        }
        }
    }
    out_bits = st[0];
    return nu[0];
}

// ---------------------------------------------------------------------------------------
// compiled ColumnPredicate conjunct (column_operator_predicate.h:41-111)
// ---------------------------------------------------------------------------------------
struct CPred {
    int32_t value_id; // which value (column) it tests
    int32_t op;       // sr_pred_op
    int32_t is_double;
    int32_t in_count;
    int64_t ilo, ihi;
    double dlo, dhi;
    int64_t in_list[SR_MAX_IN_LIST];
};

__device__ __forceinline__ bool eval_pred(const CPred& p, int64_t bits, bool is_null) {
    if (p.op == SR_PRED_IS_NULL) return is_null;
    if (p.op == SR_PRED_IS_NOT_NULL) return !is_null;
    if (is_null) return false;
    if (p.op == SR_PRED_IN || p.op == SR_PRED_NOT_IN) {
        bool found = false;
        for (int q = 0; q < p.in_count; q++) found |= (p.in_list[q] == bits);
        return (p.op == SR_PRED_IN) ? found : !found;
    }
    if (p.is_double) {
        const double v = __longlong_as_double(bits);
        switch (p.op) {
        case SR_PRED_EQ:
            return v == p.dlo;
        case SR_PRED_NE:
            return v != p.dlo;
        case SR_PRED_LT:
            return v < p.dlo;
        case SR_PRED_LE:
            return v <= p.dlo;
        case SR_PRED_GT:
            return v > p.dlo;
        case SR_PRED_GE:
            return v >= p.dlo;
        default:
            return v >= p.dlo && v <= p.dhi;
        }
    }
    switch (p.op) {
    case SR_PRED_EQ:
        return bits == p.ilo;
    case SR_PRED_NE:
        return bits != p.ilo;
    case SR_PRED_LT:
        return bits < p.ilo;
    case SR_PRED_LE:
        return bits <= p.ilo;
    case SR_PRED_GT:
        return bits > p.ilo;
    case SR_PRED_GE:
        return bits >= p.ilo;
    default:
        return bits >= p.ilo && bits <= p.ihi;
    }
}

// ---------------------------------------------------------------------------------------
// warp / block primitives
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lane_id() {
    return threadIdx.x & 31;
}
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(SR_FULL_MASK, v, o);
    return v;
}
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(SR_FULL_MASK, v, o);
        if (lane_id() >= (uint32_t)o) v += t;
    }
    return v;
}

// exclusive scan of one uint32 per thread across a block of BLOCK threads.
// returns the exclusive prefix; *total = block sum.  smem: BLOCK/32 + 1 words.
template <int BLOCK>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* smem, uint32_t* total) {
    const uint32_t incl = warp_incl_scan(v);
    const int w = threadIdx.x >> 5;
    if (lane_id() == 31) smem[w] = incl;
    __syncthreads();
    if (w == 0) {
        const int nw = BLOCK / 32;
        uint32_t x = (int)lane_id() < nw ? smem[lane_id()] : 0;
        const uint32_t xi = warp_incl_scan(x);
        if ((int)lane_id() < nw) smem[lane_id()] = xi - x;
        if ((int)lane_id() == nw - 1) smem[nw] = xi;
    }
    __syncthreads();
    const uint32_t res = incl - v + smem[w];
    *total = smem[BLOCK / 32];
    __syncthreads();
    return res;
}

} // namespace srd
