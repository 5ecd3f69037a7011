// sr_agg.cuh -- hash aggregate on the device.
// Replaces K13-K17 of SURVEY.md section 2b:
//   AggHashMap*::compute_agg_states (phmap lazy_emplace)   be/src/exec/aggregate/agg_hash_map.h:303-415,674-1263
//   AggregateFunctionBatchHelper::update_batch              be/src/exprs/agg/aggregate.h:407-412
//   Sum/Count/Avg/MaxMin ::update                           be/src/exprs/agg/sum.h:58-63, count.h:36, avg.h:84-103, maxmin.h
//   update_batch_single_state (no GROUP BY)                 sum.h:74-81, aggregator.cpp:882-905
//   Aggregator::convert_hash_map_to_chunk                   be/src/exec/aggregator.cpp:1696-1791
//
// Device layout: structure-of-arrays states (one 8-byte array per accumulator word) indexed by
// slot.  Two slot spaces:
//   * dense  -- the group-by columns have known small ranges (the FE's min/max statistics that
//               drive the reference's compressed-key maps): slot = mixed-radix index; tables of
//               <= 40 KB of state are accumulated in shared memory per CTA and flushed once;
//   * hash   -- open addressing on the packed fixed-size key (<= 8 bytes incl. a null-flag
//               byte), slot claimed with one atomicCAS on the key word; states updated with
//               red.global.add / atom.min / atom.max.
// int64 sums wrap exactly like the CPU (`sum += v`), so results are bit-exact whatever the
// order; 128-bit sums use a (lo, hi) pair with an exactly-once carry; double sums use
// atomicAdd(double) and are order dependent (tolerance 1e-6 relative in the tests).
#pragma once

#include "sr_join.cuh"

namespace srd {

enum AccMode : int32_t {
    M_COUNT_STAR = 0,
    M_COUNT,
    M_SUM_I64,
    M_SUM_I128,
    M_SUM_F64,
    M_AVG, // double sum + count
    M_MIN_I64,
    M_MAX_I64,
    M_MIN_F64, // stored as order-preserving int64 image of the double
    M_MAX_F64
};

#define SR_AGG_EMPTY 0xFFFFFFFFFFFFFFFFull

struct AggFnDev {
    int32_t kind;
    int32_t mode;
    int32_t in_is_double;
    int32_t track_n; // accn holds the non-null input count (else it equals cnt_star)
    int32_t result_type;
    int32_t n_value_id; // SR_AGG_AVG_MERGE: value id of the count state column added to accn (-1: every non-NULL input counts 1)
    long long* acc0;
    long long* acc1;
    long long* accn;
    CExpr input;
};

struct AggDev {
    int32_t num_keys, num_fns;
    int32_t dense;
    int32_t key_bytes; // packed key bytes incl. the null-flag byte
    int32_t key_value_id[SR_MAX_GROUP_KEYS];
    int32_t key_width[SR_MAX_GROUP_KEYS];
    int32_t key_type[SR_MAX_GROUP_KEYS];
    int32_t key_nullable[SR_MAX_GROUP_KEYS];
    int32_t key_shift[SR_MAX_GROUP_KEYS]; // bit offset inside the packed key
    int32_t null_shift;                   // bit offset of the null-flag byte
    int32_t wide;                         // packed key of 9..16 bytes: hkeys holds (lo, hi) pairs, claimed with a 128-bit CAS
    long long dense_min[SR_MAX_GROUP_KEYS];
    long long dense_extent[SR_MAX_GROUP_KEYS]; // range + nullable
    long long dense_stride[SR_MAX_GROUP_KEYS];
    unsigned long long cap; // slots (hash: power of two, plus one special slot at index cap)
    unsigned long long mask;
    unsigned long long limit; // admission limit for new groups
    // hash tables: a probe sequence never leaves the aligned SLICE of slice_mask + 1 slots its home slot lies in (it wraps
    // inside the slice).  A slice with all its state arrays fits the shared memory of one CTA, which is what lets the
    // radix-partitioned push (sr_agg_part.cuh) aggregate a whole slice on chip and write it back once.
    unsigned long long slice_mask;
    int32_t slice_log2;
    int32_t pad0;
    unsigned long long* hkeys;
    long long* cnt_star;
    unsigned long long* ngroups;
    int32_t* flags; // [0] overflow (new group refused), [1] key out of declared range
    AggFnDev fns[SR_MAX_AGG_FNS];
};

__device__ __forceinline__ long long f64_sortable(double d) {
    const long long b = __double_as_longlong(d);
    return b ^ ((b >> 63) & 0x7fffffffffffffffll);
}
__device__ __forceinline__ double f64_unsortable(long long s) {
    return __longlong_as_double(s ^ ((s >> 63) & 0x7fffffffffffffffll));
}

__host__ __device__ inline long long acc_init_value(int32_t mode) {
    switch (mode) {
    case M_MIN_I64:
    case M_MIN_F64:
        return 0x7fffffffffffffffll;
    case M_MAX_I64:
    case M_MAX_F64:
        return (long long)0x8000000000000000ll;
    default:
        return 0;
    }
}

struct AccPtrs {
    long long* cnt;
    long long* acc0[SR_MAX_AGG_FNS];
    long long* acc1[SR_MAX_AGG_FNS];
    long long* accn[SR_MAX_AGG_FNS];
};

// apply one (non-null) input value to the accumulators of slot
__device__ __forceinline__ void acc_apply(int32_t mode, long long* a0, long long* a1, long long slot, long long bits) {
    switch (mode) {
    case M_COUNT:
        atomicAdd((unsigned long long*)a0 + slot, 1ull);
        break;
    case M_SUM_I64:
        atomicAdd((unsigned long long*)a0 + slot, (unsigned long long)bits);
        break;
    case M_SUM_I128: {
        const unsigned long long v = (unsigned long long)bits;
        const unsigned long long old = atomicAdd((unsigned long long*)a0 + slot, v);
        const unsigned long long carry = (old + v) < old ? 1ull : 0ull;
        const unsigned long long hi = (bits < 0 ? ~0ull : 0ull) + carry;
        if (hi) atomicAdd((unsigned long long*)a1 + slot, hi);
        break;
    }
    case M_SUM_F64:
    case M_AVG:
        atomicAdd((double*)a0 + slot, __longlong_as_double(bits));
        break;
    case M_MIN_I64:
        atomicMin(a0 + slot, bits);
        break;
    case M_MAX_I64:
        atomicMax(a0 + slot, bits);
        break;
    case M_MIN_F64:
        atomicMin(a0 + slot, f64_sortable(__longlong_as_double(bits)));
        break;
    case M_MAX_F64:
        atomicMax(a0 + slot, f64_sortable(__longlong_as_double(bits)));
        break;
    default:
        break;
    }
}

// merge a partial state (s0, s1) into the accumulators of slot
__device__ __forceinline__ void acc_merge(int32_t mode, long long* a0, long long* a1, long long slot, long long s0, long long s1) {
    switch (mode) {
    case M_COUNT:
    case M_SUM_I64:
        if (s0) atomicAdd((unsigned long long*)a0 + slot, (unsigned long long)s0);
        break;
    case M_SUM_I128: {
        const unsigned long long v = (unsigned long long)s0;
        const unsigned long long old = atomicAdd((unsigned long long*)a0 + slot, v);
        const unsigned long long carry = (old + v) < old ? 1ull : 0ull;
        const unsigned long long hi = (unsigned long long)s1 + carry;
        if (hi) atomicAdd((unsigned long long*)a1 + slot, hi);
        break;
    }
    case M_SUM_F64:
    case M_AVG:
        atomicAdd((double*)a0 + slot, __longlong_as_double(s0));
        break;
    case M_MIN_I64:
    case M_MIN_F64:
        atomicMin(a0 + slot, s0);
        break;
    case M_MAX_I64:
    case M_MAX_F64:
        atomicMax(a0 + slot, s0);
        break;
    default:
        break;
    }
}

// ---- packed group key: up to 8 bytes in one word, or (wide) 9..16 bytes in a 16-byte aligned (lo, hi) pair.
// A column never straddles the two words (agg_compile lays them out that way).  An empty slot is all ones.
struct HKey {
    unsigned long long lo, hi;
};
__device__ __forceinline__ void hkey_or(HKey& k, unsigned long long bits, int shift) {
    if (shift < 64)
        k.lo |= bits << shift;
    else
        k.hi |= bits << (shift - 64);
}
__device__ __forceinline__ unsigned long long hkey_bits(const HKey& k, int shift) { return shift < 64 ? k.lo >> shift : k.hi >> (shift - 64); }
__device__ __forceinline__ bool hkey_is_empty(const AggDev& a, const HKey& k) { return k.lo == SR_AGG_EMPTY && (!a.wide || k.hi == SR_AGG_EMPTY); }
__device__ __forceinline__ bool hkey_eq(const AggDev& a, const HKey& x, const HKey& y) { return x.lo == y.lo && (!a.wide || x.hi == y.hi); }
// xorshift - multiply - xorshift: half the instructions of the murmur finaliser (mix64), and the radix-partitioned push
// hashes every row three times.  The leading fold keeps keys that differ only in their high bits (ids shifted left, packed
// second columns) apart in the LOW bits, which pick the slot inside a 256-slot probing slice.
__device__ __forceinline__ unsigned long long agg_hash64(unsigned long long x) {
    x ^= x >> 32;
    x *= 0x9E3779B97F4A7C15ull;
    return x ^ (x >> 29);
}
__device__ __forceinline__ unsigned long long hkey_hash(const AggDev& a, const HKey& k) {
    return a.wide ? agg_hash64(k.lo ^ (agg_hash64(k.hi) + 0x632BE59BD9B4E019ull)) : agg_hash64(k.lo);
}
__device__ __forceinline__ HKey hkey_load(const AggDev& a, unsigned long long s) {
    if (!a.wide) return HKey{a.hkeys[s], 0};
    HKey v; // ONE 16-byte access: a claim publishes both words at once, a split load could pair an old lo with a new hi
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.lo), "=l"(v.hi) : "l"(a.hkeys + 2 * s) : "memory");
    return v;
}
// try to claim the empty slot s for `key`; returns what the slot held before (empty = we own it now)
__device__ __forceinline__ HKey hkey_claim(const AggDev& a, unsigned long long s, const HKey& key) {
    if (!a.wide) return HKey{atomicCAS(&a.hkeys[s], SR_AGG_EMPTY, key.lo), 0};
    HKey old;
    asm volatile(
            "{ .reg .b128 c, n, o;\n"
            "  mov.b128 c, {%2, %3};\n"
            "  mov.b128 n, {%4, %5};\n"
            "  atom.global.cas.b128 o, [%6], c, n;\n"
            "  mov.b128 {%0, %1}, o; }"
            : "=l"(old.lo), "=l"(old.hi)
            : "l"(SR_AGG_EMPTY), "l"(SR_AGG_EMPTY), "l"(key.lo), "l"(key.hi), "l"(a.hkeys + 2 * s)
            : "memory");
    return old;
}

// pack the row's group-by values into the table key (hash tables only)
template <typename Loader>
__device__ __forceinline__ void agg_pack_key(const AggDev& a, Loader& ld, HKey& key) {
    key.lo = key.hi = 0;
#pragma unroll
    for (int k = 0; k < SR_MAX_GROUP_KEYS; k++) {
        if (k < a.num_keys) {
            int64_t v;
            const bool nul = ld.load(a.key_value_id[k], v);
            if (nul) {
                hkey_or(key, 1ull, a.null_shift + k);
            } else {
                const int w = a.key_width[k];
                const unsigned long long m = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1);
                hkey_or(key, (unsigned long long)v & m, a.key_shift[k]);
            }
        }
    }
}

// find or claim the slot of a packed key; -1 when it cannot be placed (flags set).  `inserted` = this call
// created the group: the CALLER adds it to a.ngroups (see agg_count_new_groups).  `known_groups` is the caller's
// register copy of the group count for admission control (refuse new groups beyond a.limit; the host grows the
// table and retries) -- a memory read of the counter per insert would make one L2 slice the bottleneck of the
// whole chip.  Pass 0 when the host has already guaranteed room for every row.
__device__ __forceinline__ long long agg_find_slot_key(const AggDev& a, const HKey& key, bool& inserted, unsigned long long known_groups) {
    inserted = false;
    if (hkey_is_empty(a, key)) return (long long)a.cap; // only possible for full 8- / 16-byte keys: the special slot
    unsigned long long s = hkey_hash(a, key) & a.mask;
    const unsigned long long sb = s & ~a.slice_mask;
    for (unsigned long long tries = 0; tries <= a.slice_mask; tries++) {
        HKey cur = hkey_load(a, s);
        if (hkey_eq(a, cur, key)) return (long long)s;
        if (hkey_is_empty(a, cur)) {
            if (known_groups >= a.limit) {
                a.flags[0] = 1;
                return -1;
            }
            cur = hkey_claim(a, s, key);
            if (hkey_is_empty(a, cur)) {
                inserted = true;
                return (long long)s;
            }
            if (hkey_eq(a, cur, key)) return (long long)s;
        }
        s = sb | ((s + 1) & a.slice_mask);
    }
    a.flags[0] = 1;
    return -1;
}

// slot of the row's group; -1 when the row cannot be placed (flags set)
template <typename Loader>
__device__ __forceinline__ long long agg_find_slot(const AggDev& a, Loader& ld) {
    if (a.num_keys == 0) return 0;
    if (a.dense) {
        long long slot = 0;
        bool bad = false;
#pragma unroll
        for (int k = 0; k < SR_MAX_GROUP_KEYS; k++) {
            if (k < a.num_keys) {
                int64_t v;
                const bool nul = ld.load(a.key_value_id[k], v);
                long long idx;
                if (nul) {
                    idx = 0;
                    bad |= !a.key_nullable[k];
                } else {
                    idx = v - a.dense_min[k] + (a.key_nullable[k] ? 1 : 0);
                    bad |= (v < a.dense_min[k]) || (idx >= a.dense_extent[k]);
                }
                slot += idx * a.dense_stride[k];
            }
        }
        if (bad) {
            a.flags[1] = 1;
            return -1;
        }
        return slot;
    }
    // callers of this form (the fused fragment kernels) have had room guaranteed by the host: no admission check
    HKey key;
    agg_pack_key(a, ld, key);
    bool inserted;
    const long long slot = agg_find_slot_key(a, key, inserted, 0ull);
    if (inserted) atomicAdd(a.ngroups, 1ull);
    return slot;
}

// Count the groups a warp just created with ONE atomic (a same-address atomic per new group serialises in L2:
// 1e8 new groups would spend tens of milliseconds on this counter alone) and refresh the callers' register copy
// of the group count from its return value.  Call from converged or diverged code.
__device__ __forceinline__ void agg_count_new_groups(const AggDev& a, bool inserted, unsigned long long& known_groups) {
    const unsigned act = __activemask();
    const unsigned b = __ballot_sync(act, inserted);
    if (b) {
        const int leader = __ffs(act) - 1;
        unsigned long long old = 0;
        if (lane_id() == (uint32_t)leader) old = atomicAdd(a.ngroups, (unsigned long long)__popc(b));
        known_groups = __shfl_sync(act, old, leader) + (unsigned long long)__popc(b);
    }
}

// shared-memory accumulators: explicit .shared reductions (a generic-address atomic on a shared
// location is far slower than red.shared)
// 64-bit add into shared memory through NATIVE 32-bit shared atomics: add the low word (atom returns the old value ->
// exactly one adder sees each wrap), then add high word + carry when that is not zero.  A 64-bit shared atomic
// compiles to a compare-and-swap spin loop (SASS ATOMS.CAST.SPIN.64), which collapses when the lanes of a warp hit
// the same few group slots.  Readers only look at the slots after a barrier, so the two halves need not move together.
__device__ __forceinline__ void smem_add_u64(long long* p, unsigned long long v) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(p);
    const uint32_t lo = (uint32_t)v;
    uint32_t hi = (uint32_t)(v >> 32);
    if (lo) {
        uint32_t old;
        asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(s), "r"(lo) : "memory");
        hi += (old + lo) < old ? 1u : 0u;
    }
    if (hi) asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(s + 4), "r"(hi) : "memory");
}
__device__ __forceinline__ void red_shared_add_u64(long long* p, unsigned long long v) {
    smem_add_u64(p, v);
}
__device__ __forceinline__ void acc_apply_shared(int32_t mode, long long* a0, long long* a1, long long slot, long long bits) {
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(a0 + slot);
    switch (mode) {
    case M_COUNT:
        smem_add_u64(a0 + slot, 1ull);
        break;
    case M_SUM_I64:
        smem_add_u64(a0 + slot, (unsigned long long)bits);
        break;
    case M_SUM_F64:
    case M_AVG:
        asm volatile("red.shared.add.f64 [%0], %1;" ::"r"(s0), "d"(__longlong_as_double(bits)) : "memory");
        break;
    case M_MIN_I64:
        asm volatile("red.shared.min.s64 [%0], %1;" ::"r"(s0), "l"(bits) : "memory");
        break;
    case M_MAX_I64:
        asm volatile("red.shared.max.s64 [%0], %1;" ::"r"(s0), "l"(bits) : "memory");
        break;
    case M_MIN_F64:
        asm volatile("red.shared.min.s64 [%0], %1;" ::"r"(s0), "l"(f64_sortable(__longlong_as_double(bits))) : "memory");
        break;
    case M_MAX_F64:
        asm volatile("red.shared.max.s64 [%0], %1;" ::"r"(s0), "l"(f64_sortable(__longlong_as_double(bits))) : "memory");
        break;
    default: // M_SUM_I128 needs the old value for the carry
        acc_apply(mode, a0, a1, slot, bits);
        break;
    }
}

template <bool SHARED = false, typename Loader>
__device__ __forceinline__ void agg_apply_row(const AggDev& a, const AccPtrs& p, long long slot, Loader& ld) {
    if (SHARED)
        red_shared_add_u64(p.cnt + slot, 1ull);
    else
        atomicAdd((unsigned long long*)p.cnt + slot, 1ull);
#pragma unroll 1
    for (int f = 0; f < a.num_fns; f++) {
        const AggFnDev& fn = a.fns[f];
        if (fn.mode == M_COUNT_STAR) continue;
        int64_t bits;
        const bool nul = eval_expr(fn.input, ld, bits);
        if (nul) continue;
        unsigned long long nadd = 1ull;
        if (fn.n_value_id >= 0) { // AVG_MERGE: the state row stands for `count` inputs
            int64_t c;
            nadd = ld.load(fn.n_value_id, c) ? 0ull : (unsigned long long)c;
            if (nadd == 0) continue;
        }
        if (SHARED) {
            acc_apply_shared(fn.mode, p.acc0[f], p.acc1[f], slot, bits);
            if (fn.track_n) red_shared_add_u64(p.accn[f] + slot, nadd);
        } else {
            acc_apply(fn.mode, p.acc0[f], p.acc1[f], slot, bits);
            if (fn.track_n) atomicAdd((unsigned long long*)p.accn[f] + slot, nadd);
        }
    }
}

__device__ __forceinline__ void acc_ptrs_global(const AggDev& a, AccPtrs& p) {
    p.cnt = a.cnt_star;
    for (int f = 0; f < SR_MAX_AGG_FNS; f++) {
        p.acc0[f] = a.fns[f].acc0;
        p.acc1[f] = a.fns[f].acc1;
        p.accn[f] = a.fns[f].accn;
    }
}

// shared-memory accumulators for a dense table: layout [cnt | per fn: acc0, acc1?, accn?]
__device__ __forceinline__ void acc_ptrs_smem(const AggDev& a, long long* smem, AccPtrs& p) {
    const long long cap = (long long)a.cap;
    long long* q = smem;
    p.cnt = q;
    q += cap;
    for (int f = 0; f < SR_MAX_AGG_FNS; f++) {
        p.acc0[f] = p.acc1[f] = p.accn[f] = nullptr;
        if (f < a.num_fns && a.fns[f].mode != M_COUNT_STAR) {
            p.acc0[f] = q;
            q += cap;
            if (a.fns[f].mode == M_SUM_I128) {
                p.acc1[f] = q;
                q += cap;
            }
            if (a.fns[f].track_n) {
                p.accn[f] = q;
                q += cap;
            }
        }
    }
}
__device__ __forceinline__ void acc_smem_init(const AggDev& a, const AccPtrs& p) {
    const long long cap = (long long)a.cap;
    for (long long i = threadIdx.x; i < cap; i += blockDim.x) {
        p.cnt[i] = 0;
        for (int f = 0; f < a.num_fns; f++) {
            if (p.acc0[f]) p.acc0[f][i] = acc_init_value(a.fns[f].mode);
            if (p.acc1[f]) p.acc1[f][i] = 0;
            if (p.accn[f]) p.accn[f][i] = 0;
        }
    }
}
__device__ __forceinline__ void acc_smem_flush(const AggDev& a, const AccPtrs& p) {
    const long long cap = (long long)a.cap;
    for (long long i = threadIdx.x; i < cap; i += blockDim.x) {
        const long long c = p.cnt[i];
        if (c == 0) continue;
        atomicAdd((unsigned long long*)a.cnt_star + i, (unsigned long long)c);
        for (int f = 0; f < a.num_fns; f++) {
            const AggFnDev& fn = a.fns[f];
            if (!p.acc0[f]) continue;
            acc_merge(fn.mode, fn.acc0, fn.acc1, i, p.acc0[f][i], p.acc1[f] ? p.acc1[f][i] : 0);
            if (p.accn[f] && p.accn[f][i]) atomicAdd((unsigned long long*)fn.accn + i, (unsigned long long)p.accn[f][i]);
        }
    }
}

constexpr int AGG_BLOCK = 256;
// the row-at-a-time push kernels wait on one DRAM access after the other (ncu: 55-60 % of the stall samples are
// long-scoreboard waits at the key / input loads), so their throughput is proportional to the warps in flight: cap the
// registers at 32 for full occupancy (the push is latency bound: fewer resident CTAs make it slower)
constexpr int AGG_MIN_BLOCKS = 8;

// standalone aggregate sink: one pass over a chunk.
//  SMEM: dense table accumulated in shared memory.  slots_out (optional): pass-1-only mode
//  (find slots, no update); slots_in (optional): pass-2 mode (slots precomputed).
template <bool SMEM>
__global__ void __launch_bounds__(AGG_BLOCK, AGG_MIN_BLOCKS) k_agg_push(const AggDev* __restrict__ ad, const __grid_constant__ VTab vt, int64_t n, long long* __restrict__ slots_out,
                                                         const long long* __restrict__ slots_in) {
    extern __shared__ long long s_acc[];
    const AggDev& a = *ad;
    AccPtrs p;
    if (SMEM) {
        acc_ptrs_smem(a, s_acc, p);
        acc_smem_init(a, p);
        __syncthreads();
    } else {
        acc_ptrs_global(a, p);
    }
    unsigned long long known_groups = (!a.dense && a.num_keys > 0) ? *(volatile unsigned long long*)a.ngroups : 0ull;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        ChunkLoader ld{vt, row};
        long long slot;
        if (slots_in) {
            slot = slots_in[row];
        } else if (a.dense || a.num_keys == 0) {
            slot = agg_find_slot(a, ld);
        } else {
            HKey key;
            agg_pack_key(a, ld, key);
            bool inserted;
            slot = agg_find_slot_key(a, key, inserted, known_groups);
            agg_count_new_groups(a, inserted, known_groups);
        }
        if (slots_out) {
            slots_out[row] = slot;
            continue;
        }
        if (slot >= 0) agg_apply_row<SMEM>(a, p, slot, ld);
    }
    if (SMEM) {
        __syncthreads();
        acc_smem_flush(a, p);
    }
}

// SELECTIVE_PREAGG (Aggregator::build_hash_map_with_selection + compute_batch_agg_states_with_selection,
// aggregate_streaming_sink_operator.cpp:173-210): a row whose group is already in the table is aggregated into it, a row
// whose group is not there creates NO group -- streaming_selection[row] = 1 sends it out as an intermediate row instead.
__device__ __forceinline__ long long agg_lookup_slot_key(const AggDev& a, const HKey& key) {
    if (hkey_is_empty(a, key)) return a.cnt_star[a.cap] != 0 ? (long long)a.cap : -1; // the special slot holds this key's group, if any
    unsigned long long s = hkey_hash(a, key) & a.mask;
    const unsigned long long sb = s & ~a.slice_mask;
    for (unsigned long long tries = 0; tries <= a.slice_mask; tries++) {
        const HKey cur = hkey_load(a, s);
        if (hkey_eq(a, cur, key)) return (long long)s;
        if (hkey_is_empty(a, cur)) return -1;
        s = sb | ((s + 1) & a.slice_mask);
    }
    return -1;
}
__global__ void __launch_bounds__(AGG_BLOCK, AGG_MIN_BLOCKS) k_agg_push_existing(const AggDev* __restrict__ ad, const __grid_constant__ VTab vt, int64_t n,
                                                                                  uint8_t* __restrict__ selection) {
    const AggDev& a = *ad;
    AccPtrs p;
    acc_ptrs_global(a, p);
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        ChunkLoader ld{vt, row};
        HKey key;
        agg_pack_key(a, ld, key);
        const long long slot = agg_lookup_slot_key(a, key);
        selection[row] = slot < 0 ? 1 : 0;
        if (slot >= 0) agg_apply_row<false>(a, p, slot, ld);
    }
}
// positions of the set selection bytes, in row order (prefix sums by cub)
__global__ void __launch_bounds__(256) k_selection_index(const uint8_t* __restrict__ selection, const uint32_t* __restrict__ pos, int64_t n, uint32_t* __restrict__ index) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (selection[i]) index[pos[i]] = (uint32_t)i;
}

// ---- radix-partitioned push (hash tables larger than one shared-memory slice, large batches): sr_agg_part.cuh,
// included at the end of the device section

// no GROUP BY: every thread keeps the single state in registers over its rows, a warp reduction and one atomic per
// warp follow at the end (update_batch_single_state).  Used by the standalone push and by the fragment's final pass --
// a per-row atomic on the one state serialises (global: in L2; shared: 64-bit shared atomics are CAS spin loops).
struct SingleAcc {
    long long cnt;
    long long acc[SR_MAX_AGG_FNS];
    long long accn[SR_MAX_AGG_FNS];
};
__device__ __forceinline__ void single_acc_init(const AggDev& a, SingleAcc& s) {
    s.cnt = 0;
    for (int f = 0; f < SR_MAX_AGG_FNS; f++) {
        s.acc[f] = f < a.num_fns ? acc_init_value(a.fns[f].mode) : 0;
        s.accn[f] = 0;
    }
}
template <typename Loader>
__device__ __forceinline__ void single_acc_row(const AggDev& a, SingleAcc& s, Loader& ld) {
    s.cnt++;
#pragma unroll 1
    for (int f = 0; f < a.num_fns; f++) {
        const AggFnDev& fn = a.fns[f];
        if (fn.mode == M_COUNT_STAR) continue;
        int64_t bits;
        if (eval_expr(fn.input, ld, bits)) continue;
        if (fn.n_value_id >= 0) { // AVG_MERGE
            int64_t c;
            if (ld.load(fn.n_value_id, c) || c == 0) continue;
            s.accn[f] += c;
        } else {
            s.accn[f]++;
        }
        switch (fn.mode) {
        case M_COUNT:
            s.acc[f]++;
            break;
        case M_SUM_I64:
            s.acc[f] = (long long)((unsigned long long)s.acc[f] + (unsigned long long)bits);
            break;
        case M_SUM_F64:
        case M_AVG:
            s.acc[f] = __double_as_longlong(__longlong_as_double(s.acc[f]) + __longlong_as_double(bits));
            break;
        case M_MIN_I64:
            s.acc[f] = min(s.acc[f], (long long)bits);
            break;
        case M_MAX_I64:
            s.acc[f] = max(s.acc[f], (long long)bits);
            break;
        case M_MIN_F64:
            s.acc[f] = min(s.acc[f], f64_sortable(__longlong_as_double(bits)));
            break;
        case M_MAX_F64:
            s.acc[f] = max(s.acc[f], f64_sortable(__longlong_as_double(bits)));
            break;
        default: // M_SUM_I128: apply directly (rare)
            acc_apply(fn.mode, fn.acc0, fn.acc1, 0, bits);
            break;
        }
    }
}
// all 32 lanes of every warp must call this (converged)
__device__ __forceinline__ void single_acc_flush(const AggDev& a, SingleAcc& s) {
    const long long cnt = warp_sum(s.cnt);
    if (lane_id() == 0 && cnt) atomicAdd((unsigned long long*)a.cnt_star, (unsigned long long)cnt);
#pragma unroll 1
    for (int f = 0; f < a.num_fns; f++) {
        const AggFnDev& fn = a.fns[f];
        if (fn.mode == M_COUNT_STAR) continue;
        long long v = s.acc[f];
        switch (fn.mode) {
        case M_SUM_F64:
        case M_AVG: {
            double d = __longlong_as_double(v);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(SR_FULL_MASK, d, o);
            v = __double_as_longlong(d);
            break;
        }
        case M_MIN_I64:
        case M_MIN_F64:
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(SR_FULL_MASK, v, o));
            break;
        case M_MAX_I64:
        case M_MAX_F64:
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(SR_FULL_MASK, v, o));
            break;
        case M_SUM_I128:
            v = 0;
            break;
        default:
            v = (long long)warp_sum((unsigned long long)v);
            break;
        }
        const long long nn = warp_sum(s.accn[f]);
        if (lane_id() == 0 && nn) {
            if (fn.mode != M_SUM_I128) acc_merge(fn.mode, fn.acc0, fn.acc1, 0, v, 0);
            if (fn.track_n) atomicAdd((unsigned long long*)fn.accn, (unsigned long long)nn);
        }
    }
}

__global__ void __launch_bounds__(AGG_BLOCK, AGG_MIN_BLOCKS) k_agg_push_single(const AggDev* __restrict__ ad, const __grid_constant__ VTab vt, int64_t n) {
    const AggDev& a = *ad;
    SingleAcc s;
    single_acc_init(a, s);
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        ChunkLoader ld{vt, row};
        single_acc_row(a, s, ld);
    }
    single_acc_flush(a, s);
}

__global__ void __launch_bounds__(256) k_fill_i64(long long* p, int64_t n, long long v) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void __launch_bounds__(256) k_copy_i64(long long* dst, const long long* src, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[i];
}

// move every occupied slot of `o` into `a` (growth) -- plain stores, slots are unique
__global__ void __launch_bounds__(256) k_agg_rehash(const AggDev* __restrict__ od, const AggDev* __restrict__ nd) {
    const AggDev& o = *od;
    const AggDev& a = *nd;
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s <= o.cap; s += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long t;
        if (s == o.cap) {
            if (o.cnt_star[s] == 0) continue;
            t = a.cap;
        } else {
            const HKey key = hkey_load(o, s);
            if (hkey_is_empty(o, key)) continue;
            t = hkey_hash(a, key) & a.mask;
            const unsigned long long tb = t & ~a.slice_mask;
            bool placed = false;
            for (unsigned long long tries = 0; tries <= a.slice_mask; tries++) {
                const HKey cur = hkey_claim(a, t, key);
                if (hkey_is_empty(a, cur)) {
                    placed = true;
                    break;
                }
                t = tb | ((t + 1) & a.slice_mask);
            }
            if (!placed) { // cannot happen when the new table is at least as large as the old one (a slice only splits)
                a.flags[0] = 1;
                continue;
            }
        }
        a.cnt_star[t] = o.cnt_star[s];
        for (int f = 0; f < a.num_fns; f++) {
            if (a.fns[f].acc0) a.fns[f].acc0[t] = o.fns[f].acc0[s];
            if (a.fns[f].acc1) a.fns[f].acc1[t] = o.fns[f].acc1[s];
            if (a.fns[f].accn) a.fns[f].accn[t] = o.fns[f].accn ? o.fns[f].accn[s] : o.cnt_star[s];
        }
    }
}

// merge every occupied slot of `o` (finished) into `a` (AggregateFunction::merge)
__global__ void __launch_bounds__(256) k_agg_merge(const AggDev* __restrict__ od, const AggDev* __restrict__ nd) {
    const AggDev& o = *od;
    const AggDev& a = *nd;
    const unsigned long long total = o.dense ? o.cap : o.cap + 1;
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < total; s += (unsigned long long)gridDim.x * blockDim.x) {
        const long long c = o.cnt_star[s];
        if (c == 0) continue;
        long long t;
        if (a.dense || a.num_keys == 0) {
            t = (long long)s;
        } else if (s == o.cap) {
            t = (long long)a.cap;
        } else {
            const HKey key = hkey_load(o, s);
            unsigned long long q = hkey_hash(a, key) & a.mask;
            const unsigned long long qb = q & ~a.slice_mask;
            t = -1;
            for (unsigned long long tries = 0; tries <= a.slice_mask; tries++) {
                HKey cur = hkey_load(a, q);
                if (hkey_is_empty(a, cur)) {
                    cur = hkey_claim(a, q, key);
                    if (hkey_is_empty(a, cur)) {
                        atomicAdd(a.ngroups, 1ull);
                        cur = key;
                    }
                }
                if (hkey_eq(a, cur, key)) {
                    t = (long long)q;
                    break;
                }
                q = qb | ((q + 1) & a.slice_mask);
            }
            if (t < 0) {
                a.flags[0] = 1;
                continue;
            }
        }
        atomicAdd((unsigned long long*)a.cnt_star + t, (unsigned long long)c);
        for (int f = 0; f < a.num_fns; f++) {
            const AggFnDev& fo = o.fns[f];
            const AggFnDev& fa = a.fns[f];
            if (fa.mode == M_COUNT_STAR) continue;
            const long long n = fo.track_n ? fo.accn[s] : c;
            if (n == 0) continue;
            acc_merge(fa.mode, fa.acc0, fa.acc1, t, fo.acc0[s], fo.acc1 ? fo.acc1[s] : 0);
            if (fa.track_n) atomicAdd((unsigned long long*)fa.accn + t, (unsigned long long)n);
        }
    }
}

// ---- output: ordered compaction of occupied slots -----------------------------------------
constexpr int EMIT_BLOCK = 256;

__device__ __forceinline__ bool agg_slot_occupied(const AggDev& a, unsigned long long s) {
    if (a.num_keys == 0) return true; // the single state always yields one row
    return a.cnt_star[s] != 0;
}

__global__ void __launch_bounds__(EMIT_BLOCK) k_agg_count(const AggDev* __restrict__ ad, unsigned long long total, uint32_t* __restrict__ block_counts) {
    __shared__ uint32_t s_cnt[EMIT_BLOCK / 32];
    const unsigned long long s = (unsigned long long)blockIdx.x * EMIT_BLOCK + threadIdx.x;
    uint32_t c = (s < total && agg_slot_occupied(*ad, s)) ? 1u : 0u;
    c = warp_sum(c);
    if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < EMIT_BLOCK / 32; w++) t += s_cnt[w];
        block_counts[blockIdx.x] = t;
    }
}

// ---------------------------------------------------------------------------------------
// COUNT(DISTINCT): fold the second-level set keyed (group keys, value) into the group states
// ---------------------------------------------------------------------------------------
// One occupied slot of the set = one distinct (group, value) pair.  The loader hands the PARENT's group-by values back
// out of the set's packed key (the set's first keys are the parent's keys, in order), so the parent's own slot lookup --
// dense index, hash probe or the single state -- finds the group.
struct DistinctKeyLoader {
    const AggDev& p;
    const AggDev& c;
    HKey key;
    __device__ __forceinline__ bool load(int id, int64_t& bits) const {
        bits = 0;
        for (int k = 0; k < p.num_keys; k++) {
            if (p.key_value_id[k] != id) continue;
            const int w = c.key_width[k];
            const unsigned long long m = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1);
            const unsigned long long raw = hkey_bits(key, c.key_shift[k]) & m;
            long long v = (long long)raw;
            if (w < 8 && c.key_type[k] != SR_TYPE_BOOLEAN) v = (long long)(raw << (64 - 8 * w)) >> (64 - 8 * w);
            bits = v;
            return c.key_nullable[k] && (hkey_bits(key, c.null_shift + k) & 1ull);
        }
        return false;
    }
};

__global__ void __launch_bounds__(256) k_agg_distinct_fold(const AggDev* __restrict__ cd, const AggDev* __restrict__ pd, int32_t f) {
    const AggDev& c = *cd;
    const AggDev& p = *pd;
    const int vk = c.num_keys - 1; // the value column is the set's last key
    for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s <= c.cap; s += (unsigned long long)gridDim.x * blockDim.x) {
        if (c.cnt_star[s] == 0) continue;
        DistinctKeyLoader ld{p, c, s == c.cap ? HKey{SR_AGG_EMPTY, SR_AGG_EMPTY} : hkey_load(c, s)};
        if (c.key_nullable[vk] && (hkey_bits(ld.key, c.null_shift + vk) & 1ull)) continue; // COUNT(DISTINCT) skips NULL
        const long long slot = agg_find_slot(p, ld);
        if (slot >= 0) atomicAdd((unsigned long long*)p.fns[f].acc0 + slot, 1ull);
    }
}

struct EmitCol {
    void* data;
    uint8_t* nulls;
    int32_t type;
    int32_t width;
};
struct EmitArgs {
    EmitCol keys[SR_MAX_GROUP_KEYS];
    EmitCol res[SR_MAX_AGG_FNS];
};

__device__ __forceinline__ void store_int_typed(void* dst, int32_t width, long long row, long long v) {
    switch (width) {
    case 1:
        ((int8_t*)dst)[row] = (int8_t)v;
        break;
    case 2:
        ((int16_t*)dst)[row] = (int16_t)v;
        break;
    case 4:
        ((int32_t*)dst)[row] = (int32_t)v;
        break;
    default:
        ((long long*)dst)[row] = v;
        break;
    }
}

// pass-through leg of the streaming (first-phase) aggregate: row i of the input becomes intermediate row i
// (Aggregator::output_chunk_by_streaming -> AggregateFunction::convert_to_serialize_format): SUM / MIN / MAX states are the
// evaluated input in the function's result type, COUNT states are 1 / 0, COUNT(*) is 1.
struct ConvertCol {
    void* data;
    uint8_t* nulls;
    int32_t width;
    int32_t type;
};
struct ConvertArgs {
    ConvertCol c[SR_MAX_AGG_FNS];
};
__global__ void __launch_bounds__(256) k_agg_convert_states(const AggDev* __restrict__ ad, const __grid_constant__ VTab vt, int64_t n, ConvertArgs ca) {
    const AggDev& a = *ad;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        ChunkLoader ld{vt, row};
#pragma unroll 1
        for (int f = 0; f < a.num_fns; f++) {
            const AggFnDev& fn = a.fns[f];
            const ConvertCol& c = ca.c[f];
            if (fn.mode == M_COUNT_STAR) {
                ((long long*)c.data)[row] = 1;
                continue;
            }
            int64_t bits;
            const bool nul = eval_expr(fn.input, ld, bits);
            if (fn.mode == M_COUNT) {
                ((long long*)c.data)[row] = nul ? 0 : 1;
                continue;
            }
            if (c.nulls) c.nulls[row] = nul ? 1 : 0;
            if (nul) bits = 0;
            if (fn.in_is_double) {
                if (c.type == SR_TYPE_FLOAT)
                    ((float*)c.data)[row] = (float)__longlong_as_double(bits);
                else
                    ((double*)c.data)[row] = __longlong_as_double(bits);
            } else {
                store_int_typed(c.data, c.width, row, bits);
            }
        }
    }
}

__global__ void __launch_bounds__(EMIT_BLOCK) k_agg_emit(const AggDev* __restrict__ ad, unsigned long long total, const uint64_t* __restrict__ block_offsets,
                                                          EmitArgs ea) {
    __shared__ uint32_t s_scan[EMIT_BLOCK / 32 + 1];
    const AggDev& a = *ad;
    const unsigned long long s = (unsigned long long)blockIdx.x * EMIT_BLOCK + threadIdx.x;
    const uint32_t occ = (s < total && agg_slot_occupied(a, s)) ? 1u : 0u;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<EMIT_BLOCK>(occ, s_scan, &tot);
    if (!occ) return;
    const long long o = (long long)(block_offsets[blockIdx.x] + ex);
    // keys
    if (a.dense) {
        unsigned long long rem = s;
        for (int k = 0; k < a.num_keys; k++) {
            const long long idx = (long long)(rem / (unsigned long long)a.dense_stride[k]);
            rem = rem % (unsigned long long)a.dense_stride[k];
            const bool nul = a.key_nullable[k] && idx == 0;
            const long long v = nul ? 0 : a.dense_min[k] + idx - (a.key_nullable[k] ? 1 : 0);
            store_int_typed(ea.keys[k].data, ea.keys[k].width, o, v);
            if (ea.keys[k].nulls) ea.keys[k].nulls[o] = nul ? 1 : 0;
        }
    } else if (a.num_keys > 0) {
        const HKey key = s == a.cap ? HKey{SR_AGG_EMPTY, SR_AGG_EMPTY} : hkey_load(a, s);
        for (int k = 0; k < a.num_keys; k++) {
            const int w = a.key_width[k];
            const unsigned long long m = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1);
            unsigned long long raw = hkey_bits(key, a.key_shift[k]) & m;
            long long v = (long long)raw;
            if (w < 8 && a.key_type[k] != SR_TYPE_BOOLEAN) v = (long long)(raw << (64 - 8 * w)) >> (64 - 8 * w); // sign extend
            const bool nul = a.key_nullable[k] && (hkey_bits(key, a.null_shift + k) & 1ull);
            store_int_typed(ea.keys[k].data, w, o, nul ? 0 : v);
            if (ea.keys[k].nulls) ea.keys[k].nulls[o] = nul ? 1 : 0;
        }
    }
    // results
    const long long c = a.cnt_star[s];
    for (int f = 0; f < a.num_fns; f++) {
        const AggFnDev& fn = a.fns[f];
        const EmitCol& ec = ea.res[f];
        const long long n = fn.mode == M_COUNT_STAR ? c : (fn.track_n ? fn.accn[s] : c);
        bool nul = false;
        switch (fn.mode) {
        case M_COUNT_STAR:
            ((long long*)ec.data)[o] = c;
            break;
        case M_COUNT:
            ((long long*)ec.data)[o] = fn.acc0[s];
            break;
        case M_SUM_I64:
            nul = n == 0;
            ((long long*)ec.data)[o] = nul ? 0 : fn.acc0[s];
            break;
        case M_SUM_I128:
            nul = n == 0;
            ((long long*)ec.data)[2 * o] = nul ? 0 : fn.acc0[s];
            ((long long*)ec.data)[2 * o + 1] = nul ? 0 : fn.acc1[s];
            break;
        case M_SUM_F64:
            nul = n == 0;
            ((double*)ec.data)[o] = nul ? 0.0 : __longlong_as_double(fn.acc0[s]);
            break;
        case M_AVG: // AvgAggregateFunction::finalize_to_column (avg.h:218-236): sum / count
            nul = n == 0;
            ((double*)ec.data)[o] = nul ? 0.0 : __longlong_as_double(fn.acc0[s]) / (double)n;
            break;
        case M_MIN_I64:
        case M_MAX_I64:
            nul = n == 0;
            store_int_typed(ec.data, ec.width, o, nul ? 0 : fn.acc0[s]);
            break;
        default: { // M_MIN_F64 / M_MAX_F64
            nul = n == 0;
            const double d = nul ? 0.0 : f64_unsortable(fn.acc0[s]);
            if (ec.type == SR_TYPE_FLOAT)
                ((float*)ec.data)[o] = (float)d;
            else
                ((double*)ec.data)[o] = d;
            break;
        }
        }
        if (ec.nulls) ec.nulls[o] = nul ? 1 : 0;
    }
}

} // namespace srd

#include "sr_agg_part.cuh"

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct sr_agg {
    sr_ctx* ctx = nullptr;
    sr_agg_desc desc;
    bool compiled = false;
    bool finished = false;
    VReg reg;
    srd::AggDev host; // host mirror of the device descriptor
    DevBuf dev;       // AggDev on device
    DevBuf hkeys, cnt_star, counters /* ngroups + flags */;
    DevBuf acc0[SR_MAX_AGG_FNS], acc1[SR_MAX_AGG_FNS], accn[SR_MAX_AGG_FNS];
    DevBuf slots_tmp;
    // radix-partitioned push (sr_agg_part.cuh): bucket histogram / bases / cursors, tile list, staged records, retry lists
    DevBuf part_cursor, part_tiles, part_rec[2], part_ovf, part_fail, part_fail64, part_fail64b;
    int64_t partitioned_pushes = 0;
    bool table_touched = false; // some kernel may have created groups since the table was allocated / reset
    Staged staged;
    int64_t ngroups_host = 0; // hash mode: groups after the last synchronising push
    size_t smem_bytes = 0;    // > 0: dense table accumulated in shared memory
    // output
    int64_t out_rows = -1;
    int64_t cursor = 0;
    DevBuf block_counts, block_offsets;
    ScanScratch scan_scratch;
    std::vector<DevBuf> out_bufs;      // device result columns (data, nulls) x (keys + fns)
    std::vector<PinnedBuf> host_bufs; // host-memory pull: page-locked, the D2H copies are plain DMA
    int32_t out_types[SR_MAX_GROUP_KEYS + SR_MAX_AGG_FNS];
    bool out_has_nulls[SR_MAX_GROUP_KEYS + SR_MAX_AGG_FNS];
    std::vector<DevBuf> conv_bufs; // sr_agg_convert_to_states: (data, nulls) per function
    DevBuf sel_flags, sel_pos, sel_index, sel_tmp; // sr_agg_push_selective: streaming selection, its prefix sums, the streamed rows
    std::vector<DevBuf> sel_bufs;                  //   compacted (data, nulls) per output column
    // COUNT(DISTINCT) functions: one (group keys, value) set each -- an aggregate of its own with no functions, fed the
    // same chunks; agg_finish_output folds it into acc0 of the function (which until then holds COUNT(value))
    sr_agg* distinct[SR_MAX_AGG_FNS] = {};
    bool has_distinct = false;
    bool distinct_folded = false;
    ~sr_agg() {
        for (sr_agg* c : distinct) delete c;
    }
};

static int32_t agg_result_type(const sr_agg_fn& f) {
    switch (f.kind) {
    case SR_AGG_COUNT:
    case SR_AGG_COUNT_STAR:
    case SR_AGG_COUNT_DISTINCT:
        return SR_TYPE_BIGINT;
    case SR_AGG_AVG:
    case SR_AGG_AVG_MERGE:
        return SR_TYPE_DOUBLE;
    case SR_AGG_SUM:
        if (srd::is_float_class(f.input_type)) return SR_TYPE_DOUBLE;
        if (srd::is_decimal(f.input_type)) return SR_TYPE_DECIMAL128;
        if (f.input_type == SR_TYPE_LARGEINT) return SR_TYPE_LARGEINT;
        return SR_TYPE_BIGINT;
    default:
        return f.input_type;
    }
}

static int32_t agg_validate_desc(sr_ctx* ctx, const sr_agg_desc* d) {
    if (d->num_group_keys < 0 || d->num_group_keys > SR_MAX_GROUP_KEYS) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "num_group_keys %d", d->num_group_keys);
    if (d->num_fns < 0 || d->num_fns > SR_MAX_AGG_FNS) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "num_fns %d", d->num_fns);
    for (int k = 0; k < d->num_group_keys; k++) {
        const int w = srd::type_width(d->group_types[k]);
        if (w == 0 || w > 8 || srd::is_float_class(d->group_types[k])) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "group key type %d", d->group_types[k]);
    }
    for (int f = 0; f < d->num_fns; f++) {
        const sr_agg_fn& fn = d->fns[f];
        if (fn.kind < SR_AGG_SUM || fn.kind > SR_AGG_COUNT_DISTINCT) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "aggregate kind %d", fn.kind);
        if (fn.kind == SR_AGG_COUNT_DISTINCT) {
            if (fn.input.num_nodes != 1 || fn.input.nodes[0].op != SR_EX_COL)
                return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) takes a column reference (fn %d)", f);
            if (srd::type_width(fn.input_type) > 8 || srd::is_float_class(fn.input_type))
                return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) on type %d (fn %d)", fn.input_type, f);
            if (d->num_group_keys + 1 > SR_MAX_GROUP_KEYS) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) with %d group keys", d->num_group_keys);
        }
        if (fn.kind != SR_AGG_COUNT_STAR && srd::type_width(fn.input_type) == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "aggregate input type %d", fn.input_type);
        if (fn.kind == SR_AGG_AVG && (srd::is_decimal(fn.input_type) || srd::type_width(fn.input_type) > 8))
            return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "AVG on decimal / largeint");
        if ((fn.kind == SR_AGG_MIN || fn.kind == SR_AGG_MAX) && srd::type_width(fn.input_type) > 8)
            return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "MIN/MAX on 128-bit values");
    }
    return SR_OK;
}

static int32_t agg_upload(sr_agg* a) {
    sr_ctx* ctx = a->ctx;
    SR_TRY(a->dev.reserve(ctx, sizeof(srd::AggDev)));
    SR_CUDA(ctx, cudaMemcpyAsync(a->dev.p, &a->host, sizeof(srd::AggDev), cudaMemcpyHostToDevice, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

// allocate + initialise state arrays for `cap` slots into the given buffers, wiring `h`
static int32_t agg_alloc_tables(sr_agg* a, srd::AggDev* h, uint64_t cap, DevBuf* hkeys, DevBuf* cnt, DevBuf* a0, DevBuf* a1, DevBuf* an) {
    sr_ctx* ctx = a->ctx;
    const bool hash = !h->dense && h->num_keys > 0;
    const uint64_t total = hash ? cap + 1 : cap;
    const int grid = std::min(grid_for((int64_t)total, 256), ctx->num_sms * 8);
    h->cap = cap;
    h->mask = cap - 1;
    h->limit = hash ? cap / 2 : ~0ull;
    if (hash) {
        int log2cap = 0;
        while ((1ull << log2cap) < cap) log2cap++;
        h->slice_log2 = std::min((int)srd::AGGP_SLICE_LOG2, log2cap);
        h->slice_mask = (1ull << h->slice_log2) - 1;
    } else {
        h->slice_log2 = 0;
        h->slice_mask = 0;
    }
    if (hash) {
        const uint64_t kwords = total * (h->wide ? 2 : 1);
        SR_TRY(hkeys->reserve(ctx, sizeof(uint64_t) * kwords));
        srd::k_fill_u64<<<grid, 256, 0, ctx->stream>>>(hkeys->as<unsigned long long>(), (int64_t)kwords, SR_AGG_EMPTY);
        SR_LAUNCH_CHECK(ctx);
        h->hkeys = hkeys->as<unsigned long long>();
    } else {
        h->hkeys = nullptr;
    }
    if (!hash) {
        // dense tables: ONE slab holds every state array back to back (cnt | per fn: acc0, acc1?, accn?), so that the
        // element-wise merge of the partial tables of several GPUs (sr_agg_dense_state + all-reduce) is one in-place
        // collective over one contiguous range per (operator, element type) instead of a cat / copy per array
        size_t words = 1;
        for (int f = 0; f < h->num_fns; f++)
            if (h->fns[f].mode != srd::M_COUNT_STAR) words += 1 + (h->fns[f].mode == srd::M_SUM_I128 ? 1 : 0) + (h->fns[f].track_n ? 1 : 0);
        SR_TRY(cnt->reserve(ctx, sizeof(int64_t) * total * words));
        SR_CUDA(ctx, cudaMemsetAsync(cnt->p, 0, sizeof(int64_t) * total * words, ctx->stream));
        long long* q = cnt->as<long long>();
        h->cnt_star = q;
        q += total;
        for (int f = 0; f < h->num_fns; f++) {
            srd::AggFnDev& fn = h->fns[f];
            fn.acc0 = fn.acc1 = fn.accn = nullptr;
            if (fn.mode == srd::M_COUNT_STAR) continue;
            fn.acc0 = q;
            q += total;
            if (srd::acc_init_value(fn.mode) != 0) {
                srd::k_fill_i64<<<grid, 256, 0, ctx->stream>>>(fn.acc0, (int64_t)total, srd::acc_init_value(fn.mode));
                SR_LAUNCH_CHECK(ctx);
            }
            if (fn.mode == srd::M_SUM_I128) {
                fn.acc1 = q;
                q += total;
            }
            if (fn.track_n) {
                fn.accn = q;
                q += total;
            }
        }
        return SR_OK;
    }
    SR_TRY(cnt->reserve(ctx, sizeof(int64_t) * total));
    SR_CUDA(ctx, cudaMemsetAsync(cnt->p, 0, sizeof(int64_t) * total, ctx->stream));
    h->cnt_star = cnt->as<long long>();
    for (int f = 0; f < h->num_fns; f++) {
        srd::AggFnDev& fn = h->fns[f];
        fn.acc0 = fn.acc1 = fn.accn = nullptr;
        if (fn.mode == srd::M_COUNT_STAR) continue;
        SR_TRY(a0[f].reserve(ctx, sizeof(int64_t) * total));
        srd::k_fill_i64<<<grid, 256, 0, ctx->stream>>>(a0[f].as<long long>(), (int64_t)total, srd::acc_init_value(fn.mode));
        SR_LAUNCH_CHECK(ctx);
        fn.acc0 = a0[f].as<long long>();
        if (fn.mode == srd::M_SUM_I128) {
            SR_TRY(a1[f].reserve(ctx, sizeof(int64_t) * total));
            SR_CUDA(ctx, cudaMemsetAsync(a1[f].p, 0, sizeof(int64_t) * total, ctx->stream));
            fn.acc1 = a1[f].as<long long>();
        }
        if (fn.track_n) {
            SR_TRY(an[f].reserve(ctx, sizeof(int64_t) * total));
            SR_CUDA(ctx, cudaMemsetAsync(an[f].p, 0, sizeof(int64_t) * total, ctx->stream));
            fn.accn = an[f].as<long long>();
        }
    }
    return SR_OK;
}

// bytes of table state one group slot owns (keys + COUNT(*) + every accumulator array)
static uint64_t agg_slot_bytes(const srd::AggDev& h) { return (uint64_t)srd::agg_slot_bytes_of(h); }

typedef int32_t (*agg_type_fn)(void* user, int32_t slot);
typedef bool (*agg_nullable_fn)(void* user, int32_t slot);

// compile the descriptor against the input's slot types (first push).
static int32_t agg_compile(sr_agg* a, slot_type_fn tf, agg_nullable_fn nf, void* user) {
    sr_ctx* ctx = a->ctx;
    const sr_agg_desc& d = a->desc;
    srd::AggDev& h = a->host;
    memset(&h, 0, sizeof(h));
    a->reg = VReg();
    h.num_keys = d.num_group_keys;
    h.num_fns = d.num_fns;
    int bits = 0;
    bool any_nullable = false;
    for (int k = 0; k < d.num_group_keys; k++) {
        const int32_t t = tf(user, d.group_slots[k]);
        if (t == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "group-by slot %d not in the input", d.group_slots[k]);
        if (srd::type_width(t) != srd::type_width(d.group_types[k]) || srd::is_float_class(t))
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "group-by slot %d: input type %d differs from group_types %d", d.group_slots[k], t, d.group_types[k]);
        const int id = a->reg.add(d.group_slots[k], t);
        if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
        h.key_value_id[k] = id;
        h.key_width[k] = srd::type_width(t);
        if (h.key_width[k] > 8) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "group-by slot %d: 128-bit group keys are not supported", d.group_slots[k]);
        h.key_type[k] = d.group_types[k];
        h.key_nullable[k] = (d.group_nullable[k] || nf(user, d.group_slots[k])) ? 1 : 0;
        any_nullable |= h.key_nullable[k] != 0;
    }
    // pack widest first: every column then starts at a multiple of its own width and never straddles the (lo, hi) words
    for (int w = 8; w >= 1; w >>= 1)
        for (int k = 0; k < d.num_group_keys; k++) {
            if (h.key_width[k] != w) continue;
            if (bits < 64 && bits + 8 * w > 64) bits = 64;
            h.key_shift[k] = bits;
            bits += 8 * w;
        }
    if (any_nullable && bits < 64 && bits + 8 > 64) bits = 64;
    h.null_shift = bits;
    h.key_bytes = bits / 8 + (any_nullable ? 1 : 0);
    h.wide = h.key_bytes > 8 ? 1 : 0;
    for (int f = 0; f < d.num_fns; f++) {
        const sr_agg_fn& fn = d.fns[f];
        srd::AggFnDev& fd = h.fns[f];
        fd.kind = fn.kind;
        fd.result_type = agg_result_type(fn);
        fd.track_n = 0;
        fd.n_value_id = -1;
        if (fn.kind == SR_AGG_COUNT_STAR) {
            fd.mode = srd::M_COUNT_STAR;
            continue;
        }
        SR_TRY(compile_expr(ctx, &fn.input, &a->reg, tf, user, &fd.input));
        fd.in_is_double = fd.input.result_is_double;
        // is any input column of the expression nullable?
        bool nullable_in = false;
        for (int k = 0; k < fn.input.num_nodes; k++)
            if (fn.input.nodes[k].op == SR_EX_COL) nullable_in |= nf(user, fn.input.nodes[k].slot_id);
        fd.track_n = nullable_in ? 1 : 0;
        const bool dbl = fd.in_is_double != 0;
        switch (fn.kind) {
        case SR_AGG_COUNT:
        case SR_AGG_COUNT_DISTINCT: // COUNT(value) while rows arrive; replaced by the folded set at sink_finish
            fd.mode = srd::M_COUNT;
            fd.track_n = 0;
            break;
        case SR_AGG_SUM:
            if (dbl)
                fd.mode = srd::M_SUM_F64;
            else
                fd.mode = (fd.result_type == SR_TYPE_DECIMAL128 || fd.result_type == SR_TYPE_LARGEINT) ? srd::M_SUM_I128 : srd::M_SUM_I64;
            if (!dbl && srd::is_float_class(fn.input_type)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fn %d: input_type is floating but the expression is integer", f);
            if (dbl && !srd::is_float_class(fn.input_type)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fn %d: input_type is integer but the expression is double", f);
            break;
        case SR_AGG_AVG:
            fd.mode = srd::M_AVG;
            if (!dbl) { // AvgAggregateState<double>: integer inputs are accumulated as double (avg.h:62-66)
                if (fd.input.num_nodes >= SR_MAX_EXPR_NODES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "expression too long");
                fd.input.nodes[fd.input.num_nodes].op = srd::C_I2D;
                fd.input.num_nodes++;
                fd.input.form = srd::F_GENERIC; // no longer the shape compile_expr recognised
                fd.input.result_is_double = 1;
            }
            break;
        case SR_AGG_AVG_MERGE: { // merge phase of AVG: acc0 += sum state, accn += count state (AvgAggregateFunction::merge, avg.h:105-118)
            if (!dbl) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fn %d: AVG_MERGE needs a DOUBLE sum state", f);
            const int32_t ct = tf(user, fn.reserved);
            if (ct == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fn %d: AVG_MERGE count state slot %d is not in the chunk", f, fn.reserved);
            if (srd::is_float_class(ct) || srd::type_width(ct) > 8) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fn %d: AVG_MERGE count state must be an integer column", f);
            const int id = a->reg.add(fn.reserved, ct);
            if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
            fd.mode = srd::M_AVG;
            fd.n_value_id = id;
            fd.track_n = 1;
            break;
        }
        case SR_AGG_MIN:
            fd.mode = dbl ? srd::M_MIN_F64 : srd::M_MIN_I64;
            break;
        default:
            fd.mode = dbl ? srd::M_MAX_F64 : srd::M_MAX_I64;
            break;
        }
    }
    // slot space
    h.dense = 0;
    uint64_t cap = 1;
    if (d.num_group_keys == 0) {
        h.dense = 1;
        cap = 1;
    } else if (d.has_ranges) {
        unsigned __int128 prod = 1;
        bool ok = true;
        for (int k = 0; k < d.num_group_keys; k++) {
            if (d.group_max[k] < d.group_min[k]) ok = false;
            const unsigned __int128 ext = (unsigned __int128)((__int128)d.group_max[k] - d.group_min[k]) + 1 + (h.key_nullable[k] ? 1 : 0);
            prod *= ext;
            if (prod > ((unsigned __int128)1 << 22)) ok = false;
            if (!ok) break;
        }
        if (ok) {
            h.dense = 1;
            cap = (uint64_t)prod;
            uint64_t stride = cap;
            for (int k = 0; k < d.num_group_keys; k++) {
                h.dense_min[k] = d.group_min[k];
                h.dense_extent[k] = d.group_max[k] - d.group_min[k] + 1 + (h.key_nullable[k] ? 1 : 0);
                stride /= (uint64_t)h.dense_extent[k];
                h.dense_stride[k] = (long long)stride;
            }
        }
    }
    if (!h.dense) {
        if (h.key_bytes > 16) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "packed group-by key of %d bytes (> 16) without usable ranges", h.key_bytes);
        cap = 1ull << 21;
        const uint64_t want = d.expected_groups > 0 ? (uint64_t)d.expected_groups * 2 : 0; // load <= 1/2: a probe sequence stays in its 256-slot slice
        while (cap < want) cap <<= 1;
    }
    SR_TRY(a->counters.reserve(ctx, 64));
    SR_CUDA(ctx, cudaMemsetAsync(a->counters.p, 0, 64, ctx->stream));
    h.ngroups = a->counters.as<unsigned long long>();
    h.flags = (int32_t*)(a->counters.as<unsigned long long>() + 1);
    SR_TRY(agg_alloc_tables(a, &h, cap, &a->hkeys, &a->cnt_star, a->acc0, a->acc1, a->accn));
    // shared-memory accumulation for small dense tables -- including the single state of a query without GROUP BY
    // inside a fused fragment (every surviving row would otherwise hit the same global address with an atomic; the
    // standalone push reduces per warp instead, k_agg_push_single)
    a->smem_bytes = 0;
    if (h.dense) {
        size_t words = 1;
        for (int f = 0; f < h.num_fns; f++) {
            if (h.fns[f].mode == srd::M_COUNT_STAR) continue;
            words += 1 + (h.fns[f].mode == srd::M_SUM_I128 ? 1 : 0) + (h.fns[f].track_n ? 1 : 0);
        }
        const size_t bytes = words * cap * sizeof(int64_t);
        if (bytes <= 40 * 1024) a->smem_bytes = bytes;
    }
    SR_TRY(agg_upload(a));
    a->compiled = true;
    // COUNT(DISTINCT value): the (group keys, value) set, an aggregate without functions over the same input
    for (int f = 0; f < d.num_fns; f++) {
        if (d.fns[f].kind != SR_AGG_COUNT_DISTINCT) continue;
        a->has_distinct = true;
        if (a->distinct[f]) continue; // recompiled after a reset: the set keeps its tables
        sr_agg* c = new sr_agg();
        a->distinct[f] = c;
        c->ctx = ctx;
        memset(&c->desc, 0, sizeof(c->desc));
        c->desc.num_group_keys = d.num_group_keys + 1;
        for (int k = 0; k < d.num_group_keys; k++) {
            c->desc.group_slots[k] = d.group_slots[k];
            c->desc.group_types[k] = d.group_types[k];
            c->desc.group_nullable[k] = d.group_nullable[k];
        }
        c->desc.group_slots[d.num_group_keys] = d.fns[f].input.nodes[0].slot_id;
        c->desc.group_types[d.num_group_keys] = d.fns[f].input_type;
        c->desc.expected_groups = d.expected_groups;
        SR_TRY(agg_compile(c, tf, nf, user));
    }
    return SR_OK;
}

static int32_t agg_grow(sr_agg* a, uint64_t new_cap) {
    sr_ctx* ctx = a->ctx;
    srd::AggDev nh = a->host;
    DevBuf nk, nc, n0[SR_MAX_AGG_FNS], n1[SR_MAX_AGG_FNS], nn[SR_MAX_AGG_FNS], ndev;
    SR_TRY(agg_alloc_tables(a, &nh, new_cap, &nk, &nc, n0, n1, nn));
    SR_TRY(ndev.reserve(ctx, sizeof(srd::AggDev)));
    SR_CUDA(ctx, cudaMemcpyAsync(ndev.p, &nh, sizeof(srd::AggDev), cudaMemcpyHostToDevice, ctx->stream));
    const int grid = std::min(grid_for((int64_t)a->host.cap + 1, 256), ctx->num_sms * 16);
    srd::k_agg_rehash<<<grid, 256, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, (const srd::AggDev*)ndev.p);
    SR_LAUNCH_CHECK(ctx);
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::swap(a->hkeys, nk);
    std::swap(a->cnt_star, nc);
    for (int f = 0; f < SR_MAX_AGG_FNS; f++) {
        std::swap(a->acc0[f], n0[f]);
        std::swap(a->acc1[f], n1[f]);
        std::swap(a->accn[f], nn[f]);
    }
    a->host = nh;
    return agg_upload(a);
}

// read ngroups + flags (synchronises)
static int32_t agg_read_counters(sr_agg* a, uint64_t* ngroups, int32_t* overflow, int32_t* bad_range) {
    sr_ctx* ctx = a->ctx;
    SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned + 8, a->counters.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *ngroups = ctx->pinned[8];
    const int32_t* fl = (const int32_t*)(ctx->pinned + 9);
    *overflow = fl[0];
    *bad_range = fl[1];
    return SR_OK;
}

static bool staged_slot_nullable(void* user, int32_t slot) {
    const Staged* st = (const Staged*)user;
    const int k = st->find(slot);
    return k >= 0 && st->cols[k].nulls != nullptr;
}

static int32_t agg_check_nullability(sr_agg* a, const VTab& vt) {
    // a column that was non-nullable at compile time must stay so (its null-tracking state was elided)
    const srd::AggDev& h = a->host;
    for (int k = 0; k < h.num_keys; k++)
        if (!h.key_nullable[k] && vt.v[h.key_value_id[k]].nulls)
            return sr_fail(a->ctx, SR_ERR_INVALID_ARGUMENT, "group-by slot %d became nullable; declare it in group_nullable", a->desc.group_slots[k]);
    for (int f = 0; f < h.num_fns; f++) {
        const srd::AggFnDev& fn = h.fns[f];
        if (fn.mode == srd::M_COUNT_STAR || fn.mode == srd::M_COUNT || fn.track_n) continue;
        for (int k = 0; k < fn.input.num_nodes; k++)
            if ((fn.input.nodes[k].op == srd::C_LOAD_I || fn.input.nodes[k].op == srd::C_LOAD_D) && vt.v[fn.input.nodes[k].arg].nulls) {
                // start tracking the non-null count: accn := cnt_star so far
                srd::AggFnDev& hf = a->host.fns[f];
                const uint64_t total = (!h.dense && h.num_keys > 0) ? h.cap + 1 : h.cap;
                SR_TRY(a->accn[f].reserve(a->ctx, sizeof(int64_t) * total));
                srd::k_copy_i64<<<std::min(grid_for((int64_t)total, 256), a->ctx->num_sms * 8), 256, 0, a->ctx->stream>>>(
                        a->accn[f].as<long long>(), a->host.cnt_star, (int64_t)total);
                SR_LAUNCH_CHECK(a->ctx);
                hf.accn = a->accn[f].as<long long>();
                hf.track_n = 1;
                a->smem_bytes = 0; // layout changed; fall back to global accumulation
                SR_TRY(agg_upload(a));
                break;
            }
    }
    return SR_OK;
}

#include "sr_agg_part_host.cuh"

static int32_t agg_push_vtab(sr_agg* a, const VTab& vt, int64_t n) {
    sr_ctx* ctx = a->ctx;
    if (n <= 0) return SR_OK;
    SR_TRY(agg_check_nullability(a, vt));
    const bool fresh = !a->table_touched; // no kernel has created a group since the table was allocated / reset
    a->table_touched = true;
    const srd::AggDev& h = a->host;
    const srd::AggDev* dev = (const srd::AggDev*)a->dev.p;
    const int grid = std::min(grid_for(n, srd::AGG_BLOCK), ctx->num_sms * 8);
    if (h.num_keys == 0) {
        srd::k_agg_push_single<<<grid, srd::AGG_BLOCK, 0, ctx->stream>>>(dev, vt, n);
        SR_LAUNCH_CHECK(ctx);
        return SR_OK;
    }
    if (h.dense) {
        if (a->smem_bytes > 0) {
            srd::k_agg_push<true><<<grid, srd::AGG_BLOCK, a->smem_bytes, ctx->stream>>>(dev, vt, n, nullptr, nullptr);
        } else {
            srd::k_agg_push<false><<<grid, srd::AGG_BLOCK, 0, ctx->stream>>>(dev, vt, n, nullptr, nullptr);
        }
        SR_LAUNCH_CHECK(ctx);
        return SR_OK;
    }
    // hash mode
    {
        // tuning knobs (also let the tests reach the partitioned path with small inputs)
        const char* e_rows = getenv("SR_AGG_PARTITION_MIN_ROWS");
        const char* e_table = getenv("SR_AGG_PARTITION_MIN_TABLE_BYTES");
        const int64_t min_rows = e_rows ? atoll(e_rows) : kPartitionedMinRows;
        (void)e_table;
        bool merge_fns = false; // the staged records of the partitioned push carry one value per function, not (sum, count)
        for (int f = 0; f < h.num_fns; f++) merge_fns |= h.fns[f].n_value_id >= 0;
        if (!merge_fns && n >= min_rows) return agg_push_partitioned(a, vt, n, fresh);
    }
    if ((uint64_t)a->ngroups_host + (uint64_t)n <= h.limit) {
        // cannot overflow: single fused pass
        srd::k_agg_push<false><<<grid, srd::AGG_BLOCK, 0, ctx->stream>>>(dev, vt, n, nullptr, nullptr);
        SR_LAUNCH_CHECK(ctx);
    } else {
        // two passes: find/insert slots (growing the table until every row is placed), then update
        SR_TRY(a->slots_tmp.reserve(ctx, sizeof(int64_t) * (size_t)n));
        while (true) {
            srd::k_agg_push<false><<<grid, srd::AGG_BLOCK, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, vt, n, a->slots_tmp.as<long long>(), nullptr);
            SR_LAUNCH_CHECK(ctx);
            uint64_t ng;
            int32_t ovf, bad;
            SR_TRY(agg_read_counters(a, &ng, &ovf, &bad));
            a->ngroups_host = (int64_t)ng;
            if (!ovf) break;
            SR_CUDA(ctx, cudaMemsetAsync((uint8_t*)a->counters.p + 8, 0, 8, ctx->stream));
            SR_TRY(agg_grow(a, a->host.cap * 4));
        }
        srd::k_agg_push<false><<<grid, srd::AGG_BLOCK, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, vt, n, nullptr, a->slots_tmp.as<long long>());
        SR_LAUNCH_CHECK(ctx);
        return SR_OK;
    }
    uint64_t ng;
    int32_t ovf, bad;
    SR_TRY(agg_read_counters(a, &ng, &ovf, &bad));
    a->ngroups_host = (int64_t)ng;
    if (ovf) return sr_fail(ctx, SR_ERR_STATE, "aggregate hash table overflow (internal)");
    return SR_OK;
}

static int32_t agg_finish_output(sr_agg* a) {
    sr_ctx* ctx = a->ctx;
    if (a->out_rows >= 0) return SR_OK;
    const sr_agg_desc& d = a->desc;
    if (!a->compiled) {
        // no input was ever pushed: GROUP BY -> zero rows; no GROUP BY -> one row of empty states
        if (d.num_group_keys > 0) {
            a->out_rows = 0;
            return SR_OK;
        }
        Staged empty;
        struct Tf {
            static int32_t f(void* u, int32_t slot) {
                // expressions over an empty input: take the declared input_type of the first fn that uses the slot
                const sr_agg_desc* dd = (const sr_agg_desc*)u;
                for (int q = 0; q < dd->num_fns; q++)
                    for (int k = 0; k < dd->fns[q].input.num_nodes; k++)
                        if (dd->fns[q].input.nodes[k].op == SR_EX_COL && dd->fns[q].input.nodes[k].slot_id == slot) return dd->fns[q].input_type;
                return 0;
            }
            static bool n(void*, int32_t) { return true; }
        };
        SR_TRY(agg_compile(a, Tf::f, Tf::n, (void*)&a->desc));
    }
    const srd::AggDev& h = a->host;
    const uint64_t total = (!h.dense && h.num_keys > 0) ? h.cap + 1 : h.cap;
    if (a->has_distinct && !a->distinct_folded) {
        for (int f = 0; f < d.num_fns; f++) {
            sr_agg* c = a->distinct[f];
            if (!c) continue;
            // acc0 held COUNT(value) so far (the state every push path maintains); from here on the distinct count
            SR_CUDA(ctx, cudaMemsetAsync(h.fns[f].acc0, 0, sizeof(int64_t) * total, ctx->stream));
            if (!c->compiled) continue;
            srd::k_agg_distinct_fold<<<std::min(grid_for((int64_t)c->host.cap + 1, 256), ctx->num_sms * 16), 256, 0, ctx->stream>>>(
                    (const srd::AggDev*)c->dev.p, (const srd::AggDev*)a->dev.p, f);
            SR_LAUNCH_CHECK(ctx);
        }
        a->distinct_folded = true;
    }
    const int blocks = grid_for((int64_t)total, srd::EMIT_BLOCK);
    SR_TRY(a->block_counts.reserve(ctx, sizeof(uint32_t) * (size_t)blocks));
    SR_TRY(a->block_offsets.reserve(ctx, sizeof(uint64_t) * (size_t)blocks));
    srd::k_agg_count<<<blocks, srd::EMIT_BLOCK, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, total, a->block_counts.as<uint32_t>());
    SR_LAUNCH_CHECK(ctx);
    SR_TRY(scan_counts(ctx, &a->scan_scratch, a->block_counts.as<uint32_t>(), blocks, a->block_offsets.as<uint64_t>()));
    // one read-back, one synchronisation: the row count and the table's status counters together
    SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned, ctx->dscratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned + 8, a->counters.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    {
        const int32_t* fl = (const int32_t*)(ctx->pinned + 9);
        if (fl[1]) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "a group-by value fell outside the declared group_min/group_max range");
        if (fl[0]) return sr_fail(ctx, SR_ERR_STATE, "aggregate hash table overflow (internal)");
    }
    const int64_t rows = (int64_t)ctx->pinned[0];
    const int nc = d.num_group_keys + d.num_fns;
    // output buffers are kept across finish/reset cycles (they only grow): a repeated query pays no cudaMalloc/cudaFree
    if (a->out_bufs.size() < 2 * (size_t)nc) {
        std::vector<DevBuf> nb(2 * (size_t)nc);
        for (size_t i = 0; i < a->out_bufs.size(); i++) std::swap(nb[i], a->out_bufs[i]);
        a->out_bufs.swap(nb);
    }
    srd::EmitArgs ea;
    memset(&ea, 0, sizeof(ea));
    for (int k = 0; k < nc; k++) {
        int32_t type;
        bool nullable;
        if (k < d.num_group_keys) {
            type = d.group_types[k];
            nullable = h.key_nullable[k] != 0;
        } else {
            const srd::AggFnDev& fn = h.fns[k - d.num_group_keys];
            type = fn.result_type;
            nullable = !(fn.mode == srd::M_COUNT || fn.mode == srd::M_COUNT_STAR);
        }
        const int w = srd::type_width(type);
        SR_TRY(a->out_bufs[2 * k].reserve(ctx, (size_t)std::max<int64_t>(rows, 1) * w));
        if (nullable) SR_TRY(a->out_bufs[2 * k + 1].reserve(ctx, (size_t)std::max<int64_t>(rows, 1)));
        srd::EmitCol ec;
        ec.data = a->out_bufs[2 * k].p;
        ec.nulls = nullable ? (uint8_t*)a->out_bufs[2 * k + 1].p : nullptr;
        ec.type = type;
        ec.width = w;
        if (k < d.num_group_keys)
            ea.keys[k] = ec;
        else
            ea.res[k - d.num_group_keys] = ec;
        a->out_types[k] = type;
        a->out_has_nulls[k] = nullable;
    }
    if (rows > 0) {
        srd::k_agg_emit<<<blocks, srd::EMIT_BLOCK, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, total, a->block_offsets.as<uint64_t>(), ea);
        SR_LAUNCH_CHECK(ctx);
    }
    a->out_rows = rows;
    a->cursor = 0;
    return SR_OK;
}
