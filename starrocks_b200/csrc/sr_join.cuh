// sr_join.cuh -- hash join build + probe on the device.
// Replaces K5-K12 of SURVEY.md section 2b:
//   JoinKeyHash / calc_bucket_num           be/src/exec/join/join_hash_map_helper.h:35-54,79-84
//   *JoinHashMap::construct_hash_table      be/src/exec/join/join_hash_map_method.hpp:37-86,133-300,542-674
//   *JoinHashMap::lookup_init               :87-126,300-370,592-618,676-706
//   JoinHashMap::_probe_from_ht (+outer/semi/anti) be/src/exec/join/join_hash_map.hpp:718-795,950-1030,1186-1255
//   _probe_output / _build_output           :163-269
//   JoinHashTable::append_chunk             be/src/exec/join/join_hash_table.cpp:712-752
//
// Device layout (GPU-first, not the CPU layout):
//  * build columns are concatenated in HBM with row 0 reserved as the sentinel (same 1-based
//    build index convention as the reference, so index pairs are comparable);
//  * DIRECT / RANGE_DIRECT_MAPPING: first[key - min] (uint32 head row) + next[] chain, built
//    with one atomicExch per row; plus a 1-bit-per-key bitmap (the RANGE_DIRECT_MAPPING_SET
//    idea) that the fused fragment kernel keeps in shared memory / L1;
//  * LINEAR_CHAINED: open addressing over {key(int64), head(uint32)} slots with linear
//    probing, equal keys chained through next[] (AreKeysInChainIdentical), claimed by
//    atomicCAS on the key word; the multiplicative JoinKeyHash picks the start slot.
#pragma once

#include <cub/device/device_scan.cuh>       // prefix sums of the other-join-conjunct emit flags
#include <thrust/iterator/transform_iterator.h>
#include <cub/device/device_radix_sort.cuh> // stable (bucket, row) sort for the deterministic-chain pass of the build (cold path)

#include "sr_scan.cuh"

namespace srd {

#define SR_HKEY_EMPTY ((int64_t)0x8000000000000000ll)

struct JoinDev {
    int32_t method;
    int32_t has_dup;
    int64_t min_value, max_value;
    const uint32_t* first;
    const uint32_t* next;
    const unsigned long long* hkeys; // LINEAR_CHAINED: cap + 1 slots (last = key == EMPTY)
    uint32_t hmask;
    uint32_t hlog;
    const uint32_t* bitmap; // range methods: bit (key - min) set when a build row has the key
    // packed keys of 9..16 bytes (SERIALIZED_FIXED_SIZE_LARGEINT, join_hash_table.cpp:221-222): the table is keyed by a
    // 64-bit FINGERPRINT of the 128-bit key -- a chain then holds every build row with that fingerprint, and every walk
    // compares the full key of each entry (wide_lo / wide_hi, one pair per build row) with the probe row's
    int32_t wide;
    int32_t pad;
    const unsigned long long* wide_lo;
    const unsigned long long* wide_hi;
};

struct WideKey {
    unsigned long long lo, hi;
};
__device__ __forceinline__ int64_t wide_fingerprint(const WideKey& k) {
    unsigned long long x = k.lo ^ (k.hi * 0x9E3779B97F4A7C15ull + 0x632BE59BD9B4E019ull);
    x ^= x >> 32;
    x *= 0xD6E8FEB86659FD93ull;
    x ^= x >> 32;
    return (int64_t)x;
}
__device__ __forceinline__ bool wide_equal(const JoinDev& j, uint32_t b, const WideKey& k) {
    return __ldg(j.wide_lo + b) == k.lo && __ldg(j.wide_hi + b) == k.hi;
}

struct KeyCols {
    DCol c[SR_MAX_JOIN_KEYS];
    int32_t n;
    int32_t pad;
};

// pack the key columns of one row; returns true when any key column is NULL
__device__ __forceinline__ bool pack_key(const KeyCols& kc, int64_t row, int64_t& key) {
    if (kc.n == 1) {
        key = load_int(kc.c[0].data, kc.c[0].type, row);
        return kc.c[0].nulls != nullptr && kc.c[0].nulls[row] != 0;
    }
    uint64_t k = 0;
    int shift = 0;
    bool nul = false;
#pragma unroll
    for (int q = 0; q < SR_MAX_JOIN_KEYS; q++) {
        if (q < kc.n) {
            const int w = kc.c[q].width;
            const uint64_t mask = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1);
            k |= ((uint64_t)load_int(kc.c[q].data, kc.c[q].type, row) & mask) << shift;
            shift += 8 * w;
            nul |= kc.c[q].nulls != nullptr && kc.c[q].nulls[row] != 0;
        }
    }
    key = (int64_t)k;
    return nul;
}

// the same for packed keys of 9..16 bytes: little-endian concatenation of the columns into 128 bits
__device__ __forceinline__ bool pack_key_wide(const KeyCols& kc, int64_t row, WideKey& key) {
    key.lo = key.hi = 0;
    int shift = 0;
    bool nul = false;
#pragma unroll
    for (int q = 0; q < SR_MAX_JOIN_KEYS; q++) {
        if (q < kc.n) {
            const int w = kc.c[q].width;
            const unsigned long long mask = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1);
            const unsigned long long v = (unsigned long long)load_int(kc.c[q].data, kc.c[q].type, row) & mask;
            if (shift < 64) {
                key.lo |= v << shift;
                if (shift + 8 * w > 64) key.hi |= v >> (64 - shift);
            } else {
                key.hi |= v << (shift - 64);
            }
            shift += 8 * w;
            nul |= kc.c[q].nulls != nullptr && kc.c[q].nulls[row] != 0;
        }
    }
    return nul;
}

__device__ __forceinline__ uint32_t hash_slot(int64_t key, uint32_t hlog) {
    return join_key_hash64((uint64_t)key, hlog);
}

// head build row of `key` (0 = no match)
__device__ __forceinline__ uint32_t join_lookup(const JoinDev& j, int64_t key) {
    if (j.method == SR_JOIN_METHOD_LINEAR_CHAINED) {
        if (key == SR_HKEY_EMPTY) return __ldg(j.first + j.hmask + 1);
        uint32_t s = hash_slot(key, j.hlog);
        while (true) {
            const int64_t k = (int64_t)__ldg(j.hkeys + s);
            if (k == key) return __ldg(j.first + s);
            if (k == SR_HKEY_EMPTY) return 0;
            s = (s + 1) & j.hmask;
        }
    }
    if (key < j.min_value || key > j.max_value) return 0;
    return __ldg(j.first + (uint64_t)(key - j.min_value));
}

// pack build keys (rows 1..n) and reduce min / max / null count
__global__ void __launch_bounds__(256) k_join_pack_keys(KeyCols kc, int64_t n_plus1, long long* __restrict__ keys, uint8_t* __restrict__ knulls,
                                                         long long* __restrict__ minmax /* [min, max, nulls] */, unsigned long long* __restrict__ wide_lo,
                                                         unsigned long long* __restrict__ wide_hi) {
    long long mn = 0x7fffffffffffffffll, mx = (long long)0x8000000000000000ll, nn = 0;
    for (int64_t i = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_plus1; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t key;
        bool nul;
        if (wide_lo) { // 9..16-byte key: the table key is its fingerprint
            WideKey wk;
            nul = pack_key_wide(kc, i, wk);
            wide_lo[i] = wk.lo;
            wide_hi[i] = wk.hi;
            key = wide_fingerprint(wk);
        } else {
            nul = pack_key(kc, i, key);
        }
        keys[i] = key;
        if (knulls) knulls[i] = nul ? 1 : 0;
        if (!nul) {
            mn = min(mn, (long long)key);
            mx = max(mx, (long long)key);
        } else {
            nn++;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = min(mn, __shfl_xor_sync(SR_FULL_MASK, mn, o));
        mx = max(mx, __shfl_xor_sync(SR_FULL_MASK, mx, o));
        nn += __shfl_xor_sync(SR_FULL_MASK, nn, o);
    }
    if (lane_id() == 0) {
        atomicMin(&minmax[0], mn);
        atomicMax(&minmax[1], mx);
        if (nn) atomicAdd((unsigned long long*)&minmax[2], (unsigned long long)nn);
    }
}

// K6/K8: next[i] = exchange(first[b], i)  (the reference's `next[i]=first[b]; first[b]=i`)
__global__ void __launch_bounds__(256) k_join_build_direct(const long long* __restrict__ keys, const uint8_t* __restrict__ knulls, int64_t n_plus1,
                                                            int64_t min_value, uint32_t* __restrict__ first, uint32_t* __restrict__ next,
                                                            uint32_t* __restrict__ bitmap, int32_t* __restrict__ has_dup) {
    for (int64_t i = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_plus1; i += (int64_t)gridDim.x * blockDim.x) {
        if (knulls && knulls[i]) continue;
        const uint64_t b = (uint64_t)(keys[i] - min_value);
        const uint32_t old = atomicExch(&first[b], (uint32_t)i);
        next[i] = old;
        if (old != 0)
            *has_dup = 1;
        else
            atomicOr(&bitmap[b >> 5], 1u << (b & 31));
    }
}

// K7 analogue: claim a slot for the key (atomicCAS on the key word), then push the row on the
// slot's chain.
__global__ void __launch_bounds__(256) k_join_build_hash(const long long* __restrict__ keys, const uint8_t* __restrict__ knulls, int64_t n_plus1,
                                                          unsigned long long* __restrict__ hkeys, uint32_t hmask, uint32_t hlog,
                                                          uint32_t* __restrict__ first, uint32_t* __restrict__ next, int32_t* __restrict__ has_dup) {
    for (int64_t i = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_plus1; i += (int64_t)gridDim.x * blockDim.x) {
        if (knulls && knulls[i]) continue;
        const int64_t key = keys[i];
        uint32_t s;
        if (key == SR_HKEY_EMPTY) {
            s = hmask + 1;
        } else {
            s = hash_slot(key, hlog);
            while (true) {
                const unsigned long long old = atomicCAS(&hkeys[s], (unsigned long long)SR_HKEY_EMPTY, (unsigned long long)key);
                if (old == (unsigned long long)SR_HKEY_EMPTY || old == (unsigned long long)key) break;
                s = (s + 1) & hmask;
            }
        }
        const uint32_t old = atomicExch(&first[s], (uint32_t)i);
        next[i] = old;
        if (old != 0) *has_dup = 1;
    }
}

// ---- deterministic chains -------------------------------------------------------------------------------------
// The parallel build links duplicate keys in arrival order.  The reference builds sequentially
// (`next[i] = first[b]; first[b] = i`, join_hash_map_method.hpp:37-86), so a chain lists its rows by DESCENDING
// build index and that is the order in which a probe row's matches are emitted.  When duplicates exist the chains are
// rebuilt to that order: bucket id per build row -> stable radix sort of (bucket, row) -> predecessor links.
__global__ void __launch_bounds__(256) k_join_bucket_ids(const long long* __restrict__ keys, const uint8_t* __restrict__ knulls, int64_t n_plus1, int32_t method,
                                                          int64_t min_value, const unsigned long long* __restrict__ hkeys, uint32_t hmask, uint32_t hlog,
                                                          uint32_t invalid, uint32_t* __restrict__ bucket, uint32_t* __restrict__ row) {
    for (int64_t i = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_plus1; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t b = invalid;
        if (!(knulls && knulls[i])) {
            const int64_t key = keys[i];
            if (method == SR_JOIN_METHOD_LINEAR_CHAINED) {
                if (key == SR_HKEY_EMPTY) {
                    b = hmask + 1;
                } else {
                    b = hash_slot(key, hlog);
                    while ((int64_t)hkeys[b] != key) b = (b + 1) & hmask; // the key was inserted by the build pass
                }
            } else {
                b = (uint32_t)(uint64_t)(key - min_value);
            }
        }
        bucket[i - 1] = b;
        row[i - 1] = (uint32_t)i;
    }
}
// sorted by (bucket, row): a row's predecessor in its bucket is its `next`, the last row of a bucket is the head
__global__ void __launch_bounds__(256) k_join_relink(const uint32_t* __restrict__ bucket, const uint32_t* __restrict__ row, int64_t n, uint32_t invalid,
                                                      uint32_t* __restrict__ first, uint32_t* __restrict__ next) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = bucket[p];
        if (b == invalid) continue;
        const uint32_t i = row[p];
        next[i] = (p > 0 && bucket[p - 1] == b) ? row[p - 1] : 0u;
        if (p + 1 == n || bucket[p + 1] != b) first[b] = i;
    }
}

__global__ void __launch_bounds__(256) k_fill_u64(unsigned long long* p, int64_t n, unsigned long long v) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// number of output rows a probe row produces for the join type, given its chain head.  `match` (joins with a POST_PROBE
// phase only): every build row of the chain is marked as matched (HashTableProbeState::build_match_index,
// join_hash_map.hpp:1352,1492 -- plain byte stores of 1, any number of probers may race on them).
__device__ __forceinline__ uint32_t probe_row_count(const JoinDev& j, int32_t join_type, uint32_t head, uint8_t* __restrict__ match = nullptr,
                                                    const WideKey* wk = nullptr) {
    uint32_t cnt = 0;
    if (wk) { // fingerprint chain: only the entries whose full key equals the probe row's count
        for (uint32_t b = head; b != 0; b = __ldg(j.next + b)) {
            if (wide_equal(j, b, *wk)) {
                cnt++;
                if (match) match[b] = 1;
            }
        }
    } else if (head != 0) {
        cnt = 1;
        if (match) match[head] = 1;
        if (j.has_dup) {
            uint32_t b = __ldg(j.next + head);
            while (b != 0) {
                cnt++;
                if (match) match[b] = 1;
                b = __ldg(j.next + b);
            }
        }
    }
    switch (join_type) {
    case SR_JOIN_INNER:
    case SR_JOIN_RIGHT_OUTER:
        return cnt;
    case SR_JOIN_LEFT_OUTER:
    case SR_JOIN_FULL_OUTER:
        return cnt ? cnt : 1;
    case SR_JOIN_LEFT_SEMI:
        return cnt ? 1 : 0;
    case SR_JOIN_RIGHT_SEMI:
    case SR_JOIN_RIGHT_ANTI:
        return 0;
    default:
        return cnt ? 0 : 1;
    }
}

// POST_PROBE: build rows 1..rows whose mark equals `want`, in build order (_search_ht_remain, join_hash_map.hpp:420-457)
constexpr int REMAIN_BLOCK = 256;
__global__ void __launch_bounds__(REMAIN_BLOCK) k_remain_count(const uint8_t* __restrict__ match, int64_t rows, uint8_t want, uint32_t* __restrict__ block_counts) {
    __shared__ uint32_t s_cnt[REMAIN_BLOCK / 32];
    const int64_t i = 1 + (int64_t)blockIdx.x * REMAIN_BLOCK + threadIdx.x;
    uint32_t c = (i <= rows && (match[i] != 0) == (want != 0)) ? 1u : 0u;
    c = warp_sum(c);
    if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < REMAIN_BLOCK / 32; w++) t += s_cnt[w];
        block_counts[blockIdx.x] = t;
    }
}
__global__ void __launch_bounds__(REMAIN_BLOCK) k_remain_write(const uint8_t* __restrict__ match, int64_t rows, uint8_t want, const uint64_t* __restrict__ block_offsets,
                                                                uint32_t* __restrict__ build_index) {
    __shared__ uint32_t s_scan[REMAIN_BLOCK / 32 + 1];
    const int64_t i = 1 + (int64_t)blockIdx.x * REMAIN_BLOCK + threadIdx.x;
    const uint32_t c = (i <= rows && (match[i] != 0) == (want != 0)) ? 1u : 0u;
    uint32_t tot;
    const uint32_t ex = block_excl_scan<REMAIN_BLOCK>(c, s_scan, &tot);
    if (c) build_index[block_offsets[blockIdx.x] + ex] = (uint32_t)i;
}
// a column of n NULLs (data zeroed: what Column::append_nulls leaves)
__global__ void __launch_bounds__(256) k_fill_u8(uint8_t* p, int64_t n, uint8_t v) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

constexpr int PROBE_BLOCK = 256;
constexpr int PROBE_ROWS = 4; // consecutive probe rows per thread: their lookups are independent and issued together
constexpr int PROBE_TILE = PROBE_BLOCK * PROBE_ROWS;

// pass 1: heads[row] + per-block output counts.
// The lookups are dependent chains (key -> table word), so one row per thread leaves the kernel waiting on a single
// L2 / DRAM access per warp.  Each thread therefore takes
// PROBE_ROWS consecutive rows: one 128-bit key load when the key is a plain int32 column, then all bitmap words, then
// all first[] words of the rows whose bit is set -- range methods read the 1-bit-per-key bitmap (32x denser than
// first[], L1/L2 resident) first, so only matching rows gather from first[].
__global__ void __launch_bounds__(PROBE_BLOCK) k_probe_count(JoinDev j, KeyCols kc, int32_t join_type, int64_t n, int32_t vec_keys, uint8_t* __restrict__ match, uint32_t* __restrict__ heads,
                                                              uint32_t* __restrict__ block_counts) {
    __shared__ unsigned long long s_cnt[PROBE_BLOCK / 32];
    const int64_t base = ((int64_t)blockIdx.x * PROBE_BLOCK + threadIdx.x) * PROBE_ROWS;
    int64_t key[PROBE_ROWS];
    uint32_t live = 0; // bit r: row exists and its key is not NULL
    const bool full = base + PROBE_ROWS <= n;
    if (vec_keys && full) {
        const int4 v = ldg_stream_v4((const int32_t*)kc.c[0].data + base);
        key[0] = v.x, key[1] = v.y, key[2] = v.z, key[3] = v.w;
        live = (1u << PROBE_ROWS) - 1;
    } else {
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++) {
            key[r] = 0;
            if (base + r < n && !pack_key(kc, base + r, key[r])) live |= 1u << r;
        }
    }
    uint32_t head[PROBE_ROWS];
    if (j.method == SR_JOIN_METHOD_LINEAR_CHAINED) {
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++) head[r] = (live >> r) & 1u ? join_lookup(j, key[r]) : 0u;
    } else {
        uint32_t word[PROBE_ROWS];
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++) {
            const bool in = ((live >> r) & 1u) && key[r] >= j.min_value && key[r] <= j.max_value;
            if (!in) live &= ~(1u << r);
            word[r] = in ? __ldg(j.bitmap + ((uint64_t)(key[r] - j.min_value) >> 5)) : 0u;
        }
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++) {
            const uint64_t off = (uint64_t)(key[r] - j.min_value);
            head[r] = (((live >> r) & 1u) && ((word[r] >> (off & 31)) & 1u)) ? __ldg(j.first + off) : 0u;
        }
    }
    // 64-bit while summing: a chain may be as long as the build side, a block's total is stored saturated (the host
    // refuses outputs of >= 2^32 - 16 rows per batch, so a saturated block makes the whole probe fail loudly instead of
    // wrapping and under-sizing the index buffers)
    unsigned long long cnt = 0;
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++)
        if (base + r < n) cnt += probe_row_count(j, join_type, head[r], match);
    if (full) {
        *(uint4*)(heads + base) = make_uint4(head[0], head[1], head[2], head[3]);
    } else {
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++)
            if (base + r < n) heads[base + r] = head[r];
    }
    cnt = warp_sum(cnt);
    if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < PROBE_BLOCK / 32; w++) t += s_cnt[w];
        block_counts[blockIdx.x] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t;
    }
}

// (Not done: ONE kernel for unique build keys -- lookup, block ranking, a decoupled look-back over per-tile status words
// for the global offset, ordered pair write.  With four rows per thread a tile is too little work to hide the serial
// look-back chain over ~200 K tiles of a 200 M-row probe.)
// pass 2: write (probe_index, build_index) pairs in probe order
__global__ void __launch_bounds__(PROBE_BLOCK) k_probe_write(JoinDev j, int32_t join_type, int64_t n, const uint32_t* __restrict__ heads,
                                                              const uint64_t* __restrict__ block_offsets, uint32_t* __restrict__ probe_index,
                                                              uint32_t* __restrict__ build_index) {
    __shared__ uint32_t s_scan[PROBE_BLOCK / 32 + 1];
    const int64_t base = ((int64_t)blockIdx.x * PROBE_BLOCK + threadIdx.x) * PROBE_ROWS;
    uint32_t head[PROBE_ROWS], cnt[PROBE_ROWS], mine = 0;
    if (base + PROBE_ROWS <= n) {
        const uint4 h = *(const uint4*)(heads + base);
        head[0] = h.x, head[1] = h.y, head[2] = h.z, head[3] = h.w;
    } else {
#pragma unroll
        for (int r = 0; r < PROBE_ROWS; r++) head[r] = base + r < n ? heads[base + r] : 0u;
    }
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++) {
        cnt[r] = base + r < n ? probe_row_count(j, join_type, head[r]) : 0u;
        mine += cnt[r];
    }
    uint32_t tot;
    const uint32_t ex = block_excl_scan<PROBE_BLOCK>(mine, s_scan, &tot);
    if (mine == 0) return;
    uint64_t o = block_offsets[blockIdx.x] + ex;
    const bool no_build = join_type == SR_JOIN_LEFT_SEMI || join_type == SR_JOIN_LEFT_ANTI;
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++) {
        if (cnt[r] == 0) continue;
        if (no_build || head[r] == 0) {
            probe_index[o] = (uint32_t)(base + r);
            build_index[o] = 0;
            o++;
            continue;
        }
        uint32_t b = head[r];
        while (b != 0) {
            probe_index[o] = (uint32_t)(base + r);
            build_index[o] = b;
            o++;
            b = j.has_dup ? __ldg(j.next + b) : 0u;
        }
    }
}

// ---- the two probe passes for packed keys of 9..16 bytes (JoinDev::wide) -----------------------------------------------
// Same tile geometry and output contract as k_probe_count / k_probe_write.  heads[] holds the head of the FINGERPRINT chain;
// both passes pack the probe row's 128-bit key again and only count / emit the chain entries whose full key equals it.
__global__ void __launch_bounds__(PROBE_BLOCK) k_probe_count_wide(JoinDev j, KeyCols kc, int32_t join_type, int64_t n, uint8_t* __restrict__ match,
                                                                   uint32_t* __restrict__ heads, uint32_t* __restrict__ block_counts) {
    __shared__ unsigned long long s_cnt[PROBE_BLOCK / 32];
    const int64_t base = ((int64_t)blockIdx.x * PROBE_BLOCK + threadIdx.x) * PROBE_ROWS;
    unsigned long long cnt = 0;
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++) {
        if (base + r >= n) continue;
        WideKey wk;
        uint32_t head = 0;
        if (!pack_key_wide(kc, base + r, wk)) head = join_lookup(j, wide_fingerprint(wk));
        heads[base + r] = head;
        cnt += probe_row_count(j, join_type, head, match, &wk);
    }
    cnt = warp_sum(cnt);
    if (lane_id() == 0) s_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < PROBE_BLOCK / 32; w++) t += s_cnt[w];
        block_counts[blockIdx.x] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t;
    }
}

__global__ void __launch_bounds__(PROBE_BLOCK) k_probe_write_wide(JoinDev j, KeyCols kc, int32_t join_type, int64_t n, const uint32_t* __restrict__ heads,
                                                                   const uint64_t* __restrict__ block_offsets, uint32_t* __restrict__ probe_index,
                                                                   uint32_t* __restrict__ build_index) {
    __shared__ uint32_t s_scan[PROBE_BLOCK / 32 + 1];
    const int64_t base = ((int64_t)blockIdx.x * PROBE_BLOCK + threadIdx.x) * PROBE_ROWS;
    uint32_t head[PROBE_ROWS], cnt[PROBE_ROWS], mine = 0;
    WideKey wk[PROBE_ROWS];
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++) {
        head[r] = cnt[r] = 0;
        wk[r].lo = wk[r].hi = 0;
        if (base + r < n) {
            head[r] = heads[base + r];
            if (head[r] != 0) (void)pack_key_wide(kc, base + r, wk[r]); // head != 0: no key column was NULL
            cnt[r] = probe_row_count(j, join_type, head[r], nullptr, &wk[r]);
        }
        mine += cnt[r];
    }
    uint32_t tot;
    const uint32_t ex = block_excl_scan<PROBE_BLOCK>(mine, s_scan, &tot);
    if (mine == 0) return;
    uint64_t o = block_offsets[blockIdx.x] + ex;
    const bool no_build = join_type == SR_JOIN_LEFT_SEMI || join_type == SR_JOIN_LEFT_ANTI;
#pragma unroll
    for (int r = 0; r < PROBE_ROWS; r++) {
        if (cnt[r] == 0) continue;
        uint32_t emitted = 0;
        if (!no_build) {
            for (uint32_t b = head[r]; b != 0; b = __ldg(j.next + b)) {
                if (!wide_equal(j, b, wk[r])) continue;
                probe_index[o] = (uint32_t)(base + r);
                build_index[o] = b;
                o++;
                emitted++;
            }
        }
        if (emitted == 0) { // semi / anti rows, and the NULL-padded row of an outer join
            probe_index[o] = (uint32_t)(base + r);
            build_index[o] = 0;
            o++;
        }
    }
}

// ---- other-join conjunct ------------------------------------------------------------------------------------------------
// (HashJoiner::_other_join_conjunct_ctxs, exec/hash_joiner.h:314-329.)  The key match produces CANDIDATE pairs (the INNER
// form of the two passes above, in probe order); the conjunct is evaluated per candidate over the probe row and the build
// row; what is emitted then depends on the join type (see sr_join_desc.other_conjunct).
struct PairLoader {
    const VTab& vt;
    int64_t prow, brow;
    __device__ __forceinline__ bool load(int id, int64_t& bits) const {
        const VDesc& d = vt.v[id];
        const int64_t row = d.src < 0 ? prow : brow;
        const bool nul = d.nulls != nullptr && d.nulls[row] != 0;
        bits = is_float_class(d.type) ? __double_as_longlong(load_double(d.data, d.type, row)) : load_int(d.data, d.type, row);
        return nul;
    }
};

// keep[c] = the conjunct holds for candidate c; probe_any[i] = some candidate of probe row i passed; match[b] (RIGHT / FULL
// joins) = build row b has a passing partner
__global__ void __launch_bounds__(256) k_conj_eval(const __grid_constant__ VTab vt, const __grid_constant__ CExpr conj, const uint32_t* __restrict__ pi,
                                                    const uint32_t* __restrict__ bi, int64_t ncand, uint8_t* __restrict__ keep, uint8_t* __restrict__ probe_any,
                                                    uint8_t* __restrict__ match) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncand; c += (int64_t)gridDim.x * blockDim.x) {
        PairLoader ld{vt, (int64_t)pi[c], (int64_t)bi[c]};
        int64_t bits;
        const bool nul = eval_expr(conj, ld, bits);
        const bool pass = !nul && bits != 0;
        keep[c] = pass ? 1 : 0;
        if (pass) {
            probe_any[pi[c]] = 1;
            if (match) match[bi[c]] = 1;
        }
    }
}
// which candidates and which probe rows appear in the output
__global__ void __launch_bounds__(256) k_conj_flags(int32_t join_type, int64_t ncand, int64_t n, uint8_t* __restrict__ keep /* in: passed, out: emit */,
                                                     uint8_t* __restrict__ probe_any /* in: any passed, out: emit the row by itself */) {
    const bool pairs = join_type == SR_JOIN_INNER || join_type == SR_JOIN_LEFT_OUTER || join_type == SR_JOIN_RIGHT_OUTER || join_type == SR_JOIN_FULL_OUTER;
    const bool row_if_none = join_type == SR_JOIN_LEFT_OUTER || join_type == SR_JOIN_FULL_OUTER || join_type == SR_JOIN_LEFT_ANTI;
    const bool row_if_any = join_type == SR_JOIN_LEFT_SEMI;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncand + n + 2; i += (int64_t)gridDim.x * blockDim.x) {
        if (i <= ncand) {
            keep[i] = (i < ncand && pairs) ? keep[i] : 0; // entry ncand: the scan's total lands behind it
        } else {
            const int64_t r = i - ncand - 1;
            const uint8_t any = r < n ? probe_any[r] : 0;
            probe_any[r] = (r < n && ((row_if_none && !any) || (row_if_any && any))) ? 1 : 0;
        }
    }
}
// ordered merge of the kept candidates and the stand-alone probe rows: a kept candidate c lands behind the kept candidates
// before it (K[c]) and the stand-alone rows of smaller probe index (U[pi[c]]); a stand-alone row i behind the kept
// candidates of smaller probe index (K[first candidate with probe index >= i]) and the stand-alone rows before it (U[i])
__global__ void __launch_bounds__(256) k_conj_emit(const uint8_t* __restrict__ keep, const uint8_t* __restrict__ row_emit, const uint32_t* __restrict__ K,
                                                    const uint32_t* __restrict__ U, const uint32_t* __restrict__ pi, const uint32_t* __restrict__ bi, int64_t ncand,
                                                    int64_t n, uint32_t* __restrict__ out_pi, uint32_t* __restrict__ out_bi) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncand + n; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < ncand) {
            if (!keep[i]) continue;
            const uint64_t o = (uint64_t)K[i] + U[pi[i]];
            out_pi[o] = pi[i];
            out_bi[o] = bi[i];
        } else {
            const int64_t r = i - ncand;
            if (!row_emit[r]) continue;
            int64_t lo = 0, hi = ncand; // first candidate whose probe index is >= r
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if ((int64_t)pi[mid] < r) lo = mid + 1; else hi = mid;
            }
            const uint64_t o = (uint64_t)K[lo] + U[r];
            out_pi[o] = (uint32_t)r;
            out_bi[o] = 0;
        }
    }
}
struct U8ToU32 {
    __host__ __device__ __forceinline__ uint32_t operator()(const uint8_t& v) const { return v; }
};

// K5 exposed for golden-vector pinning
__global__ void __launch_bounds__(256) k_join_key_hash(const void* __restrict__ keys, int32_t type, int64_t n, uint32_t log_buckets,
                                                        uint32_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t v = load_int(keys, type, i);
        out[i] = type_width(type) == 8 ? join_key_hash64((uint64_t)v, log_buckets) : join_key_hash32((uint32_t)(int32_t)v, log_buckets);
    }
}

} // namespace srd

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct BuildCol {
    int32_t slot = 0, type = 0, width = 0;
    bool nullable = false;
    DevBuf data, nulls;
};

struct ProberState {
    Staged staged;
    DevBuf heads, block_counts, block_offsets, probe_index, build_index;
    DevBuf conj_keep, conj_any, conj_k, conj_u, conj_tmp, conj_pi, conj_bi; // other-join conjunct: flags, their prefix sums, final pairs
    ScanScratch scan_scratch;
    std::vector<DevBuf> out_bufs;
    int64_t last_count = 0;
};

struct sr_join {
    sr_ctx* ctx = nullptr;
    sr_join_desc desc;
    std::vector<BuildCol*> cols;
    int64_t rows = 0;     // build rows (without the sentinel)
    int64_t capacity = 0; // rows the column buffers can hold (incl. sentinel)
    bool built = false;
    int32_t method = SR_JOIN_METHOD_NONE;
    int32_t has_dup = 0;
    int64_t min_value = 0, max_value = 0, bucket_size = 0, null_keys = 0;
    uint32_t hmask = 0, hlog = 0;
    DevBuf keys, knulls, first, next, hkeys, bitmap, flags, zero_row, wide_lo, wide_hi;
    bool wide = false; // packed key of 9..16 bytes
    bool conj_compiled = false;
    VReg conj_reg;
    srd::CExpr conj;
    // POST_PROBE phase (RIGHT / FULL joins): one mark byte per build row, written by every probe
    DevBuf match, remain_counts, remain_offsets, remain_index;
    bool match_ready = false;
    int32_t probe_types_seen[SR_MAX_JOIN_OUT] = {}; // types of the probe_out columns, from the first probed chunk
    ScanScratch remain_scan;
    std::vector<DevBuf> remain_bufs;
    Staged staged_build;
    std::vector<ProberState*> probers;
    ~sr_join() {
        for (auto* c : cols) delete c;
        for (auto* p : probers) delete p;
    }
    srd::JoinDev dev() const {
        srd::JoinDev d;
        d.method = method;
        d.has_dup = has_dup;
        d.min_value = min_value;
        d.max_value = max_value;
        d.first = first.as<uint32_t>();
        d.next = next.as<uint32_t>();
        d.hkeys = hkeys.as<unsigned long long>();
        d.wide = wide ? 1 : 0;
        d.pad = 0;
        d.wide_lo = wide_lo.as<unsigned long long>();
        d.wide_hi = wide_hi.as<unsigned long long>();
        d.hmask = hmask;
        d.hlog = hlog;
        d.bitmap = bitmap.as<uint32_t>();
        return d;
    }
    const BuildCol* find_col(int32_t slot) const {
        for (auto* c : cols)
            if (c->slot == slot) return c;
        return nullptr;
    }
};

static int32_t join_validate_desc(sr_ctx* ctx, const sr_join_desc* d) {
    if (d->num_keys < 1 || d->num_keys > SR_MAX_JOIN_KEYS) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "num_keys %d", d->num_keys);
    if (d->join_type < SR_JOIN_INNER || d->join_type > SR_JOIN_FULL_OUTER) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join type %d", d->join_type);
    int total = 0;
    for (int k = 0; k < d->num_keys; k++) {
        const int w = srd::type_width(d->key_types[k]);
        if (w == 0 || w > 8 || srd::is_float_class(d->key_types[k])) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join key type %d", d->key_types[k]);
        total += w;
    }
    if (total > 16) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "packed join key wider than 16 bytes (serialized var-length keys are not implemented)");
    if (d->num_build_out < 0 || d->num_build_out > SR_MAX_JOIN_OUT || d->num_probe_out < 0 || d->num_probe_out > SR_MAX_JOIN_OUT)
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "output slot count");
    return SR_OK;
}

static int32_t join_grow(sr_join* j, int64_t need_rows_incl_sentinel) {
    sr_ctx* ctx = j->ctx;
    if (need_rows_incl_sentinel <= j->capacity) return SR_OK;
    int64_t ncap = std::max<int64_t>(need_rows_incl_sentinel, j->capacity + j->capacity / 2);
    ncap = std::max<int64_t>(ncap, 1024);
    for (auto* c : j->cols) {
        SR_TRY(c->data.reserve(ctx, (size_t)ncap * c->width, (size_t)(j->rows + 1) * c->width));
        if (c->nullable) SR_TRY(c->nulls.reserve(ctx, (size_t)ncap, (size_t)(j->rows + 1)));
    }
    j->capacity = ncap;
    return SR_OK;
}

static int32_t join_append(sr_join* j, const sr_chunk_view* chunk) {
    sr_ctx* ctx = j->ctx;
    if (j->built) return sr_fail(ctx, SR_ERR_STATE, "append_build after build_finish");
    const cudaMemcpyKind kind = chunk->mem == SR_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (j->cols.empty()) {
        for (int k = 0; k < chunk->num_cols; k++) {
            const sr_col_view& c = chunk->cols[k];
            const int w = srd::type_width(c.type);
            if (w == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown build column type %d", c.type);
            auto* bc = new BuildCol();
            bc->slot = c.slot_id;
            bc->type = c.type;
            bc->width = w;
            j->cols.push_back(bc);
        }
        for (int k = 0; k < j->desc.num_keys; k++) {
            const BuildCol* bc = j->find_col(j->desc.build_key_slots[k]);
            if (!bc) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build chunk misses key slot %d", j->desc.build_key_slots[k]);
            if (bc->width != srd::type_width(j->desc.key_types[k])) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build key %d width differs from key_types", k);
        }
    }
    const int64_t n = chunk->num_rows;
    SR_TRY(join_grow(j, j->rows + n + 1));
    for (auto* bc : j->cols) {
        const sr_col_view* c = find_col(chunk, bc->slot);
        if (!c) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build chunk misses slot %d", bc->slot);
        if (c->type != bc->type) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build slot %d changed type", bc->slot);
        if (j->rows == 0) SR_CUDA(ctx, cudaMemsetAsync(bc->data.p, 0, (size_t)bc->width, ctx->stream)); // sentinel row 0
        if (n > 0)
            SR_CUDA(ctx, cudaMemcpyAsync((uint8_t*)bc->data.p + (size_t)(j->rows + 1) * bc->width, c->data, (size_t)n * bc->width, kind, ctx->stream));
        if (c->nulls && !bc->nullable) {
            // upgrade to nullable (join_hash_table.cpp:726-742): previous rows are non-null, row 0 NULL
            bc->nullable = true;
            SR_TRY(bc->nulls.reserve(ctx, (size_t)j->capacity));
            SR_CUDA(ctx, cudaMemsetAsync(bc->nulls.p, 0, (size_t)(j->rows + 1), ctx->stream));
            SR_CUDA(ctx, cudaMemsetAsync(bc->nulls.p, 1, 1, ctx->stream));
        }
        if (bc->nullable && n > 0) {
            if (c->nulls)
                SR_CUDA(ctx, cudaMemcpyAsync((uint8_t*)bc->nulls.p + (j->rows + 1), c->nulls, (size_t)n, kind, ctx->stream));
            else
                SR_CUDA(ctx, cudaMemsetAsync((uint8_t*)bc->nulls.p + (j->rows + 1), 0, (size_t)n, ctx->stream));
        }
    }
    if (chunk->mem != SR_MEM_DEVICE) SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // caller may free host buffers
    j->rows += n;
    return SR_OK;
}

static int32_t join_finish(sr_join* j) {
    sr_ctx* ctx = j->ctx;
    if (j->built) return SR_OK;
    if (j->rows >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "more than 2^32 build rows");
    const int64_t n1 = j->rows + 1;
    if (j->cols.empty()) {
        // empty build side: no chunk was ever appended
        j->method = SR_JOIN_METHOD_RANGE_DIRECT_MAPPING;
        j->min_value = 0;
        j->max_value = -1;
        j->bucket_size = 0;
        SR_TRY(j->first.reserve(ctx, 16));
        SR_TRY(j->next.reserve(ctx, 16));
        SR_TRY(j->bitmap.reserve(ctx, 16));
        SR_CUDA(ctx, cudaMemsetAsync(j->first.p, 0, 16, ctx->stream));
        SR_CUDA(ctx, cudaMemsetAsync(j->next.p, 0, 16, ctx->stream));
        SR_CUDA(ctx, cudaMemsetAsync(j->bitmap.p, 0, 16, ctx->stream));
        j->built = true;
        return SR_OK;
    }
    srd::KeyCols kc;
    kc.n = j->desc.num_keys;
    bool any_nullable = false;
    for (int k = 0; k < kc.n; k++) {
        const BuildCol* bc = j->find_col(j->desc.build_key_slots[k]);
        kc.c[k].data = bc->data.p;
        kc.c[k].nulls = bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr;
        kc.c[k].type = bc->type;
        kc.c[k].width = bc->width;
        any_nullable |= bc->nullable;
    }
    SR_TRY(j->keys.reserve(ctx, sizeof(int64_t) * (size_t)n1));
    if (any_nullable) SR_TRY(j->knulls.reserve(ctx, (size_t)n1));
    SR_TRY(j->flags.reserve(ctx, 64));
    long long init[4] = {0x7fffffffffffffffll, (long long)0x8000000000000000ll, 0, 0};
    SR_CUDA(ctx, cudaMemcpyAsync(j->flags.p, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    SR_CUDA(ctx, cudaMemsetAsync(j->keys.p, 0, 8, ctx->stream));
    const int grid = std::min(grid_for(j->rows, 256), ctx->num_sms * 8);
    if (j->wide) {
        SR_TRY(j->wide_lo.reserve(ctx, sizeof(uint64_t) * (size_t)n1));
        SR_TRY(j->wide_hi.reserve(ctx, sizeof(uint64_t) * (size_t)n1));
        SR_CUDA(ctx, cudaMemsetAsync(j->wide_lo.p, 0, 8, ctx->stream));
        SR_CUDA(ctx, cudaMemsetAsync(j->wide_hi.p, 0, 8, ctx->stream));
    }
    srd::k_join_pack_keys<<<grid, 256, 0, ctx->stream>>>(kc, n1, j->keys.as<long long>(), any_nullable ? j->knulls.as<uint8_t>() : nullptr,
                                                        j->flags.as<long long>(), j->wide ? j->wide_lo.as<unsigned long long>() : nullptr,
                                                        j->wide ? j->wide_hi.as<unsigned long long>() : nullptr);
    SR_LAUNCH_CHECK(ctx);
    long long mm[4];
    SR_CUDA(ctx, cudaMemcpyAsync(mm, j->flags.p, sizeof(mm), cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    j->null_keys = mm[2];
    const int64_t valid = j->rows - j->null_keys;
    const bool one_key = j->desc.num_keys == 1 && !j->wide;
    const int kw = srd::type_width(j->desc.key_types[0]);
    // --- method selection (JoinHashMapSelector::_determine_hash_map_method, join_hash_table.cpp:225-350,
    // with the CPU L2/L3 thresholds replaced by an HBM/L2 budget: a direct table is used while it
    // stays within 64x the row count or 25 MiB, half of H100's 50 MB L2) ---
    j->method = SR_JOIN_METHOD_LINEAR_CHAINED;
    if (one_key && kw <= 2) {
        j->method = SR_JOIN_METHOD_DIRECT_MAPPING;
        if (j->desc.key_types[0] == SR_TYPE_BOOLEAN) {
            j->min_value = 0;
            j->max_value = 1;
        } else {
            j->min_value = kw == 1 ? -128 : -32768;
            j->max_value = kw == 1 ? 127 : 32767;
        }
    } else if (one_key && j->desc.enable_range_direct_mapping && valid > 0) {
        const unsigned __int128 interval = (unsigned __int128)((__int128)mm[1] - (__int128)mm[0]) + 1;
        const uint64_t budget = std::max<uint64_t>((uint64_t)valid * 64, (25ull << 20) / 4);
        if (interval < 0xFFFFFFFFull && (uint64_t)interval <= budget) {
            j->method = SR_JOIN_METHOD_RANGE_DIRECT_MAPPING;
            j->min_value = mm[0];
            j->max_value = mm[1];
        }
    } else if (one_key && valid == 0) {
        j->method = SR_JOIN_METHOD_RANGE_DIRECT_MAPPING;
        j->min_value = 0;
        j->max_value = -1;
    }
    SR_TRY(j->next.reserve(ctx, sizeof(uint32_t) * (size_t)n1));
    SR_CUDA(ctx, cudaMemsetAsync(j->next.p, 0, sizeof(uint32_t) * (size_t)n1, ctx->stream));
    int32_t* has_dup_dev = (int32_t*)((long long*)j->flags.p + 3);
    if (j->method == SR_JOIN_METHOD_LINEAR_CHAINED) {
        uint64_t cap = 1024;
        while (cap < (uint64_t)std::max<int64_t>(valid, 1) * 2) cap <<= 1;
        j->hmask = (uint32_t)(cap - 1);
        j->hlog = (uint32_t)__builtin_ctzll(cap);
        j->bucket_size = (int64_t)cap + 1;
        SR_TRY(j->hkeys.reserve(ctx, sizeof(uint64_t) * (cap + 1)));
        SR_TRY(j->first.reserve(ctx, sizeof(uint32_t) * (cap + 1)));
        SR_CUDA(ctx, cudaMemsetAsync(j->first.p, 0, sizeof(uint32_t) * (cap + 1), ctx->stream));
        srd::k_fill_u64<<<std::min(grid_for((int64_t)cap + 1, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(
                j->hkeys.as<unsigned long long>(), (int64_t)cap + 1, (unsigned long long)SR_HKEY_EMPTY);
        SR_LAUNCH_CHECK(ctx);
        SR_TRY(j->bitmap.reserve(ctx, 16));
        srd::k_join_build_hash<<<grid, 256, 0, ctx->stream>>>(j->keys.as<long long>(), any_nullable ? j->knulls.as<uint8_t>() : nullptr, n1,
                                                             j->hkeys.as<unsigned long long>(), j->hmask, j->hlog, j->first.as<uint32_t>(),
                                                             j->next.as<uint32_t>(), has_dup_dev);
        SR_LAUNCH_CHECK(ctx);
    } else {
        const int64_t interval = j->max_value - j->min_value + 1;
        j->bucket_size = interval;
        const size_t fbytes = sizeof(uint32_t) * (size_t)std::max<int64_t>(interval, 4);
        const size_t bbytes = sizeof(uint32_t) * (size_t)((std::max<int64_t>(interval, 1) + 31) / 32 + 4);
        SR_TRY(j->first.reserve(ctx, fbytes));
        SR_TRY(j->bitmap.reserve(ctx, bbytes));
        SR_CUDA(ctx, cudaMemsetAsync(j->first.p, 0, fbytes, ctx->stream));
        SR_CUDA(ctx, cudaMemsetAsync(j->bitmap.p, 0, bbytes, ctx->stream));
        if (valid > 0) {
            srd::k_join_build_direct<<<grid, 256, 0, ctx->stream>>>(j->keys.as<long long>(), any_nullable ? j->knulls.as<uint8_t>() : nullptr, n1,
                                                                   j->min_value, j->first.as<uint32_t>(), j->next.as<uint32_t>(),
                                                                   j->bitmap.as<uint32_t>(), has_dup_dev);
            SR_LAUNCH_CHECK(ctx);
        }
    }
    int32_t hd = 0;
    SR_CUDA(ctx, cudaMemcpyAsync(&hd, has_dup_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    j->has_dup = hd;
    const int64_t rows = j->rows;
    if (hd && rows > 0) {
        // duplicate build keys: put every chain into the reference's order (descending build index)
        if (rows > 0x7FFFFFFFll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join build side of %lld rows with duplicate keys (the chain relink sorts int-indexed items)", (long long)rows);
        const uint64_t nb = (uint64_t)j->bucket_size;
        if (nb >= 0xFFFFFFFFull) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join table of %llu buckets with duplicate keys", (unsigned long long)nb);
        const uint32_t invalid = (uint32_t)nb; // sorts after every real bucket
        int bits = 1;
        while ((1ull << bits) <= nb) bits++;
        DevBuf b_in, b_out, r_in, r_out, tmp;
        SR_TRY(b_in.reserve(ctx, sizeof(uint32_t) * (size_t)rows));
        SR_TRY(b_out.reserve(ctx, sizeof(uint32_t) * (size_t)rows));
        SR_TRY(r_in.reserve(ctx, sizeof(uint32_t) * (size_t)rows));
        SR_TRY(r_out.reserve(ctx, sizeof(uint32_t) * (size_t)rows));
        srd::k_join_bucket_ids<<<grid, 256, 0, ctx->stream>>>(j->keys.as<long long>(), any_nullable ? j->knulls.as<uint8_t>() : nullptr, n1, j->method, j->min_value,
                                                             j->hkeys.as<unsigned long long>(), j->hmask, j->hlog, invalid, b_in.as<uint32_t>(), r_in.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
        size_t tmp_bytes = 0;
        SR_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, b_in.as<uint32_t>(), b_out.as<uint32_t>(), r_in.as<uint32_t>(), r_out.as<uint32_t>(),
                                                     (int)rows, 0, bits, ctx->stream));
        SR_TRY(tmp.reserve(ctx, std::max<size_t>(tmp_bytes, 16)));
        SR_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, b_in.as<uint32_t>(), b_out.as<uint32_t>(), r_in.as<uint32_t>(), r_out.as<uint32_t>(),
                                                     (int)rows, 0, bits, ctx->stream)); // LSD radix sort: stable, rows stay ascending inside a bucket
        srd::k_join_relink<<<grid, 256, 0, ctx->stream>>>(b_out.as<uint32_t>(), r_out.as<uint32_t>(), rows, invalid, j->first.as<uint32_t>(), j->next.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the scratch buffers go out of scope
    }
    j->built = true;
    return SR_OK;
}

static int32_t join_key_cols(sr_join* j, const Staged& st, srd::KeyCols* kc) {
    kc->n = j->desc.num_keys;
    for (int k = 0; k < kc->n; k++) {
        const int c = st.find(j->desc.probe_key_slots[k]);
        if (c < 0) return sr_fail(j->ctx, SR_ERR_INVALID_ARGUMENT, "probe chunk misses key slot %d", j->desc.probe_key_slots[k]);
        if (st.cols[c].width != srd::type_width(j->desc.key_types[k]) || srd::is_float_class(st.cols[c].type))
            return sr_fail(j->ctx, SR_ERR_INVALID_ARGUMENT, "probe key %d type differs from key_types", k);
        kc->c[k] = st.cols[c];
    }
    return SR_OK;
}

static bool join_has_post_probe(int32_t jt) {
    return jt == SR_JOIN_RIGHT_OUTER || jt == SR_JOIN_RIGHT_SEMI || jt == SR_JOIN_RIGHT_ANTI || jt == SR_JOIN_FULL_OUTER;
}

static int32_t join_match_array(sr_join* j) {
    if (j->match_ready) return SR_OK;
    sr_ctx* ctx = j->ctx;
    SR_TRY(j->match.reserve(ctx, (size_t)j->rows + 16));
    SR_CUDA(ctx, cudaMemsetAsync(j->match.p, 0, (size_t)j->rows + 16, ctx->stream));
    j->match_ready = true;
    return SR_OK;
}

// POST_PROBE: JoinHashMap::probe_remain (join_hash_map.hpp:136-143) -> _search_ht_remain + _probe_null_output / _build_output
static int32_t join_probe_remain(sr_join* j, sr_chunk_out* out) {
    sr_ctx* ctx = j->ctx;
    if (!j->built) return sr_fail(ctx, SR_ERR_STATE, "probe_remain before build_finish");
    const int32_t jt = j->desc.join_type;
    if (!join_has_post_probe(jt)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "join type %d has no post-probe phase", jt);
    SR_TRY(join_match_array(j)); // never probed: every build row is unmatched
    const bool with_probe_cols = jt == SR_JOIN_RIGHT_OUTER || jt == SR_JOIN_FULL_OUTER;
    const uint8_t want = jt == SR_JOIN_RIGHT_SEMI ? 1 : 0;
    const int64_t rows = j->rows;
    int64_t total = 0;
    const int blocks = grid_for(std::max<int64_t>(rows, 1), srd::REMAIN_BLOCK);
    if (rows > 0) {
        SR_TRY(j->remain_counts.reserve(ctx, sizeof(uint32_t) * (size_t)blocks));
        SR_TRY(j->remain_offsets.reserve(ctx, sizeof(uint64_t) * (size_t)blocks));
        srd::k_remain_count<<<blocks, srd::REMAIN_BLOCK, 0, ctx->stream>>>((const uint8_t*)j->match.p, rows, want, j->remain_counts.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
        SR_TRY(scan_counts(ctx, &j->remain_scan, j->remain_counts.as<uint32_t>(), blocks, j->remain_offsets.as<uint64_t>()));
        SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned, ctx->dscratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        total = (int64_t)ctx->pinned[0];
    }
    SR_TRY(j->remain_index.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(total, 1)));
    if (total > 0) {
        srd::k_remain_write<<<blocks, srd::REMAIN_BLOCK, 0, ctx->stream>>>((const uint8_t*)j->match.p, rows, want, j->remain_offsets.as<uint64_t>(),
                                                                           j->remain_index.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
    }
    const int np = with_probe_cols ? j->desc.num_probe_out : 0, nb = j->desc.num_build_out;
    if (np + nb > SR_MAX_OUT_COLS) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many join output columns");
    if ((int)j->remain_bufs.size() < 2 * (np + nb)) {
        std::vector<DevBuf> nbv(2 * (np + nb));
        for (size_t i = 0; i < j->remain_bufs.size(); i++) std::swap(nbv[i], j->remain_bufs[i]);
        j->remain_bufs.swap(nbv);
    }
    out->num_cols = np + nb;
    out->mem = SR_MEM_DEVICE;
    out->num_rows = total;
    srd::GatherArgs ga;
    ga.n = 0;
    const size_t cap = (size_t)std::max<int64_t>(total, 1);
    for (int k = 0; k < np + nb; k++) {
        if (k < np) { // probe side: NULL (_probe_null_output, join_hash_map.hpp:206-232)
            const int32_t type = j->desc.probe_out_types[k] ? j->desc.probe_out_types[k] : j->probe_types_seen[k];
            const int w = srd::type_width(type);
            if (w == 0)
                return sr_fail(ctx, SR_ERR_STATE, "type of probe output slot %d is unknown (never probed): declare it in sr_join_desc.probe_out_types", j->desc.probe_out_slots[k]);
            SR_TRY(j->remain_bufs[2 * k].reserve(ctx, cap * w));
            SR_TRY(j->remain_bufs[2 * k + 1].reserve(ctx, cap));
            if (total > 0) {
                SR_CUDA(ctx, cudaMemsetAsync(j->remain_bufs[2 * k].p, 0, (size_t)total * w, ctx->stream));
                SR_CUDA(ctx, cudaMemsetAsync(j->remain_bufs[2 * k + 1].p, 1, (size_t)total, ctx->stream));
            }
            out->cols[k].data = j->remain_bufs[2 * k].p;
            out->cols[k].nulls = (uint8_t*)j->remain_bufs[2 * k + 1].p;
            out->cols[k].type = type;
            out->cols[k].slot_id = j->desc.probe_out_slots[k];
            continue;
        }
        const int32_t slot = j->desc.build_out_slots[k - np];
        const BuildCol* bc = j->find_col(slot);
        if (!bc) {
            if (total > 0 || j->desc.build_out_types[k - np] == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build chunk misses output slot %d", slot);
            out->cols[k].data = nullptr; // empty build side: zero rows of the declared type
            out->cols[k].nulls = nullptr;
            out->cols[k].type = j->desc.build_out_types[k - np];
            out->cols[k].slot_id = slot;
            continue;
        }
        srd::GatherCol g;
        g.src = bc->data.p;
        g.src_nulls = bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr;
        g.width = bc->width;
        g.zero_is_null = 0;
        SR_TRY(j->remain_bufs[2 * k].reserve(ctx, cap * g.width));
        if (g.src_nulls) SR_TRY(j->remain_bufs[2 * k + 1].reserve(ctx, cap));
        g.dst = j->remain_bufs[2 * k].p;
        g.dst_nulls = g.src_nulls ? (uint8_t*)j->remain_bufs[2 * k + 1].p : nullptr;
        out->cols[k].data = g.dst;
        out->cols[k].nulls = g.dst_nulls;
        out->cols[k].type = bc->type;
        out->cols[k].slot_id = slot;
        ga.c[ga.n++] = g;
    }
    if (total > 0 && ga.n > 0) {
        srd::k_gather<<<dim3(std::min(grid_for(total, 256), ctx->num_sms * 16), ga.n), 256, 0, ctx->stream>>>(j->remain_index.as<uint32_t>(), total, ga);
        SR_LAUNCH_CHECK(ctx);
    }
    return SR_OK;
}

struct ConjTypeCtx {
    sr_join* j;
    const Staged* probe;
};
static int32_t conj_slot_type(void* user, int32_t slot) {
    ConjTypeCtx* t = (ConjTypeCtx*)user;
    const int c = t->probe->find(slot);
    if (c >= 0) return t->probe->cols[c].type;
    const BuildCol* bc = t->j->find_col(slot);
    return bc ? bc->type : 0;
}

// candidates (ps.probe_index / ps.build_index, `*total` of them, probe order) -> the join type's output pairs
static int32_t join_apply_conjunct(sr_join* j, ProberState& ps, int64_t n, int64_t* total, uint8_t* match) {
    sr_ctx* ctx = j->ctx;
    const int64_t ncand = *total;
    if (ncand >= 0x7FFFFFF0ll || n >= 0x7FFFFFF0ll)
        return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "other-join conjunct over %lld candidate pairs / %lld probe rows: probe in smaller batches (the prefix sums index with 32 bits)",
                       (long long)ncand, (long long)n);
    ConjTypeCtx tc{j, &ps.staged};
    if (!j->conj_compiled) {
        j->conj_reg = VReg();
        SR_TRY(compile_expr(ctx, &j->desc.other_conjunct, &j->conj_reg, conj_slot_type, &tc, &j->conj));
        if (j->conj.result_is_double) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "the other-join conjunct is not boolean");
        if (j->conj_reg.slots.size() > SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "other-join conjunct over too many columns");
        j->conj_compiled = true;
    }
    VTab vt;
    memset(&vt, 0, sizeof(vt));
    vt.n = (int32_t)j->conj_reg.slots.size();
    for (size_t k = 0; k < j->conj_reg.slots.size(); k++) {
        const int32_t slot = j->conj_reg.slots[k];
        const int c = ps.staged.find(slot);
        if (c >= 0) {
            vt.v[k] = VDesc{ps.staged.cols[c].data, ps.staged.cols[c].nulls, ps.staged.cols[c].type, -1};
        } else {
            const BuildCol* bc = j->find_col(slot);
            if (!bc) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "other-join conjunct: slot %d is in neither chunk", slot);
            vt.v[k] = VDesc{bc->data.p, bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr, bc->type, 0};
        }
        if (vt.v[k].type != j->conj_reg.types[k]) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "other-join conjunct: slot %d changed type", slot);
    }
    SR_TRY(ps.conj_keep.reserve(ctx, (size_t)ncand + 16));
    SR_TRY(ps.conj_any.reserve(ctx, (size_t)n + 16));
    SR_TRY(ps.conj_k.reserve(ctx, sizeof(uint32_t) * ((size_t)ncand + 2)));
    SR_TRY(ps.conj_u.reserve(ctx, sizeof(uint32_t) * ((size_t)n + 2)));
    SR_CUDA(ctx, cudaMemsetAsync(ps.conj_any.p, 0, (size_t)n + 16, ctx->stream));
    const int grid = std::min(grid_for(std::max<int64_t>(ncand + n + 2, 1), 256), ctx->num_sms * 16);
    if (ncand > 0) {
        srd::k_conj_eval<<<grid, 256, 0, ctx->stream>>>(vt, j->conj, ps.probe_index.as<uint32_t>(), ps.build_index.as<uint32_t>(), ncand, ps.conj_keep.as<uint8_t>(),
                                                       ps.conj_any.as<uint8_t>(), match);
        SR_LAUNCH_CHECK(ctx);
    }
    srd::k_conj_flags<<<grid, 256, 0, ctx->stream>>>(j->desc.join_type, ncand, n, ps.conj_keep.as<uint8_t>(), ps.conj_any.as<uint8_t>());
    SR_LAUNCH_CHECK(ctx);
    // exclusive prefix sums over ncand + 1 / n + 1 flags (the last flag is 0: its sum is the total)
    auto kin = thrust::make_transform_iterator((const uint8_t*)ps.conj_keep.as<uint8_t>(), srd::U8ToU32());
    auto uin = thrust::make_transform_iterator((const uint8_t*)ps.conj_any.as<uint8_t>(), srd::U8ToU32());
    size_t tb1 = 0, tb2 = 0;
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb1, kin, ps.conj_k.as<uint32_t>(), (int)(ncand + 1), ctx->stream));
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb2, uin, ps.conj_u.as<uint32_t>(), (int)(n + 1), ctx->stream));
    SR_TRY(ps.conj_tmp.reserve(ctx, std::max<size_t>(std::max(tb1, tb2), 16)));
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(ps.conj_tmp.p, tb1, kin, ps.conj_k.as<uint32_t>(), (int)(ncand + 1), ctx->stream));
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(ps.conj_tmp.p, tb2, uin, ps.conj_u.as<uint32_t>(), (int)(n + 1), ctx->stream));
    uint32_t* pin = (uint32_t*)ctx->pinned;
    SR_CUDA(ctx, cudaMemcpyAsync(pin, ps.conj_k.as<uint32_t>() + ncand, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaMemcpyAsync(pin + 1, ps.conj_u.as<uint32_t>() + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t out_total = (int64_t)pin[0] + (int64_t)pin[1];
    if (out_total >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join output of more than 2^32 rows in one batch; probe in smaller batches");
    SR_TRY(ps.conj_pi.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(out_total, 1)));
    SR_TRY(ps.conj_bi.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(out_total, 1)));
    if (out_total > 0) {
        srd::k_conj_emit<<<grid, 256, 0, ctx->stream>>>(ps.conj_keep.as<uint8_t>(), ps.conj_any.as<uint8_t>(), ps.conj_k.as<uint32_t>(), ps.conj_u.as<uint32_t>(),
                                                       ps.probe_index.as<uint32_t>(), ps.build_index.as<uint32_t>(), ncand, n, ps.conj_pi.as<uint32_t>(),
                                                       ps.conj_bi.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
    }
    std::swap(ps.probe_index, ps.conj_pi);
    std::swap(ps.build_index, ps.conj_bi);
    *total = out_total;
    return SR_OK;
}

static int32_t join_probe(sr_join* j, int32_t prober_id, const sr_chunk_view* probe, sr_chunk_out* out) {
    sr_ctx* ctx = j->ctx;
    if (!j->built) return sr_fail(ctx, SR_ERR_STATE, "probe before build_finish");
    if (prober_id < 0 || prober_id > 4096) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "prober_id %d", prober_id);
    if (probe->num_rows >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "probe batch of more than 2^32 rows");
    while ((int)j->probers.size() <= prober_id) j->probers.push_back(new ProberState());
    ProberState& ps = *j->probers[prober_id];
    SR_TRY(ps.staged.stage(ctx, probe));
    srd::KeyCols kc;
    SR_TRY(join_key_cols(j, ps.staged, &kc));
    const int64_t n = probe->num_rows;
    const int blocks = grid_for(n, srd::PROBE_TILE);
    const srd::JoinDev jd = j->dev();
    // the key is one plain int32-class column, 16-byte aligned: the probe reads four keys per 128-bit load
    const int32_t vec_keys = kc.n == 1 && kc.c[0].nulls == nullptr && kc.c[0].width == 4 && !srd::is_float_class(kc.c[0].type) &&
                                             (((uintptr_t)kc.c[0].data) & 15) == 0
                                     ? 1
                                     : 0;
    uint8_t* match = nullptr;
    if (join_has_post_probe(j->desc.join_type)) {
        SR_TRY(join_match_array(j));
        match = (uint8_t*)j->match.p;
        for (int k = 0; k < j->desc.num_probe_out; k++) { // remembered for the NULL padding of sr_join_probe_remain
            const int c = ps.staged.find(j->desc.probe_out_slots[k]);
            if (c >= 0) j->probe_types_seen[k] = ps.staged.cols[c].type;
        }
    }
    // with an other-join conjunct the two passes produce the key-matched CANDIDATES (INNER form, nothing marked); the
    // conjunct pass below turns them into the join type's output
    const bool has_conj = j->desc.other_conjunct.num_nodes > 0;
    const int32_t jt_run = has_conj ? (int32_t)SR_JOIN_INNER : j->desc.join_type;
    uint8_t* const match_run = has_conj ? nullptr : match;
    int64_t total = 0;
    if (n > 0) {
        SR_TRY(ps.heads.reserve(ctx, sizeof(uint32_t) * (size_t)n));
        SR_TRY(ps.block_counts.reserve(ctx, sizeof(uint32_t) * (size_t)blocks));
        SR_TRY(ps.block_offsets.reserve(ctx, sizeof(uint64_t) * (size_t)blocks));
        if (j->wide)
            srd::k_probe_count_wide<<<blocks, srd::PROBE_BLOCK, 0, ctx->stream>>>(jd, kc, jt_run, n, match_run, ps.heads.as<uint32_t>(),
                                                                                 ps.block_counts.as<uint32_t>());
        else
            srd::k_probe_count<<<blocks, srd::PROBE_BLOCK, 0, ctx->stream>>>(jd, kc, jt_run, n, vec_keys, match_run, ps.heads.as<uint32_t>(),
                                                                            ps.block_counts.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
        SR_TRY(scan_counts(ctx, &ps.scan_scratch, ps.block_counts.as<uint32_t>(), blocks, ps.block_offsets.as<uint64_t>()));
        SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned, ctx->dscratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        total = (int64_t)ctx->pinned[0];
    }
    if (total >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "join output of more than 2^32 rows in one batch; probe in smaller batches");
    SR_TRY(ps.probe_index.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(total, 1)));
    SR_TRY(ps.build_index.reserve(ctx, sizeof(uint32_t) * (size_t)std::max<int64_t>(total, 1)));
    if (total > 0) {
        if (j->wide)
            srd::k_probe_write_wide<<<blocks, srd::PROBE_BLOCK, 0, ctx->stream>>>(jd, kc, jt_run, n, ps.heads.as<uint32_t>(),
                                                                                 ps.block_offsets.as<uint64_t>(), ps.probe_index.as<uint32_t>(),
                                                                                 ps.build_index.as<uint32_t>());
        else
            srd::k_probe_write<<<blocks, srd::PROBE_BLOCK, 0, ctx->stream>>>(jd, jt_run, n, ps.heads.as<uint32_t>(),
                                                                            ps.block_offsets.as<uint64_t>(), ps.probe_index.as<uint32_t>(),
                                                                            ps.build_index.as<uint32_t>());
        SR_LAUNCH_CHECK(ctx);
    }
    if (has_conj) SR_TRY(join_apply_conjunct(j, ps, n, &total, match));
    ps.last_count = total;
    // materialise output columns: probe_out_slots (gather by probe_index) then build_out_slots
    const int32_t jt = j->desc.join_type;
    const bool semi = jt == SR_JOIN_LEFT_SEMI || jt == SR_JOIN_LEFT_ANTI;
    const bool outer = jt == SR_JOIN_LEFT_OUTER || jt == SR_JOIN_FULL_OUTER;
    const bool right_only = jt == SR_JOIN_RIGHT_SEMI || jt == SR_JOIN_RIGHT_ANTI; // no probe column in the output, no probe-phase rows
    const int np = right_only ? 0 : j->desc.num_probe_out, nb = semi ? 0 : j->desc.num_build_out;
    if (np + nb > SR_MAX_OUT_COLS) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many join output columns");
    if ((int)ps.out_bufs.size() < 2 * (np + nb)) {
        std::vector<DevBuf> nbv(2 * (np + nb));
        for (size_t i = 0; i < ps.out_bufs.size(); i++) std::swap(nbv[i], ps.out_bufs[i]);
        ps.out_bufs.swap(nbv);
    }
    srd::GatherArgs ga_p, ga_b;
    ga_p.n = 0;
    ga_b.n = 0;
    out->num_cols = np + nb;
    out->mem = SR_MEM_DEVICE;
    out->num_rows = total;
    for (int k = 0; k < np + nb; k++) {
        srd::GatherCol g;
        int32_t slot, type;
        if (k < np) {
            slot = j->desc.probe_out_slots[k];
            const int c = ps.staged.find(slot);
            if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "probe chunk misses output slot %d", slot);
            g.src = ps.staged.cols[c].data;
            g.src_nulls = ps.staged.cols[c].nulls;
            g.width = ps.staged.cols[c].width;
            g.zero_is_null = 0;
            type = ps.staged.cols[c].type;
        } else {
            slot = j->desc.build_out_slots[k - np];
            const BuildCol* bc = j->find_col(slot);
            if (bc) {
                g.src = bc->data.p;
                g.src_nulls = bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr;
                g.width = bc->width;
                type = bc->type;
            } else if (j->cols.empty() && j->desc.build_out_types[k - np] != 0) {
                // no build chunk ever arrived (a dimension scan that filtered everything out): the schema comes from the
                // desc; INNER probes to zero rows, LEFT OUTER to one all-NULL build row per probe row (index 0 = "no row")
                type = j->desc.build_out_types[k - np];
                g.width = srd::type_width(type);
                if (g.width == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build_out_types[%d] = %d is not a type", k - np, type);
                SR_TRY(j->zero_row.reserve(ctx, 16));
                SR_CUDA(ctx, cudaMemsetAsync(j->zero_row.p, 0, 16, ctx->stream));
                g.src = j->zero_row.p;
                g.src_nulls = nullptr;
            } else {
                if (j->cols.empty())
                    return sr_fail(ctx, SR_ERR_STATE, "build side is empty and the type of slot %d is unknown: declare it in sr_join_desc.build_out_types", slot);
                return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "build chunk misses output slot %d", slot);
            }
            g.zero_is_null = outer ? 1 : 0;
        }
        const bool need_nulls = g.src_nulls != nullptr || g.zero_is_null;
        SR_TRY(ps.out_bufs[2 * k].reserve(ctx, (size_t)std::max<int64_t>(total, 1) * g.width));
        if (need_nulls) SR_TRY(ps.out_bufs[2 * k + 1].reserve(ctx, (size_t)std::max<int64_t>(total, 1)));
        g.dst = ps.out_bufs[2 * k].p;
        g.dst_nulls = need_nulls ? (uint8_t*)ps.out_bufs[2 * k + 1].p : nullptr;
        out->cols[k].data = g.dst;
        out->cols[k].nulls = g.dst_nulls;
        out->cols[k].type = type;
        out->cols[k].slot_id = slot;
        if (k < np)
            ga_p.c[ga_p.n++] = g;
        else
            ga_b.c[ga_b.n++] = g;
    }
    if (total > 0) {
        const int gx = std::min(grid_for(total, 256), ctx->num_sms * 16);
        if (ga_p.n > 0) {
            srd::k_gather<<<dim3(gx, ga_p.n), 256, 0, ctx->stream>>>(ps.probe_index.as<uint32_t>(), total, ga_p);
            SR_LAUNCH_CHECK(ctx);
        }
        if (ga_b.n > 0) {
            srd::k_gather<<<dim3(gx, ga_b.n), 256, 0, ctx->stream>>>(ps.build_index.as<uint32_t>(), total, ga_b);
            SR_LAUNCH_CHECK(ctx);
        }
    }
    return SR_OK;
}
