// sr_page.cuh -- segment data pages decoded on the device (SURVEY.md 8f-4): the step in front of the scan.
//   FrameOfReferencePageDecoder  be/src/storage/rowset/frame_of_reference_page.h:113-222
//     ForDecoder::init / decode_current_frame / bit_unpack   be/src/util/frame_of_reference_coding.cpp:246-352
//   PlainPageDecoder             be/src/storage/rowset/plain_page.h:135-260
// A frame-of-reference page: frames of 128 values -- [min: 4 / 8 bytes LE][128 deltas of bit_width bits, most significant
// bit first] -- then (storage format, bit width) byte pairs of all frames, the frame size (128) and the value count
// (uint32 LE).  Storage format 0: value = min + delta; 1 (ascending input): value = previous + delta, the first previous
// being min; 2: the values themselves in 8 * sizeof(T) bits.
//
// H100 mapping (HBM- / PCIe-bound byte work): pages are read where they lie -- device memory or page-locked mapped host
// memory (the decode then IS the host->device transfer, at 4-22 bits per value instead of 32 / 64) -- or staged once when they
// are pageable.  k_page_footers reads the value counts, the host turns them into row / frame offsets (one small
// read-back per batch of pages), k_for_frames expands every page's frame table into per-frame descriptors (byte position by
// a block scan of 16 * bit_width + sizeof(T)), k_for_decode gives every frame to one warp: the packed bytes are copied to
// shared memory with coalesced word loads, every lane extracts FOUR CONSECUTIVE values with 64-bit funnel arithmetic (at
// most 9 bytes of the bit string each), ascending frames take a warp scan, and the lane stores its four values.
//
//   BitShufflePageDecoder        be/src/storage/rowset/bitshuffle_page.h (BitshufflePageBuilder::finish writes the page)
// A bitshuffle page: a 16-byte header of four little-endian uint32s -- num_elements, compressed_size (the whole page, header
// included), num_elements_after_padding = ALIGN_UP(num_elements, 8) (zero padding, never stored), elem_size_bytes -- then
// bitshuffle::compress_lz4(values, padded, elem_size, block_size = 0): blocks of bshuf_default_block_size(s) = max(128,
// (8192 / s) / 8 * 8) = 8192 / s elements (8192 bytes) for s = 1..16, the last one holding padded % block elements when
// that is non-zero.  Each block is a BIG-endian uint32 compressed length, then one LZ4 block-format stream of the
// bit-transposed block: 8 * s rows of elems / 8 bytes, row 8 * j + k holding bit k of byte j of every element (element i at
// bit i % 8 of byte i / 8).  A stream claims at most LZ4_compressBound(8192) = 8240 bytes; the blocks end exactly at
// compressed_size.  bshuf_oracle/bshuf_oracle.cpp restates the codec on the CPU, with the LZ4 end-of-block rules enforced
// here (checked against liblz4's verdicts in tests/golden/bitshuffle_lz4.npz).
// k_page_footers checks the header and counts the blocks, k_bshuf_blocks walks each page's chain of lengths into
// per-block descriptors, and k_bshuf_decode gives every block to one warp: the compressed block is staged in shared memory
// with coalesced word loads (in-place reads over PCIe move only the compressed bytes), the LZ4 sequences are parsed serially
// (warp-uniform) into an 8 KB shared buffer with the literal and match bytes copied across the lanes, and every lane then
// un-transposes 8 consecutive elements (one 8 x 8 bit transpose per byte position) and stores them.
//
//   BinaryDictPageDecoder        be/src/storage/rowset/binary_dict_page.{h,cpp} (BinaryDictPageBuilder::finish writes the page)
// A data page of a dictionary-encoded column: a 4-byte little-endian mode word (EncodingTypePB: 5 DICT_ENCODING, 2
// PLAIN_ENCODING once the dictionary overflowed), then with mode 5 a bitshuffle page of int32 codes, a code being a position
// in the segment's dictionary page.  k_page_footers checks the mode word and the embedded header, the host moves the page
// descriptors past the mode word, and k_bshuf_decode_dict is k_bshuf_decode<4> with the store translating every code
// through the decoder's table (sr_page_decoder_set_dict): the id column comes out in HBM.
//
//   RlePageDecoder               be/src/storage/rowset/rle_page.h; RleDecoder, be/src/util/rle_encoding.h
// A BOOLEAN RLE page: a uint32 value count, then an RLE stream at bit width 1 (ULEB128 run headers: bit-packed groups of 8
// or a repeated byte).  The null map of a nullable column's data page (page format 2) is that stream without the count
// (RLE_NULL) or a BIT_SHUFFLE page of one-byte flags without its header (BITSHUFFLE_NULL); the row count comes from the
// page footer.  k_rle_runs walks every page's run headers into descriptors, k_rle_expand writes the flags one aligned
// 64-bit word per thread; bitshuffle maps reuse k_bshuf_blocks / k_bshuf_decode<1>, then k_null_zero_count zeroes the pages
// without a map and counts the NULLs.
#pragma once

namespace srd {

struct PageDesc {
    const uint8_t* data; // device-visible
    long long size;
    long long row_off;   // first output row
    long long frame_off; // first frame descriptor
};

struct FrameDesc {
    const uint8_t* frame; // the frame's min value (4 / 8 bytes LE), followed by the packed deltas
    long long row;        // output row of the frame's first value
    uint32_t count;       // values in the frame (<= 128)
    uint16_t format;
    uint16_t bit_width;
};

__device__ __forceinline__ uint32_t page_le32(const uint8_t* p) {
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}

constexpr int BSHUF_BLOCK_BYTES = 8192;     // bshuf_default_block_size(s) * s for every width s in 1..16
constexpr uint32_t BSHUF_MAX_STREAM = 8240; // LZ4_compressBound(8192)

// the frames of a frame-of-reference page of n values, in 64 bits: n + 127 wraps a uint32 count from 2^32 - 127 on
__device__ __forceinline__ unsigned long long for_frame_count(unsigned long long n) { return (n + 127) / 128; }

// value count and frame (bitshuffle: block) count of every page; flags[0] |= 1 when a page cannot be a page of `encoding`,
// |= 2 for a dictionary-column page in plain mode (the column's dictionary overflowed: a page of strings, not codes)
__global__ void __launch_bounds__(256) k_page_footers(const PageDesc* __restrict__ pages, int32_t num_pages, int32_t encoding, int32_t elem_size,
                                                       unsigned long long* __restrict__ counts /* [2 * num_pages]: values, frames */, int32_t* __restrict__ flags) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= num_pages) return;
    const PageDesc& pg = pages[p];
    unsigned long long n = 0, frames = 0;
    bool bad = false;
    if (encoding == SR_PAGE_PLAIN) {
        if (pg.size < 4) {
            bad = true;
        } else {
            n = page_le32(pg.data);
            if (pg.size != 4 + (long long)n * elem_size) bad = true;
        }
    } else if (encoding == SR_PAGE_BITSHUFFLE || encoding == SR_PAGE_DICT) {
        // a dictionary data page: a 4-byte mode word (EncodingTypePB: 5 dictionary codes, 2 plain strings), then with mode
        // 5 a bitshuffle page of int32 codes
        const int hdr = encoding == SR_PAGE_DICT ? 4 : 0;
        const uint8_t* b = pg.data + hdr;
        const long long size = pg.size - hdr;
        if (hdr && pg.size >= 4 && page_le32(pg.data) == 2) {
            atomicOr(flags, 2);
        } else if (size < 16 || (hdr && page_le32(pg.data) != 5)) {
            bad = true;
        } else {
            n = page_le32(b);
            const unsigned long long padded = page_le32(b + 8), blk = BSHUF_BLOCK_BYTES / elem_size;
            if (page_le32(b + 4) != (unsigned long long)size || padded != ((n + 7) & ~7ull) || page_le32(b + 12) != (uint32_t)elem_size) bad = true;
            frames = (padded + blk - 1) / blk; // blocks
        }
    } else if (encoding == SR_PAGE_RLE) {
        // a uint32 value count, then the RLE stream; frames: the most runs the stream can hold (each takes >= 2 bytes)
        if (pg.size < 4) {
            bad = true;
        } else {
            n = page_le32(pg.data);
            frames = min(n, (unsigned long long)(pg.size - 4) / 2);
        }
    } else {
        if (pg.size < 5) {
            bad = true;
        } else {
            const uint32_t fsz = pg.data[pg.size - 5];
            n = page_le32(pg.data + pg.size - 4);
            if (fsz != 128 && n != 0) bad = true; // every writer uses ForEncoder::FRAME_VALUE_NUM = 128
            frames = for_frame_count(n);
            if (pg.size - 5 - (long long)frames * 2 < 0) bad = true;
        }
    }
    if (bad) {
        atomicOr(flags, 1);
        n = frames = 0;
    }
    counts[2 * p] = n;
    counts[2 * p + 1] = frames;
}

constexpr int FOR_FRAMES_BLOCK = 256;
// one CTA per page: frame table -> descriptors.  Frame f starts bit_width(f') * 128 / 8 + sizeof(T) bytes after frame f'
// = f - 1 (ForDecoder::init, frame_of_reference_coding.cpp:262-273 -- also for a short last frame, which has no successor).
template <typename T>
__global__ void __launch_bounds__(FOR_FRAMES_BLOCK) k_for_frames(const PageDesc* __restrict__ pages, FrameDesc* __restrict__ frames, int32_t* __restrict__ flags) {
    __shared__ uint32_t s_scan[FOR_FRAMES_BLOCK / 32 + 1];
    __shared__ unsigned long long s_base;
    const PageDesc pg = pages[blockIdx.x];
    if (pg.size < 5) return;
    const uint32_t n = page_le32(pg.data + pg.size - 4);
    const uint32_t nf = (uint32_t)for_frame_count(n); // <= 2^25
    const long long meta = pg.size - 5 - (long long)nf * 2;
    if (meta < 0) return;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (uint32_t f0 = 0; f0 < nf; f0 += FOR_FRAMES_BLOCK) {
        const uint32_t f = f0 + threadIdx.x;
        uint32_t fmt = 0, bw = 0, len = 0;
        if (f < nf) {
            fmt = pg.data[meta + 2 * f];
            bw = pg.data[meta + 2 * f + 1];
            len = bw * 16 + (uint32_t)sizeof(T);
        }
        uint32_t tot;
        const uint32_t ex = block_excl_scan<FOR_FRAMES_BLOCK>(len, s_scan, &tot);
        const unsigned long long off = s_base + ex;
        if (f < nf) {
            const uint32_t cnt = f + 1 < nf ? 128u : n - f * 128u;
            FrameDesc d;
            d.frame = pg.data + off;
            d.row = pg.row_off + (long long)f * 128;
            d.count = cnt;
            d.format = (uint16_t)fmt;
            d.bit_width = (uint16_t)bw;
            // the bytes this frame really holds must lie in front of the frame table
            const unsigned long long used = off + sizeof(T) + ((unsigned long long)cnt * bw + 7) / 8;
            if (fmt > 2 || bw > 8 * sizeof(T) || (long long)used > meta) {
                atomicOr(flags, 1);
                d.count = 0;
            }
            frames[pg.frame_off + f] = d;
        }
        __syncthreads();
        if (threadIdx.x == 0) s_base += tot;
        __syncthreads();
    }
}

constexpr int FOR_DECODE_BLOCK = 256;
constexpr int FOR_DECODE_WARPS = FOR_DECODE_BLOCK / 32;
constexpr int FOR_FRAME_WORDS = 128 * 8 / 4 + 8; // a frame: min value + at most 128 x 64 bits, + the words a 96-bit window may touch

// bits [b, b + bw) of the big-endian bit string in `words` (shared memory, 32-bit words as loaded from little-endian memory)
__device__ __forceinline__ unsigned long long for_extract(const uint32_t* words, uint32_t b, uint32_t bw) {
    const uint32_t byte = b >> 3;
    const uint32_t w = byte >> 2;
    const uint32_t pos = 8 * (byte & 3) + (b & 7); // bit position inside the 96-bit window, 0..31
    const uint32_t W0 = __byte_perm(words[w], 0, 0x0123), W1 = __byte_perm(words[w + 1], 0, 0x0123), W2 = __byte_perm(words[w + 2], 0, 0x0123);
    unsigned long long x = ((unsigned long long)W0 << 32 | W1) << pos;
    x |= (unsigned long long)(__funnelshift_l(W2, W1, pos) & ((1u << pos) - 1u)); // the pos bits shifted in from W2 (pos = 0: none)
    return x >> (64 - bw);                                                      // callers never pass bw = 0
}

template <typename T>
__global__ void __launch_bounds__(FOR_DECODE_BLOCK) k_for_decode(const FrameDesc* __restrict__ frames, long long num_frames, T* __restrict__ out) {
    __shared__ uint32_t s_words[FOR_DECODE_WARPS][FOR_FRAME_WORDS];
    typedef typename std::make_unsigned<T>::type U;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t* words = s_words[wid];
    const long long stride = (long long)gridDim.x * FOR_DECODE_WARPS;
    long long f = (long long)blockIdx.x * FOR_DECODE_WARPS + wid;
    FrameDesc nd;
    if (f < num_frames) nd = frames[f];
    for (; f < num_frames; f += stride) {
        const FrameDesc d = nd;
        if (f + stride < num_frames) nd = frames[f + stride]; // the next descriptor travels while this frame is decoded
        const uint32_t bw = d.bit_width, cnt = d.count;
        if (cnt == 0) continue; // (warp-uniform)
        U v[4] = {0, 0, 0, 0};
        // the frame (min value + packed bytes) -> shared memory.  It starts at any byte: fetch whole words from the aligned
        // address below it and remember the byte skew.  (The min value is read from this copy too: a separate read of it in
        // k_for_frames cost one extra DRAM sector -- or PCIe request -- per frame.)
        const uint32_t nbytes = (uint32_t)sizeof(T) + (cnt * bw + 7) / 8;
        const uintptr_t a0 = (uintptr_t)d.frame & ~(uintptr_t)3;
        const uint32_t skew = (uint32_t)((uintptr_t)d.frame - a0);
        const uint32_t nwords = (skew + nbytes + 3) / 4;
        __syncwarp();
        for (uint32_t i = lane; i < nwords; i += 32) words[i] = (uint32_t)ldg_stream_s32((const uint32_t*)a0 + i);
        for (uint32_t i = nwords + lane; i < nwords + 3; i += 32) words[i] = 0;
        __syncwarp();
        if (bw > 0) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t i = 4 * lane + j;
                if (i < cnt) v[j] = (U)for_extract(words, 8 * (skew + (uint32_t)sizeof(T)) + i * bw, bw);
            }
        }
        // the min value: sizeof(T) little-endian bytes at byte `skew` of the copy = a byte-swapped big-endian extraction
        const unsigned long long mn_be = for_extract(words, 8 * skew, 8 * (uint32_t)sizeof(T));
        const U mn = sizeof(T) == 4 ? (U)__byte_perm((uint32_t)mn_be, 0, 0x0123)
                                    : (U)(((unsigned long long)__byte_perm((uint32_t)mn_be, 0, 0x0123) << 32) | __byte_perm((uint32_t)(mn_be >> 32), 0, 0x0123));
        if (d.format == 1) {
            // ascending: value i = min + delta_0 + ... + delta_i (decode_current_frame, frame_of_reference_coding.cpp:338-345)
            v[1] += v[0];
            v[2] += v[1];
            v[3] += v[2];
            U run = v[3];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const U t = __shfl_up_sync(SR_FULL_MASK, run, o);
                if (lane >= o) run += t;
            }
            const U before = run - v[3] + mn;
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] += before;
        } else if (d.format == 0) {
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] += mn;
        }
        T* o = out + d.row + 4 * lane;
        if (4 * lane + 3 < (int)cnt && (((uintptr_t)o) & (4 * sizeof(T) - 1)) == 0) {
            if (sizeof(T) == 4) {
                *(uint4*)o = make_uint4((uint32_t)v[0], (uint32_t)v[1], (uint32_t)v[2], (uint32_t)v[3]);
            } else {
                ((ulonglong2*)o)[0] = make_ulonglong2((unsigned long long)v[0], (unsigned long long)v[1]);
                ((ulonglong2*)o)[1] = make_ulonglong2((unsigned long long)v[2], (unsigned long long)v[3]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (4 * lane + j < (int)cnt) o[j] = (T)v[j];
        }
    }
}

// plain pages: the values follow a 4-byte count; byte-wise when either side is not word aligned
__global__ void __launch_bounds__(256) k_plain_copy(const PageDesc* __restrict__ pages, int32_t elem_size, uint8_t* __restrict__ out) {
    const PageDesc pg = pages[blockIdx.y];
    if (pg.size < 4) return;
    const long long bytes = pg.size - 4;
    const uint8_t* src = pg.data + 4;
    uint8_t* dst = out + pg.row_off * elem_size;
    if ((((uintptr_t)src | (uintptr_t)dst) & 3) == 0) {
        const long long words = bytes >> 2;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (long long)gridDim.x * blockDim.x)
            ((uint32_t*)dst)[i] = (uint32_t)ldg_stream_s32((const uint32_t*)src + i);
    } else {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < bytes; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
    }
}

struct BshufBlock {
    const uint8_t* src; // the LZ4 stream (device-visible)
    long long row;      // output row of the block's first element
    uint32_t clen;      // stream bytes
    uint32_t elems;     // elements the stream decodes to (a multiple of 8); 0: skip the block
    uint32_t n_out;     // elements stored: the rest is padding
    uint32_t reserved;
};

__device__ __forceinline__ uint32_t page_be32(const uint8_t* p) {
    return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | (uint32_t)p[3];
}

// one thread per page: the chain of big-endian block lengths, from byte `hdr` on, -> descriptors at the page's frame_off.
// counts[2p], counts[2p + 1]: the page's value and block counts -- k_page_footers' reading of a page's 16-byte header (hdr =
// 16), or the host's for a null map (hdr = 0: no header, the count from the page footer, no blocks when the map is empty).
// A chain that overruns the page, claims more than 8240 bytes for a block or does not end at the page's end raises the
// flag; blocks from the first bad length on are skipped.
__global__ void __launch_bounds__(256) k_bshuf_blocks(const PageDesc* __restrict__ pages, int32_t num_pages, int32_t elem_size, int32_t hdr,
                                                       const unsigned long long* __restrict__ counts, BshufBlock* __restrict__ blocks, int32_t* __restrict__ flags) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= num_pages) return;
    const PageDesc pg = pages[p];
    if (pg.size < hdr) return;
    const uint32_t n = (uint32_t)counts[2 * p], blk = BSHUF_BLOCK_BYTES / elem_size, nb = (uint32_t)counts[2 * p + 1];
    const unsigned long long padded = ((unsigned long long)n + 7) & ~7ull;
    long long pos = hdr;
    bool bad = false;
    for (uint32_t b = 0; b < nb; b++) {
        BshufBlock d;
        d.src = nullptr;
        d.row = pg.row_off + (long long)b * blk;
        d.clen = d.elems = d.n_out = d.reserved = 0;
        if (!bad && pg.size - pos >= 4) {
            const uint32_t c = page_be32(pg.data + pos);
            if (c <= BSHUF_MAX_STREAM && c <= pg.size - pos - 4) {
                d.src = pg.data + pos + 4;
                d.clen = c;
                d.elems = (uint32_t)min((unsigned long long)blk, padded - (unsigned long long)b * blk);
                d.n_out = min(d.elems, n - b * blk); // n > b * blk: padding is < 8 elements and a block holds >= 8
                pos += 4 + c;
            } else {
                bad = true;
            }
        } else {
            bad = true;
        }
        blocks[pg.frame_off + b] = d;
    }
    if (bad || pos != pg.size) atomicOr(flags, 1);
}

// 8 x 8 bit matrix transpose: bit k of byte t <-> bit t of byte k (TRANS_BIT_8X8 of the bitshuffle sources)
__device__ __forceinline__ unsigned long long bshuf_trans8x8(unsigned long long x) {
    unsigned long long t;
    t = (x ^ (x >> 7)) & 0x00AA00AA00AA00AAull;
    x = x ^ t ^ (t << 7);
    t = (x ^ (x >> 14)) & 0x0000CCCC0000CCCCull;
    x = x ^ t ^ (t << 14);
    t = (x ^ (x >> 28)) & 0x00000000F0F0F0F0ull;
    x = x ^ t ^ (t << 28);
    return x;
}

// an LZ4 length nibble of 15, continued in bytes (255: another follows); stops once it passes `limit` (the caller rejects)
__device__ __forceinline__ bool lz4_len(const uint8_t* in, uint32_t n, uint32_t& ip, uint32_t& v, uint32_t limit) {
    uint32_t b;
    do {
        if (ip >= n) return false;
        b = in[ip++];
        v += b;
    } while (b == 255 && v <= limit);
    return true;
}

constexpr int BSHUF_DECODE_WARPS = 2;                                // 2 x 16.1 KB of shared memory per CTA
constexpr int BSHUF_STAGE_WORDS = (3 + (int)BSHUF_MAX_STREAM + 3) / 4; // the longest stream at the worst byte skew

// one warp per block.  S: value width in bytes.  Every length and offset is checked against the staged input and the
// block's output before it is used: a corrupt stream raises the flag and stores nothing.  DICT (S = 4, dictionary data
// pages): every decoded value is a code; it is checked against dict_size and replaced by dict[code] before the store.
template <int S, bool DICT>
__device__ __forceinline__ void bshuf_decode_blocks(const BshufBlock* __restrict__ blocks, long long num_blocks, uint8_t* __restrict__ out,
                                                    int32_t* __restrict__ flags, const int32_t* __restrict__ dict, uint32_t dict_size) {
    __shared__ uint32_t s_in[BSHUF_DECODE_WARPS][BSHUF_STAGE_WORDS];
    __shared__ uint8_t s_out[BSHUF_DECODE_WARPS][BSHUF_BLOCK_BYTES];
    constexpr int Q = (S + 7) / 8; // 64-bit words per value
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint8_t* o = s_out[wid];
    const long long stride = (long long)gridDim.x * BSHUF_DECODE_WARPS;
    for (long long bi = (long long)blockIdx.x * BSHUF_DECODE_WARPS + wid; bi < num_blocks; bi += stride) {
        const BshufBlock d = blocks[bi];
        if (d.elems == 0) continue; // (warp-uniform)
        // the stream -> shared memory: whole words from the aligned address below it (an aligned word never crosses a page
        // of the host mapping), the byte skew remembered
        const uintptr_t a0 = (uintptr_t)d.src & ~(uintptr_t)3;
        const uint32_t skew = (uint32_t)((uintptr_t)d.src - a0);
        const uint32_t nwords = (skew + d.clen + 3) / 4;
        __syncwarp();
        for (uint32_t i = lane; i < nwords; i += 32) s_in[wid][i] = (uint32_t)ldg_stream_s32((const uint32_t*)a0 + i);
        __syncwarp();
        const uint8_t* in = (const uint8_t*)s_in[wid] + skew;
        // LZ4 block decode (the end-of-block rules of bshuf_oracle.cpp).  Control flow depends only on bytes every lane reads
        // alike, so it is warp-uniform.
        const uint32_t n = d.clen, E = d.elems * S;
        uint32_t ip = 0, op = 0;
        bool ok = false;
        while (ip < n) {
            const uint32_t tok = in[ip++];
            uint32_t lit = tok >> 4;
            if (lit == 15 && !lz4_len(in, n, ip, lit, n)) break;
            if (lit > n - ip || lit > E - op) break;
            for (uint32_t k = lane; k < lit; k += 32) o[op + k] = in[ip + k];
            ip += lit;
            op += lit;
            if (ip == n) {
                ok = op == E;
                break;
            }
            if (op + 12 > E || n - ip < 2) break; // a match starts at least 12 bytes before the end
            const uint32_t off = (uint32_t)in[ip] | (uint32_t)in[ip + 1] << 8;
            ip += 2;
            if (off == 0 || off > op) break;
            uint32_t ml = tok & 15;
            if (ml == 15 && !lz4_len(in, n, ip, ml, E)) break;
            ml += 4;
            if (ml + 5 > E - op) break; // ... and ends at least 5 bytes before it
            __syncwarp();               // the bytes the match reads were written by other lanes
            // out[op + k] = out[op - off + (k mod off)]: reads only bytes before op, also when the match overlaps itself
            const uint32_t m0 = op - off;
            if (off >= ml) {
                for (uint32_t k = lane; k < ml; k += 32) o[op + k] = o[m0 + k];
            } else {
                for (uint32_t k = lane; k < ml; k += 32) o[op + k] = o[m0 + k % off];
            }
            op += ml;
        }
        if (!ok) {
            if (lane == 0) atomicOr(flags, 1);
            continue;
        }
        __syncwarp();
        // un-transpose: lane takes elements [8g, 8g + 8); byte j of them = the 8 x 8 transpose of byte g of rows 8j .. 8j + 7
        const uint32_t R = d.elems / 8;
        uint8_t* dst = out + d.row * S;
        bool bad = false;
        for (uint32_t g = lane; g < R; g += 32) {
            unsigned long long v[8][Q];
#pragma unroll
            for (int t = 0; t < 8; t++)
#pragma unroll
                for (int q = 0; q < Q; q++) v[t][q] = 0;
#pragma unroll
            for (int j = 0; j < S; j++) {
                unsigned long long x = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) x |= (unsigned long long)o[(8 * j + k) * R + g] << (8 * k);
                x = bshuf_trans8x8(x);
#pragma unroll
                for (int t = 0; t < 8; t++) v[t][j / 8] |= ((x >> (8 * t)) & 0xFF) << (8 * (j % 8));
            }
            if (DICT) {
                // code -> dict[code] through the read-only path (a low-cardinality table is <= 1 KB and stays in L1).  A code
                // outside the dictionary is a corrupt page: the reference's CPU decode would write 0 there silently.
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    const uint32_t c = (uint32_t)v[t][0];
                    const bool in = c < dict_size;
                    if (!in && 8 * g + t < d.n_out) bad = true; // padding is never stored
                    v[t][0] = in ? (uint32_t)__ldg(dict + c) : 0u;
                }
            }
            uint8_t* p = dst + (size_t)8 * g * S;
            if (8 * g + 8 <= d.n_out && ((uintptr_t)p & 7) == 0) {
                // the lane's 8 * S bytes as S little-endian 64-bit words; lanes are contiguous, so the warp's stores are too
                unsigned long long w[S];
#pragma unroll
                for (int m = 0; m < S; m++) {
                    if (S >= 8) {
                        w[m] = v[m / Q][m % Q];
                    } else {
                        w[m] = 0;
#pragma unroll
                        for (int q = 0; q < 8 / S; q++) w[m] |= v[m * (8 / S) + q][0] << (8 * S * q);
                    }
                }
                if (S >= 2 && ((uintptr_t)p & 15) == 0) {
#pragma unroll
                    for (int m = 0; m + 1 < S; m += 2) ((ulonglong2*)p)[m / 2] = make_ulonglong2(w[m], w[m + 1]);
                } else {
#pragma unroll
                    for (int m = 0; m < S; m++) ((unsigned long long*)p)[m] = w[m];
                }
            } else {
                // a partial group (the page's last), or a row offset that page boundaries left unaligned: value by value
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    if (8 * g + t >= d.n_out) break;
                    uint8_t* e = p + t * S;
                    if (S == 1) *e = (uint8_t)v[t][0];
                    else if (S == 2) *(uint16_t*)e = (uint16_t)v[t][0];
                    else if (S == 4) *(uint32_t*)e = (uint32_t)v[t][0];
                    else {
#pragma unroll
                        for (int q = 0; q < Q; q++) ((unsigned long long*)e)[q] = v[t][q];
                    }
                }
            }
        }
        if (DICT && __any_sync(SR_FULL_MASK, bad) && lane == 0) atomicOr(flags, 1); // (the block loop is warp-uniform)
    }
}

template <int S>
__global__ void __launch_bounds__(BSHUF_DECODE_WARPS * 32) k_bshuf_decode(const BshufBlock* __restrict__ blocks, long long num_blocks, uint8_t* __restrict__ out,
                                                                         int32_t* __restrict__ flags) {
    bshuf_decode_blocks<S, false>(blocks, num_blocks, out, flags, nullptr, 0);
}

// dictionary data pages: the bitshuffle blocks of int32 codes, each code translated through dict[0, dict_size)
__global__ void __launch_bounds__(BSHUF_DECODE_WARPS * 32) k_bshuf_decode_dict(const BshufBlock* __restrict__ blocks, long long num_blocks, int32_t* __restrict__ out,
                                                                              int32_t* __restrict__ flags, const int32_t* __restrict__ dict, uint32_t dict_size) {
    bshuf_decode_blocks<4, true>(blocks, num_blocks, (uint8_t*)out, flags, dict, dict_size);
}

// RLE at bit width 1 ----------------------------------------------------------------------------------------------------
// One run of a page's stream, clipped to the page's value count.  Runs are stored in stream order and cover the page's
// rows [0, covered) without gaps, so run j ends where run j + 1 starts (the last one at `covered`).
struct RleRun {
    const uint8_t* lit; // a bit-packed run: its bytes, value i at bit i % 8 of byte i / 8; nullptr: a repeated run
    uint32_t row;       // page row of the run's first value
    uint32_t value;     // a repeated run's value (0 or 1)
};

constexpr int RLE_RUNS_BLOCK = 128;
constexpr int RLE_STAGE_BYTES = 4096;

// one CTA per page: the page's bytes pass through shared memory in windows (coalesced word loads -- one pass over HBM or
// PCIe), thread 0 walks the run headers (RleDecoder::ReadHeader) into descriptors at the page's frame_off.  counts[2p]: the
// page's values; counts[2p + 1]: room for descriptors (>= the runs a stream of the page's size can hold).  meta[p] = (runs,
// rows they cover).  The walk stops at the count and reads nothing past it; it raises the flag for a header longer than 5
// bytes or cut off by the end, a zero-length run, a repeated value other than 0 / 1, a run whose values up to the count
// lie past the end, and a stream that ends before the count.  empty_is_zero: a page of no bytes is a page without NULLs (a
// null map) instead of a stream that ends at once.
__global__ void __launch_bounds__(RLE_RUNS_BLOCK) k_rle_runs(const PageDesc* __restrict__ pages, const unsigned long long* __restrict__ counts, int32_t empty_is_zero,
                                                             RleRun* __restrict__ runs, uint2* __restrict__ meta, int32_t* __restrict__ flags) {
    __shared__ uint32_t s_buf[RLE_STAGE_BYTES / 4];
    __shared__ long long s_pos; // page byte the next window starts at; -1: the walk is over
    const PageDesc pg = pages[blockIdx.x];
    const unsigned long long n = counts[2 * blockIdx.x], cap = counts[2 * blockIdx.x + 1];
    RleRun* out = runs + pg.frame_off;
    unsigned long long done = 0; // thread 0's walk: values so far, runs so far
    uint32_t nr = 0;
    bool bad = false;
    if (threadIdx.x == 0) s_pos = (n == 0 || (pg.size == 0 && empty_is_zero)) ? -1 : 0;
    __syncthreads();
    for (;;) {
        const long long pos = s_pos;
        if (pos < 0) break;
        // bytes [pos, pos + avail) of the page -> shared memory, whole words from the aligned address below them
        const long long avail = max(0ll, min(pg.size - pos, (long long)RLE_STAGE_BYTES - 4));
        const bool last = pg.size - pos <= (long long)RLE_STAGE_BYTES - 4; // the window reaches the page's end
        const uintptr_t a0 = (uintptr_t)(pg.data + pos) & ~(uintptr_t)3;
        const uint32_t skew = (uint32_t)((uintptr_t)(pg.data + pos) - a0);
        const uint32_t nwords = avail > 0 ? (uint32_t)((skew + avail + 3) / 4) : 0;
        for (uint32_t i = threadIdx.x; i < nwords; i += RLE_RUNS_BLOCK) s_buf[i] = (uint32_t)ldg_stream_s32((const uint32_t*)a0 + i);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint8_t* b = (const uint8_t*)s_buf + skew; // b[k]: page byte pos + k, k < avail
            long long k = 0, next = -1;
            while (done < n) {
                if (!last && avail - k < 6) { // a header (<= 5 bytes) and a repeated value may cross the window: move it
                    next = pos + k;
                    break;
                }
                unsigned long long h = 0;
                bool more = true;
                for (int hb = 0; hb < 5 && more && k < avail; hb++) {
                    const uint32_t c = b[k++];
                    h |= (unsigned long long)(c & 0x7F) << (7 * hb);
                    more = (c & 0x80) != 0;
                }
                const unsigned long long len = h >> 1, left = n - done;
                if (more || len == 0 || nr >= cap) { // cut off or longer than 5 bytes; a zero-length run
                    bad = true;
                    break;
                }
                RleRun r;
                r.row = (uint32_t)done;
                r.value = 0;
                if (h & 1) { // bit-packed: len groups of 8 values, one byte each; only the groups up to the count are read
                    const unsigned long long take = min(8 * len, left);
                    if (pos + k + (long long)((take + 7) / 8) > pg.size) {
                        bad = true;
                        break;
                    }
                    r.lit = pg.data + pos + k;
                    k += (long long)len;
                    done += take;
                } else { // repeated: len copies of one byte
                    if (k >= avail || b[k] > 1) {
                        bad = true;
                        break;
                    }
                    r.lit = nullptr;
                    r.value = b[k++];
                    done += min(len, left);
                }
                out[nr++] = r;
            }
            s_pos = next;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        meta[blockIdx.x] = make_uint2(nr, (uint32_t)done);
        if (bad) atomicOr(flags, 1);
    }
}

// 8 flags (bit i of b) -> 8 bytes of 0 / 1, flag i in byte i
__device__ __forceinline__ unsigned long long rle_expand8(uint32_t b) {
    return (((((unsigned long long)b * 0x0101010101010101ull) & 0x8040201008040201ull) + 0x00406070787C7E7Full) >> 7) & 0x0101010101010101ull;
}

constexpr int RLE_EXPAND_BLOCK = 256;

// grid (x, page): every thread makes one aligned 8-byte word of the output at a time: the run holding the word's first row
// by a binary search of the page's runs, then the bits of that run and the ones after it (a bit-packed run gives its bits
// straight from its bytes, a repeated run its value 8 times), expanded into bytes and stored as one 64-bit word; the page's
// first and last words, shared with its neighbours, byte by byte.  Rows past the runs' coverage (an empty null map) are 0.
// null_count (optional): += the 1s stored, a popcount per thread summed per warp.
__global__ void __launch_bounds__(RLE_EXPAND_BLOCK) k_rle_expand(const PageDesc* __restrict__ pages, const unsigned long long* __restrict__ counts,
                                                                 const RleRun* __restrict__ runs, const uint2* __restrict__ meta, uint8_t* __restrict__ out,
                                                                 unsigned long long* __restrict__ null_count) {
    const int p = blockIdx.y;
    const PageDesc pg = pages[p];
    const long long n = (long long)counts[2 * p];
    const uint2 m = meta[p];
    const RleRun* rr = runs + pg.frame_off;
    uint8_t* dst = out + pg.row_off;
    const long long skew = (long long)((uintptr_t)dst & 7);
    const long long nw = (skew + n + 7) / 8; // words the page's rows touch
    uint32_t ones = 0;
    for (long long w = (long long)blockIdx.x * RLE_EXPAND_BLOCK + threadIdx.x; w < nw; w += (long long)gridDim.x * RLE_EXPAND_BLOCK) {
        const long long r0 = 8 * w - skew; // page row of the word's byte 0
        const long long lo = max(r0, 0ll), hi = min(r0 + 8, n);
        uint32_t bits = 0; // bit r - lo: row r
        int j = -1;
        for (int a = 0, b = (int)m.x - 1; a <= b;) { // the last run starting at or before lo
            const int c = (a + b) >> 1;
            if ((long long)rr[c].row <= lo) {
                j = c;
                a = c + 1;
            } else {
                b = c - 1;
            }
        }
        for (long long r = lo; j >= 0 && (uint32_t)j < m.x && r < hi;) {
            const RleRun run = rr[j];
            const long long end = min(hi, (long long)((uint32_t)j + 1 < m.x ? rr[j + 1].row : m.y));
            if (r >= end) break; // past the runs' coverage (a stream refused part way)
            uint32_t v;
            if (run.lit) {
                const uint32_t off = (uint32_t)(r - run.row), i = off >> 3;
                v = run.lit[i];
                if ((off & 7) + (end - r) > 8) v |= (uint32_t)run.lit[i + 1] << 8;
                v >>= off & 7;
            } else {
                v = run.value ? 0xFFu : 0u;
            }
            bits |= (v & ((1u << (end - r)) - 1u)) << (r - lo);
            r = end;
            j++;
        }
        ones += __popc(bits);
        if (lo == r0 && hi == r0 + 8) {
            *(unsigned long long*)(dst + r0) = rle_expand8(bits);
        } else {
            const unsigned long long x = rle_expand8(bits << (lo - r0));
            for (long long r = lo; r < hi; r++) dst[r] = (uint8_t)(x >> (8 * (r - r0)));
        }
    }
    if (null_count) {
        ones = __reduce_add_sync(SR_FULL_MASK, ones);
        if ((threadIdx.x & 31) == 0 && ones) atomicAdd(null_count, (unsigned long long)ones);
    }
}

constexpr int NULL_COUNT_BLOCK = 256;

// bitshuffle null maps, after k_bshuf_decode<1>: grid (x, page): a page without a map (size 0) gets zeros, every other
// page's flags are counted (nonzero bytes; a popcount per thread summed per warp into null_count).  16-byte words where the
// page's rows cover them, bytes at its two ends.
__global__ void __launch_bounds__(NULL_COUNT_BLOCK) k_null_zero_count(const PageDesc* __restrict__ pages, const unsigned long long* __restrict__ counts, uint8_t* __restrict__ out,
                                                                      unsigned long long* __restrict__ null_count) {
    const int p = blockIdx.y;
    const PageDesc pg = pages[p];
    const long long n = (long long)counts[2 * p];
    const bool zero = pg.size == 0;
    uint8_t* dst = out + pg.row_off;
    const long long skew = (long long)((uintptr_t)dst & 15);
    const long long nw = (skew + n + 15) / 16;
    uint32_t ones = 0;
    for (long long w = (long long)blockIdx.x * NULL_COUNT_BLOCK + threadIdx.x; w < nw; w += (long long)gridDim.x * NULL_COUNT_BLOCK) {
        const long long r0 = 16 * w - skew;
        if (r0 >= 0 && r0 + 16 <= n) {
            uint4* q = (uint4*)(dst + r0);
            if (zero) {
                *q = make_uint4(0, 0, 0, 0);
            } else {
                const uint4 x = *q;
                const uint32_t y[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int t = 0; t < 4; t++) ones += __popc((((y[t] & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | y[t]) & 0x80808080u); // nonzero bytes
            }
        } else {
            for (long long r = max(r0, 0ll); r < min(r0 + 16, n); r++) {
                if (zero) dst[r] = 0;
                else ones += dst[r] != 0;
            }
        }
    }
    ones = __reduce_add_sync(SR_FULL_MASK, ones);
    if ((threadIdx.x & 31) == 0 && ones) atomicAdd(null_count, (unsigned long long)ones);
}

} // namespace srd

// host side ------------------------------------------------------------------------------------------------------------
struct PageScratch {
    DevBuf pages, frames, counts, flags, blob;
    PinnedBuf host_pages, host_counts;
};

// where the kernels read the pages: hp[p].data / .size of every page in sc->host_pages (the caller sets row_off / frame_off).
// View: sr_page_view or sr_null_map_view (data, size).
template <typename View>
static int32_t stage_pages(sr_ctx* ctx, PageScratch* sc, const View* pv, int32_t num_pages, int32_t mem) {
    if (!sc->host_pages.reserve(sizeof(srd::PageDesc) * (size_t)num_pages) || !sc->host_counts.reserve(16 * (size_t)num_pages + 16))
        return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "page tables");
    srd::PageDesc* hp = (srd::PageDesc*)sc->host_pages.p;
    // Host pages that lie back to back (a page cache hands out slices of large buffers) are merged into RUNS: one copy per
    // run instead of one per page.
    for (int p = 0; p < num_pages; p++)
        if (pv[p].size < 0 || (pv[p].size > 0 && !pv[p].data)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "page %d", p);
    struct Run {
        const uint8_t* begin;
        size_t bytes;
        int first, last;
    };
    std::vector<Run> runs;
    if (mem_is_host(mem)) {
        for (int p = 0; p < num_pages; p++) {
            const uint8_t* d = (const uint8_t*)pv[p].data;
            if (!runs.empty() && pv[p].size > 0 && d >= runs.back().begin + runs.back().bytes && d < runs.back().begin + runs.back().bytes + 64) {
                runs.back().bytes = (size_t)(d - runs.back().begin) + (size_t)pv[p].size;
                runs.back().last = p;
            } else {
                runs.push_back(Run{d, (size_t)pv[p].size, p, p});
            }
        }
    }
    size_t total_bytes = 0;
    for (auto& r : runs) total_bytes += r.bytes;
    // page-locked pages: long runs are copied by the DMA engines at full PCIe speed (measured: 52 GB/s against ~30 GB/s for
    // the decode kernel's word-sized reads over the bus); scattered pages are read in place (no staging buffer, no extra pass)
    const bool stage = mem == SR_MEM_HOST || (mem == SR_MEM_HOST_PINNED && !runs.empty() && total_bytes / runs.size() >= (256u << 10));
    if (stage) {
        size_t blob = 0;
        for (auto& r : runs) blob += (r.bytes + 15) & ~(size_t)15;
        SR_TRY(sc->blob.reserve(ctx, blob + 16));
        size_t at = 0;
        for (auto& r : runs) {
            if (r.bytes > 0) SR_CUDA(ctx, cudaMemcpyAsync((uint8_t*)sc->blob.p + at, r.begin, r.bytes, cudaMemcpyHostToDevice, ctx->stream));
            for (int p = r.first; p <= r.last; p++) {
                hp[p].data = (const uint8_t*)sc->blob.p + at + ((const uint8_t*)pv[p].data - r.begin);
                hp[p].size = pv[p].size;
            }
            at += (r.bytes + 15) & ~(size_t)15;
        }
    } else {
        PinnedResolver pinned;
        for (int p = 0; p < num_pages; p++) {
            const void* d = pv[p].data;
            if (mem == SR_MEM_HOST_PINNED && pv[p].size > 0) SR_TRY(pinned.resolve(ctx, pv[p].data, (size_t)pv[p].size, p, &d));
            hp[p].data = (const uint8_t*)d;
            hp[p].size = pv[p].size;
        }
    }
    return SR_OK;
}

// RLE streams at bit width 1 (sc->pages and sc->counts on the device: values, room for runs; `runs` descriptors in all)
// -> flags in out.  null_count: see k_rle_expand.
static int32_t rle_launch(sr_ctx* ctx, PageScratch* sc, int32_t num_pages, long long runs, long long max_rows, int32_t empty_is_zero, uint8_t* out,
                          unsigned long long* null_count) {
    SR_TRY(sc->frames.reserve(ctx, sizeof(srd::RleRun) * (size_t)runs + sizeof(uint2) * (size_t)num_pages));
    srd::RleRun* rr = (srd::RleRun*)sc->frames.p;
    uint2* meta = (uint2*)(rr + runs);
    const srd::PageDesc* pages = (const srd::PageDesc*)sc->pages.p;
    const unsigned long long* counts = sc->counts.as<unsigned long long>();
    srd::k_rle_runs<<<num_pages, srd::RLE_RUNS_BLOCK, 0, ctx->stream>>>(pages, counts, empty_is_zero, rr, meta, (int32_t*)sc->flags.p);
    SR_LAUNCH_CHECK(ctx);
    // about two words per thread of the longest page
    const int gx = (int)std::min<long long>(std::max<long long>((max_rows + 16 * srd::RLE_EXPAND_BLOCK - 1) / (16 * srd::RLE_EXPAND_BLOCK), 1), 64);
    for (int p0 = 0; p0 < num_pages; p0 += 65535) { // gridDim.y is limited to 65535
        srd::k_rle_expand<<<dim3(gx, std::min(num_pages - p0, 65535)), srd::RLE_EXPAND_BLOCK, 0, ctx->stream>>>(pages + p0, counts + 2 * (size_t)p0, rr, meta + p0, out, null_count);
        SR_LAUNCH_CHECK(ctx);
    }
    return SR_OK;
}

// dict / dict_words: the decoder's code -> value table (device memory; dict_words < 0: none set), read by SR_PAGE_DICT only
static int32_t pages_decode(sr_ctx* ctx, PageScratch* sc, int32_t encoding, int32_t type, const sr_page_view* pv, int32_t num_pages, int32_t mem, void* out,
                            int64_t out_capacity, int64_t* out_rows, const int32_t* dict, long long dict_words) {
    const int w = srd::type_width(type);
    if (encoding == SR_PAGE_DICT) {
        if (type != SR_TYPE_INT) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "dictionary page decode of type %d (TYPE_INT ids)", type);
        if (dict_words < 0) return sr_fail(ctx, SR_ERR_STATE, "dictionary pages decoded before sr_page_decoder_set_dict");
    } else if (encoding == SR_PAGE_BITSHUFFLE) {
        if (w == 0) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "bitshuffle page decode of type %d (fixed-width types)", type);
    } else if (encoding == SR_PAGE_RLE) {
        if (type != SR_TYPE_BOOLEAN) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "page encoding %d of type %d (RLE pages: BOOLEAN)", encoding, type);
    } else {
        if ((w != 4 && w != 8) || srd::is_float_class(type)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "page decode of type %d (4- and 8-byte integer-class types)", type);
        if (encoding != SR_PAGE_PLAIN && encoding != SR_PAGE_FOR) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "page encoding %d", encoding);
    }
    // one rule for every encoding: k_for_decode and the bitshuffle kernels store whole values where a lane's address is not
    // vector-aligned, so a column off its natural alignment would be a misaligned store (plain pages follow the same rule)
    if ((uintptr_t)out % std::min(w, 8)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "output column not aligned to %d bytes", std::min(w, 8));
    if (num_pages < 0 || (num_pages > 0 && !pv)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "pages");
    SR_TRY(mem_check(ctx, mem, "pages"));
    *out_rows = 0;
    if (num_pages == 0) return SR_OK;
    SR_TRY(stage_pages(ctx, sc, pv, num_pages, mem));
    srd::PageDesc* hp = (srd::PageDesc*)sc->host_pages.p;
    SR_TRY(sc->pages.reserve(ctx, sizeof(srd::PageDesc) * (size_t)num_pages));
    SR_TRY(sc->counts.reserve(ctx, 16 * (size_t)num_pages));
    SR_TRY(sc->flags.reserve(ctx, 16));
    SR_CUDA(ctx, cudaMemsetAsync(sc->flags.p, 0, 16, ctx->stream));
    SR_CUDA(ctx, cudaMemcpyAsync(sc->pages.p, hp, sizeof(srd::PageDesc) * (size_t)num_pages, cudaMemcpyHostToDevice, ctx->stream));
    srd::k_page_footers<<<grid_for(num_pages, 256), 256, 0, ctx->stream>>>((const srd::PageDesc*)sc->pages.p, num_pages, encoding, w, sc->counts.as<unsigned long long>(),
                                                                           (int32_t*)sc->flags.p);
    SR_LAUNCH_CHECK(ctx);
    unsigned long long* hc = (unsigned long long*)sc->host_counts.p;
    SR_CUDA(ctx, cudaMemcpyAsync(hc, sc->counts.p, 16 * (size_t)num_pages, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaMemcpyAsync(hc + 2 * (size_t)num_pages, sc->flags.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int32_t hflags = *(const int32_t*)(hc + 2 * (size_t)num_pages);
    if (hflags & 1)
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "a page is not a well-formed %s page",
                       encoding == SR_PAGE_FOR ? "frame-of-reference" : encoding == SR_PAGE_PLAIN ? "plain" : encoding == SR_PAGE_DICT ? "dictionary data"
                                                    : encoding == SR_PAGE_RLE ? "RLE" : "bitshuffle");
    if (hflags & 2) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "a dictionary data page in plain mode: the column fell back to plain pages");
    long long rows = 0, frames = 0, max_rows = 0;
    for (int p = 0; p < num_pages; p++) {
        // past the mode word: the bitshuffle page of codes (k_bshuf_blocks reads it as is); past an RLE page's value count
        if (encoding == SR_PAGE_DICT || encoding == SR_PAGE_RLE) {
            hp[p].data += 4;
            hp[p].size -= 4;
        }
        hp[p].row_off = rows;
        hp[p].frame_off = frames;
        rows += (long long)hc[2 * p];
        frames += (long long)hc[2 * p + 1];
        max_rows = std::max(max_rows, (long long)hc[2 * p]);
    }
    if (rows > out_capacity) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "the pages hold %lld values, the output column has room for %lld", rows, (long long)out_capacity);
    *out_rows = rows;
    if (rows == 0) return SR_OK;
    if (!out) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "null output");
    SR_CUDA(ctx, cudaMemcpyAsync(sc->pages.p, hp, sizeof(srd::PageDesc) * (size_t)num_pages, cudaMemcpyHostToDevice, ctx->stream));
    if (encoding == SR_PAGE_PLAIN) {
        for (int p0 = 0; p0 < num_pages; p0 += 65535) { // gridDim.y is limited to 65535
            srd::k_plain_copy<<<dim3(32, std::min(num_pages - p0, 65535)), 256, 0, ctx->stream>>>((const srd::PageDesc*)sc->pages.p + p0, w, (uint8_t*)out);
            SR_LAUNCH_CHECK(ctx);
        }
        return SR_OK;
    }
    if (encoding == SR_PAGE_RLE) {
        SR_TRY(rle_launch(ctx, sc, num_pages, frames, max_rows, 0, (uint8_t*)out, nullptr));
        SR_CUDA(ctx, cudaMemcpyAsync(hc, sc->flags.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (*(const int32_t*)hc) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "an RLE page has a malformed run stream");
        return SR_OK;
    }
    if (encoding == SR_PAGE_BITSHUFFLE || encoding == SR_PAGE_DICT) {
        SR_TRY(sc->frames.reserve(ctx, sizeof(srd::BshufBlock) * (size_t)frames));
        srd::BshufBlock* blocks = (srd::BshufBlock*)sc->frames.p;
        srd::k_bshuf_blocks<<<grid_for(num_pages, 256), 256, 0, ctx->stream>>>((const srd::PageDesc*)sc->pages.p, num_pages, w, 16, sc->counts.as<unsigned long long>(), blocks,
                                                                               (int32_t*)sc->flags.p);
        SR_LAUNCH_CHECK(ctx);
        const int bgrid = (int)std::min<long long>((frames + srd::BSHUF_DECODE_WARPS - 1) / srd::BSHUF_DECODE_WARPS, (long long)ctx->num_sms * 8);
        int32_t* flags = (int32_t*)sc->flags.p;
        if (encoding == SR_PAGE_DICT) {
            srd::k_bshuf_decode_dict<<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (int32_t*)out, flags, dict, (uint32_t)dict_words);
        } else {
            switch (w) {
            case 1: srd::k_bshuf_decode<1><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (uint8_t*)out, flags); break;
            case 2: srd::k_bshuf_decode<2><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (uint8_t*)out, flags); break;
            case 4: srd::k_bshuf_decode<4><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (uint8_t*)out, flags); break;
            case 8: srd::k_bshuf_decode<8><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (uint8_t*)out, flags); break;
            default: srd::k_bshuf_decode<16><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, (uint8_t*)out, flags); break;
            }
        }
        SR_LAUNCH_CHECK(ctx);
        // a block chain that leaves its page (k_bshuf_blocks) or a corrupt LZ4 stream (k_bshuf_decode)
        SR_CUDA(ctx, cudaMemcpyAsync(hc, sc->flags.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (*(const int32_t*)hc)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, encoding == SR_PAGE_DICT ? "a dictionary data page has a corrupt block chain or LZ4 stream, or a code outside the dictionary"
                                                                                : "a bitshuffle page has a corrupt block chain or LZ4 stream");
        return SR_OK;
    }
    SR_TRY(sc->frames.reserve(ctx, sizeof(srd::FrameDesc) * (size_t)frames));
    const int dgrid = (int)std::min<long long>((frames + srd::FOR_DECODE_WARPS - 1) / srd::FOR_DECODE_WARPS, (long long)ctx->num_sms * 8);
    if (w == 4) {
        srd::k_for_frames<int32_t><<<num_pages, srd::FOR_FRAMES_BLOCK, 0, ctx->stream>>>((const srd::PageDesc*)sc->pages.p, (srd::FrameDesc*)sc->frames.p, (int32_t*)sc->flags.p);
        SR_LAUNCH_CHECK(ctx);
        srd::k_for_decode<int32_t><<<dgrid, srd::FOR_DECODE_BLOCK, 0, ctx->stream>>>((const srd::FrameDesc*)sc->frames.p, frames, (int32_t*)out);
    } else {
        srd::k_for_frames<long long><<<num_pages, srd::FOR_FRAMES_BLOCK, 0, ctx->stream>>>((const srd::PageDesc*)sc->pages.p, (srd::FrameDesc*)sc->frames.p, (int32_t*)sc->flags.p);
        SR_LAUNCH_CHECK(ctx);
        srd::k_for_decode<long long><<<dgrid, srd::FOR_DECODE_BLOCK, 0, ctx->stream>>>((const srd::FrameDesc*)sc->frames.p, frames, (long long*)out);
    }
    SR_LAUNCH_CHECK(ctx);
    // a frame table that points outside its page is only seen by k_for_frames: report it (the frame was skipped)
    SR_CUDA(ctx, cudaMemcpyAsync(hc, sc->flags.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*(const int32_t*)hc) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "a frame-of-reference page has a corrupt frame table");
    return SR_OK;
}

// the null maps of a run of data pages -> uint8 flags (1 = NULL) in out, page k's after page k - 1's
static int32_t null_maps_decode(sr_ctx* ctx, PageScratch* sc, int32_t encoding, const sr_null_map_view* maps, int32_t num_pages, int32_t mem, uint8_t* out,
                                int64_t out_capacity, int64_t* out_rows, int64_t* out_null_count) {
    if (encoding != SR_NULL_BITSHUFFLE && encoding != SR_NULL_RLE) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "null map encoding %d", encoding);
    if (num_pages < 0 || (num_pages > 0 && !maps)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "null maps");
    SR_TRY(mem_check(ctx, mem, "null maps"));
    *out_rows = 0;
    *out_null_count = 0;
    // every row count is the page footer's: the whole layout is known before anything is copied
    long long rows = 0, max_rows = 0;
    for (int p = 0; p < num_pages; p++) {
        if (maps[p].size < 0 || (maps[p].size > 0 && !maps[p].data) || maps[p].num_rows < 0 || maps[p].num_rows > (int64_t)UINT32_MAX)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "null map %d: %lld bytes, %lld rows", p, (long long)maps[p].size, (long long)maps[p].num_rows);
        rows += maps[p].num_rows;
        max_rows = std::max(max_rows, (long long)maps[p].num_rows);
    }
    if (rows > out_capacity) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "the null maps hold %lld rows, the output column has room for %lld", rows, (long long)out_capacity);
    if (rows > 0 && !out) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "null output");
    if (num_pages == 0) return SR_OK;
    SR_TRY(stage_pages(ctx, sc, maps, num_pages, mem));
    srd::PageDesc* hp = (srd::PageDesc*)sc->host_pages.p;
    unsigned long long* hc = (unsigned long long*)sc->host_counts.p;
    long long frames = 0, at = 0;
    for (int p = 0; p < num_pages; p++) {
        const unsigned long long n = (unsigned long long)maps[p].num_rows, size = (unsigned long long)maps[p].size;
        hp[p].row_off = at;
        hp[p].frame_off = frames;
        hc[2 * p] = n;
        // bitshuffle: the blocks of ALIGN_UP(n, 8) one-byte flags (none for an absent map); RLE: room for every run the map can hold
        hc[2 * p + 1] = encoding == SR_NULL_BITSHUFFLE ? (size ? ((n + 7) / 8 * 8 + srd::BSHUF_BLOCK_BYTES - 1) / srd::BSHUF_BLOCK_BYTES : 0) : std::min(n, size / 2);
        at += (long long)n;
        frames += (long long)hc[2 * p + 1];
    }
    SR_TRY(sc->pages.reserve(ctx, sizeof(srd::PageDesc) * (size_t)num_pages));
    SR_TRY(sc->counts.reserve(ctx, 16 * (size_t)num_pages));
    SR_TRY(sc->flags.reserve(ctx, 16));
    SR_CUDA(ctx, cudaMemsetAsync(sc->flags.p, 0, 16, ctx->stream)); // the error flag, then the null count
    SR_CUDA(ctx, cudaMemcpyAsync(sc->pages.p, hp, sizeof(srd::PageDesc) * (size_t)num_pages, cudaMemcpyHostToDevice, ctx->stream));
    SR_CUDA(ctx, cudaMemcpyAsync(sc->counts.p, hc, 16 * (size_t)num_pages, cudaMemcpyHostToDevice, ctx->stream));
    int32_t* flags = (int32_t*)sc->flags.p;
    unsigned long long* null_count = (unsigned long long*)((uint8_t*)sc->flags.p + 8);
    if (encoding == SR_NULL_RLE) {
        SR_TRY(rle_launch(ctx, sc, num_pages, frames, max_rows, 1, out, null_count));
    } else {
        // a map is bitshuffle::compress_lz4 of the padded flags: a BIT_SHUFFLE page of one-byte values without its header
        const srd::PageDesc* pages = (const srd::PageDesc*)sc->pages.p;
        SR_TRY(sc->frames.reserve(ctx, sizeof(srd::BshufBlock) * (size_t)frames));
        srd::BshufBlock* blocks = (srd::BshufBlock*)sc->frames.p;
        srd::k_bshuf_blocks<<<grid_for(num_pages, 256), 256, 0, ctx->stream>>>(pages, num_pages, 1, 0, sc->counts.as<unsigned long long>(), blocks, flags);
        SR_LAUNCH_CHECK(ctx);
        if (frames > 0) {
            const int bgrid = (int)std::min<long long>((frames + srd::BSHUF_DECODE_WARPS - 1) / srd::BSHUF_DECODE_WARPS, (long long)ctx->num_sms * 8);
            srd::k_bshuf_decode<1><<<bgrid, srd::BSHUF_DECODE_WARPS * 32, 0, ctx->stream>>>(blocks, frames, out, flags);
            SR_LAUNCH_CHECK(ctx);
        }
        const int gx = (int)std::min<long long>(std::max<long long>((max_rows + 32 * srd::NULL_COUNT_BLOCK - 1) / (32 * srd::NULL_COUNT_BLOCK), 1), 64);
        for (int p0 = 0; p0 < num_pages; p0 += 65535) { // gridDim.y is limited to 65535
            srd::k_null_zero_count<<<dim3(gx, std::min(num_pages - p0, 65535)), srd::NULL_COUNT_BLOCK, 0, ctx->stream>>>(pages + p0, sc->counts.as<unsigned long long>() + 2 * (size_t)p0,
                                                                                                                       out, null_count);
            SR_LAUNCH_CHECK(ctx);
        }
    }
    unsigned long long* back = hc + 2 * (size_t)num_pages; // the 16 spare bytes of host_counts
    SR_CUDA(ctx, cudaMemcpyAsync(back, sc->flags.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*(const int32_t*)back)
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, encoding == SR_NULL_RLE ? "a null map has a malformed RLE stream" : "a null map has a corrupt block chain or LZ4 stream");
    *out_rows = rows;
    *out_null_count = (int64_t)back[1];
    return SR_OK;
}
