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

// value count and frame count of every page; flags[0] |= 1 when a page cannot be a frame-of-reference / plain page
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
    } else {
        if (pg.size < 5) {
            bad = true;
        } else {
            const uint32_t fsz = pg.data[pg.size - 5];
            n = page_le32(pg.data + pg.size - 4);
            if (fsz != 128 && n != 0) bad = true; // every writer uses ForEncoder::FRAME_VALUE_NUM = 128
            frames = (n + 127) / 128;
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
    const uint32_t nf = (n + 127) / 128;
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

} // namespace srd

// host side ------------------------------------------------------------------------------------------------------------
struct PageScratch {
    DevBuf pages, frames, counts, flags, blob;
    PinnedBuf host_pages, host_counts;
};

static int32_t pages_decode(sr_ctx* ctx, PageScratch* sc, int32_t encoding, int32_t type, const sr_page_view* pv, int32_t num_pages, int32_t mem, void* out,
                            int64_t out_capacity, int64_t* out_rows) {
    const int w = srd::type_width(type);
    if ((w != 4 && w != 8) || srd::is_float_class(type)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "page decode of type %d (4- and 8-byte integer-class types)", type);
    if (encoding != SR_PAGE_PLAIN && encoding != SR_PAGE_FOR) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "page encoding %d", encoding);
    if (num_pages < 0 || (num_pages > 0 && !pv)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "pages");
    if (mem != SR_MEM_HOST && mem != SR_MEM_DEVICE && mem != SR_MEM_HOST_PINNED) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown memory kind %d", mem);
    *out_rows = 0;
    if (num_pages == 0) return SR_OK;
    if (!sc->host_pages.reserve(sizeof(srd::PageDesc) * (size_t)num_pages) || !sc->host_counts.reserve(16 * (size_t)num_pages + 16))
        return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "page tables");
    srd::PageDesc* hp = (srd::PageDesc*)sc->host_pages.p;
    // where the kernels read the pages.  Host pages that lie back to back (a page cache hands out slices of large buffers) are
    // merged into RUNS: one copy per run instead of one per page.
    for (int p = 0; p < num_pages; p++)
        if (pv[p].size < 0 || (pv[p].size > 0 && !pv[p].data)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "page %d", p);
    struct Run {
        const uint8_t* begin;
        size_t bytes;
        int first, last;
    };
    std::vector<Run> runs;
    if (mem != SR_MEM_DEVICE) {
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
        for (int p = 0; p < num_pages; p++) {
            const void* d = pv[p].data;
            if (mem == SR_MEM_HOST_PINNED && pv[p].size > 0) SR_TRY(Staged::mapped_alias(ctx, pv[p].data, p, &d));
            hp[p].data = (const uint8_t*)d;
            hp[p].size = pv[p].size;
        }
    }
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
    if (*(const int32_t*)(hc + 2 * (size_t)num_pages)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "a page is not a well-formed %s page", encoding == SR_PAGE_FOR ? "frame-of-reference" : "plain");
    long long rows = 0, frames = 0;
    for (int p = 0; p < num_pages; p++) {
        hp[p].row_off = rows;
        hp[p].frame_off = frames;
        rows += (long long)hc[2 * p];
        frames += (long long)hc[2 * p + 1];
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
