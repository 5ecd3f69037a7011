// sr_gather.cuh -- the chunk-list form of the fragment push (sr_fragment_push_chunks): k_chunk_gather copies the columns
// of many small chunks (device memory, or page-locked host memory read over PCIe) into one contiguous device batch in
// one launch; ChunkGather launches it and gather_pieces cuts a column into its descriptor entries.
#pragma once

#include "sr_host.cuh"

namespace srd {

constexpr int CHUNK_GATHER_BLOCK = 256;
constexpr int CHUNK_GATHER_VECS = 4;                                                          // 16-byte vectors per thread
constexpr uint32_t CHUNK_GATHER_PIECE = CHUNK_GATHER_BLOCK * CHUNK_GATHER_VECS * 16;         // bytes per descriptor entry

// one descriptor entry: `bytes` (<= CHUNK_GATHER_PIECE) from `src` to `dst`; src == nullptr writes zeros (the null column
// of a chunk without one, in a batch column that is nullable)
struct GatherPiece {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t bytes;
    uint32_t pad;
};

// bytes [p, p + 16) of the 32 bytes a:b (little endian), 0 < p < 16: funnel shifts of neighbouring words
__device__ __forceinline__ int4 gather_shift(const int4 a, const int4 b, uint32_t p) {
    uint32_t w0, w1, w2, w3, w4;
    switch (p >> 2) {
    case 0: w0 = a.x, w1 = a.y, w2 = a.z, w3 = a.w, w4 = b.x; break;
    case 1: w0 = a.y, w1 = a.z, w2 = a.w, w3 = b.x, w4 = b.y; break;
    case 2: w0 = a.z, w1 = a.w, w2 = b.x, w3 = b.y, w4 = b.z; break;
    default: w0 = a.w, w1 = b.x, w2 = b.y, w3 = b.z, w4 = b.w; break;
    }
    const uint32_t r = (p & 3) * 8;
    return make_int4((int)__funnelshift_r(w0, w1, r), (int)__funnelshift_r(w1, w2, r), (int)__funnelshift_r(w2, w3, r), (int)__funnelshift_r(w3, w4, r));
}

// One CTA per entry (grid-stride over the table).  The destination is split into a byte head up to its first 16-byte
// boundary, 16-byte vectors, and a byte tail.  Every vector is stored with one 16-byte store; its source is read with
// aligned 16-byte loads: one per vector when source and destination share the phase mod 16, else the vector is funnel
// shifted out of two neighbouring aligned loads, the second taken from the next lane (lane 31 and the last vector load
// it themselves).  Each thread issues all its loads before the first store, so a CTA keeps CHUNK_GATHER_PIECE bytes of
// mapped host memory in flight over PCIe.  An aligned load may cover up to 15 bytes outside the source range, inside
// the same 16-byte block: never a page the source does not touch.
__global__ void __launch_bounds__(CHUNK_GATHER_BLOCK) k_chunk_gather(const GatherPiece* __restrict__ pieces, int32_t num_pieces) {
    const int t = threadIdx.x;
    const int lane = t & 31;
    for (int32_t e = blockIdx.x; e < num_pieces; e += gridDim.x) {
        const GatherPiece pc = pieces[e];
        const uint32_t n = pc.bytes;
        const uint32_t head = min(n, (uint32_t)(16 - ((uintptr_t)pc.dst & 15)) & 15u);
        const uint32_t nvec = (n - head) >> 4;
        const uint32_t tail = head + nvec * 16;
        if (t < (int)head) pc.dst[t] = pc.src ? pc.src[t] : 0;
        if (t < (int)(n - tail)) pc.dst[tail + t] = pc.src ? pc.src[tail + t] : 0;
        int4* dst = (int4*)(pc.dst + head);
        if (!pc.src) {
            for (uint32_t v = t; v < nvec; v += CHUNK_GATHER_BLOCK) dst[v] = make_int4(0, 0, 0, 0);
            continue;
        }
        const uintptr_t sp = (uintptr_t)(pc.src + head);
        const uint32_t p = (uint32_t)(sp & 15);
        const int4* src = (const int4*)(sp - p);
        int4 a[CHUNK_GATHER_VECS], b[CHUNK_GATHER_VECS];
#pragma unroll
        for (int k = 0; k < CHUNK_GATHER_VECS; k++) {
            const uint32_t v = (uint32_t)(k * CHUNK_GATHER_BLOCK + t);
            a[k] = v < nvec ? ldg_stream_v4(src + v) : make_int4(0, 0, 0, 0);
            b[k] = (p != 0 && v < nvec && (lane == 31 || v == nvec - 1)) ? ldg_stream_v4(src + v + 1) : make_int4(0, 0, 0, 0);
        }
        if (p == 0) {
#pragma unroll
            for (int k = 0; k < CHUNK_GATHER_VECS; k++) {
                const uint32_t v = (uint32_t)(k * CHUNK_GATHER_BLOCK + t);
                if (v < nvec) dst[v] = a[k];
            }
        } else {
#pragma unroll
            for (int k = 0; k < CHUNK_GATHER_VECS; k++) {
                const uint32_t v = (uint32_t)(k * CHUNK_GATHER_BLOCK + t);
                int4 nb;
                nb.x = __shfl_down_sync(SR_FULL_MASK, a[k].x, 1);
                nb.y = __shfl_down_sync(SR_FULL_MASK, a[k].y, 1);
                nb.z = __shfl_down_sync(SR_FULL_MASK, a[k].z, 1);
                nb.w = __shfl_down_sync(SR_FULL_MASK, a[k].w, 1);
                if (lane == 31 || v == nvec - 1) nb = b[k];
                if (v < nvec) dst[v] = gather_shift(a[k], nb, p);
            }
        }
    }
}

} // namespace srd

// What one fragment keeps for sr_fragment_push_chunks: the gathered batch columns, the descriptor table on the device
// and the page-locked copies of the table it is uploaded from.  An upload buffer is rewritten only once the copy out of
// it has run (its event), so a call never waits for the work an earlier call queued.
struct ChunkGather {
    ColBufs cols;
    DevBuf table;
    struct Upload {
        PinnedBuf buf;
        cudaEvent_t ev = nullptr;
    };
    std::vector<Upload> uploads;
    ~ChunkGather() {
        for (auto& u : uploads)
            if (u.ev) cudaEventDestroy(u.ev);
    }
    // queues the H2D copy of `pieces` into `table` and the gather launch
    int32_t launch(sr_ctx* ctx, const std::vector<srd::GatherPiece>& pieces) {
        if (pieces.empty()) return SR_OK;
        const size_t bytes = pieces.size() * sizeof(srd::GatherPiece);
        Upload* up = nullptr;
        for (auto& u : uploads)
            if (cudaEventQuery(u.ev) == cudaSuccess) {
                up = &u;
                break;
            }
        cudaGetLastError(); // cudaErrorNotReady of the busy ones
        if (!up) {
            uploads.emplace_back();
            up = &uploads.back();
            SR_CUDA(ctx, cudaEventCreateWithFlags(&up->ev, cudaEventDisableTiming));
        }
        if (!up->buf.reserve(bytes)) return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "page-locked gather table of %zu bytes", bytes);
        memcpy(up->buf.p, pieces.data(), bytes);
        SR_TRY(table.reserve(ctx, bytes));
        SR_CUDA(ctx, cudaMemcpyAsync(table.p, up->buf.p, bytes, cudaMemcpyHostToDevice, ctx->stream));
        SR_CUDA(ctx, cudaEventRecord(up->ev, ctx->stream));
        const int grid = (int)std::min<size_t>(pieces.size(), (size_t)ctx->num_sms * 8);
        srd::k_chunk_gather<<<grid, srd::CHUNK_GATHER_BLOCK, 0, ctx->stream>>>(table.as<srd::GatherPiece>(), (int32_t)pieces.size());
        SR_LAUNCH_CHECK(ctx);
        return SR_OK;
    }
};

// appends the entries that move `bytes` from `src` (nullptr: zeros) to `dst`, cut into pieces of at most
// CHUNK_GATHER_PIECE bytes; source and destination advance together, so every piece keeps the phase of the whole
static inline void gather_pieces(std::vector<srd::GatherPiece>* out, const void* src, void* dst, size_t bytes) {
    for (size_t off = 0; off < bytes; off += srd::CHUNK_GATHER_PIECE) {
        const uint32_t n = (uint32_t)std::min<size_t>(srd::CHUNK_GATHER_PIECE, bytes - off);
        out->push_back(srd::GatherPiece{src ? (const uint8_t*)src + off : nullptr, (uint8_t*)dst + off, n, 0});
    }
}
