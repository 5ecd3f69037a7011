// sr_gpu.cu -- C-ABI of libsr_gpu.so (include/sr_gpu_ops.h).  One translation unit: the device
// code lives in the headers included below.  sm_90a only; there is no CPU fallback: without a
// CUDA device every entry point fails with SR_ERR_NO_DEVICE / SR_ERR_CUDA.
#include "sr_frag.cuh"
#include "sr_serde.cuh"
#include "sr_page.cuh"

// ---------------------------------------------------------------------------------------
// exchange: hash partition (K18).  exchange_sink_operator.cpp:586-637, shuffler.h:72-89,
// column_hash.cpp:138-300
// ---------------------------------------------------------------------------------------
namespace srd {

struct PartCols {
    DCol c[SR_MAX_PART_KEYS];
    int32_t n;
    int32_t hash_fn;
    int32_t reduce;
    int32_t num_channels;
};

__device__ __forceinline__ uint32_t part_hash_row(const PartCols& pc, int64_t row) {
    uint32_t h = pc.hash_fn == SR_HASH_FNV ? 0x811C9DC5u : pc.hash_fn == SR_HASH_XXH3 ? 0x9E3779B1u : 0u; // FNV_SEED / XXH3_SEED_32
    for (int k = 0; k < pc.n; k++) {
        const DCol& c = pc.c[k];
        if (c.nulls && c.nulls[row]) {
            if (pc.hash_fn == SR_HASH_CRC32)
                h = zlib_crc32_bytes(0, 0, 4, h); // NULL hashed as int32 0 (column_hash.cpp:262-266)
            else
                h = h ^ (0x9e3779b9u + (h << 6) + (h >> 2)); // :270
            continue;
        }
        uint64_t lo = 0, hi = 0;
        switch (c.width) {
        case 1:
            lo = ((const uint8_t*)c.data)[row];
            break;
        case 2:
            lo = ((const uint16_t*)c.data)[row];
            break;
        case 4:
            lo = (uint32_t)ldg_stream_s32((const int32_t*)c.data + row);
            break;
        case 8:
            lo = (uint64_t)ldg_stream_s64((const int64_t*)c.data + row);
            break;
        default:
            lo = ((const uint64_t*)c.data)[2 * row];
            hi = ((const uint64_t*)c.data)[2 * row + 1];
            break;
        }
        h = pc.hash_fn == SR_HASH_FNV    ? fnv_hash_bytes(lo, hi, c.width, h)
            : pc.hash_fn == SR_HASH_XXH3 ? (uint32_t)xxh3_64_value(lo, hi, c.width, (uint64_t)h)
                                         : zlib_crc32_bytes(lo, hi, c.width, h);
    }
    return h;
}

constexpr int PART_BLOCK = 256;
constexpr int PART_ITEMS = 4;
constexpr int PART_TILE = PART_BLOCK * PART_ITEMS;
constexpr int PART_MAX_CH = 256;

// hash + channel per row, per-tile channel histogram written channel-major: counts[c * tiles + tile]
__global__ void __launch_bounds__(PART_BLOCK) k_part_hash(PartCols pc, int64_t n, uint32_t* __restrict__ hash_values, uint32_t* __restrict__ channel_ids,
                                                           uint32_t* __restrict__ counts, int64_t tiles) {
    __shared__ uint32_t s_hist[PART_MAX_CH];
    for (int c = threadIdx.x; c < pc.num_channels; c += PART_BLOCK) s_hist[c] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * PART_TILE;
#pragma unroll
    for (int k = 0; k < PART_ITEMS; k++) {
        const int64_t row = base + k * PART_BLOCK + threadIdx.x;
        if (row < n) {
            const uint32_t h = part_hash_row(pc, row);
            const uint32_t ch = pc.reduce == SR_REDUCE_MULHI ? reduce_op(h, (uint32_t)pc.num_channels) : h % (uint32_t)pc.num_channels;
            if (hash_values) hash_values[row] = h;
            channel_ids[row] = ch;
            if (counts) atomicAdd(&s_hist[ch], 1u);
        }
    }
    if (counts) {
        __syncthreads();
        for (int c = threadIdx.x; c < pc.num_channels; c += PART_BLOCK) counts[(int64_t)c * tiles + blockIdx.x] = s_hist[c];
    }
}

// stable scatter of row indexes: rows of channel c land at [offsets[c*tiles+tile], ...) in input order
__global__ void __launch_bounds__(PART_BLOCK) k_part_scatter(const uint32_t* __restrict__ channel_ids, int64_t n, int32_t num_channels,
                                                              const uint64_t* __restrict__ offsets, int64_t tiles, uint32_t* __restrict__ row_index) {
    __shared__ uint64_t s_base[PART_MAX_CH];
    __shared__ uint32_t s_cnt[PART_BLOCK / 32][PART_MAX_CH];
    for (int c = threadIdx.x; c < num_channels; c += PART_BLOCK) s_base[c] = offsets[(int64_t)c * tiles + blockIdx.x];
    const int w = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * PART_TILE;
#pragma unroll 1
    for (int k = 0; k < PART_ITEMS; k++) {
        for (int c = threadIdx.x; c < (PART_BLOCK / 32) * num_channels; c += PART_BLOCK) s_cnt[c / num_channels][c % num_channels] = 0;
        __syncthreads();
        const int64_t row = base + k * PART_BLOCK + threadIdx.x;
        const bool valid = row < n;
        const uint32_t vmask = __ballot_sync(SR_FULL_MASK, valid);
        uint32_t ch = 0, rank = 0;
        if (valid) {
            ch = channel_ids[row];
            const uint32_t peers = __match_any_sync(vmask, ch);
            rank = __popc(peers & lanemask_lt());
            if (rank == 0) s_cnt[w][ch] = __popc(peers);
        }
        __syncthreads();
        if (valid) {
            uint64_t pos = s_base[ch] + rank;
            for (int q = 0; q < w; q++) pos += s_cnt[q][ch];
            row_index[pos] = (uint32_t)row;
        }
        __syncthreads();
        for (int c = threadIdx.x; c < num_channels; c += PART_BLOCK) {
            uint32_t t = 0;
            for (int q = 0; q < PART_BLOCK / 32; q++) t += s_cnt[q][c];
            s_base[c] += t;
        }
        __syncthreads();
    }
}

// read-only bandwidth probe: 128-bit loads, xor-reduced so the loads cannot be elided
__global__ void __launch_bounds__(512) k_bandwidth_probe(const int4* __restrict__ p, int64_t n16, unsigned long long* __restrict__ out) {
    int4 acc = make_int4(0, 0, 0, 0);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const int4 a = ldg_stream_v4(p + i), b = ldg_stream_v4(p + i + stride), c = ldg_stream_v4(p + i + 2 * stride), d = ldg_stream_v4(p + i + 3 * stride);
        acc.x ^= a.x ^ b.x ^ c.x ^ d.x;
        acc.y ^= a.y ^ b.y ^ c.y ^ d.y;
        acc.z ^= a.z ^ b.z ^ c.z ^ d.z;
        acc.w ^= a.w ^ b.w ^ c.w ^ d.w;
    }
    for (; i < n16; i += stride) {
        const int4 a = ldg_stream_v4(p + i);
        acc.x ^= a.x;
        acc.y ^= a.y;
        acc.z ^= a.z;
        acc.w ^= a.w;
    }
    unsigned long long v = ((unsigned long long)(uint32_t)(acc.x ^ acc.z) << 32) | (uint32_t)(acc.y ^ acc.w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(SR_FULL_MASK, v, o);
    if (lane_id() == 0) atomicXor(out, v);
}

} // namespace srd

struct sr_xchg {
    sr_ctx* ctx = nullptr;
    sr_part_desc desc;
    Staged staged;
    DevBuf hash_values, channel_ids, counts, offsets, row_index;
    ScanScratch scan_scratch;
    ColBufs out_cols;
};

extern "C" {

int32_t sr_abi_version(void) {
    return SR_ABI_VERSION;
}

int32_t sr_type_width(int32_t type) {
    return srd::type_width(type);
}

sr_ctx* sr_ctx_create(int32_t device, void* cuda_stream) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        sr_fail(nullptr, SR_ERR_NO_DEVICE, "no CUDA device available (%s); libsr_gpu has no CPU fallback", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
        return nullptr;
    }
    if (device < 0 || device >= count) {
        sr_fail(nullptr, SR_ERR_INVALID_ARGUMENT, "device %d out of range (%d devices)", device, count);
        return nullptr;
    }
    if ((e = cudaSetDevice(device)) != cudaSuccess) {
        sr_fail(nullptr, SR_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
        return nullptr;
    }
    // late materialisation touches single 32-byte sectors of the later columns: do not let L2 widen those
    // misses to 64/128-byte fetches (a hint; harmless where unsupported)
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
    cudaGetLastError();
    sr_ctx* ctx = new sr_ctx();
    ctx->device = device;
    if (cuda_stream) {
        ctx->stream = (cudaStream_t)cuda_stream;
    } else {
        if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
            sr_fail(nullptr, SR_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
            delete ctx;
            return nullptr;
        }
        ctx->own_stream = true;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->num_sms = prop.multiProcessorCount;
    if (cudaMallocHost((void**)&ctx->pinned, 64 * sizeof(uint64_t)) != cudaSuccess || cudaMalloc((void**)&ctx->dscratch, 64 * sizeof(uint64_t)) != cudaSuccess) {
        sr_fail(nullptr, SR_ERR_OUT_OF_MEMORY, "context scratch allocation failed");
        delete ctx;
        return nullptr;
    }
    cudaMemset(ctx->dscratch, 0, 64 * sizeof(uint64_t));
    return ctx;
}

void sr_ctx_destroy(sr_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    if (ctx->dscratch) cudaFree(ctx->dscratch);
    if (ctx->l2_flush) cudaFree(ctx->l2_flush);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int32_t sr_ctx_sync(sr_ctx* ctx) {
    if (!ctx) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(ctx);
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

const char* sr_last_error(sr_ctx* ctx) {
    return ctx ? ctx->err.c_str() : g_create_err.c_str();
}

int32_t sr_last_error_code(sr_ctx* ctx) {
    return ctx ? ctx->err_code : SR_ERR_INVALID_ARGUMENT;
}

int64_t sr_ctx_kernel_launches(sr_ctx* ctx) {
    return ctx ? ctx->launches : 0;
}
int64_t sr_ctx_device_bytes(sr_ctx* ctx) {
    return ctx ? ctx->dev_bytes : 0;
}
void* sr_ctx_stream(sr_ctx* ctx) {
    return ctx ? (void*)ctx->stream : nullptr;
}

// validates the context, takes its lock for the rest of the calling function and makes its device current
#define SR_BIND(ctx)                            \
    if (!(ctx)) return SR_ERR_INVALID_ARGUMENT; \
    SR_LOCK(ctx);                               \
    cudaSetDevice((ctx)->device)

// ------------------------------------------------------------------ pinned host memory + events (asynchronous adapters)
int32_t sr_host_alloc(sr_ctx* ctx, int64_t bytes, void** ptr) {
    SR_BIND(ctx);
    if (!ptr || bytes <= 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_host_alloc(%lld)", (long long)bytes);
    *ptr = nullptr;
    const cudaError_t e = cudaHostAlloc(ptr, (size_t)bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "cudaHostAlloc(%lld) failed: %s", (long long)bytes, cudaGetErrorString(e));
    }
    void* dev = nullptr;
    SR_CUDA(ctx, cudaHostGetDevicePointer(&dev, *ptr, 0));
    HostRegistry& reg = host_registry();
    std::lock_guard<std::mutex> lk(reg.mu);
    reg.ranges[(uintptr_t)*ptr] = HostRange{(size_t)bytes, (uintptr_t)dev, false};
    return SR_OK;
}

int32_t sr_host_free(sr_ctx* ctx, void* ptr) {
    SR_BIND(ctx);
    if (!ptr) return SR_OK;
    {
        HostRegistry& reg = host_registry();
        std::lock_guard<std::mutex> lk(reg.mu);
        auto it = reg.ranges.find((uintptr_t)ptr);
        if (it != reg.ranges.end() && !it->second.registered) reg.ranges.erase(it);
    }
    SR_CUDA(ctx, cudaFreeHost(ptr));
    return SR_OK;
}

int32_t sr_host_register(sr_ctx* ctx, void* ptr, int64_t bytes) {
    SR_BIND(ctx);
    if (!ptr || bytes <= 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_host_register(%p, %lld)", ptr, (long long)bytes);
    HostRegistry& reg = host_registry();
    std::lock_guard<std::mutex> lk(reg.mu);
    if (reg.overlaps((uintptr_t)ptr, (size_t)bytes))
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_host_register: [%p, +%lld) overlaps a page-locked range already known", ptr, (long long)bytes);
    cudaError_t e = cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return sr_fail(ctx, e == cudaErrorHostMemoryAlreadyRegistered || e == cudaErrorInvalidValue ? SR_ERR_INVALID_ARGUMENT : SR_ERR_CUDA,
                       "cudaHostRegister(%p, %lld) failed: %s", ptr, (long long)bytes, cudaGetErrorString(e));
    }
    void* dev = nullptr;
    if ((e = cudaHostGetDevicePointer(&dev, ptr, 0)) != cudaSuccess) {
        cudaGetLastError();
        cudaHostUnregister(ptr);
        return sr_fail(ctx, SR_ERR_CUDA, "cudaHostGetDevicePointer(%p) failed: %s", ptr, cudaGetErrorString(e));
    }
    reg.ranges[(uintptr_t)ptr] = HostRange{(size_t)bytes, (uintptr_t)dev, true};
    return SR_OK;
}

int32_t sr_host_unregister(sr_ctx* ctx, void* ptr) {
    SR_BIND(ctx);
    HostRegistry& reg = host_registry();
    std::lock_guard<std::mutex> lk(reg.mu);
    auto it = reg.ranges.find((uintptr_t)ptr);
    if (it == reg.ranges.end() || !it->second.registered) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_host_unregister(%p): not a range from sr_host_register", ptr);
    reg.ranges.erase(it);
    SR_CUDA(ctx, cudaHostUnregister(ptr));
    return SR_OK;
}

// no context lock and no driver call: the registry has its own
int32_t sr_host_is_mapped(sr_ctx* ctx, const void* ptr, int64_t bytes) {
    if (!ctx || bytes < 0) return SR_ERR_INVALID_ARGUMENT;
    HostRegistry& reg = host_registry();
    std::lock_guard<std::mutex> lk(reg.mu);
    return ptr && reg.find((uintptr_t)ptr, (size_t)bytes) ? 1 : 0;
}

struct sr_event {
    sr_ctx* ctx = nullptr;
    cudaEvent_t ev = nullptr;
    bool recorded = false;
};

sr_event* sr_event_create(sr_ctx* ctx) {
    if (!ctx) return nullptr;
    SR_LOCK(ctx);
    cudaSetDevice(ctx->device);
    sr_event* e = new sr_event();
    e->ctx = ctx;
    if (cudaEventCreateWithFlags(&e->ev, cudaEventDisableTiming) != cudaSuccess) {
        cudaGetLastError();
        sr_fail(ctx, SR_ERR_CUDA, "cudaEventCreate failed");
        delete e;
        return nullptr;
    }
    return e;
}

void sr_event_destroy(sr_event* e) {
    if (!e) return;
    SR_LOCK(e->ctx);
    cudaSetDevice(e->ctx->device);
    cudaEventDestroy(e->ev);
    delete e;
}

int32_t sr_event_record(sr_event* e) {
    if (!e) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(e->ctx);
    SR_CUDA(e->ctx, cudaEventRecord(e->ev, e->ctx->stream));
    e->recorded = true;
    return SR_OK;
}

// no lock: polled from the driver / poller thread while other threads are inside library calls (cudaEventQuery is thread-safe)
int32_t sr_event_query(sr_event* e) {
    if (!e) return SR_ERR_INVALID_ARGUMENT;
    if (!e->recorded) return 1;
    const cudaError_t r = cudaEventQuery(e->ev);
    if (r == cudaSuccess) return 1;
    if (r == cudaErrorNotReady) return 0;
    return SR_ERR_CUDA;
}

int32_t sr_event_sync(sr_event* e) {
    if (!e) return SR_ERR_INVALID_ARGUMENT;
    if (!e->recorded) return SR_OK;
    return cudaEventSynchronize(e->ev) == cudaSuccess ? SR_OK : SR_ERR_CUDA;
}

// ------------------------------------------------------------------ scan
sr_scan* sr_scan_create(sr_ctx* ctx, const sr_scan_desc* desc) {
    if (!ctx || !desc) return nullptr;
    if (desc->num_preds < 0 || desc->num_filter_exprs < 0 || desc->num_out_slots < 0 || desc->num_out_slots > SR_MAX_OUT_COLS) {
        sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "scan desc counts");
        return nullptr;
    }
    sr_scan* s = new sr_scan();
    s->ctx = ctx;
    s->preds.assign(desc->preds, desc->preds + desc->num_preds);
    s->exprs.assign(desc->filter_exprs, desc->filter_exprs + desc->num_filter_exprs);
    s->out_slots.assign(desc->out_slots, desc->out_slots + desc->num_out_slots);
    return s;
}

void sr_scan_destroy(sr_scan* scan) {
    if (!scan) return;
    SR_LOCK(scan->ctx);
    cudaSetDevice(scan->ctx->device);
    cudaStreamSynchronize(scan->ctx->stream);
    delete scan;
}

int32_t sr_scan_evaluate(sr_scan* s, const sr_chunk_view* in, uint8_t* selection, int32_t sel_mem) {
    if (!s || !in || !selection) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = s->ctx;
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, sel_mem, "sel_mem"));
    int64_t total;
    SR_TRY(scan_select(s, in, false, &total));
    SR_TRY(mem_out(ctx, selection, s->sel.p, (size_t)in->num_rows, sel_mem));
    return mem_sync(ctx, sel_mem);
}

int32_t sr_scan_filter(sr_scan* s, const sr_chunk_view* in, sr_chunk_out* out) {
    if (!s || !in || !out) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = s->ctx;
    SR_BIND(ctx);
    int64_t total = 0;
    SR_TRY(scan_select(s, in, true, &total));
    const int nout = (int)s->out_slots.size();
    s->out_cols.resize(nout);
    srd::CompactArgs ca;
    ca.n = 0;
    ColBufs::header(out, nout, total);
    for (int k = 0; k < nout; k++) {
        const int c = s->staged.find(s->out_slots[k]);
        if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses output slot %d", s->out_slots[k]);
        const srd::DCol& dc = s->staged.cols[c];
        void* data;
        uint8_t* nulls;
        SR_TRY(s->out_cols.reserve(ctx, k, total, dc.width, dc.nulls != nullptr, &data, &nulls));
        const int32_t vec16 = dc.width == 16 && (((uintptr_t)dc.data | (uintptr_t)data) & 15) == 0 ? 1 : 0;
        ca.c[ca.n++] = srd::CompactCol{dc.data, data, dc.width, vec16};
        if (nulls) ca.c[ca.n++] = srd::CompactCol{dc.nulls, nulls, 1, 0};
        s->out_cols.fill(out, k, dc.type, s->out_slots[k]);
    }
    if (total > 0 && ca.n > 0) {
        const int64_t tiles = (in->num_rows + srd::SCANW_TILE - 1) / srd::SCANW_TILE;
        const int grid = (int)std::min<int64_t>((tiles + srd::SCANW_BLOCK / 32 - 1) / (srd::SCANW_BLOCK / 32), (int64_t)ctx->num_sms * 8);
        if (total * 8 >= in->num_rows)
            srd::k_scan_compact<true><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(s->mask_bits.as<uint8_t>(), s->local_excl.as<uint32_t>(), s->block_offsets.as<uint64_t>(),
                                                                                   ca, in->num_rows);
        else
            srd::k_scan_compact<false><<<grid, srd::SCANW_BLOCK, 0, ctx->stream>>>(s->mask_bits.as<uint8_t>(), s->local_excl.as<uint32_t>(), s->block_offsets.as<uint64_t>(),
                                                                                    ca, in->num_rows);
        SR_LAUNCH_CHECK(ctx);
    }
    return SR_OK;
}

// ------------------------------------------------------------------ join
sr_join* sr_join_create(sr_ctx* ctx, const sr_join_desc* desc) {
    if (!ctx || !desc) return nullptr;
    if (join_validate_desc(ctx, desc) != SR_OK) return nullptr;
    sr_join* j = new sr_join();
    j->ctx = ctx;
    j->desc = *desc;
    int total = 0;
    for (int k = 0; k < desc->num_keys; k++) total += srd::type_width(desc->key_types[k]);
    j->wide = total > 8; // SERIALIZED_FIXED_SIZE_LARGEINT (join_hash_table.cpp:221-222)
    return j;
}

void sr_join_destroy(sr_join* join) {
    if (!join) return;
    SR_LOCK(join->ctx);
    cudaSetDevice(join->ctx->device);
    cudaStreamSynchronize(join->ctx->stream);
    delete join;
}

int32_t sr_join_append_build(sr_join* join, const sr_chunk_view* chunk) {
    if (!join || !chunk) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(join->ctx);
    return join_append(join, chunk);
}

int32_t sr_join_build_finish(sr_join* join) {
    if (!join) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(join->ctx);
    return join_finish(join);
}

int32_t sr_join_is_build_done(const sr_join* join) {
    return join && join->built ? 1 : 0;
}

int32_t sr_join_get_info(const sr_join* join, sr_join_info* info) {
    if (!join || !info) return SR_ERR_INVALID_ARGUMENT;
    info->method = join->method;
    info->has_duplicates = join->has_dup;
    info->build_rows = join->rows;
    info->bucket_size = join->bucket_size;
    info->min_value = join->min_value;
    info->max_value = join->max_value;
    return SR_OK;
}

int32_t sr_join_copy_table(sr_join* join, uint32_t* first_host, uint32_t* next_host) {
    if (!join) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = join->ctx;
    SR_BIND(ctx);
    if (!join->built) return sr_fail(ctx, SR_ERR_STATE, "copy_table before build_finish");
    if (first_host && join->bucket_size > 0)
        SR_CUDA(ctx, cudaMemcpyAsync(first_host, join->first.p, sizeof(uint32_t) * (size_t)join->bucket_size, cudaMemcpyDeviceToHost, ctx->stream));
    if (next_host) SR_CUDA(ctx, cudaMemcpyAsync(next_host, join->next.p, sizeof(uint32_t) * (size_t)(join->rows + 1), cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

int32_t sr_join_probe(sr_join* join, int32_t prober_id, const sr_chunk_view* probe, sr_chunk_out* out) {
    if (!join || !probe || !out) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(join->ctx);
    return join_probe(join, prober_id, probe, out);
}

int32_t sr_join_probe_remain(sr_join* join, sr_chunk_out* out) {
    if (!join || !out) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(join->ctx);
    return join_probe_remain(join, out);
}

int32_t sr_join_probe_indexes(sr_join* join, int32_t prober_id, const uint32_t** probe_index_dev, const uint32_t** build_index_dev) {
    if (!join) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(join->ctx);
    if (prober_id < 0 || prober_id >= (int)join->probers.size()) return SR_ERR_INVALID_ARGUMENT;
    if (probe_index_dev) *probe_index_dev = join->probers[prober_id]->probe_index.as<uint32_t>();
    if (build_index_dev) *build_index_dev = join->probers[prober_id]->build_index.as<uint32_t>();
    return SR_OK;
}

// ------------------------------------------------------------------ runtime filter
static int32_t rf_insert_dcol(sr_rf* rf, const srd::DCol& col, int64_t n, int32_t insert_nulls) {
    sr_ctx* ctx = rf->ctx;
    if (srd::type_width(col.type) > 8 || srd::is_float_class(col.type)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "runtime filter on column type %d", col.type);
    if (n <= 0) return SR_OK;
    rf->stats_valid = false;
    srd::k_rf_insert_col<<<std::min(grid_for(n, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(col, n, rf->log_num_buckets ? rf->dir.as<uint32_t>() : nullptr, rf->dir_mask,
                                                                                                 rf->log_num_buckets, insert_nulls ? 1 : 0, rf->stats.as<long long>());
    SR_LAUNCH_CHECK(ctx);
    // the IN part: while the build side stays within the row limit its keys are also kept as a sorted distinct list
    if (rf->in_enabled) {
        rf->in_rows += n;
        if (rf->in_rows > SR_RF_IN_FILTER_ROW_LIMIT) {
            rf->in_enabled = false;
            rf->in_host.clear();
        } else {
            const int w = srd::type_width(col.type);
            std::vector<uint8_t> raw((size_t)n * w), nul(col.nulls ? (size_t)n : 0);
            SR_CUDA(ctx, cudaMemcpyAsync(raw.data(), col.data, raw.size(), cudaMemcpyDeviceToHost, ctx->stream));
            if (col.nulls) SR_CUDA(ctx, cudaMemcpyAsync(nul.data(), col.nulls, nul.size(), cudaMemcpyDeviceToHost, ctx->stream));
            SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (int64_t i = 0; i < n; i++) {
                if (col.nulls && nul[i]) continue;
                long long v = 0;
                if (col.type == SR_TYPE_BOOLEAN)
                    v = raw[i];
                else if (w == 1)
                    v = (int8_t)raw[i];
                else if (w == 2)
                    v = ((const int16_t*)raw.data())[i];
                else if (w == 4)
                    v = ((const int32_t*)raw.data())[i];
                else
                    v = ((const long long*)raw.data())[i];
                rf->in_host.push_back(v);
            }
            std::sort(rf->in_host.begin(), rf->in_host.end());
            rf->in_host.erase(std::unique(rf->in_host.begin(), rf->in_host.end()), rf->in_host.end());
            rf->in_dirty = true;
        }
    }
    return SR_OK;
}

sr_rf* sr_rf_create(sr_ctx* ctx, int32_t key_type, int64_t expected_rows, int32_t with_bloom) {
    if (!ctx) return nullptr;
    cudaSetDevice(ctx->device);
    sr_rf* rf = new sr_rf();
    if (rf_init(rf, ctx, key_type, expected_rows, with_bloom) != SR_OK) {
        delete rf;
        return nullptr;
    }
    return rf;
}

void sr_rf_destroy(sr_rf* rf) {
    if (!rf) return;
    SR_LOCK(rf->ctx);
    cudaSetDevice(rf->ctx->device);
    cudaStreamSynchronize(rf->ctx->stream);
    delete rf;
}

int32_t sr_rf_insert(sr_rf* rf, const sr_chunk_view* in, int32_t slot_id, int32_t insert_nulls) {
    if (!rf || !in) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = rf->ctx;
    SR_BIND(ctx);
    const std::vector<int32_t> only{slot_id};
    SR_TRY(rf->staged.stage(ctx, in, &only));
    const int c = rf->staged.find(slot_id);
    if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses slot %d", slot_id);
    SR_TRY(rf_insert_dcol(rf, rf->staged.cols[c], in->num_rows, insert_nulls));
    return mem_sync(ctx, in->mem);
}

sr_rf* sr_join_build_runtime_filter(sr_join* join, int32_t key_index, int32_t with_bloom, int32_t insert_nulls) {
    if (!join) return nullptr;
    sr_ctx* ctx = join->ctx;
    SR_LOCK(ctx);
    cudaSetDevice(ctx->device);
    if (!join->built) {
        sr_fail(ctx, SR_ERR_STATE, "build_runtime_filter before build_finish");
        return nullptr;
    }
    if (key_index < 0 || key_index >= join->desc.num_keys) {
        sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "key_index %d", key_index);
        return nullptr;
    }
    sr_rf* rf = new sr_rf();
    // the directory is sized by the hash table's row count (hash_join_build_operator.cpp:140: ht_row_count)
    if (rf_init(rf, ctx, join->desc.key_types[key_index], join->rows, with_bloom) != SR_OK) {
        delete rf;
        return nullptr;
    }
    const BuildCol* bc = join->find_col(join->desc.build_key_slots[key_index]);
    if (bc && join->rows > 0) { // build columns keep the sentinel in row 0
        srd::DCol col;
        col.data = (const uint8_t*)bc->data.p + bc->width;
        col.nulls = bc->nullable ? bc->nulls.as<uint8_t>() + 1 : nullptr;
        col.type = bc->type;
        col.width = bc->width;
        if (rf_insert_dcol(rf, col, join->rows, insert_nulls) != SR_OK) {
            delete rf;
            return nullptr;
        }
    }
    return rf;
}

int32_t sr_rf_get_info(sr_rf* rf, sr_rf_info* info) {
    if (!rf || !info) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(rf->ctx);
    SR_TRY(rf_read_stats(rf));
    info->min_value = rf->hstats[0];
    info->max_value = rf->hstats[1];
    info->num_inserted = rf->hstats[2];
    info->has_null = rf->hstats[3] != 0;
    info->log_num_buckets = rf->log_num_buckets;
    info->key_type = rf->key_type;
    info->num_in_values = rf->in_enabled ? (int32_t)rf->in_host.size() : -1;
    return SR_OK;
}

int32_t sr_rf_copy_directory(sr_rf* rf, void* dst, int64_t bytes, int32_t mem) {
    if (!rf || (!dst && bytes > 0)) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = rf->ctx;
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, mem, "sr_rf_copy_directory"));
    if (bytes != (int64_t)rf->dir_bytes()) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "directory is %zu bytes, caller passed %lld", rf->dir_bytes(), (long long)bytes);
    SR_TRY(mem_out(ctx, dst, rf->dir.p, (size_t)bytes, mem));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

int32_t sr_rf_copy_in_values(sr_rf* rf, int64_t* values_host, int32_t capacity) {
    if (!rf) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(rf->ctx);
    if (!rf->in_enabled) return -1;
    const int32_t n = (int32_t)rf->in_host.size();
    if (n > capacity || (n > 0 && !values_host)) return sr_fail(rf->ctx, SR_ERR_INVALID_ARGUMENT, "IN list of %d values, capacity %d", n, capacity);
    for (int32_t i = 0; i < n; i++) values_host[i] = rf->in_host[i];
    return n;
}

int32_t sr_rf_merge_in_values(sr_rf* rf, const int64_t* values_host, int32_t n) {
    if (!rf || (n > 0 && !values_host)) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(rf->ctx);
    if (!rf->in_enabled) return SR_OK;
    if (n < 0) { // PartialRuntimeFilterMerger: one partial filter without an IN part -> the total has none
        rf->in_enabled = false;
        rf->in_host.clear();
        return SR_OK;
    }
    for (int32_t i = 0; i < n; i++) rf->in_host.push_back(values_host[i]);
    std::sort(rf->in_host.begin(), rf->in_host.end());
    rf->in_host.erase(std::unique(rf->in_host.begin(), rf->in_host.end()), rf->in_host.end());
    if ((int64_t)rf->in_host.size() > SR_RF_IN_FILTER_ROW_LIMIT) {
        rf->in_enabled = false;
        rf->in_host.clear();
    }
    rf->in_dirty = true;
    return SR_OK;
}

int32_t sr_rf_merge_directory(sr_rf* rf, const void* directory, int64_t bytes, int32_t mem, const sr_rf_info* other) {
    if (!rf || !other) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = rf->ctx;
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, mem, "sr_rf_merge_directory"));
    if (other->log_num_buckets != rf->log_num_buckets) // SimdBlockFilter::merge DCHECKs equal sizes
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "bloom directories of different size (2^%d vs 2^%d buckets)", rf->log_num_buckets, other->log_num_buckets);
    if (bytes != (int64_t)rf->dir_bytes() || (bytes > 0 && !directory)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "directory is %zu bytes, caller passed %lld", rf->dir_bytes(), (long long)bytes);
    if (!mem_is_host(mem) && !col_aligned(directory, 4)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "device directory at %p is not 4-byte aligned", directory);
    rf->stats_valid = false;
    if (bytes > 0) {
        DevBuf tmp;
        const void* src;
        SR_TRY(mem_in(ctx, directory, (size_t)bytes, mem, &tmp, &src));
        const int64_t words = bytes / 4;
        srd::k_or_u32<<<std::min(grid_for(words, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(rf->dir.as<uint32_t>(), (const uint32_t*)src, words);
        SR_LAUNCH_CHECK(ctx);
        SR_TRY(mem_sync(ctx, mem));
    }
    srd::k_rf_merge_stats<<<1, 1, 0, ctx->stream>>>(rf->stats.as<long long>(), other->min_value, other->max_value, other->num_inserted, other->has_null ? 1 : 0);
    SR_LAUNCH_CHECK(ctx);
    return SR_OK;
}

int32_t sr_rf_evaluate(sr_rf* rf, const sr_chunk_view* in, int32_t slot_id, uint8_t* selection, int32_t sel_mem, int32_t merge_and) {
    if (!rf || !in || (!selection && in->num_rows > 0)) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = rf->ctx;
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, in->mem, "chunk"));
    SR_TRY(mem_check(ctx, sel_mem, "sel_mem"));
    const int64_t n = in->num_rows;
    if (n <= 0) return SR_OK;
    const std::vector<int32_t> only{slot_id};
    SR_TRY(rf->staged.stage(ctx, in, &only));
    const int c = rf->staged.find(slot_id);
    if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses slot %d", slot_id);
    const srd::DCol& col = rf->staged.cols[c];
    if (srd::type_width(col.type) > 8 || srd::is_float_class(col.type)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "runtime filter on column type %d", col.type);
    srd::RfDev d;
    SR_TRY(rf_device_desc(rf, &d));
    DevBuf tmp;
    const void* dsel;
    SR_TRY(mem_in(ctx, selection, (size_t)n, sel_mem, &tmp, &dsel, merge_and != 0));
    srd::k_rf_evaluate<<<std::min(grid_for(n, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(d, col, n, (uint8_t*)dsel, merge_and ? 1 : 0);
    SR_LAUNCH_CHECK(ctx);
    SR_TRY(mem_out(ctx, selection, dsel, (size_t)n, sel_mem));
    if (mem_is_host(sel_mem) || mem_is_host(in->mem)) SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

int32_t sr_scan_add_runtime_filter(sr_scan* scan, sr_rf* rf, int32_t probe_slot) {
    if (!scan || !rf) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = scan->ctx;
    SR_LOCK(ctx);
    if (rf->ctx != ctx) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "runtime filter belongs to another context");
    if (scan->rfs.size() >= SR_MAX_SCAN_RFS) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "more than %d runtime filters on one scan", SR_MAX_SCAN_RFS);
    scan->rfs.emplace_back(rf, probe_slot);
    scan->compiled = false; // the probe column joins the value table at the next batch
    return SR_OK;
}

int32_t sr_scan_get_rf_stats(sr_scan* scan, int32_t index, sr_scan_rf_stats* stats) {
    if (!scan || !stats) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(scan->ctx);
    if (index < 0 || index >= (int32_t)scan->rfs.size()) return sr_fail(scan->ctx, SR_ERR_INVALID_ARGUMENT, "runtime filter index %d", index);
    memset(stats, 0, sizeof(*stats));
    if ((size_t)index < scan->rf_use.size()) {
        const sr_scan::RfUse& u = scan->rf_use[index];
        stats->rows_tested = (int64_t)u.tested;
        stats->rows_passed = (int64_t)u.passed;
        stats->batches_skipped = u.batches_skipped;
        stats->last_selectivity = u.last_selectivity;
    }
    return SR_OK;
}

int32_t sr_scan_set_rf_adaptive(sr_scan* scan, int32_t adaptive) {
    if (!scan) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(scan->ctx);
    scan->rf_adaptive = adaptive != 0;
    return SR_OK;
}

int32_t sr_join_key_hash(sr_ctx* ctx, const void* keys, int32_t key_type, int64_t n, uint32_t log_bucket_size, uint32_t* buckets, int32_t mem) {
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, mem, "sr_join_key_hash"));
    const int w = srd::type_width(key_type);
    if ((w != 4 && w != 8) || srd::is_float_class(key_type)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "sr_join_key_hash: 4- or 8-byte integer keys only");
    if (log_bucket_size < 1 || log_bucket_size > 31) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "log_bucket_size %u", log_bucket_size);
    if (n <= 0) return SR_OK;
    if (!mem_is_host(mem) && (!col_aligned(keys, w) || !col_aligned(buckets, 4)))
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_join_key_hash: device keys or buckets are not naturally aligned");
    DevBuf kin, kout;
    const void *dk, *dout;
    SR_TRY(mem_in(ctx, keys, (size_t)n * w, mem, &kin, &dk));
    SR_TRY(mem_in(ctx, buckets, (size_t)n * 4, mem, &kout, &dout, false));
    srd::k_join_key_hash<<<std::min(grid_for(n, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(dk, key_type, n, log_bucket_size, (uint32_t*)dout);
    SR_LAUNCH_CHECK(ctx);
    SR_TRY(mem_out(ctx, buckets, dout, (size_t)n * 4, mem));
    return mem_sync(ctx, mem);
}

// ------------------------------------------------------------------ aggregate
static bool desc_has_distinct(const sr_agg_desc* d) {
    for (int f = 0; f < d->num_fns; f++)
        if (d->fns[f].kind == SR_AGG_COUNT_DISTINCT) return true;
    return false;
}

sr_agg* sr_agg_create(sr_ctx* ctx, const sr_agg_desc* desc) {
    if (!ctx || !desc) return nullptr;
    if (agg_validate_desc(ctx, desc) != SR_OK) return nullptr;
    sr_agg* a = new sr_agg();
    a->ctx = ctx;
    a->desc = *desc;
    return a;
}

void sr_agg_destroy(sr_agg* agg) {
    if (!agg) return;
    SR_LOCK(agg->ctx);
    cudaSetDevice(agg->ctx->device);
    cudaStreamSynchronize(agg->ctx->stream);
    delete agg;
}

int32_t sr_agg_push(sr_agg* a, const sr_chunk_view* chunk) {
    if (!a || !chunk) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    if (a->finished) return sr_fail(ctx, SR_ERR_STATE, "push after sink_finish");
    SR_TRY(a->staged.stage(ctx, chunk));
    if (!a->compiled) SR_TRY(agg_compile(a, staged_slot_type, staged_slot_nullable, &a->staged));
    VTab vt;
    SR_TRY(bind_vtab(ctx, a->reg, a->staged, &vt));
    SR_TRY(agg_push_vtab(a, vt, chunk->num_rows));
    for (sr_agg* c : a->distinct) { // COUNT(DISTINCT) sets see the same (already staged) columns
        if (!c) continue;
        VTab cvt;
        SR_TRY(bind_vtab(ctx, c->reg, a->staged, &cvt));
        SR_TRY(agg_push_vtab(c, cvt, chunk->num_rows));
    }
    return SR_OK;
}

int32_t sr_agg_sink_finish(sr_agg* a) {
    if (!a) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(a->ctx);
    a->finished = true;
    return SR_OK;
}

int64_t sr_agg_num_groups(sr_agg* a) {
    if (!a) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(a->ctx);
    if (!a->finished) return sr_fail(a->ctx, SR_ERR_STATE, "num_groups before sink_finish");
    const int32_t rc = agg_finish_output(a);
    if (rc != SR_OK) return rc;
    return a->out_rows;
}

int32_t sr_agg_pull(sr_agg* a, int64_t max_rows, int32_t out_mem, sr_chunk_out* out) {
    if (!a || !out || max_rows <= 0) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    if (!a->finished) return sr_fail(ctx, SR_ERR_STATE, "pull before sink_finish");
    SR_TRY(mem_check(ctx, out_mem, "out_mem"));
    SR_TRY(agg_finish_output(a));
    const sr_agg_desc& d = a->desc;
    const int nc = d.num_group_keys + d.num_fns;
    const int64_t n = std::min<int64_t>(max_rows, a->out_rows - a->cursor);
    out->num_cols = nc;
    out->mem = mem_is_host(out_mem) ? SR_MEM_HOST : SR_MEM_DEVICE;
    out->num_rows = std::max<int64_t>(n, 0);
    if (mem_is_host(out_mem) && a->host_bufs.size() < 2 * (size_t)nc) a->host_bufs.resize(2 * (size_t)nc);
    for (int k = 0; k < nc; k++) {
        const int32_t type = a->out_rows > 0 || a->compiled ? a->out_types[k] : (k < d.num_group_keys ? d.group_types[k] : agg_result_type(d.fns[k - d.num_group_keys]));
        const int w = srd::type_width(type);
        out->cols[k].type = type;
        out->cols[k].slot_id = k < d.num_group_keys ? d.group_slots[k] : d.fns[k - d.num_group_keys].out_slot;
        out->cols[k].data = nullptr;
        out->cols[k].nulls = nullptr;
        if (n <= 0) continue;
        const ColBufs::Col& oc = a->out_cols.cols[k];
        const uint8_t* ddata = (const uint8_t*)oc.data.p + (size_t)a->cursor * w;
        const uint8_t* dnull = oc.nullable ? (const uint8_t*)oc.nulls.p + a->cursor : nullptr;
        if (!mem_is_host(out_mem)) {
            out->cols[k].data = (void*)ddata;
            out->cols[k].nulls = (uint8_t*)dnull;
        } else {
            if (!a->host_bufs[2 * k].reserve((size_t)n * w)) return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "pinned host buffer of %zu bytes", (size_t)n * w);
            SR_CUDA(ctx, cudaMemcpyAsync(a->host_bufs[2 * k].p, ddata, (size_t)n * w, cudaMemcpyDeviceToHost, ctx->stream));
            out->cols[k].data = a->host_bufs[2 * k].p;
            if (dnull) {
                if (!a->host_bufs[2 * k + 1].reserve((size_t)n)) return sr_fail(ctx, SR_ERR_OUT_OF_MEMORY, "pinned host buffer of %zu bytes", (size_t)n);
                SR_CUDA(ctx, cudaMemcpyAsync(a->host_bufs[2 * k + 1].p, dnull, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
                out->cols[k].nulls = (uint8_t*)a->host_bufs[2 * k + 1].p;
            }
        }
    }
    SR_TRY(mem_sync(ctx, out_mem));
    if (n > 0) a->cursor += n;
    return SR_OK;
}

static int32_t agg_reset_impl(sr_agg* a) {
    sr_ctx* ctx = a->ctx;
    a->finished = false;
    a->out_rows = -1;
    a->cursor = 0;
    a->ngroups_host = 0;
    a->table_touched = false;
    a->distinct_folded = false;
    for (sr_agg* c : a->distinct)
        if (c) SR_TRY(agg_reset_impl(c));
    if (!a->compiled) return SR_OK;
    SR_CUDA(ctx, cudaMemsetAsync(agg_counters(a), 0, sizeof(AggCounters), ctx->stream));
    return agg_init_tables(ctx, a->host);
}

int32_t sr_agg_reset(sr_agg* a) {
    if (!a) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(a->ctx);
    return agg_reset_impl(a);
}

int32_t sr_agg_dense_state(sr_agg* a, sr_agg_state_array* arrays, int32_t max_arrays, int32_t* num_arrays) {
    if (!a || !arrays || !num_arrays) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    *num_arrays = 0;
    if (a->out_rows >= 0) return sr_fail(ctx, SR_ERR_STATE, "dense state requested after the output was materialised");
    if (a->has_distinct) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) states are not element-wise mergeable");
    if (!a->compiled) return sr_fail(ctx, SR_ERR_STATE, "dense state requested before any input was pushed");
    const srd::AggDev& h = a->host;
    if (!h.dense && h.num_keys > 0) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "hash aggregate tables have no element-wise mergeable layout");
    srd::AccPtrs p;
    srd::acc_ptrs_global(h, p);
    int n = 0, unmergeable = -1;
    srd::agg_state_arrays(h, [&](int f, srd::AccWord w) {
        int32_t type = SR_TYPE_BIGINT, reduce = SR_STATE_SUM; // the counters and accn
        if (w == srd::W_ACC0) {
            switch (h.fns[f].mode) {
            case srd::M_SUM_F64:
            case srd::M_AVG:
                type = SR_TYPE_DOUBLE;
                break;
            case srd::M_MIN_I64:
            case srd::M_MIN_F64: // doubles are kept as their order-preserving int64 image
                reduce = SR_STATE_MIN;
                break;
            case srd::M_MAX_I64:
            case srd::M_MAX_F64:
                reduce = SR_STATE_MAX;
                break;
            case srd::M_SUM_I128:
                if (unmergeable < 0) unmergeable = f;
                break;
            default: // M_COUNT, M_SUM_I64
                break;
            }
        }
        if (n < max_arrays) arrays[n] = sr_agg_state_array{srd::acc_ptr(p, f, w), (int64_t)h.cap, type, reduce};
        n++;
    });
    if (unmergeable >= 0) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "aggregate function %d keeps a state that is not element-wise mergeable", unmergeable);
    if (n > max_arrays) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%d state arrays, room for %d", n, max_arrays);
    *num_arrays = n;
    return SR_OK;
}

// ---- two-phase / streaming aggregation ----
int32_t sr_agg_two_phase_descs(const sr_agg_desc* d, sr_agg_desc* p1, sr_agg_desc* p2) {
    if (!d || !p1 || !p2) return SR_ERR_INVALID_ARGUMENT;
    if (d->num_group_keys < 0 || d->num_group_keys > SR_MAX_GROUP_KEYS || d->num_fns < 0 || d->num_fns > SR_MAX_AGG_FNS) return SR_ERR_INVALID_ARGUMENT;
    if (desc_has_distinct(d)) return SR_ERR_NOT_SUPPORTED; // plan it as GROUP BY (keys, value) below a COUNT, like the reference's FE does
    *p1 = *d;
    *p2 = *d;
    p1->num_fns = 0;
    const auto state_col = [](int32_t slot) {
        sr_expr e;
        memset(&e, 0, sizeof(e));
        e.nodes[0].op = SR_EX_COL;
        e.nodes[0].slot_id = slot;
        e.num_nodes = 1;
        return e;
    };
    for (int f = 0; f < d->num_fns; f++) {
        const sr_agg_fn& fn = d->fns[f];
        sr_agg_fn& m = p2->fns[f];
        memset(&m, 0, sizeof(m));
        m.out_slot = fn.out_slot;
        if (fn.kind == SR_AGG_AVG_MERGE) return SR_ERR_INVALID_ARGUMENT; // already a merge phase
        if (fn.kind != SR_AGG_COUNT && fn.kind != SR_AGG_COUNT_STAR && fn.kind != SR_AGG_AVG && srd::type_width(agg_result_type(fn)) > 8)
            return SR_ERR_NOT_SUPPORTED; // 128-bit states (decimal / LARGEINT sums) cannot be read back as an input column yet
        if (p1->num_fns + (fn.kind == SR_AGG_AVG ? 2 : 1) > SR_MAX_AGG_FNS) return SR_ERR_NOT_SUPPORTED;
        if (fn.kind == SR_AGG_AVG) {
            // first phase: SUM(double(x)) + COUNT(x)  (the two halves of AvgAggregateState, avg.h:62-66)
            sr_agg_fn& s1 = p1->fns[p1->num_fns++];
            s1 = fn;
            s1.kind = SR_AGG_SUM;
            s1.reserved = 0;
            if (!srd::is_float_class(fn.input_type)) {
                if (s1.input.num_nodes >= SR_MAX_EXPR_NODES) return SR_ERR_NOT_SUPPORTED;
                s1.input.nodes[s1.input.num_nodes].op = SR_EX_TO_DOUBLE;
                s1.input.num_nodes++;
                s1.input_type = SR_TYPE_DOUBLE;
            }
            sr_agg_fn& c1 = p1->fns[p1->num_fns++];
            c1 = fn;
            c1.kind = SR_AGG_COUNT;
            c1.reserved = 0;
            c1.out_slot = SR_AGG_STATE_SLOT(fn.out_slot);
            m.kind = SR_AGG_AVG_MERGE;
            m.input_type = SR_TYPE_DOUBLE;
            m.input = state_col(fn.out_slot);
            m.reserved = SR_AGG_STATE_SLOT(fn.out_slot);
            continue;
        }
        p1->fns[p1->num_fns++] = fn;
        m.input = state_col(fn.out_slot);
        switch (fn.kind) {
        case SR_AGG_COUNT:
        case SR_AGG_COUNT_STAR: // counts are summed (CountAggregateFunction::merge, count.h:60-64)
            m.kind = SR_AGG_SUM;
            m.input_type = SR_TYPE_BIGINT;
            break;
        case SR_AGG_SUM:
            m.kind = SR_AGG_SUM;
            m.input_type = agg_result_type(fn); // BIGINT or DOUBLE
            break;
        default: // MIN / MAX of the partial extrema
            m.kind = fn.kind;
            m.input_type = fn.input_type;
            break;
        }
    }
    for (int f = p1->num_fns; f < SR_MAX_AGG_FNS; f++) memset(&p1->fns[f], 0, sizeof(sr_agg_fn));
    return SR_OK;
}

int64_t sr_agg_current_groups(sr_agg* a) {
    if (!a) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    if (!a->compiled || a->host.dense || a->host.num_keys == 0) return 0;
    AggCounters st;
    SR_TRY(agg_read_status(a, &st));
    return (int64_t)st.ngroups;
}

// the body of sr_agg_convert_to_states; *vt_out receives the bound value table of the staged chunk
static int32_t agg_convert_impl(sr_agg* a, const sr_chunk_view* chunk, sr_chunk_out* out, VTab* vt_out) {
    sr_ctx* ctx = a->ctx;
    const sr_agg_desc& d = a->desc;
    if (desc_has_distinct(&d)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) has no intermediate state column");
    for (int f = 0; f < d.num_fns; f++)
        if (d.fns[f].kind == SR_AGG_AVG || d.fns[f].kind == SR_AGG_AVG_MERGE)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "convert_to_states needs a first-phase desc (sr_agg_two_phase_descs): fn %d is AVG", f);
    SR_TRY(a->staged.stage(ctx, chunk));
    if (!a->compiled) SR_TRY(agg_compile(a, staged_slot_type, staged_slot_nullable, &a->staged));
    VTab vt;
    SR_TRY(bind_vtab(ctx, a->reg, a->staged, &vt));
    SR_TRY(agg_check_nullability(a, vt));
    if (vt_out) *vt_out = vt;
    const int64_t n = chunk->num_rows;
    const srd::AggDev& h = a->host;
    a->conv_cols.resize(d.num_fns);
    ColBufs::header(out, d.num_group_keys + d.num_fns, n);
    for (int k = 0; k < d.num_group_keys; k++) { // group-by columns travel as they are (device copies of the staged input)
        const int c = a->staged.find(d.group_slots[k]);
        if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses group slot %d", d.group_slots[k]);
        out->cols[k].data = (void*)a->staged.cols[c].data;
        out->cols[k].nulls = (uint8_t*)a->staged.cols[c].nulls;
        out->cols[k].type = a->staged.cols[c].type;
        out->cols[k].slot_id = d.group_slots[k];
    }
    srd::ConvertArgs ca;
    memset(&ca, 0, sizeof(ca));
    for (int f = 0; f < d.num_fns; f++) {
        const srd::AggFnDev& fn = h.fns[f];
        const int32_t type = fn.result_type;
        const int w = srd::type_width(type);
        if (w > 8) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fn %d: 128-bit states in the intermediate format", f);
        const bool nullable = !(fn.mode == srd::M_COUNT || fn.mode == srd::M_COUNT_STAR);
        void* data;
        uint8_t* nulls;
        SR_TRY(a->conv_cols.reserve(ctx, f, n, w, nullable, &data, &nulls));
        ca.c[f] = srd::ConvertCol{data, nulls, w, type};
        out->cols[d.num_group_keys + f] = sr_col_out{data, nulls, type, d.fns[f].out_slot};
    }
    if (n > 0 && d.num_fns > 0) {
        srd::k_agg_convert_states<<<std::min(grid_for(n, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, vt, n, ca);
        SR_LAUNCH_CHECK(ctx);
    }
    return SR_OK;
}

int32_t sr_agg_convert_to_states(sr_agg* a, const sr_chunk_view* chunk, sr_chunk_out* out) {
    if (!a || !chunk || !out) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    SR_TRY(agg_convert_impl(a, chunk, out, nullptr));
    return mem_sync(ctx, chunk->mem);
}

// SELECTIVE_PREAGG leg of the streaming aggregate (aggregate_streaming_sink_operator.cpp:173-210)
int32_t sr_agg_push_selective(sr_agg* a, const sr_chunk_view* chunk, sr_chunk_out* out) {
    if (!a || !chunk || !out) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    if (a->finished) return sr_fail(ctx, SR_ERR_STATE, "push after sink_finish");
    VTab vt;
    SR_TRY(agg_convert_impl(a, chunk, out, &vt)); // every row's intermediate form; compacted to the streamed rows below
    const int64_t n = chunk->num_rows;
    const srd::AggDev& h = a->host;
    if (h.dense || h.num_keys == 0) { // every group of a range-declared (or single-state) table exists: plain pre-aggregation
        SR_TRY(agg_push_vtab(a, vt, n));
        out->num_rows = 0;
        return SR_OK;
    }
    if (n == 0) return SR_OK;
    if (n >= 0x7FFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "selective push of more than 2^31 rows: push smaller batches");
    SR_TRY(a->sel_flags.reserve(ctx, (size_t)n + 16));
    SR_TRY(a->sel_pos.reserve(ctx, sizeof(uint32_t) * ((size_t)n + 2)));
    SR_CUDA(ctx, cudaMemsetAsync((uint8_t*)a->sel_flags.p + n, 0, 1, ctx->stream)); // flag n = 0: its prefix sum is the total
    a->table_touched = true;
    srd::k_agg_push_existing<<<std::min(grid_for(n, srd::AGG_BLOCK), ctx->num_sms * 8), srd::AGG_BLOCK, 0, ctx->stream>>>((const srd::AggDev*)a->dev.p, vt, n,
                                                                                                                       a->sel_flags.as<uint8_t>());
    SR_LAUNCH_CHECK(ctx);
    auto fin = thrust::make_transform_iterator((const uint8_t*)a->sel_flags.as<uint8_t>(), srd::U8ToU32());
    size_t tb = 0;
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, fin, a->sel_pos.as<uint32_t>(), (int)(n + 1), ctx->stream));
    SR_TRY(a->sel_tmp.reserve(ctx, std::max<size_t>(tb, 16)));
    SR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(a->sel_tmp.p, tb, fin, a->sel_pos.as<uint32_t>(), (int)(n + 1), ctx->stream));
    uint32_t* pin = (uint32_t*)ctx->pinned;
    SR_CUDA(ctx, cudaMemcpyAsync(pin, a->sel_pos.as<uint32_t>() + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t m = (int64_t)pin[0];
    out->num_rows = m;
    if (m == 0 || m == n) return SR_OK; // nothing streamed, or everything: `out` already holds exactly those rows
    SR_TRY(a->sel_index.reserve(ctx, sizeof(uint32_t) * (size_t)m));
    srd::k_selection_index<<<std::min(grid_for(n, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(a->sel_flags.as<uint8_t>(), a->sel_pos.as<uint32_t>(), n,
                                                                                                 a->sel_index.as<uint32_t>());
    SR_LAUNCH_CHECK(ctx);
    a->sel_cols.resize(out->num_cols);
    srd::GatherArgs ga;
    ga.n = out->num_cols;
    for (int k = 0; k < out->num_cols; k++) {
        sr_col_out& oc = out->cols[k];
        SR_TRY(a->sel_cols.gather(ctx, k, m, oc.data, oc.nulls, srd::type_width(oc.type), false, &ga.c[k]));
        a->sel_cols.fill(out, k, oc.type, oc.slot_id);
    }
    SR_TRY(launch_gather(ctx, a->sel_index.as<uint32_t>(), m, ga));
    return mem_sync(ctx, chunk->mem);
}

int32_t sr_agg_merge(sr_agg* a, sr_agg* o) {
    if (!a || !o) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = a->ctx;
    SR_BIND(ctx);
    if (o->ctx != ctx) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "merge across contexts");
    if (a->finished) return sr_fail(ctx, SR_ERR_STATE, "merge into a finished aggregate");
    if (desc_has_distinct(&a->desc)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) states do not merge; shuffle on the group keys instead");
    if (!o->compiled) return SR_OK; // nothing was pushed into `other`
    if (memcmp(&a->desc, &o->desc, sizeof(sr_agg_desc)) != 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "merge needs identical descriptors");
    return agg_merge(a, o);
}

// ------------------------------------------------------------------ fragment
sr_fragment* sr_fragment_create(sr_ctx* ctx, const sr_fragment_desc* desc) {
    if (!ctx || !desc) return nullptr;
    SR_LOCK(ctx);
    cudaSetDevice(ctx->device);
    if (desc->num_joins < 0 || desc->num_joins > SR_MAX_FRAG_JOINS || desc->scan.num_preds < 0 || desc->scan.num_filter_exprs < 0) {
        sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fragment desc counts");
        return nullptr;
    }
    for (int j = 0; j < desc->num_joins; j++) {
        const sr_frag_join& fj = desc->joins[j];
        if (!fj.join || !fj.join->built) {
            sr_fail(ctx, SR_ERR_STATE, "fragment join %d is not built", j);
            return nullptr;
        }
        if (fj.join->ctx != ctx) {
            sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fragment join %d belongs to another context", j);
            return nullptr;
        }
        if (fj.join->desc.join_type != SR_JOIN_INNER && fj.join->desc.join_type != SR_JOIN_LEFT_SEMI) {
            sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fused fragment supports INNER / LEFT SEMI joins (join %d is type %d)", j, fj.join->desc.join_type);
            return nullptr;
        }
        if (fj.join->desc.other_conjunct.num_nodes > 0) {
            sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fused fragment: join %d has an other-join conjunct; use the per-operator path", j);
            return nullptr;
        }
        if (fj.join->desc.num_keys != 1) {
            sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fused fragment supports single-column join keys (join %d)", j);
            return nullptr;
        }
        if (fj.num_payload < 0 || fj.num_payload > SR_MAX_FRAG_PAYLOAD || (fj.num_payload > 0 && fj.join->desc.join_type != SR_JOIN_INNER)) {
            sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fragment join %d payload", j);
            return nullptr;
        }
        for (int p = 0; p < fj.num_payload; p++)
            if (!fj.join->find_col(fj.payload_build_slots[p])) {
                sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fragment join %d: payload slot %d not in the build chunk", j, fj.payload_build_slots[p]);
                return nullptr;
            }
    }
    if (agg_validate_desc(ctx, &desc->agg) != SR_OK) return nullptr;
    if (desc_has_distinct(&desc->agg)) {
        sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "COUNT(DISTINCT) inside the fused fragment; aggregate the probe output with sr_agg_push");
        return nullptr;
    }
    sr_fragment* f = new sr_fragment();
    f->ctx = ctx;
    f->preds.assign(desc->scan.preds, desc->scan.preds + desc->scan.num_preds);
    f->exprs.assign(desc->scan.filter_exprs, desc->scan.filter_exprs + desc->scan.num_filter_exprs);
    f->num_joins = desc->num_joins;
    f->force_mode = (desc->mode_hint == 1 || desc->mode_hint == 2) ? desc->mode_hint : 0;
    for (int j = 0; j < desc->num_joins; j++) {
        f->joins[j] = desc->joins[j];
        // one-to-many INNER join (duplicate build keys): always the selection-vector passes, whose final pass expands
        if (desc->joins[j].join->has_dup && desc->joins[j].join->desc.join_type == SR_JOIN_INNER) f->expand = true;
    }
    f->agg = new sr_agg();
    f->agg->ctx = ctx;
    f->agg->desc = desc->agg;
    return f;
}

void sr_fragment_destroy(sr_fragment* frag) {
    if (!frag) return;
    SR_LOCK(frag->ctx);
    cudaSetDevice(frag->ctx->device);
    cudaStreamSynchronize(frag->ctx->stream);
    delete frag->agg;
    delete frag;
}

int32_t sr_fragment_push(sr_fragment* frag, const sr_chunk_view* fact) {
    if (!frag || !fact) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(frag->ctx);
    return frag_push(frag, fact);
}

int32_t sr_fragment_push_chunks(sr_fragment* frag, const sr_chunk_view* chunks, int32_t num_chunks) {
    if (!frag) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(frag->ctx);
    return frag_push_chunks(frag, chunks, num_chunks);
}

sr_agg* sr_fragment_agg(sr_fragment* frag) {
    return frag ? frag->agg : nullptr;
}

int32_t sr_fragment_get_plan(sr_fragment* frag, sr_fragment_plan* plan) {
    if (!frag || !plan) return SR_ERR_INVALID_ARGUMENT;
    SR_LOCK(frag->ctx);
    if (!frag->compiled) return sr_fail(frag->ctx, SR_ERR_STATE, "the fragment plans on its first push");
    memset(plan, 0, sizeof(*plan));
    plan->num_joins = frag->num_joins;
    for (int q = 0; q < frag->num_joins; q++) {
        plan->order[q] = frag->order[q];
        plan->bitmap_in_smem[q] = frag->host.joins[q].smem_off >= 0 ? 1 : 0;
        plan->pass_rate[q] = frag->pass_rate[q];
    }
    plan->agg_in_smem = frag->smem_agg ? 1 : 0;
    plan->mode = frag->selective ? 2 : 1;
    plan->num_stream_joins = frag->selective ? frag->pass.num_stream_joins : 0;
    plan->num_gather_passes = frag->selective ? (int32_t)frag->gather_joins.size() : 0;
    plan->pred_rate = frag->pred_rate;
    plan->final_pass = frag->final_pass;
    // launch shape of the mode's first kernel: the streaming pass, or the cascade
    if (frag->selective) {
        plan->smem_bytes = (int32_t)frag->stream_smem;
        plan->grid = frag->stream_grid;
        plan->block = srd::STREAM_BLOCK;
    } else {
        plan->smem_bytes = (int32_t)frag->cascade_smem;
        plan->grid = frag->cascade_grid;
        plan->block = srd::FRAG_BLOCK;
    }
    return SR_OK;
}

int32_t sr_fragment_last_pass_ms(sr_fragment* frag, float ms[3]) {
    if (!frag || !ms) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = frag->ctx;
    SR_BIND(ctx);
    if (!frag->timed_push) return sr_fail(ctx, SR_ERR_STATE, "no timed push (selection-vector mode only)");
    SR_CUDA(ctx, cudaEventSynchronize(frag->ev[3]));
    for (int k = 0; k < 3; k++) SR_CUDA(ctx, cudaEventElapsedTime(&ms[k], frag->ev[k], frag->ev[k + 1]));
    return SR_OK;
}

int32_t sr_fragment_reset(sr_fragment* frag) {
    if (!frag) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = frag->ctx;
    SR_BIND(ctx);
    SR_TRY(agg_reset_impl(frag->agg));
    if (frag->compiled) SR_CUDA(ctx, cudaMemsetAsync(frag->counters.p, 0, 8, ctx->stream));
    return SR_OK;
}

int64_t sr_fragment_rows_passed(sr_fragment* frag) {
    if (!frag) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = frag->ctx;
    SR_BIND(ctx);
    if (!frag->compiled) return 0;
    SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned + 16, frag->counters.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return (int64_t)ctx->pinned[16];
}

// ------------------------------------------------------------------ exchange
sr_xchg* sr_xchg_create(sr_ctx* ctx, const sr_part_desc* desc) {
    if (!ctx || !desc) return nullptr;
    if (desc->num_channels < 1 || desc->num_channels > srd::PART_MAX_CH || desc->num_part_slots < 1 || desc->num_part_slots > SR_MAX_PART_KEYS ||
        (desc->hash_fn != SR_HASH_FNV && desc->hash_fn != SR_HASH_CRC32 && desc->hash_fn != SR_HASH_XXH3) || (desc->reduce_op != SR_REDUCE_MULHI && desc->reduce_op != SR_REDUCE_MODULO)) {
        sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "partition desc (channels 1..%d, 1..%d slots)", srd::PART_MAX_CH, SR_MAX_PART_KEYS);
        return nullptr;
    }
    sr_xchg* x = new sr_xchg();
    x->ctx = ctx;
    x->desc = *desc;
    return x;
}

void sr_xchg_destroy(sr_xchg* x) {
    if (!x) return;
    SR_LOCK(x->ctx);
    cudaSetDevice(x->ctx->device);
    cudaStreamSynchronize(x->ctx->stream);
    delete x;
}

static int32_t xchg_part_cols(sr_xchg* x, srd::PartCols* pc) {
    pc->n = x->desc.num_part_slots;
    pc->hash_fn = x->desc.hash_fn;
    pc->reduce = x->desc.reduce_op;
    pc->num_channels = x->desc.num_channels;
    for (int k = 0; k < pc->n; k++) {
        const int c = x->staged.find(x->desc.part_slots[k]);
        if (c < 0) return sr_fail(x->ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses partition slot %d", x->desc.part_slots[k]);
        pc->c[k] = x->staged.cols[c];
    }
    return SR_OK;
}

int32_t sr_xchg_hash(sr_xchg* x, const sr_chunk_view* in, uint32_t* hash_values, uint32_t* channel_ids, int32_t mem) {
    if (!x || !in) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = x->ctx;
    SR_BIND(ctx);
    SR_TRY(mem_check(ctx, mem, "sr_xchg_hash"));
    SR_TRY(x->staged.stage(ctx, in));
    srd::PartCols pc;
    SR_TRY(xchg_part_cols(x, &pc));
    const int64_t n = in->num_rows;
    if (n <= 0) return SR_OK;
    SR_TRY(x->hash_values.reserve(ctx, sizeof(uint32_t) * (size_t)n));
    SR_TRY(x->channel_ids.reserve(ctx, sizeof(uint32_t) * (size_t)n));
    const int tiles = grid_for(n, srd::PART_TILE);
    srd::k_part_hash<<<tiles, srd::PART_BLOCK, 0, ctx->stream>>>(pc, n, x->hash_values.as<uint32_t>(), x->channel_ids.as<uint32_t>(), nullptr, tiles);
    SR_LAUNCH_CHECK(ctx);
    if (hash_values) SR_TRY(mem_out(ctx, hash_values, x->hash_values.p, sizeof(uint32_t) * (size_t)n, mem));
    if (channel_ids) SR_TRY(mem_out(ctx, channel_ids, x->channel_ids.p, sizeof(uint32_t) * (size_t)n, mem));
    return mem_sync(ctx, mem);
}

int32_t sr_xchg_partition(sr_xchg* x, const sr_chunk_view* in, sr_chunk_out* out, int64_t* channel_offsets_host) {
    if (!x || !in || !out || !channel_offsets_host) return SR_ERR_INVALID_ARGUMENT;
    sr_ctx* ctx = x->ctx;
    SR_BIND(ctx);
    if (in->num_cols > SR_MAX_OUT_COLS) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many columns");
    if (in->num_rows >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "partition batch of more than 2^32 rows");
    SR_TRY(x->staged.stage(ctx, in));
    srd::PartCols pc;
    SR_TRY(xchg_part_cols(x, &pc));
    const int64_t n = in->num_rows;
    const int nch = x->desc.num_channels;
    ColBufs::header(out, in->num_cols, n);
    x->out_cols.resize(in->num_cols);
    if (n <= 0) { // zero rows of every column, with no data buffer; a nullable column keeps a (zero-row) null column
        for (int c = 0; c <= nch; c++) channel_offsets_host[c] = 0;
        for (int k = 0; k < in->num_cols; k++) {
            uint8_t* nulls = nullptr;
            if (in->cols[k].nulls) {
                DevBuf& nb = x->out_cols.cols[k].nulls;
                SR_TRY(nb.reserve(ctx, 1));
                nulls = (uint8_t*)nb.p;
            }
            out->cols[k] = sr_col_out{nullptr, nulls, in->cols[k].type, in->cols[k].slot_id};
        }
        return SR_OK;
    }
    const int tiles = grid_for(n, srd::PART_TILE);
    const int64_t ncounts = (int64_t)nch * tiles;
    SR_TRY(x->channel_ids.reserve(ctx, sizeof(uint32_t) * (size_t)n));
    SR_TRY(x->counts.reserve(ctx, sizeof(uint32_t) * (size_t)ncounts));
    SR_TRY(x->offsets.reserve(ctx, sizeof(uint64_t) * (size_t)ncounts));
    SR_TRY(x->row_index.reserve(ctx, sizeof(uint32_t) * (size_t)n));
    srd::k_part_hash<<<tiles, srd::PART_BLOCK, 0, ctx->stream>>>(pc, n, nullptr, x->channel_ids.as<uint32_t>(), x->counts.as<uint32_t>(), tiles);
    SR_LAUNCH_CHECK(ctx);
    SR_TRY(scan_counts(ctx, &x->scan_scratch, x->counts.as<uint32_t>(), ncounts, x->offsets.as<uint64_t>()));
    srd::k_part_scatter<<<tiles, srd::PART_BLOCK, 0, ctx->stream>>>(x->channel_ids.as<uint32_t>(), n, nch, x->offsets.as<uint64_t>(), tiles,
                                                                   x->row_index.as<uint32_t>());
    SR_LAUNCH_CHECK(ctx);
    // channel c starts at offsets[c * tiles]
    std::vector<uint64_t> starts(nch);
    SR_CUDA(ctx, cudaMemcpy2DAsync(starts.data(), sizeof(uint64_t), x->offsets.p, sizeof(uint64_t) * (size_t)tiles, sizeof(uint64_t), nch,
                                   cudaMemcpyDeviceToHost, ctx->stream));
    srd::GatherArgs ga;
    ga.n = in->num_cols;
    for (int k = 0; k < in->num_cols; k++) {
        const srd::DCol& dc = x->staged.cols[k];
        SR_TRY(x->out_cols.gather(ctx, k, n, dc.data, dc.nulls, dc.width, false, &ga.c[k]));
        x->out_cols.fill(out, k, dc.type, x->staged.slots[k]);
    }
    SR_TRY(launch_gather(ctx, x->row_index.as<uint32_t>(), n, ga));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int c = 0; c < nch; c++) channel_offsets_host[c] = (int64_t)starts[c];
    channel_offsets_host[nch] = n;
    return SR_OK;
}

// ------------------------------------------------------------------ misc
int32_t sr_gather(sr_ctx* ctx, const void* src, int32_t type, const uint32_t* index, int64_t n, void* dst, int32_t mem) {
    SR_BIND(ctx);
    const int w = srd::type_width(type);
    if (w == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown type %d", type);
    SR_TRY(mem_check(ctx, mem, "sr_gather"));
    if (mem_is_host(mem)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "sr_gather takes device pointers");
    if (n <= 0) return SR_OK;
    if (!col_aligned(src, w) || !col_aligned(dst, w) || !col_aligned(index, 4))
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_gather: a device pointer is not naturally aligned for width %d", w);
    srd::GatherArgs ga;
    ga.n = 1;
    ga.c[0] = srd::GatherCol{src, nullptr, dst, nullptr, w, 0, 0};
    return launch_gather(ctx, index, n, ga);
}

int32_t sr_abi_sizeof(int32_t which) {
    switch (which) {
    case 0:
        return (int32_t)sizeof(sr_col_view);
    case 1:
        return (int32_t)sizeof(sr_chunk_view);
    case 2:
        return (int32_t)sizeof(sr_chunk_out);
    case 3:
        return (int32_t)sizeof(sr_pred);
    case 4:
        return (int32_t)sizeof(sr_expr);
    case 5:
        return (int32_t)sizeof(sr_scan_desc);
    case 6:
        return (int32_t)sizeof(sr_join_desc);
    case 7:
        return (int32_t)sizeof(sr_join_info);
    case 8:
        return (int32_t)sizeof(sr_agg_fn);
    case 9:
        return (int32_t)sizeof(sr_agg_desc);
    case 10:
        return (int32_t)sizeof(sr_frag_join);
    case 11:
        return (int32_t)sizeof(sr_fragment_desc);
    case 12:
        return (int32_t)sizeof(sr_part_desc);
    case 13:
        return (int32_t)sizeof(sr_agg_state_array);
    case 14:
        return (int32_t)sizeof(sr_fragment_plan);
    case 15:
        return (int32_t)sizeof(sr_rf_info);
    case 16:
        return (int32_t)sizeof(sr_null_map_view);
    default:
        return -1;
    }
}

int32_t sr_memcpy(sr_ctx* ctx, void* dst, const void* src, int64_t bytes, int32_t kind) {
    SR_BIND(ctx);
    if (bytes < 0 || kind < 0 || kind > 2) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_memcpy arguments");
    if (bytes == 0) return SR_OK;
    const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    SR_CUDA(ctx, cudaMemcpyAsync(dst, src, (size_t)bytes, k, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

int32_t sr_bandwidth_probe(sr_ctx* ctx, const void* dev_ptr, int64_t bytes, uint64_t* checksum_host) {
    SR_BIND(ctx);
    if (!dev_ptr || bytes < 16 || ((uintptr_t)dev_ptr & 15)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "bandwidth probe needs a 16-byte aligned device buffer");
    SR_CUDA(ctx, cudaMemsetAsync(ctx->dscratch + 32, 0, 8, ctx->stream));
    srd::k_bandwidth_probe<<<ctx->num_sms * 4, 512, 0, ctx->stream>>>((const int4*)dev_ptr, bytes / 16, (unsigned long long*)(ctx->dscratch + 32));
    SR_LAUNCH_CHECK(ctx);
    if (checksum_host) {
        SR_CUDA(ctx, cudaMemcpyAsync(ctx->pinned + 32, ctx->dscratch + 32, 8, cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *checksum_host = ctx->pinned[32];
    }
    return SR_OK;
}

// ------------------------------------------------------------------ exchange wire format (ChunkPB.data)
int64_t sr_chunk_serialized_size(const sr_chunk_view* chunk, int64_t row_begin, int64_t row_end) {
    if (!chunk || row_begin < 0 || row_end < row_begin) return SR_ERR_INVALID_ARGUMENT;
    return serde_size(chunk, row_end - row_begin);
}

int32_t sr_chunk_serialize(sr_ctx* ctx, const sr_chunk_view* chunk, int64_t row_begin, int64_t row_end, void* dst, int64_t dst_capacity, int32_t dst_mem,
                           sr_chunk_pb_meta* meta) {
    SR_BIND(ctx);
    if (!chunk || !dst) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_chunk_serialize: null argument");
    return serde_serialize(ctx, chunk, row_begin, row_end, dst, dst_capacity, dst_mem, meta);
}

sr_serde* sr_serde_create(sr_ctx* ctx) {
    if (!ctx) return nullptr;
    sr_serde* h = new sr_serde();
    h->ctx = ctx;
    return h;
}

void sr_serde_destroy(sr_serde* h) {
    if (!h) return;
    SR_LOCK(h->ctx);
    cudaSetDevice(h->ctx->device);
    cudaStreamSynchronize(h->ctx->stream);
    delete h;
}

int32_t sr_chunk_deserialize(sr_serde* h, const void* src, int64_t bytes, int32_t src_mem, const sr_chunk_pb_meta* meta, sr_chunk_out* out) {
    if (!h || !src || !meta || !out) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(h->ctx);
    return serde_deserialize(h, src, bytes, src_mem, meta, out);
}

struct sr_page_decoder {
    sr_ctx* ctx = nullptr;
    PageScratch scratch;
    DevBuf dict;                // sr_page_decoder_set_dict's table: what each code of a dictionary data page decodes to
    long long dict_words = -1;  // -1: no table set
};

sr_page_decoder* sr_page_decoder_create(sr_ctx* ctx) {
    if (!ctx) return nullptr;
    sr_page_decoder* d = new sr_page_decoder();
    d->ctx = ctx;
    return d;
}

void sr_page_decoder_destroy(sr_page_decoder* d) {
    if (!d) return;
    SR_LOCK(d->ctx);
    cudaSetDevice(d->ctx->device);
    cudaStreamSynchronize(d->ctx->stream);
    delete d;
}

int32_t sr_pages_decode(sr_page_decoder* d, int32_t encoding, int32_t type, const sr_page_view* pages, int32_t num_pages, int32_t mem, void* out,
                        int64_t out_capacity, int64_t* out_rows) {
    if (!d || !out_rows) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(d->ctx);
    return pages_decode(d->ctx, &d->scratch, encoding, type, pages, num_pages, mem, out, out_capacity, out_rows, (const int32_t*)d->dict.p, d->dict_words);
}

int32_t sr_null_maps_decode(sr_page_decoder* d, int32_t null_encoding, const sr_null_map_view* maps, int32_t num_pages, int32_t mem, uint8_t* out_nulls,
                            int64_t out_capacity, int64_t* out_rows, int64_t* out_null_count) {
    if (!d || !out_rows || !out_null_count) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(d->ctx);
    return null_maps_decode(d->ctx, &d->scratch, null_encoding, maps, num_pages, mem, out_nulls, out_capacity, out_rows, out_null_count);
}

int32_t sr_page_decoder_set_dict(sr_page_decoder* d, const int32_t* values, int64_t num_words, int32_t mem) {
    if (!d) return SR_ERR_INVALID_ARGUMENT;
    SR_BIND(d->ctx);
    sr_ctx* ctx = d->ctx;
    if (num_words < 0 || num_words > INT32_MAX || (num_words > 0 && !values)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "sr_page_decoder_set_dict: %lld words", (long long)num_words);
    SR_TRY(mem_check(ctx, mem, "sr_page_decoder_set_dict"));
    d->dict_words = -1; // a failed call leaves no table
    SR_TRY(d->dict.reserve(ctx, 4 * (size_t)num_words + 4));
    if (num_words > 0) SR_CUDA(ctx, cudaMemcpyAsync(d->dict.p, values, 4 * (size_t)num_words, mem_is_host(mem) ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the caller may free `values` on return
    d->dict_words = num_words;
    return SR_OK;
}

int32_t sr_flush_l2(sr_ctx* ctx) {
    SR_BIND(ctx);
    if (!ctx->l2_flush) {
        ctx->l2_flush_bytes = 512ull << 20; // 10x the 50 MB L2
        SR_CUDA(ctx, cudaMalloc(&ctx->l2_flush, ctx->l2_flush_bytes));
    }
    SR_CUDA(ctx, cudaMemsetAsync(ctx->l2_flush, 0, ctx->l2_flush_bytes, ctx->stream));
    return SR_OK;
}

} // extern "C"
