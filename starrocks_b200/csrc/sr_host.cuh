// sr_host.cuh -- host-side plumbing of libsr_gpu.so: context, device buffers, error handling, memory kinds and the checks
// of a caller's chunks, the page-locked host registry, compilation of sr_pred / sr_expr descriptors against a chunk's slots.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "sr_device.cuh"

struct sr_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    int32_t err_code = 0;
    int64_t launches = 0;
    int64_t dev_bytes = 0;
    int num_sms = 132;
    // pinned scratch for tiny D2H results (counters) -- one slot per use inside a call
    uint64_t* pinned = nullptr; // 64 x u64
    uint64_t* dscratch = nullptr; // 64 x u64 on device
    void* l2_flush = nullptr;
    size_t l2_flush_bytes = 0;
    // Every entry point that enqueues work or touches the context's scratch (pinned / dscratch counters, err, launches,
    // dev_bytes, the per-handle prober list) holds this lock for its whole duration: handles of one context may be driven
    // from several pipeline-driver threads (build thread, N prober threads, the poller), but all their work goes to the one
    // stream anyway, so serialising the host side costs nothing and keeps the shared scratch slots private to a call.
    std::recursive_mutex mu;
};
#define SR_LOCK(ctx) std::lock_guard<std::recursive_mutex> _sr_lock((ctx)->mu)

static thread_local std::string g_create_err;

#define SR_CUDA(ctx, call)                                                                          \
    do {                                                                                            \
        cudaError_t _e = (call);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            return sr_fail((ctx), _e == cudaErrorMemoryAllocation ? SR_ERR_OUT_OF_MEMORY : SR_ERR_CUDA, \
                           "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
        }                                                                                           \
    } while (0)

#define SR_TRY(expr)                  \
    do {                              \
        int32_t _rc = (expr);         \
        if (_rc != SR_OK) return _rc; \
    } while (0)

static int32_t sr_fail(sr_ctx* ctx, int32_t code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) {
        ctx->err = buf;
        ctx->err_code = code;
    } else {
        g_create_err = buf;
    }
    return code;
}

#define SR_LAUNCH_CHECK(ctx)                                                                  \
    do {                                                                                      \
        (ctx)->launches++;                                                                    \
        cudaError_t _e = cudaGetLastError();                                                  \
        if (_e != cudaSuccess)                                                                \
            return sr_fail((ctx), SR_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                               \
    } while (0)

// grow-only device buffer
// page-locked host buffer for results handed back in host memory: a D2H copy into pageable memory is staged by the
// driver at a few GB/s, into pinned memory it is one DMA at the link rate
struct PinnedBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    PinnedBuf(PinnedBuf&& o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    PinnedBuf& operator=(PinnedBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    ~PinnedBuf() { release(); }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
    bool reserve(size_t bytes) {
        if (bytes <= cap) return true;
        release();
        const size_t ncap = (std::max<size_t>(bytes, 4096) + 4095) & ~(size_t)4095;
        if (cudaHostAlloc(&p, ncap, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            p = nullptr;
            return false;
        }
        cap = ncap;
        return true;
    }
};

struct DevBuf {
    sr_ctx* ctx = nullptr;
    void* p = nullptr;
    size_t cap = 0;
    ~DevBuf() { release(); }
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : ctx(o.ctx), p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            ctx = o.ctx;
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    void release() {
        if (p) {
            cudaFree(p);
            if (ctx) ctx->dev_bytes -= (int64_t)cap;
        }
        p = nullptr;
        cap = 0;
    }
    // ensure capacity; contents are NOT preserved unless keep > 0 (bytes to preserve)
    int32_t reserve(sr_ctx* c, size_t bytes, size_t keep = 0) {
        ctx = c;
        if (bytes <= cap) return SR_OK;
        size_t ncap = std::max(bytes, cap + cap / 2);
        ncap = (ncap + 255) & ~(size_t)255;
        void* np = nullptr;
        cudaError_t e = cudaMalloc(&np, ncap);
        if (e != cudaSuccess) {
            cudaGetLastError();
            // retry with the exact size
            ncap = (bytes + 255) & ~(size_t)255;
            e = cudaMalloc(&np, ncap);
            if (e != cudaSuccess) {
                cudaGetLastError();
                return sr_fail(c, SR_ERR_OUT_OF_MEMORY, "cudaMalloc(%zu) failed: %s", ncap, cudaGetErrorString(e));
            }
        }
        if (keep > 0 && p) {
            e = cudaMemcpyAsync(np, p, std::min(keep, cap), cudaMemcpyDeviceToDevice, c->stream);
            if (e != cudaSuccess) {
                cudaFree(np);
                return sr_fail(c, SR_ERR_CUDA, "memcpy D2D failed: %s", cudaGetErrorString(e));
            }
            cudaStreamSynchronize(c->stream);
        }
        if (p) {
            cudaFree(p);
            c->dev_bytes -= (int64_t)cap;
        }
        p = np;
        cap = ncap;
        c->dev_bytes += (int64_t)ncap;
        return SR_OK;
    }
    template <typename T>
    T* as() const {
        return (T*)p;
    }
};

// The device columns one handle stages or hands back in an sr_chunk_out: a (data, nulls) pair of grow-only buffers per
// column, kept across calls so that a repeated call pays no cudaMalloc.  What a call hands back stays valid until the
// next call on the handle (include/sr_gpu_ops.h).
struct ColBufs {
    struct Col {
        DevBuf data, nulls;
        bool nullable = false; // the last reserve gave the column a null column
    };
    std::vector<Col> cols;
    void resize(int num_cols) {
        if (cols.size() < (size_t)num_cols) cols.resize(num_cols);
    }
    // column k for `rows` values of `width` bytes, plus one null byte per row when `nullable` (*nulls is NULL
    // otherwise); a column of zero rows still gets the buffers of one row
    int32_t reserve(sr_ctx* ctx, int k, int64_t rows, int width, bool nullable, void** data, uint8_t** nulls) {
        Col& c = cols[k];
        const size_t r = (size_t)std::max<int64_t>(rows, 1);
        SR_TRY(c.data.reserve(ctx, r * width));
        if (nullable) SR_TRY(c.nulls.reserve(ctx, r));
        c.nullable = nullable;
        *data = c.data.p;
        *nulls = nullable ? (uint8_t*)c.nulls.p : nullptr;
        return SR_OK;
    }
    static void header(sr_chunk_out* out, int num_cols, int64_t rows) {
        out->num_cols = num_cols;
        out->mem = SR_MEM_DEVICE;
        out->num_rows = rows;
    }
    // out->cols[k] <- column k as the last reserve left it
    void fill(sr_chunk_out* out, int k, int32_t type, int32_t slot) const {
        const Col& c = cols[k];
        out->cols[k] = sr_col_out{c.data.p, c.nullable ? (uint8_t*)c.nulls.p : nullptr, type, slot};
    }
    // column k reserved for `rows` gathered values of a source column; it has a null column when the source has one or
    // index 0 means NULL (`zero_is_null`: the build side of an outer join)
    int32_t gather(sr_ctx* ctx, int k, int64_t rows, const void* src, const uint8_t* src_nulls, int width, bool zero_is_null, srd::GatherCol* g) {
        void* dst;
        uint8_t* dst_nulls;
        SR_TRY(reserve(ctx, k, rows, width, src_nulls != nullptr || zero_is_null, &dst, &dst_nulls));
        *g = srd::GatherCol{src, src_nulls, dst, dst_nulls, width, zero_is_null ? 1 : 0, 0};
        return SR_OK;
    }
};

static inline const sr_col_view* find_col(const sr_chunk_view* c, int32_t slot) {
    for (int k = 0; k < c->num_cols; k++)
        if (c->cols[k].slot_id == slot) return &c->cols[k];
    return nullptr;
}

// natural alignment of a column the kernels read in place: its value width, 8 bytes for 16-byte values
static inline bool col_aligned(const void* p, int width) {
    return ((uintptr_t)p & (uintptr_t)(std::min(width, 8) - 1)) == 0;
}

// memory kinds: the sr_mem rule of include/sr_gpu_ops.h.  Outside the in-place readers, which resolve pinned buffers with
// a PinnedResolver (Staged::stage for sr_fragment_push, frag_push_chunks, stage_pages), SR_MEM_HOST_PINNED is SR_MEM_HOST.
static inline bool mem_is_host(int32_t mem) {
    return mem == SR_MEM_HOST || mem == SR_MEM_HOST_PINNED;
}

// refuses an unknown kind: every entry point checks its kinds before any copy, allocation or launch
static int32_t mem_check(sr_ctx* ctx, int32_t mem, const char* what) {
    if (mem == SR_MEM_DEVICE || mem_is_host(mem)) return SR_OK;
    return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%s: unknown memory kind %d", what, mem);
}

// the caller's buffer as a device pointer: the buffer itself for device memory, else `tmp` holding an H2D copy of it
// (copy = false: an output buffer, `tmp` is only its space); `tmp` must outlive the queued work (mem_sync)
static int32_t mem_in(sr_ctx* ctx, const void* buf, size_t bytes, int32_t mem, DevBuf* tmp, const void** dev, bool copy = true) {
    *dev = buf;
    if (!mem_is_host(mem)) return SR_OK;
    SR_TRY(tmp->reserve(ctx, bytes));
    if (copy) SR_CUDA(ctx, cudaMemcpyAsync(tmp->p, buf, bytes, cudaMemcpyHostToDevice, ctx->stream));
    *dev = tmp->p;
    return SR_OK;
}

// queues the copy of a device result into the caller's buffer (none when the result is already there)
static int32_t mem_out(sr_ctx* ctx, void* dst, const void* src_dev, size_t bytes, int32_t mem) {
    if (bytes == 0 || dst == src_dev) return SR_OK;
    SR_CUDA(ctx, cudaMemcpyAsync(dst, src_dev, bytes, mem_is_host(mem) ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, ctx->stream));
    return SR_OK;
}

// for host memory, waits for the stream: a host result is complete, a host input (and its staging) free, on return
static int32_t mem_sync(sr_ctx* ctx, int32_t mem) {
    if (mem_is_host(mem)) SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SR_OK;
}

// what a refusal calls a caller's chunk: "chunk", or "chunk <index>" for chunk `index` of a list (made only on refusal)
struct ChunkName {
    char s[24] = "chunk";
    explicit ChunkName(int index) { if (index >= 0) snprintf(s, sizeof(s), "chunk %d", index); }
};

// The header of a caller's chunk, checked before any of its columns is read: a known kind, no negative row or column
// count, and a column array when it has columns.  `index`: the chunk's place in a list, -1 for a single chunk.
static int32_t chunk_check(sr_ctx* ctx, const sr_chunk_view* in, int index = -1) {
    if (in->mem != SR_MEM_DEVICE && !mem_is_host(in->mem)) return mem_check(ctx, in->mem, ChunkName(index).s);
    if (in->num_rows < 0 || in->num_cols < 0 || (in->num_cols > 0 && in->cols == nullptr))
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%s: %lld rows, %d columns at %p", ChunkName(index).s, (long long)in->num_rows, in->num_cols, (const void*)in->cols);
    return SR_OK;
}

// One column of a caller's chunk of `rows` rows: a known type (*width receives its width), data when there are rows,
// and, when the kernels read it in place, natural alignment.  `index` as for chunk_check.
static int32_t col_check(sr_ctx* ctx, const sr_col_view& c, int64_t rows, bool in_place, int* width, int index = -1) {
    const int w = srd::type_width(c.type);
    if (w == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%s: unknown column type %d (slot %d)", ChunkName(index).s, c.type, c.slot_id);
    if (rows > 0 && c.data == nullptr) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%s: null data pointer (slot %d)", ChunkName(index).s, c.slot_id);
    if (in_place && !col_aligned(c.data, w))
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%s: slot %d column at %p is not %d-byte aligned", ChunkName(index).s, c.slot_id, c.data, std::min(w, 8));
    *width = w;
    return SR_OK;
}

// ---------------------------------------------------------------------------------------
// page-locked host ranges made by sr_host_alloc / sr_host_register (process-wide: both are portable allocations)
// ---------------------------------------------------------------------------------------
struct HostRange {
    size_t bytes;
    uintptr_t dev;   // device alias of the range's first byte
    bool registered; // sr_host_register (else sr_host_alloc)
};
struct HostRegistry {
    std::mutex mu;
    std::map<uintptr_t, HostRange> ranges; // by first byte
    // the range holding [p, p + bytes), or nullptr; caller holds mu
    const std::pair<const uintptr_t, HostRange>* find(uintptr_t p, size_t bytes) {
        auto it = ranges.upper_bound(p);
        if (it == ranges.begin()) return nullptr;
        --it;
        if (p + bytes > it->first + it->second.bytes) return nullptr;
        return &*it;
    }
    bool overlaps(uintptr_t p, size_t bytes) {
        auto it = ranges.lower_bound(p);
        if (it != ranges.end() && it->first < p + bytes) return true;
        if (it == ranges.begin()) return false;
        --it;
        return it->first + it->second.bytes > p;
    }
};
static HostRegistry& host_registry() {
    static HostRegistry r;
    return r;
}

// Device aliases of SR_MEM_HOST_PINNED buffers read in place, within one call: the registry first; any other pointer costs a
// driver query, and the allocation it lies in (its extent from the driver's range query, where the driver gives one) is
// remembered for the rest of the call, so buffers cut from one allocation cost one lookup.  Unmapped memory is refused.
struct PinnedResolver {
    struct Known {
        uintptr_t base;
        size_t bytes;
        uintptr_t dev;
    };
    std::vector<Known> known;
    int32_t resolve(sr_ctx* ctx, const void* host, size_t bytes, int32_t slot, const void** dev) {
        const uintptr_t p = (uintptr_t)host;
        {
            HostRegistry& reg = host_registry();
            std::lock_guard<std::mutex> lk(reg.mu);
            if (const auto* r = reg.find(p, bytes)) {
                *dev = (const void*)(r->second.dev + (p - r->first));
                return SR_OK;
            }
        }
        for (const Known& k : known)
            if (p >= k.base && p + bytes <= k.base + k.bytes) {
                *dev = (const void*)(k.dev + (p - k.base));
                return SR_OK;
            }
        cudaPointerAttributes at;
        memset(&at, 0, sizeof(at));
        if (cudaPointerGetAttributes(&at, host) != cudaSuccess || at.type != cudaMemoryTypeHost || at.devicePointer == nullptr) {
            cudaGetLastError();
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "slot %d: SR_MEM_HOST_PINNED buffer is not page-locked mapped host memory", slot);
        }
        Known k{p, bytes, (uintptr_t)at.devicePointer};
        CUdeviceptr start = 0;
        size_t size = 0;
        if (range_query(p, &start, &size) && start <= p && p + bytes <= start + size) {
            k.base = (uintptr_t)start;
            k.bytes = size;
            k.dev = (uintptr_t)at.devicePointer - (p - (uintptr_t)start);
        }
        known.push_back(k);
        *dev = at.devicePointer;
        return SR_OK;
    }
    // cuPointerGetAttribute(RANGE_START_ADDR / RANGE_SIZE), fetched through the runtime (the library links no libcuda)
    static bool range_query(uintptr_t p, CUdeviceptr* start, size_t* size) {
        typedef CUresult (*get_attr_fn)(void*, CUpointer_attribute, CUdeviceptr);
        static get_attr_fn fn = []() -> get_attr_fn {
            void* f = nullptr;
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint("cuPointerGetAttribute", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
                cudaGetLastError();
                return nullptr;
            }
            return (get_attr_fn)f;
        }();
        return fn && fn(start, CU_POINTER_ATTRIBUTE_RANGE_START_ADDR, (CUdeviceptr)p) == CUDA_SUCCESS &&
               fn(size, CU_POINTER_ATTRIBUTE_RANGE_SIZE, (CUdeviceptr)p) == CUDA_SUCCESS && *size > 0;
    }
};

// A chunk made resident on the device: host chunks are staged (H2D on the ctx stream) into buffers owned by `Staged`;
// device chunks, and pinned ones read in place (`in_place_pinned`), are referenced in place.  Every column is checked,
// and a pinned one resolved, before anything is allocated or copied.
struct Staged {
    ColBufs bufs;
    std::vector<srd::DCol> cols;
    std::vector<int32_t> slots;
    int64_t num_rows = 0;
    int32_t stage(sr_ctx* ctx, const sr_chunk_view* in, const std::vector<int32_t>* only_slots = nullptr, bool in_place_pinned = false) {
        cols.clear();
        slots.clear();
        num_rows = in->num_rows;
        SR_TRY(chunk_check(ctx, in));
        const bool pinned = in->mem == SR_MEM_HOST_PINNED && in_place_pinned && in->num_rows > 0;
        const bool in_place = in->mem == SR_MEM_DEVICE || pinned;
        PinnedResolver resolver;
        for (int k = 0; k < in->num_cols; k++) {
            const sr_col_view& c = in->cols[k];
            if (only_slots && std::find(only_slots->begin(), only_slots->end(), c.slot_id) == only_slots->end()) continue;
            srd::DCol d{c.data, c.nulls, c.type, 0};
            SR_TRY(col_check(ctx, c, num_rows, in_place, &d.width));
            if (pinned) {
                SR_TRY(resolver.resolve(ctx, c.data, (size_t)num_rows * d.width, c.slot_id, &d.data));
                const void* nulls = nullptr;
                if (c.nulls) SR_TRY(resolver.resolve(ctx, c.nulls, (size_t)num_rows, c.slot_id, &nulls));
                d.nulls = (const uint8_t*)nulls;
            }
            cols.push_back(d);
            slots.push_back(c.slot_id);
        }
        if (in_place) return SR_OK;
        bufs.resize((int)cols.size());
        for (size_t k = 0; k < cols.size(); k++) {
            srd::DCol& d = cols[k];
            ColBufs::Col& b = bufs.cols[k];
            SR_TRY(b.data.reserve(ctx, (size_t)num_rows * d.width + 16));
            SR_CUDA(ctx, cudaMemcpyAsync(b.data.p, d.data, (size_t)num_rows * d.width, cudaMemcpyHostToDevice, ctx->stream));
            d.data = b.data.p;
            if (d.nulls) {
                SR_TRY(b.nulls.reserve(ctx, (size_t)num_rows + 16));
                SR_CUDA(ctx, cudaMemcpyAsync(b.nulls.p, d.nulls, (size_t)num_rows, cudaMemcpyHostToDevice, ctx->stream));
                d.nulls = (const uint8_t*)b.nulls.p;
            }
        }
        return SR_OK;
    }
    int find(int32_t slot) const {
        for (size_t k = 0; k < slots.size(); k++)
            if (slots[k] == slot) return (int)k;
        return -1;
    }
};

// ---------------------------------------------------------------------------------------
// value table: the columns a kernel may read, addressed by small ids
// ---------------------------------------------------------------------------------------
#define SR_MAX_VALUES 20

struct VDesc {
    const void* data;
    const uint8_t* nulls;
    int32_t type;
    int32_t src; // -1: the kernel's own row; j >= 0: row = build index of fragment join j
};
struct VTab {
    VDesc v[SR_MAX_VALUES];
    int32_t n;
    // every value read from the kernel's own row is a non-nullable int32-class column: the loaders skip the type
    // dispatch and the null probe (the common shape of fact tables: dictionary codes, keys, dates, int measures)
    int32_t plain32;
};

static inline void vt_mark_plain32(VTab* vt) {
    vt->plain32 = 1;
    for (int k = 0; k < vt->n; k++) {
        const VDesc& d = vt->v[k];
        if (d.src >= 0) continue;
        const bool i32 = d.type == SR_TYPE_INT || d.type == SR_TYPE_DATE || d.type == SR_TYPE_DECIMAL32;
        if (!i32 || d.nulls != nullptr) vt->plain32 = 0;
    }
}

// host-side registry mapping slot -> value id while compiling
struct VReg {
    std::vector<int32_t> slots;
    std::vector<int32_t> types;
    int find(int32_t slot) const {
        for (size_t k = 0; k < slots.size(); k++)
            if (slots[k] == slot) return (int)k;
        return -1;
    }
    int add(int32_t slot, int32_t type) {
        int k = find(slot);
        if (k >= 0) return k;
        slots.push_back(slot);
        types.push_back(type);
        return (int)slots.size() - 1;
    }
};

// type lookup callback: slot -> sr_type (0 when unknown)
typedef int32_t (*slot_type_fn)(void* user, int32_t slot);

static int32_t compile_expr(sr_ctx* ctx, const sr_expr* e, VReg* reg, slot_type_fn tf, void* user, srd::CExpr* out) {
    using namespace srd;
    if (e->num_nodes <= 0 || e->num_nodes > SR_MAX_EXPR_NODES) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression has %d nodes", e->num_nodes);
    // static type stack: 0 = int class, 1 = double class
    int tst[SR_EXPR_STACK + 1];
    int sp = 0;
    int n = 0;
    auto emit = [&](int32_t op, int32_t arg, int64_t ci, double cd, bool use_d) -> bool {
        if (n >= SR_MAX_EXPR_NODES) return false;
        out->nodes[n].op = op;
        out->nodes[n].arg = arg;
        if (use_d)
            out->nodes[n].c.d = cd;
        else
            out->nodes[n].c.i = ci;
        n++;
        return true;
    };
    for (int k = 0; k < e->num_nodes; k++) {
        const sr_expr_node& nd = e->nodes[k];
        bool ok = true;
        switch (nd.op) {
        case SR_EX_COL: {
            const int32_t t = tf(user, nd.slot_id);
            if (t == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression references unknown slot %d", nd.slot_id);
            if (type_width(t) > 8) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "128-bit operands in expressions (slot %d)", nd.slot_id);
            const int id = reg->add(nd.slot_id, t);
            if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
            const int d = is_float_class(t) ? 1 : 0;
            ok = emit(d ? C_LOAD_D : C_LOAD_I, id, 0, 0, false);
            tst[sp++] = d;
            break;
        }
        case SR_EX_ICONST:
            ok = emit(C_ICONST, 0, nd.ival, 0, false);
            tst[sp++] = 0;
            break;
        case SR_EX_DCONST:
            ok = emit(C_DCONST, 0, 0, nd.dval, true);
            tst[sp++] = 1;
            break;
        case SR_EX_TO_DOUBLE:
            if (sp < 1) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression stack underflow");
            if (tst[sp - 1] == 0) ok = emit(C_I2D, 0, 0, 0, false);
            tst[sp - 1] = 1;
            break;
        case SR_EX_NOT:
        case SR_EX_IS_NULL:
            if (sp < 1) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression stack underflow");
            if (nd.op == SR_EX_NOT && tst[sp - 1] == 1) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "NOT on a double");
            ok = emit(nd.op == SR_EX_NOT ? C_NOT : C_IS_NULL, 0, 0, 0, false);
            tst[sp - 1] = 0;
            break;
        case SR_EX_AND:
        case SR_EX_OR:
            if (sp < 2) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression stack underflow");
            if (tst[sp - 1] || tst[sp - 2]) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "AND/OR on a double");
            ok = emit(nd.op == SR_EX_AND ? C_AND : C_OR, 0, 0, 0, false);
            sp--;
            tst[sp - 1] = 0;
            break;
        case SR_EX_ADD:
        case SR_EX_SUB:
        case SR_EX_MUL:
        case SR_EX_DIV:
        case SR_EX_EQ:
        case SR_EX_NE:
        case SR_EX_LT:
        case SR_EX_LE:
        case SR_EX_GT:
        case SR_EX_GE: {
            if (sp < 2) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression stack underflow");
            const bool dbl = tst[sp - 1] || tst[sp - 2] || nd.op == SR_EX_DIV;
            if (dbl) {
                if (tst[sp - 2] == 0) ok = ok && emit(C_I2D2, 0, 0, 0, false);
                if (tst[sp - 1] == 0) ok = ok && emit(C_I2D, 0, 0, 0, false);
            }
            int32_t op = 0;
            bool cmp = false;
            switch (nd.op) {
            case SR_EX_ADD:
                op = dbl ? C_ADD_D : C_ADD_I;
                break;
            case SR_EX_SUB:
                op = dbl ? C_SUB_D : C_SUB_I;
                break;
            case SR_EX_MUL:
                op = dbl ? C_MUL_D : C_MUL_I;
                break;
            case SR_EX_DIV:
                op = C_DIV_D;
                break;
            case SR_EX_EQ:
                op = dbl ? C_EQ_D : C_EQ_I;
                cmp = true;
                break;
            case SR_EX_NE:
                op = dbl ? C_NE_D : C_NE_I;
                cmp = true;
                break;
            case SR_EX_LT:
                op = dbl ? C_LT_D : C_LT_I;
                cmp = true;
                break;
            case SR_EX_LE:
                op = dbl ? C_LE_D : C_LE_I;
                cmp = true;
                break;
            case SR_EX_GT:
                op = dbl ? C_GT_D : C_GT_I;
                cmp = true;
                break;
            default:
                op = dbl ? C_GE_D : C_GE_I;
                cmp = true;
                break;
            }
            ok = ok && emit(op, 0, 0, 0, false);
            sp--;
            tst[sp - 1] = cmp ? 0 : (dbl ? 1 : 0);
            break;
        }
        default:
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown expression op %d", nd.op);
        }
        if (!ok) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "compiled expression too long");
        if (sp > SR_EXPR_STACK) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "expression stack deeper than %d", SR_EXPR_STACK);
    }
    if (sp != 1) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "expression does not reduce to one value");
    out->num_nodes = n;
    out->result_is_double = tst[0];
    out->form = srd::F_GENERIC;
    out->pad = 0;
    const auto is_load = [&](int k) { return out->nodes[k].op == srd::C_LOAD_I || out->nodes[k].op == srd::C_LOAD_D; };
    const auto is_const = [&](int k) { return out->nodes[k].op == srd::C_ICONST || out->nodes[k].op == srd::C_DCONST; };
    if (n == 1 && is_load(0)) out->form = srd::F_COL;
    if (n == 3 && is_load(0) && srd::cexpr_is_simple_arith(out->nodes[2].op)) {
        if (is_load(1)) out->form = srd::F_BIN_CC;
        if (is_const(1)) out->form = srd::F_BIN_CK;
    }
    return SR_OK;
}

static int32_t compile_pred(sr_ctx* ctx, const sr_pred* p, VReg* reg, slot_type_fn tf, void* user, srd::CPred* out) {
    const int32_t t = tf(user, p->slot_id);
    if (t == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "predicate references unknown slot %d", p->slot_id);
    if (srd::type_width(t) > 8) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "predicates on 128-bit columns");
    if (p->op < SR_PRED_EQ || p->op > SR_PRED_IS_NOT_NULL) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown predicate op %d", p->op);
    if (p->in_count < 0 || p->in_count > SR_MAX_IN_LIST) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "IN list length %d", p->in_count);
    const int id = reg->add(p->slot_id, t);
    if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
    out->value_id = id;
    out->op = p->op;
    out->is_double = srd::is_float_class(t) ? 1 : 0;
    if (out->is_double && (p->op == SR_PRED_IN || p->op == SR_PRED_NOT_IN)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "IN on a double column");
    out->in_count = p->in_count;
    out->ilo = p->ilo;
    out->ihi = p->ihi;
    out->dlo = p->dlo;
    out->dhi = p->dhi;
    for (int k = 0; k < SR_MAX_IN_LIST; k++) out->in_list[k] = p->in_list[k];
    return SR_OK;
}

// The int32 values [lo, hi] an integer EQ / LT / LE / GT / GE / BETWEEN conjunct selects: the "range form" of the scan
// and streaming-pass tests.  False when the conjunct has no such form or selects no int32 value (the generic form then
// evaluates it).  The constants are clamped to one past the int32 range first, so that LT INT64_MIN and GT INT64_MAX
// cannot overflow into a range that selects every row.
static bool pred_int32_range(const srd::CPred& cp, long long* lo_out, long long* hi_out) {
    const auto clamp = [](long long c) { return std::min<long long>(std::max<long long>(c, (long long)INT32_MIN - 1), (long long)INT32_MAX + 1); };
    const long long a = clamp(cp.ilo), b = clamp(cp.ihi);
    long long lo = INT32_MIN, hi = INT32_MAX;
    switch (cp.op) {
    case SR_PRED_EQ: lo = hi = a; break;
    case SR_PRED_LT: hi = a - 1; break;
    case SR_PRED_LE: hi = a; break;
    case SR_PRED_GT: lo = a + 1; break;
    case SR_PRED_GE: lo = a; break;
    case SR_PRED_BETWEEN: lo = a; hi = b; break;
    default: return false;
    }
    lo = std::max<long long>(lo, INT32_MIN);
    hi = std::min<long long>(hi, INT32_MAX);
    if (cp.is_double || lo > hi) return false;
    *lo_out = lo;
    *hi_out = hi;
    return true;
}

// fill a VTab from a staged chunk for the slots registered in reg
static int32_t bind_vtab(sr_ctx* ctx, const VReg& reg, const Staged& st, VTab* vt) {
    vt->n = (int32_t)reg.slots.size();
    for (size_t k = 0; k < reg.slots.size(); k++) {
        const int c = st.find(reg.slots[k]);
        if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk misses slot %d", reg.slots[k]);
        if (st.cols[c].type != reg.types[k])
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "slot %d changed type (%d -> %d)", reg.slots[k], reg.types[k], st.cols[c].type);
        vt->v[k].data = st.cols[c].data;
        vt->v[k].nulls = st.cols[c].nulls;
        vt->v[k].type = st.cols[c].type;
        vt->v[k].src = -1;
    }
    vt_mark_plain32(vt);
    return SR_OK;
}

static inline int grid_for(int64_t items, int per_block) {
    int64_t g = (items + per_block - 1) / per_block;
    if (g < 1) g = 1;
    if (g > 0x7fffffff) g = 0x7fffffff;
    return (int)g;
}
