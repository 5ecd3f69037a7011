// sr_host.cuh -- host-side plumbing of libsr_gpu.so: context, device buffers, error handling,
// compilation of sr_pred / sr_expr descriptors against a chunk's slots.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
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

static inline const sr_col_view* find_col(const sr_chunk_view* c, int32_t slot) {
    for (int k = 0; k < c->num_cols; k++)
        if (c->cols[k].slot_id == slot) return &c->cols[k];
    return nullptr;
}

// A chunk made resident on the device: host chunks are staged (H2D on the ctx stream) into
// buffers owned by `Staged`; device chunks are referenced in place.
struct Staged {
    std::vector<DevBuf> bufs; // 2 per column (data, nulls)
    std::vector<srd::DCol> cols;
    std::vector<int32_t> slots;
    int64_t num_rows = 0;
    // device-visible alias of a page-locked, mapped host buffer (SR_MEM_HOST_PINNED); fails for pageable memory
    static int32_t mapped_alias(sr_ctx* ctx, const void* host, int32_t slot, const void** dev) {
        cudaPointerAttributes at;
        memset(&at, 0, sizeof(at));
        if (cudaPointerGetAttributes(&at, host) != cudaSuccess || at.type != cudaMemoryTypeHost || at.devicePointer == nullptr) {
            cudaGetLastError();
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "slot %d: SR_MEM_HOST_PINNED buffer is not page-locked mapped host memory", slot);
        }
        *dev = at.devicePointer;
        return SR_OK;
    }
    int32_t stage(sr_ctx* ctx, const sr_chunk_view* in, const std::vector<int32_t>* only_slots = nullptr, bool in_place_pinned = false) {
        cols.clear();
        slots.clear();
        num_rows = in->num_rows;
        if (in->mem != SR_MEM_HOST && in->mem != SR_MEM_DEVICE && in->mem != SR_MEM_HOST_PINNED)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown memory kind %d", in->mem);
        if ((int)bufs.size() < 2 * in->num_cols) {
            std::vector<DevBuf> nb(2 * in->num_cols);
            for (size_t i = 0; i < bufs.size(); i++) std::swap(nb[i], bufs[i]);
            bufs.swap(nb);
        }
        for (int k = 0; k < in->num_cols; k++) {
            const sr_col_view& c = in->cols[k];
            if (only_slots && std::find(only_slots->begin(), only_slots->end(), c.slot_id) == only_slots->end()) continue;
            const int w = srd::type_width(c.type);
            if (w == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown column type %d (slot %d)", c.type, c.slot_id);
            if (in->num_rows > 0 && c.data == nullptr)
                return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "null data pointer (slot %d)", c.slot_id);
            srd::DCol d;
            d.type = c.type;
            d.width = w;
            if (in->mem == SR_MEM_DEVICE) {
                d.data = c.data;
                d.nulls = c.nulls;
            } else if (in->mem == SR_MEM_HOST_PINNED && in_place_pinned && in->num_rows > 0) {
                const void* p = nullptr;
                SR_TRY(mapped_alias(ctx, c.data, c.slot_id, &p));
                d.data = p;
                d.nulls = nullptr;
                if (c.nulls) {
                    SR_TRY(mapped_alias(ctx, c.nulls, c.slot_id, &p));
                    d.nulls = (const uint8_t*)p;
                }
            } else {
                SR_TRY(bufs[2 * k].reserve(ctx, (size_t)in->num_rows * w + 16));
                SR_CUDA(ctx, cudaMemcpyAsync(bufs[2 * k].p, c.data, (size_t)in->num_rows * w, cudaMemcpyHostToDevice, ctx->stream));
                d.data = bufs[2 * k].p;
                d.nulls = nullptr;
                if (c.nulls) {
                    SR_TRY(bufs[2 * k + 1].reserve(ctx, (size_t)in->num_rows + 16));
                    SR_CUDA(ctx, cudaMemcpyAsync(bufs[2 * k + 1].p, c.nulls, (size_t)in->num_rows, cudaMemcpyHostToDevice, ctx->stream));
                    d.nulls = (const uint8_t*)bufs[2 * k + 1].p;
                }
            }
            cols.push_back(d);
            slots.push_back(c.slot_id);
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
