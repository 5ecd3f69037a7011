// sr_serde.cuh -- ChunkPB.data wire format of the exchange (SURVEY.md 8f-3), encode level 0:
//   ProtobufChunkSerde::serialize_without_meta      be/src/serde/protobuf_serde.cpp:88-140   (version, num_rows, columns)
//   FixedLengthColumnSerde::serialize / deserialize be/src/serde/column_array_serde.cpp:214-255 (fixed32 byte size + raw values)
//   NullableColumnSerde                             be/src/serde/column_array_serde.cpp:759-782 (null column, then data column)
// Column payloads are moved with one byte-exact copy each (cudaMemcpyAsync: the offsets inside the payload are only 4-byte
// aligned at best); the small header words are written by one kernel (device destination) or by the host.
#pragma once

struct sr_serde {
    sr_ctx* ctx = nullptr;
    ColBufs cols;   // the deserialized columns
    DevBuf staging; // host payloads are copied to the device once, then split
};

namespace srd {
struct SerdeWord {
    unsigned long long offset;
    uint32_t value;
    uint32_t pad;
};
struct SerdeWords {
    SerdeWord w[2 + 2 * SR_MAX_OUT_COLS];
    int32_t n;
};
// little-endian fixed32 words at arbitrary byte offsets of the payload
__global__ void k_serde_header(uint8_t* __restrict__ dst, const __grid_constant__ SerdeWords words) {
    const int i = threadIdx.x;
    if (i < words.n) {
        uint8_t* p = dst + words.w[i].offset;
        const uint32_t v = words.w[i].value;
        p[0] = (uint8_t)v;
        p[1] = (uint8_t)(v >> 8);
        p[2] = (uint8_t)(v >> 16);
        p[3] = (uint8_t)(v >> 24);
    }
}
} // namespace srd

static int64_t serde_size(const sr_chunk_view* c, int64_t rows) {
    int64_t b = 8;
    for (int k = 0; k < c->num_cols; k++) {
        const int w = srd::type_width(c->cols[k].type);
        if (c->cols[k].nulls) b += 4 + rows;
        b += 4 + rows * w;
    }
    return b;
}

static int32_t serde_serialize(sr_ctx* ctx, const sr_chunk_view* c, int64_t r0, int64_t r1, void* dst, int64_t cap, int32_t dst_mem, sr_chunk_pb_meta* meta) {
    SR_TRY(chunk_check(ctx, c));
    if (c->num_cols > SR_MAX_OUT_COLS) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%d columns", c->num_cols);
    if (r0 < 0 || r1 < r0 || r1 > c->num_rows) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "rows [%lld, %lld) of %lld", (long long)r0, (long long)r1, (long long)c->num_rows);
    const int64_t rows = r1 - r0;
    for (int k = 0; k < c->num_cols; k++) {
        int w;
        SR_TRY(col_check(ctx, c->cols[k], c->num_rows, false, &w)); // copied: any alignment
        if (rows * w >= (1ll << 32)) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "a column of %lld bytes: the format stores sizes as uint32", (long long)(rows * w));
    }
    const int64_t total = serde_size(c, rows);
    if (total > cap) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "destination of %lld bytes, %lld needed", (long long)cap, (long long)total);
    SR_TRY(mem_check(ctx, dst_mem, "dst_mem"));
    const bool dst_dev = !mem_is_host(dst_mem), src_dev = !mem_is_host(c->mem);
    const cudaMemcpyKind kind = src_dev ? (dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost) : (dst_dev ? cudaMemcpyHostToDevice : cudaMemcpyHostToHost);
    uint8_t* out = (uint8_t*)dst;
    srd::SerdeWords words;
    words.n = 0;
    auto word = [&](int64_t off, uint32_t v) {
        words.w[words.n].offset = (unsigned long long)off;
        words.w[words.n].value = v;
        words.n++;
    };
    word(0, 1u);             // version
    word(4, (uint32_t)rows); // num_rows
    int64_t off = 8;
    for (int k = 0; k < c->num_cols; k++) {
        const sr_col_view& col = c->cols[k];
        const int w = srd::type_width(col.type);
        if (col.nulls) {
            word(off, (uint32_t)rows);
            off += 4;
            if (rows) SR_CUDA(ctx, cudaMemcpyAsync(out + off, col.nulls + r0, (size_t)rows, kind, ctx->stream));
            off += rows;
        }
        word(off, (uint32_t)(rows * w));
        off += 4;
        if (rows) SR_CUDA(ctx, cudaMemcpyAsync(out + off, (const uint8_t*)col.data + r0 * w, (size_t)(rows * w), kind, ctx->stream));
        off += rows * w;
        if (meta) {
            meta->slot_ids[k] = col.slot_id;
            meta->types[k] = col.type;
            meta->is_nulls[k] = col.nulls ? 1 : 0;
            meta->is_consts[k] = 0;
        }
    }
    if (dst_dev) {
        srd::k_serde_header<<<1, 2 + 2 * SR_MAX_OUT_COLS, 0, ctx->stream>>>(out, words);
        SR_LAUNCH_CHECK(ctx);
    } else {
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the payload copies have landed; the host writes the header words
        for (int i = 0; i < words.n; i++) {
            const uint32_t v = words.w[i].value;
            uint8_t* p = out + words.w[i].offset;
            p[0] = (uint8_t)v, p[1] = (uint8_t)(v >> 8), p[2] = (uint8_t)(v >> 16), p[3] = (uint8_t)(v >> 24);
        }
    }
    if (meta) {
        meta->serialized_size = total;
        meta->num_rows = rows;
        meta->num_cols = c->num_cols;
        meta->reserved = 0;
    }
    return SR_OK;
}

// The payload must be exactly what serde_serialize writes for `meta`: a const column (ConstColumnSerde) is refused, and
// so are a header num_rows other than meta->num_rows, a size other than meta->serialized_size and bytes left after the
// last column.  The whole layout is checked before the first column is copied, so a refused payload queues no copy.
static int32_t serde_deserialize(sr_serde* h, const void* src, int64_t bytes, int32_t src_mem, const sr_chunk_pb_meta* meta, sr_chunk_out* out) {
    sr_ctx* ctx = h->ctx;
    SR_TRY(mem_check(ctx, src_mem, "src_mem"));
    if (meta->num_cols < 0 || meta->num_cols > SR_MAX_OUT_COLS) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%d columns", meta->num_cols);
    for (int k = 0; k < meta->num_cols; k++)
        if (meta->is_consts[k]) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "column %d is a const column: ConstColumnSerde payloads are not parsed", k);
    if (bytes < 8) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "payload of %lld bytes has no header", (long long)bytes);
    if (bytes != meta->serialized_size)
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "payload of %lld bytes, meta.serialized_size %lld", (long long)bytes, (long long)meta->serialized_size);
    // the header words and the per-column sizes steer the parse: read them on the host (device payload: the first pass
    // copies the whole payload's size words one by one -- at most 2 per column)
    const bool src_dev = !mem_is_host(src_mem);
    const uint8_t* in = (const uint8_t*)src;
    auto read32 = [&](int64_t off, uint32_t* v) -> int32_t {
        if (off + 4 > bytes) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "payload truncated at byte %lld", (long long)off);
        uint8_t b[4];
        if (src_dev) {
            SR_CUDA(ctx, cudaMemcpyAsync(b, in + off, 4, cudaMemcpyDeviceToHost, ctx->stream));
            SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        } else {
            memcpy(b, in + off, 4);
        }
        *v = (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
        return SR_OK;
    };
    uint32_t version = 0, rows = 0;
    SR_TRY(read32(0, &version));
    SR_TRY(read32(4, &rows));
    if (version != 1) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "ChunkPB.data version %u (expected 1)", version);
    if ((int64_t)rows != meta->num_rows)
        return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "payload header says %u rows, meta.num_rows %lld", rows, (long long)meta->num_rows);
    int64_t null_off[SR_MAX_OUT_COLS], data_off[SR_MAX_OUT_COLS], data_size[SR_MAX_OUT_COLS];
    int64_t off = 8;
    for (int k = 0; k < meta->num_cols; k++) {
        const int w = srd::type_width(meta->types[k]);
        if (w == 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "unknown column type %d", meta->types[k]);
        uint32_t sz = 0;
        null_off[k] = -1;
        if (meta->is_nulls[k]) {
            SR_TRY(read32(off, &sz));
            off += 4;
            if (sz != rows || off + sz > bytes) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "column %d: null column of %u bytes for %u rows", k, sz, rows);
            null_off[k] = off;
            off += sz;
        }
        SR_TRY(read32(off, &sz));
        off += 4;
        if ((int64_t)sz != (int64_t)rows * w || off + sz > bytes)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "column %d: %u bytes for %u rows of width %d", k, sz, rows, w);
        data_off[k] = off;
        data_size[k] = sz;
        off += sz;
    }
    if (off != bytes) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "%lld bytes after the last column", (long long)(bytes - off));
    const cudaMemcpyKind kind = src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    h->cols.resize(meta->num_cols);
    ColBufs::header(out, meta->num_cols, rows);
    for (int k = 0; k < meta->num_cols; k++) {
        void* data;
        uint8_t* nulls;
        SR_TRY(h->cols.reserve(ctx, k, rows, srd::type_width(meta->types[k]), null_off[k] >= 0, &data, &nulls));
        if (nulls && rows) SR_CUDA(ctx, cudaMemcpyAsync(nulls, in + null_off[k], rows, kind, ctx->stream));
        if (data_size[k]) SR_CUDA(ctx, cudaMemcpyAsync(data, in + data_off[k], (size_t)data_size[k], kind, ctx->stream));
        h->cols.fill(out, k, meta->types[k], meta->slot_ids[k]);
    }
    return mem_sync(ctx, src_mem); // the caller's host buffer may go away
}
