// Minimal API-compatible mirror of the StarRocks column data model for the GPU operator adapters.
// Same names / method meaning as the reference so an adapter written against this header reads like BE code:
//   Chunk                     be/src/column/chunk.h:52-354 (columns + slot_id -> index map, num_rows, append_column,
//                             get_column_by_slot_id, filter, ...)
//   FixedLengthColumnBase<T>  be/src/column/fixed_length_column_base.h:49-286 (contiguous Buffer<T>, raw_data, size)
//   NullableColumn            be/src/column/nullable_column.h:32-110 (data column + uint8 null column, 1 = NULL)
// Only what the hot path touches is here (fixed-length columns, nullable wrapper; the string column of the plan around
// it is column/binary_column.h).  In the real BE these are the
// BE's own classes; the adapters only need raw_data()/null data()/size()/slot ids.
#pragma once

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/sr_gpu_ops.h"

namespace starrocks {

using SlotId = int32_t;

class Column {
public:
    virtual ~Column() = default;
    virtual size_t size() const = 0;
    virtual bool is_nullable() const { return false; }
    virtual int32_t logical_type() const = 0; // sr_type
    virtual const uint8_t* raw_data() const = 0;
    virtual uint8_t* mutable_raw_data() = 0;
    virtual const uint8_t* null_data() const { return nullptr; }
    virtual void resize(size_t n) = 0;
    virtual size_t type_size() const = 0;
    // variable-length payload (column/binary_column.h): rows are not type_size() apart
    virtual bool is_binary() const { return false; }
    // rows [offset, offset + n) as a new column; nullptr = fixed-length payload, the caller copies n * type_size() bytes
    virtual std::shared_ptr<Column> cut(size_t offset, size_t n) const { return nullptr; }
};
using ColumnPtr = std::shared_ptr<Column>;
using Columns = std::vector<ColumnPtr>;

template <typename T>
class FixedLengthColumn final : public Column {
public:
    using Container = std::vector<T>;
    explicit FixedLengthColumn(int32_t logical_type) : _type(logical_type) {}
    FixedLengthColumn(int32_t logical_type, Container data) : _type(logical_type), _data(std::move(data)) {}
    static std::shared_ptr<FixedLengthColumn<T>> create(int32_t logical_type) { return std::make_shared<FixedLengthColumn<T>>(logical_type); }
    size_t size() const override { return _data.size(); }
    int32_t logical_type() const override { return _type; }
    const uint8_t* raw_data() const override { return reinterpret_cast<const uint8_t*>(_data.data()); }
    uint8_t* mutable_raw_data() override { return reinterpret_cast<uint8_t*>(_data.data()); }
    void resize(size_t n) override { _data.resize(n); }
    size_t type_size() const override { return sizeof(T); }
    Container& get_data() { return _data; }
    const Container& get_data() const { return _data; }
    void append(const T& v) { _data.push_back(v); }

private:
    int32_t _type;
    Container _data;
};

using Int8Column = FixedLengthColumn<int8_t>;
using Int16Column = FixedLengthColumn<int16_t>;
using Int32Column = FixedLengthColumn<int32_t>;
using Int64Column = FixedLengthColumn<int64_t>;
using DoubleColumn = FixedLengthColumn<double>;
using UInt8Column = FixedLengthColumn<uint8_t>;
using NullColumn = UInt8Column;

// A fixed-length column over memory it does not own: the reference's ContainerResource-backed columns
// (be/src/column/container_resource.h:24), which is how the buffers of a pinned ColumnAllocator pool appear in a chunk.
// `owner` keeps the memory alive (a slice of a PinnedArena, say); the column cannot grow past the borrowed rows.
class BorrowedColumn final : public Column {
public:
    BorrowedColumn(int32_t logical_type, void* data, size_t rows, std::shared_ptr<const void> owner)
            : _type(logical_type), _data((uint8_t*)data), _rows(rows), _cap(rows), _owner(std::move(owner)) {}
    size_t size() const override { return _rows; }
    int32_t logical_type() const override { return _type; }
    const uint8_t* raw_data() const override { return _data; }
    uint8_t* mutable_raw_data() override { return _data; }
    void resize(size_t n) override {
        if (n > _cap) throw std::runtime_error("BorrowedColumn: cannot grow past the " + std::to_string(_cap) + " borrowed rows");
        _rows = n;
    }
    size_t type_size() const override { return (size_t)sr_type_width(_type); }

private:
    int32_t _type;
    uint8_t* _data;
    size_t _rows, _cap;
    std::shared_ptr<const void> _owner;
};

// One page-locked, device-mapped arena (sr_host_register) handing out aligned slices: the pinned ColumnAllocator pool
// of INTEGRATION.md section 3 in miniature.  A slice is never returned to the arena; the arena is unregistered and freed
// when the last column borrowing from it is gone (every slice holds the arena).
class PinnedArena : public std::enable_shared_from_this<PinnedArena> {
public:
    static constexpr size_t ALIGN = 64;
    // StatusOr-free factory: nullptr and the library's message in *err when the registration fails
    static std::shared_ptr<PinnedArena> create(sr_ctx* ctx, size_t bytes, std::string* err) {
        auto a = std::shared_ptr<PinnedArena>(new PinnedArena(ctx, bytes));
        if (!a->_base) {
            *err = "PinnedArena: out of host memory";
            return nullptr;
        }
        if (sr_host_register(ctx, a->_base, (int64_t)a->_cap) != SR_OK) {
            *err = std::string("PinnedArena: ") + sr_last_error(ctx);
            return nullptr;
        }
        a->_registered = true;
        return a;
    }
    ~PinnedArena() {
        if (_registered) sr_host_unregister(_ctx, _base);
        free(_base);
    }
    // `bytes` at an ALIGN-byte boundary, or nullptr when the arena is full (thread-safe)
    void* slice(size_t bytes) {
        const size_t want = (bytes + ALIGN - 1) & ~(ALIGN - 1);
        size_t off = _used.fetch_add(want);
        if (off + want > _cap) return nullptr;
        return _base + off;
    }
    // a column of `rows` values of `logical_type` in a fresh slice (nullptr when full)
    std::shared_ptr<BorrowedColumn> column(int32_t logical_type, size_t rows) {
        void* p = slice(std::max<size_t>(rows, 1) * (size_t)sr_type_width(logical_type));
        return p ? std::make_shared<BorrowedColumn>(logical_type, p, rows, shared_from_this()) : nullptr;
    }
    size_t capacity() const { return _cap; }

private:
    PinnedArena(sr_ctx* ctx, size_t bytes) : _ctx(ctx), _cap((std::max<size_t>(bytes, 1) + 4095) & ~(size_t)4095) {
        _base = (uint8_t*)aligned_alloc(4096, _cap);
    }
    sr_ctx* _ctx;
    size_t _cap;
    uint8_t* _base = nullptr;
    bool _registered = false;
    std::atomic<size_t> _used{0};
};

// the data column and the uint8 null column (1 = NULL): owned (NullColumn) or borrowed (BorrowedColumn) buffers
class NullableColumn final : public Column {
public:
    NullableColumn(ColumnPtr data, ColumnPtr nulls) : _data(std::move(data)), _nulls(std::move(nulls)) {}
    size_t size() const override { return _data->size(); }
    bool is_nullable() const override { return true; }
    bool is_binary() const override { return _data->is_binary(); }
    int32_t logical_type() const override { return _data->logical_type(); }
    const uint8_t* raw_data() const override { return _data->raw_data(); }
    uint8_t* mutable_raw_data() override { return _data->mutable_raw_data(); }
    const uint8_t* null_data() const override { return _nulls->raw_data(); }
    void resize(size_t n) override {
        _data->resize(n);
        _nulls->resize(n);
    }
    size_t type_size() const override { return _data->type_size(); }
    const ColumnPtr& data_column() const { return _data; }
    const ColumnPtr& null_column() const { return _nulls; }

private:
    ColumnPtr _data;
    ColumnPtr _nulls;
};

inline ColumnPtr make_column(int32_t logical_type, size_t rows) {
    ColumnPtr c;
    switch (sr_type_width(logical_type)) {
    case 1:
        c = std::make_shared<FixedLengthColumn<int8_t>>(logical_type);
        break;
    case 2:
        c = std::make_shared<FixedLengthColumn<int16_t>>(logical_type);
        break;
    case 4:
        c = std::make_shared<FixedLengthColumn<int32_t>>(logical_type);
        break;
    case 8:
        c = std::make_shared<FixedLengthColumn<int64_t>>(logical_type);
        break;
    case 16:
        c = std::make_shared<FixedLengthColumn<__int128>>(logical_type);
        break;
    default:
        throw std::runtime_error("make_column: unsupported logical type " + std::to_string(logical_type));
    }
    c->resize(rows);
    return c;
}

class Chunk {
public:
    Chunk() = default;
    size_t num_rows() const { return _columns.empty() ? 0 : _columns[0]->size(); }
    size_t num_columns() const { return _columns.size(); }
    bool is_empty() const { return num_rows() == 0; }
    void append_column(ColumnPtr column, SlotId slot_id) {
        _slot_id_to_index[slot_id] = _columns.size();
        _slots.push_back(slot_id);
        _columns.push_back(std::move(column));
    }
    bool is_slot_exist(SlotId id) const { return _slot_id_to_index.count(id) != 0; }
    const ColumnPtr& get_column_by_slot_id(SlotId id) const { return _columns[_slot_id_to_index.at(id)]; }
    const ColumnPtr& get_column_by_index(size_t i) const { return _columns[i]; }
    SlotId slot_of_index(size_t i) const { return _slots[i]; }
    const Columns& columns() const { return _columns; }

    // rows [offset, offset + n) as a new Chunk (Chunk::clone_empty + append_safe in the reference)
    std::shared_ptr<Chunk> slice(size_t offset, size_t n) const {
        auto out = std::make_shared<Chunk>();
        for (size_t i = 0; i < _columns.size(); i++) {
            const Column& src = *_columns[i];
            const Column& payload = src.is_nullable() ? *static_cast<const NullableColumn&>(src).data_column() : src;
            ColumnPtr data = payload.cut(offset, n);
            if (!data) {
                data = make_column(src.logical_type(), n);
                memcpy(data->mutable_raw_data(), src.raw_data() + offset * src.type_size(), n * src.type_size());
            }
            if (src.is_nullable()) {
                auto nulls = std::make_shared<NullColumn>(SR_TYPE_BOOLEAN);
                nulls->resize(n);
                memcpy(nulls->mutable_raw_data(), src.null_data() + offset, n);
                out->append_column(std::make_shared<NullableColumn>(data, nulls), _slots[i]);
            } else {
                out->append_column(data, _slots[i]);
            }
        }
        return out;
    }

private:
    Columns _columns;
    std::vector<SlotId> _slots;
    std::unordered_map<SlotId, size_t> _slot_id_to_index;
};
using ChunkPtr = std::shared_ptr<Chunk>;

// Chunk -> sr_chunk_view over the columns' own host buffers (no copy).  `cols` must outlive the view.
inline sr_chunk_view make_chunk_view(const Chunk& chunk, std::vector<sr_col_view>* cols) {
    cols->clear();
    for (size_t i = 0; i < chunk.num_columns(); i++) {
        const Column& c = *chunk.get_column_by_index(i);
        cols->push_back(sr_col_view{c.raw_data(), c.null_data(), c.logical_type(), chunk.slot_of_index(i)});
    }
    return sr_chunk_view{cols->data(), (int32_t)cols->size(), SR_MEM_HOST, (int64_t)chunk.num_rows()};
}

} // namespace starrocks
