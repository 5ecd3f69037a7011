// GPU drop-in operators for the StarRocks pipeline engine, written against the reference's Operator /
// OperatorFactory interface (exec/pipeline/operator.h) and the C-ABI of libsr_gpu.so (include/sr_gpu_ops.h).
//
//   GpuScanOperator                      <- ScanOperator + OlapChunkSource filter step
//                                           (exec/pipeline/scan/scan_operator.cpp:286-309, olap_chunk_source.cpp:676-722)
//   GpuHashJoinBuildOperator             <- HashJoinBuildOperator   (exec/pipeline/hashjoin/hash_join_build_operator.cpp:41-220)
//   GpuHashJoinProbeOperator             <- HashJoinProbeOperator   (exec/pipeline/hashjoin/hash_join_probe_operator.cpp:55-117)
//   GpuAggregateBlockingSinkOperator     <- AggregateBlockingSinkOperator   (aggregate/aggregate_blocking_sink_operator.cpp:56-138)
//   GpuAggregateBlockingSourceOperator   <- AggregateBlockingSourceOperator (aggregate/aggregate_blocking_source_operator.cpp:46-72)
//   GpuFragmentSinkOperator              the fused form: the scan's downstream probes + aggregate sink collapsed into
//                                           one sink that feeds sr_fragment_push (SURVEY.md section 7: "keep the API, change
//                                           the cadence")
// Shared contexts mirror HashJoiner / Aggregator (exec/hash_joiner.h:191-330, exec/aggregator.h:253-637): one object
// shared by the build and probe (sink and source) operators, ref-counted through shared_ptr.
//
// Cadence: the pipeline contract is <= chunk_size (4096) rows per chunk.  One kernel launch per 4096 rows is hopeless
// on a GPU, so every operator accumulates `batch_chunks` input chunks (64, the IO-task batch of the reference's
// ChunkSource, scan_operator.h:119) into one contiguous batch before calling the library, and slices device results
// back into <= chunk_size chunks.  need_input() / has_output() expose exactly that buffering to the driver.
#pragma once

#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../exec/pipeline/operator.h"

namespace starrocks::pipeline {

inline Status sr_to_status(sr_ctx* ctx, int32_t rc) {
    if (rc == SR_OK) return Status::OK();
    const std::string msg = std::string("sr_gpu: ") + sr_last_error(ctx);
    switch (rc) {
    case SR_ERR_INVALID_ARGUMENT:
        return Status::InvalidArgument(msg);
    case SR_ERR_NOT_SUPPORTED:
        return Status::NotSupported(msg);
    case SR_ERR_OUT_OF_MEMORY:
        return Status::MemoryLimitExceeded(msg);
    default:
        return Status::InternalError(msg);
    }
}
#define RETURN_IF_SR_ERROR(ctx, expr) RETURN_IF_ERROR(sr_to_status((ctx), (expr)))

// contiguous accumulation of equal-schema host chunks (the batch handed to one library call)
class ChunkBatch {
public:
    void append(const Chunk& c) {
        if (_cols.empty()) {
            for (size_t i = 0; i < c.num_columns(); i++) {
                const Column& col = *c.get_column_by_index(i);
                _cols.push_back(Col{c.slot_of_index(i), col.logical_type(), col.type_size(), col.is_nullable(), {}, {}});
            }
        }
        const size_t n = c.num_rows();
        for (size_t i = 0; i < _cols.size(); i++) {
            Col& dst = _cols[i];
            const Column& col = *c.get_column_by_slot_id(dst.slot);
            const size_t old = dst.data.size();
            dst.data.resize(old + n * dst.width);
            memcpy(dst.data.data() + old, col.raw_data(), n * dst.width);
            if (col.is_nullable() && !dst.nullable) { // upgrade like JoinHashTable::append_chunk does
                dst.nullable = true;
                dst.nulls.assign(_rows, 0);
            }
            if (dst.nullable) {
                const size_t oldn = dst.nulls.size();
                dst.nulls.resize(oldn + n, 0);
                if (col.is_nullable()) memcpy(dst.nulls.data() + oldn, col.null_data(), n);
            }
        }
        _rows += n;
    }
    size_t rows() const { return _rows; }
    bool empty() const { return _rows == 0; }
    void clear() {
        for (auto& c : _cols) {
            c.data.clear();
            c.nulls.clear();
        }
        _rows = 0;
    }
    sr_chunk_view view() {
        _views.clear();
        for (auto& c : _cols) _views.push_back(sr_col_view{c.data.data(), c.nullable ? c.nulls.data() : nullptr, c.type, c.slot});
        return sr_chunk_view{_views.data(), (int32_t)_views.size(), SR_MEM_HOST, (int64_t)_rows};
    }

private:
    struct Col {
        SlotId slot;
        int32_t type;
        size_t width;
        bool nullable;
        std::vector<uint8_t> data, nulls;
    };
    std::vector<Col> _cols;
    std::vector<sr_col_view> _views;
    size_t _rows = 0;
};

// The same accumulation into PAGE-LOCKED, device-mapped buffers of a fixed row capacity (sr_host_alloc: what a
// cudaHostRegister-ed ColumnAllocator pool would be in the BE).  The library reads such a batch in place over PCIe
// (SR_MEM_HOST_PINNED) or DMA-copies it without a staging bounce; the operator may refill it only after the event it
// recorded behind the push has completed.  Non-nullable fixed-length columns (the fact tables of the hot path).
class PinnedChunkBatch {
public:
    PinnedChunkBatch() = default;
    PinnedChunkBatch(const PinnedChunkBatch&) = delete;
    PinnedChunkBatch& operator=(const PinnedChunkBatch&) = delete;
    ~PinnedChunkBatch() { release(); }
    Status init(sr_ctx* ctx, const Chunk& schema, size_t capacity_rows) {
        _ctx = ctx;
        _cap = capacity_rows;
        for (size_t i = 0; i < schema.num_columns(); i++) {
            const Column& col = *schema.get_column_by_index(i);
            if (col.is_nullable()) return Status::NotSupported("PinnedChunkBatch: nullable column (slot " + std::to_string(schema.slot_of_index(i)) + ")");
            Col c{schema.slot_of_index(i), col.logical_type(), col.type_size(), nullptr};
            void* p = nullptr;
            RETURN_IF_SR_ERROR(ctx, sr_host_alloc(ctx, (int64_t)(capacity_rows * c.width), &p));
            c.data = (uint8_t*)p;
            _cols.push_back(c);
        }
        _event = sr_event_create(ctx);
        return _event ? Status::OK() : sr_to_status(ctx, sr_last_error_code(ctx));
    }
    bool initialised() const { return _event != nullptr; }
    void release() {
        for (auto& c : _cols)
            if (c.data) sr_host_free(_ctx, c.data);
        _cols.clear();
        if (_event) sr_event_destroy(_event);
        _event = nullptr;
    }
    size_t rows() const { return _rows; }
    size_t room() const { return _cap - _rows; }
    size_t bytes() const {
        size_t b = 0;
        for (auto& c : _cols) b += _rows * c.width;
        return b;
    }
    void append(const Chunk& c, size_t from = 0) { // rows [from, from + min(room, rest)) of the chunk
        const size_t n = std::min(room(), c.num_rows() - from);
        for (auto& dst : _cols) memcpy(dst.data + _rows * dst.width, c.get_column_by_slot_id(dst.slot)->raw_data() + from * dst.width, n * dst.width);
        _rows += n;
    }
    sr_chunk_view view() {
        _views.clear();
        for (auto& c : _cols) _views.push_back(sr_col_view{c.data, nullptr, c.type, c.slot});
        return sr_chunk_view{_views.data(), (int32_t)_views.size(), SR_MEM_HOST_PINNED, (int64_t)_rows};
    }
    // in flight: handed to the library, the event behind that work has not completed yet
    Status mark_submitted() {
        RETURN_IF_SR_ERROR(_ctx, sr_event_record(_event));
        _in_flight = true;
        return Status::OK();
    }
    bool busy() { // non-blocking
        if (_in_flight && sr_event_query(_event) != 0) {
            _in_flight = false;
            _rows = 0;
        }
        return _in_flight;
    }
    void wait() {
        if (_in_flight) sr_event_sync(_event);
        _in_flight = false;
        _rows = 0;
    }

private:
    struct Col {
        SlotId slot;
        int32_t type;
        size_t width;
        uint8_t* data;
    };
    sr_ctx* _ctx = nullptr;
    std::vector<Col> _cols;
    std::vector<sr_col_view> _views;
    sr_event* _event = nullptr;
    size_t _cap = 0, _rows = 0;
    bool _in_flight = false;
};

// Chunks handed to the library as they are: every data and null buffer lies in a page-locked range the library knows
// (sr_host_is_mapped: a registered ColumnAllocator pool), so no byte is copied on the host.  The list keeps the ChunkPtrs
// of its chunks until the event recorded behind their sr_fragment_push_chunks has completed.
class ForwardedChunkList {
public:
    ForwardedChunkList() = default;
    ForwardedChunkList(const ForwardedChunkList&) = delete;
    ForwardedChunkList& operator=(const ForwardedChunkList&) = delete;
    ~ForwardedChunkList() {
        if (_event) sr_event_destroy(_event);
    }
    // true when the chunk can be forwarded: fixed-length columns whose buffers all lie in page-locked mapped ranges
    static bool forwardable(sr_ctx* ctx, const Chunk& c) {
        const size_t n = c.num_rows();
        for (size_t i = 0; i < c.num_columns(); i++) {
            const Column& col = *c.get_column_by_index(i);
            if (col.is_binary() || sr_host_is_mapped(ctx, col.raw_data(), (int64_t)(n * col.type_size())) != 1) return false;
            if (col.is_nullable() && sr_host_is_mapped(ctx, col.null_data(), (int64_t)n) != 1) return false;
        }
        return true;
    }
    Status add(sr_ctx* ctx, const ChunkPtr& c) {
        if (!_event) {
            _ctx = ctx;
            _event = sr_event_create(ctx);
            if (!_event) return sr_to_status(ctx, sr_last_error_code(ctx));
        }
        _chunks.push_back(c);
        _rows += c->num_rows();
        return Status::OK();
    }
    size_t rows() const { return _in_flight ? 0 : _rows; }
    size_t num_chunks() const { return _chunks.size(); }
    // one sr_fragment_push_chunks of the whole list, an event behind it
    Status submit(sr_fragment* frag) {
        _cols.resize(_chunks.size());
        _views.clear();
        for (size_t k = 0; k < _chunks.size(); k++) {
            sr_chunk_view v = make_chunk_view(*_chunks[k], &_cols[k]);
            v.mem = SR_MEM_HOST_PINNED;
            _views.push_back(v);
        }
        RETURN_IF_SR_ERROR(_ctx, sr_fragment_push_chunks(frag, _views.data(), (int32_t)_views.size()));
        RETURN_IF_SR_ERROR(_ctx, sr_event_record(_event));
        _in_flight = true;
        return Status::OK();
    }
    bool busy() { // non-blocking; releases the chunks once the library is done with them
        if (_in_flight && sr_event_query(_event) != 0) release();
        return _in_flight;
    }
    void wait() {
        if (_in_flight) sr_event_sync(_event);
        release();
    }

private:
    void release() {
        _in_flight = false;
        _chunks.clear();
        _rows = 0;
    }
    sr_ctx* _ctx = nullptr;
    sr_event* _event = nullptr;
    std::vector<ChunkPtr> _chunks;
    std::vector<std::vector<sr_col_view>> _cols;
    std::vector<sr_chunk_view> _views;
    size_t _rows = 0;
    bool _in_flight = false;
};

// counters every GPU operator keeps in its _unique_metrics, sampled from the context at the operator's life-cycle points
struct GpuOpCounters {
    RuntimeProfile::Counter* launches = nullptr;
    RuntimeProfile::Counter* device_bytes = nullptr;
    void init(RuntimeProfile* p) {
        launches = ADD_COUNTER(p, "GpuKernelLaunches", TUnit::UNIT);
        device_bytes = ADD_COUNTER(p, "GpuDeviceBytes", TUnit::BYTES);
    }
    void sample(sr_ctx* ctx, MemTracker* tracker) { // context-wide totals: the context is shared by the operators of a fragment
        COUNTER_SET(launches, sr_ctx_kernel_launches(ctx));
        COUNTER_SET(device_bytes, sr_ctx_device_bytes(ctx));
        if (tracker) tracker->set(sr_ctx_device_bytes(ctx));
    }
};

// device (or host) sr_chunk_out -> host Chunks of <= chunk_size rows appended to `queue`
inline Status slice_out_to_chunks(sr_ctx* ctx, const sr_chunk_out& out, int chunk_size, std::deque<ChunkPtr>* queue) {
    const int64_t n = out.num_rows;
    if (n == 0) return Status::OK();
    std::vector<ColumnPtr> cols(out.num_cols);
    std::vector<std::shared_ptr<NullColumn>> nulls(out.num_cols);
    for (int k = 0; k < out.num_cols; k++) {
        const sr_col_out& c = out.cols[k];
        cols[k] = make_column(c.type, (size_t)n);
        const int64_t bytes = n * sr_type_width(c.type);
        if (out.mem == SR_MEM_DEVICE)
            RETURN_IF_SR_ERROR(ctx, sr_memcpy(ctx, cols[k]->mutable_raw_data(), c.data, bytes, 1));
        else
            memcpy(cols[k]->mutable_raw_data(), c.data, (size_t)bytes);
        if (c.nulls != nullptr) {
            nulls[k] = std::make_shared<NullColumn>(SR_TYPE_BOOLEAN);
            nulls[k]->resize((size_t)n);
            if (out.mem == SR_MEM_DEVICE)
                RETURN_IF_SR_ERROR(ctx, sr_memcpy(ctx, nulls[k]->mutable_raw_data(), c.nulls, n, 1));
            else
                memcpy(nulls[k]->mutable_raw_data(), c.nulls, (size_t)n);
        }
    }
    Chunk whole;
    for (int k = 0; k < out.num_cols; k++) {
        if (nulls[k])
            whole.append_column(std::make_shared<NullableColumn>(cols[k], nulls[k]), out.cols[k].slot_id);
        else
            whole.append_column(cols[k], out.cols[k].slot_id);
    }
    for (int64_t off = 0; off < n; off += chunk_size) queue->push_back(whole.slice((size_t)off, (size_t)std::min<int64_t>(chunk_size, n - off)));
    return Status::OK();
}

// ------------------------------------------------------------------------------------------------------------
// runtime filters: RuntimeFilterBuildDescriptor / RuntimeFilterProbeDescriptor / RuntimeFilterCollector
// (be/src/exec/runtime_filter/runtime_filter_descriptor.h, be/src/exec/pipeline/runtime_filter_types.h:60-138)
// ------------------------------------------------------------------------------------------------------------
struct GpuRuntimeFilterBuildDesc {
    int32_t filter_id;
    int32_t key_index; // build_expr_order: which join key the filter is built from
    bool with_bloom;   // false: min/max only
    bool insert_nulls; // null-safe equal join
};
struct GpuRuntimeFilterProbeDesc {
    int32_t filter_id;
    int32_t build_plan_node_id; // the join whose holder carries the filter
    int32_t probe_slot;         // probe_expr: a plain slot ref of the scan's chunk
};
class GpuRuntimeFilterCollector { // owns the device filters of one join
public:
    ~GpuRuntimeFilterCollector() {
        for (auto& kv : _filters) sr_rf_destroy(kv.second);
    }
    void add(int32_t filter_id, sr_rf* rf) { _filters[filter_id] = rf; }
    sr_rf* find(int32_t filter_id) const {
        auto it = _filters.find(filter_id);
        return it == _filters.end() ? nullptr : it->second;
    }

private:
    std::unordered_map<int32_t, sr_rf*> _filters;
};

constexpr int kGpuBatchChunks = 64; // ScanOperator::_buffer_size / io task batch (scan_operator.h:119)

// ------------------------------------------------------------------------------------------------------------
// scan
// ------------------------------------------------------------------------------------------------------------
// The IO side of the scan (reference: ScanOperator::_trigger_next_scan submits a ScanTask to the workgroup's ScanExecutor,
// the task runs ChunkSource::buffer_next_batch_chunks_blocking and fills the operator's BalancedChunkBuffer;
// scan_operator.cpp:328-515, chunk_source.cpp:60-120, exec/workgroup/scan_executor.h).  Here the "IO" of a task is one
// sr_scan_filter call over a batch of the morsel's chunks plus the D2H slicing of its output -- the part that takes time --
// so the pipeline driver that owns the operator never waits for the GPU: pull_chunk only triggers tasks and pops the buffer.
class GpuScanExecutor {
public:
    explicit GpuScanExecutor(int threads) {
        for (int t = 0; t < std::max(1, threads); t++) _workers.emplace_back([this] { _run(); });
    }
    ~GpuScanExecutor() {
        {
            std::lock_guard<std::mutex> l(_mu);
            _stop = true;
        }
        _cv.notify_all();
        for (auto& w : _workers) w.join();
    }
    void submit(std::function<void()> task) {
        {
            std::lock_guard<std::mutex> l(_mu);
            _tasks.push_back(std::move(task));
        }
        _cv.notify_one();
    }
    int64_t tasks_run() const { return _tasks_run.load(); }

private:
    void _run() {
        while (true) {
            std::function<void()> task;
            {
                std::unique_lock<std::mutex> l(_mu);
                _cv.wait(l, [this] { return _stop || !_tasks.empty(); });
                if (_tasks.empty()) return; // stop requested and drained
                task = std::move(_tasks.front());
                _tasks.pop_front();
            }
            task();
            _tasks_run.fetch_add(1);
        }
    }
    std::mutex _mu;
    std::condition_variable _cv;
    std::deque<std::function<void()>> _tasks;
    std::vector<std::thread> _workers;
    std::atomic<int64_t> _tasks_run{0};
    bool _stop = false;
};
using GpuScanExecutorPtr = std::shared_ptr<GpuScanExecutor>;

// the operator's chunk buffer (BalancedChunkBuffer, exec/pipeline/scan/balanced_chunk_buffer.h): filled by IO tasks, drained by
// pull_chunk; `limit` chunks bound what a scan may run ahead of its consumer (ScanOperator::_buffer_size)
class GpuChunkBuffer {
public:
    explicit GpuChunkBuffer(size_t limit) : _limit(limit) {}
    void put(std::deque<ChunkPtr>&& chunks) {
        std::lock_guard<std::mutex> l(_mu);
        for (auto& c : chunks) _q.push_back(std::move(c));
        _size.store(_q.size());
    }
    ChunkPtr try_get() {
        std::lock_guard<std::mutex> l(_mu);
        if (_q.empty()) return ChunkPtr(nullptr);
        ChunkPtr c = std::move(_q.front());
        _q.pop_front();
        _size.store(_q.size());
        return c;
    }
    bool empty() const { return _size.load() == 0; }
    bool has_room() const { return _size.load() < _limit; }

private:
    mutable std::mutex _mu;
    std::deque<ChunkPtr> _q;
    std::atomic<size_t> _size{0};
    size_t _limit;
};

class GpuScanOperator final : public SourceOperator {
public:
    // `morsel`: the decoded chunks the storage layer would hand over (TabletReader -> ChunkIterator::get_next); the
    // operator owns predicate evaluation + Chunk::filter on the device.  With an executor the scan is asynchronous (the
    // reference's shape); without one every pull_chunk runs its batch inline (kept for single-threaded tests).
    GpuScanOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, sr_ctx* ctx, const sr_scan_desc& desc,
                    std::vector<ChunkPtr> morsel, GpuScanExecutorPtr executor = nullptr)
            : SourceOperator(f, id, "gpu_olap_scan", plan_node_id, false, seq), _ctx(ctx), _desc(desc), _morsel(std::move(morsel)),
              _executor(std::move(executor)), _buffer(2 * kGpuBatchChunks) {
        // the names of ScanOperator / OlapChunkSource's profile (olap_chunk_source.cpp:93-140)
        _expr_filter_timer = ADD_TIMER(_unique_metrics.get(), "ExprFilterTime");
        _rows_read_counter = ADD_COUNTER(_unique_metrics.get(), "RawRowsRead", TUnit::UNIT);
        _rows_out_counter = ADD_COUNTER(_unique_metrics.get(), "RowsRead", TUnit::UNIT);
        _io_task_counter = ADD_COUNTER(_unique_metrics.get(), "SubmitTaskCount", TUnit::UNIT);           // scan_operator.cpp: _submit_task_counter
        _buffer_empty_counter = ADD_COUNTER(_unique_metrics.get(), "PullChunkBufferEmpty", TUnit::UNIT); // pulls that found the buffer empty
        _gpu.init(_unique_metrics.get());
    }
    ~GpuScanOperator() override {
        _wait_io();
        if (_scan) sr_scan_destroy(_scan);
    }
    Status prepare(RuntimeState* state) override {
        _chunk_size = state->chunk_size();
        _scan = sr_scan_create(_ctx, &_desc);
        return _scan ? Status::OK() : sr_to_status(_ctx, sr_last_error_code(_ctx));
    }
    // ScanOperator consumes the runtime filters of the joins above it (scan_operator.h:212-225); the driver keeps this
    // operator PRECONDITION_BLOCKed until the holders returned by rf_holders() are ready.
    void set_runtime_filters(RuntimeFilterHub* hub, std::vector<GpuRuntimeFilterProbeDesc> probes) {
        _hub = hub;
        _rf_probes = std::move(probes);
    }
    std::vector<RuntimeFilterHolder*> rf_holders() const {
        std::set<int32_t> ids;
        for (auto& p : _rf_probes) ids.insert(p.build_plan_node_id);
        return _hub ? _hub->gather_holders(ids) : std::vector<RuntimeFilterHolder*>();
    }
    int64_t rows_after_scan() const { return _rows_out.load(); }
    // ScanOperator::has_output (scan_operator.cpp:130-175): a buffered chunk, or an IO task could be submitted -- the
    // driver then calls pull_chunk, which submits it and returns nothing yet
    bool has_output() const override {
        if (!_buffer.empty() || _io_failed.load()) return true;
        return _running.load() == 0 && _next.load() < _morsel.size();
    }
    bool is_finished() const override { return _buffer.empty() && _running.load() == 0 && _next.load() >= _morsel.size() && !_io_failed.load(); }
    bool pending_finish() const override { return _running.load() > 0; } // ScanOperator::pending_finish: IO tasks still hold the operator
    Status set_finished(RuntimeState* state) override {
        _cancelled.store(true);
        return Status::OK();
    }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override {
        if (!_rf_attached) RETURN_IF_ERROR(_attach_runtime_filters());
        if (_io_failed.load()) {
            std::lock_guard<std::mutex> l(_status_mu);
            return _io_status;
        }
        if (_executor) {
            _try_to_trigger_next_scan();
        } else if (_buffer.empty() && _next.load() < _morsel.size()) {
            _io_task(); // synchronous form
        }
        ChunkPtr c = _buffer.try_get();
        if (!c) COUNTER_UPDATE(_buffer_empty_counter, 1);
        return c;
    }

private:
    // one IO task per operator at a time (its chunks stay in morsel order); DOP operators give DOP concurrent tasks
    void _try_to_trigger_next_scan() {
        if (_next.load() >= _morsel.size() || !_buffer.has_room() || _cancelled.load()) return;
        int expected = 0;
        if (!_running.compare_exchange_strong(expected, 1)) return;
        COUNTER_UPDATE(_io_task_counter, 1);
        _executor->submit([this] {
            _io_task();
            _running.store(0);
        });
    }
    // ChunkSource::buffer_next_batch_chunks_blocking: read a batch, filter it on the device, buffer the output chunks
    void _io_task() {
        size_t next = _next.load();
        ChunkBatch batch;
        for (int k = 0; k < kGpuBatchChunks && next < _morsel.size(); k++) batch.append(*_morsel[next++]);
        sr_chunk_view v = batch.view();
        sr_chunk_out out;
        Status st = Status::OK();
        std::deque<ChunkPtr> chunks;
        {
            SCOPED_TIMER(_expr_filter_timer);
            const int32_t rc = sr_scan_filter(_scan, &v, &out);
            if (rc != SR_OK) st = sr_to_status(_ctx, rc);
        }
        if (st.ok()) st = slice_out_to_chunks(_ctx, out, _chunk_size, &chunks);
        if (!st.ok()) {
            {
                std::lock_guard<std::mutex> l(_status_mu);
                _io_status = st;
            }
            _io_failed.store(true);
            _next.store(_morsel.size());
            return;
        }
        COUNTER_UPDATE(_rows_read_counter, (int64_t)batch.rows());
        COUNTER_UPDATE(_rows_out_counter, out.num_rows);
        _gpu.sample(_ctx, _mem_tracker.get());
        _rows_out.fetch_add(out.num_rows);
        _buffer.put(std::move(chunks));
        _next.store(next); // published after the chunks: is_finished() never sees "exhausted" with the last batch still on its way
    }
    void _wait_io() {
        _cancelled.store(true);
        while (_running.load() > 0) std::this_thread::yield();
    }
    Status _attach_runtime_filters() {
        _rf_attached = true;
        for (auto& p : _rf_probes) {
            RuntimeFilterHolder* h = _hub ? _hub->get_holder(p.build_plan_node_id) : nullptr;
            if (!h || !h->is_ready()) return Status::InternalError("runtime filter " + std::to_string(p.filter_id) + " is not ready");
            sr_rf* rf = static_cast<GpuRuntimeFilterCollector*>(h->get_collector())->find(p.filter_id);
            if (!rf) continue; // the build side chose not to produce it
            RETURN_IF_SR_ERROR(_ctx, sr_scan_add_runtime_filter(_scan, rf, p.probe_slot));
        }
        return Status::OK();
    }
    sr_ctx* _ctx;
    sr_scan_desc _desc;
    sr_scan* _scan = nullptr;
    RuntimeFilterHub* _hub = nullptr;
    std::vector<GpuRuntimeFilterProbeDesc> _rf_probes;
    bool _rf_attached = false;
    int _chunk_size = 4096;
    std::atomic<int64_t> _rows_out{0};
    RuntimeProfile::Counter *_expr_filter_timer, *_rows_read_counter, *_rows_out_counter, *_io_task_counter, *_buffer_empty_counter;
    GpuOpCounters _gpu;
    std::vector<ChunkPtr> _morsel;
    std::atomic<size_t> _next{0};
    GpuScanExecutorPtr _executor;
    GpuChunkBuffer _buffer;
    std::atomic<int> _running{0};
    std::atomic<bool> _io_failed{false}, _cancelled{false};
    std::mutex _status_mu;
    Status _io_status;
};

// ------------------------------------------------------------------------------------------------------------
// hash join
// ------------------------------------------------------------------------------------------------------------
class GpuHashJoiner { // HashJoiner: shared by the build operator and the probe operators
public:
    GpuHashJoiner(sr_ctx* ctx, const sr_join_desc& desc) : _ctx(ctx), _desc(desc) {}
    ~GpuHashJoiner() {
        if (_join) sr_join_destroy(_join);
    }
    Status prepare() {
        if (_join) return Status::OK();
        _join = sr_join_create(_ctx, &_desc);
        return _join ? Status::OK() : sr_to_status(_ctx, sr_last_error_code(_ctx));
    }
    sr_ctx* ctx() const { return _ctx; }
    sr_join* join() const { return _join; }
    bool is_build_done() const { return _join != nullptr && sr_join_is_build_done(_join) != 0; } // HashJoiner::is_build_done
    // POST_PROBE phase of RIGHT / FULL joins (HashJoiner::_phase, exec/hash_joiner.h:161-188): every prober registers, the
    // LAST one to finish its probe input emits the unmatched build rows (hash_join_probe_operator.cpp set_finishing ->
    // HashJoiner::enter_post_probe_phase, hash_joiner.cpp:315-327)
    bool has_post_probe() const {
        return _desc.join_type == SR_JOIN_RIGHT_OUTER || _desc.join_type == SR_JOIN_RIGHT_SEMI || _desc.join_type == SR_JOIN_RIGHT_ANTI ||
               _desc.join_type == SR_JOIN_FULL_OUTER;
    }
    void add_prober() { _active_probers.fetch_add(1); }
    bool prober_finished_is_last() { return _active_probers.fetch_sub(1) == 1; }

private:
    sr_ctx* _ctx;
    sr_join_desc _desc;
    sr_join* _join = nullptr;
    std::atomic<int> _active_probers{0};
};
using GpuHashJoinerPtr = std::shared_ptr<GpuHashJoiner>;

class GpuHashJoinBuildOperator final : public Operator {
public:
    GpuHashJoinBuildOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuHashJoinerPtr joiner)
            : Operator(f, id, "gpu_hash_join_build", plan_node_id, false, seq), _joiner(std::move(joiner)) {
        // HashJoiner's build metrics (be/src/exec/hash_joiner.h:161-188)
        _copy_right_table_timer = ADD_TIMER(_unique_metrics.get(), "CopyRightTableChunkTime");
        _build_ht_timer = ADD_TIMER(_unique_metrics.get(), "BuildHashTableTime");
        _rf_build_timer = ADD_TIMER(_unique_metrics.get(), "RuntimeFilterBuildTime");
        _build_rows_counter = ADD_COUNTER(_unique_metrics.get(), "HashTableBuildRows", TUnit::UNIT);
        _rf_num_counter = ADD_COUNTER(_unique_metrics.get(), "RuntimeFilterNum", TUnit::UNIT);
        _gpu.init(_unique_metrics.get());
    }
    Status prepare(RuntimeState* state) override { return _joiner->prepare(); }
    // what HashJoinNode hands the build operator factory: the filters to build and the hub that carries them
    void set_runtime_filters(RuntimeFilterHub* hub, std::vector<GpuRuntimeFilterBuildDesc> descs) {
        _hub = hub;
        _rf_descs = std::move(descs);
    }
    bool has_output() const override { return false; }
    bool need_input() const override { return !_finished; }
    bool is_finished() const override { return _finished; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("pull_chunk on a sink"); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override { // HashJoiner::append_chunk_to_ht
        _batch.append(*chunk);
        if (_batch.rows() >= (size_t)kGpuBatchChunks * state->chunk_size()) RETURN_IF_ERROR(_flush());
        return Status::OK();
    }
    Status set_finishing(RuntimeState* state) override { // build_ht + enter_probe_phase (hash_join_build_operator.cpp:86-220)
        if (_finished) return Status::OK();
        RETURN_IF_ERROR(_flush());
        {
            SCOPED_TIMER(_build_ht_timer);
            RETURN_IF_SR_ERROR(_joiner->ctx(), sr_join_build_finish(_joiner->join()));
        }
        sr_join_info info;
        if (sr_join_get_info(_joiner->join(), &info) == SR_OK) COUNTER_SET(_build_rows_counter, info.build_rows);
        if (_hub) {
            SCOPED_TIMER(_rf_build_timer); // create_runtime_filters + set_collector (hash_join_build_operator.cpp:100-215): publish even when empty
            auto collector = std::make_shared<GpuRuntimeFilterCollector>();
            for (auto& d : _rf_descs) {
                sr_rf* rf = sr_join_build_runtime_filter(_joiner->join(), d.key_index, d.with_bloom ? 1 : 0, d.insert_nulls ? 1 : 0);
                if (!rf) return sr_to_status(_joiner->ctx(), sr_last_error_code(_joiner->ctx()));
                collector->add(d.filter_id, rf);
                COUNTER_UPDATE(_rf_num_counter, 1);
            }
            _hub->set_collector(_plan_node_id, collector);
        }
        _gpu.sample(_joiner->ctx(), _mem_tracker.get());
        _finished = true;
        return Status::OK();
    }

private:
    Status _flush() {
        if (_batch.empty()) return Status::OK();
        sr_chunk_view v = _batch.view();
        SCOPED_TIMER(_copy_right_table_timer);
        RETURN_IF_SR_ERROR(_joiner->ctx(), sr_join_append_build(_joiner->join(), &v));
        _batch.clear();
        return Status::OK();
    }
    GpuHashJoinerPtr _joiner;
    ChunkBatch _batch;
    bool _finished = false;
    RuntimeProfile::Counter *_copy_right_table_timer, *_build_ht_timer, *_rf_build_timer, *_build_rows_counter, *_rf_num_counter;
    GpuOpCounters _gpu;
    RuntimeFilterHub* _hub = nullptr;
    std::vector<GpuRuntimeFilterBuildDesc> _rf_descs;
};

class GpuHashJoinProbeOperator final : public OperatorWithDependency {
public:
    GpuHashJoinProbeOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuHashJoinerPtr joiner)
            : OperatorWithDependency(f, id, "gpu_hash_join_probe", plan_node_id, false, seq), _joiner(std::move(joiner)), _prober_id(seq) {
        _joiner->add_prober();
        _search_ht_timer = ADD_TIMER(_unique_metrics.get(), "SearchHashTableTime"); // probe + both output gathers: one library call
        _output_timer = ADD_TIMER(_unique_metrics.get(), "OutputChunkTime");        // D2H + slicing into <= chunk_size chunks
        _probe_rows_counter = ADD_COUNTER(_unique_metrics.get(), "ProbeRows", TUnit::UNIT);
        _output_rows_counter = ADD_COUNTER(_unique_metrics.get(), "OutputRows", TUnit::UNIT);
        _gpu.init(_unique_metrics.get());
    }
    Status prepare(RuntimeState* state) override { return _joiner->prepare(); }
    bool is_ready() const override { return _joiner->is_build_done(); } // hash_join_probe_operator.cpp:75-77
    bool has_output() const override { return !_out.empty(); }
    bool need_input() const override { return _out.empty() && !_finishing; }
    bool is_finished() const override { return _finishing && _out.empty() && _batch.empty(); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        _batch.append(*chunk);
        if (_batch.rows() >= (size_t)kGpuBatchChunks * state->chunk_size()) RETURN_IF_ERROR(_probe(state));
        return Status::OK();
    }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override {
        if (_out.empty()) return ChunkPtr(nullptr);
        ChunkPtr c = _out.front();
        _out.pop_front();
        return c;
    }
    Status set_finishing(RuntimeState* state) override {
        if (_finishing) return Status::OK();
        _finishing = true;
        RETURN_IF_ERROR(_probe(state));
        if (_joiner->has_post_probe() && _joiner->prober_finished_is_last()) { // probe_remain (hash_joiner.cpp:315-327)
            sr_chunk_out out;
            RETURN_IF_SR_ERROR(_joiner->ctx(), sr_join_probe_remain(_joiner->join(), &out));
            COUNTER_UPDATE(_output_rows_counter, out.num_rows);
            SCOPED_TIMER(_output_timer);
            RETURN_IF_ERROR(slice_out_to_chunks(_joiner->ctx(), out, state->chunk_size(), &_out));
        }
        return Status::OK();
    }

private:
    Status _probe(RuntimeState* state) {
        if (_batch.empty()) return Status::OK();
        sr_chunk_view v = _batch.view();
        sr_chunk_out out;
        {
            SCOPED_TIMER(_search_ht_timer);
            RETURN_IF_SR_ERROR(_joiner->ctx(), sr_join_probe(_joiner->join(), _prober_id, &v, &out));
        }
        COUNTER_UPDATE(_probe_rows_counter, (int64_t)_batch.rows());
        COUNTER_UPDATE(_output_rows_counter, out.num_rows);
        {
            SCOPED_TIMER(_output_timer);
            RETURN_IF_ERROR(slice_out_to_chunks(_joiner->ctx(), out, state->chunk_size(), &_out));
        }
        _gpu.sample(_joiner->ctx(), _mem_tracker.get());
        _batch.clear();
        return Status::OK();
    }
    GpuHashJoinerPtr _joiner;
    RuntimeProfile::Counter *_search_ht_timer, *_output_timer, *_probe_rows_counter, *_output_rows_counter;
    GpuOpCounters _gpu;
    int32_t _prober_id;
    ChunkBatch _batch;
    std::deque<ChunkPtr> _out;
    bool _finishing = false;
};

// ------------------------------------------------------------------------------------------------------------
// aggregate
// ------------------------------------------------------------------------------------------------------------
class GpuAggregator { // Aggregator: shared by the blocking sink and source
public:
    GpuAggregator(sr_ctx* ctx, const sr_agg_desc& desc) : _ctx(ctx), _desc(desc) {}
    explicit GpuAggregator(sr_ctx* ctx, sr_agg* borrowed) : _ctx(ctx), _agg(borrowed), _owned(false) {}
    ~GpuAggregator() {
        if (_agg && _owned) sr_agg_destroy(_agg);
    }
    Status prepare() {
        if (_agg) return Status::OK();
        _agg = sr_agg_create(_ctx, &_desc);
        return _agg ? Status::OK() : sr_to_status(_ctx, sr_last_error_code(_ctx));
    }
    sr_ctx* ctx() const { return _ctx; }
    sr_agg* agg() const { return _agg; }
    void bind(sr_agg* borrowed) { // the fused fragment owns its aggregate and creates it once the builds are done
        _agg = borrowed;
        _owned = false;
    }
    bool is_sink_complete() const { return _sink_complete; }
    void sink_complete() { _sink_complete = true; }

private:
    sr_ctx* _ctx;
    sr_agg_desc _desc{};
    sr_agg* _agg = nullptr;
    bool _owned = true;
    bool _sink_complete = false;
};
using GpuAggregatorPtr = std::shared_ptr<GpuAggregator>;

class GpuAggregateBlockingSinkOperator final : public Operator {
public:
    GpuAggregateBlockingSinkOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuAggregatorPtr agg)
            : Operator(f, id, "gpu_aggregate_blocking_sink", plan_node_id, false, seq), _aggregator(std::move(agg)) {
        _agg_compute_timer = ADD_TIMER(_unique_metrics.get(), "AggComputeTime"); // aggregator.h: AggComputeTime
        _input_rows_counter = ADD_COUNTER(_unique_metrics.get(), "InputRowCount", TUnit::UNIT);
        _gpu.init(_unique_metrics.get());
    }
    Status prepare(RuntimeState* state) override { return _aggregator->prepare(); }
    bool has_output() const override { return false; }
    bool need_input() const override { return !_finished; }
    bool is_finished() const override { return _finished; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("pull_chunk on a sink"); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        _batch.append(*chunk);
        if (_batch.rows() >= (size_t)kGpuBatchChunks * state->chunk_size()) RETURN_IF_ERROR(_flush());
        return Status::OK();
    }
    Status set_finishing(RuntimeState* state) override { // sink_complete (aggregate_blocking_sink_operator.cpp:56-89)
        if (_finished) return Status::OK();
        RETURN_IF_ERROR(_flush());
        RETURN_IF_SR_ERROR(_aggregator->ctx(), sr_agg_sink_finish(_aggregator->agg()));
        _aggregator->sink_complete();
        _finished = true;
        return Status::OK();
    }

private:
    Status _flush() {
        if (_batch.empty()) return Status::OK();
        sr_chunk_view v = _batch.view();
        {
            SCOPED_TIMER(_agg_compute_timer);
            RETURN_IF_SR_ERROR(_aggregator->ctx(), sr_agg_push(_aggregator->agg(), &v));
        }
        COUNTER_UPDATE(_input_rows_counter, (int64_t)_batch.rows());
        _gpu.sample(_aggregator->ctx(), _mem_tracker.get());
        _batch.clear();
        return Status::OK();
    }
    GpuAggregatorPtr _aggregator;
    ChunkBatch _batch;
    bool _finished = false;
    RuntimeProfile::Counter *_agg_compute_timer, *_input_rows_counter;
    GpuOpCounters _gpu;
};

class GpuAggregateBlockingSourceOperator final : public SourceOperator {
public:
    GpuAggregateBlockingSourceOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuAggregatorPtr agg)
            : SourceOperator(f, id, "gpu_aggregate_blocking_source", plan_node_id, false, seq), _aggregator(std::move(agg)) {}
    bool has_output() const override { return _aggregator->is_sink_complete() && !_eos; }
    bool is_finished() const override { return _aggregator->is_sink_complete() && _eos; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override { // convert_hash_map_to_chunk, chunk_size groups per call
        sr_chunk_out out;
        RETURN_IF_SR_ERROR(_aggregator->ctx(), sr_agg_pull(_aggregator->agg(), state->chunk_size(), SR_MEM_HOST, &out));
        if (out.num_rows == 0) {
            _eos = true;
            return ChunkPtr(nullptr);
        }
        std::deque<ChunkPtr> q;
        RETURN_IF_ERROR(slice_out_to_chunks(_aggregator->ctx(), out, state->chunk_size(), &q));
        return q.front();
    }

private:
    GpuAggregatorPtr _aggregator;
    bool _eos = false;
};

// ------------------------------------------------------------------------------------------------------------
// streaming (first-phase) aggregate: AggregateStreamingSinkOperator / AggregateStreamingSourceOperator
// (be/src/exec/pipeline/aggregate/aggregate_streaming_{sink,source}_operator.cpp).  The sink pre-aggregates what it can
// and hands everything else on in the intermediate format; the source drains the chunk buffer and, once the sink is done,
// the hash table.  The aggregator must be created from the FIRST-PHASE desc of sr_agg_two_phase_descs.
//
// AUTO on a GPU works on batches of kGpuBatchChunks chunks, not on single chunks, so the reference's six-state machine
// (aggregate_streaming_sink_operator.cpp:211-355) is folded into three states driven by the same quantity, the reduction
// rows_fed / groups (Aggregator::should_expand_preagg_hash_tables, STREAMING_HT_MIN_REDUCTION = 2.0 above 2 MB):
//   PREAGG        push the batch into the table.  While the table is below max_ht_bytes, or the reduction since the last
//                 flush is >= 2, stay.  Otherwise flush the table downstream (its groups are emitted as intermediate rows,
//                 the table is reset) and go to PASS_THROUGH.
//   PASS_THROUGH  convert batches row by row (sr_agg_convert_to_states) for `pass_through_batches` batches
//                 (AggrAutoContext::StableLimit), then PROBE.
//   PROBE         pre-aggregate ONE batch into the empty table (the reference's FORCE_PREAGG: "freshening the hash table
//                 with new coming rows"): reduction >= 2 -> PREAGG, else flush and PASS_THROUGH again.
// Dense tables and aggregates without GROUP BY are bounded: always PREAGG.
// ------------------------------------------------------------------------------------------------------------
// TStreamingPreaggregationMode (+ LIMITED_MEM, aggregate_streaming_sink_operator.cpp:362-372: AUTO until the table holds
// limited_memory_size bytes, FORCE_STREAMING from then on)
enum class GpuStreamingPreaggMode { AUTO = 0, FORCE_STREAMING = 1, FORCE_PREAGGREGATION = 2, LIMITED_MEM = 3 };

class GpuStreamingAggregator {
public:
    GpuStreamingAggregator(sr_ctx* ctx, const sr_agg_desc& first_phase_desc, GpuStreamingPreaggMode mode, size_t max_ht_bytes = 64u << 20,
                           int pass_through_batches = 5)
            : _ctx(ctx), _desc(first_phase_desc), _mode(mode), _max_ht_bytes(max_ht_bytes), _pass_through_batches(pass_through_batches) {
        // bytes one group occupies: packed key + COUNT(*) word + one state word per function (+ null tracking)
        _group_bytes = 16 + 8 + 16 * (size_t)_desc.num_fns;
    }
    ~GpuStreamingAggregator() {
        if (_agg) sr_agg_destroy(_agg);
    }
    Status prepare() {
        if (_agg) return Status::OK();
        _agg = sr_agg_create(_ctx, &_desc);
        return _agg ? Status::OK() : sr_to_status(_ctx, sr_last_error_code(_ctx));
    }
    // one batch of input rows (host chunks concatenated by the sink)
    Status process_batch(RuntimeState* state, const sr_chunk_view& v) {
        const bool bounded = _desc.num_group_keys == 0 || _desc.has_ranges != 0;
        if (_mode == GpuStreamingPreaggMode::FORCE_STREAMING && !bounded) return _stream(state, v);
        if (_mode == GpuStreamingPreaggMode::FORCE_PREAGGREGATION || bounded) return _preagg(v);
        if (_mode == GpuStreamingPreaggMode::LIMITED_MEM) {
            // LimitedMemAggState::has_limited (aggregator.h:639-641): Aggregator::memory_usage() >= limited_memory_size.  The
            // table's memory does not shrink when its groups are flushed, so the peak size counts
            if (_limited || _peak_table_bytes >= _max_ht_bytes) {
                _limited = true;
                return _stream(state, v);
            }
        }
        switch (_state) {
        case SELECTIVE: // SELECTIVE_PREAGG for continuous_limit batches, then back to ADJUST (aggregate_streaming_sink_operator.cpp:225-228)
            RETURN_IF_ERROR(_selective(state, v));
            if (++_pass_count >= _pass_through_batches) {
                _pass_count = 0;
                _state = PROBE;
            }
            return Status::OK();
        case PASS_THROUGH:
            RETURN_IF_ERROR(_stream(state, v));
            if (++_pass_count >= _pass_through_batches) {
                _pass_count = 0;
                _state = PROBE;
            }
            return Status::OK();
        case PROBE:
        case PREAGG: {
            RETURN_IF_ERROR(_preagg(v));
            const int64_t groups = sr_agg_current_groups(_agg);
            if (groups < 0) return sr_to_status(_ctx, (int32_t)groups);
            const double reduction = groups > 0 ? (double)_rows_in_table / (double)groups : 1e30;
            const bool big = (size_t)groups * _group_bytes > _max_ht_bytes;
            _peak_table_bytes = std::max(_peak_table_bytes, (size_t)groups * _group_bytes);
            if (_state == PROBE) {
                if (reduction >= 2.0) {
                    _state = PREAGG;
                    return Status::OK();
                }
            } else if (!big || reduction >= 2.0) {
                return Status::OK(); // small table, or pre-aggregation still pays
            }
            if (reduction >= 1.25) {
                // middling reduction ("middle cases", :194-208): keep the table, aggregate the rows of known groups into it
                // and stream the rest, so it stops growing without losing the groups that do repeat
                _state = SELECTIVE;
                _num_selective_phases++;
                return Status::OK();
            }
            // low reduction: emit what the table holds and stop building it for a while
            RETURN_IF_ERROR(flush_table(state));
            _state = PASS_THROUGH;
            _num_flushes++;
            return Status::OK();
        }
        }
        return Status::OK();
    }
    // emit every group of the table as intermediate rows and clear it
    Status flush_table(RuntimeState* state) {
        RETURN_IF_SR_ERROR(_ctx, sr_agg_sink_finish(_agg));
        while (true) {
            sr_chunk_out out;
            RETURN_IF_SR_ERROR(_ctx, sr_agg_pull(_agg, (int64_t)kGpuBatchChunks * state->chunk_size(), SR_MEM_DEVICE, &out));
            if (out.num_rows == 0) break;
            _rows_from_table += (size_t)out.num_rows;
            RETURN_IF_ERROR(slice_out_to_chunks(_ctx, out, state->chunk_size(), &_buffer));
        }
        RETURN_IF_SR_ERROR(_ctx, sr_agg_reset(_agg));
        _rows_in_table = 0;
        return Status::OK();
    }
    std::deque<ChunkPtr>& buffer() { return _buffer; } // Aggregator::_buffer (offer_chunk_to_buffer / poll_chunk_buffer)
    void sink_complete() { _sink_complete = true; }
    bool is_sink_complete() const { return _sink_complete; }
    size_t rows_streamed() const { return _rows_streamed; }
    size_t rows_selected_into_table() const { return _rows_selected; }
    int num_selective_phases() const { return _num_selective_phases; }
    bool memory_limited() const { return _limited; }
    size_t rows_from_table() const { return _rows_from_table; }
    int num_flushes() const { return _num_flushes; }

private:
    Status _preagg(const sr_chunk_view& v) {
        RETURN_IF_SR_ERROR(_ctx, sr_agg_push(_agg, &v));
        _rows_in_table += (size_t)v.num_rows;
        return Status::OK();
    }
    Status _selective(RuntimeState* state, const sr_chunk_view& v) {
        sr_chunk_out out;
        RETURN_IF_SR_ERROR(_ctx, sr_agg_push_selective(_agg, &v, &out));
        _rows_streamed += (size_t)out.num_rows;
        _rows_selected += (size_t)(v.num_rows - out.num_rows);
        _rows_in_table += (size_t)(v.num_rows - out.num_rows);
        return slice_out_to_chunks(_ctx, out, state->chunk_size(), &_buffer);
    }
    Status _stream(RuntimeState* state, const sr_chunk_view& v) {
        sr_chunk_out out;
        RETURN_IF_SR_ERROR(_ctx, sr_agg_convert_to_states(_agg, &v, &out));
        _rows_streamed += (size_t)out.num_rows;
        return slice_out_to_chunks(_ctx, out, state->chunk_size(), &_buffer);
    }
    enum AutoState { PREAGG, PASS_THROUGH, PROBE, SELECTIVE };
    sr_ctx* _ctx;
    sr_agg_desc _desc;
    GpuStreamingPreaggMode _mode;
    size_t _max_ht_bytes, _group_bytes;
    int _pass_through_batches;
    sr_agg* _agg = nullptr;
    AutoState _state = PREAGG;
    int _pass_count = 0, _num_flushes = 0, _num_selective_phases = 0;
    size_t _rows_in_table = 0, _rows_streamed = 0, _rows_from_table = 0, _rows_selected = 0;
    bool _limited = false;
    size_t _peak_table_bytes = 0;
    std::deque<ChunkPtr> _buffer;
    bool _sink_complete = false;
};
using GpuStreamingAggregatorPtr = std::shared_ptr<GpuStreamingAggregator>;

class GpuAggregateStreamingSinkOperator final : public Operator {
public:
    GpuAggregateStreamingSinkOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuStreamingAggregatorPtr agg)
            : Operator(f, id, "gpu_aggregate_streaming_sink", plan_node_id, false, seq), _aggregator(std::move(agg)) {}
    Status prepare(RuntimeState* state) override { return _aggregator->prepare(); }
    bool has_output() const override { return false; }
    bool need_input() const override { return !_finished; }
    bool is_finished() const override { return _finished; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("pull_chunk on a sink"); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        _batch.append(*chunk);
        if (_batch.rows() >= (size_t)kGpuBatchChunks * state->chunk_size()) RETURN_IF_ERROR(_flush(state));
        return Status::OK();
    }
    Status set_finishing(RuntimeState* state) override { // aggregate_streaming_sink_operator.cpp:43-66
        if (_finished) return Status::OK();
        RETURN_IF_ERROR(_flush(state));
        RETURN_IF_ERROR(_aggregator->flush_table(state)); // the source outputs the hash table after the buffered chunks
        _aggregator->sink_complete();
        _finished = true;
        return Status::OK();
    }

private:
    Status _flush(RuntimeState* state) {
        if (_batch.empty()) return Status::OK();
        sr_chunk_view v = _batch.view();
        RETURN_IF_ERROR(_aggregator->process_batch(state, v));
        _batch.clear();
        return Status::OK();
    }
    GpuStreamingAggregatorPtr _aggregator;
    ChunkBatch _batch;
    bool _finished = false;
};

class GpuAggregateStreamingSourceOperator final : public SourceOperator {
public:
    GpuAggregateStreamingSourceOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuStreamingAggregatorPtr agg)
            : SourceOperator(f, id, "gpu_aggregate_streaming_source", plan_node_id, false, seq), _aggregator(std::move(agg)) {}
    bool has_output() const override { return !_aggregator->buffer().empty(); } // aggregate_streaming_source_operator.cpp:30-52
    bool is_finished() const override { return _aggregator->is_sink_complete() && _aggregator->buffer().empty(); }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override {
        auto& q = _aggregator->buffer();
        if (q.empty()) return ChunkPtr(nullptr);
        ChunkPtr c = q.front();
        q.pop_front();
        return c;
    }

private:
    GpuStreamingAggregatorPtr _aggregator;
};

// ------------------------------------------------------------------------------------------------------------
// fused fragment sink: [probe x N -> aggregate sink] collapsed behind one sink operator
// ------------------------------------------------------------------------------------------------------------
class GpuFragment {
public:
    GpuFragment(sr_ctx* ctx, sr_fragment_desc desc, std::vector<GpuHashJoinerPtr> joiners)
            : _ctx(ctx), _desc(desc), _joiners(std::move(joiners)), _aggregator(std::make_shared<GpuAggregator>(ctx, (sr_agg*)nullptr)) {}
    ~GpuFragment() {
        if (_frag) sr_fragment_destroy(_frag);
    }
    bool builds_done() const {
        for (auto& j : _joiners)
            if (!j->is_build_done()) return false;
        return true;
    }
    Status prepare() { // needs the builds: called lazily from the first push (of any of the sinks sharing the fragment)
        std::lock_guard<std::mutex> lk(_mu);
        if (_frag) return Status::OK();
        for (size_t k = 0; k < _joiners.size(); k++) _desc.joins[k].join = _joiners[k]->join();
        _frag = sr_fragment_create(_ctx, &_desc);
        if (!_frag) return sr_to_status(_ctx, sr_last_error_code(_ctx));
        _aggregator->bind(sr_fragment_agg(_frag));
        return Status::OK();
    }
    sr_ctx* ctx() const { return _ctx; }
    sr_fragment* frag() const { return _frag; }
    GpuAggregatorPtr aggregator() const { return _aggregator; }
    // the sinks of all pipeline drivers feed the one fragment; the aggregate is complete when the last of them finishes
    // (the reference counts the sink operators of a shared Aggregator the same way, aggregator.h ref / unref)
    void add_sink() { _open_sinks.fetch_add(1); }
    Status sink_finished() {
        if (_open_sinks.fetch_sub(1) != 1) return Status::OK();
        RETURN_IF_ERROR(prepare());
        RETURN_IF_SR_ERROR(_ctx, sr_agg_sink_finish(sr_fragment_agg(_frag)));
        _aggregator->sink_complete();
        return Status::OK();
    }

private:
    sr_ctx* _ctx;
    sr_fragment_desc _desc;
    std::vector<GpuHashJoinerPtr> _joiners;
    sr_fragment* _frag = nullptr;
    GpuAggregatorPtr _aggregator;
    std::mutex _mu;
    std::atomic<int> _open_sinks{0};
};
using GpuFragmentPtr = std::shared_ptr<GpuFragment>;

// The fused sink.  push_chunk never waits for the GPU.  A chunk whose buffers all lie in a registered page-locked pool
// (ForwardedChunkList::forwardable) is forwarded: its ChunkPtr joins the current slot's list and a full list goes to
// sr_fragment_push_chunks, which gathers it on the device.  Any other chunk is copied into one of two page-locked batches
// (PinnedChunkBatch) and a full batch goes to sr_fragment_push, which reads it IN PLACE over PCIe.  A slot holds one kind
// at a time: a chunk of the other kind hands the current slot over first.  After each push an event is recorded and the
// operator switches to the other slot.  need_input() turns false only while BOTH slots are in flight -- polled by the
// driver, no blocking call (operator.h:100-118) -- and pending_finish() keeps the driver from finishing until the queued
// work has drained.
class GpuFragmentSinkOperator final : public OperatorWithDependency {
public:
    GpuFragmentSinkOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, GpuFragmentPtr frag, size_t batch_rows = 1 << 22)
            : OperatorWithDependency(f, id, "gpu_fragment_sink", plan_node_id, false, seq), _frag(std::move(frag)), _batch_rows(batch_rows) {
        _append_timer = ADD_TIMER(_unique_metrics.get(), "AppendChunkTime");
        _push_timer = ADD_TIMER(_unique_metrics.get(), "FragmentPushTime"); // host time of the (asynchronous) library call
        _batches_counter = ADD_COUNTER(_unique_metrics.get(), "FragmentBatches", TUnit::UNIT);
        _bytes_counter = ADD_COUNTER(_unique_metrics.get(), "PinnedBatchBytes", TUnit::BYTES);
        _forwarded_chunks_counter = ADD_COUNTER(_unique_metrics.get(), "ForwardedChunks", TUnit::UNIT);
        _forwarded_rows_counter = ADD_COUNTER(_unique_metrics.get(), "ForwardedRows", TUnit::UNIT);
        _no_buffer_counter = ADD_COUNTER(_unique_metrics.get(), "NeedInputFalseBothBatchesInFlight", TUnit::UNIT);
        _gpu.init(_unique_metrics.get());
        _frag->add_sink();
    }
    bool is_ready() const override { return _frag->builds_done(); }
    bool has_output() const override { return false; }
    bool need_input() const override {
        if (_finished) return false;
        auto* self = const_cast<GpuFragmentSinkOperator*>(this);
        if (_rows(_cur) < _batch_rows && !self->_busy(_cur)) return true;
        const bool ok = !self->_busy(_cur ^ 1); // the current slot is full: the other one must be free to switch
        if (!ok) COUNTER_UPDATE(self->_no_buffer_counter, 1);
        return ok;
    }
    bool is_finished() const override { return _finished; }
    bool pending_finish() const override {
        auto* self = const_cast<GpuFragmentSinkOperator*>(this);
        return _finished && (self->_busy(0) || self->_busy(1));
    }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("pull_chunk on a sink"); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        RETURN_IF_ERROR(_frag->prepare());
        if (chunk->num_rows() == 0) return Status::OK();
        if (ForwardedChunkList::forwardable(_frag->ctx(), *chunk)) {
            if (_batch[_cur].rows() > 0 || _rows(_cur) >= _batch_rows) RETURN_IF_ERROR(_next_slot());
            RETURN_IF_ERROR(_fwd[_cur].add(_frag->ctx(), chunk));
            COUNTER_UPDATE(_forwarded_chunks_counter, 1);
            COUNTER_UPDATE(_forwarded_rows_counter, (int64_t)chunk->num_rows());
            return Status::OK();
        }
        for (size_t i = 0; i < chunk->num_columns(); i++)
            if (chunk->get_column_by_index(i)->is_nullable())
                return Status::NotSupported("PinnedChunkBatch: nullable column (slot " + std::to_string(chunk->slot_of_index(i)) + ") outside a registered pool");
        if (!_batch[0].initialised())
            for (auto& b : _batch) RETURN_IF_ERROR(b.init(_frag->ctx(), *chunk, _batch_rows));
        if (_fwd[_cur].rows() > 0) RETURN_IF_ERROR(_next_slot()); // a pending forward list goes first
        size_t from = 0;
        while (from < chunk->num_rows()) {
            if (_batch[_cur].room() == 0) RETURN_IF_ERROR(_next_slot());
            const size_t before = _batch[_cur].rows();
            {
                SCOPED_TIMER(_append_timer);
                _batch[_cur].append(*chunk, from);
            }
            from += _batch[_cur].rows() - before;
        }
        return Status::OK();
    }
    Status set_finishing(RuntimeState* state) override {
        if (_finished) return Status::OK();
        RETURN_IF_ERROR(_frag->prepare());
        if (_rows(_cur) > 0) RETURN_IF_ERROR(_submit());
        _finished = true;
        return _frag->sink_finished();
    }
    Status set_finished(RuntimeState* state) override { // every driver's sink has drained (pending_finish was false)
        _gpu.sample(_frag->ctx(), _mem_tracker.get());
        return Status::OK();
    }

private:
    size_t _rows(int k) const { return _batch[k].rows() + _fwd[k].rows(); }
    bool _busy(int k) { return _batch[k].busy() | _fwd[k].busy(); }
    Status _next_slot() { // hand the current slot over and make the other one current
        RETURN_IF_ERROR(_submit());
        if (_busy(_cur)) { // cannot happen under the driver's need_input() protocol
            _batch[_cur].wait();
            _fwd[_cur].wait();
        }
        return Status::OK();
    }
    Status _submit() { // hand the current slot over, continue with the other one
        {
            SCOPED_TIMER(_push_timer);
            if (_fwd[_cur].rows() > 0) {
                RETURN_IF_ERROR(_fwd[_cur].submit(_frag->frag()));
            } else {
                sr_chunk_view v = _batch[_cur].view();
                RETURN_IF_SR_ERROR(_frag->ctx(), sr_fragment_push(_frag->frag(), &v));
                COUNTER_UPDATE(_bytes_counter, (int64_t)_batch[_cur].bytes());
                RETURN_IF_ERROR(_batch[_cur].mark_submitted());
            }
        }
        COUNTER_UPDATE(_batches_counter, 1);
        _cur ^= 1;
        return Status::OK();
    }
    GpuFragmentPtr _frag;
    size_t _batch_rows;
    PinnedChunkBatch _batch[2];
    ForwardedChunkList _fwd[2];
    int _cur = 0;
    bool _finished = false;
    RuntimeProfile::Counter *_append_timer, *_push_timer, *_batches_counter, *_bytes_counter, *_forwarded_chunks_counter, *_forwarded_rows_counter,
            *_no_buffer_counter;
    GpuOpCounters _gpu;
};

// ------------------------------------------------------------------------------------------------------------
// ExchangeSinkOperator, HASH_PARTITIONED part (exchange_sink_operator.cpp:586-637 + Shuffler, shuffler.h:72-106):
// hash the partition columns (FNV + ReduceOp, or CRC32 + modulo for BUCKET_SHUFFLE), reorder the rows so that every
// channel's rows are contiguous and in input order, hand each channel's slice to its sender.  The transport itself
// (brpc to another BE, NCCL all-to-all between the GPUs of one box) is the caller's ChannelSender.
// ------------------------------------------------------------------------------------------------------------
class GpuExchangeSinkOperator final : public Operator {
public:
    // sender(channel, chunk): called once per non-empty channel and flushed batch, rows in input order
    using ChannelSender = std::function<Status(int32_t channel, const ChunkPtr& chunk)>;
    GpuExchangeSinkOperator(OperatorFactory* f, int32_t id, int32_t plan_node_id, int32_t seq, sr_ctx* ctx, const sr_part_desc& desc, ChannelSender sender,
                            size_t batch_rows = 1 << 22)
            : Operator(f, id, "gpu_exchange_sink", plan_node_id, false, seq), _ctx(ctx), _desc(desc), _sender(std::move(sender)), _batch_rows(batch_rows) {}
    ~GpuExchangeSinkOperator() override {
        if (_xchg) sr_xchg_destroy(_xchg);
    }
    Status prepare(RuntimeState* state) override {
        _xchg = sr_xchg_create(_ctx, &_desc);
        return _xchg ? Status::OK() : sr_to_status(_ctx, sr_last_error_code(_ctx));
    }
    bool has_output() const override { return false; }
    bool need_input() const override { return !_finished; }
    bool is_finished() const override { return _finished; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("pull_chunk on a sink"); }
    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        _batch.append(*chunk);
        if (_batch.rows() >= _batch_rows) RETURN_IF_ERROR(_flush());
        return Status::OK();
    }
    Status set_finishing(RuntimeState* state) override {
        if (_finished) return Status::OK();
        RETURN_IF_ERROR(_flush());
        _finished = true;
        return Status::OK();
    }
    int64_t rows_sent(int32_t channel) const { return _rows_sent[channel]; }

private:
    Status _flush() {
        if (_batch.empty()) return Status::OK();
        sr_chunk_view v = _batch.view();
        sr_chunk_out out;
        std::vector<int64_t> offs(_desc.num_channels + 1, 0);
        RETURN_IF_SR_ERROR(_ctx, sr_xchg_partition(_xchg, &v, &out, offs.data()));
        _rows_sent.resize(_desc.num_channels, 0);
        // the partitioned columns come back as device buffers: slice them per channel into host chunks
        std::deque<ChunkPtr> whole;
        RETURN_IF_ERROR(slice_out_to_chunks(_ctx, out, (int)std::max<int64_t>(out.num_rows, 1), &whole));
        if (!whole.empty()) {
            const ChunkPtr& all = whole.front();
            for (int32_t c = 0; c < _desc.num_channels; c++) {
                const int64_t lo = offs[c], hi = offs[c + 1];
                if (hi <= lo) continue;
                ChunkPtr part = all->slice((size_t)lo, (size_t)(hi - lo));
                _rows_sent[c] += hi - lo;
                RETURN_IF_ERROR(_sender(c, part));
            }
        }
        _batch.clear();
        return Status::OK();
    }
    sr_ctx* _ctx;
    sr_part_desc _desc;
    ChannelSender _sender;
    size_t _batch_rows;
    sr_xchg* _xchg = nullptr;
    ChunkBatch _batch;
    std::vector<int64_t> _rows_sent;
    bool _finished = false;
};

// ------------------------------------------------------------------------------------------------------------
// factories (what HashJoinNode / AggregateBlockingNode::_decompose_to_pipeline<...> are instantiated with)
// ------------------------------------------------------------------------------------------------------------
class GpuScanOperatorFactory final : public SourceOperatorFactory {
public:
    // `io_threads` > 0: the scan operators share a ScanExecutor of that many IO threads (the asynchronous form); 0: every
    // pull_chunk filters its batch inline
    GpuScanOperatorFactory(int32_t id, int32_t plan_node_id, sr_ctx* ctx, sr_scan_desc desc, std::vector<std::vector<ChunkPtr>> morsels,
                           int io_threads = 2)
            : SourceOperatorFactory(id, "gpu_olap_scan", plan_node_id), _ctx(ctx), _desc(desc), _morsels(std::move(morsels)),
              _executor(io_threads > 0 ? std::make_shared<GpuScanExecutor>(io_threads) : nullptr) {
        set_degree_of_parallelism(_morsels.size());
    }
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuScanOperator>(this, _id, _plan_node_id, seq, _ctx, _desc, _morsels[seq], _executor);
    }
    GpuScanExecutorPtr executor() const { return _executor; }

private:
    sr_ctx* _ctx;
    sr_scan_desc _desc;
    std::vector<std::vector<ChunkPtr>> _morsels;
    GpuScanExecutorPtr _executor;
};

class GpuHashJoinerFactory { // HashJoinerFactory (hashjoin/hash_joiner_factory.cpp:57-79): prober i uses builder i % builder_dop
public:
    GpuHashJoinerFactory(sr_ctx* ctx, sr_join_desc desc) : _joiner(std::make_shared<GpuHashJoiner>(ctx, desc)) {}
    GpuHashJoinerPtr create_builder(int32_t, int32_t) { return _joiner; }
    GpuHashJoinerPtr create_prober(int32_t, int32_t) { return _joiner; }
    GpuHashJoinerPtr get() { return _joiner; }

private:
    GpuHashJoinerPtr _joiner;
};
using GpuHashJoinerFactoryPtr = std::shared_ptr<GpuHashJoinerFactory>;

class GpuHashJoinBuildOperatorFactory final : public OperatorFactory {
public:
    GpuHashJoinBuildOperatorFactory(int32_t id, int32_t plan_node_id, GpuHashJoinerFactoryPtr f)
            : OperatorFactory(id, "gpu_hash_join_build", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuHashJoinBuildOperator>(this, _id, _plan_node_id, seq, _f->create_builder(dop, seq));
    }

private:
    GpuHashJoinerFactoryPtr _f;
};

class GpuHashJoinProbeOperatorFactory final : public OperatorFactory {
public:
    GpuHashJoinProbeOperatorFactory(int32_t id, int32_t plan_node_id, GpuHashJoinerFactoryPtr f)
            : OperatorFactory(id, "gpu_hash_join_probe", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuHashJoinProbeOperator>(this, _id, _plan_node_id, seq, _f->create_prober(dop, seq));
    }

private:
    GpuHashJoinerFactoryPtr _f;
};

class GpuAggregatorFactory {
public:
    GpuAggregatorFactory(sr_ctx* ctx, sr_agg_desc desc) : _agg(std::make_shared<GpuAggregator>(ctx, desc)) {}
    GpuAggregatorPtr get_or_create(size_t) { return _agg; }

private:
    GpuAggregatorPtr _agg;
};
using GpuAggregatorFactoryPtr = std::shared_ptr<GpuAggregatorFactory>;

class GpuAggregateBlockingSinkOperatorFactory final : public OperatorFactory {
public:
    GpuAggregateBlockingSinkOperatorFactory(int32_t id, int32_t plan_node_id, GpuAggregatorFactoryPtr f)
            : OperatorFactory(id, "gpu_aggregate_blocking_sink", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuAggregateBlockingSinkOperator>(this, _id, _plan_node_id, seq, _f->get_or_create(seq));
    }

private:
    GpuAggregatorFactoryPtr _f;
};

class GpuAggregateBlockingSourceOperatorFactory final : public SourceOperatorFactory {
public:
    GpuAggregateBlockingSourceOperatorFactory(int32_t id, int32_t plan_node_id, GpuAggregatorFactoryPtr f)
            : SourceOperatorFactory(id, "gpu_aggregate_blocking_source", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuAggregateBlockingSourceOperator>(this, _id, _plan_node_id, seq, _f->get_or_create(seq));
    }

private:
    GpuAggregatorFactoryPtr _f;
};

// AggregateStreamingNode::decompose_to_pipeline (be/src/exec/aggregate/aggregate_streaming_node.cpp:39-50): one aggregator
// factory shared by the sink operator factory (end of the upstream pipeline) and the source operator factory (head of the
// downstream one); one aggregator per driver sequence
class GpuStreamingAggregatorFactory {
public:
    GpuStreamingAggregatorFactory(sr_ctx* ctx, sr_agg_desc first_phase_desc, GpuStreamingPreaggMode mode, size_t max_ht_bytes = 64u << 20,
                                  int pass_through_batches = 5)
            : _ctx(ctx), _desc(first_phase_desc), _mode(mode), _max_ht_bytes(max_ht_bytes), _pass_through_batches(pass_through_batches) {}
    GpuStreamingAggregatorPtr get_or_create(size_t seq) {
        if (_aggs.size() <= seq) _aggs.resize(seq + 1);
        if (!_aggs[seq]) _aggs[seq] = std::make_shared<GpuStreamingAggregator>(_ctx, _desc, _mode, _max_ht_bytes, _pass_through_batches);
        return _aggs[seq];
    }

private:
    sr_ctx* _ctx;
    sr_agg_desc _desc;
    GpuStreamingPreaggMode _mode;
    size_t _max_ht_bytes;
    int _pass_through_batches;
    std::vector<GpuStreamingAggregatorPtr> _aggs;
};
using GpuStreamingAggregatorFactoryPtr = std::shared_ptr<GpuStreamingAggregatorFactory>;

class GpuAggregateStreamingSinkOperatorFactory final : public OperatorFactory {
public:
    GpuAggregateStreamingSinkOperatorFactory(int32_t id, int32_t plan_node_id, GpuStreamingAggregatorFactoryPtr f)
            : OperatorFactory(id, "gpu_aggregate_streaming_sink", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuAggregateStreamingSinkOperator>(this, _id, _plan_node_id, seq, _f->get_or_create(seq));
    }

private:
    GpuStreamingAggregatorFactoryPtr _f;
};

class GpuAggregateStreamingSourceOperatorFactory final : public SourceOperatorFactory {
public:
    GpuAggregateStreamingSourceOperatorFactory(int32_t id, int32_t plan_node_id, GpuStreamingAggregatorFactoryPtr f)
            : SourceOperatorFactory(id, "gpu_aggregate_streaming_source", plan_node_id), _f(std::move(f)) {}
    OperatorPtr create(int32_t dop, int32_t seq) override {
        return std::make_shared<GpuAggregateStreamingSourceOperator>(this, _id, _plan_node_id, seq, _f->get_or_create(seq));
    }

private:
    GpuStreamingAggregatorFactoryPtr _f;
};

} // namespace starrocks::pipeline
