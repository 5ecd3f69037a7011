// End-to-end throughput of the C++ OPERATOR path (what a BE pipeline would run), SSB Q4.1 shape:
//
//   build pipelines (x4):   GpuScanOperator(dimension, predicate) -> GpuHashJoinBuildOperator
//   probe pipelines (x DOP): MemoryChunkSource (4096-row chunks of one lineorder shard) -> GpuFragmentSinkOperator
//   result pipeline:        GpuAggregateBlockingSourceOperator -> collect
//
// DOP pipeline drivers run on DOP host threads, like the BE's pipeline executors: each pulls <= chunk_size-row chunks from
// its source and pushes them into its sink; the sinks of all drivers feed ONE GpuFragment (one aggregate), copy the
// chunks into page-locked batches and hand full batches to sr_fragment_push without ever waiting for the GPU
// (need_input / pending_finish are polled).  The timed region starts when the probe drivers start and ends when the
// result rows are on the host: it contains the chunk copies, every byte crossing PCIe and the result D2H.
// Prints one JSON line; exit code 0 only if the groups equal a row-at-a-time evaluation done while generating the data.
//
//   operator_e2e_bench [rows=600000000] [dop=0 (hardware threads, capped at 32)] [batch_rows=4194304] [--pool pageable|pinned]
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <thread>

#include "../gpu/gpu_operators.h"

using namespace starrocks;
using namespace starrocks::pipeline;

namespace {

enum Slots { LO_ORDERDATE = 0, LO_CUSTKEY, LO_SUPPKEY, LO_PARTKEY, LO_REVENUE, LO_SUPPLYCOST, C_CUSTKEY = 10, C_REGION, C_NATION, S_SUPPKEY = 20, S_REGION,
             P_PARTKEY = 30, P_MFGR, D_DATEKEY = 40, D_YEAR, OUT_REV = 50, OUT_COST };

struct Rng {
    uint64_t s;
    uint32_t next(uint32_t lo, uint32_t hi) { // [lo, hi)
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        return lo + (uint32_t)((s >> 33) % (hi - lo));
    }
};

ChunkPtr make_chunk(const std::vector<std::pair<SlotId, std::vector<int32_t>>>& cols) {
    auto c = std::make_shared<Chunk>();
    for (auto& [slot, v] : cols) c->append_column(std::make_shared<Int32Column>(SR_TYPE_INT, v), slot);
    return c;
}
std::vector<ChunkPtr> split(const ChunkPtr& whole, size_t chunk_size) {
    std::vector<ChunkPtr> out;
    for (size_t off = 0; off < whole->num_rows(); off += chunk_size) out.push_back(whole->slice(off, std::min(chunk_size, whole->num_rows() - off)));
    return out;
}

// the scan side of a probe pipeline: one shard of lineorder in plain host arrays (the storage layer's decoded pages);
// pull_chunk materialises the next <= chunk_size rows as a Chunk of six Int32Columns (one copy: what page decoding writes):
// into pageable vectors by default, or into BorrowedColumns sliced from a registered PinnedArena (--pool pinned: the
// columns of a scan over a pinned ColumnAllocator pool, which the fused sink forwards without a host copy)
class MemoryChunkSource final : public SourceOperator {
public:
    MemoryChunkSource(int32_t seq, const std::vector<int32_t>* cols, size_t rows, std::shared_ptr<PinnedArena> arena)
            : SourceOperator(nullptr, 3, "memory_chunk_source", 3, false, seq), _cols(cols), _rows(rows), _arena(std::move(arena)) {}
    bool has_output() const override { return _next < _rows; }
    bool is_finished() const override { return _next >= _rows; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override {
        const size_t n = std::min<size_t>((size_t)state->chunk_size(), _rows - _next);
        auto c = std::make_shared<Chunk>();
        for (int k = 0; k < 6; k++) {
            if (_arena) {
                auto col = _arena->column(SR_TYPE_INT, n);
                if (!col) return Status::InternalError("pinned arena full");
                memcpy(col->mutable_raw_data(), _cols[k].data() + _next, n * sizeof(int32_t));
                c->append_column(col, (SlotId)k);
                continue;
            }
            auto col = std::make_shared<Int32Column>(SR_TYPE_INT);
            col->get_data().assign(_cols[k].begin() + (long)_next, _cols[k].begin() + (long)(_next + n));
            c->append_column(col, (SlotId)k);
        }
        _next += n;
        return c;
    }

private:
    const std::vector<int32_t>* _cols;
    size_t _rows, _next = 0;
    std::shared_ptr<PinnedArena> _arena;
};

class ResultSink final : public Operator {
public:
    ResultSink() : Operator(nullptr, 99, "result_sink", 99, false, 0) {}
    bool has_output() const override { return false; }
    bool need_input() const override { return !_finished; }
    bool is_finished() const override { return _finished; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState*) override { return Status::InternalError("sink"); }
    Status push_chunk(RuntimeState*, const ChunkPtr& c) override {
        chunks.push_back(c);
        return Status::OK();
    }
    Status set_finishing(RuntimeState*) override {
        _finished = true;
        return Status::OK();
    }
    std::vector<ChunkPtr> chunks;

private:
    bool _finished = false;
};

#define CHECK_OK(expr)                                                          \
    do {                                                                        \
        Status _st = (expr);                                                    \
        if (!_st.ok()) {                                                        \
            fprintf(stderr, "FAILED %s: %s\n", #expr, _st.to_string().c_str()); \
            exit(2);                                                            \
        }                                                                       \
    } while (0)

bool run_to_finish(PipelineDriver& d, RuntimeState* state, const char* name) {
    for (;;) {
        auto st = d.process(state);
        if (!st.ok()) {
            fprintf(stderr, "driver %s failed: %s\n", name, st.status().to_string().c_str());
            return false;
        }
        if (st.value() == PipelineDriver::FINISH) return true;
        if (st.value() == PipelineDriver::PRECONDITION_BLOCK) {
            fprintf(stderr, "driver %s is blocked on its dependency\n", name);
            return false;
        }
        std::this_thread::yield(); // READY without progress / PENDING_FINISH: the real driver parks in the poller
    }
}

sr_expr col_expr(int32_t slot) {
    sr_expr e{};
    e.nodes[0].op = SR_EX_COL;
    e.nodes[0].slot_id = slot;
    e.num_nodes = 1;
    return e;
}
using Groups = std::map<std::pair<int32_t, int32_t>, std::pair<int64_t, int64_t>>;

} // namespace

int main(int argc, char** argv) {
    std::vector<const char*> pos;
    bool pinned_pool = false;
    for (int a = 1; a < argc; a++) {
        if (std::string(argv[a]) == "--pool" && a + 1 < argc) {
            pinned_pool = std::string(argv[++a]) == "pinned";
            continue;
        }
        pos.push_back(argv[a]);
    }
    const size_t n_fact = pos.size() > 0 ? (size_t)atoll(pos[0]) : 600000000ull;
    int dop = pos.size() > 1 ? atoi(pos[1]) : 0;
    const size_t batch_rows = pos.size() > 2 ? (size_t)atoll(pos[2]) : (size_t)1 << 22;
    if (dop <= 0) dop = (int)std::min(32u, std::max(1u, std::thread::hardware_concurrency()));
    const int n_cust = 3000000, n_supp = 200000, n_part = 1400000, n_dates = 2556; // SSB SF100 dimensions
    sr_ctx* ctx = sr_ctx_create(0, nullptr);
    if (!ctx) {
        fprintf(stderr, "sr_ctx_create failed: %s\n", sr_last_error(nullptr));
        return 3;
    }
    RuntimeState state(4096);
    Rng rng{20240921};
    std::vector<int32_t> c_key(n_cust), c_region(n_cust), c_nation(n_cust), s_key(n_supp), s_region(n_supp), p_key(n_part), p_mfgr(n_part), d_key(n_dates), d_year(n_dates);
    for (int i = 0; i < n_cust; i++) {
        c_key[i] = i + 1;
        c_region[i] = rng.next(0, 5);
        c_nation[i] = c_region[i] * 5 + rng.next(0, 5);
    }
    for (int i = 0; i < n_supp; i++) {
        s_key[i] = i + 1;
        s_region[i] = rng.next(0, 5);
    }
    for (int i = 0; i < n_part; i++) {
        p_key[i] = i + 1;
        p_mfgr[i] = rng.next(0, 5);
    }
    for (int i = 0; i < n_dates; i++) {
        d_year[i] = 1992 + i / 366;
        d_key[i] = d_year[i] * 10000 + (i % 366) + 101;
    }
    // ---- lineorder shards + the expected groups, generated in parallel ----
    std::vector<std::vector<int32_t>> shard_cols((size_t)dop * 6);
    std::vector<size_t> shard_rows((size_t)dop);
    std::vector<Groups> expect_part((size_t)dop);
    {
        std::vector<std::thread> th;
        for (int t = 0; t < dop; t++)
            th.emplace_back([&, t]() {
                const size_t lo = n_fact * (size_t)t / (size_t)dop, hi = n_fact * (size_t)(t + 1) / (size_t)dop, n = hi - lo;
                shard_rows[(size_t)t] = n;
                std::vector<int32_t>* c = &shard_cols[(size_t)t * 6];
                for (int k = 0; k < 6; k++) c[k].resize(n);
                Rng r{0x9E3779B97F4A7C15ull * (uint64_t)(t + 1)};
                Groups& g = expect_part[(size_t)t];
                for (size_t i = 0; i < n; i++) {
                    const int32_t d = d_key[r.next(0, n_dates)], cu = (int32_t)r.next(1, n_cust + 1), su = (int32_t)r.next(1, n_supp + 1), pa = (int32_t)r.next(1, n_part + 1);
                    const int32_t rev = (int32_t)r.next(81000, 10400001), cost = (int32_t)r.next(54000, 125001);
                    c[0][i] = d, c[1][i] = cu, c[2][i] = su, c[3][i] = pa, c[4][i] = rev, c[5][i] = cost;
                    if (s_region[su - 1] != 1 || c_region[cu - 1] != 1 || p_mfgr[pa - 1] > 1) continue;
                    auto& e = g[{d / 10000, c_nation[cu - 1]}];
                    e.first += rev;
                    e.second += cost;
                }
            });
        for (auto& x : th) x.join();
    }
    Groups expect;
    for (auto& g : expect_part)
        for (auto& kv : g) {
            expect[kv.first].first += kv.second.first;
            expect[kv.first].second += kv.second.second;
        }
    // ---- build side through the operators ----
    auto eq_pred = [](int32_t slot, int64_t v) {
        sr_pred p{};
        p.slot_id = slot;
        p.op = SR_PRED_EQ;
        p.ilo = v;
        return p;
    };
    sr_pred supp_pred = eq_pred(S_REGION, 1), cust_pred = eq_pred(C_REGION, 1), part_pred{};
    part_pred.slot_id = P_MFGR;
    part_pred.op = SR_PRED_IN;
    part_pred.in_list[0] = 0;
    part_pred.in_list[1] = 1;
    part_pred.in_count = 2;
    struct Dim {
        const char* name;
        ChunkPtr table;
        sr_pred* pred;
        int32_t key_slot, probe_slot;
        std::vector<int32_t> payload;
    };
    std::vector<Dim> dims = {
            {"supplier", make_chunk({{S_SUPPKEY, s_key}, {S_REGION, s_region}}), &supp_pred, S_SUPPKEY, LO_SUPPKEY, {}},
            {"customer", make_chunk({{C_CUSTKEY, c_key}, {C_REGION, c_region}, {C_NATION, c_nation}}), &cust_pred, C_CUSTKEY, LO_CUSTKEY, {C_NATION}},
            {"part", make_chunk({{P_PARTKEY, p_key}, {P_MFGR, p_mfgr}}), &part_pred, P_PARTKEY, LO_PARTKEY, {}},
            {"dates", make_chunk({{D_DATEKEY, d_key}, {D_YEAR, d_year}}), nullptr, D_DATEKEY, LO_ORDERDATE, {D_YEAR}},
    };
    const auto tb0 = std::chrono::steady_clock::now();
    std::vector<GpuHashJoinerFactoryPtr> joiner_factories;
    std::vector<std::vector<int32_t>> out_slot_store(dims.size());
    for (size_t k = 0; k < dims.size(); k++) {
        Dim& dm = dims[k];
        out_slot_store[k] = {dm.key_slot};
        for (int32_t p : dm.payload) out_slot_store[k].push_back(p);
        sr_scan_desc sd{};
        sd.preds = dm.pred;
        sd.num_preds = dm.pred ? 1 : 0;
        sd.out_slots = out_slot_store[k].data();
        sd.num_out_slots = (int32_t)out_slot_store[k].size();
        sr_join_desc jd{};
        jd.join_type = SR_JOIN_INNER;
        jd.num_keys = 1;
        jd.build_key_slots[0] = dm.key_slot;
        jd.probe_key_slots[0] = dm.probe_slot;
        jd.key_types[0] = SR_TYPE_INT;
        jd.enable_range_direct_mapping = 1;
        jd.num_build_out = (int32_t)dm.payload.size();
        for (size_t p = 0; p < dm.payload.size(); p++) {
            jd.build_out_slots[p] = dm.payload[p];
            jd.build_out_types[p] = SR_TYPE_INT;
        }
        auto jf = std::make_shared<GpuHashJoinerFactory>(ctx, jd);
        joiner_factories.push_back(jf);
        GpuScanOperatorFactory scan_f(1, 1, ctx, sd, {split(dm.table, 4096)});
        GpuHashJoinBuildOperatorFactory build_f(2, 20 + (int)k, jf);
        PipelineDriver build_driver({scan_f.create(1, 0), build_f.create(1, 0)});
        CHECK_OK(build_driver.prepare(&state));
        if (!run_to_finish(build_driver, &state, dm.name)) return 2;
        build_driver.close(&state);
    }
    const double build_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - tb0).count();
    // ---- the fused fragment shared by the DOP sinks ----
    sr_agg_desc agg_desc{};
    agg_desc.num_group_keys = 2;
    agg_desc.group_slots[0] = D_YEAR;
    agg_desc.group_slots[1] = C_NATION;
    agg_desc.group_types[0] = agg_desc.group_types[1] = SR_TYPE_INT;
    agg_desc.has_ranges = 1;
    agg_desc.group_min[0] = 1992;
    agg_desc.group_max[0] = 1998;
    agg_desc.group_min[1] = 0;
    agg_desc.group_max[1] = 24;
    agg_desc.num_fns = 2;
    agg_desc.fns[0] = sr_agg_fn{SR_AGG_SUM, SR_TYPE_INT, OUT_REV, 0, col_expr(LO_REVENUE)};
    agg_desc.fns[1] = sr_agg_fn{SR_AGG_SUM, SR_TYPE_INT, OUT_COST, 0, col_expr(LO_SUPPLYCOST)};
    sr_fragment_desc fd{};
    fd.num_joins = (int32_t)dims.size();
    std::vector<GpuHashJoinerPtr> joiners;
    for (size_t k = 0; k < dims.size(); k++) {
        fd.joins[k].probe_key_slot = dims[k].probe_slot;
        fd.joins[k].num_payload = (int32_t)dims[k].payload.size();
        for (size_t p = 0; p < dims[k].payload.size(); p++) fd.joins[k].payload_build_slots[p] = dims[k].payload[p];
        joiners.push_back(joiner_factories[k]->get());
    }
    fd.agg = agg_desc;
    auto fragment = std::make_shared<GpuFragment>(ctx, fd, joiners);
    std::vector<std::shared_ptr<GpuFragmentSinkOperator>> sinks;
    std::vector<std::unique_ptr<PipelineDriver>> drivers;
    for (int t = 0; t < dop; t++) {
        std::shared_ptr<PinnedArena> arena;
        if (pinned_pool) { // one registered arena per shard, sized for its chunks (outside the timed region)
            std::string err;
            const size_t chunks = shard_rows[(size_t)t] / 4096 + 1;
            arena = PinnedArena::create(ctx, shard_rows[(size_t)t] * 6 * sizeof(int32_t) + chunks * 6 * PinnedArena::ALIGN, &err);
            if (!arena) {
                fprintf(stderr, "%s\n", err.c_str());
                return 2;
            }
        }
        auto src = std::make_shared<MemoryChunkSource>(t, &shard_cols[(size_t)t * 6], shard_rows[(size_t)t], arena);
        auto sink = std::make_shared<GpuFragmentSinkOperator>(nullptr, 8, 8, t, fragment, batch_rows);
        sinks.push_back(sink);
        drivers.push_back(std::make_unique<PipelineDriver>(Operators{src, sink}));
        CHECK_OK(drivers.back()->prepare(&state));
    }
    // ---- timed: DOP probe drivers, then the result pipeline ----
    const int64_t launches0 = sr_ctx_kernel_launches(ctx);
    std::atomic<int> failed{0};
    const auto t0 = std::chrono::steady_clock::now();
    {
        std::vector<std::thread> th;
        for (int t = 0; t < dop; t++)
            th.emplace_back([&, t]() {
                RuntimeState st(4096);
                if (!run_to_finish(*drivers[(size_t)t], &st, "probe(fused)")) failed.fetch_add(1);
            });
        for (auto& x : th) x.join();
    }
    if (failed.load()) return 2;
    const auto t1 = std::chrono::steady_clock::now();
    auto rsink = std::make_shared<ResultSink>();
    auto rsource = std::make_shared<GpuAggregateBlockingSourceOperator>(nullptr, 9, 9, 0, fragment->aggregator());
    PipelineDriver result_driver({rsource, rsink});
    CHECK_OK(result_driver.prepare(&state));
    if (!run_to_finish(result_driver, &state, "result")) return 2;
    const auto t2 = std::chrono::steady_clock::now();
    const double probe_s = std::chrono::duration<double>(t1 - t0).count(), total_s = std::chrono::duration<double>(t2 - t0).count();
    Groups got;
    int64_t d2h = 0;
    for (auto& c : rsink->chunks) {
        auto* y = (const int32_t*)c->get_column_by_slot_id(D_YEAR)->raw_data();
        auto* n = (const int32_t*)c->get_column_by_slot_id(C_NATION)->raw_data();
        auto* r = (const int64_t*)c->get_column_by_slot_id(OUT_REV)->raw_data();
        auto* s = (const int64_t*)c->get_column_by_slot_id(OUT_COST)->raw_data();
        for (size_t i = 0; i < c->num_rows(); i++) got[{y[i], n[i]}] = {r[i], s[i]};
        d2h += (int64_t)c->num_rows() * 24;
    }
    const bool ok = got == expect;
    int64_t batches = 0, bytes = 0, append_ns = 0, push_ns = 0, stalls = 0, fwd_chunks = 0, fwd_rows = 0;
    for (auto& s : sinks) {
        fwd_chunks += s->unique_metrics()->get_counter("ForwardedChunks")->value();
        fwd_rows += s->unique_metrics()->get_counter("ForwardedRows")->value();
        batches += s->unique_metrics()->get_counter("FragmentBatches")->value();
        bytes += s->unique_metrics()->get_counter("PinnedBatchBytes")->value();
        append_ns += s->unique_metrics()->get_counter("AppendChunkTime")->value();
        push_ns += s->unique_metrics()->get_counter("FragmentPushTime")->value();
        stalls += s->unique_metrics()->get_counter("NeedInputFalseBothBatchesInFlight")->value();
    }
    const std::string path = pinned_pool ? "4096-row chunks in registered pinned arenas forwarded in lists of " + std::to_string(batch_rows) +
                                                   " rows to sr_fragment_push_chunks (gathered on the device)"
                                         : "4096-row chunks, pinned double-buffered batches of " + std::to_string(batch_rows) + " rows read in place by the fragment kernels";
    printf("{\"path\": \"C++ operators: %d x (MemoryChunkSource -> GpuFragmentSinkOperator) sharing one GpuFragment, %s\", \"pool\": \"%s\", "
           "\"forwarded_chunks\": %lld, \"forwarded_rows\": %lld, \"rows\": %zu, \"dop\": %d, \"seconds\": %.6f, \"probe_seconds\": %.6f, "
           "\"rows_per_s\": %.1f, \"build_seconds\": %.4f, \"groups\": %zu, \"matches_row_at_a_time_evaluation\": %s, \"h2d_bytes_offered\": %lld, "
           "\"d2h_bytes\": %lld, \"fragment_batches\": %lld, \"append_chunk_cpu_seconds_all_threads\": %.4f, \"fragment_push_call_seconds_all_threads\": %.4f, "
           "\"need_input_false_polls\": %lld, \"gpu_launches\": %lld}\n",
           dop, path.c_str(), pinned_pool ? "pinned" : "pageable", (long long)fwd_chunks, (long long)fwd_rows, n_fact, dop, total_s, probe_s, (double)n_fact / total_s, build_s, got.size(), ok ? "true" : "false", (long long)bytes, (long long)d2h,
           (long long)batches, append_ns / 1e9, push_ns / 1e9, (long long)stalls, (long long)(sr_ctx_kernel_launches(ctx) - launches0));
    fprintf(stderr, "%s\n%s\n", sinks[0]->unique_metrics()->to_string().c_str(), sinks[0]->common_metrics()->to_string().c_str());
    for (auto& d : drivers) d->close(&state);
    sinks.clear();
    drivers.clear();
    fragment.reset();
    joiners.clear();
    joiner_factories.clear();
    sr_ctx_destroy(ctx);
    return ok ? 0 : 1;
}
