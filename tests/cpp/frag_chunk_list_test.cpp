// The fused sink fed from a registered page-locked pool: SSB Q4.1 with
//   build pipelines (x4):  GpuScanOperator(dimension, predicate) -> GpuHashJoinBuildOperator
//   probe pipeline:        PoolChunkSource (4096-row chunks materialised into a PinnedArena, LO_SUPPLYCOST nullable)
//                          -> GpuFragmentSinkOperator (chunks forwarded to sr_fragment_push_chunks, no host copy)
//   result pipeline:       GpuAggregateBlockingSourceOperator -> collect
// The groups must equal the CPU oracle (oracle/sr_oracle.cpp) run on the same rows, every chunk must have been forwarded
// (ForwardedChunks = chunk count, PinnedBatchBytes = 0), and a pageable chunk with a nullable column must still be
// refused with NotSupported.  Exit code 0 = pass; 3 = no CUDA device.
//   frag_chunk_list_test [rows=300001]
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <thread>
#include <tuple>

#include "../../oracle/sr_oracle.h"
#include "../../starrocks_b200/host/gpu/gpu_operators.h"

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

#define CHECK_OK(expr)                                                              \
    do {                                                                            \
        Status _st = (expr);                                                        \
        if (!_st.ok()) {                                                            \
            fprintf(stderr, "FAILED %s: %s\n", #expr, _st.to_string().c_str());     \
            exit(2);                                                                \
        }                                                                           \
    } while (0)

void run_to_finish(PipelineDriver& d, RuntimeState* state, const char* name) {
    CHECK_OK(d.prepare(state));
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::seconds(300);
    while (std::chrono::steady_clock::now() < deadline) {
        auto st = d.process(state);
        if (!st.ok()) {
            fprintf(stderr, "driver %s failed: %s\n", name, st.status().to_string().c_str());
            exit(2);
        }
        if (st.value() == PipelineDriver::FINISH) return;
        if (st.value() == PipelineDriver::PRECONDITION_BLOCK) {
            fprintf(stderr, "driver %s is still blocked on its dependency\n", name);
            exit(2);
        }
        // READY without progress (the asynchronous scan's IO task is still running) or PENDING_FINISH: the real driver parks
        // in the poller (pipeline_driver_poller.cpp); here the thread naps
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
    fprintf(stderr, "driver %s made no progress\n", name);
    exit(2);
}

using Groups = std::map<std::pair<int32_t, int32_t>, std::pair<int64_t, int64_t>>;

Groups collect(const ResultSink& sink) {
    Groups g;
    for (auto& c : sink.chunks) {
        auto* y = (const int32_t*)c->get_column_by_slot_id(D_YEAR)->raw_data();
        auto* n = (const int32_t*)c->get_column_by_slot_id(C_NATION)->raw_data();
        auto* r = (const int64_t*)c->get_column_by_slot_id(OUT_REV)->raw_data();
        auto* s = (const int64_t*)c->get_column_by_slot_id(OUT_COST)->raw_data();
        for (size_t i = 0; i < c->num_rows(); i++) g[{y[i], n[i]}] = {r[i], s[i]};
    }
    return g;
}

sr_expr col_expr(int32_t slot) {
    sr_expr e{};
    e.nodes[0].op = SR_EX_COL;
    e.nodes[0].slot_id = slot;
    e.num_nodes = 1;
    return e;
}

// the scan side of the probe pipeline: one lineorder shard, handed out as <= chunk_size-row chunks whose columns are
// borrowed slices of a registered arena (what a scan over a pinned ColumnAllocator pool produces)
class PoolChunkSource final : public SourceOperator {
public:
    PoolChunkSource(std::shared_ptr<PinnedArena> arena, const std::vector<int32_t>* cols, const std::vector<uint8_t>* cost_nulls, size_t rows)
            : SourceOperator(nullptr, 3, "pool_chunk_source", 3, false, 0), _arena(std::move(arena)), _cols(cols), _cost_nulls(cost_nulls), _rows(rows) {}
    bool has_output() const override { return _next < _rows; }
    bool is_finished() const override { return _next >= _rows; }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override {
        const size_t n = std::min<size_t>((size_t)state->chunk_size(), _rows - _next);
        auto c = std::make_shared<Chunk>();
        for (int k = 0; k < 6; k++) {
            auto data = _arena->column(SR_TYPE_INT, n);
            if (!data) return Status::InternalError("arena full");
            memcpy(data->mutable_raw_data(), _cols[k].data() + _next, n * 4);
            if (k != LO_SUPPLYCOST) {
                c->append_column(data, (SlotId)k);
                continue;
            }
            auto nulls = _arena->column(SR_TYPE_BOOLEAN, n);
            if (!nulls) return Status::InternalError("arena full");
            memcpy(nulls->mutable_raw_data(), _cost_nulls->data() + _next, n);
            c->append_column(std::make_shared<NullableColumn>(data, nulls), (SlotId)k);
        }
        _next += n;
        chunks++;
        return c;
    }
    size_t chunks = 0;

private:
    std::shared_ptr<PinnedArena> _arena;
    const std::vector<int32_t>* _cols;
    const std::vector<uint8_t>* _cost_nulls;
    size_t _rows, _next = 0;
};

} // namespace

int main(int argc, char** argv) {
    const size_t n_fact = argc > 1 ? (size_t)atoll(argv[1]) : 300001;
    const int n_cust = 30000, n_supp = 2000, n_part = 20000, n_dates = 2556;
    sr_ctx* ctx = sr_ctx_create(0, nullptr);
    if (!ctx) {
        fprintf(stderr, "sr_ctx_create failed: %s\n", sr_last_error(nullptr));
        return 3;
    }
    RuntimeState state(4096);
    Rng rng{20240921};
    std::vector<int32_t> c_key(n_cust), c_region(n_cust), c_nation(n_cust), s_key(n_supp), s_region(n_supp), p_key(n_part), p_mfgr(n_part), d_key(n_dates),
            d_year(n_dates);
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
    std::vector<int32_t> lo[6];
    for (auto& v : lo) v.resize(n_fact);
    std::vector<uint8_t> cost_nulls(n_fact);
    for (size_t i = 0; i < n_fact; i++) {
        lo[LO_ORDERDATE][i] = d_key[rng.next(0, n_dates)];
        lo[LO_CUSTKEY][i] = rng.next(1, n_cust + 1);
        lo[LO_SUPPKEY][i] = rng.next(1, n_supp + 1);
        lo[LO_PARTKEY][i] = rng.next(1, n_part + 1);
        lo[LO_REVENUE][i] = rng.next(81000, 10400001);
        lo[LO_SUPPLYCOST][i] = rng.next(54000, 125001);
        cost_nulls[i] = rng.next(0, 7) == 0 ? 1 : 0; // SUM skips NULL costs
    }
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

    // ---- the oracle on the same rows (LO_SUPPLYCOST nullable) ----
    Groups oracle_groups;
    {
        std::vector<orc_join*> ojoins;
        orc_fragment_desc ofd{};
        ofd.num_joins = (int32_t)dims.size();
        ofd.agg = agg_desc;
        for (size_t k = 0; k < dims.size(); k++) {
            Dim& dm = dims[k];
            std::vector<int32_t> outs = {dm.key_slot};
            for (int32_t p : dm.payload) outs.push_back(p);
            sr_scan_desc sd{};
            sd.preds = dm.pred;
            sd.num_preds = dm.pred ? 1 : 0;
            sd.out_slots = outs.data();
            sd.num_out_slots = (int32_t)outs.size();
            std::vector<sr_col_view> views;
            sr_chunk_view tv = make_chunk_view(*dm.table, &views);
            std::vector<std::vector<int32_t>> kept(outs.size(), std::vector<int32_t>(dm.table->num_rows()));
            std::vector<void*> od(outs.size());
            std::vector<uint8_t*> on(outs.size(), nullptr);
            for (size_t c = 0; c < outs.size(); c++) od[c] = kept[c].data();
            const int64_t rows = orc_scan_filter(&sd, &tv, od.data(), on.data());
            if (rows < 0) {
                fprintf(stderr, "oracle scan failed: %s\n", orc_last_error());
                return 2;
            }
            sr_join_desc jd{};
            jd.join_type = SR_JOIN_INNER;
            jd.num_keys = 1;
            jd.build_key_slots[0] = dm.key_slot;
            jd.probe_key_slots[0] = dm.probe_slot;
            jd.key_types[0] = SR_TYPE_INT;
            jd.enable_range_direct_mapping = 1;
            jd.num_build_out = (int32_t)dm.payload.size();
            for (size_t p = 0; p < dm.payload.size(); p++) jd.build_out_slots[p] = dm.payload[p];
            orc_join_options opt{1, 1, 1 << 20, 32 << 20, 0, 0};
            orc_join* oj = orc_join_create(&jd, &opt);
            std::vector<sr_col_view> bcols;
            for (size_t c = 0; c < outs.size(); c++) bcols.push_back(sr_col_view{kept[c].data(), nullptr, SR_TYPE_INT, outs[c]});
            sr_chunk_view bv{bcols.data(), (int32_t)bcols.size(), SR_MEM_HOST, rows};
            if (!oj || orc_join_append_build(oj, &bv) != SR_OK || orc_join_build(oj) != SR_OK) {
                fprintf(stderr, "oracle join build failed: %s\n", orc_last_error());
                return 2;
            }
            ojoins.push_back(oj);
            ofd.joins[k].join = oj;
            ofd.joins[k].probe_key_slot = dm.probe_slot;
            ofd.joins[k].num_payload = (int32_t)dm.payload.size();
            for (size_t p = 0; p < dm.payload.size(); p++) ofd.joins[k].payload_build_slots[p] = dm.payload[p];
        }
        std::vector<sr_col_view> fviews;
        for (int k = 0; k < 6; k++) fviews.push_back(sr_col_view{lo[k].data(), k == LO_SUPPLYCOST ? cost_nulls.data() : nullptr, SR_TYPE_INT, k});
        sr_chunk_view fv{fviews.data(), 6, SR_MEM_HOST, (int64_t)n_fact};
        orc_agg* oresult = orc_agg_create(&agg_desc);
        int64_t passed = 0;
        if (!oresult || orc_fragment_run(&ofd, &fv, 4, oresult, &passed) != SR_OK) {
            fprintf(stderr, "oracle fragment run failed: %s\n", orc_last_error());
            return 2;
        }
        const int64_t g = orc_agg_num_groups(oresult);
        std::vector<int32_t> oy((size_t)g), on_((size_t)g);
        std::vector<int64_t> orv((size_t)g), oc((size_t)g);
        std::vector<uint8_t> nul0((size_t)g), nul1((size_t)g), nul2((size_t)g), nul3((size_t)g);
        void* od[4] = {oy.data(), on_.data(), orv.data(), oc.data()};
        uint8_t* onl[4] = {nul0.data(), nul1.data(), nul2.data(), nul3.data()};
        if (orc_agg_output(oresult, od, onl) != SR_OK) {
            fprintf(stderr, "oracle output failed: %s\n", orc_last_error());
            return 2;
        }
        for (int64_t i = 0; i < g; i++) oracle_groups[{oy[(size_t)i], on_[(size_t)i]}] = {orv[(size_t)i], oc[(size_t)i]};
        orc_agg_destroy(oresult);
        for (auto* oj : ojoins) orc_join_destroy(oj);
        printf("oracle: %zu groups from %lld joined rows\n", oracle_groups.size(), (long long)passed);
    }

    // ---- build side through the operators ----
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
        run_to_finish(build_driver, &state, dm.name);
        build_driver.close(&state);
    }
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

    // ---- probe: pool chunks forwarded into the fused sink ----
    std::string err;
    auto arena = PinnedArena::create(ctx, n_fact * (6 * 4 + 1) + (n_fact / 4096 + 1) * 7 * PinnedArena::ALIGN, &err);
    if (!arena) {
        fprintf(stderr, "%s\n", err.c_str());
        return 2;
    }
    auto fragment = std::make_shared<GpuFragment>(ctx, fd, joiners);
    auto src = std::make_shared<PoolChunkSource>(arena, lo, &cost_nulls, n_fact);
    auto sink = std::make_shared<GpuFragmentSinkOperator>(nullptr, 8, 8, 0, fragment, (size_t)1 << 16); // several lists per slot
    {
        PipelineDriver probe_driver({src, sink});
        run_to_finish(probe_driver, &state, "probe(forwarded)");
        probe_driver.close(&state);
    }
    auto rsink = std::make_shared<ResultSink>();
    {
        PipelineDriver result_driver({std::make_shared<GpuAggregateBlockingSourceOperator>(nullptr, 9, 9, 0, fragment->aggregator()), rsink});
        run_to_finish(result_driver, &state, "result");
        result_driver.close(&state);
    }
    const Groups got = collect(*rsink);
    const int64_t forwarded = sink->unique_metrics()->get_counter("ForwardedChunks")->value();
    const int64_t forwarded_rows = sink->unique_metrics()->get_counter("ForwardedRows")->value();
    const int64_t copied = sink->unique_metrics()->get_counter("PinnedBatchBytes")->value();
    printf("forwarded %lld chunks (%lld rows) of %zu, copied %lld bytes, %zu groups\n%s\n", (long long)forwarded, (long long)forwarded_rows, src->chunks,
           (long long)copied, got.size(), sink->unique_metrics()->to_string().c_str());
    if (got != oracle_groups) {
        fprintf(stderr, "forwarded pipeline differs from the oracle (%zu vs %zu groups)\n", got.size(), oracle_groups.size());
        return 1;
    }
    if (forwarded != (int64_t)src->chunks || forwarded_rows != (int64_t)n_fact || copied != 0) {
        fprintf(stderr, "not every chunk was forwarded\n");
        return 1;
    }

    // ---- a pageable chunk with a nullable column still takes the copy path, which refuses it ----
    {
        auto frag2 = std::make_shared<GpuFragment>(ctx, fd, joiners);
        GpuFragmentSinkOperator sink2(nullptr, 8, 8, 0, frag2);
        auto c = std::make_shared<Chunk>();
        for (int k = 0; k < 6; k++) {
            auto data = std::make_shared<Int32Column>(SR_TYPE_INT, std::vector<int32_t>(lo[k].begin(), lo[k].begin() + 100));
            if (k == LO_SUPPLYCOST)
                c->append_column(std::make_shared<NullableColumn>(data, std::make_shared<NullColumn>(SR_TYPE_BOOLEAN, std::vector<uint8_t>(100, 0))), k);
            else
                c->append_column(data, k);
        }
        const Status st = sink2.push_chunk(&state, c);
        if (st.code() != Status::NotSupported("").code()) {
            fprintf(stderr, "pageable nullable chunk: %s (want NotSupported)\n", st.to_string().c_str());
            return 1;
        }
    }
    sink.reset();
    src.reset();
    fragment.reset();
    arena.reset();
    joiners.clear();
    joiner_factories.clear();
    sr_ctx_destroy(ctx);
    printf("FRAG_CHUNK_LIST_OK\n");
    return 0;
}
