// sr_frag.cuh -- the fused pipeline fragment: scan -> filter -> [hash-join probe]* -> aggregate
// in ONE pass over the fact columns.  This is the hot kernel of the SSB Q4.1 / Q1.1 configs.
//
// What it fuses (reference call stack, SURVEY.md section 3.3-3.5):
//   OlapChunkSource::_read_chunk_from_storage filter step   scan/olap_chunk_source.cpp:676-722
//   HashJoinProbeOperator::push_chunk/pull_chunk x N        hashjoin/hash_join_probe_operator.cpp:55-96
//     -> JoinHashMap::probe (lookup_init + _probe_from_ht + _probe_output/_build_output)
//   AggregateBlockingSinkOperator::push_chunk               aggregate/aggregate_blocking_sink_operator.cpp:101-138
//
// H100 design (HBM-bound integer/gather work, no tensor cores):
//  * persistent CTAs (grid = SMs x resident CTAs).  The main loop streams the scan-predicate
//    columns and the FIRST join's key column: each thread owns groups of 4 consecutive rows, so a
//    tile column is one 128-bit ld.global.nc.L1::no_allocate per thread and group;
//  * selection-vector cascade: rows that survive stage k are appended (warp ballot + popc) to a
//    per-warp queue in shared memory; as soon as a queue holds 32 rows the warp runs stage k+1
//    for 32 rows at once (one row per lane).  Later stages therefore always execute with full
//    warps, their column loads are issued for 32 rows together, and the dependent-load chain of
//    a tile is one DRAM round trip instead of one per join;
//  * late materialisation: a column is only loaded for rows still alive, so DRAM sectors of later
//    columns are skipped when all 8 rows of a 32-byte sector were filtered out;
//  * every range-mapped join is tested against its 1-bit-per-key bitmap; the bitmaps of the
//    earliest joins are copied into shared memory once per CTA, the others are read through
//    L1/L2 (SSB dimension bitmaps are 25-375 KB and stay L2 resident);
//  * the build row index (first[]) and payload columns are only fetched for rows that survive all
//    joins; the group-by / SUM update of the final queue goes to shared-memory accumulators when
//    the table is small, flushed once per CTA;
//  * join order: pass rates measured on a sample of the first batch (adaptive), most selective
//    first, smaller table first on a tie -- inner joins commute, the result is order independent.
//
// Host side: frag_plan chooses the mode on the first batch and plans it (frag_plan_passes: the selection-vector passes
// of sr_frag_pass.cuh, frag_plan_cascade: k_fragment); frag_push runs it on every batch, the final pass of the
// selection-vector passes through frag_launch_final.
#pragma once

#include "sr_agg.cuh"

#include "sr_frag_kernel.cuh"
#include "sr_frag_pass.cuh"
#include "sr_gather.cuh"

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct sr_fragment {
    sr_ctx* ctx = nullptr;
    std::vector<sr_pred> preds;
    std::vector<sr_expr> exprs;
    int32_t num_joins = 0;
    sr_frag_join joins[SR_MAX_FRAG_JOINS];
    sr_agg* agg = nullptr;
    bool compiled = false;
    VReg reg; // fact + payload values
    std::vector<int32_t> value_src;         // per value: -1 fact, j = payload of (ordered) join j
    std::vector<const BuildCol*> value_col; // payload column for src >= 0
    srd::FragDev host;
    DevBuf dev, counters;
    Staged staged;
    bool smem_agg = false;
    int order[SR_MAX_FRAG_JOINS];
    double pass_rate[SR_MAX_FRAG_JOINS];
    double pred_rate = 1.0;
    int force_mode = 0; // 0 = choose from the sampled pass rates, 1 = fused cascade kernel, 2 = selection-vector passes
    // cascade mode (k_fragment), planned by frag_plan_cascade
    size_t cascade_smem = 0;
    int32_t queue_word_off = 0;
    int cascade_grid = 0;
    // selective mode (sr_frag_pass.cuh): streaming pass -> gather passes -> final pass, planned by frag_plan_passes
    bool selective = false;
    bool expand = false; // some INNER / LEFT OUTER join has duplicate build keys: selection-vector passes + k_frag_gather_agg<false, SINGLE, true, CONJ>
    bool conj = false;   // some INNER / LEFT SEMI join has an other-join conjunct: selection-vector passes + k_frag_gather_agg<..., true>
    srd::PassDev pass;
    std::vector<int> gather_joins; // probe positions that get a pass of their own
    DevBuf sel[2], pass_counters;
    double est_rate = 1.0; // sampled fraction of the fact rows that reaches the aggregate
    size_t stream_smem = 0;
    int stream_grid = 0;
    int gather_grid = 0; // k_frag_gather_join
    int final_grid = 0;
    // the batched final pass (k_frag_final_dense): planned when the shape allows it, used by a push whose fact columns
    // are all plain int32 and whose aggregate still accumulates in shared memory
    bool final_dense_ok = false;
    srd::FinalDense final_dense;             // pointers into the fact chunk and the aggregate are filled per push
    int8_t final_fn_src[srd::FINAL_MAX_FNS]; // aggregate function behind each FinalDense::fn
    DevBuf digits[SR_MAX_FRAG_JOINS];        // slot-digit directories, per probe position
    int final_dense_grid = 0;
    int32_t final_pass = SR_FINAL_PASS_NONE; // the final pass of the last push
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool timed_push = false;
    ChunkGather chunk_gather; // sr_fragment_push_chunks: the batch a list of chunks is gathered into
    // payload columns of a join whose build side never received a chunk (a dimension scan that filtered everything out):
    // the type sr_join_desc.build_out_types declares over a zeroed row 0, which every probe row reads as NULL
    // (FragLoader::load) -- what sr_join_probe pads a LEFT OUTER join's rows with
    BuildCol empty_payload[SR_MAX_FRAG_JOINS][SR_MAX_FRAG_PAYLOAD];
    // the same for the build columns an other-join conjunct reads (never evaluated: such an INNER / SEMI join passes nothing)
    std::vector<std::unique_ptr<BuildCol>> empty_conj[SR_MAX_FRAG_JOINS];
    ~sr_fragment() {
        for (int e = 0; e < 4; e++)
            if (ev[e]) cudaEventDestroy(ev[e]);
    }
};

struct FragTypeCtx {
    sr_fragment* f;
};

// the slots expression `e` reads, appended to `slots`
static void expr_slots(const sr_expr& e, std::vector<int32_t>* slots) {
    for (int k = 0; k < std::min<int32_t>(e.num_nodes, SR_MAX_EXPR_NODES); k++)
        if (e.nodes[k].op == SR_EX_COL) slots->push_back(e.nodes[k].slot_id);
}
static bool expr_reads(const sr_expr& e, int32_t slot) {
    std::vector<int32_t> s;
    expr_slots(e, &s);
    return std::find(s.begin(), s.end(), slot) != s.end();
}
// the slots an aggregate reads: group keys and function inputs
static void frag_agg_slots(const sr_agg_desc& d, std::vector<int32_t>* slots) {
    slots->clear();
    for (int k = 0; k < std::min<int32_t>(d.num_group_keys, SR_MAX_GROUP_KEYS); k++) slots->push_back(d.group_slots[k]);
    for (int q = 0; q < std::min<int32_t>(d.num_fns, SR_MAX_AGG_FNS); q++) {
        if (d.fns[q].kind != SR_AGG_COUNT_STAR) expr_slots(d.fns[q].input, slots);
        if (d.fns[q].kind == SR_AGG_AVG_MERGE) slots->push_back(d.fns[q].reserved);
    }
}

// the first join (hint order) that carries `slot` as a payload, else the first whose other-join conjunct reads `slot` as
// one of its build columns (unless payload_only), and that build column; join = -1 when none does
struct FragPayload {
    const BuildCol* col;
    int join;
};
static FragPayload frag_find_payload(const sr_fragment* f, int32_t slot, bool payload_only = false) {
    for (int j = 0; j < f->num_joins; j++)
        for (int p = 0; p < f->joins[j].num_payload; p++)
            if (f->joins[j].payload_build_slots[p] == slot) {
                const BuildCol* bc = f->joins[j].join->find_col(slot);
                return FragPayload{bc ? bc : &f->empty_payload[j][p], j}; // sr_fragment_create filled the latter
            }
    for (int j = 0; j < f->num_joins && !payload_only; j++) {
        if (!expr_reads(f->joins[j].join->desc.other_conjunct, slot)) continue;
        if (const BuildCol* bc = f->joins[j].join->find_col(slot)) return FragPayload{bc, j};
        for (const auto& bc : f->empty_conj[j])
            if (bc->slot == slot) return FragPayload{bc.get(), j};
    }
    return FragPayload{nullptr, -1};
}

// the type sr_join_desc.build_out_types declares for build slot `slot`, 0 when none is declared
static int32_t join_declared_out_type(const sr_join* jn, int32_t slot) {
    for (int k = 0; k < std::min<int32_t>(jn->desc.num_build_out, SR_MAX_JOIN_OUT); k++)
        if (jn->desc.build_out_slots[k] == slot && srd::type_width(jn->desc.build_out_types[k]) > 0) return jn->desc.build_out_types[k];
    return 0;
}

// slot type: fact chunk first, then payload columns of the joins
static int32_t frag_slot_type(void* user, int32_t slot) {
    sr_fragment* f = ((FragTypeCtx*)user)->f;
    const int k = f->staged.find(slot);
    if (k >= 0) return f->staged.cols[k].type;
    const BuildCol* bc = frag_find_payload(f, slot).col;
    return bc ? bc->type : 0;
}
// a payload of a LEFT OUTER join is nullable whatever its build column is: a probe row without a build row reads NULL
static bool frag_slot_nullable(void* user, int32_t slot) {
    sr_fragment* f = ((FragTypeCtx*)user)->f;
    const int k = f->staged.find(slot);
    if (k >= 0) return f->staged.cols[k].nulls != nullptr;
    const FragPayload pl = frag_find_payload(f, slot);
    if (pl.join >= 0 && f->joins[pl.join].join->desc.join_type == SR_JOIN_LEFT_OUTER) return true;
    return pl.col && pl.col->nullable;
}

// what join j (hint order) does to a probe row (srd::FRAG_FILTER / FRAG_ANTI / FRAG_OUTER)
static int32_t frag_join_kind(const sr_fragment* f, int j) {
    const int32_t t = f->joins[j].join->desc.join_type;
    return t == SR_JOIN_LEFT_ANTI ? srd::FRAG_ANTI : t == SR_JOIN_LEFT_OUTER ? srd::FRAG_OUTER : srd::FRAG_FILTER;
}

static int32_t frag_bind_vtab(sr_fragment* f, VTab* vt) {
    sr_ctx* ctx = f->ctx;
    vt->n = (int32_t)f->reg.slots.size();
    for (size_t k = 0; k < f->reg.slots.size(); k++) {
        if (f->value_src[k] < 0) {
            const int c = f->staged.find(f->reg.slots[k]);
            if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fact chunk misses slot %d", f->reg.slots[k]);
            if (f->staged.cols[c].type != f->reg.types[k]) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fact slot %d changed type", f->reg.slots[k]);
            vt->v[k].data = f->staged.cols[c].data;
            vt->v[k].nulls = f->staged.cols[c].nulls;
            vt->v[k].type = f->staged.cols[c].type;
            vt->v[k].src = -1;
        } else {
            const BuildCol* bc = f->value_col[k];
            vt->v[k].data = bc->data.p;
            vt->v[k].nulls = bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr;
            vt->v[k].type = bc->type;
            vt->v[k].src = f->value_src[k];
        }
    }
    vt_mark_plain32(vt);
    return SR_OK;
}

static int32_t frag_compile(sr_fragment* f) {
    sr_ctx* ctx = f->ctx;
    FragTypeCtx tc{f};
    srd::FragDev& h = f->host;
    memset(&h, 0, sizeof(h));
    f->reg = VReg();
    if (f->preds.size() > 8 || f->exprs.size() > 4) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many scan conjuncts for the fused fragment");
    for (size_t k = 0; k < f->preds.size(); k++) SR_TRY(compile_pred(ctx, &f->preds[k], &f->reg, frag_slot_type, &tc, &h.preds[k]));
    for (size_t k = 0; k < f->exprs.size(); k++) {
        SR_TRY(compile_expr(ctx, &f->exprs[k], &f->reg, frag_slot_type, &tc, &h.exprs[k]));
        if (h.exprs[k].result_is_double) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "filter expression %zu is not boolean", k);
    }
    // the scan conjuncts run on fact rows ahead of every join, so each value they read must be a fact column: a join
    // payload would be indexed by fact row.  Refused before the aggregate compiles, which sets up and clears its tables
    for (size_t k = 0; k < f->reg.slots.size(); k++) {
        if (f->staged.find(f->reg.slots[k]) >= 0) continue;
        const FragPayload pl = frag_find_payload(f, f->reg.slots[k]);
        if (pl.join >= 0)
            return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "scan conjunct reads slot %d, a payload of join %d: scan predicates and filter expressions name fact slots only",
                           f->reg.slots[k], pl.join);
    }
    h.num_preds = (int32_t)f->preds.size();
    h.num_exprs = (int32_t)f->exprs.size();
    h.num_joins = f->num_joins;
    // join keys (identity order for now; reordered after sampling)
    for (int j = 0; j < f->num_joins; j++) {
        sr_join* jn = f->joins[j].join;
        const int c = f->staged.find(f->joins[j].probe_key_slot);
        if (c < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "fact chunk misses probe key slot %d", f->joins[j].probe_key_slot);
        if (srd::is_float_class(f->staged.cols[c].type) || f->staged.cols[c].width > 8)
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "probe key slot %d has a non-integer type", f->joins[j].probe_key_slot);
        if (f->staged.cols[c].width != srd::type_width(jn->desc.key_types[0]))
            return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "probe key slot %d width differs from the join's key type", f->joins[j].probe_key_slot);
        const int id = f->reg.add(f->joins[j].probe_key_slot, f->staged.cols[c].type);
        if (id >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
        h.joins[j].key_value_id = id;
        h.joins[j].j = jn->dev();
        h.joins[j].smem_off = -1;
        h.joins[j].use_bitmap = jn->method != SR_JOIN_METHOD_LINEAR_CHAINED ? 1 : 0;
        h.joins[j].bitmap_words = (int32_t)((std::max<int64_t>(jn->bucket_size, 1) + 31) / 32);
        // one-to-many INNER / LEFT OUTER join: the final pass walks the build chain of every surviving row
        h.joins[j].kind = frag_join_kind(f, j);
        h.joins[j].expand = (jn->has_dup && (jn->desc.join_type == SR_JOIN_INNER || jn->desc.join_type == SR_JOIN_LEFT_OUTER)) ? 1 : 0;
        h.joins[j].need_head = h.joins[j].expand;
        h.joins[j].idx32 = (h.joins[j].use_bitmap && jn->min_value >= INT32_MIN && jn->max_value <= INT32_MAX && jn->max_value >= jn->min_value) ? 1 : 0;
        f->order[j] = j;
        if (h.joins[j].kind != srd::FRAG_OUTER) h.num_filter_joins++;
    }
    // other-join conjuncts (INNER / LEFT SEMI, sr_fragment_create): each reads fact columns and its own join's build
    // columns, the fact chunk first as sr_join_probe resolves them.  The final pass evaluates them at the join's build rows
    for (int j = 0; j < f->num_joins; j++) {
        const sr_expr& e = f->joins[j].join->desc.other_conjunct;
        if (e.num_nodes <= 0) continue;
        for (int k = 0; k < std::min<int32_t>(e.num_nodes, SR_MAX_EXPR_NODES); k++) {
            const int32_t slot = e.nodes[k].slot_id;
            if (e.nodes[k].op != SR_EX_COL || f->staged.find(slot) >= 0) continue;
            // one slot id names one value of the fragment: a slot another join carries (a payload, a column its conjunct
            // reads, or any column of its build chunks) is that join's, even when this join's build side has one too
            const FragPayload pl = frag_find_payload(f, slot);
            int other = pl.join;
            for (int q = 0; q < f->num_joins && other < 0; q++)
                if (q != j && f->joins[q].join->find_col(slot)) other = q;
            if (other >= 0 && other != j)
                return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "other-join conjunct of join %d reads slot %d, a column of join %d: a conjunct reads fact columns and its own join's build columns",
                               j, slot, other);
            if (pl.join < 0) {
                if (f->joins[j].join->cols.empty())
                    return sr_fail(ctx, SR_ERR_STATE, "fragment join %d: build side is empty and the type of conjunct slot %d is unknown: declare it in sr_join_desc.build_out_types",
                                   j, slot);
                return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "other-join conjunct of join %d: slot %d is in neither the fact chunk nor the build chunk", j, slot);
            }
        }
        SR_TRY(compile_expr(ctx, &e, &f->reg, frag_slot_type, &tc, &h.conj[j]));
        if (h.conj[j].result_is_double) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "other-join conjunct of join %d is not boolean", j);
        h.conj_mask |= 1 << j;
        h.joins[j].need_head = 1;
    }
    // aggregate (its expressions may reference fact slots and payload slots: a build column only a conjunct reads is not
    // part of the join's output)
    {
        std::vector<int32_t> read;
        frag_agg_slots(f->agg->desc, &read);
        for (const int32_t slot : read)
            if (f->staged.find(slot) < 0 && frag_find_payload(f, slot).join >= 0 && frag_find_payload(f, slot, true).join < 0)
                return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "slot %d is neither a fact column nor a join payload", slot);
    }
    SR_TRY(agg_compile(f->agg, frag_slot_type, frag_slot_nullable, &tc));
    // the fragment and its aggregate share one value table: rebuild the aggregate's value ids on top
    // of the fragment registry
    {
        VReg merged = f->reg;
        std::vector<int> remap(f->agg->reg.slots.size());
        for (size_t k = 0; k < f->agg->reg.slots.size(); k++) {
            remap[k] = merged.add(f->agg->reg.slots[k], f->agg->reg.types[k]);
            if (remap[k] >= SR_MAX_VALUES) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "too many distinct columns");
        }
        srd::AggDev& ah = f->agg->host;
        for (int k = 0; k < ah.num_keys; k++) ah.key_value_id[k] = remap[ah.key_value_id[k]];
        for (int q = 0; q < ah.num_fns; q++)
            for (int k = 0; k < ah.fns[q].input.num_nodes; k++)
                if (ah.fns[q].input.nodes[k].op == srd::C_LOAD_I || ah.fns[q].input.nodes[k].op == srd::C_LOAD_D)
                    ah.fns[q].input.nodes[k].arg = remap[ah.fns[q].input.nodes[k].arg];
        f->agg->reg = merged;
        f->reg = merged;
        SR_TRY(agg_upload(f->agg));
    }
    // classify values: fact column or payload of join j
    f->value_src.assign(f->reg.slots.size(), -1);
    f->value_col.assign(f->reg.slots.size(), nullptr);
    for (size_t k = 0; k < f->reg.slots.size(); k++) {
        if (f->staged.find(f->reg.slots[k]) >= 0) continue;
        const FragPayload pl = frag_find_payload(f, f->reg.slots[k]);
        if (pl.join < 0) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "slot %d is neither a fact column nor a join payload", f->reg.slots[k]);
        f->value_src[k] = pl.join;
        f->value_col[k] = pl.col;
        h.joins[pl.join].need_head = 1;
    }
    SR_TRY(f->counters.reserve(ctx, 256));
    SR_CUDA(ctx, cudaMemsetAsync(f->counters.p, 0, 256, ctx->stream));
    h.rows_passed = f->counters.as<unsigned long long>();
    return SR_OK;
}

// whether the final pass of selective mode tests join q (probe order): the filtering and anti joins it was left
static bool frag_final_tests(const sr_fragment* f, int q) {
    return q >= f->pass.final_first_join && f->host.joins[q].kind != srd::FRAG_OUTER;
}

// Plan the batched final pass (k_frag_final_dense) of selective mode, once the join order is fixed.  It applies when
//  * the aggregate is dense, accumulates in shared memory and has fewer slots than the reserved digit values;
//  * every join the final pass looks up is range-mapped with unique keys and an int32 range, and its payload columns
//    are only group keys: it gets a slot-digit directory, built here (a LEFT OUTER join's directory holds the all-NULL
//    digit, 0, for keys without a build row, and the pass reads that digit for keys outside the range too);
//  * every join the final pass only tests is a bitmap test (inverted for an anti join);
//  * every aggregate input is one fact column in an integer mode acc_apply_shared handles (COUNT(*), SUM, COUNT, MIN,
//    MAX on int64 states).
// Otherwise the generic final pass runs.  That the fact columns are plain int32 is checked per push.
static int32_t frag_plan_final_dense(sr_fragment* f) {
    sr_ctx* ctx = f->ctx;
    const srd::FragDev& h = f->host;
    const srd::AggDev& ah = f->agg->host;
    srd::FinalDense& fp = f->final_dense;
    memset(&fp, 0, sizeof(fp));
    f->final_dense_ok = false;
    if (f->expand || f->conj || !f->smem_agg || !ah.dense || ah.num_keys == 0 || ah.cap >= SR_DIGIT_BAD) return SR_OK;
    const int nv = f->pass.num_final_vals;
    if (nv > srd::FINAL_MAX_VALS) return SR_OK;
    auto val_of = [&](int id) {
        for (int k = 0; k < nv; k++)
            if (f->pass.final_vals[k] == id) return k;
        return -1;
    };
    fp.num_vals = nv;
    fp.carry_val = -1;
    fp.cap = (int32_t)ah.cap;
    // group keys that are fact columns; the others must be payloads of a directory join
    bool key_of_join[SR_MAX_FRAG_JOINS] = {};
    for (int k = 0; k < ah.num_keys; k++) {
        const int id = ah.key_value_id[k];
        const int src = f->value_src[id];
        if (src >= 0) {
            key_of_join[src] = true;
            continue;
        }
        if (fp.num_fkeys == srd::FINAL_MAX_FKEYS || val_of(id) < 0) return SR_OK;
        srd::FinalDense::FKey& fk = fp.fkey[fp.num_fkeys++];
        fk.val = val_of(id);
        fk.lo = ah.dense_min[k];
        fk.base = ah.key_nullable[k] ? 1u : 0u;
        fk.span = ah.dense_extent[k] - fk.base;
        fk.stride = (uint32_t)ah.dense_stride[k];
    }
    // every value read from a build row must be a group key (then the directory stands for it)
    for (size_t id = 0; id < f->value_src.size(); id++) {
        if (f->value_src[id] < 0) continue;
        bool is_key = false;
        for (int k = 0; k < ah.num_keys; k++) is_key |= ah.key_value_id[k] == (int)id;
        if (!is_key) return SR_OK;
    }
    // aggregate functions
    int32_t acc0_off[SR_MAX_AGG_FNS] = {}; // shared-memory image of the push kernels: the state arrays, cap slots each
    int32_t off = 0;
    srd::agg_state_arrays(ah, [&](int q, srd::AccWord w) {
        if (w == srd::W_ACC0) acc0_off[q] = off;
        off += (int32_t)ah.cap;
    });
    for (int q = 0; q < ah.num_fns; q++) {
        const srd::AggFnDev& fn = ah.fns[q];
        if (fn.mode == srd::M_COUNT_STAR) continue;
        if (fn.mode != srd::M_COUNT && fn.mode != srd::M_SUM_I64 && fn.mode != srd::M_MIN_I64 && fn.mode != srd::M_MAX_I64) return SR_OK;
        if (fn.track_n || fn.n_value_id >= 0 || fn.input.num_nodes != 1 || fn.input.nodes[0].op != srd::C_LOAD_I) return SR_OK;
        const int id = fn.input.nodes[0].arg;
        if (f->value_src[id] >= 0 || val_of(id) < 0 || fp.num_fns == srd::FINAL_MAX_FNS) return SR_OK;
        f->final_fn_src[fp.num_fns] = (int8_t)q;
        srd::FinalDense::Fn& d = fp.fn[fp.num_fns++];
        d.mode = fn.mode;
        d.val = fn.mode == srd::M_COUNT ? -1 : val_of(id);
        d.smem_off = acc0_off[q];
    }
    // joins the final pass handles
    int look_join[srd::FINAL_MAX_LOOK] = {};
    for (int q = 0; q < f->num_joins; q++) {
        const srd::FragJoinDev& fj = h.joins[q];
        const bool test = frag_final_tests(f, q);
        if (!fj.need_head && !test) continue;
        const int kv = val_of(fj.key_value_id);
        if (!fj.use_bitmap || !fj.idx32 || fj.expand || kv < 0) return SR_OK;
        const uint32_t lo = (uint32_t)(int32_t)fj.j.min_value, span = (uint32_t)(fj.j.max_value - fj.j.min_value);
        if (!fj.need_head) {
            if (fp.num_test == srd::FINAL_MAX_TEST) return SR_OK;
            fp.test[fp.num_test++] = srd::FinalDense::Test{fj.j.bitmap, lo, span, kv, fj.kind == srd::FRAG_ANTI ? 1u : 0u};
            continue;
        }
        if (!key_of_join[q] || fp.num_look == srd::FINAL_MAX_LOOK) return SR_OK;
        look_join[fp.num_look] = q;
        // every payload of an outer join is a nullable group key (frag_slot_nullable): NULL is index 0 of each, digit 0
        fp.look[fp.num_look++] = srd::FinalDense::Look{nullptr, lo, span, kv, fj.kind == srd::FRAG_OUTER ? 0u : (uint32_t)SR_DIGIT_MISS};
    }
    // the directories
    for (int L = 0; L < fp.num_look; L++) {
        const int q = look_join[L];
        srd::DigitPlan dp;
        memset(&dp, 0, sizeof(dp));
        dp.miss = fp.look[L].miss;
        for (int k = 0; k < ah.num_keys; k++) {
            const int id = ah.key_value_id[k];
            if (f->value_src[id] != q) continue;
            const BuildCol* bc = f->value_col[id];
            srd::DigitKey& dk = dp.k[dp.num_keys++];
            dk.data = bc->data.p;
            dk.nulls = bc->nullable ? (const uint8_t*)bc->nulls.p : nullptr;
            dk.type = bc->type;
            dk.nullable = ah.key_nullable[k];
            dk.min = ah.dense_min[k];
            dk.extent = ah.dense_extent[k];
            dk.stride = ah.dense_stride[k];
        }
        const int64_t range = (int64_t)fp.look[L].span + 1;
        SR_TRY(f->digits[q].reserve(ctx, sizeof(uint16_t) * (size_t)range));
        srd::k_frag_build_digits<<<std::min(grid_for(range, 256), ctx->num_sms * 8), 256, 0, ctx->stream>>>(h.joins[q].j.first, range, dp,
                                                                                                             f->digits[q].as<uint16_t>());
        SR_LAUNCH_CHECK(ctx);
        fp.look[L].digit = f->digits[q].as<uint16_t>();
    }
    const size_t smem = f->agg->smem_bytes;
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_frag_final_dense<srd::FINAL_ROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 16)));
    int per_sm = 0;
    SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, srd::k_frag_final_dense<srd::FINAL_ROWS>, srd::GATHER_BLOCK, smem));
    f->final_dense_grid = std::max(per_sm, 1) * ctx->num_sms;
    f->final_dense_ok = true;
    return SR_OK;
}

// ---- selection-vector mode (sr_frag_pass.cuh) ----

// which joins the streaming pass, the gather passes and the final pass test, and the streamed join that carries its key
// (only filtering and anti joins: the outer joins behind them are looked up by the final pass and never tested)
static void frag_plan_stream_joins(sr_fragment* f) {
    const srd::FragDev& h = f->host;
    const int* ord = f->order;
    const int nf = h.num_filter_joins;
    // joins whose key column is streamed: the first one, and the second when >= 8 % of the rows reach it
    int ns = nf > 0 ? 1 : 0;
    if (nf > 1 && f->pred_rate * f->pass_rate[ord[0]] >= 0.08) ns = 2;
    // trailing joins that filter (almost) nothing are tested inline by the final pass
    int ff = nf;
    while (ff > ns && f->pass_rate[ord[ff - 1]] >= 0.9) ff--;
    f->pass.num_stream_joins = ns;
    f->pass.final_first_join = ff;
    f->gather_joins.clear();
    for (int q = ns; q < ff; q++) f->gather_joins.push_back(q);
    // a streamed join whose build row the final pass looks up (payload) hands its int32 key over through the
    // selection vector: one random fact-sector read less per surviving row
    f->pass.carry_join = -1;
    f->pass.carry_value_id = -1;
    for (int q = 0; q < ns; q++) {
        const int id = h.joins[q].key_value_id;
        const int32_t kt = f->reg.types[id];
        if (h.joins[q].need_head && srd::type_width(kt) == 4 && !srd::is_float_class(kt) && id < 127) {
            f->pass.carry_join = (int8_t)q;
            f->pass.carry_value_id = (int8_t)id;
            break;
        }
    }
}

// streaming pass shared memory: bitmaps of the streamed joins only (less the carried-key stash of
// k_frag_stream_tests<true>, so that two CTAs still fit on an SM)
static void frag_plan_stream_smem(sr_fragment* f) {
    srd::FragDev& h = f->host;
    size_t sw = 0;
    const size_t sbudget = (100 * 1024 - (f->pass.carry_join >= 0 ? sizeof(int4) * srd::FRAG_GROUPS * srd::FRAG_BLOCK : 0)) / 4;
    for (int q = 0; q < f->num_joins; q++) {
        srd::FragJoinDev& fj = h.joins[q];
        fj.smem_off = -1;
        if (q < f->pass.num_stream_joins && fj.use_bitmap && sw + (size_t)fj.bitmap_words + 1 <= sbudget) {
            fj.smem_off = (int32_t)sw;
            sw += ((size_t)fj.bitmap_words + 1 + 3) & ~(size_t)3; // + one zero guard word (stream_test_reg kind 1)
        }
    }
    f->stream_smem = sw * 4;
}

// the streaming pass in "tests" form (k_frag_stream_tests): every scan conjunct must reduce to an int32 range
// and every streamed column must be int32-class; otherwise the generic streaming kernel runs.  reach_pred0: the
// sampled fraction of the rows that pass scan conjunct 0.
static void frag_plan_stream_tests(sr_fragment* f, double reach_pred0) {
    const srd::FragDev& h = f->host;
    const int ns = f->pass.num_stream_joins;
    bool ok = h.num_exprs == 0 && h.num_preds + ns > 0 && h.num_preds + ns <= SR_MAX_STREAM_TESTS;
    int nt = 0;
    auto int32_class = [&](int id) { return srd::type_width(f->reg.types[id]) == 4 && !srd::is_float_class(f->reg.types[id]); };
    for (int p = 0; p < h.num_preds && ok; p++) {
        const srd::CPred& cp = h.preds[p];
        long long lo, hi;
        ok = pred_int32_range(cp, &lo, &hi) && int32_class(cp.value_id);
        if (!ok) break;
        srd::StreamTest& st = f->pass.tests[nt++];
        st.kind = 0;
        st.value_id = cp.value_id;
        st.join = -1;
        st.lo = (uint32_t)(int32_t)lo;
        st.span = (uint32_t)(hi - lo);
    }
    for (int q = 0; q < ns && ok; q++) {
        if (!int32_class(h.joins[q].key_value_id)) {
            ok = false;
            break;
        }
        srd::StreamTest& st = f->pass.tests[nt++];
        st.kind = 1;
        st.value_id = h.joins[q].key_value_id;
        st.join = q;
        st.lo = st.span = 0;
    }
    f->pass.num_tests = ok ? nt : 0;
    // the second test's column is streamed with vector loads as well when >= 8 % of the rows reach it
    // (most of its 64-byte DRAM bursts would be touched anyway, and the loads do not wait for test 0).  HBM does
    // move 64 bytes per access: on H100, reading every other 32-byte sector of a column costs 1.03x reading all of
    // it (scripts/hbm_sector_probe.cu), so fetching this column by the sector for the rows test 0 passed saves nothing
    double reach1 = 1.0;
    if (ok && nt > 1) reach1 = f->pass.tests[0].kind == 0 ? reach_pred0 : f->pred_rate * f->pass_rate[f->order[0]];
    f->pass.num_vec = (ok && nt > 1 && reach1 >= 0.08) ? 2 : 1;
    // the vector-column tests in the form k_frag_stream_tests runs them, with the bitmaps where frag_plan_stream_smem put them
    for (int v = 0; v < 2 && f->pass.num_tests > 0; v++) {
        const srd::StreamTest& st = f->pass.tests[v < f->pass.num_vec ? v : 0];
        srd::VecTest& t = f->pass.vec[v];
        t.kind = st.kind == 0 ? 0 : 3;
        t.lo = st.lo;
        t.span = st.span;
        t.smem_off = -1;
        t.bm = nullptr;
        t.inv = 0;
        t.pad = 0;
        if (st.kind == 1) {
            const srd::FragJoinDev& fj = h.joins[st.join];
            t.inv = fj.kind == srd::FRAG_ANTI ? ~0u : 0u;
            if (fj.use_bitmap && fj.idx32) {
                t.lo = (uint32_t)(int32_t)fj.j.min_value;
                t.span = (uint32_t)(fj.j.max_value - fj.j.min_value);
                if (fj.smem_off >= 0 && t.span != 0xFFFFFFFFu) {
                    t.kind = 1;
                    t.smem_off = fj.smem_off;
                } else {
                    t.kind = 2;
                    t.bm = fj.j.bitmap;
                }
            }
        }
    }
}

// fact values the final pass reads: keys of the joins it looks up or tests, other-join conjunct inputs, group keys,
// aggregate inputs
static void frag_plan_final_vals(sr_fragment* f) {
    const srd::FragDev& h = f->host;
    std::vector<int> need;
    auto want = [&](int id) {
        if (id >= 0 && id < (int)f->value_src.size() && f->value_src[id] < 0 && std::find(need.begin(), need.end(), id) == need.end()) need.push_back(id);
    };
    auto want_expr = [&](const srd::CExpr& e) {
        for (int k = 0; k < e.num_nodes; k++)
            if (e.nodes[k].op == srd::C_LOAD_I || e.nodes[k].op == srd::C_LOAD_D) want(e.nodes[k].arg);
    };
    for (int q = 0; q < f->num_joins; q++) {
        if (h.joins[q].need_head || frag_final_tests(f, q)) want(h.joins[q].key_value_id);
        if ((h.conj_mask >> q) & 1) want_expr(h.conj[q]);
    }
    const srd::AggDev& ah = f->agg->host;
    for (int k = 0; k < ah.num_keys; k++) want(ah.key_value_id[k]);
    for (int q = 0; q < ah.num_fns; q++) want_expr(ah.fns[q].input);
    for (int k = 0; k < SR_FINAL_PREFETCH; k++) f->pass.final_vals[k] = k < (int)need.size() ? (int8_t)need[k] : (int8_t)-1;
    f->pass.num_final_vals = (int8_t)std::min<size_t>(need.size(), 127);
}

// the instantiation of the generic final pass (k_frag_gather_agg) that runs this fragment, and its dynamic shared memory
struct FinalKernel {
    void (*fn)(const srd::FragDev*, const srd::AggDev*, const srd::PassDev, const VTab, const srd::SelEntry*, const unsigned long long*, srd::SelEntry*,
               unsigned long long*);
    size_t smem;
};
template <bool CONJ>
static FinalKernel frag_final_kernel_of(const sr_fragment* f) {
    const bool single = f->agg->host.num_keys == 0;
    if (f->expand) return {single ? srd::k_frag_gather_agg<false, true, true, CONJ> : srd::k_frag_gather_agg<false, false, true, CONJ>, 0};
    if (single) return {srd::k_frag_gather_agg<false, true, false, CONJ>, 0};
    if (f->smem_agg) return {srd::k_frag_gather_agg<true, false, false, CONJ>, f->agg->smem_bytes};
    return {srd::k_frag_gather_agg<false, false, false, CONJ>, 0};
}
static FinalKernel frag_final_kernel(const sr_fragment* f) {
    return f->conj ? frag_final_kernel_of<true>(f) : frag_final_kernel_of<false>(f);
}

// launch grids of the passes (and the dynamic shared-memory limit of the streaming kernels)
static int32_t frag_plan_pass_grids(sr_fragment* f) {
    sr_ctx* ctx = f->ctx;
    const int stream_smem_limit = (int)std::max<size_t>(f->stream_smem, 16);
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_frag_stream<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, stream_smem_limit));
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_frag_stream<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, stream_smem_limit));
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_frag_stream_tests<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, stream_smem_limit));
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_frag_stream_tests<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, stream_smem_limit));
    int per_sm = 0;
    SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, srd::k_frag_stream<false>, srd::FRAG_BLOCK, f->stream_smem));
    if (per_sm < 1) return sr_fail(ctx, SR_ERR_CUDA, "streaming pass does not fit on an SM (smem %zu)", f->stream_smem);
    f->stream_grid = per_sm * ctx->num_sms;
    // gather passes: exactly one wave of resident CTAs (grid-stride loops; a partial second wave only adds a tail)
    int gj = 0, ga = 0;
    SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&gj, srd::k_frag_gather_join, srd::GATHER_BLOCK, 0));
    const FinalKernel fk = frag_final_kernel(f);
    SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ga, fk.fn, srd::GATHER_BLOCK, fk.smem));
    f->gather_grid = std::max(gj, 1) * ctx->num_sms;
    f->final_grid = std::max(ga, 1) * ctx->num_sms;
    return SR_OK;
}

// slots of pass_counters (64-bit words): the entry count of every selection vector a push writes (the streaming pass's,
// then one per gather pass), and the entry count of the input of a hash-table retry of the final pass
constexpr int PASS_CNT_SEL = 0;
constexpr int PASS_CNT_RETRY = 8;
constexpr int PASS_CNT_WORDS = 16;
static_assert(PASS_CNT_SEL + SR_MAX_FRAG_JOINS <= PASS_CNT_RETRY && PASS_CNT_RETRY + 1 <= PASS_CNT_WORDS, "pass counter layout");

// selection-vector mode; reach_pred0: the sampled fraction of the rows that pass scan conjunct 0
static int32_t frag_plan_passes(sr_fragment* f, double reach_pred0) {
    memset(&f->pass, 0, sizeof(f->pass));
    frag_plan_stream_joins(f);
    frag_plan_stream_smem(f);
    frag_plan_stream_tests(f, reach_pred0);
    frag_plan_final_vals(f);
    SR_TRY(frag_plan_pass_grids(f));
    SR_TRY(frag_plan_final_dense(f));
    return f->pass_counters.reserve(f->ctx, PASS_CNT_WORDS * sizeof(uint64_t));
}

// ---- cascade mode (k_fragment) ----
static int32_t frag_plan_cascade(sr_fragment* f) {
    sr_ctx* ctx = f->ctx;
    srd::FragDev& h = f->host;
    // dynamic shared memory: [aggregate accumulators | bitmaps | per-warp queues]
    size_t words = 0;
    if (f->smem_agg) words += (f->agg->smem_bytes + 15) / 16 * 4;
    const size_t budget_words = (96 * 1024) / 4; // keeps 2 CTAs of 512 threads resident per SM
    const size_t queue_words = (size_t)srd::FRAG_WARPS * srd::FRAG_WARP_QWORDS;
    for (int q = 0; q < f->num_joins; q++) {
        srd::FragJoinDev& fj = h.joins[q];
        fj.smem_off = -1;
        if (q < h.num_filter_joins && fj.use_bitmap && words + (size_t)fj.bitmap_words + queue_words <= budget_words) {
            fj.smem_off = (int32_t)words;
            words += (size_t)fj.bitmap_words;
            words = (words + 3) & ~(size_t)3;
        }
    }
    f->queue_word_off = (int32_t)words;
    words += queue_words;
    f->cascade_smem = words * 4;
    // occupancy-sized persistent grid
    int per_sm = 0;
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_fragment<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)f->cascade_smem));
    SR_CUDA(ctx, cudaFuncSetAttribute(srd::k_fragment<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)f->cascade_smem));
    if (f->smem_agg)
        SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, srd::k_fragment<true>, srd::FRAG_BLOCK, f->cascade_smem));
    else
        SR_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, srd::k_fragment<false>, srd::FRAG_BLOCK, f->cascade_smem));
    if (per_sm < 1) return sr_fail(ctx, SR_ERR_CUDA, "fragment kernel does not fit on an SM (smem %zu)", f->cascade_smem);
    f->cascade_grid = per_sm * ctx->num_sms;
    return SR_OK;
}

// sample pass rates, order the joins, choose the mode and plan it, upload
static int32_t frag_plan(sr_fragment* f, const VTab& vt, int64_t n) {
    sr_ctx* ctx = f->ctx;
    srd::FragDev& h = f->host;
    SR_TRY(f->dev.reserve(ctx, sizeof(srd::FragDev)));
    SR_CUDA(ctx, cudaMemcpyAsync(f->dev.p, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    const int64_t sample = std::min<int64_t>(n, 1 << 16);
    unsigned long long counts[srd::SAMPLE_COUNTERS] = {0};
    counts[srd::SAMPLE_ALL_PREDS] = (unsigned long long)sample;
    for (int p = srd::SAMPLE_PREDS_UPTO; p < srd::SAMPLE_COUNTERS; p++) counts[p] = (unsigned long long)sample;
    if (sample > 0 && (f->num_joins > 0 || h.num_preds > 0 || h.num_exprs > 0)) {
        unsigned long long* dcounts = f->counters.as<unsigned long long>() + 8;
        SR_CUDA(ctx, cudaMemsetAsync(dcounts, 0, sizeof(counts), ctx->stream));
        srd::k_frag_sample<<<grid_for(sample, 256), 256, 0, ctx->stream>>>((const srd::FragDev*)f->dev.p, vt, sample, dcounts);
        SR_LAUNCH_CHECK(ctx);
        SR_CUDA(ctx, cudaMemcpyAsync(counts, dcounts, sizeof(counts), cudaMemcpyDeviceToHost, ctx->stream));
        SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    for (int j = 0; j < f->num_joins; j++) f->pass_rate[j] = sample > 0 ? (double)counts[j] / (double)sample : 1.0;
    f->pred_rate = sample > 0 ? (double)counts[srd::SAMPLE_ALL_PREDS] / (double)sample : 1.0;
    std::vector<int> ord(f->num_joins);
    for (int j = 0; j < f->num_joins; j++) ord[j] = j;
    // most selective first; pass rates within 15 % of each other count as a tie -> smaller table first
    // (the first join sees every row: its bitmap should fit shared memory)
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) {
        const double pa = f->pass_rate[a], pb = f->pass_rate[b];
        if (std::abs(pa - pb) > 0.15 * std::max(pa, pb)) return pa < pb;
        return h.joins[a].bitmap_words < h.joins[b].bitmap_words;
    });
    // outer joins filter nothing: they go behind every filtering join
    std::stable_partition(ord.begin(), ord.end(), [&](int j) { return h.joins[j].kind != srd::FRAG_OUTER; });
    srd::FragJoinDev reordered[SR_MAX_FRAG_JOINS];
    srd::CExpr reordered_conj[SR_MAX_FRAG_JOINS];
    int32_t conj_mask = 0;
    std::vector<int> inv(f->num_joins);
    for (int q = 0; q < f->num_joins; q++) {
        reordered[q] = h.joins[ord[q]];
        reordered_conj[q] = h.conj[ord[q]];
        conj_mask |= ((h.conj_mask >> ord[q]) & 1) << q;
        inv[ord[q]] = q;
        f->order[q] = ord[q];
    }
    for (int q = 0; q < f->num_joins; q++) {
        h.joins[q] = reordered[q];
        h.conj[q] = reordered_conj[q];
    }
    h.conj_mask = conj_mask;
    for (size_t k = 0; k < f->value_src.size(); k++)
        if (f->value_src[k] >= 0) f->value_src[k] = inv[f->value_src[k]];
    // stream the second join's key together with the first when most of its 64-byte DRAM bursts would
    // be touched anyway: 1 - (1 - p)^16 >= 0.74 for p >= 0.08
    h.eager1 = (h.num_filter_joins >= 2 && f->pass_rate[ord[0]] >= 0.08) ? 1 : 0;
    // ---- mode: when few rows reach the aggregate, run selection-vector passes instead of the cascade ----
    double total_rate = f->pred_rate;
    for (int q = 0; q < f->num_joins; q++) total_rate *= f->pass_rate[ord[q]];
    f->est_rate = total_rate;
    // (the cascade neither expands a row nor evaluates an other-join conjunct)
    f->selective = f->expand || f->conj || f->force_mode == 2 || (f->force_mode == 0 && total_rate < 0.25 && n >= (1 << 16));
    f->smem_agg = f->agg->smem_bytes > 0;
    if (f->selective)
        SR_TRY(frag_plan_passes(f, (double)counts[srd::SAMPLE_PREDS_UPTO] / (double)std::max<int64_t>(sample, 1)));
    else
        SR_TRY(frag_plan_cascade(f));
    // the kernels read the shared-memory offsets of the bitmaps the mode's plan assigned
    SR_CUDA(ctx, cudaMemcpyAsync(f->dev.p, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    SR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    f->compiled = true;
    return SR_OK;
}

// The final pass of selective mode over the selection vector `in` (its entry count at `in_count`): k_frag_final_dense
// when the push allows it, else the instantiation of k_frag_gather_agg that frag_final_kernel picks.  A hash aggregate is
// neither dense nor kept in shared memory and has group keys, so it always runs k_frag_gather_agg<false, false, EXPAND, CONJ>,
// which appends the rows its table refuses to `fail_list` (counted at `fail_count`).
static int32_t frag_launch_final(sr_fragment* f, const VTab& vt, const srd::SelEntry* in, const unsigned long long* in_count, srd::SelEntry* fail_list,
                                 unsigned long long* fail_count) {
    sr_ctx* ctx = f->ctx;
    sr_agg* a = f->agg;
    const srd::AggDev& ah = a->host;
    const srd::FragDev* fdev = (const srd::FragDev*)f->dev.p;
    const srd::AggDev* adev = (const srd::AggDev*)a->dev.p;
    const srd::PassDev& pass = f->pass;
    // the batched final pass needs plain int32 fact columns and the shared-memory accumulators it was planned for
    // (a push whose aggregate input turned nullable switches the aggregate to global accumulation)
    const bool dense_final = f->final_dense_ok && vt.plain32 && f->smem_agg && a->smem_bytes > 0;
    f->final_pass = dense_final ? SR_FINAL_PASS_DENSE : f->expand ? SR_FINAL_PASS_EXPAND : SR_FINAL_PASS_GENERIC;
    if (dense_final) {
        srd::FinalDense fp = f->final_dense;
        for (int c = 0; c < fp.num_vals; c++) {
            fp.cols[c] = (const int32_t*)vt.v[pass.final_vals[c]].data;
            if (pass.carry_join >= 0 && pass.final_vals[c] == pass.carry_value_id) fp.carry_val = c;
        }
        for (int q = 0; q < fp.num_fns; q++) fp.fn[q].gacc = ah.fns[f->final_fn_src[q]].acc0;
        fp.gcnt = ah.cnt_star;
        fp.flags = ah.flags;
        fp.rows_passed = f->host.rows_passed;
        srd::k_frag_final_dense<srd::FINAL_ROWS><<<f->final_dense_grid, srd::GATHER_BLOCK, a->smem_bytes, ctx->stream>>>(fp, in, in_count);
    } else {
        const FinalKernel fk = frag_final_kernel(f);
        fk.fn<<<f->final_grid, srd::GATHER_BLOCK, fk.smem, ctx->stream>>>(fdev, adev, pass, vt, in, in_count, fail_list, fail_count);
    }
    SR_LAUNCH_CHECK(ctx);
    return SR_OK;
}

static int32_t frag_push(sr_fragment* f, const sr_chunk_view* fact) {
    sr_ctx* ctx = f->ctx;
    if (f->agg->finished) return sr_fail(ctx, SR_ERR_STATE, "fragment push after sink_finish");
    if (fact->num_rows >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fragment batch of more than 2^32 rows; push smaller morsels");
    // page-locked mapped host columns are read in place: the passes after the first only touch the sectors of
    // surviving rows, so most of the batch never crosses PCIe
    SR_TRY(f->staged.stage(ctx, fact, nullptr, /*in_place_pinned=*/true));
    const int64_t n = fact->num_rows;
    bool first = !f->compiled;
    if (first) SR_TRY(frag_compile(f));
    VTab vt;
    SR_TRY(frag_bind_vtab(f, &vt));
    if (first) {
        SR_TRY(frag_plan(f, vt, n));
        SR_TRY(frag_bind_vtab(f, &vt)); // the plan reorders the joins: payload values now point at the new positions
    }
    if (n == 0) return SR_OK;
    SR_TRY(agg_check_nullability(f->agg, vt));
    if (f->agg->smem_bytes == 0 && f->smem_agg) f->smem_agg = false; // a nullability change forced global accumulation
    sr_agg* a = f->agg;
    a->table_touched = true;
    const srd::AggDev& ah = a->host;
    const bool hash = !ah.dense && ah.num_keys > 0;
    if (hash) {
        // Survivors are unknown before the pass.  The single-kernel cascade retries only the rows a full slice refuses, so
        // its table is made large enough for the worst case (every row a new group).  The selection-vector passes size the table
        // from the sampled survivor estimate (x2 + slack) and re-apply the rows the table refused after growing it.
        uint64_t want = (uint64_t)n;
        if (f->selective) want = std::min<uint64_t>((uint64_t)n, (uint64_t)((double)n * std::min(1.0, f->est_rate) * 2.0) + (1u << 16));
        SR_TRY(agg_grow_to_fit(a, want, 4, false));
    }
    if (f->selective) {
        const srd::FragDev* fdev = (const srd::FragDev*)f->dev.p;
        // worst case every row survives, plus one partly used chunk per warp of the writing pass
        const size_t slack = (size_t)srd::SEL_CHUNK * ((size_t)f->stream_grid * (srd::FRAG_BLOCK / 32) + (size_t)f->gather_grid * (srd::GATHER_BLOCK / 32));
        SR_TRY(f->sel[0].reserve(ctx, sizeof(srd::SelEntry) * ((size_t)n + slack)));
        if (!f->gather_joins.empty()) SR_TRY(f->sel[1].reserve(ctx, sizeof(srd::SelEntry) * ((size_t)n + slack)));
        const srd::PassDev& pass = f->pass;
        const bool carry = pass.carry_join >= 0;
        unsigned long long* cnt = f->pass_counters.as<unsigned long long>();
        SR_CUDA(ctx, cudaMemsetAsync(cnt, 0, PASS_CNT_WORDS * sizeof(uint64_t), ctx->stream));
        unsigned long long* sel_count = cnt + PASS_CNT_SEL; // [k]: entries of the selection vector after k gather passes
        const int sgrid = (int)std::min<int64_t>(f->stream_grid, (n + srd::FRAG_TILE - 1) / srd::FRAG_TILE);
        // pass boundaries are bracketed with CUDA events (bench.py reads them back as per-kernel durations)
        if (!f->ev[0])
            for (int e = 0; e < 4; e++) SR_CUDA(ctx, cudaEventCreate(&f->ev[e]));
        SR_CUDA(ctx, cudaEventRecord(f->ev[0], ctx->stream));
        // range-form conjuncts and streamed joins on plain (non-nullable) int32 columns -> the tests kernel;
        // everything else -> the generic streaming kernel
        bool tests = pass.num_tests > 0;
        for (int t = 0; t < pass.num_tests && tests; t++) {
            const VDesc& d = vt.v[pass.tests[t].value_id];
            if (d.nulls != nullptr || (t < pass.num_vec && (((uintptr_t)d.data) & 15) != 0)) tests = false;
        }
        if (tests) {
            if (carry)
                srd::k_frag_stream_tests<true><<<sgrid, srd::FRAG_BLOCK, f->stream_smem, ctx->stream>>>(fdev, pass, vt, n, f->sel[0].as<srd::SelEntry>(), sel_count);
            else
                srd::k_frag_stream_tests<false><<<sgrid, srd::FRAG_BLOCK, f->stream_smem, ctx->stream>>>(fdev, pass, vt, n, f->sel[0].as<srd::SelEntry>(), sel_count);
        } else if (carry) {
            srd::k_frag_stream<true><<<sgrid, srd::FRAG_BLOCK, f->stream_smem, ctx->stream>>>(fdev, pass, vt, n, f->sel[0].as<srd::SelEntry>(), sel_count);
        } else {
            srd::k_frag_stream<false><<<sgrid, srd::FRAG_BLOCK, f->stream_smem, ctx->stream>>>(fdev, pass, vt, n, f->sel[0].as<srd::SelEntry>(), sel_count);
        }
        SR_LAUNCH_CHECK(ctx);
        SR_CUDA(ctx, cudaEventRecord(f->ev[1], ctx->stream));
        int cur = 0, k = 0;
        for (int q : f->gather_joins) {
            srd::k_frag_gather_join<<<f->gather_grid, srd::GATHER_BLOCK, 0, ctx->stream>>>(fdev, q, vt, f->sel[cur].as<srd::SelEntry>(), sel_count + k,
                                                                                         f->sel[cur ^ 1].as<srd::SelEntry>(), sel_count + k + 1);
            SR_LAUNCH_CHECK(ctx);
            cur ^= 1;
            k++;
        }
        SR_CUDA(ctx, cudaEventRecord(f->ev[2], ctx->stream));
        // hash table: entries it refuses go to the other selection buffer (free by now) and are retried after a growth
        unsigned long long* refused = &agg_counters(a)->refused;
        if (hash) {
            SR_TRY(f->sel[cur ^ 1].reserve(ctx, sizeof(srd::SelEntry) * ((size_t)n + slack)));
            SR_CUDA(ctx, cudaMemsetAsync(refused, 0, sizeof(*refused), ctx->stream));
        }
        SR_TRY(frag_launch_final(f, vt, f->sel[cur].as<srd::SelEntry>(), sel_count + k, hash ? f->sel[cur ^ 1].as<srd::SelEntry>() : nullptr, refused));
        SR_CUDA(ctx, cudaEventRecord(f->ev[3], ctx->stream));
        f->timed_push = true;
        if (!hash) return SR_OK;
        // the refused entries become the input and the old input buffer the fail list; the launch runs the kernel of the
        // first one (a hash aggregate's, see frag_launch_final).  The kernels read the input's entry count from the
        // device, where the loop has zeroed the table's count, so it is copied in from the host.
        unsigned long long* retry_count = cnt + PASS_CNT_RETRY;
        return agg_retry_refused(a, [&](uint64_t m) -> int32_t {
            ctx->pinned[16] = m;
            SR_CUDA(ctx, cudaMemcpyAsync(retry_count, ctx->pinned + 16, sizeof(m), cudaMemcpyHostToDevice, ctx->stream));
            cur ^= 1;
            return frag_launch_final(f, vt, f->sel[cur].as<srd::SelEntry>(), retry_count, f->sel[cur ^ 1].as<srd::SelEntry>(), refused);
        });
    }
    // a hash table refuses a row only when its 256-slot slice is full (the table was sized for every row being a new
    // group): the refused fact rows are gathered and run through the cascade again after a growth.  That is exact because
    // the cascade never expands a row (a one-to-many join forces the selection-vector passes), so a refused fact row is
    // one aggregate input that applied nothing, and the same predicates and joins pass it again.
    const auto launch = [&](const VTab& v, int64_t m, uint32_t* fail_rows, unsigned long long* fail_count) -> int32_t {
        const int grid = (int)std::min<int64_t>(f->cascade_grid, (m + srd::FRAG_TILE - 1) / srd::FRAG_TILE);
        if (f->smem_agg)
            srd::k_fragment<true><<<grid, srd::FRAG_BLOCK, f->cascade_smem, ctx->stream>>>((const srd::FragDev*)f->dev.p, (const srd::AggDev*)a->dev.p, v, m,
                                                                                          f->queue_word_off, fail_rows, fail_count);
        else
            srd::k_fragment<false><<<grid, srd::FRAG_BLOCK, f->cascade_smem, ctx->stream>>>((const srd::FragDev*)f->dev.p, (const srd::AggDev*)a->dev.p, v, m,
                                                                                           f->queue_word_off, fail_rows, fail_count);
        SR_LAUNCH_CHECK(ctx);
        return SR_OK;
    };
    if (!hash) return launch(vt, n, nullptr, nullptr);
    return agg_push_rows(a, vt, n, launch);
}

// the fact slots the fragment reads: scan conjuncts, probe keys, other-join conjuncts, group keys and aggregate inputs (a
// slot of the list the fact chunk does not carry is a build column)
static void frag_read_slots(const sr_fragment* f, std::vector<int32_t>* slots) {
    slots->clear();
    for (const sr_pred& p : f->preds) slots->push_back(p.slot_id);
    for (const sr_expr& e : f->exprs) expr_slots(e, slots);
    for (int j = 0; j < f->num_joins; j++) {
        slots->push_back(f->joins[j].probe_key_slot);
        expr_slots(f->joins[j].join->desc.other_conjunct, slots);
    }
    std::vector<int32_t> agg;
    frag_agg_slots(f->agg->desc, &agg);
    slots->insert(slots->end(), agg.begin(), agg.end());
}

// sr_fragment_push_chunks: validate the whole list, gather the columns the fragment reads into one device batch (one
// k_chunk_gather launch for the device and pinned columns, H2D copies for pageable ones), and push that batch
static int32_t frag_push_chunks(sr_fragment* f, const sr_chunk_view* chunks, int32_t num_chunks) {
    sr_ctx* ctx = f->ctx;
    if (num_chunks < 0 || (chunks == nullptr && num_chunks > 0)) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk list of %d chunks at %p", num_chunks, (const void*)chunks);
    if (f->agg->finished) return sr_fail(ctx, SR_ERR_STATE, "fragment push after sink_finish");
    // headers first: the row total is refused before any column is looked at
    int64_t total = 0;
    for (int32_t c = 0; c < num_chunks; c++) {
        SR_TRY(chunk_check(ctx, &chunks[c], c));
        total += chunks[c].num_rows;
        if (total >= 0xFFFFFFF0ll) return sr_fail(ctx, SR_ERR_NOT_SUPPORTED, "fragment batch of more than 2^32 rows; push smaller chunk lists");
    }
    if (num_chunks == 0) {
        if (f->compiled) return SR_OK; // a zero-row push of a planned fragment does nothing
        const sr_chunk_view none{nullptr, 0, SR_MEM_DEVICE, 0};
        return frag_push(f, &none);
    }
    // schema: chunk 0's columns; every chunk carries the same (slot, type) set, in any order.  col_of[c * ncols + k]:
    // chunk c's column of schema column k
    const sr_chunk_view& c0 = chunks[0];
    const int ncols = c0.num_cols;
    std::vector<const sr_col_view*> col_of((size_t)num_chunks * ncols);
    for (int32_t c = 0; c < num_chunks; c++) {
        const sr_chunk_view& ch = chunks[c];
        if (ch.num_cols != ncols) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk %d has %d columns, chunk 0 has %d", c, ch.num_cols, ncols);
        for (int k = 0; k < ncols; k++) {
            const sr_col_view& s = c0.cols[k];
            const sr_col_view* m = (ch.cols[k].slot_id == s.slot_id) ? &ch.cols[k] : find_col(&ch, s.slot_id);
            if (!m || m->type != s.type) return sr_fail(ctx, SR_ERR_INVALID_ARGUMENT, "chunk %d: slot %d missing or of another type than in chunk 0", c, s.slot_id);
            int w;
            SR_TRY(col_check(ctx, *m, ch.num_rows, ch.mem == SR_MEM_DEVICE || (ch.mem == SR_MEM_HOST_PINNED && ch.num_rows > 0), &w, c));
            col_of[(size_t)c * ncols + k] = m;
        }
    }
    std::vector<int32_t> read;
    frag_read_slots(f, &read);
    std::vector<int> moved; // schema columns gathered into the batch
    std::vector<bool> nullable;
    for (int k = 0; k < ncols; k++) {
        if (std::find(read.begin(), read.end(), c0.cols[k].slot_id) == read.end()) continue;
        bool nl = false;
        for (int32_t c = 0; c < num_chunks && !nl; c++) nl = col_of[(size_t)c * ncols + k]->nulls != nullptr;
        moved.push_back(k);
        nullable.push_back(nl);
    }
    // device aliases of the pinned buffers: resolved (and refused) before anything is allocated, copied or launched
    PinnedResolver pinned;
    std::vector<const void*> src((size_t)num_chunks * moved.size() * 2, nullptr); // [c][m][data, nulls]
    for (int32_t c = 0; c < num_chunks; c++) {
        const sr_chunk_view& ch = chunks[c];
        if (ch.num_rows == 0) continue;
        for (size_t m = 0; m < moved.size(); m++) {
            const sr_col_view* col = col_of[(size_t)c * ncols + moved[m]];
            const void** s = &src[((size_t)c * moved.size() + m) * 2];
            s[0] = col->data;
            s[1] = col->nulls;
            if (ch.mem != SR_MEM_HOST_PINNED) continue;
            SR_TRY(pinned.resolve(ctx, col->data, (size_t)ch.num_rows * srd::type_width(col->type), col->slot_id, &s[0]));
            if (col->nulls) SR_TRY(pinned.resolve(ctx, col->nulls, (size_t)ch.num_rows, col->slot_id, &s[1]));
        }
    }
    // the batch: one grow-only (data, nulls) pair per moved column, filled chunk after chunk
    ChunkGather& g = f->chunk_gather;
    g.cols.resize((int)moved.size());
    std::vector<sr_col_view> view(moved.size());
    for (size_t m = 0; m < moved.size(); m++) {
        const sr_col_view& s = c0.cols[moved[m]];
        void* data;
        uint8_t* nulls;
        SR_TRY(g.cols.reserve(ctx, (int)m, total, srd::type_width(s.type), nullable[m], &data, &nulls));
        view[m] = sr_col_view{data, nulls, s.type, s.slot_id};
    }
    std::vector<srd::GatherPiece> pieces;
    int64_t row = 0;
    for (int32_t c = 0; c < num_chunks; c++) {
        const sr_chunk_view& ch = chunks[c];
        const size_t r = (size_t)ch.num_rows;
        if (r == 0) continue;
        for (size_t m = 0; m < moved.size(); m++) {
            const int w = srd::type_width(view[m].type);
            const void* const* s = &src[((size_t)c * moved.size() + m) * 2];
            uint8_t* dst = (uint8_t*)view[m].data + (size_t)row * w;
            uint8_t* dst_nulls = nullable[m] ? (uint8_t*)view[m].nulls + row : nullptr;
            if (ch.mem == SR_MEM_HOST) { // pageable: straight to its place in the batch
                SR_CUDA(ctx, cudaMemcpyAsync(dst, s[0], r * w, cudaMemcpyHostToDevice, ctx->stream));
                if (dst_nulls && s[1]) SR_CUDA(ctx, cudaMemcpyAsync(dst_nulls, s[1], r, cudaMemcpyHostToDevice, ctx->stream));
            } else {
                gather_pieces(&pieces, s[0], dst, r * w);
                if (dst_nulls && s[1]) gather_pieces(&pieces, s[1], dst_nulls, r);
            }
            if (dst_nulls && !s[1]) gather_pieces(&pieces, nullptr, dst_nulls, r);
        }
        row += (int64_t)r;
    }
    SR_TRY(g.launch(ctx, pieces));
    const sr_chunk_view batch{view.data(), (int32_t)view.size(), SR_MEM_DEVICE, total};
    return frag_push(f, &batch);
}
