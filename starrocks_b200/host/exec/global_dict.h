// The low-cardinality global dictionary around the GPU operators: strings are replaced by int32 dictionary ids below
// the DictDecodeOperator, so scan / filter / join / aggregate (the GPU path) only ever see TYPE_INT columns.
// Mirrors, on the host:
//   be/src/runtime/global_dict/config.h:22-25              DictId, LowCardDictType, DICT_DECODE_MAX_SIZE
//   be/src/runtime/global_dict/types_fwd_decl.h:27-47      GlobalDictMap / RGlobalDictMap / GlobalDictMaps
//   be/src/runtime/global_dict/fragment_dict_state.cpp:44-67   the maps built from the plan's (strings, ids) lists
//   be/src/storage/rowset/dictcode_column_iterator.cpp:53-128  segment-local codes -> global ids (the scan side)
//   be/src/runtime/global_dict/decoder.cpp:104-176         GlobalDictDecoder::decode_string
//   be/src/storage/rowset/binary_plain_page.h              BinaryPlainPageBuilder / Decoder: a segment's dictionary page
//   be/src/exec/pipeline/dict_decode_operator.{h,cpp}      DictDecodeOperator / DictDecodeOperatorFactory
// Host-only: no kernel is involved; the id columns these classes produce are what make_chunk_view hands to libsr_gpu.
#pragma once

#include <map>
#include <unordered_map>

#include "../column/binary_column.h"
#include "pipeline/operator.h"

namespace starrocks {

using DictId = int32_t;
constexpr int32_t LowCardDictType = SR_TYPE_INT;
constexpr int DICT_DECODE_MAX_SIZE = 256;

struct SliceHash {
    size_t operator()(const Slice& s) const { // FNV-1a 64; any hash does, ids come from the plan
        uint64_t h = 0xcbf29ce484222325ull;
        for (size_t i = 0; i < s.size; i++) h = (h ^ (uint8_t)s.data[i]) * 0x100000001b3ull;
        return (size_t)h;
    }
};
using GlobalDictMap = std::unordered_map<Slice, DictId, SliceHash>;
using RGlobalDictMap = std::unordered_map<DictId, Slice>;
using GlobalDictMapEntity = std::pair<GlobalDictMap, RGlobalDictMap>;
using GlobalDictMaps = std::unordered_map<uint32_t, GlobalDictMapEntity>; // column / slot id -> maps

// TGlobalDict of the plan fragment (gensrc/thrift/InternalService.thrift): the FE ships the words and their ids
struct TGlobalDict {
    int32_t columnId = 0;
    std::vector<std::string> strings;
    std::vector<int32_t> ids;
    int64_t version = 0;
};
using GlobalDictLists = std::vector<TGlobalDict>;

// FragmentDictState: owns the words (the reference copies them into the instance MemPool) and the two maps per column
class FragmentDictState {
public:
    Status init_query_global_dict(const GlobalDictLists& lists) {
        for (const auto& d : lists) {
            if (d.ids.size() != d.strings.size()) return Status::InvalidArgument("global dict: ids and strings differ in length");
            if (d.ids.size() > (size_t)DICT_DECODE_MAX_SIZE) return Status::InvalidArgument("global dict: more than DICT_DECODE_MAX_SIZE words");
            auto words = std::make_unique<BinaryColumn>();
            for (const auto& s : d.strings) words->append_string(s);
            GlobalDictMap dict;
            RGlobalDictMap rdict;
            for (size_t i = 0; i < d.ids.size(); i++) {
                const Slice w = words->get_slice(i); // stable: the column is not touched again
                dict.emplace(w, d.ids[i]);
                rdict.emplace(d.ids[i], w);
            }
            _pool.push_back(std::move(words));
            _query_global_dicts.emplace((uint32_t)d.columnId, std::make_pair(std::move(dict), std::move(rdict)));
            _versions[(uint32_t)d.columnId] = d.version;
        }
        return Status::OK();
    }
    const GlobalDictMaps& query_global_dicts() const { return _query_global_dicts; }
    GlobalDictMaps* mutable_query_global_dicts() { return &_query_global_dicts; }

private:
    std::vector<std::unique_ptr<BinaryColumn>> _pool;
    GlobalDictMaps _query_global_dicts;
    std::unordered_map<uint32_t, int64_t> _versions;
};

// What the FE's dictionary collection produces for one column: the distinct words in byte order, ids 1..n (0 is what a
// NULL row carries, dictcode_column_iterator.cpp:84-90).  Used by the tests and the benchmark data generator.
inline TGlobalDict make_sorted_global_dict(int32_t column_id, std::vector<std::string> words) {
    std::sort(words.begin(), words.end(), [](const std::string& a, const std::string& b) { return Slice(a).compare(Slice(b)) < 0; });
    words.erase(std::unique(words.begin(), words.end()), words.end());
    TGlobalDict d;
    d.columnId = column_id;
    for (size_t i = 0; i < words.size(); i++) d.ids.push_back((int32_t)i + 1);
    d.strings = std::move(words);
    return d;
}

// Scan side (GlobalDictCodeColumnIterator): a dictionary-encoded segment column stores LOCAL codes (position of the word
// in the segment's dictionary page, -1 for NULL); they are translated with a table that also answers index -1.
class GlobalDictCodeConverter {
public:
    // build_code_convert_map: table[local + 1] = global id of the local word; an unknown non-empty word is an error
    Status build_code_convert_map(const BinaryColumn& local_dict_words, const GlobalDictMap& global_dict) {
        const size_t n = local_dict_words.size();
        _table.assign(n + 2, 0);
        int16_t* local_to_global = _table.data() + 1;
        for (size_t i = 0; i < n; i++) {
            const Slice w = local_dict_words.get_slice(i);
            auto it = global_dict.find(w);
            if (it == global_dict.end()) {
                if (w.size > 0) return Status::InternalError("not found slice:" + w.to_string() + " in global dict");
            } else {
                local_to_global[i] = (int16_t)it->second;
            }
        }
        _dict_size = (int)n;
        return Status::OK();
    }
    // decode_string_dict_codes: local codes (+ the null bytes of a nullable column) -> a TYPE_INT column of global ids,
    // 0 in NULL rows.  This column is what the GPU operators scan, filter, join and group on.
    std::shared_ptr<Int32Column> decode_string_dict_codes(const int32_t* codes, const uint8_t* nulls, size_t n) const {
        auto out = std::make_shared<Int32Column>(LowCardDictType);
        out->resize(n);
        int32_t* res = out->get_data().data();
        const int16_t* local_to_global = _table.data() + 1;
        for (size_t i = 0; i < n; i++) {
            const int32_t c = codes[i];
            res[i] = (nulls && nulls[i]) || c < -1 || c >= _dict_size ? 0 : local_to_global[c];
        }
        return out;
    }
    int dict_size() const { return _dict_size; }
    // the table in code order (without the slot of index -1): global_ids()[k] is the global id of local word k.  What
    // sr_page_decoder_set_dict takes to decode this segment's dictionary data pages into ids on the device.
    std::vector<int32_t> global_ids() const {
        if (_table.empty()) return {};
        return std::vector<int32_t>(_table.begin() + 1, _table.begin() + 1 + _dict_size);
    }

private:
    std::vector<int16_t> _table;
    int _dict_size = 0;
};

// A dictionary-encoded segment column in miniature: the distinct words of `column` in first-seen order and one local code
// per row (what BinaryDictPageBuilder leaves in a segment).  Test / benchmark helper.
inline void encode_local_dict(const BinaryColumn& column, BinaryColumn* local_words, std::vector<int32_t>* codes) {
    std::unordered_map<Slice, int32_t, SliceHash> seen;
    std::vector<std::string> order;
    codes->resize(column.size());
    for (size_t i = 0; i < column.size(); i++) {
        const Slice s = column.get_slice(i);
        auto it = seen.find(s);
        if (it == seen.end()) {
            it = seen.emplace(s, (int32_t)order.size()).first; // keys point into `column`, which outlives the map
            order.push_back(s.to_string());
        }
        (*codes)[i] = it->second;
    }
    local_words->reset_column();
    for (const auto& w : order) local_words->append_string(w);
}

// A segment's dictionary page (BinaryPlainPage): the words' bytes back to back, one uint32 LE start offset per word, then
// the uint32 LE word count.  Word i runs from offset[i] to offset[i + 1], the last word to the start of the offset array.
// The parse of BinaryPlainPageDecoder::init, rejecting a count that does not fit the page and offsets that decrease or
// pass the offset array.
inline Status decode_binary_plain_page(const uint8_t* data, size_t size, BinaryColumn* words) {
    if (size < 4) return Status::InvalidArgument("binary plain page: shorter than its word count");
    uint32_t n = 0;
    memcpy(&n, data + size - 4, 4);
    if ((size - 4) / 4 < n) return Status::InvalidArgument("binary plain page: " + std::to_string(n) + " words do not fit");
    const size_t start = size - 4 - 4 * (size_t)n;
    if (start > 0xFFFFFFFFull) return Status::InvalidArgument("binary plain page: more than 4 GiB of words");
    std::vector<uint32_t> offs(n + 1);
    if (n) memcpy(offs.data(), data + start, 4 * (size_t)n);
    offs[n] = (uint32_t)start;
    for (uint32_t i = 0; i < n; i++)
        if (offs[i] > offs[i + 1]) return Status::InvalidArgument("binary plain page: word offsets decrease or pass the offset array");
    words->reset_column();
    for (uint32_t i = 0; i < n; i++) words->append(Slice(data + offs[i], offs[i + 1] - offs[i]));
    return Status::OK();
}

// BinaryPlainPageBuilder::finish of `words` (e.g. encode_local_dict's): the dictionary page a segment stores.  Test /
// benchmark helper.
inline std::vector<uint8_t> encode_binary_plain_page(const BinaryColumn& words) {
    const auto& bytes = words.get_bytes();
    std::vector<uint8_t> page(bytes.begin(), bytes.end());
    auto put32 = [&page](uint32_t v) {
        for (int k = 0; k < 4; k++) page.push_back((uint8_t)(v >> (8 * k)));
    };
    for (size_t i = 0; i < words.size(); i++) put32(words.get_offset()[i]);
    put32((uint32_t)words.size());
    return page;
}

// GlobalDictDecoder::decode_string for a plain or nullable TYPE_INT id column -> BinaryColumn / Nullable(BinaryColumn)
class GlobalDictDecoder {
public:
    explicit GlobalDictDecoder(RGlobalDictMap dict) : _dict(std::move(dict)) {}
    StatusOr<ColumnPtr> decode_string(const Column& in) const {
        if (in.logical_type() != LowCardDictType) return Status::InternalError("Dict Decode failed, the encoded column is not TYPE_INT");
        const size_t n = in.size();
        const int32_t* ids = reinterpret_cast<const int32_t*>(in.raw_data());
        const uint8_t* nulls = in.null_data();
        std::vector<Slice> words(n); // NULL rows keep the empty slice
        for (size_t i = 0; i < n; i++) {
            if (nulls && nulls[i]) continue;
            auto it = _dict.find(ids[i]);
            if (it == _dict.end()) return Status::InternalError("Dict Decode failed, Dict can't take cover all key :" + std::to_string(ids[i]));
            words[i] = it->second;
        }
        auto out = BinaryColumn::create();
        out->append_strings(words.data(), n);
        if (!in.is_nullable()) return ColumnPtr(out);
        auto out_nulls = std::make_shared<NullColumn>(SR_TYPE_BOOLEAN);
        out_nulls->resize(n);
        if (n) memcpy(out_nulls->mutable_raw_data(), nulls, n);
        return ColumnPtr(std::make_shared<NullableColumn>(out, out_nulls));
    }

private:
    RGlobalDictMap _dict;
};
using GlobalDictDecoderPtr = std::shared_ptr<GlobalDictDecoder>;
inline GlobalDictDecoderPtr create_global_dict_decoder(const RGlobalDictMap& dict) { return std::make_shared<GlobalDictDecoder>(dict); }

namespace pipeline {

// DictDecodeOperator: sits above the last operator that works on ids (here: above the GPU aggregate source) and swaps
// each encoded column for its strings, keeping the chunk's column order.
class DictDecodeOperator final : public Operator {
public:
    DictDecodeOperator(OperatorFactory* factory, int32_t id, int32_t plan_node_id, int32_t driver_sequence, const std::vector<int32_t>& encode_column_cids,
                       const std::vector<int32_t>& decode_column_cids, const std::vector<GlobalDictDecoderPtr>& decoders)
            : Operator(factory, id, "dict_decode", plan_node_id, false, driver_sequence),
              _encode_column_cids(encode_column_cids),
              _decode_column_cids(decode_column_cids),
              _decoders(decoders) {}

    bool has_output() const override { return _cur_chunk != nullptr; }
    bool need_input() const override { return !_is_finished && _cur_chunk == nullptr; }
    bool is_finished() const override { return _is_finished && _cur_chunk == nullptr; }
    Status set_finishing(RuntimeState* state) override {
        _is_finished = true;
        return Status::OK();
    }
    void close(RuntimeState* state) override { _cur_chunk.reset(); }
    StatusOr<ChunkPtr> pull_chunk(RuntimeState* state) override { return std::move(_cur_chunk); }

    Status push_chunk(RuntimeState* state, const ChunkPtr& chunk) override {
        auto out = std::make_shared<Chunk>();
        for (size_t c = 0; c < chunk->num_columns(); c++) { // original column order
            const SlotId slot = chunk->slot_of_index(c);
            const auto it = std::find(_encode_column_cids.begin(), _encode_column_cids.end(), slot);
            if (it == _encode_column_cids.end()) {
                out->append_column(chunk->get_column_by_index(c), slot);
                continue;
            }
            const size_t i = it - _encode_column_cids.begin();
            auto decoded = _decoders[i]->decode_string(*chunk->get_column_by_index(c));
            if (!decoded.ok()) return decoded.status();
            out->append_column(std::move(decoded.value()), _decode_column_cids[i]);
        }
        for (int32_t cid : _encode_column_cids)
            if (!chunk->is_slot_exist(cid)) return Status::InternalError("dict_decode: the chunk has no column for cid:" + std::to_string(cid));
        _cur_chunk = std::move(out);
        return Status::OK();
    }
    Status reset_state(RuntimeState* state, const std::vector<ChunkPtr>& refill_chunks) override {
        _cur_chunk = nullptr;
        _is_finished = false;
        return Status::OK();
    }

private:
    const std::vector<int32_t>& _encode_column_cids;
    const std::vector<int32_t>& _decode_column_cids;
    const std::vector<GlobalDictDecoderPtr>& _decoders;
    bool _is_finished = false;
    ChunkPtr _cur_chunk = nullptr;
};

class DictDecodeOperatorFactory final : public OperatorFactory {
public:
    DictDecodeOperatorFactory(int32_t id, int32_t plan_node_id, std::vector<int32_t> encode_column_cids, std::vector<int32_t> decode_column_cids,
                              const FragmentDictState* dict_state)
            : OperatorFactory(id, "dict_decode", plan_node_id),
              _encode_column_cids(std::move(encode_column_cids)),
              _decode_column_cids(std::move(decode_column_cids)),
              _dict_state(dict_state) {}

    // one decoder per encoded column, from the fragment's dictionaries; a column without one fails the plan here
    Status prepare(RuntimeState* state) override {
        if (_encode_column_cids.size() != _decode_column_cids.size()) return Status::InvalidArgument("dict_decode: cid lists differ in length");
        const auto& dicts = _dict_state->query_global_dicts();
        _decoders.clear();
        for (int32_t cid : _encode_column_cids) {
            auto it = dicts.find((uint32_t)cid);
            if (it == dicts.end()) return Status::InternalError("Not found dict for cid:" + std::to_string(cid));
            _decoders.push_back(create_global_dict_decoder(it->second.second));
        }
        return Status::OK();
    }
    OperatorPtr create(int32_t degree_of_parallelism, int32_t driver_sequence) override {
        return std::make_shared<DictDecodeOperator>(this, _id, _plan_node_id, driver_sequence, _encode_column_cids, _decode_column_cids, _decoders);
    }

private:
    std::vector<int32_t> _encode_column_cids;
    std::vector<int32_t> _decode_column_cids;
    std::vector<GlobalDictDecoderPtr> _decoders;
    const FragmentDictState* _dict_state;
};

} // namespace pipeline
} // namespace starrocks
