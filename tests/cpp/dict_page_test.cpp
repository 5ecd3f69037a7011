// CPU-only test of a dictionary-encoded segment column's host side (starrocks_b200/host/exec/global_dict.h): the
// segment's dictionary page (BinaryPlainPage, be/src/storage/rowset/binary_plain_page.h) written and parsed, malformed
// pages rejected, and GlobalDictCodeConverter::global_ids() -- the table sr_page_decoder_set_dict takes to decode the
// segment's data pages into global ids on the device -- against decode_string_dict_codes.  Needs no GPU and does not
// link libsr_gpu.so (sr_type_width is provided below).
#include <cstdio>
#include <cstdlib>
#include <random>

#include "../../starrocks_b200/host/exec/global_dict.h"

// the one libsr_gpu symbol chunk.h refers to (make_column); same table as the library
extern "C" int32_t sr_type_width(int32_t type) {
    switch (type) {
    case SR_TYPE_BOOLEAN:
    case SR_TYPE_TINYINT:
        return 1;
    case SR_TYPE_SMALLINT:
        return 2;
    case SR_TYPE_INT:
    case SR_TYPE_FLOAT:
    case SR_TYPE_DATE:
    case SR_TYPE_DECIMAL32:
        return 4;
    case SR_TYPE_BIGINT:
    case SR_TYPE_DOUBLE:
    case SR_TYPE_DATETIME:
    case SR_TYPE_DECIMAL64:
        return 8;
    case SR_TYPE_LARGEINT:
    case SR_TYPE_DECIMAL128:
        return 16;
    default:
        return 0;
    }
}

using namespace starrocks;

static int g_failed = 0, g_checks = 0;
#define CHECK(cond)                                                                  \
    do {                                                                             \
        g_checks++;                                                                  \
        if (!(cond)) {                                                               \
            g_failed++;                                                              \
            fprintf(stderr, "%s:%d: CHECK(%s) failed\n", __FILE__, __LINE__, #cond); \
        }                                                                            \
    } while (0)
#define CHECK_EQ(a, b) CHECK((a) == (b))

static std::vector<uint8_t> le32s(std::initializer_list<uint32_t> vs) {
    std::vector<uint8_t> out;
    for (uint32_t v : vs)
        for (int k = 0; k < 4; k++) out.push_back((uint8_t)(v >> (8 * k)));
    return out;
}

static bool same_words(const BinaryColumn& a, const BinaryColumn& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); i++)
        if (a.get_slice(i) != b.get_slice(i)) return false;
    return true;
}

static void test_page_bytes() {
    // "AMERICA", "", "ASIA": the bytes back to back, offsets 0 7 7, count 3
    BinaryColumn words;
    for (const char* w : {"AMERICA", "", "ASIA"}) words.append_string(w);
    const std::vector<uint8_t> page = encode_binary_plain_page(words);
    std::vector<uint8_t> want{'A', 'M', 'E', 'R', 'I', 'C', 'A', 'A', 'S', 'I', 'A'};
    const auto tail = le32s({0, 7, 7, 3});
    want.insert(want.end(), tail.begin(), tail.end());
    CHECK(page == want);
    BinaryColumn back;
    CHECK(decode_binary_plain_page(page.data(), page.size(), &back).ok());
    CHECK(same_words(back, words));
    // an empty dictionary is the count alone
    BinaryColumn none;
    const auto empty = encode_binary_plain_page(none);
    CHECK(empty == le32s({0}));
    CHECK(decode_binary_plain_page(empty.data(), empty.size(), &back).ok() && back.size() == 0);
}

static void test_round_trip() {
    std::mt19937 rng(7);
    for (size_t n : {1u, 2u, 25u, 256u, 70000u}) {
        BinaryColumn words;
        for (size_t i = 0; i < n; i++) {
            std::string w;
            const size_t len = rng() % 13; // empty words too
            for (size_t k = 0; k < len; k++) w.push_back((char)(rng() & 0xFF));
            words.append_string(w);
        }
        const auto page = encode_binary_plain_page(words);
        CHECK_EQ(page.size(), words.get_bytes().size() + 4 * n + 4);
        BinaryColumn back;
        CHECK(decode_binary_plain_page(page.data(), page.size(), &back).ok());
        CHECK(same_words(back, words));
    }
}

static void test_malformed_pages() {
    BinaryColumn words;
    for (const char* w : {"MFGR#1", "MFGR#22", "MFGR#3"}) words.append_string(w);
    const auto good = encode_binary_plain_page(words); // 19 bytes of words, offsets 0 6 13, count 3
    BinaryColumn out;
    CHECK(!decode_binary_plain_page(good.data(), 3, &out).ok()); // shorter than the count
    auto bad = good;
    bad[bad.size() - 4] = 9; // 9 words: 36 bytes of offsets do not fit in 31
    CHECK(!decode_binary_plain_page(bad.data(), bad.size(), &out).ok());
    bad = good;
    bad[bad.size() - 1] = 0x40; // a count of 2^30 + 3
    CHECK(!decode_binary_plain_page(bad.data(), bad.size(), &out).ok());
    bad = good;
    bad[19 + 4] = 14; // offsets 0 14 13: decreasing
    CHECK(!decode_binary_plain_page(bad.data(), bad.size(), &out).ok());
    bad = good;
    bad[19 + 8] = 20; // the last word would start past the offset array (at 20 of 19)
    CHECK(!decode_binary_plain_page(bad.data(), bad.size(), &out).ok());
    bad = good;
    bad[19 + 8] = 19; // ... starting exactly at it is an empty last word
    CHECK(decode_binary_plain_page(bad.data(), bad.size(), &out).ok() && out.size() == 3 && out.get_slice(2).size == 0);
    CHECK(decode_binary_plain_page(good.data(), good.size(), &out).ok() && same_words(out, words));
}

static void test_global_ids_against_decode_string_dict_codes() {
    const std::vector<std::string> regions{"AMERICA", "ASIA", "AFRICA", "EUROPE", "MIDDLE EAST"};
    GlobalDictLists lists{make_sorted_global_dict(/*columnId=*/7, regions)};
    FragmentDictState dict_state;
    CHECK(dict_state.init_query_global_dict(lists).ok());
    const auto& global = dict_state.query_global_dicts().at(7).first;
    std::mt19937 rng(11);
    for (int segment = 0; segment < 3; segment++) {
        const size_t n = 2000 + 777 * segment;
        BinaryColumn column;
        for (size_t i = 0; i < n; i++) column.append_string(segment == 2 && i % 9 == 0 ? "" : regions[rng() % (segment ? 5 : 2)]);
        BinaryColumn local_words;
        std::vector<int32_t> codes;
        encode_local_dict(column, &local_words, &codes);
        // the segment's dictionary page survives the write / parse, and the table is built from the parsed words
        const auto page = encode_binary_plain_page(local_words);
        BinaryColumn parsed;
        CHECK(decode_binary_plain_page(page.data(), page.size(), &parsed).ok() && same_words(parsed, local_words));
        GlobalDictCodeConverter conv;
        CHECK(conv.build_code_convert_map(parsed, global).ok()); // segment 2's empty word is tolerated: id 0
        const std::vector<int32_t> table = conv.global_ids();
        CHECK_EQ(table.size(), local_words.size());
        auto ids = conv.decode_string_dict_codes(codes.data(), nullptr, n);
        bool same = true;
        for (size_t i = 0; i < n; i++) same = same && ids->get_data()[i] == table[codes[i]];
        CHECK(same);
        for (size_t k = 0; k < table.size(); k++) {
            const Slice w = local_words.get_slice(k);
            CHECK_EQ(table[k], w.size ? global.at(w) : 0);
        }
    }
    CHECK(GlobalDictCodeConverter().global_ids().empty());
}

int main() {
    test_page_bytes();
    test_round_trip();
    test_malformed_pages();
    test_global_ids_against_decode_string_dict_codes();
    if (g_failed) {
        fprintf(stderr, "DICT_PAGE_TEST_FAILED %d of %d checks\n", g_failed, g_checks);
        return 1;
    }
    printf("DICT_PAGE_TEST_OK %d checks\n", g_checks);
    return 0;
}
