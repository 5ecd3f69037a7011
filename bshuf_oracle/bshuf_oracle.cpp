// bshuf_oracle.cpp -- CPU restatement of the BIT_SHUFFLE page codec (bitshuffle + LZ4).  TEST INFRASTRUCTURE ONLY: the
// reference the device decoder (starrocks_b200/csrc/sr_page.cuh) is checked against, and the encoder that writes the test
// and benchmark pages.
//
// Page body (BitshufflePageBuilder::finish, be/src/storage/rowset/bitshuffle_page.h), after page_io has stripped the
// footer, checksum and null map:
//   header: four little-endian uint32 -- num_elements, compressed_size (the whole page, header included),
//           num_elements_after_padding = ALIGN_UP(num_elements, 8) (the padding elements are zeros), elem_size_bytes
//   body:   bitshuffle::compress_lz4(data, out, padded, elem_size, block_size = 0): blocks of
//           bshuf_default_block_size(s) = max(128, (8192 / s) / 8 * 8) elements (8192 bytes each for s = 1..16), the last
//           one holding padded % block elements when that is non-zero; each block is a BIG-endian uint32 compressed length
//           followed by an LZ4 block-format stream of the bit-transposed block.
//   bit transpose (bshuf_trans_bit_elem) of n elements of s bytes: 8 * s rows of n / 8 bytes; row 8 * j + k holds bit k of
//   byte j of every element, element i at bit i % 8 of byte i / 8 (LSB first).
//
// LZ4 block format, with the end-of-block rules LZ4_decompress_safe applies when the decoded size must equal the block's
// (bshuf_decompress_lz4_block checks the returned size):
//   sequence = token (literal length << 4 | match length - 4; a nibble of 15 continues in bytes, 255 = more follow),
//   literals, then -- unless the input ends right after the literals -- a little-endian uint16 offset (1..position) and
//   the match.  The last sequence is literals only and ends exactly at the end of the input; a match starts at least 12
//   bytes before the end of the output (MFLIMIT) and ends at least 5 bytes before it (LASTLITERALS).  Matches may overlap
//   their own output (offset < length).
//   liblz4 1.9.4 has one shortcut that skips the LASTLITERALS test: a sequence with fewer than 15 literals, a match of at
//   most 18 bytes with offset >= 8, starting within 64 bytes but not within 32 bytes of the end of the output.  Such a
//   stream (never produced by an LZ4 compressor) is rejected here and on the device.
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <vector>

namespace {

constexpr int64_t kMaxBlockBytes = 8192;
constexpr int64_t kMaxCompressedBlock = 8240; // LZ4_compressBound(8192)

inline uint32_t rd32(const uint8_t* p) {
    uint32_t v;
    memcpy(&v, p, 4);
    return v;
}

// 8 x 8 bit matrix transpose: bit k of byte t <-> bit t of byte k (TRANS_BIT_8X8 of the bitshuffle sources)
inline uint64_t trans8x8(uint64_t x) {
    uint64_t t;
    t = (x ^ (x >> 7)) & 0x00AA00AA00AA00AAULL;
    x = x ^ t ^ (t << 7);
    t = (x ^ (x >> 14)) & 0x0000CCCC0000CCCCULL;
    x = x ^ t ^ (t << 14);
    t = (x ^ (x >> 28)) & 0x00000000F0F0F0F0ULL;
    x = x ^ t ^ (t << 28);
    return x;
}

int64_t block_elems(int32_t s) {
    const int64_t b = (kMaxBlockBytes / s) / 8 * 8;
    return b < 128 ? 128 : b;
}

void put_len(std::vector<uint8_t>& o, int64_t v) {
    for (; v >= 255; v -= 255) o.push_back(255);
    o.push_back((uint8_t)v);
}

void put_seq(std::vector<uint8_t>& o, const uint8_t* lit, int64_t nlit, int64_t off, int64_t ml) {
    const int64_t mcode = ml - 4;
    o.push_back((uint8_t)((nlit < 15 ? nlit : 15) << 4 | (off ? (mcode < 15 ? mcode : 15) : 0)));
    if (nlit >= 15) put_len(o, nlit - 15);
    o.insert(o.end(), lit, lit + nlit);
    if (!off) return;
    o.push_back((uint8_t)(off & 255));
    o.push_back((uint8_t)(off >> 8));
    if (mcode >= 15) put_len(o, mcode - 15);
}

// greedy single-probe hash-table matcher (the shape of LZ4_compress_default, without its acceleration and back-extension)
std::vector<uint8_t> lz4_compress(const uint8_t* src, int64_t n) {
    std::vector<uint8_t> o;
    int64_t anchor = 0;
    if (n >= 13) {
        std::vector<int32_t> table(4096, -1);
        const int64_t mflimit = n - 12, matchlimit = n - 5;
        auto hash = [&](int64_t p) { return (rd32(src + p) * 2654435761u) >> 20; };
        int64_t ip = 0;
        while (ip <= mflimit) {
            const uint32_t h = hash(ip);
            const int64_t ref = table[h];
            table[h] = (int32_t)ip;
            if (ref >= 0 && ip - ref <= 65535 && rd32(src + ref) == rd32(src + ip)) {
                int64_t ml = 4;
                while (ip + ml < matchlimit && src[ref + ml] == src[ip + ml]) ml++;
                put_seq(o, src + anchor, ip - anchor, ip - ref, ml);
                ip += ml;
                anchor = ip;
                if (ip - 2 <= n - 4) table[hash(ip - 2)] = (int32_t)(ip - 2);
            } else {
                ip++;
            }
        }
    }
    put_seq(o, src + anchor, n - anchor, 0, 0);
    return o;
}

// a length nibble of 15 continued in bytes; stops early (the caller then rejects) once it passes `limit`
int64_t read_len(const uint8_t* src, int64_t n, int64_t* ip, int64_t v, int64_t limit) {
    uint8_t b;
    do {
        if (*ip >= n) return -1;
        b = src[(*ip)++];
        v += b;
    } while (b == 255 && v <= limit);
    return v;
}

// -> expect, or -1 when the stream is malformed or does not decode to exactly `expect` bytes
int64_t lz4_decompress(const uint8_t* src, int64_t n, uint8_t* dst, int64_t expect) {
    int64_t ip = 0, op = 0;
    for (;;) {
        if (ip >= n) return -1;
        const uint8_t tok = src[ip++];
        int64_t lit = tok >> 4;
        if (lit == 15 && (lit = read_len(src, n, &ip, lit, n)) < 0) return -1;
        if (lit > n - ip || lit > expect - op) return -1;
        memcpy(dst + op, src + ip, (size_t)lit);
        ip += lit;
        op += lit;
        if (ip == n) return op == expect ? expect : -1;
        if (op > expect - 12 || n - ip < 2) return -1;
        const int64_t off = src[ip] | src[ip + 1] << 8;
        ip += 2;
        if (off == 0 || off > op) return -1;
        int64_t ml = tok & 15;
        if (ml == 15 && (ml = read_len(src, n, &ip, ml, expect)) < 0) return -1;
        ml += 4;
        if (ml > expect - 5 - op) return -1;
        for (int64_t k = 0; k < ml; k++) dst[op + k] = dst[op - off + k];
        op += ml;
    }
}

void trans_bit_elem(const uint8_t* in, uint8_t* out, int64_t n, int32_t s) {
    const int64_t rb = n / 8;
    for (int64_t g = 0; g < rb; g++)
        for (int32_t j = 0; j < s; j++) {
            uint64_t x = 0;
            for (int t = 0; t < 8; t++) x |= (uint64_t)in[(8 * g + t) * s + j] << (8 * t);
            x = trans8x8(x);
            for (int k = 0; k < 8; k++) out[(8 * j + k) * rb + g] = (uint8_t)(x >> (8 * k));
        }
}

void untrans_bit_elem(const uint8_t* in, uint8_t* out, int64_t n, int32_t s) {
    const int64_t rb = n / 8;
    for (int64_t g = 0; g < rb; g++)
        for (int32_t j = 0; j < s; j++) {
            uint64_t x = 0;
            for (int k = 0; k < 8; k++) x |= (uint64_t)in[(8 * j + k) * rb + g] << (8 * k);
            x = trans8x8(x);
            for (int t = 0; t < 8; t++) out[(8 * g + t) * s + j] = (uint8_t)(x >> (8 * t));
        }
}

bool width_ok(int32_t s) { return s == 1 || s == 2 || s == 4 || s == 8 || s == 16; }

void put_le32(uint8_t* p, uint32_t v) {
    for (int k = 0; k < 4; k++) p[k] = (uint8_t)(v >> (8 * k));
}

// RleEncoder<T> at bit width 1 (be/src/util/rle_encoding.h, the Kudu / Impala hybrid encoder): values are buffered in
// groups of 8; 8 equal values in a row turn into a repeated run (ULEB128 header count << 1, then the value in one byte) that
// lasts until the value changes; other groups go out bit-packed (one byte per group, least significant bit first) under a
// one-byte header (groups << 1 | 1) reserved in front of them, a new one once 63 groups are written.  Flush writes what is
// pending as a repeated run when it is all one value, else as a last literal group padded with zeros.
struct RleEncoder1 {
    std::vector<uint8_t> out;
    uint8_t buf[8] = {0};
    int nbuf = 0;
    int64_t literal_count = 0, indicator = -1, repeat = 0;
    uint8_t cur = 0;

    void put_vlq(uint64_t v) {
        while (v >= 0x80) {
            out.push_back((uint8_t)(v | 0x80));
            v >>= 7;
        }
        out.push_back((uint8_t)v);
    }
    void flush_literal(bool update) {
        if (indicator < 0) {
            indicator = (int64_t)out.size();
            out.push_back(0);
        }
        if (nbuf > 0) {
            uint8_t b = 0;
            for (int i = 0; i < nbuf; i++) b |= (uint8_t)(buf[i] << i);
            out.push_back(b);
        }
        nbuf = 0;
        if (update) {
            out[(size_t)indicator] = (uint8_t)(((literal_count + 7) / 8) << 1 | 1);
            indicator = -1;
            literal_count = 0;
        }
    }
    void flush_repeated() {
        put_vlq((uint64_t)repeat << 1);
        out.push_back(cur);
        nbuf = 0;
        repeat = 0;
    }
    void flush_buffered() {
        if (repeat >= 8) { // the buffered values belong to the repeated run
            nbuf = 0;
            if (literal_count != 0) flush_literal(true);
            return;
        }
        literal_count += nbuf;
        flush_literal((literal_count + 7) / 8 + 1 >= (1 << 6));
        repeat = 0;
    }
    void put(uint8_t v) {
        if (v == cur) {
            if (++repeat > 8) return;
        } else {
            if (repeat >= 8) flush_repeated();
            repeat = 1;
            cur = v;
        }
        buf[nbuf] = v;
        if (++nbuf == 8) flush_buffered();
    }
    void flush() {
        if (literal_count > 0 || repeat > 0 || nbuf > 0) {
            const bool all_repeat = literal_count == 0 && (repeat == nbuf || nbuf == 0);
            if (repeat > 0 && all_repeat) {
                flush_repeated();
            } else {
                literal_count += nbuf;
                flush_literal(true);
                repeat = 0;
            }
        }
    }
};

// n values of an RLE stream at bit width 1 -> out; false for a malformed stream.  Stops at the count (RleDecoder reads
// no further): refuses a header longer than 5 bytes or cut off, a zero-length run, a repeated value other than 0 / 1, a
// run whose values up to the count lie past the end, and a stream that ends before the count.
bool rle_decode1(const uint8_t* in, int64_t len, int64_t n, uint8_t* out) {
    int64_t pos = 0, done = 0;
    while (done < n) {
        uint64_t h = 0;
        bool more = true;
        for (int hb = 0; hb < 5 && more && pos < len; hb++) {
            const uint8_t c = in[pos++];
            h |= (uint64_t)(c & 0x7F) << (7 * hb);
            more = (c & 0x80) != 0;
        }
        const int64_t cnt = (int64_t)(h >> 1);
        if (more || cnt == 0) return false;
        if (h & 1) {
            const int64_t take = std::min<int64_t>(8 * cnt, n - done);
            if (pos + (take + 7) / 8 > len) return false;
            for (int64_t i = 0; i < take; i++) out[done + i] = (in[pos + i / 8] >> (i % 8)) & 1;
            pos += cnt;
            done += take;
        } else {
            if (pos >= len || in[pos] > 1) return false;
            const int64_t take = std::min<int64_t>(cnt, n - done);
            memset(out + done, in[pos++], (size_t)take);
            done += take;
        }
    }
    return true;
}

} // namespace

extern "C" {

// n values (0 / 1) -> an RLE stream at bit width 1; -> its size, or -(bytes needed) when cap is too small
int64_t bso_rle_encode(const uint8_t* values, int64_t n, uint8_t* out, int64_t cap) {
    RleEncoder1 e;
    for (int64_t i = 0; i < n; i++) e.put(values[i] ? 1 : 0);
    e.flush();
    if ((int64_t)e.out.size() > cap) return -(int64_t)e.out.size();
    if (!e.out.empty()) memcpy(out, e.out.data(), e.out.size());
    return (int64_t)e.out.size();
}

// the first n values of an RLE stream -> out; 0, or -1 for a malformed stream
int64_t bso_rle_decode(const uint8_t* in, int64_t len, int64_t n, uint8_t* out) { return rle_decode1(in, len, n, out) ? 0 : -1; }

// LZ4 block compress: -> compressed size, or -(bytes needed) when cap is too small
int64_t bso_lz4_compress(const uint8_t* src, int64_t n, uint8_t* dst, int64_t cap) {
    const std::vector<uint8_t> o = lz4_compress(src, n);
    if ((int64_t)o.size() > cap) return -(int64_t)o.size();
    memcpy(dst, o.data(), o.size());
    return (int64_t)o.size();
}

int64_t bso_lz4_decompress(const uint8_t* src, int64_t n, uint8_t* dst, int64_t expect) { return lz4_decompress(src, n, dst, expect); }

// bit transpose of n elements (n % 8 == 0) of s bytes, and its inverse
void bso_trans_bit_elem(const uint8_t* in, uint8_t* out, int64_t n, int32_t s) { trans_bit_elem(in, out, n, s); }
void bso_untrans_bit_elem(const uint8_t* in, uint8_t* out, int64_t n, int32_t s) { untrans_bit_elem(in, out, n, s); }

// n values of s bytes -> page body; -> page size, or -(bytes needed) when cap is too small
int64_t bso_bshuf_encode(int32_t s, const void* values, int64_t n, uint8_t* out, int64_t cap) {
    if (!width_ok(s) || n < 0 || n > 0x7FFFFFF0) return -1;
    const int64_t padded = (n + 7) / 8 * 8, blk = block_elems(s);
    std::vector<uint8_t> data((size_t)(padded * s), 0), tb((size_t)(blk * s)), page(16);
    if (n) memcpy(data.data(), values, (size_t)(n * s));
    for (int64_t b0 = 0; b0 < padded; b0 += blk) {
        const int64_t e = padded - b0 < blk ? padded - b0 : blk;
        trans_bit_elem(data.data() + b0 * s, tb.data(), e, s);
        const std::vector<uint8_t> c = lz4_compress(tb.data(), e * s);
        for (int k = 3; k >= 0; k--) page.push_back((uint8_t)(c.size() >> (8 * k)));
        page.insert(page.end(), c.begin(), c.end());
    }
    put_le32(page.data(), (uint32_t)n);
    put_le32(page.data() + 4, (uint32_t)page.size());
    put_le32(page.data() + 8, (uint32_t)padded);
    put_le32(page.data() + 12, (uint32_t)s);
    if ((int64_t)page.size() > cap) return -(int64_t)page.size();
    memcpy(out, page.data(), page.size());
    return (int64_t)page.size();
}

// page body -> values of s bytes; -> value count, -1 for a malformed page, or -(values) when cap (in values) is too small
int64_t bso_bshuf_decode(int32_t s, const uint8_t* page, int64_t len, void* out, int64_t cap) {
    if (!width_ok(s) || len < 16) return -1;
    const int64_t n = rd32(page), csize = rd32(page + 4), padded = rd32(page + 8), es = rd32(page + 12);
    if (csize != len || padded != (n + 7) / 8 * 8 || es != s) return -1;
    if (n > cap) return n > 1 ? -n : -2;
    const int64_t blk = block_elems(s);
    std::vector<uint8_t> tb((size_t)(blk * s)), vb((size_t)(blk * s));
    int64_t pos = 16;
    for (int64_t b0 = 0; b0 < padded; b0 += blk) {
        const int64_t e = padded - b0 < blk ? padded - b0 : blk;
        if (len - pos < 4) return -1;
        const int64_t c = (int64_t)page[pos] << 24 | page[pos + 1] << 16 | page[pos + 2] << 8 | page[pos + 3];
        pos += 4;
        if (c > kMaxCompressedBlock || c > len - pos) return -1;
        if (lz4_decompress(page + pos, c, tb.data(), e * s) != e * s) return -1;
        pos += c;
        untrans_bit_elem(tb.data(), vb.data(), e, s);
        const int64_t keep = (n - b0 < e ? n - b0 : e) * s;
        if (keep > 0) memcpy((uint8_t*)out + b0 * s, vb.data(), (size_t)keep);
    }
    return pos == len ? n : -1;
}

} // extern "C"
