// oracle/_ref: the REAL frame-of-reference codec of the reference (be/src/util/frame_of_reference_coding.{h,cpp}, the codec
// behind FrameOfReferencePageBuilder / FrameOfReferencePageDecoder, be/src/storage/rowset/frame_of_reference_page.h),
// compiled from the reference tree where it lies together with be/src/base/string/faststring.cc.  oracle/ref_shims/ holds
// stand-ins for the third-party headers that code pulls in but does not need here (glog, butil, fmt, arrow, boost via
// bit_stream_utils); no reference source is copied.  Built by `make -C oracle ref` only where a reference tree is given.
// tests/test_oracle_golden.py checks orc_for_encode / orc_for_decode (the restatement) byte for byte against it.
#include "util/frame_of_reference_coding.h"

#include <cstring>

using namespace starrocks;

template <typename T>
static long long encode(const T* v, long long n, unsigned char* out, long long cap) {
    faststring buf;
    ForEncoder<T> enc(&buf);
    if (n > 0) enc.put_batch(v, (size_t)n);
    enc.flush();
    if ((long long)buf.size() > cap) return -(long long)buf.size();
    memcpy(out, buf.data(), buf.size());
    return (long long)buf.size();
}

template <typename T>
static long long decode(const unsigned char* page, long long len, T* out, long long cap) {
    ForDecoder<T> dec(page, (size_t)len);
    if (!dec.init()) return -1;
    const long long n = dec.count();
    if (n > cap) return -n;
    if (n > 0 && !dec.get_batch(out, (size_t)n)) return -1;
    return n;
}

extern "C" long long ref_for_encode_i32(const int* v, long long n, unsigned char* out, long long cap) { return encode<int32_t>(v, n, out, cap); }
extern "C" long long ref_for_encode_i64(const long long* v, long long n, unsigned char* out, long long cap) { return encode<int64_t>((const int64_t*)v, n, out, cap); }
extern "C" long long ref_for_decode_i32(const unsigned char* p, long long len, int* out, long long cap) { return decode<int32_t>(p, len, out, cap); }
extern "C" long long ref_for_decode_i64(const unsigned char* p, long long len, long long* out, long long cap) { return decode<int64_t>(p, len, (int64_t*)out, cap); }
