"""ctypes binding of the BIT_SHUFFLE page codec, the RLE codec at bit width 1 (BOOLEAN pages, RLE null maps) and the
null maps of data pages, restated on the CPU (bshuf_oracle/bshuf_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

Only tests/, scripts/ and tools/ import this package: it writes the pages the device decoder is checked and measured
against, and decodes them the way the reference does.  The product package (starrocks_b200) never imports it.
"""
import ctypes as C
import ctypes.util
import hashlib
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "bshuf_oracle.cpp")
_LIB_PATH = os.path.join(_HERE, "libbshuf_oracle.so")
_LIB = None

LZ4_MAX_BLOCK = 8240          # LZ4_compressBound(8192): the most a bitshuffle block may claim


class CorruptPage(ValueError):
    pass


def _source_hash():
    with open(_SRC, "rb") as fh:
        return hashlib.sha256(fh.read()).hexdigest()


def _recorded_hash():
    try:
        with open(_LIB_PATH + ".srchash") as fh:
            return fh.read().strip()
    except OSError:
        return None


def build():
    """compile libbshuf_oracle.so (g++, a second); a no-op when the library matches the source"""
    import fcntl
    with open(_LIB_PATH + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if os.path.exists(_LIB_PATH) and _recorded_hash() == _source_hash():
                return
            tmp = _LIB_PATH + ".tmp.%d" % os.getpid()
            subprocess.check_call([os.environ.get("CXX", "g++"), "-O3", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", tmp, _SRC])
            os.replace(tmp, _LIB_PATH)
            with open(_LIB_PATH + ".srchash", "w") as fh:
                fh.write(_source_hash())
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_LIB_PATH) or _recorded_hash() != _source_hash():
            build()
        L = C.CDLL(_LIB_PATH)
        i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
        for name, res, args in (("bso_lz4_compress", i64, [vp, i64, vp, i64]), ("bso_lz4_decompress", i64, [vp, i64, vp, i64]),
                                ("bso_trans_bit_elem", None, [vp, vp, i64, i32]), ("bso_untrans_bit_elem", None, [vp, vp, i64, i32]),
                                ("bso_bshuf_encode", i64, [i32, vp, i64, vp, i64]), ("bso_bshuf_decode", i64, [i32, vp, i64, vp, i64]),
                                ("bso_rle_encode", i64, [vp, i64, vp, i64]), ("bso_rle_decode", i64, [vp, i64, i64, vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data if a.size else None


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


def lz4_compress(data):
    """LZ4 block-format stream of a byte array (greedy hash-table matcher; real matches, the format's end-of-block rules)"""
    src = np.ascontiguousarray(data, dtype=np.uint8)
    cap = len(src) + len(src) // 255 + 16
    out = np.zeros(cap, dtype=np.uint8)
    r = lib().bso_lz4_compress(_ptr(src), len(src), out.ctypes.data, cap)
    assert r >= 0
    return out[:r]


def lz4_decompress(stream, size):
    """-> the `size` bytes the stream decodes to; CorruptPage when it is malformed or decodes to another size"""
    src = np.ascontiguousarray(stream, dtype=np.uint8)
    out = np.zeros(max(size, 1), dtype=np.uint8)
    if lib().bso_lz4_decompress(_ptr(src), len(src), out.ctypes.data, size) != size:
        raise CorruptPage("LZ4 stream")
    return out[:size]


def trans_bit_elem(values):
    """bshuf_trans_bit_elem of a 1-D array (len % 8 == 0) -> 8 * itemsize rows of len / 8 bytes, as one byte array"""
    v = np.ascontiguousarray(values)
    assert v.ndim == 1 and len(v) % 8 == 0
    out = np.zeros(v.nbytes, dtype=np.uint8)
    lib().bso_trans_bit_elem(_ptr(v), _ptr(out), len(v), v.dtype.itemsize)
    return out


def untrans_bit_elem(data, width):
    """inverse of trans_bit_elem: bytes -> the elements' bytes (len(data) / width elements of `width` bytes, in order)"""
    d = np.ascontiguousarray(data, dtype=np.uint8)
    assert len(d) % (8 * width) == 0
    out = np.zeros(len(d), dtype=np.uint8)
    lib().bso_untrans_bit_elem(_ptr(d), _ptr(out), len(d) // width, width)
    return out


def bitshuffle_encode(values, width=None):
    """BIT_SHUFFLE page body (BitshufflePageBuilder::finish) of a 1-D array.  A uint8 array with width=w holds values of w
    bytes (how 16-byte LARGEINT / DECIMAL128 values are passed: numpy has no int128)."""
    v = np.ascontiguousarray(values)
    w = width or v.dtype.itemsize
    b = _bytes(v)
    assert len(b) % w == 0
    n = len(b) // w
    padded = b.nbytes + 8 * w                                   # padding, and LZ4 overhead of at most 52 bytes per block
    cap = 16 + padded + (padded // 8192 + 1) * 64
    out = np.zeros(cap, dtype=np.uint8)
    r = lib().bso_bshuf_encode(w, _ptr(b), n, out.ctypes.data, cap)
    if r < 0:
        raise ValueError("width %d" % w)
    return out[:r]


def bitshuffle_decode(page, dtype_or_width):
    """page body -> values: an array of `dtype`, or for an int width a uint8 array of count * width bytes"""
    p = np.ascontiguousarray(page, dtype=np.uint8)
    if isinstance(dtype_or_width, int):
        w, dt = dtype_or_width, np.dtype(np.uint8)
    else:
        dt = np.dtype(dtype_or_width)
        w = dt.itemsize
    n = int(np.frombuffer(p[0:4].tobytes(), dtype="<u4")[0]) if len(p) >= 16 else 0
    if n * w > 256 * len(p) + 1024:          # more than LZ4 can expand the page to: no allocation for it
        raise CorruptPage("value count")
    out = np.zeros(max(n, 1) * w, dtype=np.uint8)
    r = lib().bso_bshuf_decode(w, _ptr(p), len(p), out.ctypes.data, max(n, 1))
    if r < 0:
        raise CorruptPage("bitshuffle page")
    got = out[:r * w]
    return got if dt == np.uint8 and isinstance(dtype_or_width, int) else got.view(dt)


# ---- dictionary-encoded (DICT_ENCODING) columns: BinaryDictPageBuilder::finish / BinaryPlainPageBuilder::finish ----
DICT_ENCODING, PLAIN_ENCODING = 5, 2            # EncodingTypePB values of a dictionary data page's mode word


def dict_page_encode(codes):
    """dictionary data page body of int32 codes: the mode word 5, then the BIT_SHUFFLE page of the codes"""
    c = np.ascontiguousarray(codes, dtype=np.int32)
    return np.concatenate([np.array([DICT_ENCODING], dtype="<u4").view(np.uint8), bitshuffle_encode(c)])


def dict_page_plain_fallback(words):
    """a data page written after the column's dictionary overflowed: the mode word 2, then a BinaryPlainPage of strings"""
    return np.concatenate([np.array([PLAIN_ENCODING], dtype="<u4").view(np.uint8), binary_plain_page_encode(words)])


def dict_page_decode(page):
    """dictionary data page body -> int32 codes; CorruptPage for a short page, a mode other than 5 (2 included: strings,
    not codes) or a bad bitshuffle page"""
    p = np.ascontiguousarray(page, dtype=np.uint8)
    if len(p) < 4:
        raise CorruptPage("dictionary page shorter than its mode word")
    mode = int(np.frombuffer(p[:4].tobytes(), dtype="<u4")[0])
    if mode != DICT_ENCODING:
        raise CorruptPage("dictionary page mode %d" % mode)
    if len(p) < 20 or int(np.frombuffer(p[16:20].tobytes(), dtype="<u4")[0]) != 4:
        raise CorruptPage("dictionary codes are not a 4-byte bitshuffle page")
    return bitshuffle_decode(p[4:], np.int32)


def binary_plain_page_encode(words):
    """BinaryPlainPage of byte strings: the words back to back, one uint32 LE start offset per word, the uint32 LE count"""
    words = [bytes(w) for w in words]
    offs = np.cumsum([0] + [len(w) for w in words[:-1]]).astype("<u4") if words else np.zeros(0, dtype="<u4")
    return np.concatenate([np.frombuffer(b"".join(words), dtype=np.uint8), offs.view(np.uint8),
                           np.array([len(words)], dtype="<u4").view(np.uint8)])


def binary_plain_page_decode(page):
    """BinaryPlainPage -> list of bytes (BinaryPlainPageDecoder::init); CorruptPage for a count that does not fit, or
    offsets that decrease or pass the offset array.  Word i runs to offset[i + 1], the last one to the offset array."""
    p = np.ascontiguousarray(page, dtype=np.uint8).tobytes()
    if len(p) < 4:
        raise CorruptPage("binary plain page shorter than its count")
    n = int.from_bytes(p[-4:], "little")
    start = len(p) - 4 - 4 * n
    if start < 0:
        raise CorruptPage("word count %d" % n)
    offs = [int.from_bytes(p[start + 4 * i:start + 4 * i + 4], "little") for i in range(n)] + [start]
    if any(a > b for a, b in zip(offs, offs[1:])):
        raise CorruptPage("word offsets")
    return [p[offs[i]:offs[i + 1]] for i in range(n)]


# ---- RLE at bit width 1 (RleEncoder / RleDecoder, be/src/util/rle_encoding.h): BOOLEAN pages and RLE_NULL null maps ----
NULL_BITSHUFFLE, NULL_RLE = 0, 1                # NullEncodingPB: BITSHUFFLE_NULL, RLE_NULL


def rle_encode(values):
    """RleEncoder stream of 0 / 1 values at bit width 1 (nonzero counts as 1)"""
    v = np.ascontiguousarray(values, dtype=np.uint8)
    cap = 2 * len(v) // 8 + 16                  # literal runs: 64 bytes per 63 groups; repeated runs: <= 6 bytes per >= 8 values
    out = np.zeros(cap, dtype=np.uint8)
    r = lib().bso_rle_encode(_ptr(v), len(v), out.ctypes.data, cap)
    assert r >= 0
    return out[:r]


def rle_decode(stream, n):
    """the first n values of an RLE stream at bit width 1 (uint8 0 / 1); CorruptPage for what RleDecoder cannot decode"""
    s = np.ascontiguousarray(stream, dtype=np.uint8)
    out = np.zeros(max(n, 1), dtype=np.uint8)
    if lib().bso_rle_decode(_ptr(s), len(s), n, out.ctypes.data) != 0:
        raise CorruptPage("RLE stream")
    return out[:n]


def rle_bool_page_encode(values):
    """RLE page body of a BOOLEAN column (RlePageBuilder::finish): the uint32 LE value count, then the RLE stream"""
    v = np.ascontiguousarray(values, dtype=np.uint8)
    return np.concatenate([np.array([len(v)], dtype="<u4").view(np.uint8), rle_encode(v)])


def rle_bool_page_decode(page):
    p = np.ascontiguousarray(page, dtype=np.uint8)
    if len(p) < 4:
        raise CorruptPage("RLE page shorter than its count")
    return rle_decode(p[4:], int(np.frombuffer(p[:4].tobytes(), dtype="<u4")[0]))


def null_map_encode(flags, encoding):
    """the null map of a data page whose rows carry `flags` (nonzero = NULL) -- empty when no row is NULL (the writer then
    stores no map): bitshuffle::compress_lz4 of the flags padded to 8 (a BIT_SHUFFLE page of bytes without its 16-byte
    header), or the RleEncoder stream"""
    f = (np.ascontiguousarray(flags) != 0).astype(np.uint8)
    if not f.any():
        return np.zeros(0, dtype=np.uint8)
    if encoding == NULL_RLE:
        return rle_encode(f)
    assert encoding == NULL_BITSHUFFLE
    return bitshuffle_encode(f)[16:]


def null_map_decode(nmap, num_rows, encoding):
    """-> num_rows uint8 flags; an empty map is a page without NULLs.  CorruptPage for a malformed map"""
    m = np.ascontiguousarray(nmap, dtype=np.uint8)
    if len(m) == 0:
        return np.zeros(num_rows, dtype=np.uint8)
    if encoding == NULL_RLE:
        return rle_decode(m, num_rows)
    assert encoding == NULL_BITSHUFFLE
    padded = (num_rows + 7) // 8 * 8
    hdr = np.array([num_rows, 16 + len(m), padded, 1], dtype="<u4").view(np.uint8)
    return bitshuffle_decode(np.concatenate([hdr, m]), 1)


def system_lz4():
    """the system liblz4 (ctypes: LZ4_compress_default, LZ4_decompress_safe, LZ4_compressBound), or None when absent"""
    for name in ("liblz4.so.1", ctypes.util.find_library("lz4")):
        if not name:
            continue
        try:
            L = C.CDLL(name)
        except OSError:
            continue
        L.LZ4_compress_default.restype = C.c_int
        L.LZ4_compress_default.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.LZ4_decompress_safe.restype = C.c_int
        L.LZ4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.LZ4_compressBound.restype = C.c_int
        L.LZ4_compressBound.argtypes = [C.c_int]
        L.LZ4_versionString.restype = C.c_char_p
        return L
    return None


def system_lz4_compress(L, data):
    src = np.ascontiguousarray(data, dtype=np.uint8)
    cap = L.LZ4_compressBound(len(src))
    out = np.zeros(cap, dtype=np.uint8)
    r = L.LZ4_compress_default(_ptr(src), out.ctypes.data, len(src), cap)
    assert r > 0
    return out[:r]


def system_lz4_decompress(L, stream, size):
    """-> (verdict, output): liblz4's LZ4_decompress_safe with capacity `size`; verdict True when it returned exactly `size`"""
    src = np.ascontiguousarray(stream, dtype=np.uint8)
    out = np.zeros(max(size, 1) + 64, dtype=np.uint8)       # slack past the capacity: a decoder that overran it would show
    r = L.LZ4_decompress_safe(_ptr(src), out.ctypes.data, len(src), size)
    return r == size, out[:size]


def bitshuffle_encode_with(L, values, width=None):
    """a page body whose LZ4 blocks come from the system liblz4's LZ4_compress_default (what the golden pages hold)"""
    v = np.ascontiguousarray(values)
    w = width or v.dtype.itemsize
    b = _bytes(v)
    n = len(b) // w
    padded = (n + 7) // 8 * 8
    data = np.zeros(padded * w, dtype=np.uint8)
    data[:len(b)] = b
    blk = max(128, (8192 // w) // 8 * 8)
    parts = []
    for b0 in range(0, padded, blk):
        e = min(blk, padded - b0)
        rows = trans_bit_elem(data[b0 * w:(b0 + e) * w].view(_UINT[w]) if w <= 8 else _as_u8_elems(data[b0 * w:(b0 + e) * w], w))
        c = system_lz4_compress(L, rows)
        parts.append(np.frombuffer(len(c).to_bytes(4, "big"), dtype=np.uint8))
        parts.append(c)
    body = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
    hdr = np.array([n, 16 + len(body), padded, w], dtype="<u4").view(np.uint8)
    return np.concatenate([hdr, body])


_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _as_u8_elems(b, w):
    """16-byte elements as a structured view trans_bit_elem accepts (itemsize w)"""
    return b.view(np.dtype((np.void, w)))
