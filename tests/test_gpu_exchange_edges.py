"""Exchange edges: the hash partition (sr_xchg_hash / sr_xchg_partition: k_part_hash, k_part_scatter, k_gather) and the
ChunkPB.data wire format (sr_chunk_serialize / sr_chunk_deserialize) at the edges of their types, NULLs, channel counts,
row counts and memory kinds.

The exchange is where the device has to agree with a CPU BE bit for bit: the same key must land on the same channel on
both, and each side must parse the other's ChunkPB bytes.  A wrong hash raises no error -- it splits a group over two
nodes -- so every hash value, channel id, row position and payload byte is compared exactly with a reference written
here in plain Python (ints and bytes, no oracle):
  FNV-1a 32        h = ((h ^ b) * 0x01000193) mod 2^32 per byte, seed 0x811C9DC5
  CRC32            zlib.crc32(data, h) (zlib's crc32(seed, data, len)), seed 0
  XXH3             XXH3_64bits_withSeed of 1..16 bytes (len_1to3 / len_4to8 / len_9to16, default secret) truncated to
                   32 bits, the row's hash so far as the seed; seed 0x9E3779B1
  NULL row         CRC32 hashes 4 zero bytes; FNV and XXH3 mix h ^ (0x9e3779b9 + (h << 6) + (h >> 2)); the bytes under
                   a NULL are never read
  channel          MULHI (h * n) >> 32, MODULO h % n; rows of a channel in input order (a stable sort by channel)
  wire format      fixed32 version 1, fixed32 num_rows, then per column the null column (if nullable) and the data
                   column, each a fixed32 byte size and the raw bytes
The CPU tests pin the reference to stored goldens and to the oracle on every case the GPU tests use.
"""
import ctypes as C
import functools
import os
import struct
import zlib

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
FNV, CRC, XXH3 = abi.HASH_FNV, abi.HASH_CRC32, abi.HASH_XXH3
MULHI, MODULO = abi.REDUCE_MULHI, abi.REDUCE_MODULO
HASH_NAME = {FNV: "fnv", CRC: "crc32", XXH3: "xxh3"}
REDUCE_NAME = {MULHI: "mulhi", MODULO: "modulo"}
SEED = {FNV: 0x811C9DC5, CRC: 0, XXH3: 0x9E3779B1}


# =============================================================================================
# the reference
# =============================================================================================
def fnv1a32(data, h):
    for b in data:
        h = ((h ^ b) * 0x01000193) & M32
    return h


XXH3_SECRET = bytes.fromhex(
    "b8fe6c3923a44bbe7c01812cf721ad1cded46de9839097db7240a4a4b7b3671f"
    "cb79e64eccc0e578825ad07dccff7221b8084674f743248ee03590e6813a264c")


def _r32(b, o):
    return int.from_bytes(b[o:o + 4], "little")


def _r64(b, o):
    return int.from_bytes(b[o:o + 8], "little")


def _rotl64(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _bswap(x, nbytes):
    return int.from_bytes(x.to_bytes(nbytes, "little"), "big")


def xxh3_64(data, seed):
    """XXH3_64bits_withSeed for 1 <= len(data) <= 16"""
    n = len(data)
    assert 1 <= n <= 16
    if n <= 3:
        combined = (data[0] << 16) | (data[n >> 1] << 24) | data[n - 1] | (n << 8)
        h = combined ^ (((_r32(XXH3_SECRET, 0) ^ _r32(XXH3_SECRET, 4)) + seed) & M64)
        h ^= h >> 33                                        # XXH64_avalanche
        h = (h * 0xC2B2AE3D27D4EB4F) & M64
        h ^= h >> 29
        h = (h * 0x165667B19E3779F9) & M64
        return h ^ (h >> 32)
    if n <= 8:
        seed ^= _bswap(seed & M32, 4) << 32
        keyed = (_r32(data, n - 4) + (_r32(data, 0) << 32)) ^ (((_r64(XXH3_SECRET, 8) ^ _r64(XXH3_SECRET, 16)) - seed) & M64)
        h = keyed ^ _rotl64(keyed, 49) ^ _rotl64(keyed, 24)  # XXH3_rrmxmx
        h = (h * 0x9FB21C651E98DF25) & M64
        h ^= (h >> 35) + n
        h = (h * 0x9FB21C651E98DF25) & M64
        return h ^ (h >> 28)
    lo = _r64(data, 0) ^ (((_r64(XXH3_SECRET, 24) ^ _r64(XXH3_SECRET, 32)) + seed) & M64)
    hi = _r64(data, n - 8) ^ (((_r64(XXH3_SECRET, 40) ^ _r64(XXH3_SECRET, 48)) - seed) & M64)
    prod = lo * hi
    h = (n + _bswap(lo, 8) + hi + ((prod & M64) ^ (prod >> 64))) & M64
    h ^= h >> 37                                            # XXH3_avalanche
    h = (h * 0x165667919E3779F9) & M64
    return h ^ (h >> 32)


def hash_value(fn, data, h):
    if fn == FNV:
        return fnv1a32(data, h)
    if fn == CRC:
        return zlib.crc32(data, h)
    return xxh3_64(data, h) & M32


def hash_null(fn, h):
    if fn == CRC:
        return zlib.crc32(b"\0\0\0\0", h)
    return (h ^ ((0x9E3779B9 + (h << 6) + (h >> 2)) & M32)) & M32


def hash_key(fn, values):
    """values: one bytes (or None for NULL) per partition column"""
    h = SEED[fn]
    for v in values:
        h = hash_null(fn, h) if v is None else hash_value(fn, v, h)
    return h


def reduce_channel(reduce_op, h, n):
    return (h * n) >> 32 if reduce_op == MULHI else h % n


class Col:
    """one fixed-width column as raw little-endian bytes (+ a null byte per row, 1 = NULL)"""

    def __init__(self, slot, typ, raw, nulls=None):
        self.slot, self.typ, self.w = slot, typ, abi.TYPE_WIDTH[typ]
        self.raw = bytes(raw)
        self.nulls = None if nulls is None else bytes(nulls)
        assert len(self.raw) % self.w == 0
        self.n = len(self.raw) // self.w
        assert self.nulls is None or len(self.nulls) == self.n

    def value(self, i):
        if self.nulls is not None and self.nulls[i]:
            return None
        return self.raw[i * self.w:(i + 1) * self.w]


def ref_hashes(cols, key_slots, fn, n):
    keys = [next(c for c in cols if c.slot == s) for s in key_slots]
    memo = {}
    out = np.zeros(n, dtype=np.uint32)
    for i in range(n):
        k = tuple(c.value(i) for c in keys)
        h = memo.get(k)
        if h is None:
            h = memo[k] = hash_key(fn, k)
        out[i] = h
    return out


def ref_partition(hv, reduce_op, nch):
    """-> channel ids, row order (stable by channel), channel offsets (nch + 1)"""
    h = hv.astype(np.uint64)
    ch = ((h * np.uint64(nch)) >> np.uint64(32)) if reduce_op == MULHI else h % np.uint64(nch)
    ch = ch.astype(np.uint32)
    order = np.argsort(ch, kind="stable")
    offs = np.concatenate([[0], np.cumsum(np.bincount(ch, minlength=nch))]).astype(np.int64)
    return ch, order, offs


def take_rows(c, order):
    """column c with its rows in `order`: the data bytes (garbage under NULLs included) and the null bytes"""
    raw = np.frombuffer(c.raw, dtype=np.uint8).reshape(-1, c.w)[order].tobytes() if c.n else b""
    nul = None if c.nulls is None else np.frombuffer(c.nulls, dtype=np.uint8)[order].tobytes()
    return raw, nul


def ref_serialize(cols, lo, hi):
    rows = hi - lo
    out = [struct.pack("<II", 1, rows)]
    for c in cols:
        if c.nulls is not None:
            out.append(struct.pack("<I", rows) + c.nulls[lo:hi])
        out.append(struct.pack("<I", rows * c.w) + c.raw[lo * c.w:hi * c.w])
    return b"".join(out)


# =============================================================================================
# cases
# =============================================================================================
TYPES = [abi.TYPE_BOOLEAN, abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_FLOAT, abi.TYPE_DATE, abi.TYPE_DECIMAL32,
         abi.TYPE_BIGINT, abi.TYPE_DOUBLE, abi.TYPE_DATETIME, abi.TYPE_DECIMAL64, abi.TYPE_LARGEINT, abi.TYPE_DECIMAL128]
TYPE_NAME = {abi.TYPE_BOOLEAN: "boolean", abi.TYPE_TINYINT: "tinyint", abi.TYPE_SMALLINT: "smallint", abi.TYPE_INT: "int",
             abi.TYPE_FLOAT: "float", abi.TYPE_DATE: "date", abi.TYPE_DECIMAL32: "decimal32", abi.TYPE_BIGINT: "bigint",
             abi.TYPE_DOUBLE: "double", abi.TYPE_DATETIME: "datetime", abi.TYPE_DECIMAL64: "decimal64",
             abi.TYPE_LARGEINT: "largeint", abi.TYPE_DECIMAL128: "decimal128"}
WIDTH_TYPE = {1: abi.TYPE_TINYINT, 2: abi.TYPE_SMALLINT, 4: abi.TYPE_INT, 8: abi.TYPE_BIGINT, 16: abi.TYPE_DECIMAL128}

FLOAT_BITS = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000,
              0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0xBF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FC00001, 0x7FFFFFFF,
              0xFFFFFFFF]
DOUBLE_BITS = [0x0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x1, 0x8000000000000001, 0x000FFFFFFFFFFFFF,
               0x800FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x3FF0000000000000,
               0xBFF0000000000000, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8000000000001,
               0x7FF4000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF]


def edge_values(typ):
    """the value edges of a type as raw bytes: min, max, 0, +-1, all ones; around 2^64 and +-2^127 for 16-byte types;
    +-0.0, +-inf, subnormals and NaNs of different payloads for FLOAT / DOUBLE"""
    w = abi.TYPE_WIDTH[typ]
    if typ == abi.TYPE_FLOAT:
        return [b.to_bytes(4, "little") for b in FLOAT_BITS]
    if typ == abi.TYPE_DOUBLE:
        return [b.to_bytes(8, "little") for b in DOUBLE_BITS]
    if typ == abi.TYPE_BOOLEAN:
        return [bytes([0]), bytes([1]), bytes([0xFF])]
    lo, hi = -(1 << (8 * w - 1)), (1 << (8 * w - 1)) - 1
    vals = [lo, hi, 0, 1, -1, lo + 1, hi - 1, 2, -2]
    if w == 16:
        vals += [(1 << 64) - 1, 1 << 64, (1 << 64) + 1, -(1 << 64), -(1 << 64) - 1, 1 << 63, -(1 << 63), (1 << 63) - 1,
                 (1 << 126), -(1 << 126), (1 << 32) - 1, 1 << 32]
    return [v.to_bytes(w, "little", signed=True) for v in vals]


def edge_column(typ, nullable, seed, n=320, slot=0):
    """the edges (never NULL) followed by random bytes; nullable: ~30% NULLs with random garbage under them"""
    rng = np.random.default_rng(seed)
    w = abi.TYPE_WIDTH[typ]
    edges = edge_values(typ)
    raw = bytearray(rng.integers(0, 256, n * w, dtype=np.uint8).tobytes())
    for i, e in enumerate(edges * 3):                       # every edge at three positions: start, middle, end
        p = [i, n // 2 + i, n - 1 - i][i // len(edges)]
        raw[p * w:(p + 1) * w] = e
    nulls = None
    if nullable:
        nl = (rng.random(n) < 0.3).astype(np.uint8)
        nl[:len(edges)] = 0
        nulls = nl.tobytes()
    return Col(slot, typ, raw, nulls)


def random_column(slot, typ, n, rng, null_rate=None):
    w = abi.TYPE_WIDTH[typ]
    raw = rng.integers(0, 256, n * w, dtype=np.uint8).tobytes()
    nulls = None if null_rate is None else (rng.random(n) < null_rate).astype(np.uint8).tobytes()
    return Col(slot, typ, raw, nulls)


MULTI_KEY_CASES = {
    "int_tinyint": [13, 10],
    "decimal128_smallint_int": [14, 11, 12],
    "four_widths": [10, 14, 13, 11],
    "same_slot_twice": [12, 12],
    "decimal128_twice_and_tinyint": [14, 14, 10],
    "reverse_of_chunk_order": [14, 13, 12, 11],
}


def multi_key_columns(seed=5, n=3000):
    """slots 10..14 of widths 1, 2, 4, 8, 16, each with its own NULLs (and edge values in the first rows)"""
    rng = np.random.default_rng(seed)
    cols = []
    for k, w in enumerate((1, 2, 4, 8, 16)):
        typ = WIDTH_TYPE[w]
        c = random_column(10 + k, typ, n, rng, null_rate=0.1 + 0.05 * k)
        raw = bytearray(c.raw)
        for i, e in enumerate(edge_values(typ)):
            raw[(7 * i + k) * w:(7 * i + k + 1) * w] = e
        cols.append(Col(10 + k, typ, raw, c.nulls))
    return cols


def int_key(v):
    return (v & M32).to_bytes(4, "little")


@functools.lru_cache(maxsize=None)
def extreme_int_keys(fn, count=8):
    """INT keys whose reference hash is below 2^20 (MULHI: channel 0 for every n <= 4096) and keys above 2^32 - 2^20
    (channel n - 1)"""
    low, high = [], []
    for v in range(1 << 20):
        h = hash_key(fn, [int_key(v)])
        if h < (1 << 20) and len(low) < count:
            low.append(v)
        elif h >= (1 << 32) - (1 << 20) and len(high) < count:
            high.append(v)
        if len(low) == count and len(high) == count:
            return tuple(low), tuple(high)
    raise AssertionError("no extreme keys found")


def channel_count_columns(fn, nch, seed):
    rng = np.random.default_rng(seed + nch)
    low, high = extreme_int_keys(fn)
    n = 4 * nch + 600
    keys = rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64)
    keys[:len(low)] = low
    keys[-len(high):] = high
    raw = b"".join(int_key(int(v)) for v in keys)
    return [Col(0, abi.TYPE_INT, raw), random_column(1, abi.TYPE_DECIMAL128, n, rng, 0.2)]


CHANNEL_COUNTS = [1, 2, 3, 31, 32, 33, 255, 256]
LAYOUT_ROWS = [0, 1, 1023, 1024, 1025, 4097, 250_001]
LAYOUT_SKEWS = ["uniform", "all_first", "all_last", "one_middle", "two_alternating"]
LAYOUT_NCH = 33


@functools.lru_cache(maxsize=None)
def keys_by_channel(fn, reduce_op, nch, per_channel=4):
    """INT keys and their reference hashes, per channel"""
    pool = [[] for _ in range(nch)]
    v = 0
    while any(len(p) < per_channel for p in pool):
        h = hash_key(fn, [int_key(v)])
        c = reduce_channel(reduce_op, h, nch)
        if len(pool[c]) < per_channel:
            pool[c].append((v, h))
        v += 1
    return pool


def layout_columns(n, skew, seed=17):
    """partition key (slot 0, FNV / MULHI over 33 channels) drawn per the skew, payload columns of every width with and
    without NULLs.  -> (cols, reference hash values)"""
    rng = np.random.default_rng(seed + n)
    pool = keys_by_channel(FNV, MULHI, LAYOUT_NCH)
    if skew == "uniform":
        chans = rng.integers(0, LAYOUT_NCH, n)
    elif skew == "all_first":
        chans = np.zeros(n, dtype=np.int64)
    elif skew == "all_last":
        chans = np.full(n, LAYOUT_NCH - 1)
    elif skew == "one_middle":
        chans = np.full(n, LAYOUT_NCH // 2)
    else:
        chans = np.where(np.arange(n) % 2 == 0, 3, LAYOUT_NCH - 2)
    pick = rng.integers(0, 4, n)
    keys = np.array([[v for v, _ in p] for p in pool], dtype=np.int64)[chans, pick]
    hv = np.array([[h for _, h in p] for p in pool], dtype=np.uint32)[chans, pick]
    cols = [Col(0, abi.TYPE_INT, keys.astype(np.int32).tobytes())]
    for k, w in enumerate((1, 2, 4, 8, 16)):
        cols.append(random_column(1 + k, WIDTH_TYPE[w], n, rng))
        cols.append(random_column(6 + k, WIDTH_TYPE[w], n, rng, null_rate=0.25))
    return cols, hv


def wire_columns(n, seed=29):
    """every type, plain and nullable, and an all-NULL column"""
    rng = np.random.default_rng(seed)
    cols = []
    for k, typ in enumerate(TYPES):
        cols.append(random_column(2 * k, typ, n, rng))
        cols.append(random_column(2 * k + 1, typ, n, rng, null_rate=0.3))
    cols.append(Col(99, abi.TYPE_BIGINT, rng.integers(0, 256, 8 * n, dtype=np.uint8).tobytes(), bytes([1]) * n))
    return cols


def host_chunk(cols, n):
    spec = []
    for c in cols:
        a = np.frombuffer(c.raw, dtype=np.uint8).copy().view(np.dtype((np.void, c.w))) if c.n else np.zeros(0, dtype=np.dtype((np.void, c.w)))
        nl = None if c.nulls is None else np.frombuffer(c.nulls, dtype=np.uint8).copy()
        spec.append((c.slot, a, nl, c.typ))
    return Chunk(spec, num_rows=n)


# =============================================================================================
# CPU: the reference against stored goldens, the xxhash package and the oracle
# =============================================================================================
def _golden(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    offs = np.concatenate([[0], np.cumsum(g["lengths"])])
    return [g["data"][offs[k]:offs[k + 1]].tobytes() for k in range(len(g["lengths"]))], g


def test_reference_hashes_equal_the_goldens():
    bufs, g = _golden("exchange_hashes")
    for k, b in enumerate(bufs):
        for j, seed in enumerate(int(s) for s in g["seeds"]):
            assert fnv1a32(b, seed) == int(g["fnv_hash"][k, j]), ("fnv", len(b), seed)
            assert zlib.crc32(b, seed) == int(g["zlib_crc_hash"][k, j]), ("crc32", len(b), seed)
    bufs, g = _golden("xxh3_64")
    checked = 0
    for b, seed, want in zip(bufs, g["seeds"], g["hashes"]):
        if 1 <= len(b) <= 16:
            assert xxh3_64(b, int(seed)) == int(want), (len(b), int(seed))
            checked += 1
    assert checked == 16 * 200


def test_reference_xxh3_against_the_xxhash_package():
    xxhash = pytest.importorskip("xxhash")
    rng = np.random.default_rng(3)
    for n in range(1, 17):
        for _ in range(100):
            b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            seed = int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2))
            assert xxh3_64(b, seed) == xxhash.xxh3_64_intdigest(b, seed), (n, seed)
            assert xxh3_64(b, seed & M32) == xxhash.xxh3_64_intdigest(b, seed & M32), (n, seed)


def test_reference_known_answers():
    assert fnv1a32(b"", 0x811C9DC5) == 0x811C9DC5 and fnv1a32(b"a", 0x811C9DC5) == 0xE40C292C     # FNV-1a 32 test vector
    assert zlib.crc32(b"123456789", 0) == 0xCBF43926                                                # CRC-32 check value
    assert hash_null(FNV, 0) == 0x9E3779B9 and hash_null(CRC, 0) == zlib.crc32(b"\0\0\0\0")
    assert reduce_channel(MULHI, M32, 256) == 255 and reduce_channel(MULHI, (1 << 20) - 1, 4096) == 0
    # +0.0 and -0.0 are different bytes and hash differently
    assert hash_key(FNV, [struct.pack("<d", 0.0)]) != hash_key(FNV, [struct.pack("<d", -0.0)])


def _oracle_partition_cases():
    for typ in TYPES:
        for nullable in (False, True):
            cols = [edge_column(typ, nullable, seed=typ)]
            for fn in (FNV, CRC, XXH3):
                for red in (MULHI, MODULO):
                    yield f"edge/{TYPE_NAME[typ]}/{nullable}/{fn}/{red}", cols, [0], fn, red, 37
    mk = multi_key_columns()
    for name, slots in MULTI_KEY_CASES.items():
        for fn in (FNV, CRC, XXH3):
            yield f"multi/{name}/{fn}", mk, slots, fn, MULHI, 37
    for fn in (FNV, CRC, XXH3):
        for nch in CHANNEL_COUNTS:
            for red in (MULHI, MODULO):
                yield f"nch/{fn}/{nch}/{red}", channel_count_columns(fn, nch, 7), [0], fn, red, nch
    for n in LAYOUT_ROWS[:-1]:
        for skew in LAYOUT_SKEWS:
            yield f"layout/{n}/{skew}", layout_columns(n, skew)[0], [0], FNV, MULHI, LAYOUT_NCH


def test_reference_partition_equals_the_oracle(oracle):
    # hash values, channels, row order and offsets, on every partition case of the GPU tests (the 250 001-row layouts
    # draw the same keys as the smaller ones)
    for label, cols, slots, fn, red, nch in _oracle_partition_cases():
        n = cols[0].n
        d = abi.make_part_desc(slots, nch, hash_fn=fn, reduce_op=red)
        ohv, och, ori, ost = oracle.hash_partition(d, host_chunk(cols, n))
        hv = ref_hashes(cols, slots, fn, n)
        ch, order, offs = ref_partition(hv, red, nch)
        assert np.array_equal(hv, ohv) and np.array_equal(ch, och), label
        assert np.array_equal(order, ori) and offs.tolist() == ost.tolist(), label


def test_layout_keys_hash_as_drawn():
    for skew in LAYOUT_SKEWS:
        cols, hv = layout_columns(1025, skew)
        assert np.array_equal(ref_hashes(cols, [0], FNV, 1025), hv), skew


def test_reference_serialize_equals_the_oracle(oracle):
    for n in (0, 1, 7, 1000):
        cols = wire_columns(n)
        for lo, hi in {(0, n), (n, n), (max(n - 1, 0), n), (min(3, n), max(n - 2, min(3, n)))}:
            assert ref_serialize(cols, lo, hi) == oracle.chunk_serialize(host_chunk(cols, n), lo, hi).tobytes(), (n, lo, hi)
    cols = [random_column(k, TYPES[k % 13], 50, np.random.default_rng(k), 0.5 if k % 3 else None) for k in range(32)]
    assert ref_serialize(cols, 5, 45) == oracle.chunk_serialize(host_chunk(cols, 50), 5, 45).tobytes()
    assert ref_serialize([], 0, 0) == struct.pack("<II", 1, 0)


# =============================================================================================
# GPU helpers
# =============================================================================================
MEM = {"host": abi.MEM_HOST, "pinned": abi.MEM_HOST_PINNED, "device": abi.MEM_DEVICE}


class Placed:
    """columns copied into `mem` (host, pinned or device).  offset: each column starts at row 1 of a larger buffer, and a
    16-byte column 8 bytes in, so that no column is 16-byte aligned (the null bytes start 1 byte in)"""

    def __init__(self, cols, n, mem, offset=False):
        self.keep = []
        spec = []
        for c in cols:
            off = (8 if c.w == 16 else c.w) if offset else 0
            dp = self._place(c.raw, mem, off)
            if offset and c.n:
                assert dp % 16 != 0 and dp % min(c.w, 8) == 0
            np_ = None if c.nulls is None else self._place(c.nulls, mem, 1 if offset else 0)
            spec.append((c.slot, dp, np_, c.typ))
        self.chunk = Chunk(spec, num_rows=n, mem=MEM[mem])

    def _place(self, raw, mem, off):
        size = len(raw) + off + 16
        if mem == "host":
            a = np.zeros(size, dtype=np.uint8)
            a[off:off + len(raw)] = np.frombuffer(raw, dtype=np.uint8)
            self.keep.append(a)
            return a.ctypes.data + off
        import torch
        if mem == "pinned":
            t = torch.zeros(size, dtype=torch.uint8).pin_memory()
            t.numpy()[off:off + len(raw)] = np.frombuffer(raw, dtype=np.uint8)
        else:
            t = torch.zeros(size, dtype=torch.uint8, device="cuda")
            if raw:
                t[off:off + len(raw)] = torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).cuda()
        self.keep.append(t)
        return t.data_ptr() + off


def check_hash(gpu, ctx, cols, slots, fn, red, nch, chunk=None, label=""):
    n = cols[0].n
    x = gpu.Xchg(ctx, abi.make_part_desc(slots, nch, hash_fn=fn, reduce_op=red))
    try:
        hv, ch = x.hash(chunk if chunk is not None else host_chunk(cols, n))
    finally:
        x.close()
    want = ref_hashes(cols, slots, fn, n)
    wch, _, _ = ref_partition(want, red, nch)
    bad = np.flatnonzero(hv != want)
    assert len(bad) == 0, f"{label}: {len(bad)} hash values differ, first at row {bad[0]}: {hv[bad[0]]:#x} vs {want[bad[0]]:#x}"
    assert np.array_equal(ch, wch), f"{label}: channel ids differ"
    return want


def check_partition(gpu, ctx, cols, slots, fn, red, nch, chunk=None, hv=None, label=""):
    n = cols[0].n
    x = gpu.Xchg(ctx, abi.make_part_desc(slots, nch, hash_fn=fn, reduce_op=red))
    try:
        out, offs = x.partition(chunk if chunk is not None else host_chunk(cols, n))
        got = gpu.chunk_out_to_host(ctx, out)
    finally:
        x.close()
    hv = ref_hashes(cols, slots, fn, n) if hv is None else hv
    _, order, woffs = ref_partition(hv, red, nch)
    assert offs.tolist() == woffs.tolist(), f"{label}: channel offsets differ"
    assert len(got) == len(cols)
    for c, (slot, typ, data, nulls) in zip(cols, got):
        raw, nul = take_rows(c, order)
        assert slot == c.slot and typ == c.typ
        assert data.view(np.uint8).tobytes() == raw, f"{label}: slot {c.slot} (width {c.w}) data out of place"
        assert (nulls is None) == (nul is None), f"{label}: slot {c.slot} null column"
        assert nul is None or nulls.tobytes() == nul, f"{label}: slot {c.slot} null bytes out of place"
    return offs


# =============================================================================================
# GPU: hash values and channels
# =============================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("nullable", [False, True], ids=["plain", "nullable"])
@pytest.mark.parametrize("red", [MULHI, MODULO], ids=[REDUCE_NAME[r] for r in (MULHI, MODULO)])
@pytest.mark.parametrize("fn", [FNV, CRC, XXH3], ids=[HASH_NAME[f] for f in (FNV, CRC, XXH3)])
@pytest.mark.parametrize("typ", TYPES, ids=[TYPE_NAME[t] for t in TYPES])
def test_hash_at_type_edges(gpu, ctx, typ, fn, red, nullable):
    cols = [edge_column(typ, nullable, seed=typ)]
    check_hash(gpu, ctx, cols, [0], fn, red, 37, label=f"{TYPE_NAME[typ]}")


@pytest.mark.gpu
@pytest.mark.parametrize("fn", [FNV, CRC, XXH3], ids=[HASH_NAME[f] for f in (FNV, CRC, XXH3)])
@pytest.mark.parametrize("case", list(MULTI_KEY_CASES))
def test_hash_multi_key(gpu, ctx, case, fn):
    cols = multi_key_columns()
    check_hash(gpu, ctx, cols, MULTI_KEY_CASES[case], fn, MULHI, 37, label=case)


@pytest.mark.gpu
@pytest.mark.parametrize("red", [MULHI, MODULO], ids=[REDUCE_NAME[r] for r in (MULHI, MODULO)])
@pytest.mark.parametrize("fn", [FNV, CRC, XXH3], ids=[HASH_NAME[f] for f in (FNV, CRC, XXH3)])
@pytest.mark.parametrize("nch", CHANNEL_COUNTS)
def test_channel_counts(gpu, ctx, nch, fn, red):
    cols = channel_count_columns(fn, nch, 7)
    hv = check_hash(gpu, ctx, cols, [0], fn, red, nch, label=f"{nch} channels")
    offs = check_partition(gpu, ctx, cols, [0], fn, red, nch, hv=hv, label=f"{nch} channels")
    if red == MULHI:      # the extreme keys: channel 0 and channel n - 1 both hold rows
        assert offs[1] > 0 and offs[nch] - offs[nch - 1] > 0


@pytest.mark.gpu
def test_xchg_create_refuses_bad_descs(gpu, ctx):
    def refused(d):
        with pytest.raises(gpu.GpuError) as ei:
            gpu.Xchg(ctx, d)
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
    for nch in (0, 257, -1):
        refused(abi.make_part_desc([0], nch))
    d = abi.make_part_desc([], 8)
    refused(d)
    d = abi.make_part_desc([0, 1, 2, 3], 8)
    d.num_part_slots = 5
    refused(d)
    for fn in (-1, 3):
        refused(abi.make_part_desc([0], 8, hash_fn=fn))
    for red in (-1, 2):
        refused(abi.make_part_desc([0], 8, reduce_op=red))
    gpu.Xchg(ctx, abi.make_part_desc([0, 1, 2, 3], 256, hash_fn=XXH3, reduce_op=MODULO)).close()


# =============================================================================================
# GPU: partition layout
# =============================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("skew", LAYOUT_SKEWS)
@pytest.mark.parametrize("n", LAYOUT_ROWS)
def test_partition_layout(gpu, ctx, n, skew):
    cols, hv = layout_columns(n, skew)
    offs = check_partition(gpu, ctx, cols, [0], FNV, MULHI, LAYOUT_NCH, hv=hv, label=f"{n} rows, {skew}")
    sizes = np.diff(offs)
    if n and skew != "uniform":
        assert np.count_nonzero(sizes) == (2 if skew == "two_alternating" and n > 1 else 1)


@pytest.mark.gpu
def test_partition_column_limit(gpu, ctx):
    rng = np.random.default_rng(9)
    n = 1500
    cols = [Col(0, abi.TYPE_INT, rng.integers(0, 256, 4 * n, dtype=np.uint8).tobytes())]
    cols += [random_column(k, TYPES[k % 13], n, rng, 0.2 if k % 2 else None) for k in range(1, abi.SR_MAX_OUT_COLS)]
    check_partition(gpu, ctx, cols, [0, 5], XXH3, MULHI, 19, label="32 columns")
    x = gpu.Xchg(ctx, abi.make_part_desc([0], 19))
    try:
        with pytest.raises(gpu.GpuError):
            x.partition(host_chunk(cols + [random_column(40, abi.TYPE_INT, n, rng)], n))
    finally:
        x.close()


# =============================================================================================
# GPU: input and output memory
# =============================================================================================
def _mixed_columns(n, seed=13):
    rng = np.random.default_rng(seed)
    cols = []
    for k, w in enumerate((1, 2, 4, 8, 16)):
        cols.append(random_column(k, WIDTH_TYPE[w], n, rng, 0.2 if k % 2 else None))
        cols.append(random_column(10 + k, WIDTH_TYPE[w], n, rng, None if k % 2 else 0.3))
    cols.append(random_column(20, abi.TYPE_LARGEINT, n, rng, 0.15))
    return cols


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [False, True], ids=["aligned", "natural_not_16"])
@pytest.mark.parametrize("mem", ["host", "pinned", "device"])
def test_partition_input_memory(gpu, ctx, mem, offset):
    # a 16-byte column 8 bytes into a device buffer takes k_gather's two-word copies
    cols = _mixed_columns(5000)
    p = Placed(cols, 5000, mem, offset)
    for fn, slots in ((FNV, [14, 1]), (CRC, [20]), (XXH3, [4, 12, 0])):
        check_hash(gpu, ctx, cols, slots, fn, MULHI, 29, chunk=p.chunk, label=f"{mem}/{HASH_NAME[fn]}")
        check_partition(gpu, ctx, cols, slots, fn, MULHI, 29, chunk=p.chunk, label=f"{mem}/{HASH_NAME[fn]}")


@pytest.mark.gpu
def test_hash_into_device_memory_and_after_a_refused_call(gpu, ctx):
    import torch
    cols = _mixed_columns(3001)
    chunk = host_chunk(cols, 3001)
    x = gpu.Xchg(ctx, abi.make_part_desc([14, 2], 64, hash_fn=XXH3, reduce_op=MODULO))
    try:
        hv = torch.zeros(3001 + 1, dtype=torch.int32, device="cuda")
        ch = torch.zeros(3001 + 1, dtype=torch.int32, device="cuda")
        ctx.check(gpu.lib().sr_xchg_hash(x.h, chunk.ref(), hv.data_ptr() + 4, ch.data_ptr() + 4, abi.MEM_DEVICE))
        ctx.sync()
        want = ref_hashes(cols, [14, 2], XXH3, 3001)
        wch, order, woffs = ref_partition(want, MODULO, 64)
        assert np.array_equal(hv.cpu().numpy()[1:].view(np.uint32), want)
        assert np.array_equal(ch.cpu().numpy()[1:].view(np.uint32), wch)
        missing = host_chunk([c for c in cols if c.slot != 2], 3001)
        for call in (lambda: x.hash(missing), lambda: x.partition(missing)):
            with pytest.raises(gpu.GpuError) as ei:
                call()
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
            got_hv, got_ch = x.hash(chunk)
            assert np.array_equal(got_hv, want) and np.array_equal(got_ch, wch)
            out, offs = x.partition(chunk)
            assert offs.tolist() == woffs.tolist()
            assert gpu.chunk_out_to_host(ctx, out)[9][2].view(np.uint8).tobytes() == take_rows(cols[9], order)[0]
    finally:
        x.close()


@pytest.mark.gpu
def test_device_columns_must_be_naturally_aligned(gpu, ctx):
    # a device column 1 byte short of its natural alignment is refused before any launch; the next call with an aligned
    # view of the same bytes runs
    import torch
    n = 2000
    rng = np.random.default_rng(4)
    for w in (2, 4, 8, 16):
        c = random_column(0, WIDTH_TYPE[w], n, rng)
        buf = torch.from_numpy(np.frombuffer(c.raw + bytes(32), dtype=np.uint8).copy()).cuda()
        x = gpu.Xchg(ctx, abi.make_part_desc([0], 8))
        try:
            for bad in ({2: 1, 4: 2, 8: 4, 16: 4}[w], 1):
                with pytest.raises(gpu.GpuError) as ei:
                    x.partition(Chunk([(0, buf.data_ptr() + bad, None, c.typ)], num_rows=n, mem=abi.MEM_DEVICE))
                assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
            ok = Placed([c], n, "device", offset=True)
            check_partition(gpu, ctx, [c], [0], FNV, MULHI, 8, chunk=ok.chunk, label=f"width {w}")
        finally:
            x.close()
    # the other entry points that take device columns in place
    sc = gpu.Scan(ctx, abi.ScanDesc([abi.make_pred(0, abi.PRED_GT, 0)], out_slots=[0]))
    try:
        buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
        with pytest.raises(gpu.GpuError) as ei:
            sc.evaluate(Chunk([(0, buf.data_ptr() + 2, None, abi.TYPE_INT)], num_rows=8, mem=abi.MEM_DEVICE))
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
        assert sc.evaluate(Chunk([(0, buf.data_ptr() + 4, None, abi.TYPE_INT)], num_rows=8, mem=abi.MEM_DEVICE)).tolist() == [0] * 8
    finally:
        sc.close()
    keys = torch.zeros(64, dtype=torch.uint8, device="cuda")
    buckets = torch.zeros(8, dtype=torch.int32, device="cuda")
    L = gpu.lib()
    assert L.sr_join_key_hash(ctx.h, keys.data_ptr() + 4, abi.TYPE_BIGINT, 4, 8, buckets.data_ptr(), abi.MEM_DEVICE) == abi.SR_ERR_INVALID_ARGUMENT
    ctx.check(L.sr_join_key_hash(ctx.h, keys.data_ptr() + 8, abi.TYPE_BIGINT, 4, 8, buckets.data_ptr(), abi.MEM_DEVICE))
    ctx.sync()
    assert buckets.cpu().tolist()[:4] == [ctx.join_key_hash(np.zeros(1, dtype=np.int64), 8)[0]] * 4


@pytest.mark.gpu
@pytest.mark.parametrize("src_off,dst_off", [(0, 0), (8, 0), (0, 8), (8, 8)])
def test_gather_sixteen_byte_values(gpu, ctx, src_off, dst_off):
    # sr_gather of a 16-byte column: int4 copies when source and destination are 16-byte aligned, two 8-byte words when
    # either is only 8-byte aligned; a pointer that is not 8-byte aligned is refused
    import torch
    rng = np.random.default_rng(src_off * 3 + dst_off)
    n_src, n = 777, 5000
    src_raw = rng.integers(0, 256, 16 * n_src, dtype=np.uint8)
    index = rng.integers(0, n_src, n).astype(np.uint32)
    index[:2] = [0, n_src - 1]
    src = torch.from_numpy(np.concatenate([np.zeros(src_off, np.uint8), src_raw])).cuda()
    dst = torch.zeros(16 * n + dst_off, dtype=torch.uint8, device="cuda")
    idx = torch.from_numpy(index.view(np.int32)).cuda()
    L = gpu.lib()
    ctx.check(L.sr_gather(ctx.h, src.data_ptr() + src_off, abi.TYPE_DECIMAL128, idx.data_ptr(), n, dst.data_ptr() + dst_off, abi.MEM_DEVICE))
    ctx.sync()
    assert dst.cpu().numpy()[dst_off:].tobytes() == src_raw.reshape(-1, 16)[index].tobytes()
    for bad_src, bad_dst in ((4, 0), (0, 4), (1, 1)):
        rc = L.sr_gather(ctx.h, src.data_ptr() + bad_src, abi.TYPE_DECIMAL128, idx.data_ptr(), n, dst.data_ptr() + bad_dst, abi.MEM_DEVICE)
        assert rc == abi.SR_ERR_INVALID_ARGUMENT


@pytest.mark.gpu
@pytest.mark.parametrize("threshold", [100, 50, 3], ids=["all_pass", "half_pass", "sparse"])
@pytest.mark.parametrize("offset", [False, True], ids=["aligned", "natural_not_16"])
def test_scan_filter_carries_16_byte_device_columns(gpu, ctx, offset, threshold):
    # sr_scan_filter compacts the device columns in place (k_scan_compact): 16-byte values by int4 only when the column is
    # 16-byte aligned.  half_pass takes the staged kernel (a quarter or more of the rows survive), sparse the direct one.
    n = 5003
    rng = np.random.default_rng(threshold + offset)
    v = rng.integers(0, 100, n, dtype=np.int32)
    cols = [Col(0, abi.TYPE_INT, v.tobytes()), random_column(1, abi.TYPE_DECIMAL128, n, rng),
            random_column(2, abi.TYPE_LARGEINT, n, rng, 0.3), random_column(3, abi.TYPE_BIGINT, n, rng, 0.2)]
    p = Placed(cols, n, "device", offset=offset)
    sc = gpu.Scan(ctx, abi.ScanDesc([abi.make_pred(0, abi.PRED_LT, threshold)], out_slots=[0, 1, 2, 3]))
    try:
        got = gpu.chunk_out_to_host(ctx, sc.filter(p.chunk))
    finally:
        sc.close()
    sel = np.flatnonzero(v < threshold)
    for c, (slot, typ, data, nulls) in zip(cols, got):
        raw, nul = take_rows(c, sel)
        assert slot == c.slot and data.view(np.uint8).tobytes() == raw, f"slot {c.slot} (width {c.w})"
        assert (nulls is None) == (nul is None) and (nul is None or nulls.tobytes() == nul), f"slot {c.slot} nulls"


@pytest.mark.gpu
def test_rf_merge_reads_a_device_directory_in_place(gpu, ctx):
    # the bloom directory of another filter, merged from device memory: 4-byte aligned is read in place, less is refused
    import torch
    rng = np.random.default_rng(21)
    a = Chunk([(0, rng.integers(-10**6, 10**6, 3000, dtype=np.int32), None)])
    b = Chunk([(0, rng.integers(-10**6, 10**6, 3000, dtype=np.int32), None)])
    rfs = [gpu.RuntimeFilter(ctx, abi.TYPE_INT, 6000) for _ in range(3)]
    try:
        for rf, ch in zip(rfs, (a, a, b)):
            rf.insert(ch, 0)
        d, info = rfs[2].directory(), rfs[2].info()
        rfs[0].merge(d, info)                                         # host directory: the expected result
        dev = torch.zeros(d.nbytes + 8, dtype=torch.uint8, device="cuda")
        dev[4:4 + d.nbytes] = torch.from_numpy(d.view(np.uint8)).cuda()
        L = gpu.lib()
        assert L.sr_rf_merge_directory(rfs[1].h, dev.data_ptr() + 2, d.nbytes, abi.MEM_DEVICE, C.byref(info)) == abi.SR_ERR_INVALID_ARGUMENT
        ctx.check(L.sr_rf_merge_directory(rfs[1].h, dev.data_ptr() + 4, d.nbytes, abi.MEM_DEVICE, C.byref(info)))
        ctx.sync()
        assert np.array_equal(rfs[1].directory(), rfs[0].directory())
        i0, i1 = rfs[0].info(), rfs[1].info()
        assert (i1.min_value, i1.max_value, i1.num_inserted) == (i0.min_value, i0.max_value, i0.num_inserted)
    finally:
        for rf in rfs:
            rf.close()


@pytest.mark.gpu
def test_join_carries_an_8_byte_aligned_16_byte_probe_column(gpu, ctx):
    # the probe side's output gather reads the device column in place
    n = 3000
    rng = np.random.default_rng(12)
    keys = rng.permutation(n).astype(np.int32)
    dec = random_column(1, abi.TYPE_DECIMAL128, n, rng, 0.2)
    kc = Col(0, abi.TYPE_INT, keys.tobytes())
    p = Placed([kc, dec], n, "device", offset=True)
    build = Chunk([(10, np.arange(n, dtype=np.int32), None), (11, np.arange(n, dtype=np.int64) * 3, None)])
    j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [10], [0], [abi.TYPE_INT], build_out=[11], probe_out=[0, 1]))
    try:
        j.append_build(build)
        j.build_finish()
        got = gpu.chunk_out_to_host(ctx, j.probe(p.chunk))
    finally:
        j.close()
    gk = got[0][2]
    assert sorted(gk.tolist()) == list(range(n))
    raw, nul = take_rows(dec, np.argsort(keys)[gk])             # the probe row holding each output row's key
    assert got[1][2].view(np.uint8).tobytes() == raw and got[1][3].tobytes() == nul
    assert np.array_equal(got[2][2], gk.astype(np.int64) * 3)


# =============================================================================================
# GPU: the wire format
# =============================================================================================
def serialize(gpu, ctx, chunk, lo, hi, dst_mem):
    """sr_chunk_serialize into a host, pinned or device (3 bytes into the buffer) destination -> (bytes, meta)"""
    import torch
    L = gpu.lib()
    size = L.sr_chunk_serialized_size(chunk.ref(), lo, hi)
    assert size >= 8
    meta = abi.sr_chunk_pb_meta()
    if dst_mem == "host":
        buf = np.full(size, 0xAB, dtype=np.uint8)
        ctx.check(L.sr_chunk_serialize(ctx.h, chunk.ref(), lo, hi, buf.ctypes.data, size, abi.MEM_HOST, C.byref(meta)))
        return buf.tobytes(), meta
    if dst_mem == "pinned":
        t = torch.full((size,), 0xAB, dtype=torch.uint8).pin_memory()
        ctx.check(L.sr_chunk_serialize(ctx.h, chunk.ref(), lo, hi, t.data_ptr(), size, abi.MEM_HOST_PINNED, C.byref(meta)))
        return t.numpy().tobytes(), meta
    t = torch.full((size + 3,), 0xAB, dtype=torch.uint8, device="cuda")
    ctx.check(L.sr_chunk_serialize(ctx.h, chunk.ref(), lo, hi, t.data_ptr() + 3, size, abi.MEM_DEVICE, C.byref(meta)))
    ctx.sync()
    return t.cpu().numpy()[3:].tobytes(), meta


def deserialize(gpu, ctx, sd, payload, meta, src_mem):
    """-> (status, columns on the host or None)"""
    import torch
    out = abi.sr_chunk_out()
    if src_mem == "host":
        a = np.frombuffer(payload, dtype=np.uint8).copy() if payload else np.zeros(1, dtype=np.uint8)
        rc = gpu.lib().sr_chunk_deserialize(sd.h, a.ctypes.data, len(payload), abi.MEM_HOST, C.byref(meta), C.byref(out))
    else:
        t = torch.zeros(len(payload) + 1, dtype=torch.uint8, device="cuda")
        if payload:
            t[1:] = torch.from_numpy(np.frombuffer(payload, dtype=np.uint8).copy()).cuda()
        rc = gpu.lib().sr_chunk_deserialize(sd.h, t.data_ptr() + 1, len(payload), abi.MEM_DEVICE, C.byref(meta), C.byref(out))
        ctx.sync()
    if rc != 0:
        return rc, None
    return 0, (out.num_rows, gpu.chunk_out_to_host(ctx, out))


def check_columns_back(cols, lo, hi, back, label):
    rows, got = back
    assert rows == hi - lo and len(got) == len(cols), label
    for c, (slot, typ, data, nulls) in zip(cols, got):
        assert slot == c.slot and typ == c.typ, label
        assert data.view(np.uint8).tobytes() == c.raw[lo * c.w:hi * c.w], f"{label}: slot {c.slot}"
        assert (nulls is None) == (c.nulls is None), f"{label}: slot {c.slot}"
        assert nulls is None or nulls.tobytes() == c.nulls[lo:hi], f"{label}: slot {c.slot}"


def _meta_for(cols, rows):
    m = abi.sr_chunk_pb_meta()
    m.num_cols, m.num_rows = len(cols), rows
    m.serialized_size = len(ref_serialize(cols, 0, 0)) + sum((rows if c.nulls is not None else 0) + rows * c.w for c in cols)
    for k, c in enumerate(cols):
        m.slot_ids[k], m.types[k], m.is_nulls[k] = c.slot, c.typ, 1 if c.nulls is not None else 0
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("dst_mem", ["host", "pinned", "device"])
@pytest.mark.parametrize("src_mem", ["host", "pinned", "device"])
def test_wire_format_memory_kinds(gpu, ctx, src_mem, dst_mem):
    n = 1000
    cols = wire_columns(n)
    p = Placed(cols, n, src_mem, offset=src_mem == "device")
    sd = gpu.Serde(ctx)
    try:
        for lo, hi in ((0, n), (n, n), (n - 1, n), (3, n - 2), (0, 1)):
            label = f"{src_mem}->{dst_mem} [{lo}, {hi})"
            payload, meta = serialize(gpu, ctx, p.chunk, lo, hi, dst_mem)
            assert payload == ref_serialize(cols, lo, hi), label
            assert meta.serialized_size == len(payload) and meta.num_rows == hi - lo and meta.num_cols == len(cols)
            assert list(meta.is_nulls[:len(cols)]) == [int(c.nulls is not None) for c in cols]
            assert list(meta.is_consts[:len(cols)]) == [0] * len(cols)
            for from_mem in ("host", "device"):
                rc, back = deserialize(gpu, ctx, sd, payload, meta, from_mem)
                assert rc == 0, label
                check_columns_back(cols, lo, hi, back, f"{label}, parsed from {from_mem}")
    finally:
        sd.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["zero_rows", "zero_cols", "max_cols"])
def test_wire_format_shapes(gpu, ctx, shape):
    rng = np.random.default_rng(6)
    n = {"zero_rows": 0, "zero_cols": 5, "max_cols": 300}[shape]
    if shape == "zero_cols":
        cols = []
    elif shape == "zero_rows":
        cols = wire_columns(0)
    else:
        cols = [random_column(k, TYPES[k % 13], n, rng, 0.4 if k % 3 else None) for k in range(abi.SR_MAX_OUT_COLS)]
    sd = gpu.Serde(ctx)
    try:
        for mem in ("host", "device"):
            p = Placed(cols, n, mem)
            for dst in ("host", "device"):
                payload, meta = serialize(gpu, ctx, p.chunk, 0, n, dst)
                assert payload == ref_serialize(cols, 0, n)
                for from_mem in ("host", "device"):
                    rc, back = deserialize(gpu, ctx, sd, payload, meta, from_mem)
                    assert rc == 0
                    check_columns_back(cols, 0, n, back, shape)
        if shape == "max_cols":
            over = host_chunk(cols + [random_column(77, abi.TYPE_INT, n, rng)], n)
            with pytest.raises(gpu.GpuError):
                gpu.chunk_serialize(ctx, over)
    finally:
        sd.close()


def _malformed_cases():
    """(label, payload, meta, expected status) built from a good payload of 3 columns x 5 rows"""
    rng = np.random.default_rng(8)
    rows = 5
    cols = [random_column(1, abi.TYPE_INT, rows, rng, 0.4), random_column(2, abi.TYPE_DECIMAL128, rows, rng),
            random_column(3, abi.TYPE_SMALLINT, rows, rng, 0.4)]
    good = ref_serialize(cols, 0, rows)
    INV, NS = abi.SR_ERR_INVALID_ARGUMENT, abi.SR_ERR_NOT_SUPPORTED

    def meta(size=None, **kw):
        m = _meta_for(cols, rows)
        m.serialized_size = len(good) if size is None else size
        for k, v in kw.items():
            setattr(m, k, v)
        return m
    yield "version 0", struct.pack("<I", 0) + good[4:], meta(), INV
    yield "version 2", struct.pack("<I", 2) + good[4:], meta(), INV
    for k in range(8):
        yield f"{k} bytes", good[:k], meta(k), INV
    # every header word of the columns and a cut inside each column's bytes
    words, off = [], 8
    for c in cols:
        if c.nulls is not None:
            words.append(off)
            off += 4 + rows
        words.append(off)
        off += 4 + rows * c.w
    for w in words:
        for cut in (w, w + 2, w + 4 + 1):
            yield f"truncated at {cut}", good[:cut], meta(cut), INV
    yield "truncated by 1", good[:-1], meta(len(good) - 1), INV
    # null column of 0 bytes, the rest consistent (the header num_rows and the data sizes still say 5 rows)
    no_nulls = good[:8] + struct.pack("<I", 0) + good[8 + 4 + rows:]
    yield "null column of 0 bytes", no_nulls, meta(len(no_nulls)), INV
    short_null = good[:8] + struct.pack("<I", rows - 1) + good[12:12 + rows - 1] + good[12 + rows:]
    yield "null column of rows - 1 bytes", short_null, meta(len(short_null)), INV
    # data column one value short (the rest consistent)
    d0 = 8 + 4 + rows
    short_data = good[:d0] + struct.pack("<I", 4 * (rows - 1)) + good[d0 + 4:d0 + 4 + 4 * (rows - 1)] + good[d0 + 4 + 4 * rows:]
    yield "data column of rows - 1 values", short_data, meta(len(short_data)), INV
    long_data = good[:d0] + struct.pack("<I", 4 * rows + 4) + good[d0 + 4:]
    yield "data size word too large", long_data, meta(), INV
    m = meta()
    m.types[1] = 0
    yield "type 0", good, m, INV
    m = meta()
    m.types[2] = 14
    yield "type 14", good, m, INV
    yield "num_cols -1", good, meta(num_cols=-1), INV
    yield "num_cols 33", good + bytes(64), meta(num_cols=33), INV
    yield "trailing byte", good + b"\0", meta(len(good) + 1), INV
    yield "trailing column", good + struct.pack("<I", 20) + bytes(20), meta(len(good) + 24), INV
    yield "serialized_size != bytes", good, meta(len(good) + 1), INV
    m = meta()
    m.is_consts[1] = 1
    yield "is_consts", good, m, NS
    yield "meta.num_rows 4", good, meta(num_rows=4), INV
    yield "meta.num_rows 6", good, meta(num_rows=6), INV
    header_rows = good[:4] + struct.pack("<I", 4) + good[8:]
    yield "header num_rows 4", header_rows, meta(), INV
    yield "good", good, meta(), (cols, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("src_mem", ["host", "device"])
def test_deserialize_refuses_malformed_payloads(gpu, ctx, src_mem):
    cases = list(_malformed_cases())
    _, good, good_meta, (cols, rows) = cases[-1]
    sd = gpu.Serde(ctx)
    try:
        for label, payload, meta, want in cases[:-1]:
            rc, _ = deserialize(gpu, ctx, sd, payload, meta, src_mem)
            assert rc == want, f"{label}: status {rc}, want {want}"
            rc, back = deserialize(gpu, ctx, sd, good, good_meta, src_mem)      # the handle is still good
            assert rc == 0, f"after {label}"
            check_columns_back(cols, 0, rows, back, f"after {label}")
    finally:
        sd.close()


# =============================================================================================
# GPU: end to end -- partition, one payload per channel, parse on the receiver
# =============================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("fn", [FNV, CRC, XXH3], ids=[HASH_NAME[f] for f in (FNV, CRC, XXH3)])
def test_exchange_end_to_end(gpu, ctx, fn):
    import torch
    n, nch = 20_000, 13
    rng = np.random.default_rng(40 + fn)
    cols = [random_column(k, typ, n, rng, 0.2 if k % 2 else None) for k, typ in enumerate(TYPES)]
    slots = [3, 12, 1]
    hv = ref_hashes(cols, slots, fn, n)
    _, order, woffs = ref_partition(hv, MULHI, nch)
    moved = [Col(c.slot, c.typ, *take_rows(c, order)) for c in cols]
    x = gpu.Xchg(ctx, abi.make_part_desc(slots, nch, hash_fn=fn))
    sd = gpu.Serde(ctx)
    try:
        out, offs = x.partition(host_chunk(cols, n))
        assert offs.tolist() == woffs.tolist()
        view = gpu.chunk_out_as_view(out)
        L = gpu.lib()
        for c in range(nch):
            lo, hi = int(offs[c]), int(offs[c + 1])
            size = L.sr_chunk_serialized_size(view.ref(), lo, hi)
            buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
            meta = abi.sr_chunk_pb_meta()
            ctx.check(L.sr_chunk_serialize(ctx.h, view.ref(), lo, hi, buf.data_ptr(), size, abi.MEM_DEVICE, C.byref(meta)))
            assert buf.cpu().numpy().tobytes() == ref_serialize(moved, lo, hi), f"channel {c}"
            res = abi.sr_chunk_out()
            ctx.check(L.sr_chunk_deserialize(sd.h, buf.data_ptr(), size, abi.MEM_DEVICE, C.byref(meta), C.byref(res)))
            sel = np.flatnonzero(((hv.astype(np.uint64) * np.uint64(nch)) >> np.uint64(32)) == c)     # the rows the reference sends to c
            check_columns_back([Col(k.slot, k.typ, *take_rows(k, sel)) for k in cols], 0, hi - lo, (res.num_rows, gpu.chunk_out_to_host(ctx, res)),
                               f"channel {c}")
    finally:
        sd.close()
        x.close()
