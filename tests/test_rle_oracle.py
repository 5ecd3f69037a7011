"""The RLE codec at bit width 1 (BOOLEAN RLE pages, RLE_NULL null maps) and the bitshuffle null maps, restated on the CPU in
bshuf_oracle: known answers, hand-built streams the encoder never writes, every malformed case, round trips.  No GPU."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _b(*xs):
    return np.array(xs, dtype=np.uint8)


def _vlq(v):
    out = []
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    return out + [v]


def test_expand_word_formula_all_bytes():
    # the device's literal expansion: one byte -> 8 flag bytes in one 64-bit word, flag i = bit i
    b = np.arange(256, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = ((((b * np.uint64(0x0101010101010101)) & np.uint64(0x8040201008040201)) + np.uint64(0x00406070787C7E7F)) >> np.uint64(7)) \
            & np.uint64(0x0101010101010101)
    got = x.astype("<u8").view(np.uint8).reshape(256, 8)
    want = ((np.arange(256)[:, None] >> np.arange(8)[None, :]) & 1).astype(np.uint8)
    assert (got == want).all()


def test_known_answer(bo):
    v = _b(*([0] * 100 + [1, 1, 1]))
    # a literal group for the last three values: a stream the decoder takes as written
    assert (bo.rle_decode(_b(0xC8, 0x01, 0x00, 0x03, 0x07), 103) == v).all()
    assert (bo.rle_bool_page_decode(_b(0x67, 0, 0, 0, 0xC8, 0x01, 0x00, 0x03, 0x07)) == v).all()
    # RleEncoder::Flush writes a pending tail of one value as a repeated run
    assert bo.rle_encode(v).tobytes() == bytes([0xC8, 0x01, 0x00, 0x06, 0x01])
    assert bo.rle_bool_page_encode(v).tobytes() == bytes([0x67, 0, 0, 0, 0xC8, 0x01, 0x00, 0x06, 0x01])


def test_encoder_greedy_rules(bo):
    # 8 equal values make a repeated run; literal runs hold at most 63 groups per header
    assert bo.rle_encode(_b(*[1] * 8)).tobytes() == bytes([0x10, 0x01])
    alt = np.tile(_b(0, 1), 63 * 4)                                  # 63 groups of 01010101
    s = bo.rle_encode(alt)
    assert s[0] == (63 << 1 | 1) and len(s) == 64 and (s[1:] == 0xAA).all()
    s = bo.rle_encode(np.tile(_b(0, 1), 64 * 4))                      # 64 groups: 63, then a second literal run of 1
    assert s.tobytes() == bytes([127] + [0xAA] * 63 + [3, 0xAA])
    s = bo.rle_encode(np.tile(np.repeat(_b(0, 1), 8), 3))              # alternating runs of 8: repeated runs
    assert s.tobytes() == bytes([0x10, 0x00, 0x10, 0x01] * 3)


def test_multibyte_headers(bo):
    for count in (2 ** 14, 2 ** 14 + 3, 2 ** 21, 2 ** 21 + 5):
        h = _vlq(count << 1)
        assert len(h) == (3 if count < 2 ** 20 else 4)
        s = _b(*h, 1, 0x03, 0x05)                                     # count ones, then a literal group 1, 0, 1
        got = bo.rle_decode(s, count + 3)
        assert got[:count].all() and got[count:].tolist() == [1, 0, 1]
    # a 5-byte header (35 bits): the largest the format has
    s = _b(0x80 | 0x10, 0x80, 0x80, 0x80, 0x00, 0x01)                 # count 8 in a padded 5-byte header
    assert bo.rle_decode(s, 8).tolist() == [1] * 8


def test_literal_run_longer_than_the_encoder_writes(bo):
    groups = 200                                                      # header 401 (2 bytes); the encoder stops at 63
    rng = np.random.default_rng(1)
    body = rng.integers(0, 256, groups, dtype=np.uint8)
    s = np.concatenate([_b(*_vlq(groups << 1 | 1)), body])
    want = np.unpackbits(body, bitorder="little")
    assert (bo.rle_decode(s, 8 * groups) == want).all()
    assert (bo.rle_decode(s, 8 * groups - 5) == want[:-5]).all()


def test_values_and_bytes_past_the_count_are_not_read(bo):
    # padding of the last group, a repeated run the count cuts short, trailing bytes -- garbage included
    assert bo.rle_decode(_b(0x03, 0xFF, 0xEE, 0x99), 3).tolist() == [1, 1, 1]
    assert bo.rle_decode(_b(0x20, 0x01, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0xFF), 5).tolist() == [1] * 5
    # a literal run claiming more groups than the stream holds: only the groups up to the count are read
    assert bo.rle_decode(_b(63 << 1 | 1, 0x0F), 4).tolist() == [1, 1, 1, 1]
    # count 0: nothing is read at all
    assert len(bo.rle_decode(_b(0xFF, 0xFF), 0)) == 0
    assert len(bo.rle_bool_page_decode(_b(0, 0, 0, 0, 0x00))) == 0


MALFORMED = [
    ("header longer than 5 bytes", _b(0x80, 0x80, 0x80, 0x80, 0x80, 0x01, 0x01), 8),
    ("header cut off by the end", _b(0x10, 0x01, 0x80), 9),
    ("header cut off at once", _b(0x80), 1),
    ("literal bytes past the end", _b(0x05, 0xFF), 9),
    ("repeated value past the end", _b(0x10), 8),
    ("zero-length repeated run", _b(0x00, 0x01, 0x10, 0x01), 8),
    ("zero-length literal run", _b(0x01, 0x10, 0x01), 8),
    ("repeated value 2", _b(0x10, 0x02), 8),
    ("repeated value 255", _b(0x10, 0xFF), 3),
    ("stream ends before the count", _b(0x10, 0x01), 9),
    ("empty stream, rows to decode", _b(), 1),
]


@pytest.mark.parametrize("name,stream,n", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_malformed_streams(bo, name, stream, n):
    with pytest.raises(bo.CorruptPage):
        bo.rle_decode(stream, n)
    with pytest.raises(bo.CorruptPage):
        bo.rle_bool_page_decode(np.concatenate([np.array([n], dtype="<u4").view(np.uint8), stream]))


def test_short_bool_page(bo):
    for k in range(4):
        with pytest.raises(bo.CorruptPage):
            bo.rle_bool_page_decode(np.zeros(k, dtype=np.uint8))


def _patterns(n, rng):
    yield "zeros", np.zeros(n, np.uint8)
    yield "ones", np.ones(n, np.uint8)
    yield "random", rng.integers(0, 2, n).astype(np.uint8)
    yield "sparse", (rng.random(n) < 0.01).astype(np.uint8)
    yield "runs", np.repeat(np.arange((n + 999) // 1000) % 2, 1000)[:n].astype(np.uint8)
    yield "alternating_8", np.repeat(np.arange((n + 7) // 8) % 2, 8)[:n].astype(np.uint8)


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 8191, 8192, 8193])
def test_round_trips(bo, n):
    rng = np.random.default_rng(n)
    for name, v in _patterns(n, rng):
        assert (bo.rle_decode(bo.rle_encode(v), n) == v).all(), name
        assert (bo.rle_bool_page_decode(bo.rle_bool_page_encode(v)) == v).all(), name
        for enc in (bo.NULL_BITSHUFFLE, bo.NULL_RLE):
            m = bo.null_map_encode(v, enc)
            assert (len(m) == 0) == (not v.any()), name
            assert (bo.null_map_decode(m, n, enc) == v).all(), (name, enc)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 8191, 8192, 8193, 65_536])
def test_bitshuffle_map_is_the_padded_flags(bo, n):
    # the map is the block chain of a BIT_SHUFFLE page of ALIGN_UP(n, 8) one-byte flags: decoded with the padding, the
    # padding is zeros
    rng = np.random.default_rng(n)
    f = (rng.random(n) < 0.3).astype(np.uint8)
    f[0] = 1
    m = bo.null_map_encode(f, bo.NULL_BITSHUFFLE)
    padded = (n + 7) // 8 * 8
    hdr = np.array([padded, 16 + len(m), padded, 1], dtype="<u4").view(np.uint8)
    got = bo.bitshuffle_decode(np.concatenate([hdr, m]), 1)
    assert len(got) == padded and (got[:n] == f).all() and not got[n:].any()
    with pytest.raises(bo.CorruptPage):                               # the chain must end exactly at the map's size
        bo.null_map_decode(np.concatenate([m, _b(0)]), n, bo.NULL_BITSHUFFLE)
    with pytest.raises(bo.CorruptPage):
        bo.null_map_decode(m[:-1], n, bo.NULL_BITSHUFFLE)
