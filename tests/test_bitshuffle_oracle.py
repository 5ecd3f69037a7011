"""The CPU restatement of BIT_SHUFFLE pages (bshuf_oracle): the bit transpose, the LZ4 block codec with its end-of-block
rules, and whole pages, pinned against liblz4's output and verdicts (tests/golden/bitshuffle_lz4.npz, written by
scripts/make_bitshuffle_golden.py) and, where the system liblz4 is present, against the library itself."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bitshuffle_lz4.npz")


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def golden():
    """-> [(name, kind, width, size, verdict, input bytes, output bytes)]"""
    g = np.load(GOLDEN)
    offs = np.concatenate([[0], np.cumsum(g["lengths"])])
    s = [np.ascontiguousarray(g["data"][offs[k]:offs[k + 1]]) for k in range(len(g["lengths"]))]
    return [(str(g["names"][i]), str(g["kind"][i]), int(g["width"][i]), int(g["size"][i]), int(g["verdict"][i]), s[2 * i], s[2 * i + 1])
            for i in range(len(g["names"]))]


def test_transpose_known_answer(bo):
    # bshuf_trans_bit_elem: row 8 * j + k = bit k of byte j of every element, element i at bit i % 8 of byte i / 8
    v = np.array([0xFF, 0x100, 0, 0, 0, 0, 0, 0x80000000], dtype=np.uint32)
    want = bytes([1] * 8 + [2] + [0] * 22 + [0x80])
    assert bo.trans_bit_elem(v).tobytes() == want
    assert bo.untrans_bit_elem(np.frombuffer(want, dtype=np.uint8), 4).view(np.uint32).tolist() == v.tolist()


@pytest.mark.parametrize("width", [1, 2, 4, 8, 16])
def test_transpose_matches_its_definition(bo, width):
    rng = np.random.default_rng(width)
    n = 8 * 37
    raw = rng.integers(0, 256, n * width).astype(np.uint8)
    bits = np.unpackbits(raw.reshape(n, width), axis=1, bitorder="little")          # [element, 8 * byte + bit]
    want = np.packbits(bits.T, axis=1, bitorder="little").reshape(-1)              # row r: bit r of every element, LSB first
    got = bo.trans_bit_elem(raw.view(np.dtype((np.void, width))))
    assert (got == want).all()
    assert (bo.untrans_bit_elem(got, width) == raw).all()


def test_golden_pages_and_streams(bo):
    # pages whose LZ4 blocks came from liblz4, and hand-built streams with liblz4's verdict and output
    cases = golden()
    assert {c[1] for c in cases} == {"page", "lz4"}
    for name, kind, width, size, verdict, data, want in cases:
        if kind == "page":
            assert (bo.bitshuffle_decode(data, width) == want).all(), name
            assert len(bo.bitshuffle_decode(bo.bitshuffle_encode(want, width), width)) == len(want), name
        elif verdict:
            assert (bo.lz4_decompress(data, size) == want).all(), name
        else:
            with pytest.raises(bo.CorruptPage):
                bo.lz4_decompress(data, size)


@pytest.mark.parametrize("width", [1, 2, 4, 8, 16])
def test_round_trip_edge_sizes(bo, width):
    rng = np.random.default_rng(100 + width)
    blk = 8192 // width
    for n in (0, 1, 7, 8, 9, blk, blk + 8, blk * 7 // 2):
        for raw in (rng.integers(0, 256, n * width).astype(np.uint8),                     # incompressible
                    np.repeat(rng.integers(0, 4, n * width // 50 + 1), 50)[:n * width].astype(np.uint8)):   # runs
            page = bo.bitshuffle_encode(raw, width)
            hdr = page[:16].view("<u4")
            assert hdr.tolist() == [n, len(page), (n + 7) // 8 * 8, width]
            assert (bo.bitshuffle_decode(page, width) == raw).all(), (width, n)


def test_compressor_emits_matches(bo):
    # a typical key column: the high bit rows are zero and must compress to matches, not literal-only blocks
    v = np.random.default_rng(3).integers(1, 3_000_000, 2048).astype(np.int32)
    page = bo.bitshuffle_encode(v)
    assert len(page) < 0.8 * v.nbytes
    assert (bo.bitshuffle_decode(page, np.int32) == v).all()


def test_malformed_pages_are_rejected(bo):
    v = np.arange(3000, dtype=np.int32) * 7
    good = bo.bitshuffle_encode(v)

    def with_word(k, x):
        p = good.copy()
        p[4 * k:4 * k + 4] = np.array([x], dtype="<u4").view(np.uint8)
        return p

    chain = good.copy()
    chain[16:20] = np.frombuffer((len(good)).to_bytes(4, "big"), dtype=np.uint8)        # the first block overruns the page
    big = good.copy()
    big[16:20] = np.frombuffer((8241).to_bytes(4, "big"), dtype=np.uint8)
    for bad in (good[:15], with_word(1, len(good) + 1), with_word(2, 3008), with_word(3, 8), chain, big, good[:-1]):
        with pytest.raises(bo.CorruptPage):
            bo.bitshuffle_decode(bad, np.int32)
    with pytest.raises(bo.CorruptPage):
        bo.bitshuffle_decode(good, np.int64)                                             # elem_size_bytes != the width asked for


def test_system_liblz4_interoperates(bo):
    # liblz4 decodes the oracle's streams and the oracle decodes liblz4's, on random and structured inputs
    L = bo.system_lz4()
    if L is None:
        pytest.skip("no system liblz4")
    rng = np.random.default_rng(9)
    inputs = [rng.integers(0, 256, n).astype(np.uint8) for n in (0, 1, 12, 13, 100, 8192)]
    inputs += [rng.integers(0, 3, n).astype(np.uint8) for n in (13, 64, 8192)]
    inputs += [np.zeros(8192, dtype=np.uint8), np.tile(np.arange(7, dtype=np.uint8), 1000), np.repeat(rng.integers(0, 256, 300), 27).astype(np.uint8)]
    inputs += [bo.trans_bit_elem(rng.integers(1, 3_000_000, 2048).astype(np.int32)), bo.trans_bit_elem(np.sort(rng.integers(0, 10**6, 1024)))]
    for x in inputs:
        ours = bo.lz4_compress(x)
        ok, out = bo.system_lz4_decompress(L, ours, len(x))
        assert ok and (out == x).all(), len(x)
        if len(x):
            theirs = bo.system_lz4_compress(L, x)
            assert (bo.lz4_decompress(theirs, len(x)) == x).all(), len(x)
    for w, dt in ((1, np.int8), (2, np.int16), (4, np.int32), (8, np.int64)):
        v = rng.integers(-100, 100, 8192 // w * 3 + 5).astype(dt)
        assert (bo.bitshuffle_decode(bo.bitshuffle_encode_with(L, v), dt) == v).all()
