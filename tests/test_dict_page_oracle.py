"""Dictionary-encoded (DICT_ENCODING) column pages restated on the CPU (bshuf_oracle): the segment's dictionary page
(BinaryPlainPage) and its data pages (a mode word, then a BIT_SHUFFLE page of int32 codes), pinned by pages spelled out
byte by byte; and the host side of the same pages (starrocks_b200/host/exec/global_dict.h) through tests/cpp."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _le32(*vs):
    return b"".join(int(v).to_bytes(4, "little") for v in vs)


def test_dictionary_page_spelled_out(bo):
    # BinaryPlainPageBuilder::finish: the words back to back, their start offsets, the count
    want = b"AMERICA" + b"ASIA" + _le32(0, 7, 7, 3)
    page = bo.binary_plain_page_encode([b"AMERICA", b"", b"ASIA"])
    assert page.tobytes() == want
    assert bo.binary_plain_page_decode(np.frombuffer(want, dtype=np.uint8)) == [b"AMERICA", b"", b"ASIA"]
    assert bo.binary_plain_page_encode([]).tobytes() == _le32(0)
    assert bo.binary_plain_page_decode(bo.binary_plain_page_encode([])) == []


def test_data_page_spelled_out(bo):
    # codes 2, 0, 1: mode word 5, then a bitshuffle page -- header (3 values, 54 bytes, padded to 8, 4-byte elements) and
    # one block: the 32 bytes of the transposed codes (row 0 = bit 0 of byte 0 of the 8 values = 0b100, row 1 = 0b001)
    # as one LZ4 sequence of 32 literals (token 0xF0, length byte 17), behind its big-endian length 34
    rows = bytes([4, 1] + [0] * 30)
    stream = bytes([0xF0, 17]) + rows
    page = _le32(5) + _le32(3, 16 + 4 + len(stream), 8, 4) + len(stream).to_bytes(4, "big") + stream
    p = np.frombuffer(page, dtype=np.uint8)
    assert bo.dict_page_decode(p).tolist() == [2, 0, 1]
    mine = bo.dict_page_encode(np.array([2, 0, 1], dtype=np.int32))
    assert mine[:4].tobytes() == _le32(5) and mine[4:8].tobytes() == _le32(3)
    assert mine[12:20].tobytes() == _le32(8, 4) and int.from_bytes(mine[8:12].tobytes(), "little") == len(mine) - 4
    assert bo.lz4_decompress(mine[24:], 32).tobytes() == rows                 # the same transposed block
    # the plain-mode page of a column whose dictionary overflowed: mode word 2, then a BinaryPlainPage of strings
    assert bo.dict_page_plain_fallback([b"x", b"yz"]).tobytes() == _le32(2) + b"xyz" + _le32(0, 1, 2)


@pytest.mark.parametrize("n", [0, 1, 7, 8, 2048, 2049, 65_536])
def test_data_page_round_trip(bo, n):
    rng = np.random.default_rng(n)
    for hi in (1, 25, 256, 70_000):
        codes = rng.integers(0, hi, n).astype(np.int32)
        page = bo.dict_page_encode(codes)
        assert page[:4].tobytes() == _le32(5)
        assert (bo.dict_page_decode(page) == codes).all()
        assert (bo.bitshuffle_decode(page[4:], np.int32) == codes).all()      # the body is a plain bitshuffle page
    words = [bytes(rng.integers(0, 256, rng.integers(0, 12)).astype(np.uint8)) for _ in range(n % 3000)]
    assert bo.binary_plain_page_decode(bo.binary_plain_page_encode(words)) == words


def test_malformed_pages(bo):
    good = bo.dict_page_encode(np.arange(100, dtype=np.int32) % 7)
    for mode in (0, 2, 6, 0xFFFFFFFF):
        bad = good.copy()
        bad[:4] = np.frombuffer(_le32(mode), dtype=np.uint8)
        with pytest.raises(bo.CorruptPage):
            bo.dict_page_decode(bad)
    for bad in (good[:3], good[:18]):
        with pytest.raises(bo.CorruptPage):
            bo.dict_page_decode(bad)
    bad = good.copy()
    bad[16:20] = np.frombuffer(_le32(8), dtype=np.uint8)                     # 8-byte elements: not codes
    with pytest.raises(bo.CorruptPage):
        bo.dict_page_decode(bad)
    dpage = bo.binary_plain_page_encode([b"MFGR#1", b"MFGR#22", b"MFGR#3"])   # 19 bytes of words, offsets 0 6 13
    for at, v in ((-4, 9), (19 + 4, 14), (19 + 8, 20)):                       # a count that does not fit; offsets decrease / pass the array
        bad = dpage.copy()
        bad[at] = v
        with pytest.raises(bo.CorruptPage):
            bo.binary_plain_page_decode(bad)
    with pytest.raises(bo.CorruptPage):
        bo.binary_plain_page_decode(dpage[:3])


def test_host_dictionary_page_and_global_ids(tmp_path):
    """tests/cpp/dict_page_test: the host parse of a dictionary page (decode_binary_plain_page), its writer, and
    GlobalDictCodeConverter::global_ids() against decode_string_dict_codes.  Needs no GPU; built outside the tree."""
    binary = str(tmp_path / "dict_page_test")
    subprocess.check_call(["make", "-C", CPP, "-s", "-f", "dict_page_test.mk", "OUT=" + binary])
    r = subprocess.run([binary], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "DICT_PAGE_TEST_OK" in r.stdout
