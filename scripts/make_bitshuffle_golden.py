"""Writes tests/golden/bitshuffle_lz4.npz: BIT_SHUFFLE pages and LZ4 streams with the system liblz4's verdicts.

    python scripts/make_bitshuffle_golden.py

Needs the system liblz4 (liblz4.so.1).  The file lets the tests check the CPU codec (bshuf_oracle) and the device decoder
against real-library output on hosts without liblz4.  Layout (np.savez_compressed): `data` holds every byte string end to
end and `lengths` their sizes; case i owns strings 2i (a page or an LZ4 stream) and 2i + 1 (the raw values of the page, or
what liblz4 decoded the stream to -- empty when it rejected it).  Per case: `names`, `kind` ("page" / "lz4"), `width` (the
page's value width), `size` (the size the stream must decode to: LZ4_decompress_safe's capacity), `verdict` (1: liblz4
returned exactly `size`).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bshuf_oracle as bo  # noqa: E402


def _len_bytes(v):
    out = []
    while v >= 255:
        out.append(255)
        v -= 255
    return out + [v]


def seq(lits, off=None, ml=None):
    """one LZ4 sequence: literals, then (unless off is None) a match of ml bytes at offset off"""
    lits = list(lits)
    lcode = min(len(lits), 15)
    mcode = 0 if off is None else min(ml - 4, 15)
    out = [lcode << 4 | mcode] + (_len_bytes(len(lits) - 15) if len(lits) >= 15 else []) + lits
    if off is not None:
        out += [off & 255, off >> 8] + (_len_bytes(ml - 19) if ml >= 19 else [])
    return out


def decoded_size(stream):
    """the size a stream decodes to when every offset is in range (its sequences' literal and match lengths)"""
    ip = op = 0
    s = list(stream)
    while ip < len(s):
        tok = s[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = s[ip]
                ip += 1
                lit += b
                if b != 255:
                    break
        ip += lit
        op += lit
        if ip >= len(s):
            break
        ip += 2
        ml = tok & 15
        if ml == 15:
            while True:
                b = s[ip]
                ip += 1
                ml += b
                if b != 255:
                    break
        op += ml + 4
    return op


def lz4_cases(rng):
    """(name, stream, size).  Sizes are multiples of 8 where the case allows, so that a stream is also one bitshuffle
    block of a 1-byte-wide page."""
    r = lambda k: [int(x) for x in rng.integers(0, 256, k)]     # noqa: E731

    def end(s, skew=0):
        """s + a last literal run of 5..12 bytes that brings the decoded size to skew (mod 8)"""
        return s + seq(r(5 + (skew - decoded_size(s) - 5) % 8))

    c = []
    for off in (1, 2, 3):                                         # overlapping matches: the match reads its own output
        s = end(seq(r(off + 5), off, 40) + seq(r(3), off, 21))
        c.append(("overlap_offset_%d" % off, s, decoded_size(s)))
    for n in (14, 15, 270):                                       # literal runs: 14 in the nibble, 15 / 270 with extension bytes
        s = end(seq(r(n), 4, 20))
        c.append(("literal_run_%d" % n, s, decoded_size(s)))
    for ml in (18, 19, 274):                                      # match lengths: 18 in the nibble, 19 / 274 with extension bytes
        s = end(seq(r(8), 8, ml))
        c.append(("match_length_%d" % ml, s, decoded_size(s)))
    s = end(seq(r(16), 16, 65535) + seq(r(5), 65535, 30))         # a 65551-byte window, then a match 65535 bytes back
    c.append(("offset_65535", s, decoded_size(s)))
    s = end(seq(r(20), 21, 8))                                    # the match starts one byte before the block
    c.append(("offset_before_block_start", s, decoded_size(s)))
    s = end(seq(r(16), 8, 40))
    c.append(("truncated_stream", s[:-3], decoded_size(s)))
    s = end(seq(r(16), 8, 40), skew=7)                            # decodes to one byte less than the block holds
    c.append(("output_one_byte_short", s, decoded_size(s) + 1))
    s = end(seq(r(16), 8, 40), skew=1)                            # decodes to one byte more than the capacity
    c.append(("capacity_one_byte_short", s, decoded_size(s) - 1))
    s = seq(r(16), 8, 44) + seq(r(4))                             # the match ends 4 bytes before the end; a match of more than
    c.append(("match_into_last_5_bytes", s, decoded_size(s)))     # 18 bytes, so not through liblz4's short-sequence shortcut
    s = seq(r(16), 8, 40) + seq(r(4), 8, 4) + seq(r(5))           # a match starting 9 bytes before the end (MFLIMIT is 12)
    c.append(("match_starts_in_last_12_bytes", s, decoded_size(s)))
    return c


def page_cases(rng):
    c = []
    for w in (1, 2, 4, 8, 16):
        blk = 8192 // w
        n = blk + blk // 2 + 3                                    # a full block, a partial last block, n % 8 != 0
        if w <= 8:
            dt = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[w]
            v = (np.sort(rng.integers(-3, 200, n)) * (1 if w == 1 else 37)).astype(dt)
        else:
            v = np.zeros((n, 16), dtype=np.uint8)
            v[:, :3] = rng.integers(0, 256, (n, 3))
            v[::7, 15] = 0x80                                     # some negative LARGEINTs
        c.append(("width_%d" % w, w, np.ascontiguousarray(v).view(np.uint8).reshape(-1)))
    c.append(("width_4_five_values", 4, np.array([-1, 0, 1, 2**31 - 1, -2**31], dtype=np.int32).view(np.uint8)))
    c.append(("width_8_empty", 8, np.zeros(0, dtype=np.uint8)))
    return c


def main():
    L = bo.system_lz4()
    if L is None:
        sys.exit("liblz4.so.1 not found")
    rng = np.random.default_rng(20261015)
    strings, names, kind, width, size, verdict = [], [], [], [], [], []
    for name, w, raw in page_cases(rng):
        page = bo.bitshuffle_encode_with(L, raw.view(np.uint8), w)
        strings += [page, raw]
        names.append(name)
        kind.append("page")
        width.append(w)
        size.append(len(raw))
        verdict.append(1)
    for name, s, sz in lz4_cases(rng):
        s = np.array(s, dtype=np.uint8)
        ok, out = bo.system_lz4_decompress(L, s, sz)
        strings += [s, out if ok else np.zeros(0, dtype=np.uint8)]
        names.append(name)
        kind.append("lz4")
        width.append(0)
        size.append(sz)
        verdict.append(int(ok))
        print("%-30s size %6d  liblz4 %s" % (name, sz, "accepts" if ok else "rejects"))
    path = os.path.join(ROOT, "tests", "golden", "bitshuffle_lz4.npz")
    np.savez_compressed(path, data=np.concatenate(strings), lengths=np.array([len(x) for x in strings], dtype=np.int64),
                        names=np.array(names), kind=np.array(kind), width=np.array(width, dtype=np.int32),
                        size=np.array(size, dtype=np.int64), verdict=np.array(verdict, dtype=np.int32),
                        lz4_version=np.array(L.LZ4_versionString().decode()))
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
