"""Frame-of-reference (FOR) and PLAIN data pages decoded on the device by sr_pages_decode, against a reference written here
in plain Python ints: a frame writer, a page assembler and ForDecoder's reading of a page, pinned on the CPU to the
oracle's codec (oracle.for_encode / oracle.for_decode).

A crafted corpus spans every (value width, storage format, bit width) and, through four byte skews of the page, every start
bit position of for_extract's 96-bit window that a width can meet.  The GPU tests decode it, then page shapes at every
residue of the last frame and every output alignment, the accepted and the refused types, the four memory kinds and the
host's merging of pages into runs, columns long enough that every page decode kernel's grid-stride loop turns at least
twice, malformed pages, the reference's reading of a format-2 frame that another frame follows, misaligned output columns,
and one decoder used across encodings and sizes."""
import functools
import math
import random

import numpy as np
import pytest

from starrocks_b200 import abi

FRAME = 128                                                  # ForEncoder::FRAME_VALUE_NUM
SENTINEL = 0xA5                                              # every byte of an output buffer before a decode
SKEWS = (0, 1, 2, 3)                                         # byte alignments of the crafted pages in device memory
UNSIGNED = {4: np.uint32, 8: np.uint64}
SIGNED = {4: np.int32, 8: np.int64}
TYPES = {4: (abi.TYPE_INT, abi.TYPE_DATE, abi.TYPE_DECIMAL32), 8: (abi.TYPE_BIGINT, abi.TYPE_DATETIME, abi.TYPE_DECIMAL64)}
REFUSED_TYPES = (abi.TYPE_BOOLEAN, abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_LARGEINT, abi.TYPE_DECIMAL128, abi.TYPE_FLOAT,
                 abi.TYPE_DOUBLE)
F2_WIDTHS = {4: (1, 7, 16, 31, 32), 8: (1, 13, 32, 33, 47, 63, 64)}   # format 2 (raw bits) at 8W and narrower
# value counts of the shape pages, in an order that starts later pages at rows = 1, 2 and 3 mod 4; 32767 .. 32769 values
# are 256 and 257 frames, the edge of k_for_frames' 256-frame pass that carries the byte offset over
SHAPE_COUNTS = (1, 32767, 2, 32768, 3, 65536, 5, 32769, 0, 127, 4, 128, 129, 255, 256, 257)
FOR_MSG = "a page is not a well-formed frame-of-reference page"
TABLE_MSG = "a frame-of-reference page has a corrupt frame table"
PLAIN_MSG = "a page is not a well-formed plain page"


# ---- the reference, in plain Python ints ---------------------------------------------------------------------------
class Refused(ValueError):
    """a page the device refuses"""


def pack(deltas, bw):
    """bit_pack: every delta in bw bits, most significant bit first, the bit string zero-padded to whole bytes"""
    if bw == 0:
        return b""
    acc, mask = 0, (1 << bw) - 1
    for d in deltas:
        acc = (acc << bw) | (d & mask)
    nbits = len(deltas) * bw
    return (acc << (-nbits % 8)).to_bytes((nbits + 7) // 8, "big")


def page(W, frames, layout="reader", table=None, frame_size=FRAME, count=None, body=None):
    """a FOR page of W-byte values: the frames, then the (format, bit width) pair of every frame, then the frame-size byte,
    then the uint32 value count.  A frame is (format, bit width, min, deltas): the min in W little-endian bytes, then the
    packed deltas.  layout "reader": a frame that another frame follows takes bw * 128 / 8 + W bytes, where
    ForDecoder::init looks for the next one; "encoder": the bytes ForEncoder writes, a format-2 frame taking count * bw
    BYTES (see test_oracle_golden).  table, frame_size and count override what the frames imply; body maps a frame index to
    the bytes that replace that frame's."""
    parts = []
    for k, (fmt, bw, mn, deltas) in enumerate(frames):
        b = (mn % (1 << 8 * W)).to_bytes(W, "little") + pack(deltas, bw)
        if layout == "encoder" and fmt == 2:
            b += bytes(W + len(deltas) * bw - len(b))
        elif k + 1 < len(frames):
            b += bytes(W + bw * FRAME // 8 - len(b))
        parts.append(body[k] if body and k in body else b)
    if table is None:
        table = bytes(x for fmt, bw, _, _ in frames for x in (fmt, bw))
    n = sum(len(f[3]) for f in frames) if count is None else count
    return np.frombuffer(b"".join(parts) + table + bytes([frame_size]) + n.to_bytes(4, "little"), dtype=np.uint8).copy()


def walk(pg, W):
    """the frames ForDecoder::init finds in a page: (byte offset, format, bit width, value count) of each; Refused for a page
    the device refuses by its footer or frame table (short, frame size not 128 with values, a table that does not fit, a
    format above 2, a width above 8 * W, frame bits that run into the table)"""
    b = bytes(pg)
    if len(b) < 5:
        raise Refused("shorter than the footer")
    n = int.from_bytes(b[-4:], "little")
    if n == 0:
        return []
    if b[-5] != FRAME:
        raise Refused("frame size")
    nf = (n + FRAME - 1) // FRAME
    meta = len(b) - 5 - 2 * nf
    if meta < 0:
        raise Refused("frame table longer than the page")
    out, off = [], 0
    for f in range(nf):
        fmt, bw, cnt = b[meta + 2 * f], b[meta + 2 * f + 1], min(FRAME, n - f * FRAME)
        if fmt > 2 or bw > 8 * W or off + W + (cnt * bw + 7) // 8 > meta:
            raise Refused("frame %d" % f)
        out.append((off, fmt, bw, cnt))
        off += bw * FRAME // 8 + W                           # also after a format-2 frame
    return out


def read(pg, W):
    """ForDecoder's values of a page as unsigned W-byte ints: format 0 min + delta, format 1 min + the deltas up to the
    value, format 2 the raw bits -- all modulo 2^(8W)"""
    b, M, out = bytes(pg), 1 << 8 * W, []
    for off, fmt, bw, cnt in walk(pg, W):
        mn = int.from_bytes(b[off:off + W], "little")
        nbytes = (cnt * bw + 7) // 8
        bits = int.from_bytes(b[off + W:off + W + nbytes], "big") >> (8 * nbytes - cnt * bw)
        deltas = [(bits >> (cnt - 1 - i) * bw) & ((1 << bw) - 1) for i in range(cnt)]
        if fmt == 2:
            out += deltas
        elif fmt == 1:
            for d in deltas:
                mn = (mn + d) % M
                out.append(mn)
        else:
            out += [(mn + d) % M for d in deltas]
    return out


def encoder_frames(values, W):
    """ForEncoder's frames of a column (bit_packing_one_frame_value): (format, bit width, min, deltas) of every 128 values"""
    B = 8 * W
    M, half_max = 1 << B, (1 << (B - 2)) - 1
    wrap = lambda x: (x + M // 2) % M - M // 2                # to T
    bits = lambda x: (x % (1 << 64)).bit_length()             # of the value sign-extended to 64 bits
    frames = []
    for lo in range(0, len(values), FRAME):
        v = [int(x) for x in values[lo:lo + FRAME]]
        asc, keep, bw = True, False, 0
        for a, b in zip(v, v[1:]):
            if asc:
                if b < a:
                    asc = False
                elif wrap((b >> 1) - (a >> 1)) > half_max:
                    keep = True
                else:
                    bw = max(bw, bits(wrap(b - a)))
        mn, mx = min(v), max(v)
        if not asc and wrap((mx >> 1) - (mn >> 1)) > half_max:
            keep = True
        if keep:
            frames.append((2, B, mn, v))
        elif asc:
            frames.append((1, bw, mn, [0] + [wrap(b - a) for a, b in zip(v, v[1:])]))
        else:
            frames.append((0, bits(wrap(mx - mn)), mn, [x - mn for x in v]))
    return frames


def as_bytes(values, W):
    return np.array(values, dtype=UNSIGNED[W]).view(np.uint8)


def plain_page(values, W):
    return np.concatenate([np.array([len(values)], dtype="<u4").view(np.uint8), as_bytes(values, W)])


# ---- the crafted corpus --------------------------------------------------------------------------------------------
def _deltas(bw, rng):
    """128 deltas of bw bits: all ones, alternating bits both ways, a single bit at every position, then random ones"""
    if bw == 0:
        return [0] * FRAME
    ones = (1 << bw) - 1
    alt = int("10" * 32, 2) & ones
    return ([ones, alt, ones ^ alt] + [1 << j for j in range(bw)] + [rng.getrandbits(bw) for _ in range(FRAME)])[:FRAME]


@functools.lru_cache(maxsize=None)
def corpus_frames(W):
    """formats 0 and 1 at every width 0 .. 8W, format 2 at F2_WIDTHS; mins at the type's minimum and maximum, -1 and 0"""
    B, rng = 8 * W, random.Random(W)
    mins = (-(1 << (B - 1)), (1 << (B - 1)) - 1, -1, 0)
    frames = [(fmt, bw, mins[(bw + fmt) % 4], _deltas(bw, rng)) for fmt in (0, 1) for bw in range(B + 1)]
    return frames + [(2, bw, mins[k % 4], _deltas(bw, rng)) for k, bw in enumerate(F2_WIDTHS[W])]


def _cut(frames, cnt):
    """the frames with the last one cut to cnt values"""
    fmt, bw, mn, d = frames[-1]
    return frames[:-1] + [(fmt, bw, mn, d[:cnt])]


@functools.lru_cache(maxsize=None)
def corpus_pages(W):
    """one page per format and one of every frame in a shuffled order, each with a short last frame"""
    fr = corpus_frames(W)
    mixed = list(fr)
    random.Random(7 * W).shuffle(mixed)
    groups = [[f for f in fr if f[0] == fmt] for fmt in (0, 1, 2)] + [mixed]
    return [page(W, _cut(g, cnt)) for g, cnt in zip(groups, (77, 3, 1, 50))]


def coverage(W, pages):
    """what for_extract meets when the pages lie at every byte skew of SKEWS: the (format, bit width) pairs, the start bit
    positions inside the 96-bit window per width, and the widths with a value whose window start + width passes 64 bits
    (its last bits come from the third word).  Positions follow k_for_decode: bit b = 8 * (skew + frame offset + W) + i * bw."""
    fmts, pos, third = set(), {}, set()
    for pg in pages:
        for off, fmt, bw, cnt in walk(pg, W):
            fmts.add((fmt, bw))
            for skew in SKEWS if bw else ():
                for i in range(cnt):
                    b = 8 * (skew + off + W) + i * bw
                    p = 8 * ((b >> 3) & 3) + (b & 7)
                    pos.setdefault(bw, set()).add(p)
                    if p + bw > 64:
                        third.add(bw)
    return fmts, pos, third


@functools.lru_cache(maxsize=None)
def shape_pages(W):
    """one FOR page per count of SHAPE_COUNTS, its frames cycling through the formats and widths, random mins and deltas;
    -> (pages, the values of every page)"""
    B, rng = 8 * W, random.Random(100 + W)
    pages, values = [], []
    for p, c in enumerate(SHAPE_COUNTS):
        frames = []
        for k in range((c + FRAME - 1) // FRAME):
            bw = (5 * k + 3 * p) % (B + 1)
            frames.append(((k + p) % 3, bw, rng.getrandbits(B), [rng.getrandbits(bw) for _ in range(min(FRAME, c - k * FRAME))]))
        pg = page(W, frames)
        pages.append(pg)
        values.append(read(pg, W))
    return pages, values


def _natural(W):
    """columns as a writer sees them; format 2 only in single-frame columns (test_oracle_golden: the reference cannot read
    its own page back when another frame follows a format-2 frame)"""
    rng = np.random.default_rng(31 + W)
    info = np.iinfo(SIGNED[W])
    yield "empty", np.zeros(0, dtype=SIGNED[W])
    yield "one", np.array([2019], dtype=SIGNED[W])
    yield "two_and_a_half_frames", np.arange(320, dtype=SIGNED[W])
    yield "constant", np.full(300, -7, dtype=SIGNED[W])
    yield "small_range", rng.integers(1000, 1000 + (1 << 22), 5000).astype(SIGNED[W])
    yield "negative", rng.integers(-500, 500, 777).astype(SIGNED[W])
    yield "ascending_big_steps", np.cumsum(rng.integers(0, 1 << 20, 1000)).astype(SIGNED[W])
    yield "ascending_then_not", np.concatenate([np.arange(128), rng.integers(0, 50, 128), np.arange(40)]).astype(SIGNED[W])
    yield "half_range", rng.integers(info.min // 2 + 1, info.max // 2, 999, dtype=SIGNED[W])
    yield "extremes_single_frame", np.array([info.min, info.max, 0, -1, 1, info.min, info.max] * 18, dtype=SIGNED[W])[:128]
    yield "ascending_overflow_single_frame", np.array([info.min, info.max] + [info.max] * 126, dtype=SIGNED[W])
    yield "full_range_single_frame", rng.integers(info.min, info.max, 100, dtype=SIGNED[W])


# ---- CPU: the reference against the oracle, and the corpus' coverage -----------------------------------------------
@pytest.mark.parametrize("W", [4, 8])
def test_reader_matches_the_oracle_on_every_page(oracle, W):
    pages = list(corpus_pages(W)) + list(shape_pages(W)[0])
    pages += [oracle.for_encode(v) for _, v in _natural(W)]
    for k, pg in enumerate(pages):
        assert as_bytes(read(pg, W), W).tobytes() == oracle.for_decode(pg, SIGNED[W]).tobytes(), k


@pytest.mark.parametrize("W", [4, 8])
def test_writer_reproduces_the_encoder(oracle, W):
    for name, v in _natural(W):
        frames = encoder_frames(v, W)
        mine = page(W, frames, layout="encoder")
        assert mine.tobytes() == oracle.for_encode(v).tobytes(), name
        assert (np.array(read(mine, W), dtype=UNSIGNED[W]).view(SIGNED[W]) == v).all(), name
        if name.endswith("single_frame"):
            assert [f[0] for f in frames] == [2], name
    # test_oracle_golden's known answer: ascending, deltas 0, 1, 2, 4 in 3 bits
    assert page(W, [(1, 3, 101, [0, 1, 2, 4])]).tobytes() == \
        (101).to_bytes(W, "little") + bytes([0b00000101, 0b01000000, 1, 3, 128]) + (4).to_bytes(4, "little")
    assert page(W, []).tobytes() == bytes([128, 0, 0, 0, 0])


@pytest.mark.parametrize("W", [4, 8])
def test_corpus_covers_the_format_space(W):
    B = 8 * W
    fmts, pos, third = coverage(W, corpus_pages(W))
    assert fmts >= {(fmt, bw) for fmt in (0, 1) for bw in range(B + 1)} | {(2, B)}
    assert {bw for fmt, bw in fmts if fmt == 2} >= {1, B // 2, B - 1, B}
    for bw in range(1, B + 1):
        # pos = 8 * skew + i * bw (mod 32): a width meets the multiples of gcd(bw, 8), all 32 positions when it is odd
        assert pos[bw] == set(range(0, 32, math.gcd(bw, 8))), bw
    assert third == {bw for bw in range(1, B + 1) if 32 - math.gcd(bw, 8) + bw > 64}
    assert (W == 4) == (not third)                                        # 96 bits are needed from width 35 on
    M = 1 << B
    wraps = [f for f in corpus_frames(W) if f[0] == 1 and any(s >= M for s in np.cumsum([f[2] % M] + f[3], dtype=object))]
    assert len(wraps) >= 8 and {1, B} <= {f[1] for f in wraps}            # format-1 frames whose running sum wraps
    mins = {f[2] for f in corpus_frames(W)}
    assert mins == {-(1 << (B - 1)), (1 << (B - 1)) - 1, -1, 0}
    assert {f[2] for f in corpus_frames(W) if f[0] == 2} - {0}            # format 2 ignores a nonzero min


def test_shape_pages_start_at_every_row_alignment():
    starts = np.cumsum((0,) + SHAPE_COUNTS)[:-1]
    assert {s % 4 for s, c in zip(starts, SHAPE_COUNTS) if c} == {0, 1, 2, 3}
    assert {c % 4 for c in SHAPE_COUNTS} == {0, 1, 2, 3} and {c % FRAME % 4 for c in SHAPE_COUNTS if c % FRAME} == {0, 1, 2, 3}
    assert {(c + FRAME - 1) // FRAME for c in SHAPE_COUNTS} >= {256, 257, 512}


@pytest.mark.parametrize("W", [4, 8])
def test_reader_refuses_what_the_device_refuses(oracle, W):
    # the reader keeps the device's rule; oracle.for_decode (ForDecoder) is laxer and reads some of these pages
    for name, pg, msg in _malformed_for(W):
        with pytest.raises(Refused):
            read(pg, W)
    lax = {n for n, pg, _ in _malformed_for(W) if _oracle_reads(oracle, pg, W)}
    assert lax == {"frame_size_127", "format_3", "width_8W_plus_1", "bits_overlap_table"}
    for name, pg, want in _accepted_edges(W):
        assert read(pg, W) == want, name
    assert read(page(W, FULL_THEN_SHORT), W)[FRAME:] == [(-9 + 7) % (1 << 8 * W), (-9 + 8) % (1 << 8 * W), 126]


def _oracle_reads(oracle, pg, W):
    try:
        oracle.for_decode(pg, SIGNED[W])
        return True
    except oracle.OracleError:
        return False


FULL_THEN_SHORT = [(0, 9, 1, list(range(FRAME))), (1, 7, -9, [7, 1, 127])]   # the short frame's 21 bits end mid-byte


def _malformed_for(W):
    """(name, page, message) of FOR pages the device refuses"""
    B = 8 * W
    one = [(0, 3, 5, [1, 2, 3, 4, 5])]
    last = FULL_THEN_SHORT[1]
    return [
        ("empty_page", np.zeros(0, dtype=np.uint8), FOR_MSG),
        ("short", np.zeros(4, dtype=np.uint8), FOR_MSG),
        ("frame_size_127", page(W, one, frame_size=127), FOR_MSG),
        ("frame_size_0", page(W, one, frame_size=0), FOR_MSG),
        ("table_longer_than_page", page(W, one, count=10 * FRAME), FOR_MSG),
        ("format_3", page(W, FULL_THEN_SHORT[:1] + [(3,) + last[1:]]), TABLE_MSG),
        ("width_8W_plus_1", page(W, FULL_THEN_SHORT[:1] + [(0, B + 1) + last[2:]]), TABLE_MSG),
        # the last frame's packed bits one byte short: they reach one byte into the frame table
        ("bits_overlap_table", page(W, FULL_THEN_SHORT, body={1: page(W, [last])[:W + 2].tobytes()}), TABLE_MSG),
    ]


def _accepted_edges(W):
    """(name, page, values) of FOR pages at the edge of the device's rule that it accepts"""
    return [("no_values_frame_size_%d" % fs, page(W, [], frame_size=fs), []) for fs in (0, 1, 127, 255)] + \
           [("frame_ends_at_the_table", page(W, FULL_THEN_SHORT), read(page(W, FULL_THEN_SHORT), W))]


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _column(n, W, shift=0, extra=8):
    """a device buffer of shift + n + extra values of W bytes, every byte SENTINEL, from a 256-byte-aligned allocation;
    -> (buffer, pointer to value `shift`)"""
    import torch
    t = torch.full(((shift + n + extra) * W,), SENTINEL, dtype=torch.uint8, device="cuda")
    assert t.data_ptr() % 256 == 0
    return t, t.data_ptr() + shift * W


def _check(ctx, t, W, shift, want, what=None):
    """the buffer holds the bytes `want` from value `shift` on, and SENTINEL everywhere else"""
    ctx.sync()
    got = t.cpu().numpy()
    lo, hi = shift * W, shift * W + len(want)
    assert (got[:lo] == SENTINEL).all(), what
    assert np.array_equal(got[lo:hi], want), what
    assert (got[hi:] == SENTINEL).all(), what                     # nothing written past the column


def _decode(dec, enc, typ, pages, ptr, cap, mem="host", skew=None):
    """decode `pages` into ptr from `mem`: host (pageable: staged); device, every page at byte `skew` of its own
    allocation (page k at k % 4 + 1 when skew is None); pinned_run: back to back in one page-locked buffer (runs of >= 256
    KiB are staged by DMA); pinned_scattered: 100 + k % 3 byte gaps (read in place over PCIe).  -> rows"""
    import torch
    keep = []
    if mem == "host":
        rows = dec.decode(enc, typ, pages, ptr, cap)
    elif mem == "device":
        views = []
        for k, pg in enumerate(pages):
            s = k % 4 + 1 if skew is None else skew
            b = torch.from_numpy(np.concatenate([np.zeros(s, dtype=np.uint8), pg])).cuda()
            keep.append(b)
            views.append((b.data_ptr() + s, len(pg)))
        rows = dec.decode(enc, typ, views, ptr, cap, mem=abi.MEM_DEVICE)
    else:
        offs, at = [], 0
        for k, pg in enumerate(pages):
            at += 0 if mem == "pinned_run" else 100 + k % 3
            offs.append(at)
            at += len(pg)
        blob = torch.zeros(max(at, 1), dtype=torch.uint8).pin_memory()
        for o, pg in zip(offs, pages):
            blob.numpy()[o:o + len(pg)] = pg
        keep.append(blob)
        rows = dec.decode(enc, typ, [(blob.data_ptr() + o, len(pg)) for o, pg in zip(offs, pages)], ptr, cap, mem=abi.MEM_HOST_PINNED)
    dec.ctx.sync()                                                  # the pages are read asynchronously
    return rows


def _refused(gpu, ctx, call, code, msg):
    """call() fails with `code` and `msg` before any kernel launch or device allocation"""
    launches, nbytes = ctx.launches, ctx.device_bytes
    with pytest.raises(gpu.GpuError) as ei:
        call()
    assert ei.value.code == code and msg in str(ei.value), str(ei.value)
    assert (ctx.launches, ctx.device_bytes) == (launches, nbytes), msg


def _shape_job(W, enc):
    """(pages, expected bytes, rows) of the shape pages as FOR or PLAIN pages"""
    fpages, values = shape_pages(W)
    pages = list(fpages) if enc == abi.PAGE_FOR else [plain_page(v, W) for v in values]
    want = as_bytes([x for v in values for x in v], W)
    return pages, want, len(want) // W


ENCS = [abi.PAGE_FOR, abi.PAGE_PLAIN]
ENC_IDS = ["for", "plain"]


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_crafted_corpus_at_every_skew_and_type(gpu, ctx, W):
    pages = corpus_pages(W)
    want = as_bytes([x for pg in pages for x in read(pg, W)], W)
    n = len(want) // W
    dec = gpu.PageDecoder(ctx)
    try:
        for typ in TYPES[W]:                                        # the 4- or 8-byte types decode to the same bytes
            for skew in SKEWS:
                t, ptr = _column(n, W)
                assert _decode(dec, abi.PAGE_FOR, typ, pages, ptr, n, "device", skew) == n
                _check(ctx, t, W, 0, want, (typ, skew))
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
@pytest.mark.parametrize("enc", ENCS, ids=ENC_IDS)
def test_page_shapes_in_one_call(gpu, ctx, W, enc):
    # every residue of the last frame, later pages at rows = 1, 2, 3 mod 4, the output at 0 .. 3 values from a 256-byte
    # boundary; the exact capacity is accepted, one value less is refused
    pages, want, n = _shape_job(W, enc)
    dec = gpu.PageDecoder(ctx)
    try:
        for shift in range(4):
            typ = TYPES[W][shift % 3]
            t, ptr = _column(n, W, shift)
            with pytest.raises(gpu.GpuError) as ei:
                dec.decode(enc, typ, pages, ptr, n - 1)
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT and "room for %d" % (n - 1) in str(ei.value)
            assert dec.decode(enc, typ, pages, ptr, n) == n
            _check(ctx, t, W, shift, want, shift)
    finally:
        dec.close()


@pytest.mark.gpu
def test_refused_types_and_encodings_launch_nothing(gpu, ctx):
    pages, want, n = _shape_job(4, abi.PAGE_FOR)
    t, ptr = _column(n, 8)
    dec = gpu.PageDecoder(ctx)
    try:
        for first in (True, False):                                  # a fresh decoder, then one with scratch
            for enc in ENCS:
                for typ in REFUSED_TYPES:
                    _refused(gpu, ctx, lambda: dec.decode(enc, typ, pages, ptr, n), abi.SR_ERR_NOT_SUPPORTED, "page decode of type %d" % typ)
            for enc in (4, -1):
                for typ in TYPES[4] + TYPES[8]:
                    _refused(gpu, ctx, lambda: dec.decode(enc, typ, pages, ptr, n), abi.SR_ERR_NOT_SUPPORTED, "page encoding %d" % enc)
            _check(ctx, t, 8, 0, np.zeros(0, dtype=np.uint8))
            if first:
                assert dec.decode(abi.PAGE_FOR, abi.TYPE_INT, pages, ptr, n) == n
                _check(ctx, t, 4, 0, want)
                t, ptr = _column(n, 8)
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
@pytest.mark.parametrize("enc", ENCS, ids=ENC_IDS)
@pytest.mark.parametrize("mem", ["host", "device", "pinned_run", "pinned_scattered"])
def test_memory_kinds(gpu, ctx, W, enc, mem):
    pages, want, n = _shape_job(W, enc)
    total = sum(len(p) for p in pages)
    if mem == "pinned_run":
        assert total >= 256 << 10                                   # one run, staged
    if mem == "pinned_scattered":
        assert total / len(pages) < 256 << 10                       # one run per page, read in place
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(n, W)
        assert _decode(dec, enc, TYPES[W][0], pages, ptr, n, mem) == n
        _check(ctx, t, W, 0, want)
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("enc", ENCS, ids=ENC_IDS)
@pytest.mark.parametrize("mem", [abi.MEM_HOST, abi.MEM_HOST_PINNED], ids=["host", "pinned"])
def test_host_run_merging(gpu, ctx, enc, mem):
    # host pages less than 64 bytes after the previous one are copied with it as one run.  Laid out as
    # a |1| b |63| c |64| d |5| g | f | e  (gap bytes 0xEE) and listed a b c d e f g a: b and c join a's run, d starts a
    # new one, e f g are listed in reverse address order, and a is listed twice
    import torch
    W = 8
    fpages, values = shape_pages(W)
    pages = list(fpages) if enc == abi.PAGE_FOR else [plain_page(v, W) for v in values]
    a, b, c, d, e, f, g = 9, 2, 12, 1, 13, 10, 15
    layout = [(a, 0), (b, 1), (c, 63), (d, 64), (g, 5), (f, 0), (e, 0)]
    offs, at = {}, 0
    for k, gap in layout:
        offs[k] = at + gap
        at += gap + len(pages[k])
    blob = torch.full((at,), 0xEE, dtype=torch.uint8)
    blob = blob.pin_memory() if mem == abi.MEM_HOST_PINNED else blob
    for k, _ in layout:
        blob.numpy()[offs[k]:offs[k] + len(pages[k])] = pages[k]
    listed = [a, b, c, d, e, f, g, a]
    want = as_bytes([x for k in listed for x in values[k]], W)
    n = len(want) // W
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(n, W)
        assert dec.decode(enc, abi.TYPE_BIGINT, [(blob.data_ptr() + offs[k], len(pages[k])) for k in listed], ptr, n, mem=mem) == n
        _check(ctx, t, W, 0, want)
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_for_column_sweeps_the_grid(gpu, ctx, oracle, W):
    sweep = 64 * _sms()                          # k_for_decode: at most 8 * SMs CTAs of 8 warps, one frame per warp at a time
    n = int(2.6 * sweep) * FRAME - 77
    rng = np.random.default_rng(41 + W)
    v = np.empty(n, dtype=SIGNED[W])
    rows = 65536
    for k, lo in enumerate(range(0, n, rows)):
        bits = 1 + 7 * k % (8 * W - 2)
        x = rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), min(rows, n - lo), dtype=np.int64)
        v[lo:lo + rows] = np.sort(x) if k % 3 == 1 else x           # format-1 pages among format-0 ones
    pages = [oracle.for_encode(v[lo:lo + rows]) for lo in range(0, n, rows)]
    assert sum((min(rows, n - lo) + FRAME - 1) // FRAME for lo in range(0, n, rows)) > 2.5 * sweep
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(n, W)
        assert dec.decode(abi.PAGE_FOR, TYPES[W][0], pages, ptr, n) == n
        _check(ctx, t, W, 0, v.view(np.uint8))
    finally:
        dec.close()


def _bshuf_blocks(rows, w):
    blk = 8192 // w
    return ((rows + 7) // 8 * 8 + blk - 1) // blk


@pytest.mark.gpu
@pytest.mark.parametrize("w", [1, 4, 8, 16])
def test_bitshuffle_column_sweeps_the_grid(gpu, ctx, bo, w):
    sweep = 16 * _sms()                          # k_bshuf_decode: at most 8 * SMs CTAs of 2 warps, one 8 KB block per warp
    n = int(2.6 * sweep) * (8192 // w) - 3
    rng = np.random.default_rng(51 + w)
    raw = rng.integers(0, 16, n * w, dtype=np.uint8) & (rng.integers(0, 2, n * w, dtype=np.uint8) * np.uint8(0xFF))
    rows = 64 * 8192 // w
    pages = [bo.bitshuffle_encode(raw[lo * w:(lo + rows) * w], w) for lo in range(0, n, rows)]
    assert sum(_bshuf_blocks(min(rows, n - lo), w) for lo in range(0, n, rows)) > 2.5 * sweep
    typ = {1: abi.TYPE_TINYINT, 4: abi.TYPE_INT, 8: abi.TYPE_BIGINT, 16: abi.TYPE_LARGEINT}[w]
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(n, w)
        assert dec.decode(abi.PAGE_BITSHUFFLE, typ, pages, ptr, n) == n
        _check(ctx, t, w, 0, raw)
    finally:
        dec.close()


@pytest.mark.gpu
def test_dict_column_sweeps_the_grid(gpu, ctx, bo):
    sweep = 16 * _sms()
    n = int(2.6 * sweep) * 2048 - 5
    rng = np.random.default_rng(61)
    words = rng.integers(-2**31, 2**31, 1000, dtype=np.int64).astype(np.int32)
    codes = rng.integers(0, len(words), n).astype(np.int32)
    rows = 64 * 2048
    pages = [bo.dict_page_encode(codes[lo:lo + rows]) for lo in range(0, n, rows)]
    assert sum(_bshuf_blocks(min(rows, n - lo), 4) for lo in range(0, n, rows)) > 2.5 * sweep
    dec = gpu.PageDecoder(ctx)
    try:
        dec.set_dict(words)
        t, ptr = _column(n, 4)
        assert dec.decode(abi.PAGE_DICT, abi.TYPE_INT, pages, ptr, n) == n
        _check(ctx, t, 4, 0, words[codes].view(np.uint8))
    finally:
        dec.close()


@pytest.mark.gpu
def test_plain_call_over_65535_pages(gpu, ctx):
    # k_plain_copy takes one page per gridDim.y: more than 65535 pages take a second launch
    rng = np.random.default_rng(71)
    counts = rng.integers(1, 4, 70_000)
    v = rng.integers(-2**31, 2**31, int(counts.sum()), dtype=np.int64).astype(np.int32)
    ends = np.cumsum(counts)
    blob = np.concatenate([x for lo, hi in zip(ends - counts, ends) for x in (np.array([hi - lo], dtype="<u4").view(np.uint8), v[lo:hi].view(np.uint8))])
    offs = 4 * (ends - counts) + 4 * np.arange(len(counts))
    views = [(blob.ctypes.data + int(o), 4 + 4 * int(c)) for o, c in zip(offs, counts)]
    assert len(views) > 65535
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(len(v), 4)
        assert dec.decode(abi.PAGE_PLAIN, abi.TYPE_INT, views, ptr, len(v)) == len(v)
        _check(ctx, t, 4, 0, v.view(np.uint8))
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_malformed_pages_then_a_good_call(gpu, ctx, oracle, W):
    # oracle.for_decode reads some of these pages (test_reader_refuses_what_the_device_refuses): the device is stricter
    typ = TYPES[W][0]
    fpages, values = shape_pages(W)
    pick = (9, 12, 13)                                                  # 127, 129 and 255 values
    good = {abi.PAGE_FOR: [fpages[k] for k in pick], abi.PAGE_PLAIN: [plain_page(values[k], W) for k in pick]}
    want = as_bytes([x for k in pick for x in values[k]], W)
    n = len(want) // W
    p = plain_page(values[6], W)
    bad = {abi.PAGE_FOR: _malformed_for(W),
           abi.PAGE_PLAIN: [("short", p[:3], PLAIN_MSG), ("one_byte_more", np.concatenate([p, p[-1:]]), PLAIN_MSG),
                            ("one_byte_less", p[:-1], PLAIN_MSG)]}
    dec = gpu.PageDecoder(ctx)
    try:
        for enc in ENCS:
            for name, pg, msg in bad[enc]:
                t, ptr = _column(n + 2 * FRAME, W)
                with pytest.raises(gpu.GpuError) as ei:                 # behind good pages
                    dec.decode(enc, typ, good[enc] + [pg], ptr, n + 2 * FRAME)
                assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT and msg in str(ei.value), (name, str(ei.value))
                t, ptr = _column(n, W)
                assert dec.decode(enc, typ, good[enc], ptr, n) == n, name
                _check(ctx, t, W, 0, want, name)
        for name, pg, vals in _accepted_edges(W):
            e = as_bytes(vals, W)
            t, ptr = _column(n + len(vals), W)
            assert dec.decode(abi.PAGE_FOR, typ, good[abi.PAGE_FOR] + [pg], ptr, n + len(vals)) == n + len(vals), name
            _check(ctx, t, W, 0, np.concatenate([want, e]), name)
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W", [4, 8])
def test_format2_frame_followed_by_another_reads_as_the_reference(gpu, ctx, oracle, W):
    # ForEncoder writes count * bw BYTES for a format-2 frame, while ForDecoder::init looks for the next frame bw * 128 / 8
    # + W bytes on, inside that frame's padding.  The device reads what ForDecoder reads -- which is not the column written.
    info = np.iinfo(SIGNED[W])
    rng = np.random.default_rng(81 + W)
    extremes = np.array([info.min, info.max, 0, -1, 1, info.min, info.max] * 19, dtype=SIGNED[W])[:FRAME]
    small = rng.integers(-1000, 1000, 300).astype(SIGNED[W])
    cols = [np.concatenate([extremes, small]), np.concatenate([small[:FRAME], extremes, small[:40]])]
    pages = [oracle.for_encode(v) for v in cols]
    assert [[f[0] for f in encoder_frames(v, W)] for v in cols] == [[2, 0, 0, 0], [0, 2, 0]]
    reads = [oracle.for_decode(pg, SIGNED[W]) for pg in pages]
    for pg, v, r in zip(pages, cols, reads):
        assert as_bytes(read(pg, W), W).tobytes() == r.tobytes()
        assert (r[:len(v)] != v).any()                              # not the source values
    want = np.concatenate(reads).view(np.uint8)
    n = len(want) // W
    dec = gpu.PageDecoder(ctx)
    try:
        t, ptr = _column(n, W)
        assert dec.decode(abi.PAGE_FOR, TYPES[W][0], pages, ptr, n) == n
        _check(ctx, t, W, 0, want)
    finally:
        dec.close()


@pytest.mark.gpu
def test_misaligned_output_is_refused_without_a_launch(gpu, ctx, oracle, bo):
    rng = np.random.default_rng(91)
    dec = gpu.PageDecoder(ctx)
    try:
        for typ, W, shifts in ((abi.TYPE_INT, 4, (1, 2, 3)), (abi.TYPE_BIGINT, 8, (4,))):
            v = rng.integers(-10**6, 10**6, 1001).astype(SIGNED[W])
            for enc, pages in ((abi.PAGE_FOR, [oracle.for_encode(v)]), (abi.PAGE_PLAIN, [oracle.plain_encode(v)]),
                               (abi.PAGE_BITSHUFFLE, [bo.bitshuffle_encode(v)])):
                t, ptr = _column(len(v), W, 1)
                for s in shifts:
                    _refused(gpu, ctx, lambda: dec.decode(enc, typ, pages, ptr - W + s, len(v)), abi.SR_ERR_INVALID_ARGUMENT,
                             "output column not aligned to %d bytes" % W)
                _check(ctx, t, W, 1, np.zeros(0, dtype=np.uint8))
                assert dec.decode(enc, typ, pages, ptr, len(v)) == len(v)
                _check(ctx, t, W, 1, v.view(np.uint8), enc)
        raw16 = np.arange(16 * 16, dtype=np.uint8)                  # 16-byte values: 8-byte alignment
        page16 = bo.bitshuffle_encode(raw16, 16)
        t, ptr = _column(2 * 16, 8, 2)                              # (in 8-byte slots)
        _refused(gpu, ctx, lambda: dec.decode(abi.PAGE_BITSHUFFLE, abi.TYPE_LARGEINT, [page16], ptr - 4, 16), abi.SR_ERR_INVALID_ARGUMENT,
                 "output column not aligned to 8 bytes")
        assert dec.decode(abi.PAGE_BITSHUFFLE, abi.TYPE_LARGEINT, [page16], ptr, 16) == 16
        _check(ctx, t, 8, 2, raw16)
        codes = np.arange(100, dtype=np.int32) % 7                   # dictionary pages: 4-byte ids
        dec.set_dict(np.arange(7, dtype=np.int32) * 3)
        t, ptr = _column(len(codes), 4, 1)
        _refused(gpu, ctx, lambda: dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [bo.dict_page_encode(codes)], ptr - 2, len(codes)),
                 abi.SR_ERR_INVALID_ARGUMENT, "output column not aligned to 4 bytes")
        _check(ctx, t, 4, 1, np.zeros(0, dtype=np.uint8))
    finally:
        dec.close()


def _jobs(oracle, bo, rng, words):
    """(encoding, type, value width, pages, expected bytes) of columns of every encoding, sizes growing and shrinking"""
    def ints(n, W, bits):
        return rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), n, dtype=np.int64).astype(SIGNED[W])

    def split(v, rows):
        return [v[lo:lo + rows] for lo in range(0, max(len(v), 1), rows)]

    for enc, W, n, rows in ((abi.PAGE_FOR, 4, 200_000, 1000), (abi.PAGE_PLAIN, 8, 3000, 1000), (abi.PAGE_BITSHUFFLE, 4, 300_000, 8192),
                            (abi.PAGE_DICT, 4, 50_000, 4096), (abi.PAGE_FOR, 8, 1, 1), (abi.PAGE_FOR, 4, 600_001, 5000),
                            (abi.PAGE_BITSHUFFLE, 8, 999, 100), (abi.PAGE_PLAIN, 4, 20_000, 7), (abi.PAGE_DICT, 4, 700_000, 65_536),
                            (abi.PAGE_FOR, 8, 70_000, 65_536), (abi.PAGE_FOR, 4, 130, 129)):
        if enc == abi.PAGE_DICT:
            codes = rng.integers(0, len(words), n).astype(np.int32)
            yield enc, abi.TYPE_INT, 4, [bo.dict_page_encode(c) for c in split(codes, rows)], words[codes].view(np.uint8)
            continue
        v = ints(n, W, 1 + n % (8 * W - 1))
        encode = {abi.PAGE_FOR: oracle.for_encode, abi.PAGE_PLAIN: oracle.plain_encode, abi.PAGE_BITSHUFFLE: bo.bitshuffle_encode}[enc]
        yield enc, TYPES[W][n % 3], W, [encode(x) for x in split(v, rows)], v.view(np.uint8)


@pytest.mark.gpu
def test_one_decoder_across_encodings_and_sizes(gpu, ctx, oracle, bo):
    # the decoder's scratch (page tables, frame / block descriptors, staging) grows and shrinks between calls of every
    # encoding; then two decoders on one context take turns
    rng = np.random.default_rng(101)
    words = rng.integers(-2**31, 2**31, 500, dtype=np.int64).astype(np.int32)
    jobs = list(_jobs(oracle, bo, rng, words))
    decs = [gpu.PageDecoder(ctx), gpu.PageDecoder(ctx)]
    try:
        for d in decs:
            d.set_dict(words)
        order = jobs + jobs[::-1]
        for turn in ([decs[0]] * len(order), [decs[k % 2] for k in range(len(order))]):
            for dec, (enc, typ, W, pages, want) in zip(turn, order):
                n = len(want) // W
                t, ptr = _column(n, W)
                assert dec.decode(enc, typ, pages, ptr, n) == n
                _check(ctx, t, W, 0, want, (enc, n))
    finally:
        for d in decs:
            d.close()
