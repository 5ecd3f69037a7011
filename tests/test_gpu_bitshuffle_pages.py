"""BIT_SHUFFLE (bitshuffle + LZ4) data pages decoded on the device by sr_pages_decode, bit-exact against the CPU codec
(bshuf_oracle) and against pages whose LZ4 blocks came from liblz4 (tests/golden/bitshuffle_lz4.npz)."""
import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from tests.test_bitshuffle_oracle import golden

pytestmark = pytest.mark.gpu

# (numpy dtype or None for 16-byte values carried as bytes, sr_type)
TYPES = [(np.uint8, abi.TYPE_BOOLEAN), (np.int8, abi.TYPE_TINYINT), (np.int16, abi.TYPE_SMALLINT), (np.int32, abi.TYPE_INT),
         (np.float32, abi.TYPE_FLOAT), (np.int64, abi.TYPE_BIGINT), (np.float64, abi.TYPE_DOUBLE), (None, abi.TYPE_LARGEINT),
         (None, abi.TYPE_DECIMAL128)]


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _columns(dt, typ, rng):
    """(name, raw bytes of the values): shaped like the frame-of-reference page tests' columns, plus float specials"""
    w = abi.TYPE_WIDTH[typ]
    if dt is None:                                                   # 16-byte two's-complement values as bytes
        def wide(lo):
            v = np.zeros((len(lo), 16), dtype=np.uint8)
            v[:, :8] = lo.astype(np.int64).view(np.uint8).reshape(-1, 8)
            v[:, 8:] = np.where(lo < 0, 255, 0)[:, None]
            return v.reshape(-1)
        yield "ssb_keys_22bit", wide(rng.integers(1, 3_000_000, 20_003))
        yield "negative_mixed", wide(rng.integers(-10**6, 10**6, 5_001))
        yield "full_range", rng.integers(0, 256, 16 * 3000).astype(np.uint8)
        yield "one_value", wide(np.array([-7]))
        yield "empty", np.zeros(0, dtype=np.uint8)
        return
    if np.dtype(dt).kind == "f":
        yield "ssb_like", rng.normal(0, 1e6, 100_003).astype(dt).view(np.uint8)
        yield "specials", np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1e-40, -1.5] * 301, dtype=dt).view(np.uint8)
        yield "payload_nan", (np.array([0x7FC00001, 0xFFF00002] * 50, dtype=np.uint32 if w == 4 else np.uint64)).view(np.uint8)
        yield "constant", np.full(1000, 42.5, dtype=dt).view(np.uint8)
        yield "one_value", np.array([-0.0], dtype=dt).view(np.uint8)
        yield "empty", np.zeros(0, dtype=np.uint8)
        return
    info = np.iinfo(dt)
    yield "ssb_keys_22bit", rng.integers(0, min(3_000_000, int(info.max)), 100_003).astype(dt).view(np.uint8)
    yield "dates_ascending", np.sort(rng.integers(19920101, 19981231, 70_000)).astype(dt).view(np.uint8)
    yield "constant", np.full(1000, 42, dtype=dt).view(np.uint8)
    yield "negative_mixed", rng.integers(max(-10**6, int(info.min)), min(10**6, int(info.max)), 12_345).astype(dt).view(np.uint8)
    yield "full_range", rng.integers(int(info.min), int(info.max), 5000, dtype=dt, endpoint=True).view(np.uint8)
    yield "one_value", np.array([7], dtype=dt).view(np.uint8)
    yield "empty", np.zeros(0, dtype=np.uint8)


def _pages(bo, raw, w, page_rows):
    n = len(raw) // w
    return [bo.bitshuffle_encode(raw[lo * w:(lo + page_rows) * w], w) for lo in range(0, max(n, 1), page_rows)]


def _decode(gpu, ctx, dec, typ, pages, n, mem, w, cap=None, sentinel=8):
    """decode into a fresh device byte column with `sentinel` values of 0xA5 past the column; -> (rows, host bytes)"""
    import torch
    out = torch.full(((n + sentinel) * w,), 0xA5, dtype=torch.uint8, device="cuda")
    cap = n if cap is None else cap
    keep = []
    if mem == "host":
        rows = dec.decode(abi.PAGE_BITSHUFFLE, typ, pages, out.data_ptr(), cap)
    elif mem == "device":                                            # every page at a different byte alignment
        views = []
        for k, pg in enumerate(pages):
            b = torch.from_numpy(np.concatenate([np.zeros(k % 4 + 1, dtype=np.uint8), pg])).cuda()
            keep.append(b)
            views.append((b.data_ptr() + k % 4 + 1, len(pg)))
        rows = dec.decode(abi.PAGE_BITSHUFFLE, typ, views, out.data_ptr(), cap, mem=abi.MEM_DEVICE)
    else:
        # pinned_run: pages back to back (one run of >= 256 KB is staged by DMA); pinned_scattered: 100-byte gaps, odd
        # alignments (read in place over PCIe)
        gap = 0 if mem == "pinned_run" else 100
        offs, at = [], 0
        for k, pg in enumerate(pages):
            at += 0 if gap == 0 else gap + k % 3
            offs.append(at)
            at += len(pg)
        blob = torch.zeros(max(at, 1), dtype=torch.uint8).pin_memory()
        bn = blob.numpy()
        for o, pg in zip(offs, pages):
            bn[o:o + len(pg)] = pg
        keep.append(blob)
        rows = dec.decode(abi.PAGE_BITSHUFFLE, typ, [(blob.data_ptr() + o, len(pg)) for o, pg in zip(offs, pages)], out.data_ptr(), cap,
                          mem=abi.MEM_HOST_PINNED)
    ctx.sync()
    return rows, out.cpu().numpy()


@pytest.mark.parametrize("dt,typ", TYPES, ids=lambda x: getattr(x, "__name__", str(x)))
@pytest.mark.parametrize("page_rows", [1000, 65_536])
@pytest.mark.parametrize("mem", ["host", "device", "pinned_run", "pinned_scattered"])
def test_bitshuffle_pages_decode_parity(gpu, ctx, bo, dt, typ, page_rows, mem):
    rng = np.random.default_rng(11)
    w = abi.TYPE_WIDTH[typ]
    dec = gpu.PageDecoder(ctx)
    try:
        for name, raw in _columns(dt, typ, rng):
            n = len(raw) // w
            pages = _pages(bo, raw, w, page_rows)
            assert (np.concatenate([bo.bitshuffle_decode(p, w) for p in pages]) == raw).all(), name
            rows, got = _decode(gpu, ctx, dec, typ, pages, n, mem, w)
            assert rows == n, name
            assert (got[:n * w] == raw).all(), name                  # bit for bit: NaN payloads and -0.0 included
            assert (got[n * w:] == 0xA5).all(), name                 # nothing written past the column
    finally:
        dec.close()


def test_many_pages_of_different_sizes(gpu, ctx, bo):
    # one call over pages of 1 .. 70 000 values (odd counts shift every later page's first row off alignment)
    rng = np.random.default_rng(12)
    dec = gpu.PageDecoder(ctx)
    try:
        for typ in (abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_BIGINT, abi.TYPE_LARGEINT):
            w = abi.TYPE_WIDTH[typ]
            sizes = [1, 7, 8, 9, 8192 // w, 8192 // w + 8, 8192 // w * 7 // 2, 70_000, 3, 0, 12_345]
            raws = [rng.integers(0, 1 << min(8 * w - 1, 40), s).astype(np.int64).view(np.uint8).reshape(-1, 8)[:, :w].reshape(-1).copy()
                    if w <= 8 else rng.integers(0, 256, 16 * s).astype(np.uint8) for s in sizes]
            pages = [bo.bitshuffle_encode(r, w) for r in raws]
            raw = np.concatenate(raws)
            for mem in ("host", "device", "pinned_scattered"):
                rows, got = _decode(gpu, ctx, dec, typ, pages, len(raw) // w, mem, w)
                assert rows == len(raw) // w
                assert (got[:len(raw)] == raw).all(), (typ, mem)
                assert (got[len(raw):] == 0xA5).all()
    finally:
        dec.close()


def test_golden_liblz4_pages_and_streams(gpu, ctx, bo):
    # pages whose blocks liblz4 compressed, and every hand-built stream that fits one block of a 1-byte-wide page: the ones
    # liblz4 accepts decode to its output, the ones it rejects are refused
    dec = gpu.PageDecoder(ctx)
    types = {1: abi.TYPE_TINYINT, 2: abi.TYPE_SMALLINT, 4: abi.TYPE_INT, 8: abi.TYPE_BIGINT, 16: abi.TYPE_LARGEINT}
    tried = 0
    try:
        for name, kind, width, size, verdict, data, want in golden():
            if kind == "page":
                rows, got = _decode(gpu, ctx, dec, types[width], [data], len(want) // width, "device", width)
                assert rows == len(want) // width and (got[:len(want)] == want).all(), name
                continue
            if size % 8 or size > 8192:
                continue
            page = _stream_page(data, size)
            tried += 1
            if verdict:
                rows, got = _decode(gpu, ctx, dec, abi.TYPE_TINYINT, [page], size, "host", 1)
                assert rows == size and (got[:size] == bo.untrans_bit_elem(want, 1)).all(), name
            else:
                with pytest.raises(gpu.GpuError) as ei:
                    _decode(gpu, ctx, dec, abi.TYPE_TINYINT, [page], size, "host", 1)
                assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
        assert tried >= 12
    finally:
        dec.close()


def _stream_page(stream, size):
    """a 1-byte-wide page of `size` values (size % 8 == 0, <= 8192: one block) holding one LZ4 stream"""
    stream = np.asarray(stream, dtype=np.uint8)
    hdr = np.array([size, 16 + 4 + len(stream), size, 1], dtype="<u4").view(np.uint8)
    return np.concatenate([hdr, np.frombuffer(len(stream).to_bytes(4, "big"), dtype=np.uint8), stream])


def test_malformed_pages_then_a_good_call(gpu, ctx, bo):
    import torch
    v = np.random.default_rng(13).integers(0, 1 << 20, 5000).astype(np.int32)
    good = bo.bitshuffle_encode(v)
    out = torch.zeros(2 * len(v) + 8, dtype=torch.int32, device="cuda")

    def with_word(k, x):
        p = good.copy()
        p[4 * k:4 * k + 4] = np.array([x], dtype="<u4").view(np.uint8)
        return p

    def with_len(pos, x):
        p = good.copy()
        p[pos:pos + 4] = np.frombuffer(int(x).to_bytes(4, "big"), dtype=np.uint8)
        return p

    first = int.from_bytes(good[16:20].tobytes(), "big")
    bad = {"short_header": good[:12], "size_mismatch": with_word(1, len(good) + 4), "wrong_padded_count": with_word(2, 5008),
           "wrong_element_size": with_word(3, 8), "chain_overruns_page": with_len(16, len(good)),
           "block_over_8240": with_len(16, 8241), "chain_ends_early": np.concatenate([good, np.zeros(4, dtype=np.uint8)]),
           "second_block_overruns": with_len(20 + first, len(good))}
    bad["chain_ends_early"][4:8] = np.array([len(good) + 4], dtype="<u4").view(np.uint8)
    dec = gpu.PageDecoder(ctx)
    try:
        for name, page in list(bad.items()) + [("corrupt_stream_%s" % nm, _stream_page(d, sz)) for nm, kind, _, sz, ok, d, _ in golden()
                                                 if kind == "lz4" and not ok and sz % 8 == 0 and sz <= 8192]:
            typ = abi.TYPE_TINYINT if name.startswith("corrupt_stream") else abi.TYPE_INT
            pages, cap = ([good, page], 2 * len(v)) if typ == abi.TYPE_INT else ([page], 4 * len(v))     # behind a good page
            with pytest.raises(gpu.GpuError) as ei:
                dec.decode(abi.PAGE_BITSHUFFLE, typ, pages, out.data_ptr(), cap)
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
        with pytest.raises(gpu.GpuError) as ei:                                                      # output capacity too small
            dec.decode(abi.PAGE_BITSHUFFLE, abi.TYPE_INT, [good], out.data_ptr(), len(v) - 1)
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
        with pytest.raises(gpu.GpuError) as ei:                                                      # a width that is not fixed
            dec.decode(abi.PAGE_BITSHUFFLE, 0, [good], out.data_ptr(), len(v))
        assert ei.value.code == abi.SR_ERR_NOT_SUPPORTED
        assert dec.decode(abi.PAGE_BITSHUFFLE, abi.TYPE_INT, [good], out.data_ptr(), len(v)) == len(v)   # the decoder still works
        ctx.sync()
        assert (out.cpu().numpy()[:len(v)] == v).all()
    finally:
        dec.close()


def test_bitshuffle_pages_feed_the_scan(gpu, ctx, bo):
    # lineorder-shaped columns written as bitshuffle pages, decoded, then scanned: equal to the oracle's scan of the raw values
    import torch
    from oracle import oracle
    rng = np.random.default_rng(14)
    n = 300_000
    custkey = rng.integers(1, 3_000_000, n).astype(np.int32)
    orderdate = np.sort(rng.integers(19920101, 19981231, n)).astype(np.int32)
    revenue = rng.integers(1, 10_000_000, n).astype(np.int64)
    dec = gpu.PageDecoder(ctx)
    try:
        cols = []
        for v, typ, rows in ((custkey, abi.TYPE_INT, 16_384), (orderdate, abi.TYPE_DATE, 16_384), (revenue, abi.TYPE_BIGINT, 8_192)):
            d = torch.empty(n, dtype=torch.int32 if v.dtype == np.int32 else torch.int64, device="cuda")
            pages = [bo.bitshuffle_encode(v[lo:lo + rows]) for lo in range(0, n, rows)]
            assert dec.decode(abi.PAGE_BITSHUFFLE, typ, pages, d.data_ptr(), n) == n
            cols.append(d)
        ctx.sync()
        sd = abi.ScanDesc(preds=[abi.make_pred(0, abi.PRED_LT, 1_000_000), abi.make_pred(1, abi.PRED_BETWEEN, 19940101, 19941231)], out_slots=[0, 1, 2])
        sc = gpu.Scan(ctx, sd)
        try:
            got = gpu.chunk_out_to_host(ctx, sc.filter(Chunk([(0, cols[0], None), (1, cols[1], None), (2, cols[2], None)], num_rows=n, mem=abi.MEM_DEVICE)))
        finally:
            sc.close()
        rows, ores = oracle.scan_filter(sd, Chunk([(0, custkey, None), (1, orderdate, None), (2, revenue, None)]))
        gcols = {s: d for s, _, d, _ in got}
        assert rows > 0 and len(gcols[0]) == rows
        for s in (0, 1, 2):
            assert (gcols[s] == ores[s][0]).all()
    finally:
        dec.close()
