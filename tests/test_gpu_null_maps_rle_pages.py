"""Null maps of nullable columns (BITSHUFFLE_NULL and RLE_NULL) and BOOLEAN RLE pages decoded on the device
(sr_null_maps_decode, sr_pages_decode with SR_PAGE_RLE), bit-exact against the CPU codec in bshuf_oracle, and the decoded
columns carried through the scan, the aggregate and the fragment."""
import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

pytestmark = pytest.mark.gpu

MEMS = ["host", "device", "pinned_run", "pinned_scattered"]
ENCS = [abi.NULL_BITSHUFFLE, abi.NULL_RLE]
ENC_IDS = ["bitshuffle", "rle"]


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _flags(kind, n, rng):
    if kind == "none":
        return np.zeros(n, np.uint8)
    if kind == "all":
        return np.ones(n, np.uint8)
    if kind == "clustered":                                           # runs of ~1000 NULLs, ~10 % of the rows
        f = np.zeros(n, np.uint8)
        for s in rng.integers(0, max(n, 1), max(1, n // 10_000)):
            f[s:s + 1000] = 1
        return f
    return (rng.random(n) < float(kind)).astype(np.uint8)


NULL_KINDS = ["none", "0.001", "0.01", "0.1", "0.5", "clustered", "all"]


def _bools(kind, n, rng):
    if kind == "random":
        return rng.integers(0, 2, n).astype(np.uint8)
    if kind == "long_runs":
        return np.repeat(rng.integers(0, 2, n // 5000 + 1), 5000)[:n].astype(np.uint8)
    if kind == "alternating_8":
        return np.repeat(np.arange(n // 8 + 1) % 2, 8)[:n].astype(np.uint8)
    return np.ones(n, np.uint8)


def _place(bufs, mem, keep):
    """byte buffers -> [(pointer, size)] in `mem` (host: the arrays themselves), as sr_pages_decode's memory tests lay them"""
    import torch
    if mem == "host":
        return bufs, abi.MEM_HOST
    if mem == "device":                                               # every buffer at a different byte alignment
        out = []
        for k, b in enumerate(bufs):
            t = torch.from_numpy(np.concatenate([np.zeros(k % 4 + 1, np.uint8), b])).cuda()
            keep.append(t)
            out.append((t.data_ptr() + k % 4 + 1, len(b)))
        return out, abi.MEM_DEVICE
    gap = 0 if mem == "pinned_run" else 100                           # one staged run / scattered, read in place
    offs, at = [], 0
    for k, b in enumerate(bufs):
        at += 0 if gap == 0 else gap + k % 3
        offs.append(at)
        at += len(b)
    blob = torch.zeros(max(at, 1), dtype=torch.uint8).pin_memory()
    bn = blob.numpy()
    for o, b in zip(offs, bufs):
        bn[o:o + len(b)] = b
    keep.append(blob)
    return [(blob.data_ptr() + o, len(b)) for o, b in zip(offs, bufs)], abi.MEM_HOST_PINNED


def _out(n, skew=0, sentinel=16):
    import torch
    return torch.full((n + skew + sentinel,), 0xA5, dtype=torch.uint8, device="cuda")


def _decode_nulls(ctx, dec, enc, maps, rows, mem, skew=0, cap=None):
    """-> (rows, null_count, host bytes of the column with its sentinels)"""
    keep = []
    n = int(sum(rows))
    placed, m = _place(maps, mem, keep)
    views = [(p, r) if m == abi.MEM_HOST else (p[0], p[1], r) for p, r in zip(placed, rows)]
    out = _out(n, skew)
    got = dec.decode_nulls(enc, views, out.data_ptr() + skew, n if cap is None else cap, mem=m)
    ctx.sync()
    return got[0], got[1], out.cpu().numpy()[skew:]


def _decode_rle(ctx, dec, pages, n, mem, skew=0):
    keep = []
    placed, m = _place(pages, mem, keep)
    out = _out(n, skew)
    rows = dec.decode(abi.PAGE_RLE, abi.TYPE_BOOLEAN, placed, out.data_ptr() + skew, n, mem=m)
    ctx.sync()
    return rows, out.cpu().numpy()[skew:]


def _split(n, page_rows):
    return [(lo, min(lo + page_rows, n)) for lo in range(0, n, page_rows)]


@pytest.mark.parametrize("enc", ENCS, ids=ENC_IDS)
@pytest.mark.parametrize("page_rows", [1000, 65_536])
@pytest.mark.parametrize("mem", MEMS)
def test_null_maps_parity(gpu, ctx, bo, enc, page_rows, mem):
    rng = np.random.default_rng(31)
    dec = gpu.PageDecoder(ctx)
    try:
        for kind in NULL_KINDS:
            n = 7 * page_rows + 333                                   # an odd last page
            f = _flags(kind, n, rng)
            parts = _split(n, page_rows)
            maps = [bo.null_map_encode(f[a:b], enc) for a, b in parts]
            assert (np.concatenate([bo.null_map_decode(m, b - a, enc) for m, (a, b) in zip(maps, parts)]) == f).all(), kind
            for skew in (0, 3):
                rows, cnt, got = _decode_nulls(ctx, dec, enc, maps, [b - a for a, b in parts], mem, skew)
                assert rows == n and cnt == int(f.sum()), (kind, skew)
                assert (got[:n] == f).all(), (kind, skew)
                assert (got[n:] == 0xA5).all(), (kind, skew)
    finally:
        dec.close()


@pytest.mark.parametrize("page_rows", [1000, 65_536])
@pytest.mark.parametrize("mem", MEMS)
def test_bool_rle_pages_parity(gpu, ctx, bo, page_rows, mem):
    rng = np.random.default_rng(32)
    dec = gpu.PageDecoder(ctx)
    try:
        for kind in ["random", "long_runs", "alternating_8", "ones"]:
            n = 5 * page_rows + 77
            v = _bools(kind, n, rng)
            pages = [bo.rle_bool_page_encode(v[a:b]) for a, b in _split(n, page_rows)]
            assert (np.concatenate([bo.rle_bool_page_decode(p) for p in pages]) == v).all()
            rows, got = _decode_rle(ctx, dec, pages, n, mem, skew=1)
            assert rows == n, kind
            assert (got[:n] == v).all(), kind
            assert (got[n:] == 0xA5).all(), kind
    finally:
        dec.close()


def test_staged_pinned_run(gpu, ctx, bo):
    # maps and pages back to back in page-locked memory, >= 256 KB in all: one run, staged by DMA
    rng = np.random.default_rng(39)
    n = 3_000_000
    f = (rng.random(n) < 0.5).astype(np.uint8)
    parts = _split(n, 65_536)
    dec = gpu.PageDecoder(ctx)
    try:
        for enc in ENCS:
            maps = [bo.null_map_encode(f[a:b], enc) for a, b in parts]
            assert sum(len(m) for m in maps) >= 256 << 10
            rows, cnt, got = _decode_nulls(ctx, dec, enc, maps, [b - a for a, b in parts], "pinned_run", skew=5)
            assert rows == n and cnt == int(f.sum()) and (got[:n] == f).all() and (got[n:] == 0xA5).all(), enc
        pages = [bo.rle_bool_page_encode(f[a:b]) for a, b in parts]
        assert sum(len(p) for p in pages) >= 256 << 10
        rows, got = _decode_rle(ctx, dec, pages, n, "pinned_run", skew=5)
        assert rows == n and (got[:n] == f).all() and (got[n:] == 0xA5).all()
    finally:
        dec.close()


def test_pages_of_odd_sizes_in_one_call(gpu, ctx, bo):
    # page sizes that put every later page's first row at another byte offset, empty pages and maps among them
    rng = np.random.default_rng(33)
    sizes = [1, 7, 0, 1000, 13, 8, 9, 65_536, 3, 8191, 8193, 5, 0, 64, 65]
    n = sum(sizes)
    v = rng.integers(0, 2, n).astype(np.uint8)
    v[1000:2000] = 1
    f = (rng.random(n) < 0.2).astype(np.uint8)
    at = np.cumsum([0] + sizes)
    f[at[4]:at[7]] = 0                                                # pages with no NULL: empty maps
    dec = gpu.PageDecoder(ctx)
    try:
        pages = [bo.rle_bool_page_encode(v[at[k]:at[k + 1]]) for k in range(len(sizes))]
        for skew in range(8):
            rows, got = _decode_rle(ctx, dec, pages, n, "device", skew)
            assert rows == n and (got[:n] == v).all() and (got[n:] == 0xA5).all(), skew
        for enc in ENCS:
            maps = [bo.null_map_encode(f[at[k]:at[k + 1]], enc) for k in range(len(sizes))]
            assert any(len(m) == 0 and s > 0 for m, s in zip(maps, sizes))
            for skew in range(8):
                rows, cnt, got = _decode_nulls(ctx, dec, enc, maps, sizes, "pinned_scattered", skew)
                assert rows == n and cnt == int(f.sum()), (enc, skew)
                assert (got[:n] == f).all() and (got[n:] == 0xA5).all(), (enc, skew)
    finally:
        dec.close()


def test_hand_built_streams(gpu, ctx, bo):
    # what the encoder never writes but the reference decodes: multi-byte repeat headers, long literal runs, values and bytes
    # past the count, the known-answer stream with a literal tail
    def vlq(x):
        o = []
        while x >= 0x80:
            o.append(x & 0x7F | 0x80)
            x >>= 7
        return o + [x]
    body = np.random.default_rng(34).integers(0, 256, 200, dtype=np.uint8)
    cases = [(np.array([0xC8, 0x01, 0x00, 0x03, 0x07], np.uint8), 103),
             (np.array(vlq(2 ** 14 << 1) + [1, 0x03, 0x05], np.uint8), 2 ** 14 + 3),
             (np.array(vlq((2 ** 21 + 5) << 1) + [0, 0x03, 0x05], np.uint8), 2 ** 21 + 3),
             (np.concatenate([np.array(vlq(200 << 1 | 1), np.uint8), body]), 1597),
             (np.array([0x20, 0x01, 0xFF, 0xFF, 0xFF], np.uint8), 5),
             (np.array([63 << 1 | 1, 0x0F], np.uint8), 4),
             (np.array([0x90, 0x80, 0x80, 0x80, 0x00, 0x01], np.uint8), 8)]
    dec = gpu.PageDecoder(ctx)
    try:
        for k, (s, n) in enumerate(cases):
            want = bo.rle_decode(s, n)
            rows, cnt, got = _decode_nulls(ctx, dec, abi.NULL_RLE, [s], [n], "device", skew=k % 8)
            assert rows == n and cnt == int(want.sum()) and (got[:n] == want).all() and (got[n:] == 0xA5).all(), k
            page = np.concatenate([np.array([n], "<u4").view(np.uint8), s])
            rows, got = _decode_rle(ctx, dec, [page], n, "host", skew=k % 8)
            assert rows == n and (got[:n] == want).all() and (got[n:] == 0xA5).all(), k
    finally:
        dec.close()


def _malformed_rle():
    from tests.test_rle_oracle import MALFORMED
    return [(name, s, n) for name, s, n in MALFORMED]


def test_malformed_maps_and_pages_then_a_good_call(gpu, ctx, bo):
    rng = np.random.default_rng(35)
    f = (rng.random(20_000) < 0.1).astype(np.uint8)
    good = {e: bo.null_map_encode(f, e) for e in ENCS}
    gpage = bo.rle_bool_page_encode(f)
    bs = good[abi.NULL_BITSHUFFLE]
    bad_bs = {"chain_longer": np.concatenate([bs, np.zeros(1, np.uint8)]), "chain_shorter": bs[:-1],
              "length_overruns": np.concatenate([np.frombuffer((len(bs) + 100).to_bytes(4, "big"), np.uint8), bs[4:]]),
              "length_over_8240": np.concatenate([np.frombuffer((9000).to_bytes(4, "big"), np.uint8), bs[4:]]),
              "lz4_garbage": np.concatenate([bs[:4], np.full(len(bs) - 4, 0xF0, np.uint8)]), "map_of_zero_rows": bs}
    dec = gpu.PageDecoder(ctx)
    try:
        def good_call():
            for e in ENCS:
                rows, cnt, got = _decode_nulls(ctx, dec, e, [good[e]], [len(f)], "host")
                assert rows == len(f) and cnt == int(f.sum()) and (got[:len(f)] == f).all()
            rows, got = _decode_rle(ctx, dec, [gpage], len(f), "host")
            assert rows == len(f) and (got[:len(f)] == f).all()

        for name, m in bad_bs.items():
            n = 0 if name == "map_of_zero_rows" else len(f)
            with pytest.raises(gpu.GpuError) as ei:
                _decode_nulls(ctx, dec, abi.NULL_BITSHUFFLE, [good[abi.NULL_BITSHUFFLE], m], [len(f), n], "device")
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
            good_call()
        for name, s, n in _malformed_rle():
            if len(s):                                                # (an empty map is a page without NULLs)
                with pytest.raises(gpu.GpuError) as ei:               # behind a good map
                    _decode_nulls(ctx, dec, abi.NULL_RLE, [good[abi.NULL_RLE], s], [len(f), n], "device")
                assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
                good_call()
            page = np.concatenate([np.array([n], "<u4").view(np.uint8), s])
            with pytest.raises(gpu.GpuError) as ei:
                _decode_rle(ctx, dec, [gpage, page], len(f) + n, "device")
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
            good_call()
        for k in range(4):                                            # shorter than the page's value count
            with pytest.raises(gpu.GpuError) as ei:
                _decode_rle(ctx, dec, [np.zeros(k, np.uint8)], 8, "host")
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
            good_call()
        # a malformed map writes nothing past the pages' rows
        rows_n = len(f) + 9
        out = _out(rows_n)
        with pytest.raises(gpu.GpuError):
            dec.decode_nulls(abi.NULL_RLE, [(good[abi.NULL_RLE], len(f)), (np.array([0x10, 0x01], np.uint8), 9)], out.data_ptr(), rows_n)
        ctx.sync()
        assert (out.cpu().numpy()[rows_n:] == 0xA5).all()
        good_call()
    finally:
        dec.close()


def test_argument_errors_launch_nothing(gpu, ctx, bo):
    f = np.zeros(1000, np.uint8)
    f[::7] = 1
    m = bo.null_map_encode(f, abi.NULL_RLE)
    out = _out(2000)
    dec = gpu.PageDecoder(ctx)
    try:
        for first in (True, False):
            before = ctx.launches
            cases = [(abi.SR_ERR_NOT_SUPPORTED, lambda: dec.decode_nulls(2, [(m, 1000)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_NOT_SUPPORTED, lambda: dec.decode_nulls(-1, [(m, 1000)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m, 1000)], out.data_ptr(), 999)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m, -1)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m.ctypes.data, -5, 1000)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(None, 5, 1000)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m, 2 ** 32)], out.data_ptr(), 2 ** 33)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m, 1000)], 0, 2000)),
                     (abi.SR_ERR_INVALID_ARGUMENT, lambda: dec.decode_nulls(abi.NULL_RLE, [(m, 1000)], out.data_ptr(), 2000, mem=7)),
                     (abi.SR_ERR_NOT_SUPPORTED, lambda: dec.decode(abi.PAGE_RLE, abi.TYPE_INT, [bo.rle_bool_page_encode(f)], out.data_ptr(), 2000)),
                     (abi.SR_ERR_NOT_SUPPORTED, lambda: dec.decode(abi.PAGE_RLE, abi.TYPE_TINYINT, [bo.rle_bool_page_encode(f)], out.data_ptr(), 2000))]
            for code, call in cases:
                with pytest.raises(gpu.GpuError) as ei:
                    call()
                assert ei.value.code == code
            assert ctx.launches == before
            assert dec.decode_nulls(abi.NULL_RLE, [], out.data_ptr(), 0) == (0, 0)
            assert dec.decode_nulls(abi.NULL_RLE, [(m, 1000)], out.data_ptr(), 1000) == (1000, int(f.sum()))
    finally:
        dec.close()


def test_other_encodings_unchanged_after_rle_and_map_calls(gpu, ctx, bo, oracle):
    import torch
    v = np.random.default_rng(36).integers(-10**6, 10**6, 70_001).astype(np.int32)
    pages = {abi.PAGE_BITSHUFFLE: [bo.bitshuffle_encode(v[lo:lo + 8192]) for lo in range(0, len(v), 8192)],
             abi.PAGE_FOR: [oracle.for_encode(v[lo:lo + 8192]) for lo in range(0, len(v), 8192)],
             abi.PAGE_DICT: [bo.dict_page_encode(np.abs(v[lo:lo + 8192]) % 7) for lo in range(0, len(v), 8192)]}
    want = {abi.PAGE_BITSHUFFLE: v, abi.PAGE_FOR: v, abi.PAGE_DICT: (np.abs(v) % 7) + 100}
    f = (np.random.default_rng(37).random(len(v)) < 0.1).astype(np.uint8)
    nulls = _out(len(v))
    dec = gpu.PageDecoder(ctx)
    try:
        dec.set_dict(np.arange(100, 107, dtype=np.int32))
        for enc, pg in pages.items():
            before = torch.zeros(len(v), dtype=torch.int32, device="cuda")
            after = torch.zeros(len(v), dtype=torch.int32, device="cuda")
            assert dec.decode(enc, abi.TYPE_INT, pg, before.data_ptr(), len(v)) == len(v)
            for e in ENCS:
                assert dec.decode_nulls(e, [(bo.null_map_encode(f, e), len(f))], nulls.data_ptr(), len(f))[0] == len(f)
            assert dec.decode(abi.PAGE_RLE, abi.TYPE_BOOLEAN, [bo.rle_bool_page_encode(f)], nulls.data_ptr(), len(f)) == len(f)
            assert dec.decode(enc, abi.TYPE_INT, pg, after.data_ptr(), len(v)) == len(v)
            ctx.sync()
            assert (before.cpu().numpy() == want[enc]).all() and (after.cpu().numpy() == want[enc]).all(), enc
    finally:
        dec.close()


# ---- end to end: nullable SSB-shaped columns decoded from value pages + null maps, and a BOOLEAN RLE column ------------
def _decoded_columns(gpu, ctx, bo, oracle, n, null_frac, enc):
    """lo_custkey (BIT_SHUFFLE values + map), lo_revenue (FOR values + map), lo_flag (BOOLEAN RLE) -> device tensors and the
    host arrays they must equal.  -> (cols: name -> (data, nulls or None when the batch has no NULL), values, null flags,
    null counts)"""
    import torch
    rng = np.random.default_rng(38)
    host = {"custkey": rng.integers(1, 30_000, n).astype(np.int32), "revenue": rng.integers(1, 10_000_000, n).astype(np.int32),
            "flag": rng.integers(0, 2, n).astype(np.uint8)}
    nul = {"custkey": (rng.random(n) < null_frac).astype(np.uint8), "revenue": (rng.random(n) < null_frac).astype(np.uint8)}
    parts = _split(n, 65_536)
    dec = gpu.PageDecoder(ctx)
    cols, counts = {}, {}
    try:
        for name, vpage, code in (("custkey", bo.bitshuffle_encode, abi.PAGE_BITSHUFFLE), ("revenue", oracle.for_encode, abi.PAGE_FOR)):
            t = torch.empty(n, dtype=torch.int32, device="cuda")
            nt = torch.empty(n, dtype=torch.uint8, device="cuda")
            # a page body is `values | null map`: split by the footer's nullmap_size
            bodies = [np.concatenate([vpage(host[name][a:b]), bo.null_map_encode(nul[name][a:b], enc)]) for a, b in parts]
            sizes = [len(bo.null_map_encode(nul[name][a:b], enc)) for a, b in parts]
            vals = [body[:len(body) - s] for body, s in zip(bodies, sizes)]
            maps = [(body[len(body) - s:], b - a) for body, s, (a, b) in zip(bodies, sizes, parts)]
            rows = dec.decode(code, abi.TYPE_INT, vals, t.data_ptr(), n)
            nrows, cnt = dec.decode_nulls(enc, maps, nt.data_ptr(), n)
            assert rows == nrows == n
            counts[name] = cnt
            cols[name] = (t, nt if cnt > 0 else None)
        ft = torch.empty(n, dtype=torch.uint8, device="cuda")
        assert dec.decode(abi.PAGE_RLE, abi.TYPE_BOOLEAN, [bo.rle_bool_page_encode(host["flag"][a:b]) for a, b in parts], ft.data_ptr(), n) == n
        cols["flag"] = (ft, None)
    finally:
        dec.close()
    return cols, host, nul, counts


CUST, REV, FLAG, OUT_SUM, OUT_CNT, OUT_CNT_STAR, DIM_KEY, DIM_NATION = 1, 2, 3, 10, 11, 12, 20, 21


@pytest.mark.parametrize("null_frac", [0.1, 0.0], ids=["nulls", "no_nulls"])
@pytest.mark.parametrize("enc", ENCS, ids=ENC_IDS)
def test_end_to_end_scan_agg_fragment(gpu, ctx, bo, oracle, null_frac, enc):
    import torch
    n = 300_007
    cols, h, nul, counts = _decoded_columns(gpu, ctx, bo, oracle, n, null_frac, enc)
    for k in ("custkey", "revenue"):
        assert counts[k] == int(nul[k].sum())
        assert (cols[k][1] is None) == (null_frac == 0.0)               # no NULL in the batch: passed as nulls = NULL
        if cols[k][1] is not None:
            assert (cols[k][1].cpu().numpy() == nul[k]).all()
    chunk = Chunk([(CUST, cols["custkey"][0], cols["custkey"][1], abi.TYPE_INT), (REV, cols["revenue"][0], cols["revenue"][1], abi.TYPE_INT),
                   (FLAG, cols["flag"][0], None, abi.TYPE_BOOLEAN)], num_rows=n, mem=abi.MEM_DEVICE)
    cn, rn = nul["custkey"].astype(bool), nul["revenue"].astype(bool)

    # scan: IS NULL, IS NOT NULL, a range on a nullable column, EQ on the boolean
    scans = [([abi.make_pred(CUST, abi.PRED_IS_NULL)], cn),
             ([abi.make_pred(REV, abi.PRED_IS_NOT_NULL)], ~rn),
             ([abi.make_pred(CUST, abi.PRED_BETWEEN, 1000, 9000)], ~cn & (h["custkey"] >= 1000) & (h["custkey"] <= 9000)),
             ([abi.make_pred(FLAG, abi.PRED_EQ, 1), abi.make_pred(REV, abi.PRED_LT, 5_000_000)], (h["flag"] == 1) & ~rn & (h["revenue"] < 5_000_000))]
    for preds, keep in scans:
        scan = gpu.Scan(ctx, abi.ScanDesc(preds=preds, out_slots=[CUST, REV]))
        try:
            out = gpu.chunk_out_to_host(ctx, scan.filter(chunk))
            assert len(out[0][2]) == int(keep.sum())
            assert (out[0][2][~cn[keep]] == h["custkey"][keep][~cn[keep]]).all()
            assert (out[1][2][~rn[keep]] == h["revenue"][keep][~rn[keep]]).all()
            if out[0][3] is not None:
                assert (out[0][3].astype(bool) == cn[keep]).all()
            else:
                assert not cn[keep].any()
        finally:
            scan.close()

    # aggregate: GROUP BY the boolean, SUM / COUNT / COUNT(*) of the nullable revenue
    agg = gpu.Agg(ctx, abi.make_agg_desc([FLAG], [abi.TYPE_BOOLEAN], fns=[(abi.AGG_SUM, abi.TYPE_INT, OUT_SUM, [("col", REV)]),
                                                                           (abi.AGG_COUNT, abi.TYPE_INT, OUT_CNT, [("col", REV)]),
                                                                           (abi.AGG_COUNT_STAR, 0, OUT_CNT_STAR, None)]))
    try:
        agg.push(chunk)
        res = {slot: (d, nl) for slot, _, d, nl in agg.result()}
        for g, key in enumerate(res[FLAG][0].tolist()):
            m = h["flag"] == key
            assert int(res[OUT_SUM][0][g]) == int(h["revenue"][m & ~rn].astype(np.int64).sum()), key
            assert int(res[OUT_CNT][0][g]) == int((m & ~rn).sum()), key
            assert int(res[OUT_CNT_STAR][0][g]) == int(m.sum()), key
        assert sorted(res[FLAG][0].tolist()) == [0, 1]
    finally:
        agg.close()

    # fragment: the nullable custkey is the foreign key of an INNER join (its NULL rows drop out); SUM(revenue) by nation
    dim_keys = np.arange(1, 30_000, 2, dtype=np.int32)                # half the keys have a dimension row
    dim_nation = (dim_keys % 25).astype(np.int32)
    j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [DIM_KEY], [CUST], [abi.TYPE_INT], build_out=[DIM_NATION], probe_out=[]))
    try:
        j.append_build(Chunk([(DIM_KEY, torch.from_numpy(dim_keys).cuda(), None, abi.TYPE_INT),
                              (DIM_NATION, torch.from_numpy(dim_nation).cuda(), None, abi.TYPE_INT)], num_rows=len(dim_keys), mem=abi.MEM_DEVICE))
        j.build_finish()
        desc = abi.make_agg_desc([DIM_NATION], [abi.TYPE_INT], fns=[(abi.AGG_SUM, abi.TYPE_INT, OUT_SUM, [("col", REV)]),
                                                                    (abi.AGG_COUNT_STAR, 0, OUT_CNT_STAR, None)])
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [(j, CUST, [DIM_NATION])], desc)
        try:
            frag.push(chunk)
            res = {slot: d for slot, _, d, _ in frag.agg.result()}
        finally:
            frag.close()
        hit = ~cn & (h["custkey"] % 2 == 1)
        nat = h["custkey"] % 25
        want = {}
        for g in np.unique(nat[hit]):
            m = hit & (nat == g)
            want[int(g)] = (int(h["revenue"][m & ~rn].astype(np.int64).sum()), int(m.sum()))
        got = {int(g): (int(s), int(c)) for g, s, c in zip(res[DIM_NATION], res[OUT_SUM], res[OUT_CNT_STAR])}
        assert got == want
    finally:
        j.close()
