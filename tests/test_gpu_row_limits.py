"""Every entry point past 2^31 rows and up to its 2^32 limit, against closed-form references.

The row ids, selection entries, join indexes and per-tile counts inside the library are 32 bits wide beside 64-bit bases
and totals; between 2^31 and 2^32 rows a signed reinterpretation or a 32-bit product of them gives a wrong answer without
an error.  These tests push batches of n = 2^31 + 65 rows (the last row has residue 0 mod 251) and, where the device memory
allows, of 0xFFFFFFEF rows, the largest count the row limits accept, and check:

- the exact answer, from Python integers: counts of r < n with r = k (mod 251), and sums over those rows;
- whole output columns (scan survivors, decoded pages, join indexes, partitioned rows) chunk by chunk on the device
  against the closed-form expected sequence built with torch.arange arithmetic (torch only compares);
- the refusals at each documented limit: the first refused count gives its error code before any launch or allocation.

Inputs are made on the device from the row index r: the shared 1-byte column is r % 251 (as TINYINT: 0..127, -128..-6).
Each GPU test states its device budget and skips when the device has less free; the CPU tests check every closed form
against numpy brute force.
"""
import ctypes as C

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

TINYINT, INT, BIGINT, BOOLEAN = abi.TYPE_TINYINT, abi.TYPE_INT, abi.TYPE_BIGINT, abi.TYPE_BOOLEAN
DEV = abi.MEM_DEVICE
GB = 1 << 30
M = 251                                     # the shared column: r % M
N31 = (1 << 31) + 65                        # past 2^31, odd; (N31 - 1) % M == 0
NMAX = 0xFFFFFFEF                           # the largest batch the 0xFFFFFFF0 limits accept
REFUSED = 0xFFFFFFF0                        # the first refused batch
SEL_LIMIT = 0x7FFFFFF0                      # sr_agg_push_selective's first refused batch
STEP = 1 << 26                              # rows per comparison chunk on the device


# =============================================================================================
# closed forms (Python integers)
# =============================================================================================
def tinyint(k):
    """the TINYINT value of the byte k"""
    return k - 256 if k >= 128 else k


def residue_count(n, m, k):
    """#{r < n : r = k (mod m)}, 0 <= k < m"""
    return max(0, (n - k + m - 1) // m)


def range_count(lo, hi, m, k):
    """#{lo <= r < hi : r = k (mod m)}"""
    return residue_count(hi, m, k) - residue_count(lo, m, k)


def shifted_sum(n, m, k, shift, bias):
    """sum of ((r >> shift) - bias) over r < n, r = k (mod m)"""
    total = 0
    for b in range(0, ((n - 1) >> shift) + 1):
        total += (b - bias) * range_count(b << shift, min((b + 1) << shift, n), m, k)
    return total


def last_with_residue(n, m, k):
    return k + m * (residue_count(n, m, k) - 1)


def nth_with_residue(o, s, m):
    """row of the o-th r (from 0, in order) whose residue mod m lies in the sorted list s (o: int or torch tensor)"""
    return (o // len(s)) * m + _index(s, o % len(s))


def _index(s, i):
    if isinstance(i, int):
        return s[i]
    import torch
    return torch.tensor(s, dtype=torch.int64, device=i.device)[i]


def rle_runs_bytes(runs):
    """RLE stream at bit width 1: runs of ("rep", count, bit) or ("lit", [8-bit groups])"""
    out = []

    def vlq(x):
        while x >= 0x80:
            out.append(x & 0x7F | 0x80)
            x >>= 7
        out.append(x)
    for r in runs:
        if r[0] == "rep":
            vlq(r[1] << 1)
            out.append(r[2])
        else:
            vlq(len(r[1]) << 1 | 1)
            out.extend(r[1])
    return np.array(out, np.uint8)


def big_bool_runs(n, head, lit):
    """the runs of a BOOLEAN column of n rows: `head` ones, the 8 bits of `lit`, zeros, a final one"""
    return [("rep", head, 1), ("lit", [lit]), ("rep", n - head - 8 - 1, 0), ("rep", 1, 1)]


def big_bool_expected(r, n, head, lit):
    """value of row r (a torch int64 tensor) of big_bool_runs(n, head, lit)"""
    import torch
    lit_bit = (torch.full_like(r, lit) >> (r - head).clamp(0, 7)) & 1
    return torch.where(r < head, 1, torch.where(r < head + 8, lit_bit, (r == n - 1).long()))


def big_bool_ones(n, head, lit):
    return head + bin(lit).count("1") + 1


KM = 4099                                   # SMALLINT key: (r % KM) - 2049, coprime to M


def smallint_groups(n):
    """{key: (COUNT(*), SUM(tinyint(r % M)))} of GROUP BY (r % KM) - 2049 over r < n, by whole periods of KM * M rows"""
    period = KM * M
    r = np.arange(period, dtype=np.int64)
    g, v = r % KM, r % M
    v = np.where(v >= 128, v - 256, v)
    q, rem = divmod(n, period)
    cnt = [q * int(a) + int(b) for a, b in zip(np.bincount(g, minlength=KM), np.bincount(g[:rem], minlength=KM))]
    sm = [q * int(a) + int(b) for a, b in zip(np.bincount(g, weights=v, minlength=KM).round().astype(np.int64),
                                                np.bincount(g[:rem], weights=v[:rem], minlength=KM).round().astype(np.int64))]
    return {k - 2049: (cnt[k], sm[k]) for k in range(KM) if cnt[k]}


BLK = 8192                                  # one-byte values per bitshuffle block (BSHUF_BLOCK_BYTES)
PATTERN = ((np.arange(BLK) & 0xFF) ^ 0x5A).astype(np.uint8)          # value of row r: (r & 0xFF) ^ 0x5A
NULL_BYTES = (3, 77, 200)
NULL_PATTERN = np.isin(np.arange(BLK) & 0xFF, NULL_BYTES).astype(np.uint8)   # NULL where r & 0xFF is one of NULL_BYTES


def bshuf_block(bo, values):
    """one block of a one-byte bitshuffle stream: the big-endian length and the LZ4 stream of len(values) <= 8192 values"""
    return bo.bitshuffle_encode(values)[16:]


def big_bshuf_page(bo, n):
    """BIT_SHUFFLE page of n (a multiple of 8) one-byte values (r & 0xFF) ^ 0x5A: the block of PATTERN n // 8192 times,
    then the block of the tail, behind the 16-byte header (count, page bytes, padded count, width)"""
    nfull, tail = divmod(n, BLK)
    body = [np.tile(bshuf_block(bo, PATTERN), nfull)] + ([bshuf_block(bo, PATTERN[:tail])] if tail else [])
    body = np.concatenate(body)
    assert n % 8 == 0 and 16 + len(body) < 1 << 32
    return np.concatenate([np.array([n, 16 + len(body), n, 1], "<u4").view(np.uint8), body])


def big_bshuf_null_map(bo, rows):
    """bitshuffle null map of rows (up to UINT32_MAX) whose NULLs follow NULL_PATTERN: one block per 8192 padded rows; the
    padding rows have r & 0xFF = 0xFF, not NULL, so the last block is the same block"""
    assert 0 <= -rows % BLK < 8 and 0xFF not in NULL_BYTES
    return np.tile(bshuf_block(bo, NULL_PATTERN), (rows + 7) // BLK)


# =============================================================================================
# CPU: the closed forms against brute force
# =============================================================================================
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_residue_forms_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    n = 1_000_000 + int(rng.integers(0, 5000))
    r = np.arange(n, dtype=np.int64)
    for m in (M, 7, 1000):
        for k in {0, 1, m // 2, m - 1, int(rng.integers(0, m))}:
            sel = r[r % m == k]
            assert residue_count(n, m, k) == len(sel), (m, k)
            lo, hi = sorted(int(x) for x in rng.integers(0, n, 2))
            assert range_count(lo, hi, m, k) == int(((r >= lo) & (r < hi) & (r % m == k)).sum())
            assert last_with_residue(n, m, k) == int(sel[-1])
            for shift, bias in ((12, 64), (17, 0), (5, 1000)):
                assert shifted_sum(n, m, k, shift, bias) == int(((sel >> shift) - bias).sum()), (m, k, shift)
        s = sorted({int(x) for x in rng.integers(0, m, 7)})
        rows = r[np.isin(r % m, s)]
        o = np.arange(len(rows))
        assert all(nth_with_residue(int(q), s, m) == int(rows[q]) for q in rng.integers(0, len(rows), 200))
        assert np.array_equal((o // len(s)) * m + np.array(s)[o % len(s)], rows)
    assert [tinyint(k) for k in range(256)] == np.arange(256, dtype=np.uint8).view(np.int8).tolist()
    assert (N31 - 1) % M == 0 and N31 % 2 == 1


def test_scan_output_forms_against_brute_force():
    # the survivor sequences the scan tests compare with, on a short prefix of the same column
    n = 1_000_003
    v = (np.arange(n) % M).astype(np.uint8).view(np.int8)
    sparse = v[(v >= 0) & (v <= 9)]
    o = np.arange(len(sparse))
    assert np.array_equal(sparse, (o % 10).astype(np.int8))
    dense = v[v != 5]
    o = np.arange(len(dense))
    j = o % 250
    assert np.array_equal(dense, (j + (j >= 5)).astype(np.uint8).view(np.int8))


@pytest.mark.parametrize("n,head,lit", [(10_000, 4_001, 0x4D), (4097, 2049, 0xB2), (20, 3, 0xFF)])
def test_big_bool_stream_against_the_codec(n, head, lit):
    import torch
    bo = pytest.importorskip("bshuf_oracle")
    bo.lib()
    s = rle_runs_bytes(big_bool_runs(n, head, lit))
    want = big_bool_expected(torch.arange(n), n, head, lit).numpy().astype(np.uint8)
    assert np.array_equal(bo.rle_decode(s, n), want)
    page = np.concatenate([np.array([n], "<u4").view(np.uint8), s])
    assert np.array_equal(bo.rle_bool_page_decode(page), want)
    assert int(want.sum()) == big_bool_ones(n, head, lit)


def test_smallint_groups_against_brute_force():
    n = 3 * KM * M + 12_345
    r = np.arange(n, dtype=np.int64)
    g = r % KM
    v = r % M
    v = np.where(v >= 128, v - 256, v)
    cnt, sm = np.bincount(g, minlength=KM), np.bincount(g, weights=v, minlength=KM).round().astype(np.int64)
    assert smallint_groups(n) == {k - 2049: (int(cnt[k]), int(sm[k])) for k in range(KM)}
    assert smallint_groups(100) == {k - 2049: (1, tinyint(k % M)) for k in range(100)}


def test_big_bitshuffle_builders_against_the_codec():
    bo = pytest.importorskip("bshuf_oracle")
    bo.lib()
    for n in (3 * BLK + 8184, 2 * BLK, 8):
        page = big_bshuf_page(bo, n)
        want = ((np.arange(n) & 0xFF) ^ 0x5A).astype(np.uint8)
        assert np.array_equal(bo.bitshuffle_decode(page, 1), want)
        assert page.tobytes() == bo.bitshuffle_encode(want).tobytes()
    for rows in (3 * BLK - 1, 2 * BLK - 7, 2 * BLK):
        m = big_bshuf_null_map(bo, rows)
        want = np.isin(np.arange(rows) & 0xFF, NULL_BYTES).astype(np.uint8)
        assert np.array_equal(bo.null_map_decode(m, rows, abi.NULL_BITSHUFFLE), want)
        assert m.tobytes() == bo.null_map_encode(want, abi.NULL_BITSHUFFLE).tobytes()


def test_channel_counts_against_brute_force():
    from tests.test_gpu_exchange_edges import FNV, hash_key
    n = 1_000_033
    keys = np.arange(n) % M
    hv = np.array([hash_key(FNV, [bytes([k])]) for k in range(M)], np.uint64)
    ch = ((hv[keys] * np.uint64(16)) >> np.uint64(32)).astype(np.int64)
    want = np.bincount(ch, minlength=16)
    assert channel_counts(n, 16).tolist() == want.tolist()


def channel_of(k, nch):
    from tests.test_gpu_exchange_edges import FNV, MULHI, hash_key, reduce_channel
    return reduce_channel(MULHI, hash_key(FNV, [bytes([k])]), nch)


def channel_counts(n, nch):
    out = np.zeros(nch, np.int64)
    for k in range(M):
        out[channel_of(k, nch)] += residue_count(n, M, k)
    return out


# =============================================================================================
# GPU helpers
# =============================================================================================
# ctx.device_bytes measured at the end of each case on an H100 80GB HBM3 (700 W): the library's own device memory.  Each
# case asks for this, plus the buffers it allocates itself and 1 GB of slack, beside the shared 4 GB column.
PEAK = {
    "scan sparse": 2_568_691_200,          # 2.4 GB: filter scratch + the n-byte selection of sr_scan_evaluate
    "scan dense": 4_949_147_392,           # 4.6 GB: 4.27 G survivors + the tile masks
    "dense aggregate": 17_152,
    "selective push": 10_862_129_408,      # 10.1 GB: the flags n, the prefix sums 4n, the streamed rows
    "smallint direct": 17_230_206_720,     # 16.0 GB: the two-pass direct push keeps an 8-byte slot per row
    "join probe": 9_307_978_496,           # 8.7 GB: heads 4n + the pairs
    "join pairs": 17_181_183_232,          # 16.0 GB: 8 bytes per output pair
    "exchange": 19_864_619_520,            # 18.5 GB: channel ids 4n, row index 4n, the output column n, tile counts
    "rle page": 1_280,
    "bitshuffle": 68_158_720,              # 65 MB: the staged pages and one 32-byte descriptor per 8 KB block
    "fragment cascade": 16_128,
    "fragment passes": 17_205_839_104,     # 16.0 GB: 8-byte selection entries
    "fragment chunk list": 19_356_468_992,  # 18.0 GB: the gathered batch + the passes
}


def need(nbytes, what):
    """skip unless the device has nbytes free (and 1 GB to spare)"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + GB:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB of device memory; {free / GB:.1f} GB are free")


def report(ctx, what):
    print(f"[row limits] {what}: ctx.device_bytes = {ctx.device_bytes} ({ctx.device_bytes / GB:.2f} GB)")


def release():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


_DT = {"i1": ("|i1", "int8"), "u1": ("|u1", "uint8"), "i4": ("<i4", "int32"), "i8": ("<i8", "int64")}


def dev_view(ptr, n, kind):
    """a zero-copy torch view of n device elements at ptr"""
    import torch

    class _View:
        pass
    v = _View()
    v.__cuda_array_interface__ = {"shape": (n,), "typestr": _DT[kind][0], "data": (int(ptr), False), "version": 2}
    t = torch.as_tensor(v, device="cuda")
    assert t.dtype == getattr(torch, _DT[kind][1])
    return t


def compare(got, expected_of, lo=0, hi=None, what=""):
    """got[o] == expected_of(o) for o in [lo, hi), chunk by chunk: expected_of maps an int64 tensor of positions to values"""
    import torch
    hi = got.numel() if hi is None else hi
    first, wrong = None, 0
    for a in range(lo, hi, STEP):
        b = min(a + STEP, hi)
        o = torch.arange(a, b, dtype=torch.int64, device="cuda")
        want = expected_of(o)
        g = got[a:b].to(torch.int64)
        bad = (g != want).nonzero()
        wrong += bad.numel()
        if bad.numel() and first is None:
            i = int(bad[0])
            first = (a + i, int(g[i]), int(want[i]), got[max(a + i - 8, 0):a + i + 24].tolist())
    if wrong:
        raise AssertionError(f"{what}: {wrong} positions differ; the first, {first[0]}: got {first[1]}, want {first[2]}; from 8 before: {first[3]}")


def filled(n, byte=0xA5):
    """n device bytes of `byte`, complete before the library's stream touches them"""
    import torch
    t = torch.full((n,), byte, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    return t


def tinyint_of(k):
    """torch: the TINYINT value of residues k (int64 tensor)"""
    import torch
    return torch.where(k >= 128, k - 256, k)


@pytest.fixture(autouse=True)
def _device(request):
    """the GPU cases skip on a machine without a CUDA device; the CPU checks above run everywhere"""
    if request.node.get_closest_marker("gpu"):
        import torch
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")


@pytest.fixture(scope="module")
def col():
    """the shared device column: REFUSED bytes, byte r = r % 251"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    free, _ = torch.cuda.mem_get_info()
    if free < REFUSED + 8 * GB:
        pytest.skip(f"the shared 4 GB column and its cases need more than {free / GB:.1f} GB free")
    t = torch.empty(REFUSED, dtype=torch.uint8, device="cuda")
    for a in range(0, REFUSED, STEP):
        b = min(a + STEP, REFUSED)
        t[a:b] = (torch.arange(a, b, dtype=torch.int64, device="cuda") % M).to(torch.uint8)
    torch.cuda.synchronize()
    yield t
    del t
    release()


def col_chunk(col, n, offset=0, slot=1, typ=TINYINT):
    return Chunk([(slot, col.data_ptr() + offset, None, typ)], num_rows=n, mem=DEV)


def gpu_error(ctx):
    from starrocks_b200.gpu import lib
    return lib().sr_last_error(ctx.h)


# =============================================================================================
# scan
# =============================================================================================
@pytest.mark.gpu
def test_scan_sparse_survivors_past_2_31(gpu, ctx, col):
    """v BETWEEN 0 AND 9 over 2^31 + 65 rows: the last row and every 251-row period past 2^31 survive"""
    import torch
    n = N31
    need(PEAK["scan sparse"] + n, "scan sparse")
    L = gpu.lib()
    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_BETWEEN, 0, 9)], out_slots=[1]))
    try:
        out = scan.filter(col_chunk(col, n))
        ctx.sync()
        want = sum(residue_count(n, M, k) for k in range(10))
        assert out.num_rows == want
        compare(dev_view(out.cols[0].data, want, "i1"), lambda o: o % 10, what="scan sparse survivors")
        report(ctx, "scan filter, 2^31 + 65 rows, 10 of 251 survive")
        sel = filled(n + 16)
        whole = col_chunk(col, n)
        assert L.sr_scan_evaluate(scan.h, whole.ref(), sel.data_ptr(), DEV) == 0, gpu_error(ctx)
        ctx.sync()
        compare(sel, lambda r: (r % M <= 9).long(), 0, n, what="scan selection bytes")
        assert (sel[n:] == 0xA5).all()
        report(ctx, "scan filter + evaluate, 2^31 + 65 rows")
        del sel
    finally:
        scan.close()
        release()


@pytest.mark.gpu
def test_scan_dense_output_past_2_31(gpu, ctx, col):
    """v != 5 over 0xFFFFFFEF rows: more than 2^31 survivors, output positions past 2^31"""
    n = NMAX
    need(PEAK["scan dense"], "scan dense")
    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_NE, 5)], out_slots=[1]))
    try:
        out = scan.filter(col_chunk(col, n))
        ctx.sync()
        want = n - residue_count(n, M, 5)
        assert want > 1 << 31 and out.num_rows == want
        got = dev_view(out.cols[0].data, want, "i1")

        def expected(o):
            j = o % 250
            return tinyint_of(j + (j >= 5).long())
        compare(got, expected, what="scan dense survivors")
        report(ctx, "scan filter, 0xFFFFFFEF rows, 250 of 251 survive")
    finally:
        scan.close()
        release()


# =============================================================================================
# aggregate
# =============================================================================================
@pytest.mark.gpu
def test_agg_dense_tinyint_key_twice_past_2_32(gpu, ctx, col):
    """GROUP BY a range-declared TINYINT key: COUNT(*), SUM, MIN, MAX of w = (r >> 25) - 64 (negative before 2^31, not
    after) from one push of 0xFFFFFFEF rows, then the same columns again; beside it one scalar aggregate whose COUNT(*)
    passes 2^32"""
    import torch
    from starrocks_b200.gpu import chunk_out_to_host
    n = NMAX
    need(PEAK["dense aggregate"] + n, "dense aggregate")
    w = torch.empty(n, dtype=torch.int8, device="cuda")
    for a in range(0, n, STEP):
        b = min(a + STEP, n)
        w[a:b] = ((torch.arange(a, b, dtype=torch.int64, device="cuda") >> 25) - 64).to(torch.int8)
    torch.cuda.synchronize()                                    # torch fills on its own stream; the library on the context's
    fns = [(abi.AGG_COUNT_STAR, 0, 10, None), (abi.AGG_SUM, TINYINT, 11, [("col", 2)]), (abi.AGG_MIN, TINYINT, 12, [("col", 2)]),
           (abi.AGG_MAX, TINYINT, 13, [("col", 2)])]
    keyed = gpu.Agg(ctx, abi.make_agg_desc([1], [TINYINT], fns, ranges=[(-128, 127)]))
    scalar = gpu.Agg(ctx, abi.make_agg_desc(fns=fns[:2]))
    chunk = Chunk([(1, col.data_ptr(), None, TINYINT), (2, w.data_ptr(), None, TINYINT)], num_rows=n, mem=DEV)
    try:
        for _ in range(2):
            keyed.push(chunk)
            scalar.push(chunk)
        ctx.sync()
        report(ctx, "dense aggregate + scalar aggregate, 2 x 0xFFFFFFEF rows")
        keyed.finish()
        got = {s: d for s, _, d, _ in chunk_out_to_host(ctx, keyed.pull())}
        rows = sorted(zip(got[1].tolist(), got[10].tolist(), got[11].tolist(), got[12].tolist(), got[13].tolist()))
        want = sorted((tinyint(k), 2 * residue_count(n, M, k), 2 * shifted_sum(n, M, k, 25, 64), -64,
                       (last_with_residue(n, M, k) >> 25) - 64) for k in range(M))
        assert rows == want
        scalar.finish()
        got = {s: d for s, _, d, _ in chunk_out_to_host(ctx, scalar.pull())}
        assert (int(got[10][0]), int(got[11][0])) == (2 * n, 2 * sum(shifted_sum(n, M, k, 25, 64) for k in range(M)))
        assert 2 * n > 1 << 32
    finally:
        scalar.close()
        keyed.close()
        del w
        release()


@pytest.mark.gpu
def test_agg_push_selective_limit(gpu, ctx, col):
    """a keyed hash aggregate's selective push of 0x7FFFFFF0 rows is refused before it allocates or launches anything,
    and the handle stays usable"""
    from starrocks_b200.gpu import chunk_out_to_host
    L = gpu.lib()
    first, _ = abi.two_phase_descs(abi.make_agg_desc([1], [TINYINT], [(abi.AGG_COUNT_STAR, 0, 10, None)]))
    agg = gpu.Agg(ctx, first)
    small = Chunk([(1, (np.arange(300) % M).astype(np.uint8).view(np.int8), None)])
    try:
        agg.push(Chunk([(1, np.arange(100, dtype=np.int8), None)]))         # groups 0..99 exist
        o = agg.push_selective(small)                                       # compiles; streams the other groups' rows
        assert o.num_rows == int(((np.arange(300) % M) >= 100).sum())
        out = abi.sr_chunk_out()
        launches, nbytes = ctx.launches, ctx.device_bytes
        over = col_chunk(col, SEL_LIMIT)
        rc = L.sr_agg_push_selective(agg.h, over.ref(), C.byref(out))
        assert rc == abi.SR_ERR_NOT_SUPPORTED, (rc, gpu_error(ctx))
        assert (ctx.launches, ctx.device_bytes) == (launches, nbytes)
        o = agg.push_selective(small)
        assert o.num_rows == int(((np.arange(300) % M) >= 100).sum())
        agg.finish()
        res = {s: d for s, _, d, _ in chunk_out_to_host(ctx, agg.pull())}
        counts = dict(zip(res[1].tolist(), res[10].tolist()))
        assert counts == {k: 1 + 2 * int(((np.arange(300) % M) == k).sum()) for k in range(100)}
    finally:
        agg.close()


@pytest.mark.gpu
def test_agg_push_selective_accepted_below_limit(gpu, ctx, col):
    """a keyed selective push of 0x7FFFFFEF rows (the largest accepted) into a GROUP BY table holding every residue but 5
    and 250: exactly their rows stream out, in input order, and no group is created"""
    from starrocks_b200.gpu import chunk_out_to_host
    n = SEL_LIMIT - 1
    need(PEAK["selective push"], "selective push")
    missing = [5, 250]
    agg = gpu.Agg(ctx, abi.make_agg_desc([1], [TINYINT], []))
    try:
        agg.push(Chunk([(1, np.array([tinyint(k) for k in range(M) if k not in missing], np.int8), None)]))
        out = agg.push_selective(col_chunk(col, n))
        ctx.sync()
        report(ctx, "selective push, 0x7FFFFFEF rows")
        want = sum(residue_count(n, M, k) for k in missing)
        assert out.num_rows == want and out.num_cols == 1
        compare(dev_view(out.cols[0].data, want, "i1"), lambda o: tinyint_of(nth_with_residue(o, missing, M) % M), what="streamed keys")
        agg.finish()
        keys = {s: d for s, _, d, _ in chunk_out_to_host(ctx, agg.pull())}[1]
        assert sorted(keys.tolist()) == sorted(tinyint(k) for k in range(M) if k not in missing)
    finally:
        agg.close()
        release()


@pytest.mark.gpu
def test_agg_smallint_hash_key_direct_push(gpu, ctx, col, monkeypatch):
    """GROUP BY a SMALLINT hash key (r % 4099) - 2049 over 2^31 + 65 rows in one push through the direct (unpartitioned)
    hash push: COUNT(*) and SUM of the TINYINT column"""
    import torch
    from starrocks_b200.gpu import chunk_out_to_host
    n = N31
    need(PEAK["smallint direct"] + 2 * n, "SMALLINT hash aggregate")
    monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", str(1 << 40))     # the library's knob: no partitioned push
    key = torch.empty(n, dtype=torch.int16, device="cuda")
    for a in range(0, n, STEP):
        b = min(a + STEP, n)
        key[a:b] = (torch.arange(a, b, dtype=torch.int64, device="cuda") % KM - 2049).to(torch.int16)
    torch.cuda.synchronize()
    agg = gpu.Agg(ctx, abi.make_agg_desc([3], [abi.TYPE_SMALLINT], [(abi.AGG_COUNT_STAR, 0, 10, None), (abi.AGG_SUM, TINYINT, 11, [("col", 1)])]))
    try:
        agg.push(Chunk([(1, col.data_ptr(), None, TINYINT), (3, key.data_ptr(), None, abi.TYPE_SMALLINT)], num_rows=n, mem=DEV))
        ctx.sync()
        report(ctx, "SMALLINT hash aggregate, direct push, 2^31 + 65 rows")
        agg.finish()
        got = {s: d for s, _, d, _ in chunk_out_to_host(ctx, agg.pull())}
        assert dict(zip(got[3].tolist(), zip(got[10].tolist(), got[11].tolist()))) == smallint_groups(n)
    finally:
        agg.close()
        del key
        release()


# =============================================================================================
# join
# =============================================================================================
def _probe_last_chunk(gpu, ctx, join, total, tail=1 << 20):
    """(first position, probe_index, build_index) of the last `tail` output pairs, as int64 host arrays"""
    from starrocks_b200.gpu import _copy_dev_to_host
    pi, bi = C.c_void_p(), C.c_void_p()
    ctx.check(gpu.lib().sr_join_probe_indexes(join.h, 0, C.byref(pi), C.byref(bi)))
    ctx.sync()
    lo = max(0, total - tail)
    p = _copy_dev_to_host(ctx, pi.value + 4 * lo, 4 * (total - lo)).view(np.uint32).astype(np.int64)
    b = _copy_dev_to_host(ctx, bi.value + 4 * lo, 4 * (total - lo)).view(np.uint32).astype(np.int64)
    return lo, p, b, pi.value, bi.value


@pytest.mark.gpu
@pytest.mark.parametrize("jt", [abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI], ids=["inner", "left_semi", "left_anti"])
def test_join_probe_batch_past_2_31(gpu, ctx, col, jt):
    """2^31 + 65 probe rows of the 1-byte key against a small build: the rows with residue 0..9 come out, the last one
    past 2^31 included"""
    n = N31
    need(PEAK["join probe"], "join probe")
    matched = list(range(10))
    build_keys = matched if jt != abi.JOIN_LEFT_ANTI else list(range(10, M))
    join = gpu.Join(ctx, abi.make_join_desc(jt, [1], [1], [TINYINT]))
    try:
        join.append_build(Chunk([(1, np.array([tinyint(k) for k in build_keys], np.int8), None)]))
        join.build_finish()
        out = join.probe(col_chunk(col, n))
        ctx.sync()
        total = sum(residue_count(n, M, k) for k in matched)
        assert out.num_rows == total
        report(ctx, f"join probe {jt}, 2^31 + 65 rows")
        lo, p, b, _, _ = _probe_last_chunk(gpu, ctx, join, total)
        o = np.arange(lo, total)
        assert np.array_equal(p, (o // 10) * M + o % 10)
        assert p[-1] == n - 1 and p[0] < 1 << 31 < p[-1]
        assert np.array_equal(b, o % 10 + 1 if jt == abi.JOIN_INNER else np.zeros_like(o))
    finally:
        join.close()
        release()


@pytest.mark.gpu
def test_join_output_of_2_32_pairs_refused(gpu, ctx):
    """B build rows and P probe rows of one key with B * P = 2^32 + 65536: refused, never wrapped to 65536 pairs"""
    L = gpu.lib()
    B, P = 1 << 16, (1 << 16) + 1
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT]))
    try:
        join.append_build(Chunk([(1, np.zeros(B, np.int32), None)]))
        join.build_finish()
        out = abi.sr_chunk_out()
        probe = Chunk([(1, np.zeros(P, np.int32), None)])                # kept alive through the call
        rc = L.sr_join_probe(join.h, 0, probe.ref(), C.byref(out))
        assert rc == abi.SR_ERR_NOT_SUPPORTED and b"2^32" in gpu_error(ctx), (rc, gpu_error(ctx))
        assert out.num_rows == 0
        o = join.probe(Chunk([(1, np.zeros(3, np.int32), None)]))            # the handle still probes
        assert o.num_rows == 3 * B
    finally:
        join.close()
    # 4096 build rows, 2^24 + 1 probe rows: every 1024 probe blocks of 1024 rows sum to exactly 2^32 pairs -- the block
    # sums of the scan over the probe blocks must saturate, or 2^36 + 4096 pairs wrap to 4096
    B, P = 1 << 12, (1 << 24) + 1
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT]))
    try:
        join.append_build(Chunk([(1, np.zeros(B, np.int32), None)]))
        join.build_finish()
        out = abi.sr_chunk_out()
        probe = Chunk([(1, np.zeros(P, np.int32), None)])                # kept alive through the call
        rc = L.sr_join_probe(join.h, 0, probe.ref(), C.byref(out))
        assert rc == abi.SR_ERR_NOT_SUPPORTED and b"2^32" in gpu_error(ctx), (rc, gpu_error(ctx))
        assert out.num_rows == 0
    finally:
        join.close()


@pytest.mark.gpu
def test_join_output_past_2_31_pairs(gpu, ctx):
    """B = 2^15 build rows, P = 2^16 + 1 probe rows of one key: 2^31 + 2^15 pairs, output positions past 2^31"""
    B, P = 1 << 15, (1 << 16) + 1
    total = B * P
    need(PEAK["join pairs"], "join output past 2^31")
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT]))
    try:
        join.append_build(Chunk([(1, np.zeros(B, np.int32), None)]))
        join.build_finish()
        out = join.probe(Chunk([(1, np.zeros(P, np.int32), None)]))
        ctx.sync()
        assert out.num_rows == total
        report(ctx, "join probe, 2^31 + 2^15 output pairs")
        lo, p, b, _, bi = _probe_last_chunk(gpu, ctx, join, total, tail=4 * B)
        assert np.array_equal(p, np.arange(lo, total) // B)
        from starrocks_b200.gpu import _copy_dev_to_host
        chain = _copy_dev_to_host(ctx, bi, 4 * B).view(np.uint32).astype(np.int64)   # probe row 0's pairs
        assert np.array_equal(np.sort(chain), np.arange(1, B + 1))
        assert np.array_equal(b, np.tile(chain, 4))                          # every probe row walks the same chain
    finally:
        join.close()
        release()


# =============================================================================================
# exchange
# =============================================================================================
@pytest.mark.gpu
def test_xchg_partition_past_2_31(gpu, ctx, col):
    """2^31 + 65 rows of the 1-byte key into 16 channels: each channel holds exactly the rows of its residues, in input
    order, the channels after the first starting past 2^31 where the counts put them"""
    n, nch = N31, 16
    need(PEAK["exchange"], "exchange partition")
    x = gpu.Xchg(ctx, abi.make_part_desc([1], nch))
    try:
        out, offs = x.partition(col_chunk(col, n))
        ctx.sync()
        report(ctx, "exchange partition, 2^31 + 65 rows, 16 channels")
        counts = channel_counts(n, nch)
        assert offs.tolist() == [0] + np.cumsum(counts).tolist()
        assert out.num_rows == n
        got = dev_view(out.cols[0].data, n, "u1")
        for c in range(nch):
            s = sorted(k for k in range(M) if channel_of(k, nch) == c)
            if not s:
                continue
            a, b = int(offs[c]), int(offs[c + 1])
            for lo, hi in ((a, min(b, a + STEP)), (max(a, b - STEP), b)):      # the head and the tail of every channel
                compare(got, lambda o: nth_with_residue(o - a, s, M) % M, lo, hi, what=f"channel {c}")
    finally:
        x.close()
        release()


# =============================================================================================
# pages
# =============================================================================================
@pytest.mark.gpu
def test_rle_bool_page_of_2_32_minus_1_values(gpu, ctx):
    """one RLE BOOLEAN page whose value count is 0xFFFFFFFF, from 21 bytes of runs: a run of 2^31 + 1 ones, a literal
    group, zeros, a final one; the 16 sentinel bytes past the column stay untouched"""
    import torch
    n = 0xFFFFFFFF
    need(PEAK["rle page"] + n, "RLE page")
    head, lit = (1 << 31) + 1, 0x4D
    page = np.concatenate([np.array([n], "<u4").view(np.uint8), rle_runs_bytes(big_bool_runs(n, head, lit))])
    assert len(page) < 32
    out = filled(n + 16)
    dec = gpu.PageDecoder(ctx)
    try:
        assert dec.decode(abi.PAGE_RLE, BOOLEAN, [page], out.data_ptr(), n) == n
        ctx.sync()
        report(ctx, "RLE BOOLEAN page, 0xFFFFFFFF values")
        compare(out, lambda r: big_bool_expected(r, n, head, lit), 0, n, what="RLE page")
        assert (out[n:] == 0xA5).all()
        assert int(out[:n].sum(dtype=torch.int64)) == big_bool_ones(n, head, lit)
    finally:
        dec.close()
        del out
        release()


@pytest.mark.gpu
def test_rle_null_maps_with_a_page_past_2_32(gpu, ctx):
    """RLE null maps of UINT32_MAX, 7 and 9 rows in one call: the third map's first row is 2^32 + 6"""
    import torch
    big = 0xFFFFFFFF
    head, lit = (1 << 31) + 3, 0xB2
    maps = [(rle_runs_bytes(big_bool_runs(big, head, lit)), big), (rle_runs_bytes([("lit", [0x55])]), 7),
            (rle_runs_bytes([("rep", 9, 1)]), 9)]
    n = big + 16
    need(PEAK["rle page"] + n, "RLE null maps")
    out = filled(n + 16)
    dec = gpu.PageDecoder(ctx)
    try:
        rows, nulls = dec.decode_nulls(abi.NULL_RLE, maps, out.data_ptr(), n)
        ctx.sync()
        report(ctx, "RLE null maps, UINT32_MAX + 16 rows")
        assert rows == n and nulls == big_bool_ones(big, head, lit) + 4 + 9

        def expected(r):
            return torch.where(r < big, big_bool_expected(r, big, head, lit),
                               torch.where(r < big + 7, (torch.full_like(r, 0x55) >> (r - big).clamp(0, 7)) & 1, 1))
        compare(out, expected, 0, n, what="null maps")
        assert (out[n:] == 0xA5).all()
    finally:
        dec.close()
        del out
        release()


@pytest.mark.gpu
def test_bitshuffle_pages_with_a_page_past_2_32(gpu, ctx):
    """BIT_SHUFFLE data pages of 2^32 - 8, 16 and 24 one-byte values in one call (the third starts at row 2^32 + 8): the
    first page is 524 288 blocks, its last one of 8184 values"""
    import torch
    bo = pytest.importorskip("bshuf_oracle")
    bo.lib()
    big = (1 << 32) - 8
    rng = np.random.default_rng(41)
    smalls = [rng.integers(0, 256, k).astype(np.uint8) for k in (16, 24)]
    pages = [big_bshuf_page(bo, big)] + [bo.bitshuffle_encode(v) for v in smalls]
    n = big + 40
    need(PEAK["bitshuffle"] + n, "bitshuffle pages")
    out = filled(n + 16)
    dec = gpu.PageDecoder(ctx)
    try:
        assert dec.decode(abi.PAGE_BITSHUFFLE, TINYINT, pages, out.data_ptr(), n) == n
        ctx.sync()
        report(ctx, "BIT_SHUFFLE pages, 2^32 + 32 values")
        compare(out, lambda r: (r & 0xFF) ^ 0x5A, 0, big, what="bitshuffle page")
        assert np.array_equal(out[big:].cpu().numpy(), np.concatenate(smalls + [np.full(16, 0xA5, np.uint8)]))
    finally:
        dec.close()
        del out
        release()


@pytest.mark.gpu
def test_bitshuffle_null_maps_with_a_page_past_2_32(gpu, ctx):
    """bitshuffle null maps of UINT32_MAX, 7 and 9 rows in one call: the third map's first row is 2^32 + 6"""
    import torch
    bo = pytest.importorskip("bshuf_oracle")
    bo.lib()
    big = 0xFFFFFFFF
    smalls = [np.array([1, 0, 1, 1, 0, 0, 1], np.uint8), np.array([0, 1, 0, 0, 0, 0, 0, 1, 1], np.uint8)]
    maps = [(big_bshuf_null_map(bo, big), big)] + [(bo.null_map_encode(f, abi.NULL_BITSHUFFLE), len(f)) for f in smalls]
    n = big + 16
    need(PEAK["bitshuffle"] + n, "bitshuffle null maps")
    out = filled(n + 16)
    dec = gpu.PageDecoder(ctx)
    try:
        rows, nulls = dec.decode_nulls(abi.NULL_BITSHUFFLE, maps, out.data_ptr(), n)
        ctx.sync()
        report(ctx, "bitshuffle null maps, UINT32_MAX + 16 rows")
        assert rows == n and nulls == len(NULL_BYTES) * (1 << 24) + sum(int(f.sum()) for f in smalls)
        lut = torch.tensor(np.isin(np.arange(256), NULL_BYTES).astype(np.int64), device="cuda")
        compare(out, lambda r: lut[r & 0xFF], 0, big, what="bitshuffle null map")
        assert np.array_equal(out[big:].cpu().numpy(), np.concatenate(smalls + [np.full(16, 0xA5, np.uint8)]))
    finally:
        dec.close()
        del out
        release()


# =============================================================================================
# fused fragment
# =============================================================================================
def _dim(gpu, ctx, keys):
    """a range-direct-mapped dimension: the TINYINT key of each residue k in keys, payload slot 2 = k % 7"""
    dim = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [TINYINT], build_out=[2]))
    dim.append_build(Chunk([(1, np.array([tinyint(k) for k in keys], np.int8), None), (2, np.array([k % 7 for k in keys], np.int32), None)]))
    dim.build_finish()
    return dim


DIM_KEYS = list(range(0, 50)) + [250]                    # residue 250 (TINYINT -6) is the last of each period


def _frag_want(n):
    want = {}
    for k in DIM_KEYS:
        c, s = want.get(k % 7, (0, 0))
        want[k % 7] = (c + residue_count(n, M, k), s + tinyint(k) * residue_count(n, M, k))
    return sorted((g, c, s) for g, (c, s) in want.items())


def _frag_passed(n):
    """the fact rows that survive the join"""
    return sum(residue_count(n, M, k) for k in DIM_KEYS)


def _frag_result(ctx, frag):
    from starrocks_b200.gpu import chunk_out_to_host
    frag.agg.finish()
    got = {s: d for s, _, d, _ in chunk_out_to_host(ctx, frag.agg.pull())}
    return sorted(zip(got[2].tolist(), got[10].tolist(), got[11].tolist()))


FRAG_AGG = dict(group_slots=[2], group_types=[INT], ranges=[(0, 6)],
                fns=[(abi.AGG_COUNT_STAR, 0, 10, None), (abi.AGG_SUM, TINYINT, 11, [("col", 1)])])


@pytest.mark.gpu
@pytest.mark.parametrize("mode,n", [(1, N31), (2, N31), (1, NMAX)], ids=["cascade-2^31+65", "passes-2^31+65", "cascade-0xFFFFFFEF"])
def test_fragment_join_group_past_2_31(gpu, ctx, col, mode, n):
    """fact key (1 byte) JOIN a 51-key dimension GROUP BY its payload: COUNT(*), SUM(fact key); survivors up to the last
    row, whose ids pass 2^31"""
    need(PEAK["fragment cascade" if mode == 1 else "fragment passes"], "fragment")
    dim = _dim(gpu, ctx, DIM_KEYS)
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [2])], abi.make_agg_desc(**FRAG_AGG), mode=mode)
    try:
        frag.push(col_chunk(col, n))
        ctx.sync()
        report(ctx, f"fragment mode {mode}, {n} rows, plan {frag.plan()['mode']}")
        assert frag.rows_passed == _frag_passed(n)
        assert _frag_result(ctx, frag) == _frag_want(n)
    finally:
        frag.close()
        dim.close()
        release()


@pytest.mark.gpu
def test_fragment_push_chunks_past_2_31(gpu, ctx, col):
    """a list of three device chunks, 2^31 + 65 rows in all, gathered into one batch: the same answer as one chunk"""
    n = N31
    need(PEAK["fragment chunk list"], "fragment chunk list")
    cuts = [0, (1 << 30) + 7, (1 << 31) - 3, n]
    dim = _dim(gpu, ctx, DIM_KEYS)
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [2])], abi.make_agg_desc(**FRAG_AGG), mode=2)
    try:
        frag.push_chunks([col_chunk(col, b - a, offset=a) for a, b in zip(cuts, cuts[1:])])
        ctx.sync()
        report(ctx, "fragment push_chunks, 2^31 + 65 rows in 3 chunks")
        assert frag.rows_passed == _frag_passed(n)
        assert _frag_result(ctx, frag) == _frag_want(n)
    finally:
        frag.close()
        dim.close()
        release()


# =============================================================================================
# refusals at the documented limits
# =============================================================================================
def refused(ctx, call, code=abi.SR_ERR_NOT_SUPPORTED):
    launches, nbytes = ctx.launches, ctx.device_bytes
    rc = call()
    assert rc == code, (rc, gpu_error(ctx))
    assert (ctx.launches, ctx.device_bytes) == (launches, nbytes)


SMALL = np.arange(-50, 50, dtype=np.int8)                 # a good 100-row TINYINT batch


@pytest.mark.gpu
def test_refuse_fragment_push_and_chunk_list(gpu, ctx, col):
    """0xFFFFFFF0 fact rows, in one chunk and in a list of two, then a good push"""
    L = gpu.lib()
    dim = _dim(gpu, ctx, DIM_KEYS)
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [2])], abi.make_agg_desc(**FRAG_AGG))
    try:
        frag.push(col_chunk(col, 1000))
        over = col_chunk(col, REFUSED)
        refused(ctx, lambda: L.sr_fragment_push(frag.h, over.ref()))
        half = REFUSED // 2
        pieces = [col_chunk(col, half), col_chunk(col, REFUSED - half, offset=half)]
        views = (abi.sr_chunk_view * 2)(*[c.view for c in pieces])
        refused(ctx, lambda: L.sr_fragment_push_chunks(frag.h, views, 2))
        frag.push(col_chunk(col, 1000))
        assert frag.rows_passed == 2 * _frag_passed(1000)
    finally:
        frag.close()
        dim.close()


@pytest.mark.gpu
def test_refuse_join_probe_batch(gpu, ctx, col):
    """0xFFFFFFF0 probe rows, then a good probe"""
    L = gpu.lib()
    out = abi.sr_chunk_out()
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [TINYINT]))
    try:
        join.append_build(Chunk([(1, SMALL, None)]))
        join.build_finish()
        over = col_chunk(col, REFUSED)
        refused(ctx, lambda: L.sr_join_probe(join.h, 0, over.ref(), C.byref(out)))
        assert join.probe(Chunk([(1, SMALL, None)])).num_rows == 100
    finally:
        join.close()


@pytest.mark.gpu
def test_refuse_join_build_side(gpu, ctx, col):
    """0xFFFFFFF0 build rows are appended (a 4 GB copy) and refused by build_finish"""
    L = gpu.lib()
    need(REFUSED, "build-side refusal")
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [TINYINT]))
    try:
        join.append_build(col_chunk(col, REFUSED))
        refused(ctx, lambda: L.sr_join_build_finish(join.h))
    finally:
        join.close()
        release()


@pytest.mark.gpu
def test_refuse_xchg_partition(gpu, ctx, col):
    """0xFFFFFFF0 rows into the hash partition, then a good one"""
    L = gpu.lib()
    out = abi.sr_chunk_out()
    x = gpu.Xchg(ctx, abi.make_part_desc([1], 16))
    offs = np.zeros(17, np.int64)
    try:
        x.partition(Chunk([(1, SMALL, None)]))
        over = col_chunk(col, REFUSED)
        refused(ctx, lambda: L.sr_xchg_partition(x.h, over.ref(), C.byref(out), offs.ctypes.data))
        _, o = x.partition(Chunk([(1, SMALL, None)]))
        assert o[-1] == 100
    finally:
        x.close()


@pytest.mark.gpu
def test_refuse_null_map_rows(gpu, ctx):
    """a null map of UINT32_MAX + 1 rows (its stream holds them; so does the output column), then a good map"""
    L = gpu.lib()
    need((1 << 32) + 16, "null map refusal")
    dst = filled((1 << 32) + 16)
    dec = gpu.PageDecoder(ctx)
    try:
        s = rle_runs_bytes([("rep", 1 << 32, 1)])
        views = (abi.sr_null_map_view * 1)()
        views[0].data, views[0].size, views[0].num_rows = s.ctypes.data, len(s), 1 << 32
        rows, nulls = C.c_int64(0), C.c_int64(0)
        refused(ctx, lambda: L.sr_null_maps_decode(dec.h, abi.NULL_RLE, views, 1, abi.MEM_HOST, dst.data_ptr(), (1 << 32) + 16,
                                                   C.byref(rows), C.byref(nulls)), abi.SR_ERR_INVALID_ARGUMENT)
        assert dec.decode_nulls(abi.NULL_RLE, [(rle_runs_bytes([("rep", 5, 1)]), 5)], dst.data_ptr(), 5) == (5, 5)
    finally:
        dec.close()
        del dst
        release()


@pytest.mark.gpu
def test_refuse_chunk_pb_column_of_2_32_bytes(gpu, ctx):
    """ChunkPB stores a column's byte size as uint32: a SMALLINT column of 2^31 rows (2^32 bytes) is refused, one row fewer
    is sized exactly"""
    import torch
    from starrocks_b200.abi import TYPE_SMALLINT
    L = gpu.lib()
    need(1 << 32, "ChunkPB refusal")
    big = torch.zeros(1 << 31, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    chunk = Chunk([(1, big.data_ptr(), None, TYPE_SMALLINT)], num_rows=1 << 31, mem=DEV)
    dst = np.zeros(64, np.uint8)
    meta = abi.sr_chunk_pb_meta()
    try:
        refused(ctx, lambda: L.sr_chunk_serialize(ctx.h, chunk.ref(), 0, 1 << 31, dst.ctypes.data, len(dst), abi.MEM_HOST, C.byref(meta)))
        assert L.sr_chunk_serialized_size(chunk.ref(), 0, (1 << 31) - 1) == 8 + 4 + ((1 << 32) - 2)
        payload, m = gpu.chunk_serialize(ctx, chunk, 0, 5)               # the handle's context still serialises
        assert m.num_rows == 5 and payload.tobytes() == np.array([1, 5, 10], "<u4").tobytes() + bytes(10)
    finally:
        del big
        release()
