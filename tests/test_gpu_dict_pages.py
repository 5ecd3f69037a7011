"""Dictionary-encoded (DICT_ENCODING) data pages decoded on the device by sr_pages_decode(SR_PAGE_DICT) into the ids of
the decoder's table (sr_page_decoder_set_dict): parity against numpy values[codes], several segments with their own
local dictionaries into one column, every malformed page, and SSB Q4.1 with its string columns carried as words."""
import numpy as np
import pytest

from starrocks_b200 import abi, ssb
from starrocks_b200.abi import Chunk

pytestmark = pytest.mark.gpu

SENTINEL = -0x5A5A5A5B


@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


def _pages(bo, codes, page_rows):
    return [bo.dict_page_encode(codes[lo:lo + page_rows]) for lo in range(0, max(len(codes), 1), page_rows)]


def _set_dict(dec, values, mem, keep):
    import torch
    if mem == "host":
        dec.set_dict(values)
    elif mem == "device":
        t = torch.from_numpy(values).cuda()
        keep.append(t)
        dec.set_dict((t.data_ptr(), len(values)), mem=abi.MEM_DEVICE)
    else:
        t = torch.from_numpy(values).pin_memory()
        keep.append(t)
        dec.set_dict((t.data_ptr(), len(values)), mem=abi.MEM_HOST_PINNED)


def _decode(ctx, dec, pages, out, row0, cap, mem):
    """pages -> out[row0:] (a device int32 tensor) from `mem`: host, device at odd byte alignments, pinned back to back
    (staged by DMA) or pinned with gaps (read in place); -> rows"""
    import torch
    keep = []
    dst = out.data_ptr() + 4 * row0
    if mem == "host":
        rows = dec.decode(abi.PAGE_DICT, abi.TYPE_INT, pages, dst, cap)
    elif mem == "device":
        views = []
        for k, pg in enumerate(pages):
            b = torch.from_numpy(np.concatenate([np.zeros(k % 4 + 1, dtype=np.uint8), pg])).cuda()
            keep.append(b)
            views.append((b.data_ptr() + k % 4 + 1, len(pg)))
        rows = dec.decode(abi.PAGE_DICT, abi.TYPE_INT, views, dst, cap, mem=abi.MEM_DEVICE)
    else:
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
        rows = dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [(blob.data_ptr() + o, len(pg)) for o, pg in zip(offs, pages)], dst, cap,
                          mem=abi.MEM_HOST_PINNED)
    ctx.sync()
    return rows


def _column(n, extra=8):
    import torch
    return torch.full((n + extra,), SENTINEL, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("words", [1, 7, 25, 256, 70_000])
@pytest.mark.parametrize("order", ["random", "sorted"])
@pytest.mark.parametrize("page_rows", [1000, 65_536])
@pytest.mark.parametrize("mem", ["host", "device", "pinned_run", "pinned_scattered"])
def test_dict_pages_decode_parity(gpu, ctx, bo, words, order, page_rows, mem):
    rng = np.random.default_rng(words + page_rows)
    n = 100_003
    codes = rng.integers(0, words, n).astype(np.int32)
    if order == "sorted":
        codes.sort()
    values = rng.integers(-2**31, 2**31, words, dtype=np.int64).astype(np.int32)     # any int32 table, not only small ids
    pages = _pages(bo, codes, page_rows)
    dec = gpu.PageDecoder(ctx)
    keep = []
    try:
        _set_dict(dec, values, "host" if mem == "host" else "device" if mem == "device" else "pinned", keep)
        out = _column(n)
        assert _decode(ctx, dec, pages, out, 0, n, mem) == n
        got = out.cpu().numpy()
        assert (got[:n] == values[codes]).all()
        assert (got[n:] == SENTINEL).all()                                           # nothing written past the column
    finally:
        dec.close()


def _first_seen(words):
    """encode_local_dict: the distinct words in first-seen order and one local code per row"""
    local, codes = {}, np.empty(len(words), dtype=np.int32)
    for i, w in enumerate(words):
        codes[i] = local.setdefault(w, len(local))
    return list(local), codes


def _global_ids(local_words, global_dict):
    """GlobalDictCodeConverter::global_ids: the global id of each local word, 0 for an empty word the dictionary lacks"""
    return np.array([global_dict.get(w, 0) for w in local_words], dtype=np.int32)


def _decode_segments(ctx, dec, bo, words, global_dict, bounds, page_rows, mem="host"):
    """a string column written as segments [bounds[k], bounds[k + 1]), each with its own first-seen dictionary, decoded into
    one device column of global ids: one table per segment, `out` advanced by the segment's rows"""
    n = bounds[-1]
    out = _column(n)
    for lo, hi in zip(bounds, bounds[1:]):
        local_words, codes = _first_seen(words[lo:hi])
        dpage = bo.binary_plain_page_encode(local_words)                 # the segment's dictionary page, read back
        dec.set_dict(_global_ids(bo.binary_plain_page_decode(dpage), global_dict))
        assert _decode(ctx, dec, _pages(bo, codes, page_rows), out, lo, n - lo, mem) == hi - lo
    return out


def test_several_segments_into_one_column(gpu, ctx, bo):
    rng = np.random.default_rng(21)
    vocab = [b"AFRICA", b"AMERICA", b"ASIA", b"EUROPE", b"MIDDLE EAST", b""]
    global_dict = {w: i + 1 for i, w in enumerate(sorted(w for w in vocab if w))}
    n = 50_000
    words = [vocab[k] for k in rng.integers(0, 6, n)]
    words[:3000] = [vocab[k] for k in rng.integers(0, 2, 3000)]              # the first segment sees two words only
    bounds = [0, 3000, 17_777, 17_778, n]
    dec = gpu.PageDecoder(ctx)
    try:
        for mem in ("host", "device", "pinned_scattered"):
            out = _decode_segments(ctx, dec, bo, words, global_dict, bounds, 4096, mem)
            got = out.cpu().numpy()
            assert (got[:n] == [global_dict.get(w, 0) for w in words]).all(), mem
            assert (got[n:] == SENTINEL).all()
    finally:
        dec.close()


def _with_word(page, at, x):
    p = page.copy()
    p[at:at + 4] = np.array([x], dtype="<u4").view(np.uint8)
    return p


def test_malformed_pages_then_a_good_call(gpu, ctx, bo):
    rng = np.random.default_rng(22)
    words = 25
    values = np.arange(100, 100 + words, dtype=np.int32)
    codes = rng.integers(0, words, 5000).astype(np.int32)
    good = bo.dict_page_encode(codes)
    with_code = lambda c: bo.dict_page_encode(np.concatenate([codes[:1234], np.array([c], dtype=np.uint32).view(np.int32), codes[1235:]]))
    bad = {"too_short": good[:3], "mode_0": _with_word(good, 0, 0), "mode_6": _with_word(good, 0, 6), "mode_ffffffff": _with_word(good, 0, 0xFFFFFFFF),
           "header_size_mismatch": _with_word(good, 8, len(good)), "header_padded_count": _with_word(good, 12, 5008),
           "elem_size_8": _with_word(good, 16, 8), "chain_overruns_page": np.concatenate([good[:20], np.frombuffer(len(good).to_bytes(4, "big"), dtype=np.uint8), good[24:]]),
           "code_num_words": with_code(words), "code_ffffffff": with_code(0xFFFFFFFF),
           "bad_behind_plain_mode": None}
    plain = bo.dict_page_plain_fallback([b"x", b"yz"])
    out = _column(2 * len(codes))
    dec = gpu.PageDecoder(ctx)
    try:
        dec.set_dict(values)
        for name, page in bad.items():
            pages = [plain, good[:3]] if page is None else [good, page]                 # behind a good page (a plain one: INVALID wins)
            with pytest.raises(gpu.GpuError) as ei:
                dec.decode(abi.PAGE_DICT, abi.TYPE_INT, pages, out.data_ptr(), 2 * len(codes))
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, name
            assert dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [good], out.data_ptr(), len(codes)) == len(codes), name
            ctx.sync()
            assert (out.cpu().numpy()[:len(codes)] == values[codes]).all(), name
    finally:
        dec.close()


def test_plain_mode_no_table_and_other_types(gpu, ctx, bo):
    codes = np.arange(3000, dtype=np.int32) % 5
    good = bo.dict_page_encode(codes)
    plain = bo.dict_page_plain_fallback([b"AMERICA", b"ASIA"])
    out = _column(2 * len(codes))
    dec = gpu.PageDecoder(ctx)
    try:
        with pytest.raises(gpu.GpuError) as ei:                                       # no table yet
            dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [good], out.data_ptr(), len(codes))
        assert ei.value.code == abi.SR_ERR_STATE
        dec.set_dict(np.arange(5, dtype=np.int32) + 1)
        for pages in ([plain], [good, plain]):                                        # the column fell back to plain pages
            with pytest.raises(gpu.GpuError) as ei:
                dec.decode(abi.PAGE_DICT, abi.TYPE_INT, pages, out.data_ptr(), 2 * len(codes))
            assert ei.value.code == abi.SR_ERR_NOT_SUPPORTED
        for typ in (abi.TYPE_BIGINT, abi.TYPE_DATE, abi.TYPE_SMALLINT):                # ids are TYPE_INT
            with pytest.raises(gpu.GpuError) as ei:
                dec.decode(abi.PAGE_DICT, typ, [good], out.data_ptr(), len(codes))
            assert ei.value.code == abi.SR_ERR_NOT_SUPPORTED
        with pytest.raises(gpu.GpuError) as ei:                                       # out must be 4-byte aligned
            dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [good], out.data_ptr() + 2, len(codes))
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
        assert dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [good], out.data_ptr(), len(codes)) == len(codes)
        ctx.sync()
        assert (out.cpu().numpy()[:len(codes)] == codes + 1).all()
        dec.set_dict(np.zeros(0, dtype=np.int32))                                     # an empty table: every code is out of range
        with pytest.raises(gpu.GpuError) as ei:
            dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [good], out.data_ptr(), len(codes))
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
        assert dec.decode(abi.PAGE_DICT, abi.TYPE_INT, [bo.dict_page_encode(np.zeros(0, dtype=np.int32))], out.data_ptr(), 0) == 0
    finally:
        dec.close()


def test_other_encodings_unchanged_after_set_dict(gpu, ctx, bo, oracle):
    import torch
    v = np.random.default_rng(23).integers(-10**6, 10**6, 70_001).astype(np.int32)
    pages = {abi.PAGE_BITSHUFFLE: [bo.bitshuffle_encode(v[lo:lo + 8192]) for lo in range(0, len(v), 8192)],
             abi.PAGE_FOR: [oracle.for_encode(v[lo:lo + 8192]) for lo in range(0, len(v), 8192)]}
    dec = gpu.PageDecoder(ctx)
    try:
        for enc, pg in pages.items():
            before = torch.zeros(len(v), dtype=torch.int32, device="cuda")
            after = torch.zeros(len(v), dtype=torch.int32, device="cuda")
            assert dec.decode(enc, abi.TYPE_INT, pg, before.data_ptr(), len(v)) == len(v)
            dec.set_dict(np.arange(7, dtype=np.int32))
            assert dec.decode(enc, abi.TYPE_INT, pg, after.data_ptr(), len(v)) == len(v)
            ctx.sync()
            assert (before.cpu().numpy() == v).all() and (after.cpu().numpy() == v).all(), enc
    finally:
        dec.close()


# ---- SSB Q4.1 with c_region, c_nation, s_region and p_mfgr as words --------------------------------------------------
REGIONS = [b"AFRICA", b"AMERICA", b"ASIA", b"EUROPE", b"MIDDLE EAST"]          # ssb.py's codes 0..4 (AMERICA = 1)
NATIONS = [b"ALGERIA", b"ETHIOPIA", b"KENYA", b"MOROCCO", b"MOZAMBIQUE", b"ARGENTINA", b"BRAZIL", b"CANADA", b"PERU",
           b"UNITED STATES", b"CHINA", b"INDIA", b"INDONESIA", b"JAPAN", b"VIETNAM", b"FRANCE", b"GERMANY", b"ROMANIA",
           b"RUSSIA", b"UNITED KINGDOM", b"EGYPT", b"IRAN", b"IRAQ", b"JORDAN", b"SAUDI ARABIA"]   # region * 5 + k
MFGRS = [b"MFGR#1", b"MFGR#2", b"MFGR#3", b"MFGR#4", b"MFGR#5"]                     # MFGR#1 = 0, MFGR#2 = 1


def _sorted_global_dict(vocab):
    """make_sorted_global_dict: the distinct words in byte order, ids 1..n"""
    return {w: i + 1 for i, w in enumerate(sorted(set(vocab)))}


def test_ssb_q41_with_dictionary_string_columns(gpu, ctx, bo, oracle):
    import torch
    from starrocks_b200.rows import assert_rows_equal, gpu_rows, oracle_rows
    dims = ssb.gen_dims(0.05)
    lo = ssb.gen_lineorder(0.05, n=200_000)
    strings = {("customer", "c_region"): REGIONS, ("customer", "c_nation"): NATIONS, ("supplier", "s_region"): REGIONS,
               ("part", "p_mfgr"): MFGRS}
    gdicts = {k: _sorted_global_dict(v) for k, v in strings.items()}
    dec = gpu.PageDecoder(ctx)
    try:
        # every dimension column on the device: keys as they are, strings written as dictionary pages in three segments
        # (each with its own first-seen dictionary) and decoded into global ids
        ddims = {}
        for table in ("customer", "supplier", "part", "dates"):
            cols = {}
            for name, v in dims[table].items():
                if (table, name) in strings:
                    words = [strings[table, name][c] for c in v]
                    n = len(words)
                    bounds = [0, n // 3, n // 3 + 1 + n // 5, n]
                    out = _decode_segments(ctx, dec, bo, words, gdicts[table, name], bounds, 512)
                    assert (out.cpu().numpy()[:n] == [gdicts[table, name][w] for w in words]).all(), name
                    cols[name] = out[:n]
                else:
                    cols[name] = torch.from_numpy(v).cuda()
            ddims[table] = cols
    finally:
        dec.close()
    america_c, america_s = gdicts["customer", "c_region"][b"AMERICA"], gdicts["supplier", "s_region"][b"AMERICA"]
    mfgr = gdicts["part", "p_mfgr"]
    plans = []
    for table, key_col, key_slot, probe_slot, payload, preds, slotmap in ssb.dim_plans_q41():
        preds = {"supplier": [abi.make_pred(ssb.S_REGION, abi.PRED_EQ, america_s)],
                 "customer": [abi.make_pred(ssb.C_REGION, abi.PRED_EQ, america_c)],
                 "part": [abi.make_pred(ssb.P_MFGR, abi.PRED_IN, in_list=[mfgr[b"MFGR#1"], mfgr[b"MFGR#2"]])],
                 "dates": []}[table]
        plans.append((table, key_col, key_slot, probe_slot, payload, preds, slotmap))
    gjoins, keep = [], []
    for table, key_col, key_slot, probe_slot, payload, preds, slotmap in plans:
        cols = ddims[table]
        chunk = Chunk([(slotmap[nm], cols[nm], None, abi.TYPE_INT) for nm in cols], num_rows=len(cols[key_col]), mem=abi.MEM_DEVICE)
        scan = gpu.Scan(ctx, abi.ScanDesc(preds=preds, out_slots=[key_slot] + [s for _, s in payload]))
        out = scan.filter(chunk)
        bchunk = Chunk([(out.cols[k].slot_id, out.cols[k].data, out.cols[k].nulls, out.cols[k].type) for k in range(out.num_cols)],
                       num_rows=out.num_rows, mem=abi.MEM_DEVICE)
        j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [key_slot], [probe_slot], [abi.TYPE_INT], build_out=[s for _, s in payload], probe_out=[]))
        j.append_build(bchunk)
        j.build_finish()
        keep.append((scan, chunk, bchunk))
        gjoins.append((j, probe_slot, [s for _, s in payload]))
    nation_ids = gdicts["customer", "c_nation"]
    agg_desc = abi.make_agg_desc([ssb.D_YEAR, ssb.C_NATION], [abi.TYPE_INT, abi.TYPE_INT],
                                 fns=[(abi.AGG_SUM, abi.TYPE_INT, ssb.OUT_SUM_REVENUE, [("col", ssb.LO_REVENUE)]),
                                      (abi.AGG_SUM, abi.TYPE_INT, ssb.OUT_SUM_SUPPLYCOST, [("col", ssb.LO_SUPPLYCOST)])],
                                 ranges=[(1992, 1998), (1, len(nation_ids))])
    frag = gpu.Fragment(ctx, abi.ScanDesc(), gjoins, agg_desc)
    try:
        chunk = ssb.fact_chunk(lo, ssb.Q41_FACT_COLS)
        frag.push(chunk)
        by_id = {i: w for w, i in nation_ids.items()}
        got = sorted((r[0], by_id[r[1]]) + tuple(r[2:]) for r in gpu_rows(frag.agg.result()))
        passed = frag.rows_passed
    finally:
        frag.close()
        for j, _, _ in gjoins:
            j.close()
        for item in keep:
            item[0].close()
    # the oracle on the original arrays (ssb.py's fixed codes), its groups mapped to words
    ojoins, okeep = ssb.build_dims(oracle, dims, ssb.dim_plans_q41())
    ores, opassed = oracle.fragment_run(abi.ScanDesc(), ojoins, ssb.q41_agg_desc(), chunk, num_threads=2)
    want = sorted((r[0], NATIONS[r[1]]) + tuple(r[2:]) for r in oracle_rows(ores))
    assert passed == opassed
    assert len(want) == 35
    assert_rows_equal(got, want)
