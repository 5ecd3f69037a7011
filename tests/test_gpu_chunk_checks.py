"""The checks every entry point makes on a caller's sr_chunk_view (include/sr_gpu_ops.h), and the one resolver of the
page-locked buffers the in-place readers take:

- Each entry point that takes a chunk refuses a malformed one (an unknown kind, num_rows < 0, cols == NULL with columns,
  an unknown column type, data == NULL with rows) with SR_ERR_INVALID_ARGUMENT before any launch or device allocation,
  and the next good call on the same handle returns the right result.  None of the malformed pointers is read.
- sr_fragment_push, sr_pages_decode and sr_null_maps_decode read SR_MEM_HOST_PINNED buffers in place: pageable memory
  passed as pinned is refused, and a range registered with sr_host_register and a torch page-locked tensor outside that
  registry both give the bytes SR_MEM_DEVICE gives.
"""
import ctypes as C

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from starrocks_b200.rows import gpu_rows
from tests.test_gpu_for_plain_pages import plain_page

INT, BIGINT = abi.TYPE_INT, abi.TYPE_BIGINT
N = 3000
K = (np.arange(N) - N // 2).astype(np.int32)           # slot 1: distinct keys, half of them negative
V = K.astype(np.int64) * 10 + 7                          # slot 2
MALFORMED = ("unknown_kind", "negative_rows", "no_column_array", "unknown_type", "null_data")


def good_chunk():
    return Chunk([(1, K, None), (2, V, None)], num_rows=N)


def malformed(form):
    """the two-column host chunk of K and V, broken in one way"""
    c = good_chunk()
    if form == "unknown_kind":
        c.view.mem = 7
    elif form == "negative_rows":
        c.view.num_rows = -1
    elif form == "no_column_array":
        c.view.cols = None
    elif form == "unknown_type":
        c._cols[0].type = 1000
    else:
        c._cols[0].data = None
    return c


def refuse_each(ctx, call, good):
    """call(chunk) -> status, once per malformed form: each refused before any launch or device allocation, then
    good() on the same handle"""
    for form in MALFORMED:
        bad = malformed(form)
        launches, nbytes = ctx.launches, ctx.device_bytes
        rc = call(bad)
        assert rc == abi.SR_ERR_INVALID_ARGUMENT, (form, rc, gpu_error(ctx))
        assert (ctx.launches, ctx.device_bytes) == (launches, nbytes), form
        good()


def gpu_error(ctx):
    from starrocks_b200.gpu import lib
    return lib().sr_last_error(ctx.h)


def out_col(ctx, out, slot):
    from starrocks_b200.gpu import chunk_out_to_host
    return {s: (d, nl) for s, _, d, nl in chunk_out_to_host(ctx, out)}[slot]


# =============================================================================================
# malformed chunks, at every entry point that takes one
# =============================================================================================
@pytest.mark.gpu
def test_scan(gpu, ctx):
    L = gpu.lib()
    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_LT, 0)], out_slots=[1, 2]))
    sel = np.zeros(N, np.uint8)
    out = abi.sr_chunk_out()
    try:
        def good_evaluate():
            assert np.array_equal(scan.evaluate(good_chunk()), (K < 0).astype(np.uint8))

        def good_filter():
            o = scan.filter(good_chunk())
            assert o.num_rows == int((K < 0).sum())
            assert np.array_equal(out_col(ctx, o, 1)[0], K[K < 0]) and np.array_equal(out_col(ctx, o, 2)[0], V[K < 0])
        refuse_each(ctx, lambda c: L.sr_scan_evaluate(scan.h, c.ref(), sel.ctypes.data, abi.MEM_HOST), good_evaluate)
        refuse_each(ctx, lambda c: L.sr_scan_filter(scan.h, c.ref(), C.byref(out)), good_filter)
    finally:
        scan.close()


@pytest.mark.gpu
def test_join_append_build_and_probe(gpu, ctx):
    L = gpu.lib()
    desc = abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT], build_out=[2])
    join = gpu.Join(ctx, desc)
    probed = gpu.Join(ctx, desc)
    out = abi.sr_chunk_out()
    try:
        appends = []

        def good_append():
            join.append_build(good_chunk())
            appends.append(1)
        refuse_each(ctx, lambda c: L.sr_join_append_build(join.h, c.ref()), good_append)
        join.build_finish()
        assert join.info().build_rows == len(appends) * N
        o = join.probe(good_chunk())                                   # every key is in the build side once per append
        assert o.num_rows == len(appends) * N
        assert np.array_equal(np.sort(out_col(ctx, o, 2)[0]), np.sort(np.tile(V, len(appends))))

        probed.append_build(good_chunk())
        probed.build_finish()

        def good_probe():
            o = probed.probe(good_chunk())
            assert o.num_rows == N and np.array_equal(np.sort(out_col(ctx, o, 2)[0]), np.sort(V))
        refuse_each(ctx, lambda c: L.sr_join_probe(probed.h, 0, c.ref(), C.byref(out)), good_probe)
    finally:
        probed.close()
        join.close()


@pytest.mark.gpu
def test_agg(gpu, ctx):
    L = gpu.lib()
    desc = abi.make_agg_desc([1], [INT], fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)])])
    first, _ = abi.two_phase_descs(desc)
    agg, conv, sel = gpu.Agg(ctx, desc), gpu.Agg(ctx, first), gpu.Agg(ctx, first)
    out = abi.sr_chunk_out()
    try:
        pushes = []

        def good_push():
            agg.push(good_chunk())
            pushes.append(1)

        def good_states(h):
            def check():
                o = h.convert_to_states(good_chunk()) if h is conv else h.push_selective(good_chunk())
                assert o.num_rows == N                                # an empty table: every row is streamed
                assert np.array_equal(out_col(ctx, o, 1)[0], K)
            return check
        refuse_each(ctx, lambda c: L.sr_agg_push(agg.h, c.ref()), good_push)
        refuse_each(ctx, lambda c: L.sr_agg_convert_to_states(conv.h, c.ref(), C.byref(out)), good_states(conv))
        refuse_each(ctx, lambda c: L.sr_agg_push_selective(sel.h, c.ref(), C.byref(out)), good_states(sel))
        assert gpu_rows(agg.result()) == sorted(zip(K.tolist(), (V * len(pushes)).tolist()))
    finally:
        for h in (sel, conv, agg):
            h.close()


@pytest.mark.gpu
def test_xchg(gpu, ctx):
    L = gpu.lib()
    desc = abi.make_part_desc([1], 8)
    x, ref = gpu.Xchg(ctx, desc), gpu.Xchg(ctx, desc)
    hv, ch = np.zeros(N, np.uint32), np.zeros(N, np.uint32)
    out, offs = abi.sr_chunk_out(), np.zeros(9, np.int64)
    try:
        want_hv, want_ch = ref.hash(good_chunk())
        want_out, want_offs = ref.partition(good_chunk())
        want_k = out_col(ctx, want_out, 1)[0].copy()

        def good_hash():
            got_hv, got_ch = x.hash(good_chunk())
            assert np.array_equal(got_hv, want_hv) and np.array_equal(got_ch, want_ch)

        def good_partition():
            o, offsets = x.partition(good_chunk())
            assert np.array_equal(offsets, want_offs) and np.array_equal(out_col(ctx, o, 1)[0], want_k)
        refuse_each(ctx, lambda c: L.sr_xchg_hash(x.h, c.ref(), hv.ctypes.data, ch.ctypes.data, abi.MEM_HOST), good_hash)
        refuse_each(ctx, lambda c: L.sr_xchg_partition(x.h, c.ref(), C.byref(out), offs.ctypes.data), good_partition)
    finally:
        ref.close()
        x.close()


@pytest.mark.gpu
def test_runtime_filter(gpu, ctx):
    L = gpu.lib()
    rf, probed = gpu.RuntimeFilter(ctx, INT, N), gpu.RuntimeFilter(ctx, INT, N)
    sel = np.zeros(N, np.uint8)
    outside = Chunk([(1, K + 10 * N, None)])                             # above the inserted keys' max
    try:
        def good_insert():
            rf.insert(good_chunk(), 1)
            assert rf.evaluate(good_chunk(), 1).all() and not rf.evaluate(outside, 1).any()
        refuse_each(ctx, lambda c: L.sr_rf_insert(rf.h, c.ref(), 1, 0), good_insert)

        probed.insert(good_chunk(), 1)

        def good_evaluate():
            assert probed.evaluate(good_chunk(), 1).all() and not probed.evaluate(outside, 1).any()
        refuse_each(ctx, lambda c: L.sr_rf_evaluate(probed.h, c.ref(), 1, sel.ctypes.data, abi.MEM_HOST, 0), good_evaluate)
    finally:
        probed.close()
        rf.close()


@pytest.mark.gpu
def test_chunk_serialize(gpu, ctx):
    L = gpu.lib()
    cap = L.sr_chunk_serialized_size(good_chunk().ref(), 0, N)
    dst = np.zeros(cap, np.uint8)
    meta = abi.sr_chunk_pb_meta()
    sd = gpu.Serde(ctx)
    try:
        def good():
            payload, m = gpu.chunk_serialize(ctx, good_chunk())
            o = sd.deserialize(payload, m)
            assert np.array_equal(out_col(ctx, o, 1)[0], K) and np.array_equal(out_col(ctx, o, 2)[0], V)
        refuse_each(ctx, lambda c: L.sr_chunk_serialize(ctx.h, c.ref(), 0, N, dst.ctypes.data, cap, abi.MEM_HOST, C.byref(meta)), good)
    finally:
        sd.close()


def _dim(gpu, ctx):
    """a dimension holding every key of K"""
    dim = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT]))
    dim.append_build(Chunk([(1, K.copy(), None)]))
    dim.build_finish()
    return dim


@pytest.mark.gpu
def test_fragment_push_and_push_chunks(gpu, ctx):
    L = gpu.lib()
    dim = _dim(gpu, ctx)
    count = abi.make_agg_desc(fns=[(abi.AGG_COUNT_STAR, 0, 10, None)])
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [])], count)
    listed = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [])], count)
    try:
        pushed = {frag: 0, listed: 0}

        def good_push():
            frag.push(good_chunk())
            pushed[frag] += N
            assert frag.rows_passed == pushed[frag]
        refuse_each(ctx, lambda c: L.sr_fragment_push(frag.h, c.ref()), good_push)

        def list_call(chunks):
            views = (abi.sr_chunk_view * len(chunks))(*[c.view for c in chunks])
            return L.sr_fragment_push_chunks(listed.h, views, len(chunks))

        def good_list():
            listed.push_chunks([good_chunk(), good_chunk()])
            pushed[listed] += 2 * N
            assert listed.rows_passed == pushed[listed]
        refuse_each(ctx, lambda c: list_call([c]), good_list)                  # the malformed chunk first
        refuse_each(ctx, lambda c: list_call([good_chunk(), c]), good_list)    # and behind a good one
        assert gpu_rows(frag.agg.result()) == [(pushed[frag],)]
        assert gpu_rows(listed.agg.result()) == [(pushed[listed],)]
    finally:
        listed.close()
        frag.close()
        dim.close()


# =============================================================================================
# the in-place readers of page-locked memory
# =============================================================================================
@pytest.fixture(scope="module")
def bo():
    import bshuf_oracle
    bshuf_oracle.lib()
    return bshuf_oracle


class Placed:
    """byte buffers laid out in one memory: "device" (torch CUDA), "registered" (one numpy arena registered with
    sr_host_register), "torch_pinned" (torch pin_memory, outside the library's registry) or "pageable" (numpy)"""

    def __init__(self, ctx, kind, bufs):
        import torch
        self.ctx, self.kind, self.registered = ctx, kind, None
        offs, at = [], 0
        for b in bufs:                                                 # 64-byte aligned, 100-byte gaps: scattered
            at = (at + 100 + 63) & ~63
            offs.append(at)
            at += len(b)
        blob = np.zeros(at + 64, np.uint8)
        for o, b in zip(offs, bufs):
            blob[o:o + len(b)] = b
        if kind == "device":
            self.keep = torch.from_numpy(blob).cuda()
            base = self.keep.data_ptr()
        elif kind == "torch_pinned":
            self.keep = torch.from_numpy(blob).pin_memory()
            base = self.keep.data_ptr()
            assert not ctx.host_is_mapped(base, blob.nbytes)
        else:
            self.keep = blob
            base = blob.ctypes.data
            if kind == "registered":
                ctx.host_register(blob)
                self.registered = blob
        self.mem = abi.MEM_DEVICE if kind == "device" else abi.MEM_HOST_PINNED
        self.ptrs = [base + o for o in offs]

    def close(self):
        if self.registered is not None:
            self.ctx.sync()
            self.ctx.host_unregister(self.registered)


IN_PLACE = ("device", "registered", "torch_pinned")


def _fact(n=N, seed=5):
    """fact columns: the join key, a nullable BIGINT measure (its null column) and an INT group key"""
    rng = np.random.default_rng(seed)
    key = rng.choice(K, n).astype(np.int32)
    val = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    nulls = (rng.random(n) < 0.2).astype(np.uint8)
    grp = (key % 13).astype(np.int32)
    return key, val, nulls, grp


def _fact_chunk(placed, n):
    p = placed.ptrs
    return Chunk([(1, p[0], None, INT), (2, p[1], p[2], BIGINT), (3, p[3], None, INT)], num_rows=n, mem=placed.mem)


@pytest.mark.gpu
def test_fragment_push_in_place(gpu, ctx):
    L = gpu.lib()
    dim = _dim(gpu, ctx)
    desc = abi.make_agg_desc([3], [INT], fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)]), (abi.AGG_COUNT_STAR, 0, 11, None)])
    key, val, nulls, grp = _fact()
    bufs = [key.view(np.uint8), val.view(np.uint8), nulls, grp.view(np.uint8)]
    want = sorted((g, int(val[(grp == g) & (nulls == 0)].sum()) if ((grp == g) & (nulls == 0)).any() else None, int((grp == g).sum()))
                  for g in np.unique(grp).tolist())
    try:
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [])], desc)
        pageable = Placed(ctx, "pageable", bufs)
        try:
            launches, nbytes = ctx.launches, ctx.device_bytes
            rc = L.sr_fragment_push(frag.h, _fact_chunk(pageable, N).ref())
            assert rc == abi.SR_ERR_INVALID_ARGUMENT and b"page-locked" in gpu_error(ctx), gpu_error(ctx)
            assert (ctx.launches, ctx.device_bytes) == (launches, nbytes)
            dev = Placed(ctx, "device", bufs)
            frag.push(_fact_chunk(dev, N))
            assert gpu_rows(frag.agg.result()) == want
        finally:
            frag.close()
        for kind in IN_PLACE:
            frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [])], desc)
            placed = Placed(ctx, kind, bufs)
            try:
                frag.push(_fact_chunk(placed, N))
                assert gpu_rows(frag.agg.result()) == want, kind
            finally:
                frag.close()
                placed.close()
    finally:
        dim.close()


def _pages(n_pages=5, rows=700, seed=7):
    rng = np.random.default_rng(seed)
    values = [rng.integers(-(1 << 31), 1 << 31, rows + k).astype(np.int32) for k in range(n_pages)]
    return [plain_page(v.view(np.uint32), 4) for v in values], np.concatenate(values)


def _decode(dec, pages_at, mem, n):
    import torch
    out = torch.zeros(n, dtype=torch.int32, device="cuda")
    rows = dec.decode(abi.PAGE_PLAIN, INT, pages_at, out.data_ptr(), n, mem=mem)
    return rows, out.cpu().numpy()


@pytest.mark.gpu
def test_pages_decode_in_place(gpu, ctx):
    import torch
    L = gpu.lib()
    pages, values = _pages()
    n = len(values)
    dec = gpu.PageDecoder(ctx)
    try:
        pageable = Placed(ctx, "pageable", pages)
        views = (abi.sr_page_view * len(pages))()
        for k, (p, pg) in enumerate(zip(pageable.ptrs, pages)):
            views[k].data, views[k].size = p, len(pg)
        out = torch.zeros(n, dtype=torch.int32, device="cuda")
        rows = C.c_int64(0)
        launches, nbytes = ctx.launches, ctx.device_bytes
        rc = L.sr_pages_decode(dec.h, abi.PAGE_PLAIN, INT, views, len(pages), abi.MEM_HOST_PINNED, out.data_ptr(), n, C.byref(rows))
        assert rc == abi.SR_ERR_INVALID_ARGUMENT and b"page-locked" in gpu_error(ctx), gpu_error(ctx)
        assert (ctx.launches, ctx.device_bytes) == (launches, nbytes)
        results = {}
        for kind in IN_PLACE:
            placed = Placed(ctx, kind, pages)
            try:
                results[kind] = _decode(dec, list(zip(placed.ptrs, [len(p) for p in pages])), placed.mem, n)
                ctx.sync()
            finally:
                placed.close()
        assert results["device"][0] == n and np.array_equal(results["device"][1], values)
        for kind in IN_PLACE:
            assert results[kind][0] == n and results[kind][1].tobytes() == results["device"][1].tobytes(), kind
    finally:
        dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("enc", [abi.NULL_BITSHUFFLE, abi.NULL_RLE], ids=["bitshuffle", "rle"])
def test_null_maps_decode_in_place(gpu, ctx, bo, enc):
    import torch
    L = gpu.lib()
    rng = np.random.default_rng(11)
    rows = [900, 1000, 1, 4096]
    flags = [(rng.random(r) < 0.3).astype(np.uint8) for r in rows]
    maps = [bo.null_map_encode(f, enc) for f in flags]
    n = sum(rows)
    want = np.concatenate(flags)
    dec = gpu.PageDecoder(ctx)
    try:
        pageable = Placed(ctx, "pageable", maps)
        views = (abi.sr_null_map_view * len(maps))()
        for k, (p, m, r) in enumerate(zip(pageable.ptrs, maps, rows)):
            views[k].data, views[k].size, views[k].num_rows = p, len(m), r
        out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        got_rows, got_nulls = C.c_int64(0), C.c_int64(0)
        launches, nbytes = ctx.launches, ctx.device_bytes
        rc = L.sr_null_maps_decode(dec.h, enc, views, len(maps), abi.MEM_HOST_PINNED, out.data_ptr(), n, C.byref(got_rows), C.byref(got_nulls))
        assert rc == abi.SR_ERR_INVALID_ARGUMENT and b"page-locked" in gpu_error(ctx), gpu_error(ctx)
        assert (ctx.launches, ctx.device_bytes) == (launches, nbytes)
        results = {}
        for kind in IN_PLACE:
            placed = Placed(ctx, kind, maps)
            try:
                out = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
                got = dec.decode_nulls(enc, [(p, len(m), r) for p, m, r in zip(placed.ptrs, maps, rows)], out.data_ptr(), n, mem=placed.mem)
                ctx.sync()
                results[kind] = (got, out.cpu().numpy())
            finally:
                placed.close()
        assert results["device"][0] == (n, int(want.sum())) and np.array_equal(results["device"][1], want)
        for kind in IN_PLACE:
            assert results[kind][0] == results["device"][0] and results[kind][1].tobytes() == results["device"][1].tobytes(), kind
    finally:
        dec.close()
