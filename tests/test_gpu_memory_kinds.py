"""Every entry point that takes a memory kind (an `sr_mem` argument or `sr_chunk_view.mem`) follows the one rule stated in
include/sr_gpu_ops.h:

- SR_MEM_HOST, SR_MEM_HOST_PINNED and SR_MEM_DEVICE give byte-identical results, with the same number of kernel
  launches: outside sr_fragment_push and sr_pages_decode, SR_MEM_HOST_PINNED is host memory like SR_MEM_HOST.
- A result written into host memory (either host kind) is complete when the call returns.  Each call below runs behind
  a ~50 ms spin queued on the context's stream, with its output pre-filled with a sentinel, and its host output is read
  with no sr_ctx_sync: a call that returned before its copy ran would leave the sentinel in place.
- An unknown kind is refused with SR_ERR_INVALID_ARGUMENT before any launch or device allocation.

Every buffer passed as SR_MEM_HOST_PINNED or with an unknown kind is page-locked, so it is a valid address both for the
host and for the device whichever way a build reads the tag.
"""
import ctypes as C

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

HOST, DEVICE, PINNED = abi.MEM_HOST, abi.MEM_DEVICE, abi.MEM_HOST_PINNED
KINDS = {"host": HOST, "pinned": PINNED, "device": DEVICE}
INT, BIGINT = abi.TYPE_INT, abi.TYPE_BIGINT
SENTINEL = 0xAB
SPIN_CYCLES = 100_000_000   # ~50-60 ms at the H100's SM clock


def spin(ctx):
    """a bounded busy kernel on the context's stream: whatever the next call queues runs after it"""
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(ctx.stream)):
        torch.cuda._sleep(SPIN_CYCLES)


class Buf:
    """`nbytes` in memory kind `kind`, filled with `fill`: a pageable numpy array (host), a page-locked tensor (pinned,
    and any unknown kind) or a device tensor"""

    def __init__(self, kind, nbytes, fill=SENTINEL):
        import torch
        self.kind, self.nbytes = kind, nbytes
        if kind == HOST:
            self.a = np.full(max(nbytes, 1), fill, dtype=np.uint8)
            self.ptr = self.a.ctypes.data
        else:
            dev = "cuda" if kind == DEVICE else "cpu"
            self.t = torch.full((max(nbytes, 1),), fill, dtype=torch.uint8, device=dev)
            if kind != DEVICE:
                self.t = self.t.pin_memory()
            self.ptr = self.t.data_ptr()

    @classmethod
    def of(cls, kind, arr):
        """a copy of numpy array `arr` in `kind`"""
        import torch
        raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        b = cls(kind, raw.size, 0)
        if kind == HOST:
            b.a[:raw.size] = raw
        else:
            b.t[:raw.size].copy_(torch.from_numpy(raw.copy()))
            if kind == DEVICE:
                torch.cuda.synchronize()
        return b

    def read(self):
        """the buffer's bytes; a host buffer is read as it is now, without waiting for any stream"""
        if self.kind == HOST:
            return self.a[:self.nbytes].tobytes()
        return self.t[:self.nbytes].cpu().numpy().tobytes()


def placed_chunk(kind, cols, n):
    """cols: [(slot, numpy array)] copied into `kind` -> (Chunk, buffers to keep alive)"""
    bufs = [Buf.of(kind, a) for _, a in cols]
    spec = [(slot, b.ptr, None, abi.NUMPY_TYPE[a.dtype]) for (slot, a), b in zip(cols, bufs)]
    return Chunk(spec, num_rows=n, mem=kind), bufs


def run_kinds(ctx, call):
    """call(kind) -> (output Buf or host bytes getter, expected bytes) for each kind, behind a spin; checks the host
    result before any sync and the device result after one, and that every kind made the same number of launches"""
    launches = {}
    for name, kind in KINDS.items():
        spin(ctx)
        before = ctx.launches
        read, want = call(kind)
        launches[name] = ctx.launches - before
        if kind != DEVICE:
            assert read() == want, f"{name}: host result not complete when the call returned"
        ctx.sync()
        assert read() == want, f"{name}: wrong result"
    assert len(set(launches.values())) == 1, f"launches per kind differ: {launches}"


def keys(n, seed=1):
    return np.random.default_rng(seed).integers(-(1 << 30), 1 << 30, n).astype(np.int32)


# =============================================================================================
# same result, complete on return, same launches
# =============================================================================================
@pytest.mark.gpu
def test_scan_evaluate(gpu, ctx):
    n = 300_000
    x = keys(n)
    chunk, keep = placed_chunk(HOST, [(1, x)], n)
    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_LT, 0)]))
    want = (x < 0).astype(np.uint8).tobytes()
    scan.evaluate(chunk)   # compiles the scan: its launches are not part of the comparison

    def call(kind):
        out = Buf(kind, n)
        ctx.check(gpu.lib().sr_scan_evaluate(scan.h, chunk.ref(), out.ptr, kind))
        return out.read, want
    try:
        run_kinds(ctx, call)
    finally:
        scan.close()


@pytest.mark.gpu
def test_xchg_hash(gpu, ctx):
    n = 300_000
    chunk, keep = placed_chunk(HOST, [(1, keys(n))], n)
    x = gpu.Xchg(ctx, abi.make_part_desc([1], 17))
    try:
        hv, ch = x.hash(chunk)           # the SR_MEM_HOST result, pinned down by test_gpu_exchange_edges.py
        want = hv.tobytes() + ch.tobytes()

        def call(kind):
            h, c = Buf(kind, 4 * n), Buf(kind, 4 * n)
            ctx.check(gpu.lib().sr_xchg_hash(x.h, chunk.ref(), h.ptr, c.ptr, kind))
            return (lambda: h.read() + c.read()), want
        run_kinds(ctx, call)
    finally:
        x.close()


@pytest.mark.gpu
def test_join_key_hash(gpu, ctx):
    n = 300_000
    k = keys(n).astype(np.int64) * 3
    want = ctx.join_key_hash(k, 20).tobytes()  # the SR_MEM_HOST result, pinned down by the golden-vector tests

    def call(kind):
        out = Buf(kind, 4 * n)
        out.keys = Buf.of(kind, k)   # lives as long as the output is read
        ctx.check(gpu.lib().sr_join_key_hash(ctx.h, out.keys.ptr, BIGINT, n, 20, out.ptr, kind))
        return out.read, want
    run_kinds(ctx, call)


RF_KEYS = 5000


def _rf(gpu, ctx):
    rf = gpu.RuntimeFilter(ctx, INT, RF_KEYS)
    chunk, keep = placed_chunk(HOST, [(1, keys(RF_KEYS, seed=2))], RF_KEYS)
    rf.insert(chunk, 1)
    return rf


@pytest.mark.gpu
def test_rf_copy_directory(gpu, ctx):
    rf = _rf(gpu, ctx)
    try:
        want = rf.directory().tobytes()
        assert any(want)

        def call(kind):
            out = Buf(kind, len(want))
            ctx.check(gpu.lib().sr_rf_copy_directory(rf.h, out.ptr, len(want), kind))
            return out.read, want
        run_kinds(ctx, call)
    finally:
        rf.close()


@pytest.mark.gpu
def test_rf_merge_directory(gpu, ctx):
    src = _rf(gpu, ctx)
    try:
        other, info = src.directory(), src.info()
        for name, kind in KINDS.items():
            dst = gpu.RuntimeFilter(ctx, INT, RF_KEYS)
            try:
                d = Buf.of(kind, other)
                spin(ctx)
                before = ctx.launches
                ctx.check(gpu.lib().sr_rf_merge_directory(dst.h, d.ptr, other.nbytes, kind, C.byref(info)))
                assert ctx.launches - before == 2, name
                assert dst.directory().tobytes() == other.tobytes(), name
            finally:
                dst.close()
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("merge_and", [0, 1])
def test_rf_evaluate(gpu, ctx, merge_and):
    n = 300_000
    rf = _rf(gpu, ctx)
    probe = keys(n, seed=3)
    probe[::7] = np.resize(keys(RF_KEYS, seed=2), len(probe[::7]))   # every 7th row holds an inserted key
    chunk, keep = placed_chunk(HOST, [(1, probe)], n)
    prior = (np.arange(n) % 3 != 0).astype(np.uint8)
    try:
        want = rf.evaluate(chunk, 1, prior if merge_and else None).tobytes()   # the SR_MEM_HOST result

        def call(kind):
            sel = Buf.of(kind, prior) if merge_and else Buf(kind, n)
            ctx.check(gpu.lib().sr_rf_evaluate(rf.h, chunk.ref(), 1, sel.ptr, kind, merge_and))
            return sel.read, want
        run_kinds(ctx, call)
    finally:
        rf.close()


@pytest.mark.gpu
def test_agg_pull(gpu, ctx):
    """each kind pulls the second half of the groups on its own handle; the first half is pulled as SR_MEM_HOST, and its
    host buffers, which the second pull reuses, are overwritten with the sentinel"""
    n, g = 200_000, 4096
    k = (np.arange(n) % g).astype(np.int32)
    v = keys(n).astype(np.int64)
    want = {i: int(v[k == i].sum()) for i in range(g)}
    chunk, keep = placed_chunk(HOST, [(1, k), (2, v)], n)
    desc = abi.make_agg_desc([1], [INT], fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)])])
    launches = {}
    for name, kind in KINDS.items():
        a = gpu.Agg(ctx, desc)
        try:
            a.push(chunk)
            a.finish()
            first = a.pull(max_rows=g // 2, mem=HOST)
            got = {}
            for key, s in zip(*[col[2] for col in gpu.chunk_out_to_host(ctx, first)]):
                got[int(key)] = int(s)
            for c in first.cols[:first.num_cols]:
                C.memset(c.data, SENTINEL, first.num_rows * abi.TYPE_WIDTH[c.type])
            spin(ctx)
            before = ctx.launches
            out = a.pull(max_rows=g // 2, mem=kind)
            launches[name] = ctx.launches - before
            assert out.num_rows == g // 2, name
            if kind != DEVICE:
                kcol = np.ctypeslib.as_array(C.cast(out.cols[0].data, C.POINTER(C.c_int32)), shape=(g // 2,)).copy()
                scol = np.ctypeslib.as_array(C.cast(out.cols[1].data, C.POINTER(C.c_int64)), shape=(g // 2,)).copy()
                rows = list(zip(kcol.tolist(), scol.tolist()))
            else:
                rows = list(zip(*[col[2].tolist() for col in gpu.chunk_out_to_host(ctx, out)]))
            got.update(rows)
            assert got == want, f"{name}: result incomplete or wrong"
            assert out.mem == (DEVICE if kind == DEVICE else HOST), name
        finally:
            a.close()
    assert len(set(launches.values())) == 1, f"launches per kind differ: {launches}"


@pytest.mark.gpu
def test_chunk_deserialize(gpu, ctx):
    """an input only: a ChunkPB payload read from each kind gives the same device columns"""
    n = 20_000
    x = keys(n)
    chunk, keep = placed_chunk(HOST, [(1, x)], n)
    payload, meta = gpu.chunk_serialize(ctx, chunk)
    sd = gpu.Serde(ctx)
    try:
        for name, kind in KINDS.items():
            src = Buf.of(kind, payload)
            out = abi.sr_chunk_out()
            before = ctx.launches
            ctx.check(gpu.lib().sr_chunk_deserialize(sd.h, src.ptr, payload.nbytes, kind, C.byref(meta), C.byref(out)))
            assert ctx.launches == before, name
            (slot, typ, data, nulls), = gpu.chunk_out_to_host(ctx, out)
            assert slot == 1 and data.tobytes() == x.tobytes() and nulls is None, name
    finally:
        sd.close()


# =============================================================================================
# unknown kinds
# =============================================================================================
def _pinned(arr):
    return Buf.of(PINNED, arr)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [3, -1])
def test_unknown_kind_refused(gpu, ctx, bad):
    L = gpu.lib()
    n = 1000
    x = keys(n)
    good, keep_good = placed_chunk(PINNED, [(1, x), (2, x.astype(np.int64))], n)
    badc, keep_bad = placed_chunk(PINNED, [(1, x), (2, x.astype(np.int64))], n)
    badc.view.mem = bad
    out_buf = _pinned(np.zeros(16 * n, dtype=np.uint8))
    sel = _pinned(np.ones(n, dtype=np.uint8))
    idx = _pinned(np.arange(n, dtype=np.uint32))

    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_LT, 0)], out_slots=[1]))
    xchg = gpu.Xchg(ctx, abi.make_part_desc([1], 8))
    rf = _rf(gpu, ctx)
    directory = rf.directory()
    info = rf.info()
    dir_buf = _pinned(directory)
    desc = abi.make_agg_desc([1], [INT], fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)])])
    agg = gpu.Agg(ctx, desc)
    p1, _ = abi.two_phase_descs(desc)
    first = gpu.Agg(ctx, p1)
    pulled = gpu.Agg(ctx, desc)
    pulled.push(good)
    pulled.finish()
    join = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT], build_out=[2]))
    probed = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT], build_out=[2]))
    probed.append_build(good)
    probed.build_finish()
    dim = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [1], [1], [INT]))
    dim.append_build(Chunk([(1, np.unique(x), None)]))
    dim.build_finish()
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [(dim, 1, [])], abi.make_agg_desc(fns=[(abi.AGG_COUNT_STAR, 0, 10, None)]))
    sd = gpu.Serde(ctx)
    dec = gpu.PageDecoder(ctx)
    payload, meta = gpu.chunk_serialize(ctx, good)
    payload_buf = _pinned(payload)
    pages = (abi.sr_page_view * 1)()
    pages[0].data, pages[0].size = payload_buf.ptr, payload.nbytes
    rows = C.c_int64(0)
    co = abi.sr_chunk_out()
    offs = np.zeros(9, dtype=np.int64)
    pmeta = abi.sr_chunk_pb_meta()
    calls = {
        "sr_scan_evaluate sel_mem": lambda: L.sr_scan_evaluate(scan.h, good.ref(), sel.ptr, bad),
        "sr_scan_evaluate chunk": lambda: L.sr_scan_evaluate(scan.h, badc.ref(), sel.ptr, PINNED),
        "sr_scan_filter chunk": lambda: L.sr_scan_filter(scan.h, badc.ref(), C.byref(co)),
        "sr_xchg_hash mem": lambda: L.sr_xchg_hash(xchg.h, good.ref(), out_buf.ptr, None, bad),
        "sr_xchg_hash chunk": lambda: L.sr_xchg_hash(xchg.h, badc.ref(), out_buf.ptr, None, PINNED),
        "sr_xchg_partition chunk": lambda: L.sr_xchg_partition(xchg.h, badc.ref(), C.byref(co), offs.ctypes.data),
        "sr_join_key_hash": lambda: L.sr_join_key_hash(ctx.h, idx.ptr, INT, n, 20, out_buf.ptr, bad),
        "sr_rf_copy_directory": lambda: L.sr_rf_copy_directory(rf.h, dir_buf.ptr, directory.nbytes, bad),
        "sr_rf_merge_directory": lambda: L.sr_rf_merge_directory(rf.h, dir_buf.ptr, directory.nbytes, bad, C.byref(info)),
        "sr_rf_evaluate sel_mem": lambda: L.sr_rf_evaluate(rf.h, good.ref(), 1, sel.ptr, bad, 1),
        "sr_rf_evaluate chunk": lambda: L.sr_rf_evaluate(rf.h, badc.ref(), 1, sel.ptr, PINNED, 1),
        "sr_rf_insert chunk": lambda: L.sr_rf_insert(rf.h, badc.ref(), 1, 0),
        "sr_agg_push chunk": lambda: L.sr_agg_push(agg.h, badc.ref()),
        "sr_agg_convert_to_states chunk": lambda: L.sr_agg_convert_to_states(first.h, badc.ref(), C.byref(co)),
        "sr_agg_push_selective chunk": lambda: L.sr_agg_push_selective(first.h, badc.ref(), C.byref(co)),
        "sr_agg_pull out_mem": lambda: L.sr_agg_pull(pulled.h, 100, bad, C.byref(co)),
        "sr_join_append_build chunk": lambda: L.sr_join_append_build(join.h, badc.ref()),
        "sr_join_probe chunk": lambda: L.sr_join_probe(probed.h, 0, badc.ref(), C.byref(co)),
        "sr_fragment_push chunk": lambda: L.sr_fragment_push(frag.h, badc.ref()),
        "sr_gather": lambda: L.sr_gather(ctx.h, out_buf.ptr, INT, idx.ptr, n, out_buf.ptr, bad),
        "sr_chunk_serialize dst_mem": lambda: L.sr_chunk_serialize(ctx.h, good.ref(), 0, n, out_buf.ptr, 16 * n, bad, C.byref(pmeta)),
        "sr_chunk_serialize chunk": lambda: L.sr_chunk_serialize(ctx.h, badc.ref(), 0, n, out_buf.ptr, 16 * n, PINNED, C.byref(pmeta)),
        "sr_chunk_deserialize src_mem": lambda: L.sr_chunk_deserialize(sd.h, payload_buf.ptr, payload.nbytes, bad, C.byref(meta), C.byref(co)),
        "sr_page_decoder_set_dict": lambda: L.sr_page_decoder_set_dict(dec.h, idx.ptr, n, bad),
        "sr_pages_decode": lambda: L.sr_pages_decode(dec.h, abi.PAGE_PLAIN, INT, pages, 1, bad, out_buf.ptr, n, C.byref(rows)),
    }
    try:
        ctx.sync()
        for name, call in calls.items():
            launches, dev_bytes = ctx.launches, ctx.device_bytes
            assert call() == abi.SR_ERR_INVALID_ARGUMENT, name
            assert b"unknown memory kind" in L.sr_last_error(ctx.h), name
            assert (ctx.launches, ctx.device_bytes) == (launches, dev_bytes), name
        ctx.sync()
        # a host kind of sr_gather stays unsupported
        assert L.sr_gather(ctx.h, out_buf.ptr, INT, idx.ptr, n, out_buf.ptr, PINNED) == abi.SR_ERR_NOT_SUPPORTED
    finally:
        for h in (frag, dim, probed, join, pulled, first, agg, rf, xchg, scan, sd, dec):
            h.close()
