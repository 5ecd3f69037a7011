"""sr_fragment_push_chunks: a list of chunks, each in its own memory kind, pushed into the fused fragment as one batch,
gathered on the device by k_chunk_gather.  Every plan of tests/test_gpu_frag_plans.py through random chunk lists (sizes
0, 1, 3, 4095, 4096, 4097 and random ones up to 9000; device, device one element off, torch-pinned, a registered numpy
arena and pageable host memory), the load phases of the gather, null columns present in only some chunks, the push
lifecycle, the refusals and the page-locked registry (sr_host_register / sr_host_is_mapped).  The forwarding fragment sink
of the C++ operators runs in tests/cpp/frag_chunk_list_test.cpp."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from tests.test_gpu_frag_plans import CASES, Run, _check, build_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
KINDS = ("device", "device_off", "pinned", "arena", "host")
SIZES = (0, 1, 3, 4095, 4096, 4097)


class Copies:
    """the fact columns in every memory kind: one allocation per column and kind (device_off: one element into it), and
    one registered numpy arena holding all of them; chunks are slices, so successive chunks land at every phase"""

    def __init__(self, ctx, cols):
        import torch
        self.ctx, self.cols, self.keep = ctx, cols, []
        self.base = {k: {} for k in KINDS}            # kind -> slot -> (data pointer, nulls pointer or None)
        total = sum(d.nbytes + (0 if nl is None else nl.nbytes) + 128 for _, d, nl, _ in cols)
        self.arena = np.zeros(total + 4096, np.uint8)
        off = (-self.arena.ctypes.data) % 64
        for s, d, nl, t in cols:
            raw = np.ascontiguousarray(d).view(np.uint8).ravel()
            nraw = None if nl is None else np.ascontiguousarray(nl, dtype=np.uint8)
            w = abi.TYPE_WIDTH[t]
            ptrs = {}
            for kind in ("device", "device_off", "pinned"):
                pad = w if kind == "device_off" else 0
                td = torch.zeros(len(raw) + pad + 1, dtype=torch.uint8, device="cuda" if kind != "pinned" else "cpu")
                if kind == "pinned":
                    td = td.pin_memory()
                td[pad:pad + len(raw)] = torch.from_numpy(raw)
                tn = None
                if nraw is not None:
                    tn = torch.from_numpy(nraw.copy())
                    tn = tn.pin_memory() if kind == "pinned" else tn.cuda()
                self.keep += [td, tn]
                ptrs[kind] = (td.data_ptr() + pad, None if tn is None else tn.data_ptr())
            self.arena[off:off + len(raw)] = raw
            ptrs["arena"] = (self.arena.ctypes.data + off, None)
            off += len(raw) + 64 - len(raw) % 64
            if nraw is not None:
                self.arena[off:off + len(nraw)] = nraw
                ptrs["arena"] = (ptrs["arena"][0], self.arena.ctypes.data + off)
                off += len(nraw) + 64 - len(nraw) % 64
            ptrs["host"] = (raw.ctypes.data, None if nraw is None else nraw.ctypes.data)
            self.keep += [raw, nraw]
            for kind, p in ptrs.items():
                self.base[kind][s] = p
        ctx.host_register(self.arena)

    def chunk(self, kind, a, b, order):
        mem = {"device": abi.MEM_DEVICE, "device_off": abi.MEM_DEVICE, "pinned": abi.MEM_HOST_PINNED,
               "arena": abi.MEM_HOST_PINNED, "host": abi.MEM_HOST}[kind]
        cols = []
        for k in order:
            s, _, _, t = self.cols[k]
            d, nl = self.base[kind][s]
            cols.append((s, d + a * abi.TYPE_WIDTH[t], None if nl is None else nl + a, t))
        return Chunk(cols, num_rows=b - a, mem=mem)

    def close(self):
        self.ctx.sync()
        self.ctx.host_unregister(self.arena)


def _cuts(rng, n):
    cuts = [0]
    while cuts[-1] < n:
        size = int(rng.choice(SIZES)) if rng.random() < 0.5 else int(rng.integers(0, 9001))
        cuts.append(min(n, cuts[-1] + size))
    return cuts


def _lists(rng, cuts, max_chunks):
    """the chunk boundaries grouped into lists of 1..max_chunks chunks"""
    out, k = [], 0
    while k < len(cuts) - 1:
        m = int(rng.integers(1, max_chunks + 1))
        out.append(list(zip(cuts[k:k + m], cuts[k + 1:k + m + 1])))
        k += m
    return out


def _push_lists(r, copies, lists, rng):
    ncols = len(copies.cols)
    for lst in lists:
        chunks = []
        for a, b in lst:
            kind = KINDS[int(rng.integers(0, len(KINDS)))]
            order = list(range(ncols)) if rng.random() < 0.5 else list(rng.permutation(ncols))
            chunks.append(copies.chunk(kind, a, b, order))
        r.frag.push_chunks(chunks)


def _contiguous(gpu, ctx, c, cols=None):
    r = Run(gpu, ctx, c)
    try:
        r.push(cols or c.fact_cols, 0, c.n)
        return r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_plan_case_as_chunk_lists(gpu, ctx, name):
    c = build_case(name)
    rng = np.random.default_rng(sorted(CASES).index(name))
    cuts = _cuts(rng, c.n)
    want_plan, want_passed, want_out = _contiguous(gpu, ctx, c)
    r = Run(gpu, ctx, c)
    copies = Copies(ctx, c.fact_cols)
    try:
        # the first list holds the whole sampled prefix, so the plan is made from the same rows as the contiguous push's
        first = next(k for k, x in enumerate(cuts) if x >= min(c.n, 1 << 16))
        _push_lists(r, copies, [list(zip(cuts[:first], cuts[1:first + 1]))] + _lists(rng, cuts[first:], 40), rng)
        plan, passed, out = r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()
        copies.close()
    _check(c, out, passed, label=f"{name} as chunk lists")
    assert passed == want_passed
    for k in ("mode", "order", "num_stream_joins", "num_gather_passes", "bitmap_in_smem", "agg_in_smem", "pass_rate"):
        assert plan[k] == want_plan[k], (name, k, plan[k], want_plan[k])
    assert [t for t, _, _ in out] == [t for t, _, _ in want_out]
    assert sorted(len(d) for _, d, _ in out) == sorted(len(d) for _, d, _ in want_out)


def _gather_roundtrip(gpu, ctx, typ, dtype, phase_elems, sizes, kind):
    """SUM and COUNT of one column gathered from chunks that start `phase_elems` elements into their buffer"""
    import torch
    n = sum(sizes)
    rng = np.random.default_rng(n + phase_elems)
    vals = rng.integers(-1000, 1000, n).astype(dtype)
    agg = abi.make_agg_desc(fns=[(abi.AGG_SUM, typ, 90, [("col", 1)]), (abi.AGG_COUNT_STAR, 0, 91, None)])
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [], agg)
    keep, chunks, a = [], [], 0
    try:
        for sz in sizes:
            buf = np.zeros(sz + phase_elems + 1, dtype)
            buf[phase_elems:phase_elems + sz] = vals[a:a + sz]
            t = torch.from_numpy(buf)
            t = t.cuda() if kind == "device" else t.pin_memory()
            keep.append(t)
            ptr = t.data_ptr() + phase_elems * buf.itemsize
            chunks.append(Chunk([(1, ptr, None, typ)], num_rows=sz, mem=abi.MEM_DEVICE if kind == "device" else abi.MEM_HOST_PINNED))
            a += sz
        frag.push_chunks(chunks)
        got = frag.agg.result()
        ctx.sync()
    finally:
        frag.close()
    return int(got[0][2][0]), int(got[1][2][0]), int(vals.astype(np.int64).sum()), n


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("typ,dtype,phases", [(abi.TYPE_INT, np.int32, (0, 1, 2, 3)), (abi.TYPE_BIGINT, np.int64, (0, 1))])
def test_gather_alignment_phases(gpu, ctx, kind, typ, dtype, phases):
    # int32 sources at 0/4/8/12 bytes mod 16, int64 at 0/8; chunk sizes that are not multiples of 4 shift every later
    # destination, so source and destination phases disagree in every combination
    sizes = [4097, 1, 3, 4095, 6, 9001, 2, 4096, 5, 13]
    for ph in phases:
        s, cnt, want_s, want_n = _gather_roundtrip(gpu, ctx, typ, dtype, ph, sizes, kind)
        assert (s, cnt) == (want_s, want_n), (kind, typ, ph)


@pytest.mark.gpu
def test_null_columns_in_some_chunks(gpu, ctx):
    # the SUM input (slot 6) has a null column in some chunks of the list, one of them all NULL, and none in the others
    c = build_case("dense_at_limits", 120_001)
    rng = np.random.default_rng(7)
    cuts = [0, 4097, 8193, 20_000, 20_003, 40_000, 65_536, 65_537, 90_000, 120_001]
    with_nulls = {1, 3, 5, 7}
    nulls = np.zeros(c.n, np.uint8)
    for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        if k in with_nulls:
            nulls[a:b] = 1 if k == 5 else (rng.random(b - a) < 0.3)
    cols = [(s, d, nulls if s == 6 else nl, t) for s, d, nl, t in c.fact_cols]
    assert any(s == 6 for s, _, _, _ in cols)
    want_plan, want_passed, _ = _contiguous(gpu, ctx, c, cols)
    r = Run(gpu, ctx, c)
    copies = Copies(ctx, cols)
    try:
        chunks = []
        for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            ch = copies.chunk(KINDS[k % len(KINDS)], a, b, list(range(len(cols))))
            if k not in with_nulls:         # the chunks without a null column contribute zeros
                for q in range(ch.view.num_cols):
                    if ch._cols[q].slot_id == 6:
                        ch._cols[q].nulls = None
            chunks.append(ch)
        r.frag.push_chunks(chunks)
        plan, passed, out = r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()
        copies.close()
    assert passed == want_passed and plan["final_pass"] == want_plan["final_pass"] == "generic"
    _check(c, out, passed, cols, "null columns in some chunks")


@pytest.mark.gpu
def test_no_nulls_keeps_the_final_pass(gpu, ctx):
    # no chunk has a null column: the batch has none either, so the batched final pass stays eligible
    c = build_case("stream_bitmap_750k_carry", 120_001)
    want_plan, _, _ = _contiguous(gpu, ctx, c)
    r = Run(gpu, ctx, c)
    copies = Copies(ctx, c.fact_cols)
    try:
        cuts = list(range(0, c.n, 4096)) + [c.n]
        r.frag.push_chunks([copies.chunk(KINDS[k % 5], a, b, list(range(len(c.fact_cols)))) for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))])
        plan, passed, out = r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()
        copies.close()
    assert plan["final_pass"] == want_plan["final_pass"] == "dense-batched"
    _check(c, out, passed, label="no nulls")


@pytest.mark.gpu
def test_lifecycle_push_chunks_push_reset_finish(gpu, ctx):
    c = build_case("gather4_six_joins", 100_001)
    r = Run(gpu, ctx, c)
    copies = Copies(ctx, c.fact_cols)
    order = list(range(len(c.fact_cols)))
    try:
        r.frag.push_chunks([copies.chunk("host", 0, 0, order), copies.chunk("arena", 0, 0, order)])   # only empty chunks: plans
        assert r.plan()["mode"] in ("fused-cascade", "selection-vector-passes")
        r.frag.push_chunks([])
        r.frag.push_chunks([copies.chunk("pinned", 0, 30_000, order), copies.chunk("device_off", 30_000, 30_001, order)])
        r.push(c.fact_cols, 30_001, 60_000)
        r.frag.push_chunks([copies.chunk("arena", 60_000, c.n, order)])
        _check(c, r.result(), r.frag.rows_passed, label="mixed pushes")
        r.frag.reset()
        r.frag.push_chunks([copies.chunk("device", 0, 50_000, order), copies.chunk("host", 50_000, c.n, order)])
        passed = r.frag.rows_passed
        out = r.result()
        _check(c, out, passed, label="after reset")
        with pytest.raises(gpu.GpuError) as ei:
            r.frag.push_chunks([copies.chunk("device", 0, 100, order)])
        assert ei.value.code == abi.SR_ERR_STATE
    finally:
        r.close()
        copies.close()


@pytest.mark.gpu
def test_refusals_launch_nothing(gpu, ctx):
    from starrocks_b200.gpu import lib
    c = build_case("cascade_eager1", 20_000)
    r = Run(gpu, ctx, c)
    copies = Copies(ctx, c.fact_cols)
    order = list(range(len(c.fact_cols)))
    try:
        r.frag.push_chunks([copies.chunk("device", 0, 1000, order)])
        ctx.sync()

        def refused(chunks, code, n=None):
            before = ctx.launches
            views = (abi.sr_chunk_view * max(1, len(chunks)))(*[ch.view for ch in chunks])
            rc = lib().sr_fragment_push_chunks(r.frag.h, views, len(chunks) if n is None else n)
            assert rc == code, (rc, lib().sr_last_error(ctx.h))
            assert ctx.launches == before

        good = copies.chunk("device", 1000, 2000, order)
        refused([good], abi.SR_ERR_INVALID_ARGUMENT, n=-1)
        rc = lib().sr_fragment_push_chunks(r.frag.h, None, 2)
        assert rc == abi.SR_ERR_INVALID_ARGUMENT
        bad = copies.chunk("device", 1000, 2000, order)
        bad.view.mem = 7
        refused([good, bad], abi.SR_ERR_INVALID_ARGUMENT)
        neg = copies.chunk("device", 1000, 2000, order)
        neg.view.num_rows = -5
        refused([good, neg], abi.SR_ERR_INVALID_ARGUMENT)
        other = copies.chunk("device", 1000, 2000, order[:-1])                 # one slot missing
        refused([good, other], abi.SR_ERR_INVALID_ARGUMENT)
        retyped = copies.chunk("device", 1000, 2000, order)
        retyped._cols[0].type = abi.TYPE_BIGINT if retyped._cols[0].type != abi.TYPE_BIGINT else abi.TYPE_INT
        refused([good, retyped], abi.SR_ERR_INVALID_ARGUMENT)
        nodata = copies.chunk("host", 1000, 2000, order)
        nodata._cols[0].data = None
        refused([good, nodata], abi.SR_ERR_INVALID_ARGUMENT)
        mis = copies.chunk("device", 1000, 2000, order)
        wide = [q for q in range(mis.view.num_cols) if abi.TYPE_WIDTH[mis._cols[q].type] >= 4][0]
        mis._cols[wide].data = mis._cols[wide].data + 2
        refused([good, mis], abi.SR_ERR_INVALID_ARGUMENT)
        pageable = np.zeros(1 << 16, np.uint8)
        unpinned = copies.chunk("pinned", 1000, 2000, order)
        unpinned._cols[0].data = (pageable.ctypes.data + 63) & ~63
        refused([good, unpinned], abi.SR_ERR_INVALID_ARGUMENT)
        # the row total is refused before any buffer is read: these pointers lead nowhere
        huge = [Chunk([(s, 0x10000, None, t) for s, _, _, t in c.fact_cols], num_rows=0x7FFFFFF8, mem=abi.MEM_HOST_PINNED) for _ in range(2)]
        refused(huge, abi.SR_ERR_NOT_SUPPORTED)
    finally:
        r.close()
        copies.close()


@pytest.mark.gpu
def test_host_register_registry(gpu, ctx):
    a = np.zeros(1 << 20, np.uint8)
    base, n = a.ctypes.data, a.nbytes
    assert not ctx.host_is_mapped(base, 1)
    ctx.host_register(base, n)
    try:
        assert ctx.host_is_mapped(base, n) and ctx.host_is_mapped(base + n - 1, 1) and ctx.host_is_mapped(base, 0)
        assert not ctx.host_is_mapped(base - 1, 1) and not ctx.host_is_mapped(base, n + 1) and not ctx.host_is_mapped(base + n, 1)
        for p, sz in ((base, n), (base + 4096, 4096), (base - 4096, 8192), (base + n - 1, 4096)):
            with pytest.raises(gpu.GpuError) as ei:
                ctx.host_register(p, sz)
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT, (p - base, sz)
        with pytest.raises(gpu.GpuError) as ei:
            ctx.host_register(base + n + 4096, 0)
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
        with pytest.raises(gpu.GpuError) as ei:
            ctx.host_unregister(base + 4096)
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
    finally:
        ctx.host_unregister(base)
    assert not ctx.host_is_mapped(base, 1)
    with pytest.raises(gpu.GpuError) as ei:
        ctx.host_unregister(base)
    assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT
    # sr_host_alloc ranges are in the registry until sr_host_free; they cannot be unregistered
    import ctypes as C
    from starrocks_b200.gpu import lib
    p = C.c_void_p()
    ctx.check(lib().sr_host_alloc(ctx.h, 12345, C.byref(p)))
    assert ctx.host_is_mapped(p.value, 12345) and not ctx.host_is_mapped(p.value, 12346)
    with pytest.raises(gpu.GpuError):
        ctx.host_unregister(p.value)
    ctx.check(lib().sr_host_free(ctx.h, p))
    assert not ctx.host_is_mapped(p.value, 1)


@pytest.mark.gpu
def test_forwarding_fragment_sink(gpu, oracle):
    with tempfile.TemporaryDirectory() as d:
        binary = os.path.join(d, "frag_chunk_list_test")
        subprocess.check_call(["make", "-C", CPP, "-s", "-f", "frag_chunk_list_test.mk", f"OUT={binary}"])
        r = subprocess.run([binary, "300001"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "FRAG_CHUNK_LIST_OK" in r.stdout and "ForwardedChunks" in r.stdout
