"""The device columns each producer hands back in an `sr_chunk_out`, across the life of one handle.

A handle keeps its output columns across calls and only ever grows them.  Each test below drives one handle through
outputs of a few rows, many rows, a few rows again and zero rows, and checks every output against a reference: the
grow-only reuse path.  It also pins each producer's zero-row shape, because callers test `nulls != NULL` and so the
shape is part of the ABI:

- `sr_scan_filter` and `sr_chunk_deserialize`: every column has a data buffer; a nullable input keeps a null column.
- `sr_xchg_partition`: no data buffer; a nullable input gets an (empty) null column.
- `sr_agg_pull`: no row left means `data == nulls == NULL` in every column.
- `sr_agg_convert_to_states` / `sr_agg_push_selective`: group keys pass through as the input's own device pointers;
  COUNT states have no null column.
- `sr_join_probe`: the build columns of a LEFT OUTER join always have a null column, an empty build side included.
- `sr_join_probe_remain`: probe-side columns always have a null column; a build slot of an empty build side that was
  declared in `build_out_types` has `data == nulls == NULL`.

`sr_join_probe` is also driven by two probers in turn: prober 0's output must still read back after prober 1 probed.
"""
import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from starrocks_b200.rows import col_to_py, rand_nulls, rows_sorted

INT, BIGINT, DOUBLE = abi.TYPE_INT, abi.TYPE_BIGINT, abi.TYPE_DOUBLE
SIZES = (1000, 150_000, 37, 0)   # a few rows, many, a few again, none


def _py(data, nulls=None):
    return [None if nulls is not None and nulls[i] else x for i, x in enumerate(data.tolist())]


def _table(seed, n, kmax):
    """(k int32 in [0, kmax), v int64 with 20 % NULLs, its null bytes, d double)"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, max(kmax, 1), n).astype(np.int32)
    v = rng.integers(-10 ** 12, 10 ** 12, n).astype(np.int64)
    return k, v, rand_nulls(rng, n, 0.2), rng.standard_normal(n)


def shape(out):
    """(num_cols, mem, [(slot, type, has data buffer, has null column)])"""
    return out.num_cols, out.mem, [(c.slot_id, c.type, bool(c.data), bool(c.nulls)) for c in out.cols[:out.num_cols]]


def values(gpu, ctx, out):
    """the output's columns as lists of Python values (None = NULL)"""
    return [col_to_py(t, d, nl) for _, t, d, nl in gpu.chunk_out_to_host(ctx, out)]


def rows(gpu, ctx, out):
    return rows_sorted(values(gpu, ctx, out))


@pytest.mark.gpu
def test_scan_filter_output_columns(gpu, ctx):
    scan = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(1, abi.PRED_LT, 300)], out_slots=[2, 1, 3]))
    try:
        for step, n in enumerate(SIZES):
            k, v, vn, d = _table(step, n, 1000)
            out = scan.filter(Chunk([(1, k, None), (2, v, vn), (3, d, None)]))
            keep = k < 300
            assert shape(out) == (3, abi.MEM_DEVICE, [(2, BIGINT, True, True), (1, INT, True, False), (3, DOUBLE, True, False)])
            assert out.num_rows == int(keep.sum())
            assert values(gpu, ctx, out) == [_py(v[keep], vn[keep]), _py(k[keep]), _py(d[keep])], f"step {step}"
    finally:
        scan.close()


AGG_DESC = dict(group_slots=[1], group_types=[INT],
                fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)]), (abi.AGG_COUNT_STAR, 0, 11, None)])


def _ref_groups(k, v, vn):
    sums, counts = {}, {}
    for key, x, nl in zip(k.tolist(), v.tolist(), vn.tolist()):
        counts[key] = counts.get(key, 0) + 1
        if not nl:
            sums[key] = sums.get(key, 0) + x
    return rows_sorted([list(counts), [sums.get(key) for key in counts], list(counts.values())])


@pytest.mark.gpu
def test_agg_pull_output_columns(gpu, ctx):
    # a hash aggregate whose group count rises and falls between resets; each result is pulled on the device in two
    # slices (sr_agg_pull reads the emitted columns at its cursor), then once more with no row left
    a = gpu.Agg(ctx, abi.make_agg_desc(**AGG_DESC))
    try:
        for step, n in enumerate(SIZES):
            if step:
                a.reset()
            k, v, vn, _ = _table(10 + step, n, n // 2)
            a.push(Chunk([(1, k, None), (2, v, vn)]))
            a.finish()
            got = [[], [], []]
            groups = a.num_groups
            for max_rows in (max(groups // 3, 1), 1 << 62):
                out = a.pull(max_rows=max_rows, mem=abi.MEM_DEVICE)
                if out.num_rows:
                    assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, True, False), (10, BIGINT, True, True), (11, BIGINT, True, False)])
                for c, col in enumerate(values(gpu, ctx, out)):
                    got[c] += col
            assert rows_sorted(got) == _ref_groups(k, v, vn), f"step {step}"
            out = a.pull(mem=abi.MEM_DEVICE)
            assert out.num_rows == 0
            assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, False, False), (10, BIGINT, False, False), (11, BIGINT, False, False)])
    finally:
        a.close()


FIRST_PHASE = dict(group_slots=[1], group_types=[INT],
                   fns=[(abi.AGG_SUM, BIGINT, 10, [("col", 2)]), (abi.AGG_COUNT, BIGINT, 11, [("col", 2)])])
STATE_SHAPE = [(1, INT, True, False), (10, BIGINT, True, True), (11, BIGINT, True, False)]


def _device_chunk(k, v, vn):
    import torch
    dev = [torch.from_numpy(x.copy()).cuda() for x in (k, v, vn)]
    torch.cuda.synchronize()        # the library reads them on its own stream
    return Chunk([(1, dev[0], None, INT), (2, dev[1], dev[2], BIGINT)], num_rows=len(k), mem=abi.MEM_DEVICE), dev


@pytest.mark.gpu
def test_agg_convert_to_states_output_columns(gpu, ctx, oracle):
    desc = abi.make_agg_desc(**FIRST_PHASE)
    a = gpu.Agg(ctx, desc)
    try:
        for step, n in enumerate(SIZES):
            k, v, vn, _ = _table(20 + step, n, 500)
            ch, dev = _device_chunk(k, v, vn)
            out = a.convert_to_states(ch)
            # the group key is the input's own column (an empty tensor's is NULL)
            assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, n > 0, False)] + STATE_SHAPE[1:])
            assert out.num_rows == n
            assert (out.cols[0].data or 0) == dev[0].data_ptr()
            exp = [col_to_py(t, d, nl) for _, t, d, nl in oracle.convert_to_states(desc, Chunk([(1, k, None), (2, v, vn)]))]
            assert values(gpu, ctx, out) == exp, f"step {step}"
    finally:
        a.close()


@pytest.mark.gpu
def test_agg_push_selective_output_columns(gpu, ctx, oracle):
    # a hash table warmed with keys [0, 400): rows of other keys are streamed out, compacted into the handle's own columns
    desc = abi.make_agg_desc(**FIRST_PHASE)
    a, ref = gpu.Agg(ctx, desc), oracle.Agg(desc)
    try:
        warm = np.arange(400, dtype=np.int32)
        for agg in (a, ref):
            agg.push(Chunk([(1, warm, None), (2, warm.astype(np.int64), None)]))
        for step, n in enumerate(SIZES):
            k, v, vn, _ = _table(30 + step, n, 500)
            host = Chunk([(1, k, None), (2, v, vn)])
            sel = ref.streaming_selection(host) == 1
            out = a.push_selective(host)
            assert shape(out) == (3, abi.MEM_DEVICE, STATE_SHAPE)
            assert out.num_rows == int(sel.sum())
            exp = [col_to_py(t, d[sel], None if nl is None else nl[sel]) for _, t, d, nl in oracle.convert_to_states(desc, host)]
            assert values(gpu, ctx, out) == exp, f"step {step}"
            ch, dev = _device_chunk(k, v, vn)
            if 0 < sel.sum() < n:
                out = a.push_selective(ch)
                assert out.cols[0].data != dev[0].data_ptr()      # compacted: the handle's own column
                assert values(gpu, ctx, out) == exp, f"step {step}, device input"
    finally:
        a.close()


@pytest.mark.gpu
def test_xchg_partition_output_columns(gpu, ctx):
    nch = 4
    x = gpu.Xchg(ctx, abi.make_part_desc([1], nch))
    try:
        for step, n in enumerate(SIZES):
            k, v, vn, d = _table(40 + step, n, 1 << 30)
            ch = Chunk([(1, k, None), (2, v, vn), (3, d, None)])
            out, offs = x.partition(ch)
            assert out.num_rows == n and offs[0] == 0 and offs[-1] == n
            if n == 0:
                assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, False, False), (2, BIGINT, False, True), (3, DOUBLE, False, False)])
                assert list(offs) == [0] * (nch + 1)
                continue
            assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, True, False), (2, BIGINT, True, True), (3, DOUBLE, True, False)])
            got = list(zip(*values(gpu, ctx, out)))
            _, channel = x.hash(ch)
            inp = list(zip(_py(k), _py(v, vn), _py(d)))
            for c in range(nch):
                exp = [r for r, cc in zip(inp, channel.tolist()) if cc == c]
                assert rows_sorted(list(zip(*got[offs[c]:offs[c + 1]]))) == rows_sorted(list(zip(*exp))), f"step {step} channel {c}"
    finally:
        x.close()


@pytest.mark.gpu
def test_serde_output_columns(gpu, ctx):
    s = gpu.Serde(ctx)
    try:
        for step, n in enumerate(SIZES):
            k, v, vn, d = _table(50 + step, n, 1000)
            payload, meta = gpu.chunk_serialize(ctx, Chunk([(1, k, None), (2, v, vn), (3, d, None)]))
            out = s.deserialize(payload, meta)
            assert shape(out) == (3, abi.MEM_DEVICE, [(1, INT, True, False), (2, BIGINT, True, True), (3, DOUBLE, True, False)])
            assert out.num_rows == n
            assert values(gpu, ctx, out) == [_py(k), _py(v, vn), _py(d)], f"step {step}"
    finally:
        s.close()


# joins: build (100: key, 101: nullable BIGINT payload), probe (1: key, 2: BIGINT); output probe 2, 1 then build 101, 100
NB = 50_000
JOIN_OUT = dict(build_out=[101, 100], probe_out=[2, 1])


def _build(seed=60):
    rng = np.random.default_rng(seed)
    bk = rng.permutation(4 * NB)[:NB].astype(np.int32)
    bv = rng.integers(-10 ** 12, 10 ** 12, NB).astype(np.int64)
    return bk, bv, rand_nulls(rng, NB, 0.2)


def _join(gpu, ctx, jt, bk=None, bv=None, bvn=None, **kw):
    j = gpu.Join(ctx, abi.make_join_desc(jt, [100], [1], [INT], **JOIN_OUT, **kw))
    if bk is not None:
        j.append_build(Chunk([(100, bk, None), (101, bv, bvn)]))
    j.build_finish()
    return j


def _probe(seed, n):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 4 * NB, n).astype(np.int32), rng.integers(-10 ** 12, 10 ** 12, n).astype(np.int64)


def _ref_probe(jt, build, pk, pv):
    bk, bv, bvn = build
    payload = dict(zip(bk.tolist(), _py(bv, bvn)))
    out = []
    for key, x in zip(pk.tolist(), pv.tolist()):
        if key in payload:
            out.append((x, key, payload[key], key))
        elif jt == abi.JOIN_LEFT_OUTER:
            out.append((x, key, None, None))
    return rows_sorted(list(zip(*out))) if out else []


@pytest.mark.gpu
@pytest.mark.parametrize("jt", [abi.JOIN_INNER, abi.JOIN_LEFT_OUTER], ids=["inner", "left_outer"])
def test_join_probe_output_columns_two_probers(gpu, ctx, jt):
    build = _build()
    j = _join(gpu, ctx, jt, *build)
    outer = jt == abi.JOIN_LEFT_OUTER
    want = (4, abi.MEM_DEVICE, [(2, BIGINT, True, False), (1, INT, True, False), (101, BIGINT, True, True), (100, INT, True, outer)])
    try:
        for step, n in enumerate(SIZES):
            m = SIZES[(step + 1) % len(SIZES)]      # prober 1 runs one size ahead
            p0, p1 = _probe(70 + step, n), _probe(80 + step, m)
            out0 = j.probe(Chunk([(1, p0[0], None), (2, p0[1], None)]), prober_id=0)
            out1 = j.probe(Chunk([(1, p1[0], None), (2, p1[1], None)]), prober_id=1)
            assert shape(out0) == want and shape(out1) == want
            assert rows(gpu, ctx, out0) == _ref_probe(jt, build, *p0), f"step {step}, prober 0 after prober 1"
            assert rows(gpu, ctx, out1) == _ref_probe(jt, build, *p1), f"step {step}, prober 1"
    finally:
        j.close()


@pytest.mark.gpu
@pytest.mark.parametrize("jt", [abi.JOIN_INNER, abi.JOIN_LEFT_OUTER], ids=["inner", "left_outer"])
def test_join_probe_of_empty_build_side(gpu, ctx, jt):
    # no build chunk: the build columns take their declared types and read the all-zero row 0
    j = _join(gpu, ctx, jt, build_out_types=[BIGINT, INT])
    outer = jt == abi.JOIN_LEFT_OUTER
    try:
        for step, n in enumerate(SIZES):
            pk, pv = _probe(90 + step, n)
            out = j.probe(Chunk([(1, pk, None), (2, pv, None)]))
            assert shape(out) == (4, abi.MEM_DEVICE, [(2, BIGINT, True, False), (1, INT, True, False), (101, BIGINT, True, outer),
                                                      (100, INT, True, outer)])
            exp = rows_sorted([_py(pv), _py(pk), [None] * n, [None] * n]) if outer else []
            assert rows(gpu, ctx, out) == exp, f"step {step}"
    finally:
        j.close()


def _ref_remain(build, matched, with_probe_cols):
    bk, bv, bvn = build
    keep = np.array([(key in matched) != with_probe_cols for key in bk.tolist()], dtype=bool)
    n = int(keep.sum())
    return rows_sorted(([[None] * n] * 2 if with_probe_cols else []) + [_py(bv[keep], bvn[keep]), _py(bk[keep])])


@pytest.mark.gpu
def test_join_probe_remain_output_columns(gpu, ctx):
    # RIGHT OUTER: the unmatched build rows shrink from all to none; RIGHT SEMI: the matched ones grow from none.  Each
    # handle calls probe_remain after every probe.
    build = _build()
    bk = build[0]
    outer = _join(gpu, ctx, abi.JOIN_RIGHT_OUTER, *build, probe_out_types=[BIGINT, INT])
    semi = _join(gpu, ctx, abi.JOIN_RIGHT_SEMI, *build)
    try:
        matched = set()
        for step, keys in enumerate((bk[:0], bk[:40], bk[: NB - 30], bk)):
            pv = np.arange(len(keys), dtype=np.int64)
            for j in (outer, semi):
                j.probe(Chunk([(1, keys, None), (2, pv, None)]))
            matched.update(keys.tolist())
            out = outer.probe_remain()
            assert shape(out) == (4, abi.MEM_DEVICE, [(2, BIGINT, True, True), (1, INT, True, True), (101, BIGINT, True, True),
                                                      (100, INT, True, False)])
            assert out.num_rows == NB - len(matched)
            assert rows(gpu, ctx, out) == _ref_remain(build, matched, True), f"right outer, step {step}"
            out = semi.probe_remain()
            assert shape(out) == (2, abi.MEM_DEVICE, [(101, BIGINT, True, True), (100, INT, True, False)])
            assert out.num_rows == len(matched)
            assert rows(gpu, ctx, out) == _ref_remain(build, matched, False), f"right semi, step {step}"
    finally:
        outer.close()
        semi.close()


@pytest.mark.gpu
def test_join_probe_remain_of_empty_build_side(gpu, ctx):
    j = _join(gpu, ctx, abi.JOIN_FULL_OUTER, build_out_types=[BIGINT, INT], probe_out_types=[BIGINT, INT])
    try:
        out = j.probe_remain()
        assert out.num_rows == 0
        assert shape(out) == (4, abi.MEM_DEVICE, [(2, BIGINT, True, True), (1, INT, True, True), (101, BIGINT, False, False),
                                                  (100, INT, False, False)])
    finally:
        j.close()
