"""The aggregate's state arrays across their lifecycle: reset and a second stream for every table kind, an input that turns
nullable after the tables were laid out, merges that start counting non-NULL inputs, and the dense-state export's list."""
import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from tests.helpers import assert_rows_equal, gpu_rows, oracle_rows, rand_nulls

pytestmark = pytest.mark.gpu

# MIN / MAX start from non-zero values, the DECIMAL64 sum keeps a second word (acc1), the sum over the nullable column 3
# counts its non-NULL inputs (accn)
FNS = [(abi.AGG_COUNT_STAR, 0, 20, None), (abi.AGG_MIN, abi.TYPE_BIGINT, 21, [("col", 2)]), (abi.AGG_MAX, abi.TYPE_BIGINT, 22, [("col", 2)]),
       (abi.AGG_SUM, abi.TYPE_DECIMAL64, 23, [("col", 4)]), (abi.AGG_SUM, abi.TYPE_INT, 24, [("col", 3)]),
       (abi.AGG_AVG, abi.TYPE_DOUBLE, 25, [("col", 5)]), (abi.AGG_MIN, abi.TYPE_DOUBLE, 26, [("col", 5)])]
AVG = 5   # position of the AVG in FNS: its result column, nk + AVG, is compared with a tolerance (double sums)


def _desc(kind):
    if kind == "nogroup":
        return abi.make_agg_desc(fns=FNS), 0
    if kind == "dense_smem":      # 7 x 7 slots: the state fits shared memory
        return abi.make_agg_desc([0, 1], [abi.TYPE_INT, abi.TYPE_INT], fns=FNS, ranges=[(0, 6), (-3, 3)]), 2
    if kind == "dense_global":    # 7 x 1000 slots, over 40 KB of state: accumulated in global memory
        return abi.make_agg_desc([0, 1], [abi.TYPE_INT, abi.TYPE_INT], fns=FNS, ranges=[(0, 6), (-3, 996)]), 2
    return abi.make_agg_desc([0, 2], [abi.TYPE_INT, abi.TYPE_BIGINT], fns=FNS), 2   # hash: the int64 value is a key too


def _stream(kind, n, seed, nullable=True, null_k0=False):
    rng = np.random.default_rng(seed)
    k0 = rng.integers(0, 7, n, dtype=np.int32)
    k1 = rng.integers(-3, 997 if kind == "dense_global" else 4, n).astype(np.int32)
    k2 = rng.integers(-10**12, 10**12, n, dtype=np.int64)
    if kind.startswith("hash"):
        k2 = k2 % (n // 3 + 1)    # about three rows per group
    v3 = rng.integers(-10**6, 10**6, n, dtype=np.int32)
    dec = rng.integers(-2**62, 2**62, n, dtype=np.int64)
    vd = rng.normal(10, 5, n)
    nulls = rand_nulls(rng, n, 0.2) if nullable else None
    if null_k0:                   # every group with k0 == 0 sees only NULLs in column 3: its SUM is NULL
        nulls[k0 == 0] = 1
    return Chunk([(0, k0, None), (1, k1, None), (2, k2, None), (3, v3, nulls),
                  (4, dec, None, abi.TYPE_DECIMAL64), (5, vd, None)])


@pytest.mark.parametrize("kind", ["dense_smem", "dense_global", "hash_direct", "hash_partitioned", "nogroup"])
def test_agg_reset_then_other_stream(gpu, ctx, oracle, monkeypatch, kind):
    # reset() must bring every state array back to its initial value: the second result is the second stream's alone
    if kind == "hash_partitioned":
        monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", "100000")
    n = 300_000 if kind == "hash_partitioned" else 40_000
    d, nk = _desc(kind)
    first, second = _stream(kind, n, 1), _stream(kind, n, 2)
    ga = gpu.Agg(ctx, d)
    try:
        o1, o2 = oracle.Agg(d), oracle.Agg(d)
        ga.push(first)
        o1.push(first)
        assert_rows_equal(gpu_rows(ga.result()), oracle_rows(o1), float_cols=(nk + AVG,))
        ga.reset()
        ga.push(second)
        o2.push(second)
        assert_rows_equal(gpu_rows(ga.result()), oracle_rows(o2), float_cols=(nk + AVG,))
    finally:
        ga.close()


@pytest.mark.parametrize("kind", ["dense_smem", "hash_direct", "hash_grows"])
def test_agg_input_turns_nullable_then_grow_and_reset(gpu, ctx, oracle, kind):
    # column 3 has no NULLs in the first push (no non-NULL count kept for the SUM over it), NULLs in the second; hash_grows:
    # the table then grows past its first 2^21 slots.  After a reset a third stream is aggregated alone; in it the groups
    # with k0 == 0 see only NULLs, so a non-NULL count the reset left behind would turn their NULL SUM into a value.
    d, nk = _desc("dense_smem" if kind == "dense_smem" else "hash_direct")
    ga, oa = gpu.Agg(ctx, d), oracle.Agg(d)
    try:
        chunks = [_stream(kind, 30_000, 3, nullable=False), _stream(kind, 30_000, 4)]
        if kind == "hash_grows":
            chunks.append(_stream(kind, 1_500_000, 5))     # ~1.2 M groups: over the 2^20-group limit of the first table
        for ch in chunks:
            ga.push(ch)
            oa.push(ch)
        if kind == "hash_grows":
            assert ga.current_groups() > 1 << 20
        assert_rows_equal(gpu_rows(ga.result()), oracle_rows(oa), float_cols=(nk + AVG,))
        ga.reset()
        third, o3 = _stream(kind, 30_000, 7, null_k0=True), oracle.Agg(d)
        ga.push(third)
        o3.push(third)
        assert_rows_equal(gpu_rows(ga.result()), oracle_rows(o3), float_cols=(nk + AVG,))
    finally:
        ga.close()


@pytest.mark.parametrize("kind", ["dense_smem", "hash_direct"])
@pytest.mark.parametrize("case", ["into_never_pushed", "only_source_counts"])
def test_agg_merge_starts_non_null_counts(gpu, ctx, oracle, kind, case):
    # into_never_pushed: the target adopts the layout of a source whose input turned nullable after its first push.
    # only_source_counts: the target's input never had a NULL, the source's had from the start.
    d, nk = _desc(kind)
    a, o, oa = gpu.Agg(ctx, d), gpu.Agg(ctx, d), oracle.Agg(d)
    try:
        if case == "into_never_pushed":
            src = [_stream(kind, 20_000, 8, nullable=False), _stream(kind, 20_000, 9)]
            dst = []
        else:
            src = [_stream(kind, 20_000, 10)]
            dst = [_stream(kind, 20_000, 11, nullable=False)]
        for ch in src:
            o.push(ch)
            oa.push(ch)
        for ch in dst:
            a.push(ch)
            oa.push(ch)
        o.finish()
        a.merge(o)
        after = _stream(kind, 20_000, 12)   # pushed with the layout the target now has (into_never_pushed: its accn in its slab)
        a.push(after)
        oa.push(after)
        assert_rows_equal(gpu_rows(a.result()), oracle_rows(oa), float_cols=(nk + AVG,))
    finally:
        a.close()
        o.close()


B, D, SUM, MIN, MAX = abi.TYPE_BIGINT, abi.TYPE_DOUBLE, abi.STATE_REDUCE_SUM, abi.STATE_REDUCE_MIN, abi.STATE_REDUCE_MAX


# int_min: MIN over int, MAX over double; else the other way round (eight functions at most)
@pytest.mark.parametrize("int_min", [True, False])
def test_agg_dense_state_list(gpu, ctx, oracle, int_min):
    # the exported list: one array per state word in table order, each with its element type and reduce op, back to back
    # in one slab; after an input turns nullable its non-NULL count joins the list right after that function's state
    ext = [(abi.AGG_MIN, abi.TYPE_INT, 25, [("col", 2)]), (abi.AGG_MAX, abi.TYPE_DOUBLE, 26, [("col", 5)])] if int_min else \
          [(abi.AGG_MIN, abi.TYPE_DOUBLE, 25, [("col", 5)]), (abi.AGG_MAX, abi.TYPE_INT, 26, [("col", 2)])]
    fns = [(abi.AGG_COUNT_STAR, 0, 20, None), (abi.AGG_COUNT, abi.TYPE_INT, 21, [("col", 3)]), (abi.AGG_SUM, abi.TYPE_INT, 22, [("col", 3)]),
           (abi.AGG_SUM, abi.TYPE_DOUBLE, 23, [("col", 5)]), (abi.AGG_AVG, abi.TYPE_INT, 24, [("col", 2)])] + ext
    d = abi.make_agg_desc([0, 1], [abi.TYPE_INT, abi.TYPE_INT], fns=fns, ranges=[(0, 6), (-3, 3)])
    rng = np.random.default_rng(12)
    n = 20_000

    def chunk(null2):
        return Chunk([(0, rng.integers(0, 7, n, dtype=np.int32), None), (1, rng.integers(-3, 4, n, dtype=np.int32), None),
                      (2, rng.integers(-1000, 1000, n, dtype=np.int32), rand_nulls(rng, n, 0.3) if null2 else None),
                      (3, rng.integers(-1000, 1000, n, dtype=np.int32), rand_nulls(rng, n, 0.2)), (5, rng.normal(0, 1, n), None)])

    ga, oa = gpu.Agg(ctx, d), oracle.Agg(d)
    try:
        ch = chunk(False)
        ga.push(ch)
        oa.push(ch)
        arrays = ga.dense_state()
        #          cnt        COUNT      SUM int + accn (nullable input)  SUM dbl    AVG        MIN        MAX
        expect = [(B, SUM), (B, SUM), (B, SUM), (B, SUM),             (D, SUM), (D, SUM), (B, MIN), (B, MAX)]
        assert [(t, r) for _, _, t, r in arrays] == expect
        assert all(c == 49 for _, c, _, _ in arrays)
        assert all(arrays[i + 1][0] == arrays[i][0] + 8 * 49 for i in range(len(arrays) - 1))
        ch = chunk(True)   # column 2 turns nullable: AVG and the integer MIN / MAX over it start counting their non-NULL inputs
        ga.push(ch)
        oa.push(ch)
        arrays = ga.dense_state()
        late = (6, 8) if int_min else (6, 9)
        expect = expect[:6] + [(B, SUM)] + ([(B, MIN), (B, SUM), (B, MAX)] if int_min else [(B, MIN), (B, MAX), (B, SUM)])
        assert [(t, r) for _, _, t, r in arrays] == expect
        slab = [a for i, a in enumerate(arrays) if i not in late]
        assert all(slab[i + 1][0] == slab[i][0] + 8 * 49 for i in range(len(slab) - 1))
        assert_rows_equal(gpu_rows(ga.result()), oracle_rows(oa), float_cols=(2 + 3, 2 + 4))
    finally:
        ga.close()
