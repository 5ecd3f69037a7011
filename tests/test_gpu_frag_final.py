"""The batched final pass of selection-vector mode (k_frag_final_dense) and its slot-digit directories, against the
oracle.  Each case is a small star join that the plan routes through the final pass; `final_pass` in the fragment's
plan says which kernel ran, so a case that must fall back to the generic kernel is checked as well.
"""
import numpy as np
import pytest

from starrocks_b200 import abi, ssb
from starrocks_b200.abi import Chunk
from tests.helpers import assert_rows_equal, gpu_rows, oracle_rows

pytestmark = pytest.mark.gpu

N = 400_000
P1_RANGE = (0, 6)


def _star(case, rng):
    """fact slots 0..5: key of A, key of B, key of C, two measures, a small fact column.  A filters (5 % pass) and is
    streamed; B (payload: slots 21, 22) and C (no payload) pass >= 90 % and are handled by the final pass."""
    fact = Chunk([(0, rng.integers(0, 1000, N, dtype=np.int32), None), (1, rng.integers(0, 2000, N, dtype=np.int32), None),
                  (2, rng.integers(0, 3000, N, dtype=np.int32), None), (3, rng.integers(-10**6, 10**6, N, dtype=np.int32), None),
                  (4, rng.integers(0, 10**5, N, dtype=np.int32), None), (5, rng.integers(0, 10, N, dtype=np.int32), None)])
    dim_a = Chunk([(10, np.arange(0, 50, dtype=np.int32), None)])
    kb = np.arange(2000, dtype=np.int32)
    if case == "miss":
        kb = kb[rng.random(2000) >= 0.07]                 # ~7 % of the fact rows find no B row in the final pass
    rng.shuffle(kb)
    p1 = rng.integers(0, 10 if case == "out_of_range" else 7, len(kb), dtype=np.int32)
    p1_nulls = (rng.random(len(kb)) < 0.1).astype(np.uint8) if case.startswith("nullable_payload") else None
    dim_b = Chunk([(20, kb, None), (21, p1, p1_nulls), (22, rng.integers(0, 4, len(kb), dtype=np.int32), None)])
    kc = np.arange(3000, dtype=np.int32)
    kc = kc[rng.random(3000) >= 0.03]
    dim_c = Chunk([(30, kc, None)])
    return fact, [dim_a, dim_b, dim_c]


def _agg_desc(case):
    fns = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 3)]), (abi.AGG_COUNT_STAR, 0, 41, None), (abi.AGG_MIN, abi.TYPE_INT, 42, [("col", 4)]),
           (abi.AGG_MAX, abi.TYPE_INT, 43, [("col", 4)]), (abi.AGG_COUNT, abi.TYPE_BIGINT, 44, [("col", 3)])]
    keys, types, ranges, nullable = [21], [abi.TYPE_INT], [P1_RANGE], None
    if case == "fact_group_key":
        keys, types, ranges = [21, 5], [abi.TYPE_INT] * 2, [P1_RANGE, (0, 9)]
    elif case == "two_keys_one_join":
        keys, types, ranges = [21, 22], [abi.TYPE_INT] * 2, [P1_RANGE, (0, 3)]
    elif case in ("nullable_payload_declared", "nullable_key_no_nulls"):
        nullable = [True]
    elif case == "fallback_payload_sum":
        fns = fns + [(abi.AGG_SUM, abi.TYPE_BIGINT, 45, [("col", 21)])]
    return abi.make_agg_desc(keys, types, fns=fns, ranges=ranges, group_nullable=nullable)


CASES = ["basic", "out_of_range", "nullable_payload", "nullable_payload_declared", "nullable_key_no_nulls", "fact_group_key",
         "two_keys_one_join", "miss", "fallback_payload_sum"]


@pytest.mark.parametrize("case", CASES)
def test_final_pass_dense_parity(gpu, ctx, oracle, case):
    rng = np.random.default_rng(100 + CASES.index(case))
    fact, dims = _star(case, rng)
    descs = [abi.make_join_desc(abi.JOIN_INNER, [10 * (k + 1)], [k], [abi.TYPE_INT]) for k in range(3)]
    payload = [[], [21, 22] if case == "two_keys_one_join" else [21], []]
    gj = [gpu.Join(ctx, d) for d in descs]
    oj = [oracle.Join(d) for d in descs]
    frag = None
    try:
        for g, o, ch in zip(gj, oj, dims):
            g.append_build(ch)
            o.append_build(ch)
            g.build_finish()
            o.build()
        agg_desc = _agg_desc(case)
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [(g, k, payload[k]) for k, g in enumerate(gj)], agg_desc, mode=2)
        half = N // 2 + 7
        for lo, hi in ((0, half), (half, N)):
            frag.push(Chunk([(sl, d[lo:hi], None if nl is None else nl[lo:hi]) for sl, d, nl in fact.columns()]))
        plan = frag.plan()
        assert plan["mode"] == "selection-vector-passes" and plan["num_stream_joins"] == 1 and plan["num_gather_passes"] == 0
        assert plan["final_pass"] == ("generic" if case == "fallback_payload_sum" else "dense-batched")
        ores, opassed = oracle.fragment_run(abi.ScanDesc(), [(o, k, payload[k]) for k, o in enumerate(oj)], agg_desc, fact, num_threads=3)
        assert frag.rows_passed == opassed > 10_000
        if case == "out_of_range":
            # payloads 7..9 lie outside the declared range: the rows pass the joins (counted above), reach no group,
            # and the aggregate reports the broken range when its result is asked for
            with pytest.raises(gpu.GpuError) as ei:
                frag.agg.result()
            assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT and "declared" in str(ei.value)
            return
        got = gpu_rows(frag.agg.result())
        assert_rows_equal(got, oracle_rows(ores))
        if case.startswith("nullable_payload"):
            assert got[0][0] is None
    finally:
        if frag:
            frag.close()
        for g in gj:
            g.close()


@pytest.mark.parametrize("pinned", [False, True])
def test_final_pass_dense_q41(gpu, ctx, oracle, pinned):
    # SSB Q4.1 takes the batched final pass, with the customer key carried through the selection vector for pinned input
    import torch
    dims = ssb.gen_dims(0.1)
    lo = ssb.gen_lineorder(0.1, n=600_000)
    gjoins, gkeep = ssb.build_dims(gpu, dims, ssb.dim_plans_q41(), ctx=ctx)
    ojoins, okeep = ssb.build_dims(oracle, dims, ssb.dim_plans_q41())
    agg_desc = ssb.q41_agg_desc()
    frag = gpu.Fragment(ctx, abi.ScanDesc(), gjoins, agg_desc, mode=2)
    try:
        if pinned:
            pin = {k: torch.from_numpy(lo[k]).pin_memory() for k in ssb.Q41_FACT_COLS}
            frag.push(Chunk([(ssb.LO_SLOTS[k], pin[k].data_ptr(), None, abi.TYPE_INT) for k in ssb.Q41_FACT_COLS],
                            num_rows=len(lo[ssb.Q41_FACT_COLS[0]]), mem=abi.MEM_HOST_PINNED))
            ctx.sync()
            del pin
        else:
            frag.push(ssb.fact_chunk(lo, ssb.Q41_FACT_COLS))
        assert frag.plan()["final_pass"] == "dense-batched"
        got = gpu_rows(frag.agg.result())
        ores, opassed = oracle.fragment_run(abi.ScanDesc(), ojoins, agg_desc, ssb.fact_chunk(lo, ssb.Q41_FACT_COLS), num_threads=4)
        assert frag.rows_passed == opassed > 0
        assert_rows_equal(got, oracle_rows(ores))
        assert len(got) == 35
    finally:
        frag.close()
        for j, _, _ in gjoins:
            j.close()
        for item in gkeep:
            item[0].close()
