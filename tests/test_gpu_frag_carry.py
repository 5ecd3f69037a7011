"""The streamed join key carried through the selection vector (selection-vector mode): the streaming pass stores the key
of the streamed join whose build row the final pass needs next to each surviving row id, and the final pass reads it
from there instead of gathering it from the fact column again.  Every case runs on fact columns in device memory (and
one on pinned host memory) and is compared with the oracle; the cases choose pass rates and layouts so that the carried
join is the first or the second vector-loaded test or a later predicated test, with and without a gather pass, through
the dense and the generic final pass, the tests kernel and the generic streaming kernel, and over a ragged last tile.
"""
import numpy as np
import pytest

from starrocks_b200 import abi, ssb
from starrocks_b200.abi import Chunk
from tests.helpers import assert_rows_equal, gpu_rows, oracle_rows

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
N = 4096 * 97 + 1237  # not a multiple of the streaming pass's 4096-row tile: the last tile is ragged
PAY_RANGE = (0, 6)
# fact slots: 0 carried join key, 1 other streamed join key, 2 key of a join that passes >= 90 %, 3 / 4 measures,
# 5 scan-predicate column.  Build slots: 10 carried key, 11 its group payload, 20 other key, 30 third key.
FNS = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 3)]), (abi.AGG_COUNT_STAR, 0, 41, None), (abi.AGG_MIN, abi.TYPE_INT, 42, [("col", 4)]),
       (abi.AGG_MAX, abi.TYPE_INT, 43, [("col", 4)])]

# case -> (rows, carried join pass rate, other join pass rate, carried key range low end, scan predicate pass rate)
CASES = {
    "carried_first": (N, 0.10, 0.25, 1000, None),       # most selective: test 0
    "carried_second": (N, 0.25, 0.10, 1000, None),      # test 1
    "carried_later": (N, 0.10, 0.25, 1000, 0.05),       # after a 5 % scan predicate: a predicated test, not vector-loaded
    "keys_at_int32_max": (N, 0.10, 0.25, I32_MAX - 1999, None),
    "keys_at_int32_min": (N, 0.25, 0.10, I32_MIN, None),
    "one_ragged_tile": (3001, 0.10, 0.25, 1000, None),  # fewer rows than one tile
    "unaligned": (N, 0.25, 0.10, 1000, None),           # columns 4 bytes off 16: the generic streaming kernel
    "generic_final": (N, 0.25, 0.10, 1000, None),       # the payload is also an aggregate input: the generic final pass
    "pinned": (N, 0.25, 0.10, 1000, None),
}


def _keys_hitting(rng, n, rate, keys, lo):
    """n fact keys: a `rate` share drawn from the build keys, the rest misses -- absent keys inside the build range
    [lo, lo + 1999] and keys outside it, the int32 extremes among them"""
    inside = np.setdiff1d(np.arange(lo, lo + 2000, dtype=np.int64), keys)
    outside = np.array([v for v in (lo - 1, lo + 2000, I32_MIN, I32_MIN + 1, I32_MAX - 1, I32_MAX, 0, -1)
                        if I32_MIN <= v <= I32_MAX and not lo <= v < lo + 2000], dtype=np.int64)
    out = np.where(rng.random(n) < 0.5, inside[rng.integers(0, len(inside), n)], outside[rng.integers(0, len(outside), n)])
    hit = rng.random(n) < rate
    out[hit] = keys[rng.integers(0, len(keys), int(hit.sum()))]
    return out.astype(np.int32)


def _star(case, rng):
    n, rate_c, rate_o, lo, pred_rate = CASES[case]
    kc = (lo + np.concatenate([[0, 1999], 1 + rng.choice(1998, 1398, replace=False)])).astype(np.int32)  # both ends of the range
    pay = rng.integers(PAY_RANGE[0], PAY_RANGE[1] + 1, len(kc), dtype=np.int32)
    ko = np.arange(5000, dtype=np.int32)
    k3 = np.arange(3000, dtype=np.int32)
    k3 = k3[rng.random(3000) >= 0.03]
    fc = _keys_hitting(rng, n, rate_c, kc, lo)
    for p in (0, n // 2, n - 8):  # both ends of the build range and the int32 extremes in the first, a middle and the last tile
        fc[p:p + 8] = [lo, lo + 1999, I32_MIN, I32_MAX, lo, lo + 1999, lo, lo + 1999]
    fo = np.where(rng.random(n) < rate_o, rng.integers(0, 5000, n), rng.integers(5000, 10**6, n)).astype(np.int32)
    fo[:8] = fo[n // 2:n // 2 + 8] = fo[n - 8:] = 7  # let the planted rows of fc through the other join
    f3 = rng.integers(0, 3000, n, dtype=np.int32)
    pred = np.where(rng.random(n) < (pred_rate or 1.0), 1, 2).astype(np.int32)
    pred[:8] = pred[n // 2:n // 2 + 8] = pred[n - 8:] = 1
    fact = [(0, fc), (1, fo), (2, f3), (3, rng.integers(-10**6, 10**6, n, dtype=np.int32)),
            (4, rng.integers(-(1 << 30), 1 << 30, n, dtype=np.int32)), (5, pred)]
    dims = [Chunk([(10, kc, None), (11, pay, None)]), Chunk([(20, ko, None)]), Chunk([(30, k3, None)])]
    scan = abi.ScanDesc([abi.make_pred(5, abi.PRED_EQ, 1)]) if pred_rate is not None else abi.ScanDesc()
    fns = FNS + ([(abi.AGG_SUM, abi.TYPE_BIGINT, 44, [("col", 11)])] if case == "generic_final" else [])
    agg = abi.make_agg_desc([11], [abi.TYPE_INT], fns=fns, ranges=[PAY_RANGE])
    return fact, dims, scan, agg


def _device_chunk(torch, fact, offset):
    """the fact columns in device memory; offset > 0 places each column `offset` elements into a larger buffer"""
    keep = []
    for slot, a in fact:
        buf = torch.empty(len(a) + offset, dtype=torch.int32, device="cuda")
        buf[offset:] = torch.from_numpy(a).cuda()
        keep.append((slot, buf[offset:], None, abi.TYPE_INT))
    return Chunk(keep, mem=abi.MEM_DEVICE)


def _push(torch, frag, fact, case):
    n = len(fact[0][1])
    if case == "pinned":
        pin = [(slot, torch.from_numpy(a).pin_memory()) for slot, a in fact]
        frag.push(Chunk([(slot, t.data_ptr(), None, abi.TYPE_INT) for slot, t in pin], num_rows=n, mem=abi.MEM_HOST_PINNED))
        frag.ctx.sync()
        return
    chunk = _device_chunk(torch, fact, 1 if case == "unaligned" else 0)
    if case == "unaligned":
        assert all(c[1].data_ptr() % 16 == 4 for c in chunk.columns())
    frag.push(chunk)
    frag.ctx.sync()


@pytest.mark.parametrize("case", list(CASES))
def test_carried_key_parity(gpu, ctx, oracle, case):
    import torch
    rng = np.random.default_rng(500 + list(CASES).index(case))
    fact, dims, scan, agg = _star(case, rng)
    descs = [abi.make_join_desc(abi.JOIN_INNER, [10 * (k + 1)], [k], [abi.TYPE_INT]) for k in range(3)]
    payload = [[11], [], []]
    gj = [gpu.Join(ctx, d) for d in descs]
    oj = [oracle.Join(d) for d in descs]
    frag = None
    try:
        for g, o, ch in zip(gj, oj, dims):
            g.append_build(ch)
            o.append_build(ch)
            g.build_finish()
            o.build()
        frag = gpu.Fragment(ctx, scan, [(g, k, payload[k]) for k, g in enumerate(gj)], agg, mode=2)
        _push(torch, frag, fact, case)
        plan = frag.plan()
        # (after the 5 % predicate only the carried join is streamed; the other one gets a gather pass)
        later = case == "carried_later"
        assert plan["mode"] == "selection-vector-passes", plan
        assert (plan["num_stream_joins"], plan["num_gather_passes"]) == ((1, 1) if later else (2, 0)), plan
        assert plan["final_pass"] == ("generic" if case == "generic_final" else "dense-batched"), plan
        first = 0 if case in ("carried_first", "carried_later", "keys_at_int32_max", "one_ragged_tile") else 1
        assert plan["order"][first] == 0, plan
        ores, opassed = oracle.fragment_run(scan, [(o, k, payload[k]) for k, o in enumerate(oj)], agg,
                                            Chunk([(slot, a, None) for slot, a in fact]), num_threads=3)
        assert frag.rows_passed == opassed > (10 if case == "one_ragged_tile" else 200)
        assert_rows_equal(gpu_rows(frag.agg.result()), oracle_rows(ores))
    finally:
        if frag:
            frag.close()
        for g in gj:
            g.close()


def test_carried_key_q41_device(gpu, ctx, oracle):
    # SSB Q4.1 on device-resident columns: supplier and customer streamed, the customer key carried, part in a gather
    # pass between the streaming and the final pass, dates tested by the final pass; pushed in two batches, the second
    # one with a ragged last tile
    import torch
    dims = ssb.gen_dims(0.1)
    lo = ssb.gen_lineorder(0.1, n=600_000)
    gjoins, gkeep = ssb.build_dims(gpu, dims, ssb.dim_plans_q41(), ctx=ctx)
    ojoins, okeep = ssb.build_dims(oracle, dims, ssb.dim_plans_q41())
    agg_desc = ssb.q41_agg_desc()
    frag = gpu.Fragment(ctx, abi.ScanDesc(), gjoins, agg_desc, mode=2)
    try:
        dev = {k: torch.from_numpy(lo[k]).cuda() for k in ssb.Q41_FACT_COLS}
        cut = 4096 * 60
        for a, b in ((0, cut), (cut, 600_000)):
            frag.push(ssb.fact_chunk({k: v[a:b] for k, v in dev.items()}, ssb.Q41_FACT_COLS, mem=abi.MEM_DEVICE))
        ctx.sync()
        plan = frag.plan()
        assert plan["num_stream_joins"] == 2 and plan["num_gather_passes"] == 1 and plan["final_pass"] == "dense-batched", plan
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
