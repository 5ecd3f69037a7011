"""The hash aggregate's table geometry: a model of it in plain Python ints, and the routes into the table driven with keys
that crowd its 256-slot probing slices.

A probe never leaves the aligned 256-slot slice of its home slot (sr_agg.cuh, AggDev::slice_mask), and the table is kept
at load <= 1/2.  That is safe only while the hash spreads real keys over the slices as a uniform one would, and only while
every route into the table can take back a row a full slice refuses.  The model below restates the hash, the key packing,
the table sizing and the routes of a push; the CPU tests check it and bound the fullest slice for arithmetic-progression
key families, and the GPU tests pin it to the device (groups are emitted in slot order) and then use it to build inputs
that provably take each route and fill a slice: clustered real keys, keys crafted by inverting the hash, and skewed keys
that overflow the partitioned push's bucket regions.  Every result is compared exactly with a reference (numpy sorts and
Python ints; doubles only through MIN / MAX, which are exact).
"""
import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

M64 = (1 << 64) - 1
EMPTY = M64
SLICE_LOG2 = 8

# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
FMIX_C1, FMIX_C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
WIDE_ADD = 0x632BE59BD9B4E019


def agg_hash64(x):
    """sr_agg.cuh agg_hash64: the murmur3 finaliser fmix64"""
    x ^= x >> 33
    x = (x * FMIX_C1) & M64
    x ^= x >> 33
    x = (x * FMIX_C2) & M64
    return x ^ (x >> 33)


def agg_unhash64(h):
    """the inverse of agg_hash64: x ^= x >> 33 is its own inverse on 64 bits, the multipliers are odd"""
    h ^= h >> 33
    h = (h * pow(FMIX_C2, -1, 1 << 64)) & M64
    h ^= h >> 33
    h = (h * pow(FMIX_C1, -1, 1 << 64)) & M64
    return h ^ (h >> 33)


def hkey_hash(lo, hi, wide):
    """sr_agg.cuh hkey_hash: a wide (9..16 byte) key folds its high word in first"""
    return agg_hash64(lo ^ ((agg_hash64(hi) + WIDE_ADD) & M64)) if wide else agg_hash64(lo)


def hash64_np(x):
    """agg_hash64 over a numpy uint64 array (the same expression, for the large key families)"""
    u = np.uint64
    with np.errstate(over="ignore"):
        x = x ^ (x >> u(33))
        x = x * u(FMIX_C1)
        x = x ^ (x >> u(33))
        x = x * u(FMIX_C2)
        return x ^ (x >> u(33))


def key_layout(widths, nullable):
    """sr_agg.cuh agg_compile: columns packed widest first, each at a multiple of its width, never straddling the two
    words; the null bits after them -> (shifts, null_shift, wide)"""
    bits, shifts = 0, [0] * len(widths)
    for w in (8, 4, 2, 1):
        for k, wk in enumerate(widths):
            if wk != w:
                continue
            if bits < 64 < bits + 8 * w:
                bits = 64
            shifts[k] = bits
            bits += 8 * w
    if any(nullable) and bits < 64 < bits + 8:
        bits = 64
    key_bytes = bits // 8 + (1 if any(nullable) else 0)
    return shifts, bits, key_bytes > 8


def pack_key(values, widths, nullable):
    """one row's group-by values (None = NULL) -> (lo, hi, wide), as agg_pack_key builds it"""
    shifts, null_shift, wide = key_layout(widths, nullable)
    k = 0
    for i, (v, w) in enumerate(zip(values, widths)):
        k |= (1 << (null_shift + i)) if v is None else ((v & ((1 << (8 * w)) - 1)) << shifts[i])
    return k & M64, k >> 64, wide


def home_slot(cap, lo, hi=0, wide=False):
    """the slot a key's probe starts at; the all-ones key lives in the special slot `cap`"""
    if lo == EMPTY and (not wide or hi == EMPTY):
        return cap
    return hkey_hash(lo, hi, wide) & (cap - 1)


def slice_of(cap, slot):
    return slot >> SLICE_LOG2


def table_cap(expected_groups=0):
    """sr_agg.cuh agg_compile: 2^21 slots, or 2 expected_groups rounded up to a power of two"""
    cap = 1 << 21
    while cap < 2 * expected_groups:
        cap <<= 1
    return cap


def admission_limit(cap):
    return cap // 2    # agg_alloc_tables


PARTITION_MIN_ROWS = 1 << 20   # sr_agg_part_host.cuh kPartitionedMinRows


def push_route(n, ngroups, cap, min_rows=PARTITION_MIN_ROWS):
    """sr_agg.cuh agg_push_vtab, hash tables without AVG_MERGE -> (route, growth factor when the table refuses a row)"""
    if n >= min_rows:
        return "partitioned", 2
    if ngroups + n <= admission_limit(cap):
        return "fused", 2     # the refused rows are pushed again after at least a doubling
    return "two_pass", 4


def state_words(fns_modes):
    """agg_state_words: COUNT(*)'s counter, then per other function acc0, acc1 (128-bit sums), accn (nullable input);
    fns_modes: [(is_count_star, is_i128, track_n)]"""
    return 1 + sum(0 if cs else 1 + int(i128) + int(tn) for cs, i128, tn in fns_modes)


def region_cap(mean):
    """sr_agg_part_host.cuh aggp_region_cap"""
    c = int(mean * 1.1 + 6.0 * max(mean, 1.0) ** 0.5 + 64.0) + 1
    return (c + 1) & ~1


def part_plan(cap, m, wide, words_state, force_l2=False):
    """sr_agg_part_host.cuh agg_push_partitioned: bucket geometry of a push of m rows -> dict"""
    log2cap = cap.bit_length() - 1
    slot_bytes = 8 * ((2 if wide else 1) + words_state)
    nw = 8
    while nw > 1 and (nw << SLICE_LOG2) * slot_bytes > 48 * 1024:
        nw >>= 1
    log2nw = nw.bit_length() - 1
    apply_smem = (nw << SLICE_LOG2) * slot_bytes
    bucket_log2 = SLICE_LOG2 + log2nw
    smem = (log2cap > bucket_log2 and log2cap - bucket_log2 <= 18 and apply_smem <= 200 * 1024 and not force_l2)
    if smem:
        bits, shift = log2cap - bucket_log2, bucket_log2
    else:
        table_bytes = (cap + 1) * slot_bytes
        log2p = 1
        while log2p < 9 and (table_bytes >> log2p) > (32 << 20):
            log2p += 1
        bits = min(log2p, log2cap)
        shift = log2cap - bits
    bits2 = bits // 2 if bits > 9 else 0
    P, F1 = 1 << bits, 1 << (bits - bits2)
    return {"smem": smem, "nw": nw, "bits": bits, "bits2": bits2, "bucket_shift": shift,
            "cap2": region_cap(m / P), "cap1": region_cap(m / F1) if bits2 else 0}


def craft_keys(cap, target_slice, count, seed=0, hi=None):
    """`count` distinct keys whose home slot lies in `target_slice` of a table of `cap` slots, with bit log2(cap) of the
    hash alternating: after one doubling they split into two slices of count / 2 each, and no further.  8-byte keys as
    unsigned words; with `hi` given, the lo words of wide keys (lo, hi)."""
    log2cap = cap.bit_length() - 1
    rng = np.random.default_rng(seed)
    keys, seen = [], set()
    while len(keys) < count:
        top = int(rng.integers(0, 1 << (63 - log2cap))) << 1 | (len(keys) & 1)
        h = (top << log2cap) | (target_slice << SLICE_LOG2) | int(rng.integers(0, 1 << SLICE_LOG2))
        k = agg_unhash64(h)
        if hi is not None:
            k ^= (agg_hash64(hi) + WIDE_ADD) & M64
        if k == EMPTY or k in seen:
            continue
        seen.add(k)
        keys.append(k)
    return keys


def signed64(u):
    return u - (1 << 64) if u >> 63 else u


def slice_counts_np(keys_u64, cap):
    return np.bincount(((hash64_np(keys_u64) & np.uint64(cap - 1)) >> np.uint64(SLICE_LOG2)).astype(np.int64), minlength=cap >> SLICE_LOG2)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model
# ---------------------------------------------------------------------------------------------------------------------
def test_model_hash_and_inverse():
    rng = np.random.default_rng(1)
    xs = [0, 1, M64, 1 << 63, 1000, 0x123456789ABCDEF] + [int(v) for v in rng.integers(0, 1 << 63, 200, dtype=np.int64)]
    for x in xs:
        assert agg_unhash64(agg_hash64(x)) == x
    got = hash64_np(np.array(xs, dtype=np.uint64))
    assert [int(v) for v in got] == [agg_hash64(x) for x in xs]
    assert agg_hash64(0) == 0


def test_model_key_packing():
    # BIGINT alone: one word; nullable BIGINT: the null bit opens the second word; INT + BIGINT: BIGINT first
    assert key_layout([8], [False]) == ([0], 64, False)
    assert key_layout([8], [True]) == ([0], 64, True)
    assert key_layout([4, 8], [False, False]) == ([64, 0], 96, True)
    assert key_layout([4, 4], [False, False]) == ([0, 32], 64, False)
    assert key_layout([4, 2, 1], [True, False, False]) == ([0, 32, 48], 56, False)
    assert pack_key([0, 7], [4, 4], [False, False]) == (7 << 32, 0, False)
    assert pack_key([-1], [8], [False]) == (M64, 0, False)
    assert home_slot(1 << 21, M64) == 1 << 21
    assert pack_key([None], [8], [True]) == (0, 1, True)
    assert pack_key([5, -2], [4, 8], [False, False]) == (M64 - 1, 5, True)


def test_model_routes():
    cap = table_cap()
    assert cap == 1 << 21 and table_cap(3_000_000) == 1 << 23 and admission_limit(cap) == 1 << 20
    assert push_route(1_000_000, 0, cap) == ("fused", 2)
    assert push_route(1_000_000, 1_000_000, cap) == ("two_pass", 4)
    assert push_route(1 << 20, 0, cap) == ("partitioned", 2)
    assert push_route(10_300, 0, cap, min_rows=1000) == ("partitioned", 2)
    # the partitioned plans the GPU tests use: SUM + COUNT(*) over an 8-byte key
    p = part_plan(cap, 3_000_000, False, state_words([(False, False, False), (True, False, False)]))
    assert p["smem"] and p["nw"] == 8 and p["bits"] == 10 and p["bits2"] == 5
    pl2 = part_plan(cap, 3_000_000, False, 2, force_l2=True)
    assert not pl2["smem"] and pl2["bits"] == 1 and pl2["bits2"] == 0


def test_craft_keys_land_in_one_slice_and_split_once():
    cap = 1 << 21
    for s, hi in ((5, None), (4000, 77)):
        keys = craft_keys(cap, s, 300, seed=s, hi=hi)
        wide = hi is not None
        assert len(set(keys)) == 300
        assert {slice_of(cap, home_slot(cap, k, hi or 0, wide)) for k in keys} == {s}
        after = [slice_of(2 * cap, home_slot(2 * cap, k, hi or 0, wide)) for k in keys]
        assert sorted(set(after)) == [s, s + (cap >> SLICE_LOG2)] and after.count(s) == 150


# slice-load families (all keys distinct) at load 1/2; the uniform expectation for the fullest of 2^13..2^15 slices is
# about 175
SLICE_LOAD_BOUND = 200
FAMILIES = {"1000i": lambda n: np.uint64(1000) * np.arange(n, dtype=np.uint64),
            "i<<32": lambda n: np.arange(n, dtype=np.uint64) << np.uint64(32),
            "1.6e12+10000i": lambda n: np.uint64(1_600_000_000_000) + np.uint64(10000) * np.arange(n, dtype=np.uint64),
            "100000i": lambda n: np.uint64(100000) * np.arange(n, dtype=np.uint64),
            "125i": lambda n: np.uint64(125) * np.arange(n, dtype=np.uint64)}


@pytest.mark.parametrize("log2cap", [21, 22, 23])
def test_slice_load_of_arithmetic_progressions(log2cap):
    cap = 1 << log2cap
    worst = {name: int(slice_counts_np(f(cap // 2), cap).max()) for name, f in FAMILIES.items()}
    assert max(worst.values()) <= SLICE_LOAD_BOUND, f"fullest slice per family at 2^{log2cap} slots: {worst}"


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers: an exact reference over sorted numpy arrays
# ---------------------------------------------------------------------------------------------------------------------
SUM_COUNT = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 10)]), (abi.AGG_COUNT_STAR, 0, 41, None)]


def _groups(key_cols):
    """key columns [(data, nulls)] -> (unique key columns as [(data, nulls)], inverse index)"""
    parts = []
    for d, nl in key_cols:
        parts.append(np.zeros(len(d), np.int64) if nl is None else nl.astype(np.int64))
        parts.append(np.where(nl.astype(bool), 0, d).astype(np.int64) if nl is not None else d.astype(np.int64))
    rec = np.stack(parts, axis=1)
    uniq, inv = np.unique(rec, axis=0, return_inverse=True)
    out = []
    for k in range(len(key_cols)):
        nl = uniq[:, 2 * k].astype(bool)
        out.append((uniq[:, 2 * k + 1], nl))
    return out, inv.reshape(-1)


def _reduce(inv, ng, vals, nulls, kind):
    """exact per-group SUM (Python ints, 128-bit capable) / MIN / MAX / COUNT of non-NULL values -> (values, is_null)"""
    keep = np.ones(len(vals), bool) if nulls is None else ~nulls.astype(bool)
    g, v = inv[keep], vals[keep]
    cnt = np.bincount(g, minlength=ng)
    if kind == abi.AGG_COUNT:
        return cnt, np.zeros(ng, bool)
    if kind == abi.AGG_SUM:
        vi = v.astype(np.int64)
        hi = np.zeros(ng, np.int64)
        lo = np.zeros(ng, np.int64)
        np.add.at(hi, g, vi >> 32)
        np.add.at(lo, g, vi & 0xFFFFFFFF)
        return [int(h) * (1 << 32) + int(l) for h, l in zip(hi, lo)], cnt == 0
    init = np.inf if vals.dtype.kind == "f" else np.iinfo(np.int64).max
    if kind == abi.AGG_MAX:
        init = -init if vals.dtype.kind == "f" else np.iinfo(np.int64).min
    r = np.full(ng, init, dtype=np.float64 if vals.dtype.kind == "f" else np.int64)
    (np.minimum if kind == abi.AGG_MIN else np.maximum).at(r, g, v)
    return r, cnt == 0


def check_exact(res, key_cols, fns, val_cols, label):
    """res: Agg.result() -> assert it equals the reference exactly.  key_cols [(data, nulls)]; val_cols {slot: (data, nulls)}"""
    nk = len(key_cols)
    uk, inv = _groups(key_cols)
    ng = len(uk[0][0])
    got_keys = []
    for k in range(nk):
        _, _, d, nl = res[k]
        nlb = np.zeros(len(d), bool) if nl is None else nl.astype(bool)
        got_keys.append((np.where(nlb, 0, d).astype(np.int64), nlb))
    assert len(got_keys[0][0]) == ng, f"{label}: {len(got_keys[0][0])} groups, want {ng}"
    parts = []
    for d, nl in got_keys:
        parts += [nl.astype(np.int64), d]
    order = np.lexsort(parts[::-1])
    for k in range(nk):
        assert np.array_equal(got_keys[k][1][order], uk[k][1]), f"{label}: key {k} nulls"
        assert np.array_equal(got_keys[k][0][order], uk[k][0]), f"{label}: key {k} values"
    cnt_star = np.bincount(inv, minlength=ng)
    for f, (kind, ityp, _, rpn) in enumerate(fns):
        _, rt, d, nl = res[nk + f]
        d = d[order]
        if kind == abi.AGG_COUNT_STAR:
            assert np.array_equal(d, cnt_star), f"{label}: COUNT(*)"
            continue
        vd, vn = val_cols[rpn[0][1]]
        want, wnull = _reduce(inv, ng, vd, vn, kind)
        gnull = np.zeros(ng, bool) if nl is None else nl[order].astype(bool)
        if kind == abi.AGG_COUNT:
            assert np.array_equal(d, want), f"{label}: fn {f}"
            continue
        assert np.array_equal(gnull, wnull), f"{label}: fn {f} nulls"
        if rt == abi.TYPE_DECIMAL128:
            pairs = np.frombuffer(np.ascontiguousarray(d).tobytes(), np.int64).reshape(-1, 2)
            bad = [i for i in np.flatnonzero(~wnull) if int(pairs[i, 0]) % (1 << 64) + (int(pairs[i, 1]) << 64) != want[i]]
        elif kind == abi.AGG_SUM:
            w = np.array([((x + (1 << 63)) % (1 << 64)) - (1 << 63) for x in want], dtype=np.int64)
            bad = np.flatnonzero(~wnull & (d != w))
        else:
            bad = np.flatnonzero(~wnull & (d.astype(want.dtype) != want))
        assert len(bad) == 0, f"{label}: fn {f}: {len(bad)} groups differ, first at {bad[:3]}"


def _chunk(cols, lo=0, hi=None):
    return Chunk([(s, d[lo:hi], None if nl is None else nl[lo:hi], t) for s, d, nl, t in cols])


def _run(gpu, ctx, route, desc, cols, pushes, monkeypatch):
    """push `cols` in `pushes` equal parts through one route -> (result, device bytes before the result, after the first
    push).  Routes: agg (whatever agg_push_vtab chooses), part, part_l2, merge (one partial per part), frag1, frag2."""
    n = len(cols[0][1])
    cuts = [n * i // pushes for i in range(pushes + 1)]
    if route.startswith("part"):
        monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", "1000")
        if route == "part_l2":
            monkeypatch.setenv("SR_AGG_PARTITION_FORCE_L2", "1")
    if route.startswith("frag"):
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [], desc, mode=1 if route == "frag1" else 2)
        try:
            frag.push(_chunk(cols, cuts[0], cuts[1]))
            b1 = ctx.device_bytes
            for i in range(1, pushes):
                frag.push(_chunk(cols, cuts[i], cuts[i + 1]))
            assert frag.plan()["mode"] == ("fused-cascade" if route == "frag1" else "selection-vector-passes")
            assert frag.rows_passed == n
            b = ctx.device_bytes
            return frag.agg.result(), b, b1
        finally:
            frag.close()
    if route == "merge":
        parts = [gpu.Agg(ctx, desc) for _ in range(pushes)]
        a = gpu.Agg(ctx, desc)
        try:
            for i, p in enumerate(parts):
                p.push(_chunk(cols, cuts[i], cuts[i + 1]))
                p.finish()
            a.merge(parts[0])
            b1 = ctx.device_bytes
            for p in parts[1:]:
                a.merge(p)
            b = ctx.device_bytes
            return a.result(), b, b1
        finally:
            for p in parts:
                p.close()
            a.close()
    a = gpu.Agg(ctx, desc)
    try:
        a.push(_chunk(cols, cuts[0], cuts[1]))
        b1 = ctx.device_bytes
        for i in range(1, pushes):
            a.push(_chunk(cols, cuts[i], cuts[i + 1]))
        b = ctx.device_bytes
        return a.result(), b, b1
    finally:
        a.close()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the model is the device's
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["bigint", "nullable_bigint", "int_bigint"])
def test_groups_come_out_in_model_slot_order(gpu, ctx, shape):
    cap = table_cap()
    rng = np.random.default_rng(7)
    widths, nullable = ([8], [shape == "nullable_bigint"]) if shape != "int_bigint" else ([4, 8], [False, False])
    rows, used = [], set()
    while len(rows) < 1000:
        b = int(rng.integers(-(1 << 62), 1 << 62))
        vals = [b] if shape != "int_bigint" else [int(rng.integers(-(1 << 31), 1 << 31)), b]
        lo, hi, wide = pack_key(vals, widths, nullable)
        assert wide == (shape != "bigint")
        s = home_slot(cap, lo, hi, wide)
        if s in used:
            continue
        used.add(s)
        rows.append((s, vals))
    arr = list(zip(*[v for _, v in rows]))
    if shape == "int_bigint":
        cols = [(0, np.array(arr[0], np.int32), None, abi.TYPE_INT), (1, np.array(arr[1], np.int64), None, abi.TYPE_BIGINT)]
        slots, types = [0, 1], [abi.TYPE_INT, abi.TYPE_BIGINT]
    else:
        nl = np.zeros(1000, np.uint8) if shape == "nullable_bigint" else None
        cols = [(1, np.array(arr[0], np.int64), nl, abi.TYPE_BIGINT)]
        slots, types = [1], [abi.TYPE_BIGINT]
    desc = abi.make_agg_desc(slots, types, fns=[(abi.AGG_COUNT_STAR, 0, 40, None)], group_nullable=nullable if shape == "nullable_bigint" else None)
    a = gpu.Agg(ctx, desc)
    try:
        a.push(Chunk(cols))
        res = a.result()
    finally:
        a.close()
    want = [v for _, v in sorted(rows)]
    got = list(zip(*[res[k][2].tolist() for k in range(len(slots))]))
    assert [list(g) for g in got] == want, "group order differs from the model's home-slot order"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: clustered real keys through every route
# ---------------------------------------------------------------------------------------------------------------------
def _bigint_case(keys_i64, rng):
    n = len(keys_i64)
    v = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    cols = [(1, keys_i64, None, abi.TYPE_BIGINT), (10, v, None, abi.TYPE_BIGINT)]
    desc = abi.make_agg_desc([1], [abi.TYPE_BIGINT], fns=SUM_COUNT)
    return desc, cols, [(keys_i64, None)], {10: (v, None)}


CLUSTER_ROUTES = ["agg", "agg3", "merge", "part", "part_l2", "frag1", "frag2"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", CLUSTER_ROUTES)
def test_clustered_keys_1000i(gpu, ctx, monkeypatch, route):
    # GROUP BY k = 1000 i, i < 2^20, every key once.  Under the xorshift hash a slice of the 2^21-slot table received
    # 268 of them; the model now keeps every slice at the uniform bound
    n = 1 << 20
    keys = np.arange(n, dtype=np.int64) * 1000
    cap = table_cap()
    assert slice_counts_np(keys.astype(np.uint64), cap).max() <= SLICE_LOAD_BOUND
    if route == "agg":
        assert push_route(n - 1, 0, cap)[0] == "fused"
        keys = keys[:n - 1]        # below the partitioned threshold: the fused pass
    pushes = {"agg": 1, "agg3": 3, "merge": 2}.get(route, 2)
    desc, cols, kc, vc = _bigint_case(keys, np.random.default_rng(11))
    res, _, _ = _run(gpu, ctx, "agg" if route == "agg3" else route, desc, cols, pushes, monkeypatch)
    check_exact(res, kc, SUM_COUNT, vc, route)


@pytest.mark.gpu
def test_clustered_int_pairs_three_pushes(gpu, ctx):
    # GROUP BY (a INT, b INT), a = 0, b = i: the packed key is i << 32.  Three pushes of 1,000,000 rows: the first two are
    # fused then two-pass (growing to 2^23 slots), the third is fused into the grown table
    n = 3_000_000
    b = np.arange(n, dtype=np.int32)
    a = np.zeros(n, np.int32)
    assert slice_counts_np(b.astype(np.uint64) << np.uint64(32), 1 << 23).max() <= SLICE_LOAD_BOUND
    cap, ng, routes = table_cap(), 0, []
    for _ in range(3):
        r, grow = push_route(1_000_000, ng, cap)
        routes.append(r)
        if r == "two_pass":
            while ng + 1_000_000 > admission_limit(cap):
                cap *= grow
        ng += 1_000_000
    assert routes == ["fused", "two_pass", "fused"] and cap == 1 << 23
    v = np.random.default_rng(3).integers(-1000, 1000, n, dtype=np.int64)
    cols = [(0, a, None, abi.TYPE_INT), (1, b, None, abi.TYPE_INT), (10, v, None, abi.TYPE_BIGINT)]
    desc = abi.make_agg_desc([0, 1], [abi.TYPE_INT, abi.TYPE_INT], fns=SUM_COUNT)
    agg = gpu.Agg(ctx, desc)
    try:
        for i in range(3):
            agg.push(_chunk(cols, i * 1_000_000, (i + 1) * 1_000_000))
        res = agg.result()
    finally:
        agg.close()
    check_exact(res, [(a, None), (b, None)], SUM_COUNT, {10: (v, None)}, "int pairs")


@pytest.mark.gpu
def test_clustered_keys_count_distinct(gpu, ctx):
    # COUNT(DISTINCT v) GROUP BY g: the inner set is keyed (g, v), a wide key; v = 1000 i over 1,000,000 rows
    n = 1_000_000
    rng = np.random.default_rng(5)
    g = rng.integers(0, 50, n).astype(np.int32)
    v = np.arange(n, dtype=np.int64) * 1000
    fns = [(abi.AGG_COUNT_DISTINCT, abi.TYPE_BIGINT, 40, [("col", 10)]), (abi.AGG_COUNT_STAR, 0, 41, None)]
    desc = abi.make_agg_desc([0], [abi.TYPE_INT], fns=fns)
    a = gpu.Agg(ctx, desc)
    try:
        a.push(_chunk([(0, g, None, abi.TYPE_INT), (10, v, None, abi.TYPE_BIGINT)], 0, n // 2))
        a.push(_chunk([(0, g, None, abi.TYPE_INT), (10, v, None, abi.TYPE_BIGINT)], n // 2, n))
        res = a.result()
    finally:
        a.close()
    order = np.argsort(res[0][2])
    assert np.array_equal(res[0][2][order], np.arange(50))
    assert np.array_equal(res[1][2][order], np.bincount(g, minlength=50))   # every v distinct
    assert np.array_equal(res[2][2][order], np.bincount(g, minlength=50))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: crafted keys that fill one slice, on every route, against a uniform control
# ---------------------------------------------------------------------------------------------------------------------
CRAFT_SLICE = 1234


def _crafted_case(crafted, rows_per_key=1, seed=0):
    """10,000 uniform BIGINT keys plus 300 crafted ones (or 300 more uniform ones), each repeated rows_per_key times,
    shuffled"""
    rng = np.random.default_rng(seed)
    cap = table_cap()
    uni = rng.integers(-(1 << 62), 1 << 62, 10_300, dtype=np.int64)
    if crafted:
        uni[10_000:] = [signed64(k) for k in craft_keys(cap, CRAFT_SLICE, 300, seed=seed)]
    keys = np.repeat(uni, rows_per_key)
    rng.shuffle(keys)
    return keys


CRAFT_ROUTES = ["agg", "two_pass", "merge", "part", "part_l2", "frag1", "frag2"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", CRAFT_ROUTES)
def test_crafted_keys_fill_a_slice(gpu, ctx, monkeypatch, route):
    cap = table_cap()
    results = {}
    for crafted in (True, False):
        if route == "two_pass":
            # 10,300 groups over 2^20 - 1 rows, pushed after 10,000 rows: below the partitioned threshold and above
            # the admission limit, so the find-slots pass runs; only a full slice makes it grow
            keys = _crafted_case(crafted, rows_per_key=102)[:(1 << 20) - 1]
            keys = np.concatenate([np.arange(10_000, dtype=np.int64) * 7 + 1, keys])
            assert push_route(len(keys) - 10_000, 10_000, cap) == ("two_pass", 4)
            pushes = None
        else:
            keys = _crafted_case(crafted)
            pushes = 2
        u = keys.astype(np.uint64)
        worst = slice_counts_np(np.unique(u), cap).max()
        assert (worst > 256) == crafted, f"model: fullest slice {worst}"
        desc, cols, kc, vc = _bigint_case(keys, np.random.default_rng(2))
        if route == "two_pass":
            a = gpu.Agg(ctx, desc)
            try:
                a.push(_chunk(cols, 0, 10_000))
                b1 = ctx.device_bytes
                a.push(_chunk(cols, 10_000, None))
                res, b = a.result(), ctx.device_bytes
            finally:
                a.close()
        else:
            if route == "merge":   # each partial alone fits its slice, the merged table does not
                half_u = np.unique(u[: len(u) // 2])
                assert slice_counts_np(half_u, cap).max() <= 256 or not crafted
            res, b, b1 = _run(gpu, ctx, route, desc, cols, pushes, monkeypatch)
        check_exact(res, kc, SUM_COUNT, vc, f"{route} crafted={crafted}")
        results[crafted] = (b, b1)
        monkeypatch.delenv("SR_AGG_PARTITION_MIN_ROWS", raising=False)
        monkeypatch.delenv("SR_AGG_PARTITION_FORCE_L2", raising=False)
    # the crafted keys made the route grow its table; the same number of uniform keys did not
    assert results[True][0] > results[False][0], f"{route}: device bytes crafted {results[True]}, uniform {results[False]}"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: skewed keys overflow the partitioned push's bucket regions
# ---------------------------------------------------------------------------------------------------------------------
SKEW_CASES = ["half_one_key", "sixteen_keys_90pct", "heavy_minus1_simple", "heavy_minus1_general", "nullable_decimal_double",
              "overflow_and_failed_bucket"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SKEW_CASES)
def test_partitioned_skew(gpu, ctx, monkeypatch, case):
    n = 2_000_000
    rng = np.random.default_rng(SKEW_CASES.index(case))
    cap = table_cap()
    keys = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64) % 200_000 * 7919
    heavy = [-1] if "minus1" in case else [123456789]
    if case == "half_one_key" or "minus1" in case or case == "nullable_decimal_double":
        keys[rng.random(n) < 0.5] = heavy[0]
    elif case == "sixteen_keys_90pct":
        heavy = [int(x) for x in rng.integers(-(1 << 62), 1 << 62, 16)]
        hot = rng.random(n) < 0.9
        keys[hot] = np.array(heavy, np.int64)[rng.integers(0, 16, int(hot.sum()))]
    else:   # a heavy key and a crafted slice in the same push
        keys[rng.random(n) < 0.5] = heavy[0]
        keys[:300] = [signed64(k) for k in craft_keys(cap, CRAFT_SLICE, 300, seed=9)]
    v = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    d = rng.standard_normal(n) * 1e6
    vn = dn = None
    if case == "nullable_decimal_double":
        vn = (rng.random(n) < 0.2).astype(np.uint8)
        dn = (rng.random(n) < 0.2).astype(np.uint8)
        fns = [(abi.AGG_SUM, abi.TYPE_DECIMAL64, 40, [("col", 10)]), (abi.AGG_MIN, abi.TYPE_DOUBLE, 41, [("col", 11)]),
               (abi.AGG_MAX, abi.TYPE_DOUBLE, 42, [("col", 11)]), (abi.AGG_COUNT_STAR, 0, 43, None)]
        vtype = abi.TYPE_DECIMAL64
    elif case == "heavy_minus1_general":
        fns = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 10)]), (abi.AGG_MAX, abi.TYPE_DOUBLE, 41, [("col", 11)]),
               (abi.AGG_COUNT_STAR, 0, 43, None)]
        vtype = abi.TYPE_BIGINT
        vn = (rng.random(n) < 0.1).astype(np.uint8)   # a null word: the general scatter kernel
    else:
        fns = SUM_COUNT
        vtype = abi.TYPE_BIGINT
    cols = [(1, keys, None, abi.TYPE_BIGINT), (10, v, vn, vtype), (11, d, dn, abi.TYPE_DOUBLE)]
    nulls_of = {10: vn, 11: dn}
    modes = [(k == abi.AGG_COUNT_STAR, t == abi.TYPE_DECIMAL64, r is not None and nulls_of[r[0][1]] is not None) for k, t, _, r in fns]
    plan = part_plan(cap, n // 2, False, state_words(modes))
    assert plan["smem"] and plan["bits2"] > 0
    # every heavy key alone fills its bucket's region at both scatter levels: its records go to the overflow list
    fewest = min(int((keys[: n // 2] == h).sum()) for h in heavy)
    assert fewest > plan["cap1"] and fewest > plan["cap2"], (fewest, plan)
    monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", "1000")
    a = gpu.Agg(ctx, abi.make_agg_desc([1], [abi.TYPE_BIGINT], fns=fns))
    try:
        a.push(_chunk(cols, 0, n // 2))        # into a fresh table
        a.push(_chunk(cols, n // 2, None))     # into loaded slices
        res = a.result()
    finally:
        a.close()
    check_exact(res, [(keys, None)], fns, {10: (v, vn), 11: (d, dn)}, case)
