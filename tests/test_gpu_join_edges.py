"""Hash joins, the fragment's joins and runtime filters at the edges of their key domains, against an exact reference in
plain Python.

The join tests elsewhere use moderate random keys and judge the device only against the oracle.  Here the keys sit where
the delicate arithmetic is: range-mapped tables whose build range ends at a type's extreme and is probed from the other
end (key - min), the method limits of `join_finish`, the INT64_MIN "empty" marker as a legal key, narrow packed keys with
negative columns (masking), 9- to 16-byte keys whose BIGINT column straddles bit 64, colliding 64-bit fingerprints of
16-byte keys, build chunks that turn a column nullable, the fragment's 32-bit bitmap tests with their guard word, and
runtime filters at INT64_MIN / INT64_MAX.  `ref_join` below compares keys as tuples of Python values and packs nothing,
so it cannot share a packing bug with the device; `test_reference_agrees_with_the_oracle` checks it against the oracle on
the CPU, under the oracle's own method choice and under every forced method that applies, before it judges the kernels.
Every other test needs the device and is marked `gpu`.
"""
import functools

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from starrocks_b200.rows import col_to_py
from tests.test_gpu_value_edges import I8, I16, I32, I64, check_agg, col_values, ref_agg, ref_expr, wrap

INF, NAN = float("inf"), float("nan")
RANGE, LINEAR, DIRECT = abi.JOIN_METHOD_RANGE_DIRECT_MAPPING, abi.JOIN_METHOD_LINEAR_CHAINED, abi.JOIN_METHOD_DIRECT_MAPPING
JOIN_TYPES = [abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_RIGHT_OUTER,
              abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL_OUTER]
JT_NAME = {abi.JOIN_INNER: "inner", abi.JOIN_LEFT_OUTER: "left_outer", abi.JOIN_LEFT_SEMI: "left_semi",
           abi.JOIN_LEFT_ANTI: "left_anti", abi.JOIN_RIGHT_OUTER: "right_outer", abi.JOIN_RIGHT_SEMI: "right_semi",
           abi.JOIN_RIGHT_ANTI: "right_anti", abi.JOIN_FULL_OUTER: "full_outer"}
PAIR_TYPES = (abi.JOIN_INNER, abi.JOIN_LEFT_OUTER, abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER)
ROW_IF_NONE = (abi.JOIN_LEFT_OUTER, abi.JOIN_FULL_OUTER, abi.JOIN_LEFT_ANTI)
POST_PROBE = (abi.JOIN_RIGHT_OUTER, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL_OUTER)
TYPE_RANGE = {abi.TYPE_BOOLEAN: (0, 1), abi.TYPE_TINYINT: I8, abi.TYPE_SMALLINT: I16, abi.TYPE_INT: I32, abi.TYPE_BIGINT: I64}


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def ref_join(build_rows, probe_rows, join_type, conjunct=None):
    """build_rows / probe_rows: key tuples of Python values (None = NULL).  conjunct: optional callable
    (probe_index, build_index) -> bool, the other-join conjunct.  -> (probe-phase pairs [(probe_index, build_index)],
    POST_PROBE build indexes).  Build indexes are 1-based; 0 stands for "no build row"."""
    index = {}
    for b, key in enumerate(build_rows, 1):
        if None not in key:
            index.setdefault(key, []).append(b)
    pairs, matched = [], set()
    for i, key in enumerate(probe_rows):
        cands = [] if None in key else index.get(key, [])[::-1]          # a key's matches by descending build index
        if conjunct is not None:
            cands = [b for b in cands if conjunct(i, b)]
        if join_type in PAIR_TYPES:
            pairs.extend((i, b) for b in cands)
        if not cands and join_type in ROW_IF_NONE:
            pairs.append((i, 0))
        if cands and join_type == abi.JOIN_LEFT_SEMI:
            pairs.append((i, 0))
        matched.update(cands)
    if join_type == abi.JOIN_RIGHT_SEMI:
        remain = sorted(matched)
    elif join_type in POST_PROBE:
        remain = [b for b in range(1, len(build_rows) + 1) if b not in matched]
    else:
        remain = []
    return pairs, remain


def ref_conjunct(rpn, types, probe_cols, build_cols):
    """the other-join conjunct of one (probe row, build row) pair through ref_expr: true when not NULL and not zero"""
    def holds(i, b):
        cols = {s: [v[i]] for s, v in probe_cols.items()}
        cols.update({s: [v[b - 1]] for s, v in build_cols.items()})
        v, nl = ref_expr(rpn, cols, types, 0)
        return not nl and v != 0
    return holds


# wide_fingerprint of csrc/sr_join.cuh:53 (the 64-bit table key of a 9..16-byte packed key), restated over Python ints
FP_MUL_HI, FP_ADD_HI, FP_MUL = 0x9E3779B97F4A7C15, 0x632BE59BD9B4E019, 0xD6E8FEB86659FD93
M64 = (1 << 64) - 1


def wide_fingerprint(lo, hi):
    x = (lo & M64) ^ (((hi & M64) * FP_MUL_HI + FP_ADD_HI) & M64)
    x ^= x >> 32
    x = (x * FP_MUL) & M64
    x ^= x >> 32
    return wrap(x, 64)


def wide_fingerprint_lo(fp, hi):
    """the low 64 bits `lo` with wide_fingerprint(lo, hi) == fp: each `x ^= x >> 32` is its own inverse, the multiply is
    undone by the inverse of the odd multiplier modulo 2^64"""
    x = fp & M64
    x ^= x >> 32
    x = (x * pow(FP_MUL, -1, 1 << 64)) & M64
    x ^= x >> 32
    return x ^ (((hi & M64) * FP_MUL_HI + FP_ADD_HI) & M64)


def test_reference_known_answers():
    b = [(1,), (2,), (1,), (None,)]
    p = [(1,), (3,), (None,), (2,)]
    assert ref_join(b, p, abi.JOIN_INNER) == ([(0, 3), (0, 1), (3, 2)], [])
    assert ref_join(b, p, abi.JOIN_LEFT_OUTER)[0] == [(0, 3), (0, 1), (1, 0), (2, 0), (3, 2)]
    assert ref_join(b, p, abi.JOIN_LEFT_SEMI)[0] == [(0, 0), (3, 0)]
    assert ref_join(b, p, abi.JOIN_LEFT_ANTI)[0] == [(1, 0), (2, 0)]
    assert ref_join(b, p, abi.JOIN_RIGHT_SEMI) == ([], [1, 2, 3])
    assert ref_join(b, p, abi.JOIN_RIGHT_ANTI) == ([], [4])
    assert ref_join(b, p, abi.JOIN_FULL_OUTER)[1] == [4]
    assert ref_join(b, p, abi.JOIN_INNER, lambda i, bi: bi != 3)[0] == [(0, 1), (3, 2)]
    for lo, hi in ((0, 0), (M64, M64), (12345, 1 << 63), (1 << 63, 7)):
        assert wide_fingerprint_lo(wide_fingerprint(lo, hi), hi) == lo


# ---------------------------------------------------------------------------------------------------------------------
# standalone join cases.  Build slots: keys 10.., row number 20 (1-based: it IS the build index), BIGINT payload 21,
# DOUBLE payload 22.  Probe slots: keys 0.., row number 5, BIGINT 6, DOUBLE 7.
# ---------------------------------------------------------------------------------------------------------------------
B_ROW, B_BIG, B_DBL, P_ROW, P_BIG, P_DBL = 20, 21, 22, 5, 6, 7
BIG_EDGES = [I64[0], I64[0] + 3, I64[1], I64[1] - 5, 1 << 62, -(1 << 62), -1, 0]
DBL_EDGES = [NAN, INF, -INF, 0.0, -0.0, 1.5, -1.5, 1e308]


def _pick(rng, values, n, dtype):
    return np.array(values, dtype=object)[rng.integers(0, len(values), n)].astype(dtype)


def _mix(rng, n, dtype, parts):
    """n values: parts = [(probability, array of candidates)], the rest uniform over the type"""
    lo, hi = I64 if dtype == np.int64 else (int(np.iinfo(dtype).min), int(np.iinfo(dtype).max))
    out = rng.integers(lo, hi, n, dtype=dtype, endpoint=True) if dtype != np.uint8 else rng.integers(0, 2, n).astype(np.uint8)
    r = rng.random(n)
    acc = 0.0
    for p, cand in parts:
        cand = np.asarray(cand, dtype=dtype)
        sel = (r >= acc) & (r < acc + p)
        out[sel] = cand[rng.integers(0, len(cand), int(sel.sum()))]
        acc += p
    return out


class JoinCase:
    """inputs of one join: key columns of both sides with NULL masks, payloads, the build chunking and the method the
    case is written for"""

    def __init__(self, rng, ktypes, bkeys, pkeys, method, bnull=0.05, pnull=0.05, chunks=None, conj=None):
        self.ktypes, self.method, self.conj = ktypes, method, conj
        nb, npr = len(bkeys[0]), len(pkeys[0])
        self.bkeys, self.pkeys = bkeys, pkeys
        self.bnulls = [(rng.random(nb) < bnull).astype(np.uint8) if bnull else None for _ in bkeys]
        self.pnulls = [(rng.random(npr) < pnull).astype(np.uint8) if pnull else None for _ in pkeys]
        self.brow = np.arange(1, nb + 1, dtype=np.int32)
        self.bbig = _mix(rng, nb, np.int64, [(0.6, BIG_EDGES)])
        self.bbign = (rng.random(nb) < 0.1).astype(np.uint8)
        self.bdbl = _pick(rng, DBL_EDGES, nb, np.float64)
        self.prow = np.arange(npr, dtype=np.int32)
        self.pbig = _mix(rng, npr, np.int64, [(0.6, BIG_EDGES)])
        self.pdbl = _pick(rng, DBL_EDGES, npr, np.float64)
        # chunks: [(lo, hi, nullable)]; a non-nullable chunk carries no NULL arrays (its rows are not NULL)
        self.chunks = chunks or [(0, nb // 3, True), (nb // 3, nb, True)]
        for lo, hi, nullable in self.chunks:
            if not nullable:
                for m in self.bnulls + [self.bbign]:
                    if m is not None:
                        m[lo:hi] = 0

    @property
    def nb(self):
        return len(self.brow)

    def desc(self, jt):
        nk = len(self.ktypes)
        return abi.make_join_desc(jt, [10 + k for k in range(nk)], list(range(nk)), self.ktypes,
                                  build_out=[B_ROW, B_BIG] + [10 + k for k in range(nk)], probe_out=[P_ROW, P_BIG] + list(range(nk)),
                                  other_conjunct=self.conj)

    def build_chunks(self):
        out = []
        for lo, hi, nullable in self.chunks:
            cols = [(10 + k, c[lo:hi].copy(), None if (nl is None or not nullable) else nl[lo:hi].copy(), t)
                    for k, (c, nl, t) in enumerate(zip(self.bkeys, self.bnulls, self.ktypes))]
            cols += [(B_ROW, self.brow[lo:hi].copy(), None), (B_BIG, self.bbig[lo:hi].copy(), self.bbign[lo:hi].copy() if nullable else None),
                     (B_DBL, self.bdbl[lo:hi].copy(), None)]
            out.append(Chunk(cols))
        return out

    def probe_cols(self, rows=None):
        sl = slice(None) if rows is None else slice(0, rows)
        cols = [(k, c[sl].copy(), None if nl is None else nl[sl].copy(), t) for k, (c, nl, t) in enumerate(zip(self.pkeys, self.pnulls, self.ktypes))]
        return cols + [(P_ROW, self.prow[sl].copy(), None), (P_BIG, self.pbig[sl].copy(), None), (P_DBL, self.pdbl[sl].copy(), None)]

    def probe_chunk(self):
        return Chunk(self.probe_cols())

    @functools.cached_property
    def build_rows(self):
        return list(zip(*[col_values(c, nl) for c, nl in zip(self.bkeys, self.bnulls)]))

    @functools.cached_property
    def probe_rows(self):
        return list(zip(*[col_values(c, nl) for c, nl in zip(self.pkeys, self.pnulls)]))

    @functools.cached_property
    def build_vals(self):
        """Python values of the build_out columns, in build order"""
        return [col_values(self.brow, None), col_values(self.bbig, self.bbign)] + [col_values(c, nl) for c, nl in zip(self.bkeys, self.bnulls)]

    @functools.cached_property
    def probe_vals(self):
        return [col_values(self.prow, None), col_values(self.pbig, None)] + [col_values(c, nl) for c, nl in zip(self.pkeys, self.pnulls)]

    @functools.cached_property
    def conjunct(self):
        if self.conj is None:
            return None
        types = {P_BIG: abi.TYPE_BIGINT, B_BIG: abi.TYPE_BIGINT, P_DBL: abi.TYPE_DOUBLE, B_DBL: abi.TYPE_DOUBLE}
        holds = ref_conjunct(self.conj, types, {P_BIG: self.probe_vals[1], P_DBL: col_values(self.pdbl, None)},
                             {B_BIG: self.build_vals[1], B_DBL: col_values(self.bdbl, None)})
        return functools.lru_cache(maxsize=None)(holds)        # every join type asks for the same pairs

    def ref(self, jt, probe_rows=None):
        if probe_rows is None:
            return self._ref(jt)
        return ref_join(self.build_rows, probe_rows, jt, self.conjunct)

    @functools.lru_cache(maxsize=None)
    def _ref(self, jt):
        return ref_join(self.build_rows, self.probe_rows, jt, self.conjunct)

    def expected_columns(self, jt, pairs, probe_vals=None):
        """the output columns the reference gathers for the probe-phase pairs: probe_out, then build_out (NULL where the
        build index is 0)"""
        cols = []
        if jt not in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
            cols += [[v[i] for i, _ in pairs] for v in (probe_vals or self.probe_vals)]
        if jt not in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):          # RIGHT SEMI / ANTI: build columns, no rows
            cols += [[v[b - 1] if b else None for _, b in pairs] for v in self.build_vals]
        return cols

    def expected_remain(self, jt, remain):
        cols = [[None] * len(remain) for _ in self.probe_vals] if jt in (abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER) else []
        return cols + [[v[b - 1] for b in remain] for v in self.build_vals]


def _int32_range_case(rng, lo, hi, nb=3000, npr=20_000):
    bk = rng.integers(lo, hi, nb, dtype=np.int32, endpoint=True)
    bk[:2] = [lo, hi]
    specials = [v for v in (lo - 1, lo, hi, hi + 1, I32[0], I32[1], -1, 0) if I32[0] <= v <= I32[1]]
    pk = _mix(rng, npr, np.int32, [(0.5, bk), (0.3, specials)])
    pk[:len(specials)] = specials
    return JoinCase(rng, [abi.TYPE_INT], [bk], [pk], RANGE)


def _int64_range_case(rng, lo, hi, nb=3000, npr=20_000):
    bk = (np.int64(lo) + rng.integers(0, hi - lo + 1, nb, dtype=np.int64)).astype(np.int64)
    bk[:2] = [lo, hi]
    specials = [v for v in (lo - 1, lo, hi, hi + 1, I64[0], I64[0] + 1, I64[1], I64[1] - 1, -1, 0) if I64[0] <= v <= I64[1]]
    pk = _mix(rng, npr, np.int64, [(0.5, bk), (0.3, specials)])
    pk[:len(specials)] = specials
    return JoinCase(rng, [abi.TYPE_BIGINT], [bk], [pk], RANGE)


def _two_point_case(rng, a, b, method, dtype=np.int32, typ=abi.TYPE_INT):
    bk = np.array([a, b], dtype=dtype)[rng.integers(0, 2, 40)]
    specials = [v for v in (a - 1, a, a + 1, b - 1, b, b + 1, -1, 0, 1) + TYPE_RANGE[typ] if TYPE_RANGE[typ][0] <= v <= TYPE_RANGE[typ][1]]
    pk = _mix(rng, 20_000, dtype, [(0.5, bk), (0.4, specials)])
    return JoinCase(rng, [typ], [bk], [pk], method)


def _limit_case(rng, extra):
    # 102 401 distinct keys whose interval is 64 x valid (+ extra), ending at INT32_MAX; NULL rows carry the top key
    valid = 102_401
    interval = 64 * valid + extra
    base = I32[1] - interval + 1
    inner = rng.choice(interval - 2, valid - 2, replace=False) + 1
    bk = (base + np.concatenate([[0, interval - 1], inner])).astype(np.int32)
    bk = bk[rng.permutation(valid)]
    nulls = np.zeros(valid + 50, dtype=np.uint8)
    bk = np.concatenate([bk, np.full(50, I32[1], dtype=np.int32)])
    nulls[valid:] = 1
    specials = [base - 1, base, I32[1], I32[0], -1, 0]
    pk = _mix(rng, 20_000, np.int32, [(0.6, bk[:valid]), (0.2, specials)])
    case = JoinCase(rng, [abi.TYPE_INT], [bk], [pk], RANGE if extra == 0 else LINEAR, bnull=0)
    case.bnulls = [nulls]
    return case


def _pool_case(rng, ktypes, pools, method, nb=600, npr=8000):
    # keys from a small pool: fewer rows than the other cases, so that the duplicate chains keep the pair count small
    dts = [abi.TYPE_NUMPY[t] for t in ktypes]
    bks = [_pick(rng, p, nb, dt) for p, dt in zip(pools, dts)]
    pks = [_pick(rng, p, npr, dt) for p, dt in zip(pools, dts)]
    return JoinCase(rng, ktypes, bks, pks, method)


def _narrow_pool(t):
    lo, hi = TYPE_RANGE[t]
    return [lo, lo + 1, -1, 0, 1, hi - 1, hi]


def _wide_bigint_pool(rng):
    v = int(rng.integers(1, 1 << 30))
    return [v, v + (1 << 32), v + (5 << 40), v - (1 << 63) if v - (1 << 63) >= I64[0] else v, I64[0], I64[1], -1, 0, (1 << 32) - 1, -(1 << 32)]


def _fingerprint_case(rng):
    # (BIGINT, BIGINT) keys: 40 distinct keys that share one fingerprint, 12 whose fingerprint is INT64_MIN (the table's
    # empty marker, kept in the special slot), 300 random keys; every build key distinct.  The probe side also carries
    # keys with those two fingerprints that the build side does not have.
    fp = wide_fingerprint(123456789, 987654321)
    his = rng.choice(1 << 40, 80, replace=False).astype(object) - (1 << 39)
    shared = [(wrap(wide_fingerprint_lo(fp, h), 64), int(h)) for h in his[:40]]
    absent = [(wrap(wide_fingerprint_lo(fp, h), 64), int(h)) for h in his[40:60]]
    empty = [(wrap(wide_fingerprint_lo(I64[0], h), 64), int(h)) for h in his[60:72]]
    empty_absent = [(wrap(wide_fingerprint_lo(I64[0], h), 64), int(h)) for h in his[72:]]
    rand = {(int(a), int(b)) for a, b in rng.integers(I64[0], I64[1], (300, 2), dtype=np.int64)}
    build = shared + empty + sorted(rand - set(shared) - set(empty))
    build = [build[i] for i in rng.permutation(len(build))]
    probe_pool = build + absent + empty_absent
    probe = [probe_pool[i] for i in rng.integers(0, len(probe_pool), 20_000)]
    bk = [np.array([k[c] for k in build], dtype=np.int64) for c in range(2)]
    pk = [np.array([k[c] for k in probe], dtype=np.int64) for c in range(2)]
    case = JoinCase(rng, [abi.TYPE_BIGINT, abi.TYPE_BIGINT], bk, pk, LINEAR, bnull=0, pnull=0.02)
    assert all(wide_fingerprint(lo & M64, hi & M64) == fp for lo, hi in shared + absent)
    assert all(wide_fingerprint(lo & M64, hi & M64) == I64[0] for lo, hi in empty + empty_absent)
    return case


def _chunks_case(rng, shape):
    case = _int32_range_case(rng, -2000, 2000, nb=3000)
    third = case.nb // 3
    case.chunks = {"empty_first": [(0, 0, True), (0, third, True), (third, case.nb, False)],
                   "plain_then_nullable": [(0, third, False), (third, 2 * third, True), (2 * third, case.nb, False)],
                   "nullable_then_plain": [(0, third, True), (third, case.nb, False)]}[shape]
    for lo, hi, nullable in case.chunks:
        if not nullable:
            for m in case.bnulls + [case.bbign]:
                m[lo:hi] = 0
    return case


def _conjunct_case(rng):
    # BIGINT + BIGINT near +-2^63 wraps; DOUBLE comparisons with NaN and +-inf; NULLs in the build BIGINT column
    bk = rng.integers(0, 400, 3000, dtype=np.int32)
    pk = rng.integers(-10, 410, 20_000, dtype=np.int32)
    conj = [("col", P_BIG), ("col", B_BIG), "+", ("i", 0), "<", ("col", P_DBL), ("col", B_DBL), ">=", "or"]
    return JoinCase(rng, [abi.TYPE_INT], [bk], [pk], RANGE, conj=conj)


JOIN_CASES = {
    "int32_top": lambda r: _int32_range_case(r, I32[1] - 4095, I32[1]),
    "int32_bottom": lambda r: _int32_range_case(r, I32[0], I32[0] + 999),
    "int64_top": lambda r: _int64_range_case(r, I64[1] - 2999, I64[1]),
    "int64_bottom": lambda r: _int64_range_case(r, I64[0], I64[0] + 2999),
    "budget_at_limit": lambda r: _two_point_case(r, 0, 6_553_599, RANGE),
    "budget_over_limit": lambda r: _two_point_case(r, 0, 6_553_600, LINEAR),
    "interval_64_valid": lambda r: _limit_case(r, 0),
    "interval_64_valid_plus_1": lambda r: _limit_case(r, 1),
    "int64_whole_range": lambda r: _two_point_case(r, I64[0], I64[1], LINEAR, np.int64, abi.TYPE_BIGINT),
    "empty_marker_bigint": lambda r: _pool_case(r, [abi.TYPE_BIGINT], [[I64[0]] * 5 + [int(x) for x in r.integers(-(1 << 62), 1 << 62, 500)] + [I64[1], -1, 0]], LINEAR),
    "empty_marker_int_int": lambda r: _pool_case(r, [abi.TYPE_INT, abi.TYPE_INT], [[0, -1, I32[0], I32[1], 1]] * 2, LINEAR),
    "narrow_tiny_small_int": lambda r: _pool_case(r, [abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT],
                                                  [_narrow_pool(abi.TYPE_TINYINT), _narrow_pool(abi.TYPE_SMALLINT), _narrow_pool(abi.TYPE_INT)], LINEAR, nb=3000, npr=20_000),
    "narrow_small_tiny": lambda r: _pool_case(r, [abi.TYPE_SMALLINT, abi.TYPE_TINYINT], [_narrow_pool(abi.TYPE_SMALLINT), _narrow_pool(abi.TYPE_TINYINT)], LINEAR),
    "wide_int_bigint": lambda r: _pool_case(r, [abi.TYPE_INT, abi.TYPE_BIGINT], [_narrow_pool(abi.TYPE_INT), _wide_bigint_pool(r)], LINEAR),
    "wide_tiny_bigint": lambda r: _pool_case(r, [abi.TYPE_TINYINT, abi.TYPE_BIGINT], [_narrow_pool(abi.TYPE_TINYINT), _wide_bigint_pool(r)], LINEAR),
    "wide_small_bigint_small": lambda r: _pool_case(r, [abi.TYPE_SMALLINT, abi.TYPE_BIGINT, abi.TYPE_SMALLINT],
                                                    [_narrow_pool(abi.TYPE_SMALLINT), _wide_bigint_pool(r), _narrow_pool(abi.TYPE_SMALLINT)], LINEAR),
    "fingerprint_collisions": _fingerprint_case,
    "direct_tinyint": lambda r: _pool_case(r, [abi.TYPE_TINYINT], [[I8[0], I8[0] + 1, -1, 0, 1, I8[1] - 1, I8[1]] + list(range(-20, 20))], DIRECT),
    "direct_smallint": lambda r: _pool_case(r, [abi.TYPE_SMALLINT], [[I16[0], I16[0] + 1, -1, 0, 1, I16[1] - 1, I16[1]] + list(range(-300, 300, 7))], DIRECT),
    "direct_boolean": lambda r: _pool_case(r, [abi.TYPE_BOOLEAN], [[0, 1]], DIRECT, nb=40),
    "chunks_empty_first": lambda r: _chunks_case(r, "empty_first"),
    "chunks_plain_then_nullable": lambda r: _chunks_case(r, "plain_then_nullable"),
    "chunks_nullable_then_plain": lambda r: _chunks_case(r, "nullable_then_plain"),
    "conjunct_extremes": _conjunct_case,
}


@functools.lru_cache(maxsize=None)
def join_case(name):
    return JOIN_CASES[name](np.random.default_rng(2000 + sorted(JOIN_CASES).index(name)))


def _remain_rows(remain_cols):
    """build indexes of POST_PROBE output: the build row number column (slot 20)"""
    for slot, data, nulls in remain_cols:
        if slot == B_ROW:
            return data.tolist()
    raise AssertionError("no build row column")


def _force_methods(case):
    """the oracle's forced methods valid for the case: the chained ones always, the range ones when the interval over
    every build row (NULL rows too, as the oracle computes it) is small -- a forced range method allocates all of it"""
    from oracle import oracle as orc
    methods = [0, orc.LINEAR_CHAINED, orc.BUCKET_CHAINED]
    if len(case.ktypes) == 1:
        interval = int(case.bkeys[0].max()) - int(case.bkeys[0].min()) + 1
    elif sum(abi.TYPE_WIDTH[t] for t in case.ktypes) > 8:
        interval = len(set(zip(*[c.tolist() for c in case.bkeys])))      # 16-byte keys are interned: ids 0..distinct - 1
    else:
        interval = None
    if interval is not None and interval <= (1 << 23):
        methods += [orc.RANGE_DIRECT_MAPPING, orc.DENSE_RANGE_DIRECT_MAPPING]
    return methods


def _fanout_expected(nb, npr):
    pi = np.repeat(np.arange(npr, dtype=np.uint32), nb)
    bi = np.tile(np.arange(nb, 0, -1, dtype=np.uint32), npr)
    return pi, bi


FANOUT_KEY = I32[1]


def _fanout_inputs():
    build = Chunk([(10, np.full(3000, FANOUT_KEY, dtype=np.int32), None), (B_ROW, np.arange(1, 3001, dtype=np.int32), None)])
    probe = Chunk([(0, np.full(2000, FANOUT_KEY, dtype=np.int32), None), (P_ROW, np.arange(2000, dtype=np.int32), None)])
    return build, probe


def test_reference_agrees_with_the_oracle(oracle):
    # CPU only: every join case, every join type, under the oracle's own method and every forced method that applies
    bad = []
    for name in JOIN_CASES:
        case = join_case(name)
        probe = case.probe_chunk()
        for jt in JOIN_TYPES:
            pairs, remain = case.ref(jt)
            epi = np.array([p for p, _ in pairs], dtype=np.uint32)
            ebi = np.array([b for _, b in pairs], dtype=np.uint32)
            for m in _force_methods(case):
                oj = oracle.Join(case.desc(jt), force_method=m)
                for ch in case.build_chunks():
                    oj.append_build(ch)
                oj.build()
                pi, bi = oj.probe_all(probe)
                if not (np.array_equal(pi, epi) and np.array_equal(bi, ebi)):
                    bad.append(f"{name}/{JT_NAME[jt]}/method {m}: pairs differ ({len(pi)} vs {len(epi)})")
                if jt in POST_PROBE:
                    ptypes = [probe.types[probe.slots.index(s)] for s in [P_ROW, P_BIG] + list(range(len(case.ktypes)))]
                    got = _remain_rows(oj.probe_remain(ptypes))
                    if got != remain:
                        bad.append(f"{name}/{JT_NAME[jt]}/method {m}: POST_PROBE rows differ")
    build, probe = _fanout_inputs()
    oj = oracle.Join(abi.make_join_desc(abi.JOIN_INNER, [10], [0], [abi.TYPE_INT], build_out=[B_ROW], probe_out=[P_ROW]))
    oj.append_build(build)
    oj.build()
    pi, bi = oj.probe_all(probe, cap=6_000_000)
    epi, ebi = _fanout_expected(3000, 2000)
    if not (np.array_equal(pi, epi) and np.array_equal(bi, ebi)):
        bad.append("fan-out pairs differ")
    assert not bad, "; ".join(bad[:10])


# ---------------------------------------------------------------------------------------------------------------------
# standalone joins on the device
# ---------------------------------------------------------------------------------------------------------------------
def run_join(gpu, ctx, case, jt, probe):
    j = gpu.Join(ctx, case.desc(jt))
    try:
        for ch in case.build_chunks():
            j.append_build(ch)
        j.build_finish()
        info = j.info()
        out = j.probe(probe)
        n = out.num_rows
        rows = gpu.chunk_out_to_host(ctx, out)
        pi, bi = j.probe_indexes(n)
        remain = gpu.chunk_out_to_host(ctx, j.probe_remain()) if jt in POST_PROBE else None
        return info, pi, bi, rows, remain
    finally:
        j.close()


def check_join(case, jt, pi, bi, rows, remain, probe_rows=None, probe_vals=None, label=""):
    pairs, exp_remain = case.ref(jt, probe_rows)
    epi = np.array([p for p, _ in pairs], dtype=np.uint32)
    ebi = np.array([b for _, b in pairs], dtype=np.uint32)
    assert len(pi) == len(epi), f"{label}: {len(pi)} pairs, want {len(epi)}"
    bad = np.flatnonzero((pi != epi) | (bi != ebi))
    assert not len(bad), f"{label}: pair {bad[0]} is {(int(pi[bad[0]]), int(bi[bad[0]]))}, want {pairs[bad[0]]} ({len(bad)} differ)"
    got = [col_to_py(t, d, nl) for _, t, d, nl in rows]
    exp = case.expected_columns(jt, pairs, probe_vals)
    assert len(got) == len(exp), f"{label}: {len(got)} output columns, want {len(exp)}"
    for c, (g, e) in enumerate(zip(got, exp)):
        assert g == e, f"{label}: output column {c} differs"
    if jt in POST_PROBE:
        got = [col_to_py(t, d, nl) for _, t, d, nl in remain]
        assert got == case.expected_remain(jt, exp_remain), f"{label}: POST_PROBE rows differ"


@pytest.mark.gpu
@pytest.mark.parametrize("jt", JOIN_TYPES, ids=[JT_NAME[t] for t in JOIN_TYPES])
@pytest.mark.parametrize("name", list(JOIN_CASES))
def test_join_at_key_edges(gpu, ctx, name, jt):
    case = join_case(name)
    info, pi, bi, rows, remain = run_join(gpu, ctx, case, jt, case.probe_chunk())
    assert info.method == case.method, f"method {info.method}, the case is written for {case.method}"
    if name == "fingerprint_collisions":
        assert info.has_duplicates == 1, "the colliding fingerprints did not reach the table: wide_fingerprint's restatement is stale"
    check_join(case, jt, pi, bi, rows, remain, label=f"{name}/{JT_NAME[jt]}")


def _offset_device(a, offset4):
    import torch
    if not offset4:
        return torch.from_numpy(a).cuda()
    t = torch.from_numpy(np.concatenate([a[:1], a])).cuda()[1:]
    assert t.data_ptr() % 16 == 4
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["host", "device_aligned", "device_offset4"])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 1025])
def test_probe_key_layouts_and_lengths(gpu, ctx, layout, n):
    # a plain int32 key 16-byte aligned on the device takes k_probe_count's 128-bit key loads; 4 bytes off it does not.
    # The lengths leave the last 4-row group of a thread and the last 1024-row block ragged.
    case = join_case("int32_top")
    keys = case.pkeys[0][:n].copy()
    keys[: min(n, 4)] = [I32[1], I32[1] - 4096, I32[0], I32[1] - 4095][: min(n, 4)]
    keys[-1] = I32[1]
    probe_rows = [(k,) for k in keys.tolist()]
    probe_vals = [col_values(case.prow[:n], None), col_values(case.pbig[:n], None), col_values(keys, None)]
    cols = [(0, keys), (P_ROW, case.prow[:n].copy()), (P_BIG, case.pbig[:n].copy()), (P_DBL, case.pdbl[:n].copy())]
    if layout == "host":
        probe = Chunk([(s, d, None) for s, d in cols])
    else:
        probe = Chunk([(s, _offset_device(d, layout == "device_offset4" and s == 0), None) for s, d in cols], mem=abi.MEM_DEVICE)
    for jt in JOIN_TYPES:
        info, pi, bi, rows, remain = run_join(gpu, ctx, case, jt, probe)
        assert info.method == RANGE
        check_join(case, jt, pi, bi, rows, remain, probe_rows, probe_vals, label=f"{layout}/{n}/{JT_NAME[jt]}")


@pytest.mark.gpu
def test_join_fan_out(gpu, ctx):
    # one key, 3 000 build rows, 2 000 probe rows: 6 M pairs, each probe row's chain in descending build index
    build, probe = _fanout_inputs()
    j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [10], [0], [abi.TYPE_INT], build_out=[B_ROW], probe_out=[P_ROW]))
    try:
        j.append_build(build)
        j.build_finish()
        assert j.info().method == RANGE and j.info().has_duplicates == 1
        out = j.probe(probe)
        assert out.num_rows == 6_000_000
        pi, bi = j.probe_indexes(out.num_rows)
        epi, ebi = _fanout_expected(3000, 2000)
        assert np.array_equal(pi, epi) and np.array_equal(bi, ebi)
        (_, _, prow, _), (_, _, brow, _) = gpu.chunk_out_to_host(ctx, out)
        assert np.array_equal(prow, epi.astype(np.int32)) and np.array_equal(brow, ebi.astype(np.int32))
    finally:
        j.close()


@pytest.mark.gpu
def test_join_output_over_2_32_pairs_fails_loudly(gpu, ctx):
    # 70 000 x 70 000 rows of one key: 4.9e9 pairs in one batch (each 1 024-row probe block stays below 2^32).  The probe
    # refuses it instead of wrapping the 32-bit indexes, and the join stays usable.  This test is only safe while the scan
    # of the per-block pair counts (scan_counts: k_scan_counts / k_scan_lvl1<true>) sums in 64 bits: were that sum to wrap
    # again, the probe would size its index buffers from the wrapped total and write past them instead of failing here.
    # Keep that in mind when changing scan_counts.
    n = 70_000
    j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [10], [0], [abi.TYPE_INT], build_out=[B_ROW], probe_out=[P_ROW]))
    try:
        j.append_build(Chunk([(10, np.full(n, 7, dtype=np.int32), None), (B_ROW, np.arange(1, n + 1, dtype=np.int32), None)]))
        j.build_finish()
        with pytest.raises(gpu.GpuError) as ei:
            j.probe(Chunk([(0, np.full(n, 7, dtype=np.int32), None), (P_ROW, np.arange(n, dtype=np.int32), None)]))
        assert ei.value.code == abi.SR_ERR_NOT_SUPPORTED
        out = j.probe(Chunk([(0, np.array([6, 7, 8], dtype=np.int32), None), (P_ROW, np.arange(3, dtype=np.int32), None)]))
        assert out.num_rows == n
        pi, bi = j.probe_indexes(n)
        assert (pi == 1).all() and np.array_equal(bi, np.arange(n, 0, -1, dtype=np.uint32))
    finally:
        j.close()


# ---------------------------------------------------------------------------------------------------------------------
# the fragment's joins at the edges: ref_join (INNER), then ref_agg grouped by a build payload
# ---------------------------------------------------------------------------------------------------------------------
FRAG_N = 8 * 4096 + 1234               # not a multiple of STREAM_TILE (4096): the last tile is ragged
F_KEY, F_KEY2, F_VAL, F_PRED = 0, 1, 3, 4
D_KEY, D_PAY, D_KEY2 = 10, 11, 20
FRAG_FNS = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", F_VAL)]), (abi.AGG_COUNT_STAR, 0, 41, None)]
PAY_RANGE = (0, 6)
PRED_LO, PRED_HI = -40, 39                 # mode2_pred: a range conjunct on another int32 column that passes ~4 % of the rows


def _fact_keys(rng, n, bkeys, specials, dtype):
    """fact keys: build keys, the specials and uniform values; every special also sits in the first tile, in the middle
    and in the ragged last tile"""
    pool = np.array(specials, dtype=dtype)
    k = _mix(rng, n, dtype, ([(0.3, bkeys)] if len(bkeys) else []) + [(0.15, pool)])
    positions = (3, n // 2, n - 2 * len(pool) - 5)
    for p in positions:
        k[p:p + len(pool)] = pool
    return k, positions


def _specials(lo, hi, typ):
    tlo, thi = TYPE_RANGE[typ]
    return sorted({v for v in (lo - 1, lo, lo + 1, hi - 1, hi, hi + 1, tlo, thi, -1, 0) if tlo <= v <= thi})


FRAG_CASES = {
    # name: (key type, build key lo, hi, build rows, duplicates, NULL fraction of build keys)
    "guard_on_word_boundary": (abi.TYPE_INT, I32[1] - 1023, I32[1], 800, False, 0.0),
    "guard_inside_last_word": (abi.TYPE_INT, I32[0], I32[0] + 999, 800, False, 0.0),
    "global_bitmap": (abi.TYPE_INT, I32[1] - 6_553_599, I32[1], 3000, False, 0.0),
    "bigint_range_top": (abi.TYPE_BIGINT, I64[1] - 2999, I64[1], 2000, False, 0.0),
    "bigint_linear_min": (abi.TYPE_BIGINT, I64[0], I64[1], 3000, True, 0.05),
    "all_null_build": (abi.TYPE_INT, 0, -1, 500, False, 1.0),
    "empty_build": (abi.TYPE_INT, 0, -1, 0, False, 0.0),
    "expand_extremes": (abi.TYPE_INT, I32[1] - 500, I32[1], 1500, True, 0.03),
}
FRAG_VARIANTS = ["mode1", "mode2", "mode2_pred", "mode2_nullable"]


def _frag_build(rng, name):
    typ, lo, hi, nb, dups, bnull = FRAG_CASES[name]
    dt = abi.TYPE_NUMPY[typ]
    if name == "bigint_linear_min":
        pool = np.concatenate([[I64[0], I64[1], -1, 0], rng.integers(I64[0], I64[1], 1200, dtype=np.int64)])
        bk = pool[rng.integers(0, len(pool), nb)]
        bk[:6] = I64[0]
    elif nb == 0:
        bk = np.empty(0, dtype=dt)
    elif hi < lo:
        bk = rng.integers(-100, 100, nb).astype(dt)                      # all NULL: the data bytes are arbitrary
    elif dups:
        bk = (np.int64(lo) + rng.integers(0, hi - lo + 1, nb)).astype(dt)
    else:                                                               # unique keys, both ends of the range among them
        bk = (np.int64(lo) + np.concatenate([[0, hi - lo], 1 + rng.choice(hi - lo - 1, nb - 2, replace=False)])).astype(dt)
    if dups:
        bk[:2] = [lo, hi]
    bn = (rng.random(nb) < bnull).astype(np.uint8) if bnull else None
    if bn is not None and hi >= lo:
        bn[:2] = 0
    pay = rng.integers(PAY_RANGE[0], PAY_RANGE[1] + 1, nb, dtype=np.int32)
    return typ, bk, bn, pay


def _frag_expect(name, variant):
    typ, lo, hi, nb, dups, bnull = FRAG_CASES[name]
    expand = dups
    selective = variant != "mode1" or expand
    linear = name == "bigint_linear_min"
    smem = 0 if linear or name == "global_bitmap" else 1
    plan = {"mode": "selection-vector-passes" if selective else "fused-cascade", "bitmap_in_smem": [smem]}
    if selective:
        plan.update(num_stream_joins=1, final_pass="expand" if expand else "generic")
    return plan


def _run_fragment(gpu, ctx, joins, agg, fact_cols, mode, n, mem=abi.MEM_HOST, scan=None):
    frag = gpu.Fragment(ctx, scan or abi.ScanDesc(), joins, agg, mode=mode)
    try:
        cut = n // 3 + 1
        if mem == abi.MEM_HOST:
            for a, b in ((0, cut), (cut, n)):
                frag.push(Chunk([(s, d[a:b].copy(), None if nl is None else nl[a:b].copy(), t) for s, d, nl, t in fact_cols]))
        else:
            import torch
            pin = [torch.from_numpy(d).pin_memory() for _, d, _, _ in fact_cols]
            frag.push(Chunk([(s, p.data_ptr(), None, t) for (s, _, _, t), p in zip(fact_cols, pin)], num_rows=n, mem=mem))
            ctx.sync()
            del pin
        return frag.plan(), frag.rows_passed, [(t, d, nl) for _, t, d, nl in frag.agg.result()]
    finally:
        frag.close()


def _check_plan(plan, want, label):
    for k, v in want.items():
        assert plan[k] == v, f"{label}: plan {k} = {plan[k]!r}, the case is written for {v!r}"


@pytest.mark.gpu
@pytest.mark.parametrize("variant", FRAG_VARIANTS)
@pytest.mark.parametrize("name", list(FRAG_CASES))
def test_fragment_join_at_key_edges(gpu, ctx, name, variant):
    rng = np.random.default_rng(3000 + sorted(FRAG_CASES).index(name) * 10 + FRAG_VARIANTS.index(variant))
    typ, bk, bn, pay = _frag_build(rng, name)
    _, lo, hi, _, _, _ = FRAG_CASES[name]
    dt = abi.TYPE_NUMPY[typ]
    n = FRAG_N
    valid = bk if bn is None else bk[bn == 0]
    specials = _specials(lo, hi, typ) if hi >= lo else _specials(I32[0], I32[1], typ) + [0]
    if name == "bigint_linear_min":
        specials = _specials(I64[0], I64[1], typ) + [I64[0] + 1, 1]
    fk, positions = _fact_keys(rng, n, valid, specials, dt)
    fkn = None
    if variant == "mode2_nullable":
        fkn = (rng.random(n) < 0.1).astype(np.uint8)
        if len(valid):
            fk[fkn == 1] = valid[rng.integers(0, len(valid), int(fkn.sum()))]    # a NULL row's data bytes are a build key
    val = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    c = rng.integers(-1000, 1000, n, dtype=np.int32)               # PRED_LO <= c <= PRED_HI for ~4 % of the rows
    for p in positions:
        c[p:p + len(specials)] = rng.integers(PRED_LO, PRED_HI + 1, len(specials), dtype=np.int32)
    fact_cols = [(F_KEY, fk, fkn, typ), (F_VAL, val, None, abi.TYPE_BIGINT), (F_PRED, c, None, abi.TYPE_INT)]
    scan = abi.ScanDesc([abi.make_pred(F_PRED, abi.PRED_BETWEEN, PRED_LO, PRED_HI)]) if variant == "mode2_pred" else None
    d = abi.make_join_desc(abi.JOIN_INNER, [D_KEY], [F_KEY], [typ])
    j = gpu.Join(ctx, d)
    try:
        j.append_build(Chunk([(D_KEY, bk, bn, typ), (D_PAY, pay, None)]))
        j.build_finish()
        inf = j.info()
        if hi < lo:
            assert inf.method == RANGE and inf.min_value == 0 and inf.max_value == -1
        else:
            assert inf.method == (LINEAR if name == "bigint_linear_min" else RANGE)
        agg = abi.make_agg_desc([D_PAY], [abi.TYPE_INT], fns=FRAG_FNS, ranges=[PAY_RANGE])
        plan, passed, out = _run_fragment(gpu, ctx, [(j, F_KEY, [D_PAY])], agg, fact_cols, 1 if variant == "mode1" else 2, n, scan=scan)
    finally:
        j.close()
    label = f"{name}/{variant}"
    _check_plan(plan, _frag_expect(name, variant), label)
    if variant == "mode2_pred":
        assert plan["pred_rate"] < 0.08, "the predicate must pass < 8 % so that the join is a later, non-vector test"
    probe_vals = col_values(fk, fkn)
    if scan is not None:
        probe_vals = [v if PRED_LO <= cc <= PRED_HI else None for v, cc in zip(probe_vals, c.tolist())]
    pairs, _ = ref_join([(v,) for v in col_values(bk, bn)], [(v,) for v in probe_vals], abi.JOIN_INNER)
    vals, pays = val.tolist(), pay.tolist()
    cols = {D_PAY: [pays[b - 1] for _, b in pairs], F_VAL: [vals[i] for i, _ in pairs]}
    # rows_passed counts the rows that reach the aggregate: one per (fact row, build row) pair, also in the expand pass
    assert passed == len(pairs), f"{label}: {passed} rows passed, want {len(pairs)}"
    if hi < lo:
        assert passed == 0 and len(pairs) == 0
    check_agg(out, cols, {D_PAY: abi.TYPE_INT, F_VAL: abi.TYPE_BIGINT}, [D_PAY], FRAG_FNS, label)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["mode1", "mode2", "mode2_pinned"])
def test_fragment_two_joins_negative_keys(gpu, ctx, variant):
    # join A: build keys [INT32_MIN, INT32_MIN + 1999] with the group payload, ~5 % of the fact rows pass, streamed.
    # Join B: negative build keys, >= 90 % pass, tested by the final pass.  Plain int32 fact columns (the measure too),
    # so mode 2 takes the batched dense final pass: its directory lookup and its bitmap test both start at a negative
    # lo.  Pinned input carries A's key through the selection vector (k_frag_stream_tests<true>).
    rng = np.random.default_rng(77 + ["mode1", "mode2", "mode2_pinned"].index(variant))
    n = FRAG_N
    ka = (I32[0] + np.concatenate([[0, 1999], 1 + rng.choice(1998, 1698, replace=False)])).astype(np.int32)
    pay = rng.integers(PAY_RANGE[0], PAY_RANGE[1] + 1, len(ka), dtype=np.int32)
    kb = np.arange(-5000, 0, dtype=np.int32)
    kb = kb[(rng.random(len(kb)) >= 0.02) | (kb == -5000) | (kb == -1)]
    sa = _specials(I32[0], I32[0] + 1999, abi.TYPE_INT)
    sb = _specials(-5000, -1, abi.TYPE_INT)
    fa = rng.integers(0, I32[1], n, dtype=np.int32, endpoint=True)      # misses; A lets ~5 % of the rows through
    hit = rng.random(n) < 0.04
    fa[hit] = ka[rng.integers(0, len(ka), int(hit.sum()))]
    for p in (2, n // 2, n - 30):
        fa[p:p + len(sa)] = sa
    fb = np.where(rng.random(n) < 0.97, rng.integers(-5000, 0, n, dtype=np.int32), _pick(rng, sb, n, np.int32)).astype(np.int32)
    for p in (2, n // 2, n - 30):
        fb[p:p + len(sb)] = sb
    val = rng.integers(-10**6, 10**6, n, dtype=np.int32)
    fact_cols = [(F_KEY, fa, None, abi.TYPE_INT), (F_KEY2, fb, None, abi.TYPE_INT), (F_VAL, val, None, abi.TYPE_INT)]
    ja = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [D_KEY], [F_KEY], [abi.TYPE_INT]))
    jb = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [D_KEY2], [F_KEY2], [abi.TYPE_INT]))
    try:
        ja.append_build(Chunk([(D_KEY, ka, None), (D_PAY, pay, None)]))
        jb.append_build(Chunk([(D_KEY2, kb, None)]))
        for j in (ja, jb):
            j.build_finish()
            assert j.info().method == RANGE
        agg = abi.make_agg_desc([D_PAY], [abi.TYPE_INT], fns=FRAG_FNS, ranges=[PAY_RANGE])
        mem = abi.MEM_HOST_PINNED if variant == "mode2_pinned" else abi.MEM_HOST
        plan, passed, out = _run_fragment(gpu, ctx, [(ja, F_KEY, [D_PAY]), (jb, F_KEY2, [])], agg, fact_cols,
                                          1 if variant == "mode1" else 2, n, mem=mem)
    finally:
        ja.close()
        jb.close()
    if variant == "mode1":
        _check_plan(plan, {"mode": "fused-cascade", "bitmap_in_smem": [1, 1]}, variant)
    else:
        _check_plan(plan, {"mode": "selection-vector-passes", "order": [0, 1], "num_stream_joins": 1, "num_gather_passes": 0,
                           "final_pass": "dense-batched"}, variant)
        assert plan["pass_rate"][1] >= 0.9
    pa, _ = ref_join([(v,) for v in ka.tolist()], [(v,) for v in fa.tolist()], abi.JOIN_INNER)
    pb, _ = ref_join([(v,) for v in kb.tolist()], [(v,) for v in fb.tolist()], abi.JOIN_INNER)
    hit_b = {i for i, _ in pb}
    rows = [(i, b) for i, b in pa if i in hit_b]
    vals, pays = val.tolist(), pay.tolist()
    assert passed == len(rows) > 1000
    cols = {D_PAY: [pays[b - 1] for _, b in rows], F_VAL: [vals[i] for i, _ in rows]}
    types = {D_PAY: abi.TYPE_INT, F_VAL: abi.TYPE_INT}
    assert len(ref_agg(cols, types, [D_PAY], FRAG_FNS)) == PAY_RANGE[1] - PAY_RANGE[0] + 1
    check_agg(out, cols, types, [D_PAY], FRAG_FNS, variant)


# ---------------------------------------------------------------------------------------------------------------------
# runtime filters at the edges
# ---------------------------------------------------------------------------------------------------------------------
RF_TYPES = [abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_BIGINT]
RF_INFO = ("min_value", "max_value", "num_inserted", "has_null", "log_num_buckets", "key_type", "num_in_values")


def _same_info(a, b, label):
    for f in RF_INFO:
        assert getattr(a, f) == getattr(b, f), f"{label}: info.{f} {getattr(a, f)} vs {getattr(b, f)}"


def _rf_keys(rng, typ, shape, n):
    lo, hi = TYPE_RANGE[typ]
    dt = abi.TYPE_NUMPY[typ]
    nulls = (rng.random(n) < 0.1).astype(np.uint8)
    if shape == "extremes":
        k = rng.integers(lo, hi, n, dtype=dt, endpoint=True)
        edge = [lo, lo + 1, -1, 0, 1, hi - 1, hi]
        k[:len(edge)] = edge
        nulls[:len(edge)] = 0
    elif shape == "single":
        k = np.full(n, hi - 1, dtype=dt)
        nulls[0] = 0
    else:
        k = rng.integers(-50, 50, n).astype(dt)
        nulls[:] = 1
    return k, nulls


def _rf_probe(rng, typ, keys, m=8000):
    lo, hi = TYPE_RANGE[typ]
    dt = abi.TYPE_NUMPY[typ]
    edge = sorted({lo, lo + 1, -2, -1, 0, 1, hi - 2, hi - 1, hi})
    p = _mix(rng, m, dt, [(0.3, keys), (0.3, edge)])
    p[:len(edge)] = edge
    pn = (rng.random(m) < 0.05).astype(np.uint8)
    pn[:len(edge)] = 0
    return p, pn


def _check_rf_facts(sel, info, probe, pnulls, keys, knulls, with_bloom, is_in, label):
    valid = [int(v) for v, nl in zip(keys.tolist(), knulls.tolist()) if not nl]
    vals = probe.tolist()
    pn = pnulls.astype(bool)
    sel = sel.astype(bool)
    if valid:
        assert (info.min_value, info.max_value) == (min(valid), max(valid)), f"{label}: min / max"
    else:
        assert info.num_inserted == 0
    assert (sel[pn] == bool(info.has_null)).all(), f"{label}: NULL rows"
    in_range = np.array([bool(valid) and min(valid) <= v <= max(valid) for v in vals])
    members = np.isin(np.array(vals, dtype=np.int64), np.array(valid, dtype=np.int64))
    nn = ~pn
    if not with_bloom:
        assert np.array_equal(sel[nn], in_range[nn]), f"{label}: the range filter is not exact"
    elif is_in:
        assert np.array_equal(sel[nn], members[nn]), f"{label}: the IN filter is not exact"
    else:
        assert sel[nn & members].all(), f"{label}: bloom false negative"
        assert not sel[nn & ~in_range].any(), f"{label}: a value outside [min, max] passed"
    if valid:
        lo, hi = TYPE_RANGE[abi.NUMPY_TYPE[probe.dtype]]
        for v in (min(valid) - 1, max(valid) + 1):
            if lo <= v <= hi:
                assert not sel[nn & (np.array(vals) == v)].any(), f"{label}: {v} passed, outside [min, max]"


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["in_filter", "bloom"])
@pytest.mark.parametrize("shape", ["extremes", "single", "all_null"])
@pytest.mark.parametrize("typ", RF_TYPES)
def test_runtime_filter_at_extremes(gpu, ctx, oracle, typ, shape, size):
    rng = np.random.default_rng(typ * 100 + ["extremes", "single", "all_null"].index(shape) * 10 + (size == "bloom"))
    n = 700 if size == "in_filter" else 5000
    keys, knulls = _rf_keys(rng, typ, shape, n)
    probe, pnulls = _rf_probe(rng, typ, keys[knulls == 0] if (knulls == 0).any() else keys)
    pch = Chunk([(3, probe, pnulls, typ)])
    pch_plain = Chunk([(3, probe.copy(), None, typ)])
    half = n // 2
    b1 = Chunk([(0, keys[:half].copy(), knulls[:half].copy(), typ)])
    b2 = Chunk([(0, keys[half:].copy(), knulls[half:].copy(), typ)])
    prior = rng.integers(0, 2, len(probe)).astype(np.uint8)
    for with_bloom in (True, False):
        label = f"bloom={with_bloom}"
        is_in = with_bloom and n <= abi.RF_IN_FILTER_ROW_LIMIT
        g, o = gpu.RuntimeFilter(ctx, typ, n, with_bloom), oracle.RuntimeFilter(typ, n, with_bloom)
        e, oe = gpu.RuntimeFilter(ctx, typ, n, with_bloom), oracle.RuntimeFilter(typ, n, with_bloom)
        j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [0], [3], [typ]))
        scan = gpu.Scan(ctx, abi.ScanDesc(out_slots=[3]))
        try:
            for f in (g, o):
                f.insert(b1, 0)
                f.insert(b2, 0, insert_nulls=True)
            _same_info(g.info(), o.info(), label)
            assert np.array_equal(g.directory(), o.directory()), f"{label}: directory"
            sel = g.evaluate(pch, 3)
            assert np.array_equal(sel, o.evaluate(pch, 3)), f"{label}: selection"
            assert np.array_equal(g.evaluate(pch, 3, prior), o.evaluate(pch, 3, prior)), f"{label}: selection over a prior one"
            if is_in and (knulls == 0).any():
                assert g.in_values().tolist() == sorted(set(int(v) for v in keys[knulls == 0].tolist()))
            _check_rf_facts(sel, g.info(), probe, pnulls, keys, knulls, with_bloom, is_in, label)
            # a scan with the filter attached (rf_test_rows), with and without NULLs in the probe column
            scan.add_runtime_filter(g, 3)
            scan.set_rf_adaptive(False)                   # an unselective filter stays on for every batch
            for ch in (pch, pch_plain):
                sd = abi.ScanDesc(out_slots=[3])
                assert np.array_equal(scan.evaluate(ch), o.evaluate(ch, 3, oracle.scan_evaluate(sd, ch))), f"{label}: scan"
            # the filter a join publishes for its key
            j.append_build(b1)
            j.append_build(b2)
            j.build_finish()
            jf = gpu.RuntimeFilter.from_join(j, 0, with_bloom, insert_nulls=True)
            try:
                oj = oracle.RuntimeFilter(typ, n, with_bloom)
                oj.insert(Chunk([(0, keys, knulls, typ)]), 0, insert_nulls=True)
                _same_info(jf.info(), oj.info(), f"{label} from_join")
                assert np.array_equal(jf.directory(), oj.directory()), f"{label} from_join: directory"
                assert np.array_equal(jf.evaluate(pch, 3), oj.evaluate(pch, 3)), f"{label} from_join: selection"
            finally:
                jf.close()
            # an empty filter merged into the full one changes nothing
            g.merge(e.directory(), e.info())
            o.merge(oe)
            before = g.in_values()
            g.merge_in_values(e.in_values())
            _same_info(g.info(), o.info(), f"{label} merged")
            assert np.array_equal(g.directory(), o.directory()), f"{label} merged: directory"
            assert np.array_equal(g.evaluate(pch, 3), sel), f"{label} merged: selection changed"
            got = g.in_values()
            assert (got is None and before is None) or np.array_equal(got, before)
        finally:
            scan.close()
            j.close()
            for f in (g, e):
                f.close()
