"""Aggregate, scan and fragment kernels at the edges of their value domains, against an exact reference in plain Python.

The parity tests elsewhere compare the kernels with the CPU oracle on moderate random values.  Here the inputs sit where
the delicate code is: 64- and 128-bit sums that wrap and carry, MIN / MAX at the accumulator sentinels, doubles with
signs, infinities, subnormals and -0.0, group keys at their type's extremes and all-ones packed images, declared key
ranges met by keys near the int64 extremes, and predicate constants at and beyond the column type's range.  The
reference below uses Python ints, math.fsum and dicts only, so it shares no code (and no numpy reduction) with either
implementation; `test_reference_agrees_with_the_oracle` checks it against the oracle on the CPU before it judges the
kernels.  Every other test needs the device and is marked `gpu`.
"""
import math
import os

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

I8, I16, I32, I64 = (-(1 << 7), (1 << 7) - 1), (-(1 << 15), (1 << 15) - 1), (-(1 << 31), (1 << 31) - 1), (-(1 << 63), (1 << 63) - 1)
INF, NAN = float("inf"), float("nan")
FLOATS = (abi.TYPE_FLOAT, abi.TYPE_DOUBLE)
TYPE_RANGE = {abi.TYPE_BOOLEAN: (0, 1), abi.TYPE_TINYINT: I8, abi.TYPE_SMALLINT: I16, abi.TYPE_INT: I32, abi.TYPE_DATE: I32,
              abi.TYPE_DECIMAL32: I32, abi.TYPE_BIGINT: I64, abi.TYPE_DECIMAL64: I64}


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def wrap(v, bits):
    """two's complement wrap of a Python int to `bits` bits"""
    m = 1 << bits
    v &= m - 1
    return v - m if v >> (bits - 1) else v


def col_values(data, nulls):
    """numpy column -> Python values (None for NULL); FLOAT values are the exact float32 values as Python floats"""
    vals = data.tolist()
    if nulls is not None:
        vals = [None if nl else v for v, nl in zip(vals, nulls.tolist())]
    return vals


def ref_expr(rpn, cols, types, i):
    """evaluate an abi.make_expr token list on row i -> (value, is_null).  Integer arithmetic wraps at 64 bits, '/' and
    any operand of a DOUBLE make the operation DOUBLE, a zero divisor (-0.0 too) gives NULL, comparisons give 0 / 1
    (false for NaN), AND / OR are SQL's three-valued logic."""
    st = []     # (value, is_null, is_double)
    for tok in rpn:
        if isinstance(tok, tuple):
            kind, x = tok
            if kind == "col":
                v = cols[x][i]
                st.append((v, v is None, types[x] in FLOATS))
            else:
                st.append((float(x) if kind == "d" else int(x), False, kind == "d"))
            continue
        if tok == "todouble":
            v, nl, d = st.pop()
            st.append((v if d or nl else float(v), nl, True))
            continue
        if tok == "isnull":
            v, nl, d = st.pop()
            st.append((1 if nl else 0, False, False))
            continue
        if tok == "not":
            v, nl, d = st.pop()
            st.append((None if nl else (0 if v else 1), nl, False))
            continue
        (a, an, ad), (b, bn, bd) = st.pop(-2), st.pop()
        if tok in ("and", "or"):
            av, bv = (not an and a != 0), (not bn and b != 0)
            af, bf = (not an and not av), (not bn and not bv)
            if tok == "and":
                rv, rn = not (af or bf) and not (an or bn), not (af or bf) and (an or bn)
            else:
                rv, rn = av or bv, not (av or bv) and (an or bn)
            st.append((1 if rv else 0, rn, False))
            continue
        dbl = ad or bd or tok == "/"
        if an or bn:
            st.append((None, True, dbl and tok in "+-*/"))
            continue
        if dbl:
            a, b = float(a), float(b)
        if tok in ("+", "-", "*"):
            r = a + b if tok == "+" else a - b if tok == "-" else a * b
            st.append((r if dbl else wrap(r, 64), False, dbl))
        elif tok == "/":
            st.append((None, True, True) if b == 0.0 else (a / b, False, True))
        else:
            r = {"==": a == b, "!=": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[tok]
            st.append((1 if r else 0, False, False))
    (v, nl, _), = st
    return (None if nl else v), nl


def ref_pred(op, v, lo=0, hi=0, in_list=()):
    """a ColumnPredicate on one value (None = NULL): Python comparisons, so NaN compares false and NE is true for it"""
    if op == abi.PRED_IS_NULL:
        return v is None
    if op == abi.PRED_IS_NOT_NULL:
        return v is not None
    if v is None:
        return False
    if op == abi.PRED_IN:
        return v in in_list
    if op == abi.PRED_NOT_IN:
        return v not in in_list
    return {abi.PRED_EQ: v == lo, abi.PRED_NE: v != lo, abi.PRED_LT: v < lo, abi.PRED_LE: v <= lo, abi.PRED_GT: v > lo,
            abi.PRED_GE: v >= lo, abi.PRED_BETWEEN: lo <= v <= hi}[op]


class DoubleSum:
    """expected SUM (or AVG, count > 0) of DOUBLE inputs: NaN when a NaN or both infinities are summed, the infinity
    when one is, else math.fsum within (n + 1) 2^-52 sum|x| -- a bound that holds whatever the summation order"""

    def __init__(self, xs, count=None):
        self.xs, self.count = xs, count

    def check(self, got):
        xs, c = self.xs, self.count or 1
        pinf, ninf = INF in xs, -INF in xs
        if any(math.isnan(x) for x in xs) or (pinf and ninf):
            return got is not None and math.isnan(got)
        if pinf or ninf:
            return got == (INF if pinf else -INF) / c
        exp = math.fsum(xs) / c
        bound = (len(xs) + 1) * 2.0 ** -52 * math.fsum(abs(x) for x in xs) / c + 2.0 ** -52 * abs(exp)
        return got is not None and abs(got - exp) <= bound

    def __repr__(self):
        return f"DoubleSum(fsum={math.fsum(x for x in self.xs if math.isfinite(x))}, n={len(self.xs)}, count={self.count})"


def ref_agg(cols, types, key_slots, fns):
    """cols: {slot: Python values}; fns: (kind, input_type, out_slot, rpn) as abi.make_agg_desc takes them.
    -> {key tuple: [expected result per function]}; DOUBLE sums and averages are DoubleSum objects"""
    n = len(next(iter(cols.values())))
    groups = {}
    for i in range(n):
        key = tuple(cols[s][i] for s in key_slots)
        acc = groups.get(key)
        if acc is None:
            acc = groups[key] = [0] + [[] for _ in fns]
        acc[0] += 1
        for f, (kind, _, _, rpn) in enumerate(fns):
            if kind != abi.AGG_COUNT_STAR:
                v, nl = ref_expr(rpn, cols, types, i)
                if not nl:
                    acc[1 + f].append(v)
    out = {}
    for key, acc in groups.items():
        res = []
        for f, (kind, ityp, _, _) in enumerate(fns):
            xs = acc[1 + f]
            rt = abi.agg_result_type(kind, ityp)
            if kind == abi.AGG_COUNT_STAR:
                res.append(acc[0])
            elif kind == abi.AGG_COUNT:
                res.append(len(xs))
            elif not xs:
                res.append(None)
            elif kind == abi.AGG_SUM:
                res.append(DoubleSum(xs) if rt == abi.TYPE_DOUBLE else wrap(sum(xs), abi.TYPE_WIDTH[rt] * 8))
            elif kind == abi.AGG_AVG:
                res.append(DoubleSum([float(x) for x in xs], len(xs)))
            else:
                res.append(min(xs) if kind == abi.AGG_MIN else max(xs))
        out[key] = res
    return out


def check_agg(out_cols, cols, types, key_slots, fns, label=""):
    """out_cols: [(type, data, nulls)] keys first, then one column per function (GPU or oracle) -> assert they are the
    reference's answer: exact, by value for floats (-0.0 == 0.0), DoubleSum within its bound, NULL where a group has no
    non-NULL input"""
    from starrocks_b200.rows import col_to_py
    exp = ref_agg(cols, types, key_slots, fns)
    nk = len(key_slots)
    want_types = [types[s] for s in key_slots] + [abi.agg_result_type(k, t) for k, t, _, _ in fns]
    assert [t for t, _, _ in out_cols] == want_types, f"{label}: result types"
    pyc = [col_to_py(t, d, nl) for t, d, nl in out_cols]
    got = {tuple(r[:nk]): list(r[nk:]) for r in zip(*pyc)} if pyc else {}
    assert set(got) == set(exp), f"{label}: groups {sorted(got, key=repr)[:8]} vs {sorted(exp, key=repr)[:8]}"
    bad = []
    for key, er in exp.items():
        for f, (e, g) in enumerate(zip(er, got[key])):
            ok = e.check(g) if isinstance(e, DoubleSum) else (g is None if e is None else (g is not None and g == e))
            if not ok:
                bad.append(f"group {key} fn {f}: got {g!r}, want {e!r}")
    assert not bad, f"{label}: " + "; ".join(bad[:6])


# ---------------------------------------------------------------------------------------------------------------------
# aggregate cases: crafted rows over random filler in 7 groups (g = 0..6), value columns at slots >= 10
# ---------------------------------------------------------------------------------------------------------------------
def _in_group(g, k, m=1):
    return np.flatnonzero(g == k)[:m]


def _case_bigint(rng, n):
    # SUM over +-2^62 + noise: wraps many times, most low-word adds carry; MIN / MAX at INT64_MIN / INT64_MAX, which are
    # the accumulators' initial values; a nullable column with an all-NULL group and groups whose only value is a sentinel
    g = rng.integers(0, 7, n)
    sign = np.where(rng.random(n) < 0.5, -1, 1).astype(np.int64)
    v = sign * ((1 << 62) + rng.integers(0, 1 << 40, n, dtype=np.int64))
    v[g == 0] = np.abs(v[g == 0])
    v[_in_group(g, 1)] = I64[1]
    v[_in_group(g, 2)] = I64[0]
    w = rng.integers(I64[0], I64[1], n, dtype=np.int64, endpoint=True)
    wn = (rng.random(n) < 0.3).astype(np.uint8)
    wn[g >= 4] = 1
    for grp, val in ((4, I64[1]), (5, I64[0])):
        i = _in_group(g, grp)
        w[i], wn[i] = val, 0
    cols = [(10, v, None, abi.TYPE_BIGINT), (11, w, wn, abi.TYPE_BIGINT)]
    fns = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 10)]), (abi.AGG_MIN, abi.TYPE_BIGINT, 41, [("col", 10)]),
           (abi.AGG_MAX, abi.TYPE_BIGINT, 42, [("col", 10)]), (abi.AGG_COUNT_STAR, 0, 43, None),
           (abi.AGG_SUM, abi.TYPE_BIGINT, 44, [("col", 11)]), (abi.AGG_MIN, abi.TYPE_BIGINT, 45, [("col", 11)]),
           (abi.AGG_MAX, abi.TYPE_BIGINT, 46, [("col", 11)]), (abi.AGG_COUNT, abi.TYPE_BIGINT, 47, [("col", 11)])]
    return g, cols, fns


def _case_decimal(rng, n):
    # SUM(DECIMAL64) -> DECIMAL128: group 0 climbs far past 2^64, group 1 alternates INT64_MAX / INT64_MIN (crosses 2^64
    # and comes back through zero, in whatever order the device adds), group 2 descends past -2^64
    g = rng.integers(0, 7, n)
    v = rng.integers(I64[0], I64[1], n, dtype=np.int64, endpoint=True)
    v[g == 0] = I64[1] - rng.integers(0, 1 << 20, int((g == 0).sum()), dtype=np.int64)
    i1 = np.flatnonzero(g == 1)
    v[i1] = np.where(np.arange(len(i1)) % 2 == 0, I64[1], I64[0])
    v[g == 2] = I64[0]
    w = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    wn = (rng.random(n) < 0.25).astype(np.uint8)
    wn[g == 6] = 1
    cols = [(12, v, None, abi.TYPE_DECIMAL64), (13, w, wn, abi.TYPE_DECIMAL64)]
    fns = [(abi.AGG_SUM, abi.TYPE_DECIMAL64, 40, [("col", 12)]), (abi.AGG_SUM, abi.TYPE_DECIMAL64, 41, [("col", 13)]),
           (abi.AGG_COUNT, abi.TYPE_DECIMAL64, 42, [("col", 13)]), (abi.AGG_COUNT_STAR, 0, 43, None),
           (abi.AGG_MIN, abi.TYPE_DECIMAL64, 44, [("col", 12)]), (abi.AGG_MAX, abi.TYPE_DECIMAL64, 45, [("col", 13)])]
    return g, cols, fns


def _case_int32(rng, n):
    # runs of INT32_MAX / INT32_MIN: the BIGINT sum must not truncate to 32 bits.  Plain non-NULL int32 columns and at
    # most four functions besides COUNT(*), so that a fragment's final pass may take the batched dense kernel
    g = rng.integers(0, 7, n)
    v = rng.integers(I32[0], I32[1], n, dtype=np.int32, endpoint=True)
    v[g == 0] = I32[1]
    v[g == 1] = I32[0]
    i2 = np.flatnonzero(g == 2)
    v[i2] = np.where(np.arange(len(i2)) % 3 == 0, I32[0], I32[1])
    w = rng.integers(-5, 6, n, dtype=np.int32)
    w[_in_group(g, 3)] = I32[0]
    w[_in_group(g, 4)] = I32[1]
    cols = [(14, v, None, abi.TYPE_INT), (15, w, None, abi.TYPE_INT)]
    fns = [(abi.AGG_SUM, abi.TYPE_INT, 40, [("col", 14)]), (abi.AGG_MIN, abi.TYPE_INT, 41, [("col", 15)]),
           (abi.AGG_MAX, abi.TYPE_INT, 42, [("col", 15)]), (abi.AGG_COUNT_STAR, 0, 43, None),
           (abi.AGG_SUM, abi.TYPE_INT, 44, [("col", 15)])]
    return g, cols, fns


def _case_narrow(rng, n):
    # MIN / MAX of TINYINT / SMALLINT at their extremes, returned at their own width; group 0 holds only the minimum and
    # group 1 only the maximum, so a value widened without its sign, or truncated wrongly, shows
    g = rng.integers(0, 7, n)
    t = rng.integers(I8[0], I8[1], n, dtype=np.int8, endpoint=True)
    s = rng.integers(I16[0], I16[1], n, dtype=np.int16, endpoint=True)
    t[g == 0], s[g == 0] = I8[0], I16[0]
    t[g == 1], s[g == 1] = I8[1], I16[1]
    sn = (rng.random(n) < 0.2).astype(np.uint8)
    sn[g == 6] = 1
    cols = [(16, t, None, abi.TYPE_TINYINT), (17, s, sn, abi.TYPE_SMALLINT)]
    fns = [(abi.AGG_MIN, abi.TYPE_TINYINT, 40, [("col", 16)]), (abi.AGG_MAX, abi.TYPE_TINYINT, 41, [("col", 16)]),
           (abi.AGG_SUM, abi.TYPE_TINYINT, 42, [("col", 16)]), (abi.AGG_MIN, abi.TYPE_SMALLINT, 43, [("col", 17)]),
           (abi.AGG_MAX, abi.TYPE_SMALLINT, 44, [("col", 17)]), (abi.AGG_SUM, abi.TYPE_SMALLINT, 45, [("col", 17)]),
           (abi.AGG_COUNT_STAR, 0, 46, None)]
    return g, cols, fns


def _fill_doubles(rng, g, dt, tiny, huge):
    n = len(g)
    x = (rng.standard_normal(n) * 1e3).astype(dt)
    x[g == 0] = -(rng.random(int((g == 0).sum())) * huge + tiny).astype(dt)          # all negative
    i1 = _in_group(g, 1, 2)
    x[i1] = np.array([INF, -INF], dtype=dt)                                        # both infinities among finite values
    x[g == 2] = (np.where(rng.random(int((g == 2).sum())) < 0.5, -1, 1) * tiny * rng.integers(1, 4, int((g == 2).sum()))).astype(dt)
    x[g == 3] = np.where(rng.random(int((g == 3).sum())) < 0.5, -0.0, 0.0).astype(dt)  # only zeros of both signs
    x[g == 4] = dt(-0.0)
    x[g == 5] = (-rng.random(int((g == 5).sum())) * huge).astype(dt)
    x[_in_group(g, 5)] = dt(-INF)
    return x


def _case_double_minmax(rng, n):
    g = rng.integers(0, 7, n)
    d = _fill_doubles(rng, g, np.float64, 5e-324, 1e300)
    f = _fill_doubles(rng, g, np.float32, np.float32(1e-45), np.float32(1e38))
    dn = (rng.random(n) < 0.3).astype(np.uint8)
    dn[g == 6] = 1
    cols = [(20, d, None, abi.TYPE_DOUBLE), (21, f, None, abi.TYPE_FLOAT), (22, d.copy(), dn, abi.TYPE_DOUBLE)]
    fns = [(abi.AGG_MIN, abi.TYPE_DOUBLE, 40, [("col", 20)]), (abi.AGG_MAX, abi.TYPE_DOUBLE, 41, [("col", 20)]),
           (abi.AGG_MIN, abi.TYPE_FLOAT, 42, [("col", 21)]), (abi.AGG_MAX, abi.TYPE_FLOAT, 43, [("col", 21)]),
           (abi.AGG_COUNT_STAR, 0, 44, None), (abi.AGG_MIN, abi.TYPE_DOUBLE, 45, [("col", 22)]),
           (abi.AGG_MAX, abi.TYPE_DOUBLE, 46, [("col", 22)])]
    return g, cols, fns


def _case_double_sum(rng, n):
    # heavy cancellation (1e16, 1, -1e16 triples: the exact sum is the number of ones), +-inf, inf + -inf and NaN
    # (SUM / AVG propagate them; NaN never reaches MIN / MAX here, where its order is not defined)
    g = rng.integers(0, 7, n)
    x = rng.standard_normal(n) * 1e3
    i0 = np.flatnonzero(g == 0)
    x[i0] = np.array([1e16, 1.0, -1e16])[np.arange(len(i0)) % 3]
    i1 = np.flatnonzero(g == 1)
    x[i1] = np.where(np.arange(len(i1)) % 2 == 0, 1e15, -1e15) + rng.random(len(i1))
    x[_in_group(g, 2)] = INF
    x[_in_group(g, 3)] = -INF
    x[_in_group(g, 4, 2)] = [INF, -INF]
    x[_in_group(g, 5)] = NAN
    y = np.where(rng.random(n) < 0.5, 1e300, -1e300) * rng.random(n)
    yn = (rng.random(n) < 0.3).astype(np.uint8)
    yn[g == 6] = 1
    f = (rng.standard_normal(n) * 1e30).astype(np.float32)
    cols = [(23, x, None, abi.TYPE_DOUBLE), (24, y, yn, abi.TYPE_DOUBLE), (25, f, None, abi.TYPE_FLOAT)]
    # two AVGs: each is two first-phase functions, and the two-phase split must fit SR_MAX_AGG_FNS
    fns = [(abi.AGG_SUM, abi.TYPE_DOUBLE, 40, [("col", 23)]), (abi.AGG_AVG, abi.TYPE_DOUBLE, 41, [("col", 23)]),
           (abi.AGG_SUM, abi.TYPE_DOUBLE, 42, [("col", 24)]), (abi.AGG_AVG, abi.TYPE_DOUBLE, 43, [("col", 24)]),
           (abi.AGG_SUM, abi.TYPE_FLOAT, 44, [("col", 25)]), (abi.AGG_COUNT_STAR, 0, 45, None)]
    return g, cols, fns


def _case_expr(rng, n):
    # eval_expr at the int64 extremes: a * b, a + k, a - b wrap (three-node fast forms), longer stack programs, INT64_MAX
    # converted to DOUBLE, division by -0.0 (NULL), and three-valued AND / OR counted through COUNT(expr)
    g = rng.integers(0, 7, n)
    a = rng.integers(I64[0], I64[1], n, dtype=np.int64, endpoint=True)
    a[g == 0] = I64[1]
    a[g == 1] = I64[0]
    b = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    b[_in_group(g, 2, 4)] = [I64[0], I64[1], -1, 3]
    bn = (rng.random(n) < 0.2).astype(np.uint8)
    x = rng.standard_normal(n) * 1e6
    y = rng.standard_normal(n)
    y[rng.random(n) < 0.2] = -0.0
    y[rng.random(n) < 0.1] = 0.0
    cols = [(26, a, None, abi.TYPE_BIGINT), (27, b, bn, abi.TYPE_BIGINT), (28, x, None, abi.TYPE_DOUBLE), (29, y, None, abi.TYPE_DOUBLE)]
    fns = [(abi.AGG_SUM, abi.TYPE_BIGINT, 40, [("col", 26), ("col", 27), "*"]),
           (abi.AGG_SUM, abi.TYPE_BIGINT, 41, [("col", 26), ("i", I64[1]), "+"]),
           (abi.AGG_SUM, abi.TYPE_BIGINT, 42, [("col", 26), ("col", 27), "-", ("i", 3), "*", ("col", 26), "+"]),
           (abi.AGG_SUM, abi.TYPE_DOUBLE, 43, [("col", 26), "todouble"]),
           (abi.AGG_SUM, abi.TYPE_DOUBLE, 44, [("col", 28), ("col", 29), "/"]),
           (abi.AGG_COUNT, abi.TYPE_DOUBLE, 45, [("col", 28), ("col", 29), "/"]),
           (abi.AGG_COUNT, abi.TYPE_BIGINT, 46, [("col", 27), ("i", 0), ">", ("col", 29), ("d", 0.0), "<", "and"]),
           (abi.AGG_SUM, abi.TYPE_BIGINT, 47, [("col", 27), ("i", 0), ">", ("col", 26), ("i", 0), "<", "or"])]
    return g, cols, fns


AGG_CASES = {"bigint": _case_bigint, "decimal": _case_decimal, "int32": _case_int32, "narrow": _case_narrow,
             "double_minmax": _case_double_minmax, "double_sum": _case_double_sum, "expr": _case_expr}
CASE_SEED = {name: 1000 + k for k, name in enumerate(AGG_CASES)}

# group keys of each aggregate path, derived from g: slot 0 = g (INT), slot 1 = 1429 g (INT, declared 0..9999: a dense
# table beyond 40 KB of state lives in global memory), slot 2 = a BIGINT image of g (INT + BIGINT = a 12-byte hash key)
PATH_KEYS = {"nogroup": ([], [], None), "dense_smem": ([0], [abi.TYPE_INT], [(0, 6)]),
             "dense_global": ([1], [abi.TYPE_INT], [(0, 9999)]), "hash8": ([0], [abi.TYPE_INT], None),
             "hash16": ([0, 2], [abi.TYPE_INT, abi.TYPE_BIGINT], None), "part": ([0], [abi.TYPE_INT], None),
             "part_l2": ([0], [abi.TYPE_INT], None), "two_phase": ([0], [abi.TYPE_INT], None),
             "dense_state": ([0], [abi.TYPE_INT], [(0, 6)]), "frag1": ([0], [abi.TYPE_INT], [(0, 6)]),
             "frag2": ([0], [abi.TYPE_INT], [(0, 6)])}
N_ROWS = 6000


def build_case(name, path="hash8", n=N_ROWS):
    g, vcols, fns = AGG_CASES[name](np.random.default_rng(CASE_SEED[name]), n)
    key_cols = {0: (g.astype(np.int32), abi.TYPE_INT), 1: ((g * 1429).astype(np.int32), abi.TYPE_INT),
                2: (g.astype(np.int64) * 1_000_000_007 - 3, abi.TYPE_BIGINT)}
    slots, ktypes, ranges = PATH_KEYS[path]
    cols = [(s, key_cols[s][0], None, key_cols[s][1]) for s in slots] + vcols
    desc = abi.make_agg_desc(slots, ktypes, fns=fns, ranges=ranges)
    return desc, cols, slots, fns


def py_cols(cols):
    return {c[0]: col_values(c[1], c[2]) for c in cols}, {c[0]: c[3] for c in cols}


def sub_chunk(cols, lo, hi):
    return Chunk([(s, d[lo:hi].copy(), None if nl is None else nl[lo:hi].copy(), t) for s, d, nl, t in cols])


# two-phase aggregation and the element-wise dense merge have no 128-bit intermediate states
AGG_PARAMS = [(c, p) for c in AGG_CASES for p in PATH_KEYS if not (c == "decimal" and p in ("two_phase", "dense_state"))]


def test_reference_agrees_with_the_oracle(oracle):
    # CPU only: every aggregate case, grouped and not, through the oracle and the reference
    for name in AGG_CASES:
        for path in ("hash8", "nogroup", "hash16"):
            desc, cols, slots, fns = build_case(name, path)
            oa = oracle.Agg(desc)
            oa.push(sub_chunk(cols, 0, 1000))
            oa.push(sub_chunk(cols, 1000, N_ROWS))
            pc, types = py_cols(cols)
            check_agg(oa.output(), pc, types, slots, fns, f"oracle {name}/{path}")


def test_reference_known_answers():
    assert wrap((1 << 63) + 5, 64) == -(1 << 63) + 5 and wrap(-(1 << 127) - 1, 128) == (1 << 127) - 1
    assert ref_expr([("col", 0), ("col", 1), "*"], {0: [I64[1]], 1: [2]}, {0: abi.TYPE_BIGINT, 1: abi.TYPE_BIGINT}, 0) == (-2, False)
    assert ref_expr([("d", 1.0), ("d", -0.0), "/"], {}, {}, 0) == (None, True)
    t = {0: abi.TYPE_BIGINT}
    assert ref_expr([("col", 0), ("i", 0), ">", ("i", 0), ("i", 1), ">", "and"], {0: [None]}, t, 0) == (0, False)   # NULL AND false
    assert ref_expr([("col", 0), ("i", 0), ">", ("i", 1), ("i", 0), ">", "or"], {0: [None]}, t, 0) == (1, False)    # NULL OR true
    assert ref_expr([("col", 0), ("i", 0), ">", ("i", 1), ("i", 0), ">", "and"], {0: [None]}, t, 0) == (None, True)
    assert not ref_pred(abi.PRED_LT, NAN, 1.0) and ref_pred(abi.PRED_NE, NAN, 1.0) and not ref_pred(abi.PRED_EQ, None, 0)
    assert DoubleSum([1e16, 1.0, -1e16]).check(1.0) and not DoubleSum([1e16, 1.0, -1e16, 1.0]).check(50.0)
    assert DoubleSum([INF, 1.0]).check(INF) and DoubleSum([INF, -INF]).check(NAN) and DoubleSum([NAN, 1.0], 2).check(NAN)


# ---------------------------------------------------------------------------------------------------------------------
# aggregate cases x every path that applies them
# ---------------------------------------------------------------------------------------------------------------------
def _host_cols(res):
    return [(t, d, nl) for _, t, d, nl in res]


def run_agg_path(gpu, ctx, path, desc, cols, monkeypatch, batched=False):
    """push the case through one aggregate path -> result columns [(type, data, nulls)]"""
    n = len(cols[0][1])
    cut = n // 3
    halves = ((0, cut), (cut, n))
    if path.startswith("frag"):
        mode = 1 if path == "frag1" else 2
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [], desc, mode=mode)
        try:
            for lo, hi in halves:
                frag.push(sub_chunk(cols, lo, hi))
            plan = frag.plan()
            assert plan["mode"] == ("fused-cascade" if mode == 1 else "selection-vector-passes")
            if mode == 2:   # plain int32 columns only (the "int32" case) take the batched dense kernel
                assert plan["final_pass"] == ("dense-batched" if batched else "generic")
            assert frag.rows_passed == n
            return _host_cols(frag.agg.result())
        finally:
            frag.close()
    if path == "two_phase":
        p1, p2 = gpu.two_phase_descs(desc)
        first, final = gpu.Agg(ctx, p1), gpu.Agg(ctx, p2)
        try:
            first.push(sub_chunk(cols, *halves[0]))       # pre-aggregated, pulled as a device chunk
            first.finish()
            final.push(gpu.chunk_out_as_view(first.pull(mem=abi.MEM_DEVICE)))
            final.push(gpu.chunk_out_as_view(first.convert_to_states(sub_chunk(cols, *halves[1]))))   # passed through
            return _host_cols(final.result())
        finally:
            first.close()
            final.close()
    if path == "dense_state":
        import torch
        from starrocks_b200.distributed import dense_state_views
        a, b = gpu.Agg(ctx, desc), gpu.Agg(ctx, desc)
        try:
            a.push(sub_chunk(cols, *halves[0]))
            b.push(sub_chunk(cols, *halves[1]))
            ctx.sync()
            for (ta, ra), (tb, _) in zip(dense_state_views(a.dense_state(), "cuda:0"), dense_state_views(b.dense_state(), "cuda:0")):
                ta.copy_(ta + tb if ra == abi.STATE_REDUCE_SUM else torch.minimum(ta, tb) if ra == abi.STATE_REDUCE_MIN else torch.maximum(ta, tb))
            torch.cuda.synchronize()
            return _host_cols(a.result())
        finally:
            a.close()
            b.close()
    if path.startswith("part"):
        monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", "1000")
        if path == "part_l2":
            monkeypatch.setenv("SR_AGG_PARTITION_FORCE_L2", "1")
    a = gpu.Agg(ctx, desc)
    try:
        for lo, hi in halves:
            a.push(sub_chunk(cols, lo, hi))
        return _host_cols(a.result())
    finally:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,path", AGG_PARAMS)
def test_agg_value_edges(gpu, ctx, monkeypatch, name, path):
    desc, cols, slots, fns = build_case(name, path)
    out = run_agg_path(gpu, ctx, path, desc, cols, monkeypatch, batched=name == "int32")
    pc, types = py_cols(cols)
    check_agg(out, pc, types, slots, fns, f"{name}/{path}")


# ---------------------------------------------------------------------------------------------------------------------
# group keys at their type's extremes, and packed keys that are all ones (the hash table's empty marker: special slot)
# ---------------------------------------------------------------------------------------------------------------------
KEY_TYPES = [abi.TYPE_BOOLEAN, abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_DATE, abi.TYPE_BIGINT]


def _extreme_values(typ, rng, n):
    lo, hi = TYPE_RANGE[typ]
    pool = sorted({lo, lo + 1, -1 if lo < 0 else 0, 0, 1, hi - 1, hi})
    return np.array(pool, dtype=object)[rng.integers(0, len(pool), n)].astype(abi.TYPE_NUMPY[typ])


@pytest.mark.gpu
@pytest.mark.parametrize("typ", KEY_TYPES)
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("layout", ["hash", "dense", "with_int"])
def test_group_keys_at_extremes(gpu, ctx, typ, nullable, layout):
    if layout == "dense" and typ in (abi.TYPE_INT, abi.TYPE_DATE, abi.TYPE_BIGINT):
        pytest.skip("a declared range of the whole type is too wide for a dense table")
    rng = np.random.default_rng(typ * 10 + nullable)
    n = 5000
    k = _extreme_values(typ, rng, n)
    kn = (rng.random(n) < 0.1).astype(np.uint8) if nullable else None
    k2 = np.where(rng.random(n) < 0.5, -1, I32[1]).astype(np.int32)        # with_int: -1 packs to all ones
    v = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    cols = [(0, k, kn, typ), (1, k2, None, abi.TYPE_INT), (2, v, None, abi.TYPE_BIGINT)]
    keys = [0, 1] if layout == "with_int" else [0]
    fns = [(abi.AGG_COUNT_STAR, 0, 10, None), (abi.AGG_SUM, abi.TYPE_BIGINT, 11, [("col", 2)]), (abi.AGG_MIN, typ, 12, [("col", 0)])]
    ranges = [TYPE_RANGE[typ]] if layout == "dense" else None
    desc = abi.make_agg_desc(keys, [typ, abi.TYPE_INT][:len(keys)], fns=fns, ranges=ranges, group_nullable=[nullable, False][:len(keys)])
    a = gpu.Agg(ctx, desc)
    try:
        a.push(sub_chunk(cols, 0, 1700))
        a.push(sub_chunk(cols, 1700, n))
        out = _host_cols(a.result())
    finally:
        a.close()
    pc, types = py_cols(cols)
    check_agg(out, pc, types, keys, fns, f"keys {typ} nullable={nullable} {layout}")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["bigint", "int_int", "bigint_bigint", "bigint_bigint_partitioned"])
def test_all_ones_packed_keys(gpu, ctx, monkeypatch, shape):
    # 8-byte images (one BIGINT, two INTs) and 16-byte images (two BIGINTs) equal to the empty marker when every key is -1
    rng = np.random.default_rng(7)
    n = 20_000
    wide = shape.startswith("bigint_bigint")
    dt, typ = (np.int32, abi.TYPE_INT) if shape == "int_int" else (np.int64, abi.TYPE_BIGINT)
    lo, hi = TYPE_RANGE[typ]
    a_ = np.array([-1, 0, lo, hi], dtype=dt)[rng.integers(0, 4, n)]
    b_ = np.array([-1, 0, lo, hi], dtype=dt)[rng.integers(0, 4, n)]
    v = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    cols = [(0, a_, None, typ), (1, b_, None, typ), (2, v, None, abi.TYPE_BIGINT)]
    keys = [0] if shape == "bigint" else [0, 1]
    fns = [(abi.AGG_COUNT_STAR, 0, 10, None), (abi.AGG_SUM, abi.TYPE_BIGINT, 11, [("col", 2)]), (abi.AGG_MAX, abi.TYPE_BIGINT, 12, [("col", 2)])]
    if shape.endswith("partitioned"):
        monkeypatch.setenv("SR_AGG_PARTITION_MIN_ROWS", "1000")
    desc = abi.make_agg_desc(keys, [typ] * len(keys), fns=fns)
    ag = gpu.Agg(ctx, desc)
    try:
        ag.push(sub_chunk(cols, 0, n // 2))
        ag.push(sub_chunk(cols, n // 2, n))
        out = _host_cols(ag.result())
    finally:
        ag.close()
    pc, types = py_cols(cols)
    assert (-1, -1) in {(x, y) for x, y in zip(pc[0], pc[1])} or not wide
    check_agg(out, pc, types, keys, fns, shape)


# ---------------------------------------------------------------------------------------------------------------------
# declared key ranges met by keys outside them, near the int64 extremes
# ---------------------------------------------------------------------------------------------------------------------
RANGE = (-5, 5)
OUTSIDE = {"int64_max": I64[1], "int64_min": I64[0], "min_minus_1": RANGE[0] - 1, "max_plus_1": RANGE[1] + 1}


def _expect_declared_range_error(gpu, agg):
    with pytest.raises(gpu.GpuError) as ei:
        agg.result()
    assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT and "declared" in str(ei.value)


def _range_keys(rng, n, bad, nullable):
    k = rng.integers(RANGE[0], RANGE[1] + 1, n, dtype=np.int64)
    k[n // 2] = bad
    kn = None
    if nullable:
        kn = (rng.random(n) < 0.1).astype(np.uint8)
        kn[n // 2] = 0
    return k, kn


@pytest.mark.gpu
@pytest.mark.parametrize("bad", list(OUTSIDE))
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("where", ["agg", "frag1"])
def test_declared_range_of_a_bigint_key(gpu, ctx, bad, nullable, where):
    rng = np.random.default_rng(3)
    n = 4000
    k, kn = _range_keys(rng, n, OUTSIDE[bad], nullable)
    v = rng.integers(-1000, 1000, n, dtype=np.int64)
    desc = abi.make_agg_desc([0], [abi.TYPE_BIGINT], fns=[(abi.AGG_SUM, abi.TYPE_BIGINT, 10, [("col", 1)]), (abi.AGG_COUNT_STAR, 0, 11, None)],
                             ranges=[RANGE], group_nullable=[nullable])
    ch = Chunk([(0, k, kn, abi.TYPE_BIGINT), (1, v, None, abi.TYPE_BIGINT)])
    if where == "agg":
        a = gpu.Agg(ctx, desc)
        try:
            a.push(ch)
            _expect_declared_range_error(gpu, a)
        finally:
            a.close()
        return
    frag = gpu.Fragment(ctx, abi.ScanDesc(), [], desc, mode=1)
    try:
        frag.push(ch)
        assert frag.plan()["mode"] == "fused-cascade"
        _expect_declared_range_error(gpu, frag.agg)
    finally:
        frag.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bad", list(OUTSIDE))
@pytest.mark.parametrize("nullable", [False, True])
def test_declared_range_of_a_bigint_payload_key(gpu, ctx, bad, nullable):
    # mode 2: the BIGINT payload of a join is the group key, folded into the join's slot-digit directory
    rng = np.random.default_rng(4)
    n, nb = 200_000, 2000
    fa, fb = rng.integers(0, 100, n, dtype=np.int32), rng.integers(0, nb, n, dtype=np.int32)
    fa[0], fb[0] = 0, nb // 2                                                  # one fact row passes A and meets the bad key
    fact = Chunk([(0, fa, None), (1, fb, None), (3, rng.integers(-1000, 1000, n, dtype=np.int32), None)])
    dim_a = Chunk([(10, np.arange(0, 5, dtype=np.int32), None)])               # streamed: 5 % of the rows pass
    p, pn = _range_keys(rng, nb, OUTSIDE[bad], nullable)
    dim_b = Chunk([(20, np.arange(nb, dtype=np.int32), None), (21, p, pn, abi.TYPE_BIGINT)])
    descs = [abi.make_join_desc(abi.JOIN_INNER, [10 * (k + 1)], [k], [abi.TYPE_INT]) for k in range(2)]
    joins = [gpu.Join(ctx, d) for d in descs]
    frag = None
    try:
        for j, ch in zip(joins, (dim_a, dim_b)):
            j.append_build(ch)
            j.build_finish()
        agg = abi.make_agg_desc([21], [abi.TYPE_BIGINT], fns=[(abi.AGG_SUM, abi.TYPE_INT, 40, [("col", 3)]), (abi.AGG_COUNT_STAR, 0, 41, None)],
                                ranges=[RANGE], group_nullable=[nullable])
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [(joins[0], 0, []), (joins[1], 1, [21])], agg, mode=2)
        frag.push(fact)
        plan = frag.plan()
        assert plan["mode"] == "selection-vector-passes" and plan["final_pass"] == "dense-batched"
        assert frag.rows_passed > 0
        _expect_declared_range_error(gpu, frag.agg)
    finally:
        if frag:
            frag.close()
        for j in joins:
            j.close()


# ---------------------------------------------------------------------------------------------------------------------
# predicates at the boundaries
# ---------------------------------------------------------------------------------------------------------------------
INT_PRED_TYPES = [abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_DATE, abi.TYPE_DECIMAL32, abi.TYPE_BIGINT, abi.TYPE_DECIMAL64]
INT32_CLASS = (abi.TYPE_INT, abi.TYPE_DATE, abi.TYPE_DECIMAL32)
CMP_OPS = [abi.PRED_EQ, abi.PRED_NE, abi.PRED_LT, abi.PRED_LE, abi.PRED_GT, abi.PRED_GE]


def _int_constants(typ):
    lo, hi = TYPE_RANGE[typ]
    beyond = {abi.TYPE_TINYINT: [200, -200], abi.TYPE_SMALLINT: [40_000, -40_000]}.get(typ, [1 << 31, -(1 << 31) - 1, 1 << 40])
    return sorted({lo - 1, lo, lo + 1, -1, 0, 1, hi - 1, hi, hi + 1, I64[0], I64[0] + 1, I64[1] - 1, I64[1], *beyond})


def _int_preds(typ):
    """[(label, sr_pred, op, lo, hi, in_list)] for one column at slot 0; every constant fits the int64 the ABI carries"""
    def fits(*cs):
        return all(I64[0] <= c <= I64[1] for c in cs)
    cs = [c for c in _int_constants(typ) if fits(c)]
    lo, hi = TYPE_RANGE[typ]
    out = [(f"op{op} {c}", abi.make_pred(0, op, c), op, c, 0, ()) for op in CMP_OPS for c in cs]
    for a, b in [(lo, hi), (I64[0], I64[1]), (hi, lo), (lo - 1, lo), (hi, hi + 1), (-1, 1), (I64[0], lo), (hi, I64[1])]:
        if fits(a, b):
            out.append((f"between {a} {b}", abi.make_pred(0, abi.PRED_BETWEEN, a, b), abi.PRED_BETWEEN, a, b, ()))
    ins = [c for c in cs if c != hi + 1][:abi.SR_MAX_IN_LIST]
    for op in (abi.PRED_IN, abi.PRED_NOT_IN):
        out.append((f"in{op}", abi.make_pred(0, op, in_list=ins), op, 0, 0, tuple(ins)))
        out.append((f"in{op} wrapped", abi.make_pred(0, op, in_list=[lo + (1 << 32), hi - (1 << 32), lo]), op, 0, 0,
                    (lo + (1 << 32), hi - (1 << 32), lo)))
    return out


def _boundary_chunk(typ, rng, n, variant):
    """-> (chunk with the column at slot 0, its Python values).  offset4: a device column 4 bytes into its allocation,
    so not 16-byte aligned (a host column would be staged into an aligned buffer)"""
    lo, hi = TYPE_RANGE[typ]
    dt = abi.TYPE_NUMPY[typ]
    x = rng.integers(lo, hi, n + 1, dtype=dt, endpoint=True)
    x[1: 1 + 8 * 16: 16] = np.array([lo, lo + 1, -1, 0, 1, hi - 1, hi, lo], dtype=dt)
    if variant == "offset4":
        import torch
        dev = torch.from_numpy(x).cuda()[1:]
        assert dev.data_ptr() % 16 == 4
        return Chunk([(0, dev, None, typ)], mem=abi.MEM_DEVICE), col_values(x[1:], None)
    x = x[1:].copy()
    xn = (rng.random(n) < 0.15).astype(np.uint8) if variant == "nullable" else None
    return Chunk([(0, x, xn, typ)]), col_values(x, xn)


def _selection_mismatches(sel, vals, op, a, b, ins):
    want = np.array([ref_pred(op, v, a, b, ins) for v in vals], dtype=bool)
    return int(np.count_nonzero(sel.astype(bool) != want)), int(want.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("typ", INT_PRED_TYPES)
@pytest.mark.parametrize("variant", ["plain", "nullable", "offset4"])
def test_int_predicates_at_boundaries(gpu, ctx, typ, variant):
    if variant == "offset4" and typ not in INT32_CLASS:
        pytest.skip("the misaligned view is an int32-class column")
    ch, vals = _boundary_chunk(typ, np.random.default_rng(typ), 3000, variant)
    bad = []
    for label, pred, op, a, b, ins in _int_preds(typ):
        sc = gpu.Scan(ctx, abi.ScanDesc([pred], out_slots=[0]))
        try:
            miss, want = _selection_mismatches(sc.evaluate(ch), vals, op, a, b, ins)
            if miss:
                bad.append(f"{label}: {miss} rows differ (want {want} selected)")
            rows = sc.filter(ch).num_rows
            if rows != want:
                bad.append(f"{label}: filter kept {rows} rows, want {want}")
        finally:
            sc.close()
    assert not bad, "; ".join(bad[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("typ", INT32_CLASS)
@pytest.mark.parametrize("variant", ["plain", "nullable", "offset4"])
def test_int32_predicates_in_the_streaming_pass(gpu, ctx, typ, variant):
    # a join-free selection-vector fragment: its streaming pass runs the range form ("tests") of the conjunct
    ch, vals = _boundary_chunk(typ, np.random.default_rng(50 + typ), 3000, variant)
    agg =abi.make_agg_desc(fns=[(abi.AGG_COUNT_STAR, 0, 10, None)])
    bad = []
    for label, pred, op, a, b, ins in _int_preds(typ):
        if op in (abi.PRED_NE, abi.PRED_IN, abi.PRED_NOT_IN):
            continue
        frag = gpu.Fragment(ctx, abi.ScanDesc([pred]), [], agg, mode=2)
        try:
            frag.push(ch)
            want = sum(ref_pred(op, v, a, b, ins) for v in vals)
            if frag.rows_passed != want:
                bad.append(f"{label}: {frag.rows_passed} rows passed, want {want}")
        finally:
            frag.close()
    assert not bad, "; ".join(bad[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("typ", FLOATS)
@pytest.mark.parametrize("nullable", [False, True])
def test_double_predicates_at_boundaries(gpu, ctx, typ, nullable):
    rng = np.random.default_rng(60 + typ)
    n = 3000
    dt = abi.TYPE_NUMPY[typ]
    special = np.array([INF, -INF, 0.0, -0.0, NAN, 5e-324, -5e-324, 1.5, -1.5, np.finfo(dt).max, np.finfo(dt).min], dtype=dt)
    x = np.where(rng.random(n) < 0.5, special[rng.integers(0, len(special), n)], rng.standard_normal(n).astype(dt)).astype(dt)
    xn = (rng.random(n) < 0.15).astype(np.uint8) if nullable else None
    ch = Chunk([(0, x, xn, typ)])
    vals = col_values(x, xn)
    consts = [INF, -INF, 0.0, -0.0, NAN, 1.5, float(np.finfo(dt).max)]
    preds = [(op, c, 0.0) for op in CMP_OPS for c in consts]
    preds += [(abi.PRED_BETWEEN, a, b) for a, b in [(-INF, INF), (-0.0, 0.0), (0.0, -0.0), (NAN, INF), (-INF, NAN), (-1.5, 1.5)]]
    bad = []
    for op, a, b in preds:
        sc = gpu.Scan(ctx, abi.ScanDesc([abi.make_pred(0, op, a, b, is_double=True)]))
        try:
            miss, want = _selection_mismatches(sc.evaluate(ch), vals, op, a, b, ())
            if miss:
                bad.append(f"op{op} {a} {b}: {miss} rows differ (want {want} selected)")
        finally:
            sc.close()
    assert not bad, "; ".join(bad[:8])


# ---------------------------------------------------------------------------------------------------------------------
# filter expressions at the edges (aggregate inputs go through the "expr" case above)
# ---------------------------------------------------------------------------------------------------------------------
FILTERS = [
    [("col", 0), ("col", 1), "*", ("i", 0), "<"],                                   # wraps at the extremes
    [("col", 0), ("i", I64[1]), "+", ("i", 0), ">="],
    [("col", 0), ("col", 1), "-", ("i", 1), "+", ("i", 0), ">"],
    [("col", 0), "todouble", ("d", 9.223372036854776e18), "=="],                    # INT64_MAX as a DOUBLE
    [("col", 2), ("col", 3), "/", ("d", 0.0), ">"],                                 # x / -0.0 is NULL, never true
    [("col", 2), ("col", 3), "/", "isnull"],
    [("col", 1), ("i", 0), ">", ("col", 3), ("d", 0.0), "<", "and", "not"],         # NOT (NULL AND ...) stays NULL
    [("col", 1), ("i", 0), ">", ("col", 0), ("i", 0), "<", "or"],
]


@pytest.mark.gpu
def test_filter_expressions_at_edges(gpu, ctx):
    _, cols, _, _ = build_case("expr", "nogroup", n=4000)
    cols = [(0, cols[0][1], None, abi.TYPE_BIGINT), (1, cols[1][1], cols[1][2], abi.TYPE_BIGINT),
            (2, cols[2][1], None, abi.TYPE_DOUBLE), (3, cols[3][1], None, abi.TYPE_DOUBLE)]
    ch = Chunk(cols)
    pc, types = py_cols(cols)
    bad = []
    for k, rpn in enumerate(FILTERS):
        sc = gpu.Scan(ctx, abi.ScanDesc(filter_exprs=[abi.make_expr(rpn)]))
        try:
            sel = sc.evaluate(ch)
            want = [(lambda r: not r[1] and r[0] != 0)(ref_expr(rpn, pc, types, i)) for i in range(ch.num_rows)]
            miss = int(np.count_nonzero(sel.astype(bool) != np.array(want)))
            if miss:
                bad.append(f"filter {k}: {miss} rows differ (want {sum(want)} selected)")
        finally:
            sc.close()
    assert not bad, "; ".join(bad)


@pytest.mark.gpu
def test_sum_nan_propagates(gpu, ctx):
    # only SUM / AVG are defined for NaN inputs (DESIGN.md: NaN in MIN / MAX)
    x = np.array([1.0, NAN, 2.0, 3.0, INF], dtype=np.float64)
    g = np.array([0, 0, 1, 1, 1], dtype=np.int32)
    fns = [(abi.AGG_SUM, abi.TYPE_DOUBLE, 10, [("col", 1)]), (abi.AGG_AVG, abi.TYPE_DOUBLE, 11, [("col", 1)])]
    a = gpu.Agg(ctx, abi.make_agg_desc([0], [abi.TYPE_INT], fns=fns, ranges=[(0, 1)]))
    try:
        a.push(Chunk([(0, g, None), (1, x, None)]))
        res = _host_cols(a.result())
    finally:
        a.close()
    assert res[0][1].tolist() == [0, 1]
    assert math.isnan(res[1][1][0]) and math.isnan(res[2][1][0]) and res[1][1][1] == INF and res[2][1][1] == INF
