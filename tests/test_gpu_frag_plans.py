"""The fused fragment across its plan space and its push lifecycle, against an exact star-join reference in plain Python.

The fragment plans once, on its first push: it samples the pass rates, orders the joins, picks the fused cascade or the
selection-vector passes, splits the joins between the streaming pass, the gather passes and the final pass, puts some
bitmaps in shared memory and picks the final-pass kernel.  Every case below is a seeded builder plus the plan it is
written for (`CASES`); `test_plan_table_covers_the_plan_space` checks on the CPU that the table as a whole reaches every
branch of the planner, and `test_fragment_plan_case` checks on the device that each case gets its plan and the right
answer.  The lifecycle tests push several morsels into one fragment and change what the plan was made for between them.

`ref_fragment` joins with dicts of Python values and aggregates with `ref_agg`, so it shares no code with the kernels
or the oracle; `test_reference_agrees_with_the_oracle` checks it against the oracle on every case at a reduced size.
"""
import collections

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from tests.test_gpu_join_edges import DIRECT, LINEAR, RANGE, _check_plan
from tests.test_gpu_value_edges import I8, I16, I32, I64, check_agg, col_values, ref_agg, ref_expr, ref_pred

INT, BIG, DBL, DEC, TINY, SMALL = abi.TYPE_INT, abi.TYPE_BIGINT, abi.TYPE_DOUBLE, abi.TYPE_DECIMAL64, abi.TYPE_TINYINT, abi.TYPE_SMALLINT
TYPE_RANGE = {TINY: I8, SMALL: I16, INT: I32, BIG: I64}
CASCADE, PASSES = "fused-cascade", "selection-vector-passes"
SAMPLE = 1 << 16          # rows of the first push the planner samples (frag_plan)


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
RefJoin = collections.namedtuple("RefJoin", "semi probe keys payload")   # payload: {build slot: (Python values, type)}


def _used_slots(agg):
    keys, fns = agg
    used = list(keys)
    for _, _, _, rpn in fns:
        used += [tok[1] for tok in rpn or () if isinstance(tok, tuple) and tok[0] == "col"]
    return set(used)


def star_rows(scan, joins, agg, fact_cols):
    """the rows that reach the aggregate -> ({slot: Python values}, {slot: type}, rows_passed).  scan: (preds, exprs) with
    preds as (slot, op, lo, hi, in_list); joins: RefJoin in the fragment's (hint) order; agg: (key slots, fns).  A NULL
    key never matches; INNER emits one row per matching build row, LEFT SEMI only tests; payloads are read from the
    matched build row.  rows_passed counts (fact row, build-row combination) pairs."""
    fc = {s: col_values(d, nl) for s, d, nl, _ in fact_cols}
    types = {s: t for s, _, _, t in fact_cols}
    n = len(next(iter(fc.values())))
    preds, exprs = scan
    rows = range(n)
    for slot, op, lo, hi, ins in preds:
        col = fc[slot]
        rows = [i for i in rows if ref_pred(op, col[i], lo, hi, ins)]
    for rpn in exprs:
        rows = [i for i in rows if (lambda r: not r[1] and r[0] != 0)(ref_expr(rpn, fc, types, i))]
    combos = [(i,) for i in rows]
    for rj in joins:
        index = {}
        for b, k in enumerate(rj.keys):
            if k is not None:
                index.setdefault(k, []).append(b)
        col = fc[rj.probe]
        nxt = []
        for c in combos:
            k = col[c[0]]
            m = index.get(k) if k is not None else None
            if m:
                if rj.semi:
                    nxt.append(c + (-1,))
                else:
                    nxt.extend(c + (b,) for b in m)
        combos = nxt
    cols = {}
    for s in _used_slots(agg):
        if s in fc:
            v = fc[s]
            cols[s] = [v[c[0]] for c in combos]
            continue
        for j, rj in enumerate(joins):
            if s in rj.payload:
                v, types[s] = rj.payload[s]
                cols[s] = [v[c[1 + j]] for c in combos]
                break
        else:
            raise KeyError(f"slot {s} is neither a fact column nor a payload")
    return cols, types, len(combos)


def ref_fragment(scan, joins, agg, fact_cols):
    """-> ({group key tuple: [expected result per function]}, rows_passed), see star_rows"""
    cols, types, passed = star_rows(scan, joins, agg, fact_cols)
    if not cols:
        cols = {-1: [0] * passed}
    return ref_agg(cols, types, agg[0], agg[1]), passed


def test_reference_known_answers():
    # fact rows 0..5; A: INNER with a duplicate key 1 and a NULL build key, payload 11; B: LEFT SEMI with duplicates;
    # C: INNER on a nullable probe key, payload 31
    fact = [(0, np.array([1, 2, 1, 3, 0, 1], np.int32), np.array([0, 0, 0, 0, 1, 0], np.uint8), INT),
            (1, np.array([5, 5, 6, 5, 5, 7], np.int32), None, INT),
            (2, np.array([9, 9, 9, 9, 9, 8], np.int32), np.array([0, 0, 0, 0, 0, 1], np.uint8), INT),
            (6, np.array([10, 20, 30, 40, 50, 60], np.int64), None, BIG)]
    a = RefJoin(False, 0, [1, 1, 2, None, 0], {11: ([100, 101, 200, 300, 400], INT)})
    b = RefJoin(True, 1, [5, 5, 6], {})
    c = RefJoin(False, 2, [9, 8], {31: ([7, 8], INT)})
    fns = [(abi.AGG_COUNT_STAR, 0, 40, None), (abi.AGG_SUM, BIG, 41, [("col", 6)])]
    got, passed = ref_fragment(([], []), [a, b, c], ([11, 31], fns), fact)
    # row 0 (key 1: two A rows) x B hit x C 9 -> 2 rows; row 1 (key 2) -> 1; row 2 (key 1) x B on 6 -> 2; row 3: no A row
    # for 3; row 4: NULL A key; row 5: B misses 7 (and the C key is NULL)
    assert passed == 5
    assert got == {(100, 7): [2, 40], (101, 7): [2, 40], (200, 7): [1, 20]}
    # a scan conjunct and a filter expression ahead of the joins
    preds = [(1, abi.PRED_LE, 5, 0, ())]
    got, passed = ref_fragment((preds, [[("col", 6), ("i", 15), ">"]]), [a, b, c], ([11], fns), fact)
    assert passed == 1 and got == {(200,): [1, 20]}


# ---------------------------------------------------------------------------------------------------------------------
# case builders.  Fact slots: join k probes slot k; measures below.  Build slots: join k keys at 10 (k + 1), its
# payloads at 10 (k + 1) + 1 and + 2.
# ---------------------------------------------------------------------------------------------------------------------
def _fact_int(rng, n, lo, hi):
    return rng.integers(lo, hi, n, dtype=np.int32, endpoint=True)


def _measure(rng, n):
    v = rng.integers(-10**6, 10**6, n, dtype=np.int32)
    v[rng.random(n) < 0.01] = I32[1]
    v[rng.random(n) < 0.01] = I32[0]
    return v


def _wide(rng, n):
    v = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    v[rng.random(n) < 0.01] = I64[1]
    v[rng.random(n) < 0.01] = I64[0]
    return v


def _doubles(rng, n):
    x = rng.standard_normal(n) * 1e3
    x[rng.random(n) < 0.02] = -0.0
    return x


FACTS = {   # slot: (type, generator(rng, n) -> (data, nulls))
    6: (INT, lambda r, n: (_measure(r, n), None)), 7: (INT, lambda r, n: (_fact_int(r, n, -5, 5), None)),
    8: (INT, lambda r, n: (_measure(r, n), None)), 9: (INT, lambda r, n: (_fact_int(r, n, 0, 100), None)),
    60: (INT, lambda r, n: (_fact_int(r, n, 0, 6), None)), 61: (INT, lambda r, n: (_fact_int(r, n, 0, 3), None)),
    62: (INT, lambda r, n: (_fact_int(r, n, 0, 2), None)), 63: (INT, lambda r, n: (r.permutation(n).astype(np.int32), None)),
    70: (BIG, lambda r, n: (_wide(r, n), None)), 71: (DBL, lambda r, n: (_doubles(r, n), None)),
    72: (DEC, lambda r, n: (_wide(r, n) >> 12, (r.random(n) < 0.2).astype(np.uint8))),
    **{50 + k: (INT, lambda r, n: (_fact_int(r, n, 0, 999), None)) for k in range(8)},
}
PAYLOADS = {   # kind: (type, generator(rng, nb) -> (data, nulls))
    "g7": (INT, lambda r, nb: (_fact_int(r, nb, 0, 6), None)),
    "g4": (INT, lambda r, nb: (_fact_int(r, nb, 0, 3), None)),
    "gbig": (BIG, lambda r, nb: (np.array([I64[0], I64[1], -1, 0, 1 << 40, -(1 << 40), 7], np.int64)[r.integers(0, 7, nb)], None)),
    "int": (INT, lambda r, nb: (_measure(r, nb), None)),
    "big": (BIG, lambda r, nb: (_wide(r, nb), None)),
    "dbl": (DBL, lambda r, nb: (_doubles(r, nb), None)),
    "dec": (DEC, lambda r, nb: (_wide(r, nb) >> 10, (r.random(nb) < 0.2).astype(np.uint8))),
}


class J:
    """one join of a case: `rate` of the fact rows find a build key (`rate0` of the first SAMPLE rows when given).
    kind "range": build keys in [lo, lo + span], both ends among them; "spread": keys over the whole type (a hash
    table for INT / BIGINT, direct mapping for TINYINT / SMALLINT)."""

    def __init__(self, rate, lo=0, span=2999, nb=None, typ=INT, kind="range", dup=False, semi=False, pays=(), fnull=0.0,
                 bnull=0.0, rate0=None):
        self.rate, self.lo, self.span, self.typ, self.kind = rate, lo, span, typ, kind
        self.nb = nb or min(span + 1, 3000)
        self.dup, self.semi, self.pays, self.fnull, self.bnull, self.rate0 = dup, semi, list(pays), fnull, bnull, rate0

    def method(self):
        if abi.TYPE_WIDTH[self.typ] <= 2:
            return DIRECT
        return LINEAR if self.kind == "spread" else RANGE


class Case:
    def __init__(self, mode, fact_cols, joins, preds, exprs, agg_keys, fns):
        self.mode, self.fact_cols, self.joins, self.preds, self.exprs = mode, fact_cols, joins, preds, exprs
        self.agg_keys, self.fns = agg_keys, fns          # agg_keys: [(slot, type, range or None, nullable)]

    @property
    def n(self):
        return len(self.fact_cols[0][1])

    def scan_desc(self):
        return abi.ScanDesc([abi.make_pred(s, op, lo, hi, in_list=list(ins) or None) for s, op, lo, hi, ins in self.preds],
                            [abi.make_expr(rpn) for rpn in self.exprs])

    def agg_desc(self):
        ks = self.agg_keys
        ranges = [r for _, _, r, _ in ks] if ks and all(r is not None for _, _, r, _ in ks) else None
        return abi.make_agg_desc([s for s, _, _, _ in ks], [t for _, t, _, _ in ks], fns=self.fns, ranges=ranges,
                                 group_nullable=[nl for _, _, _, nl in ks] or None)

    def key_slots(self):
        return [s for s, _, _, _ in self.agg_keys]

    def ref_joins(self):
        return [RefJoin(j["semi"], j["probe"], col_values(j["keys"], j["knulls"]),
                        {s: (col_values(d, nl), t) for s, d, nl, t in j["pay"]}) for j in self.joins]

    def reference(self, fact_cols=None):
        return star_rows((self.preds, self.exprs), self.ref_joins(), (self.key_slots(), self.fns), fact_cols or self.fact_cols)


def _build_keys(rng, j):
    tlo, thi = TYPE_RANGE[j.typ]
    dt = abi.TYPE_NUMPY[j.typ]
    if j.kind == "spread":
        pool = np.setdiff1d(np.concatenate([[-1, 0], rng.integers(tlo, thi, j.nb * 2, endpoint=True)]), [tlo, thi])
        keys = np.concatenate([[tlo, thi], rng.choice(pool, j.nb - 2, replace=j.dup)])
    elif j.dup:
        keys = j.lo + rng.integers(0, j.span + 1, j.nb)
        keys[:2] = [j.lo, j.lo + j.span]
    else:
        inner = rng.choice(j.span - 1, j.nb - 2, replace=False) + 1 if j.nb > 2 else np.empty(0, np.int64)
        keys = j.lo + np.concatenate([[0, j.span], inner])
    keys = np.asarray(keys).astype(dt)
    rng.shuffle(keys)
    knulls = None
    if j.bnull:
        knulls = (rng.random(j.nb) < j.bnull).astype(np.uint8)
        knulls[np.isin(keys, [keys.min(), keys.max()])] = 0
    return keys, knulls


def _miss_pool(rng, j, valid):
    tlo, thi = TYPE_RANGE[j.typ]
    if j.kind == "spread":
        cand = rng.integers(tlo, thi, 4000, endpoint=True)
    else:
        lo, hi = j.lo, j.lo + j.span
        cand = rng.integers(max(tlo, lo - j.span // 2 - 10), min(thi, hi + j.span // 2 + 10), 4000, endpoint=True)
    cand = np.concatenate([cand, [v for v in (j.lo - 1, j.lo + j.span + 1, tlo, thi) if tlo <= v <= thi]])
    return cand[~np.isin(cand, valid)]


def _fact_keys(rng, n, j, keys, knulls):
    dt = abi.TYPE_NUMPY[j.typ]
    tlo, thi = TYPE_RANGE[j.typ]
    valid = keys if knulls is None else keys[knulls == 0]
    miss = _miss_pool(rng, j, valid)
    rate = np.full(n, j.rate)
    if j.rate0 is not None:
        rate[:SAMPLE] = j.rate0
    hit = rng.random(n) < rate
    k = np.where(hit, valid[rng.integers(0, len(valid), n)], miss[rng.integers(0, len(miss), n)]).astype(dt)
    # both ends of the build range and the values just outside it, in the first tile, a middle one and the ragged last
    hi = j.lo + j.span
    specials = np.array(sorted({v for v in (j.lo - 1, j.lo, j.lo + 1, hi - 1, hi, hi + 1, tlo, thi) if tlo <= v <= thi}), dtype=dt)
    if n > 8 * len(specials):
        for p in (3, n // 2, n - len(specials) - 5):
            k[p:p + len(specials)] = specials
    nulls = None
    if j.fnull:
        nulls = (rng.random(n) < j.fnull).astype(np.uint8)
        k[nulls == 1] = valid[rng.integers(0, len(valid), int(nulls.sum()))]    # a NULL row's data bytes are a build key
    return k, nulls


def make_case(seed, n, mode, joins, agg_keys, fns, facts=(), preds=(), exprs=()):
    rng = np.random.default_rng(seed)
    fact_cols, built = [], []
    for k, j in enumerate(joins):
        keys, knulls = _build_keys(rng, j)
        pay = []
        for p, kind in enumerate(j.pays):
            t, gen = PAYLOADS[kind]
            d, nl = gen(rng, j.nb)
            pay.append((10 * (k + 1) + 1 + p, d, nl, t))
        fk, fkn = _fact_keys(rng, n, j, keys, knulls)
        fact_cols.append((k, fk, fkn, j.typ))
        built.append({"semi": j.semi, "probe": k, "key_slot": 10 * (k + 1), "typ": j.typ, "keys": keys, "knulls": knulls,
                      "pay": pay, "method": j.method()})
    for s in sorted(set(facts)):
        t, gen = FACTS[s]
        d, nl = gen(rng, n)
        fact_cols.append((s, d, nl, t))
    return Case(mode, fact_cols, built, list(preds), list(exprs), agg_keys, fns)


def SUM(s, t, o):
    return (abi.AGG_SUM, t, o, [("col", s)])


def MIN(s, t, o):
    return (abi.AGG_MIN, t, o, [("col", s)])


def MAX(s, t, o):
    return (abi.AGG_MAX, t, o, [("col", s)])


def COUNT(s, t, o):
    return (abi.AGG_COUNT, t, o, [("col", s)])


STAR = (abi.AGG_COUNT_STAR, 0, 99, None)
G7, G4 = (0, 6), (0, 3)
TOP = I32[1] - 2999      # build ranges that end at INT32_MAX / start at INT32_MIN
BOT = I32[0]


# ---------------------------------------------------------------------------------------------------------------------
# the plan-space table: name -> (builder(n, seed, mode) -> Case, full size, declared plan, dense-limit counts)
# ---------------------------------------------------------------------------------------------------------------------
Entry = collections.namedtuple("Entry", "build n plan limits")
CASES = {}


def case(name, n, plan, limits=None):
    def deco(fn):
        CASES[name] = Entry(fn, n, plan, limits or {})
        return fn
    return deco


def _casc(order, smem, agg_smem, methods):
    return {"mode": CASCADE, "order": order, "bitmap_in_smem": smem, "agg_in_smem": agg_smem, "num_stream_joins": 0,
            "num_gather_passes": 0, "final_pass": None, "method": methods}


def _pass(ns, gp, final, smem, agg_smem, methods, order=None):
    p = {"mode": PASSES, "num_stream_joins": ns, "num_gather_passes": gp, "final_pass": final, "bitmap_in_smem": smem,
         "agg_in_smem": agg_smem, "method": methods}
    if order is not None:
        p["order"] = order
    return p


# -- the fused cascade --
@case("cascade_eager1", 100_003, _casc([0, 1, 2], [1, 1, 1], True, [RANGE] * 3))
def _(n, seed, mode=1):
    # three bitmaps in shared memory, the second key streamed with the first (join 0 passes >= 8 %); dense shared aggregate
    return make_case(seed, n, mode, [J(0.3, 0, 1999, pays=["g7", "big"]), J(0.5, TOP, 2999, pays=["dbl"]), J(0.7, BOT, 999)],
                     [(11, INT, G7, False)], [SUM(6, INT, 40), STAR, MIN(12, BIG, 41), SUM(21, DBL, 42), MAX(70, BIG, 43)],
                     facts=[6, 70])


@case("cascade_budget", 100_003, _casc([0, 1, 2, 3], [1, 1, 0, 1], False, [RANGE] * 4))
def _(n, seed, mode=1):
    # the 96 KB budget: two 300 K-key bitmaps do not both fit next to the queues, the small one after them does; eager1
    # off (join 0 passes 3 %); a hash aggregate on a BIGINT payload; a LEFT SEMI join with duplicate build keys
    return make_case(seed, n, mode, [J(0.03, -500, 1000), J(0.3, 0, 300_000, pays=["gbig"]),
                                     J(0.6, -300_000, 300_000, pays=["dec"]), J(0.95, TOP + 999, 1999, dup=True, semi=True)],
                     [(21, BIG, None, False)], [STAR, SUM(31, DEC, 40), SUM(6, INT, 41), MAX(31, DEC, 42)], facts=[6])


@case("cascade_auto_first_push_65535", 65_535, _casc([0, 1], [1, 1], True, [RANGE] * 2))
def _(n, seed, mode=0):
    # total rate 2.5 % < 25 %, but a first push of 65 535 rows stays in the cascade; no GROUP BY
    return make_case(seed, n, mode, [J(0.05, 0, 4999, nb=4000), J(0.5, 100, 9999, nb=8000)], [],
                     [SUM(6, INT, 40), STAR, SUM(71, DBL, 41), MAX(70, BIG, 42)], facts=[6, 70, 71])


@case("auto_selective_first_push_65536", 65_536 + 4097, _pass(1, 1, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]))
def _(n, seed, mode=0):
    # the same rates with a first push of >= 65 536 rows: selection-vector passes, one gather pass, the batched final
    # pass with join 0's key carried
    return make_case(seed, n, mode, [J(0.05, 0, 4999, nb=4000, pays=["g7"]), J(0.5, 100, 9999, nb=8000)], [(11, INT, G7, False)],
                     [SUM(6, INT, 40), STAR], facts=[6])


@case("auto_cascade_high_rate", 70_001, _casc([0, 1], [1, 1], False, [RANGE] * 2))
def _(n, seed, mode=0):
    # total rate 40 % >= 25 %: the cascade for a large first push; hash aggregate on a fact column
    return make_case(seed, n, mode, [J(0.5, BOT, 2999), J(0.8, -999, 999)], [(60, INT, None, False)],
                     [STAR, SUM(70, BIG, 40)], facts=[60, 70])


# -- selection-vector passes: the streaming pass --
@case("stream2_mixed_smem", 120_007, _pass(2, 0, "generic", [1, 0, 0], True, [RANGE] * 3, [0, 1, 2]))
def _(n, seed, mode=2):
    # join 0 passes 12 % >= 8 %: two streamed joins; its 700 K-key bitmap takes the shared memory, the second one is read
    # from global memory; the trailing join is tested inline; BIGINT / DOUBLE / nullable DECIMAL64 measures
    return make_case(seed, n, mode, [J(0.12, 0, 700_000), J(0.4, -200_000, 200_000), J(0.93, BOT, 4999, nb=4500, pays=["g7"])],
                     [(31, INT, G7, False)], [SUM(70, BIG, 40), STAR, SUM(71, DBL, 41), SUM(72, DEC, 42), COUNT(72, DEC, 43)],
                     facts=[70, 71, 72])


@case("stream1_pred_below_8pct", 120_007, _pass(1, 1, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]))
def _(n, seed, mode=2):
    # a range conjunct passes 50 %, join 0 14 %: 7 % of the rows reach join 1, which gets a gather pass
    return make_case(seed, n, mode, [J(0.14, 0, 2999, pays=["g7"]), J(0.5, 0, 9999, nb=8000)], [(11, INT, G7, False)],
                     [SUM(6, INT, 40), STAR, MIN(7, INT, 41)], facts=[6, 7, 50], preds=[(50, abi.PRED_BETWEEN, 0, 499, ())])


@case("stream2_pred_above_8pct", 120_007, _pass(2, 1, "dense-batched", [1, 1, 0], True, [RANGE] * 3, [0, 1, 2]))
def _(n, seed, mode=2):
    # 50 % x 20 % = 10 % of the rows reach join 1: two streamed joins behind a conjunct, then a gather pass
    return make_case(seed, n, mode, [J(0.2, 0, 2999, pays=["g7"]), J(0.45, TOP, 2999), J(0.7, 0, 1999)], [(11, INT, G7, False)],
                     [SUM(6, INT, 40), STAR], facts=[6, 50], preds=[(50, abi.PRED_LE, 499, 0, ())])


@case("stream_hash_int32", 120_007, _pass(1, 1, "dense-batched", [0, 0], True, [LINEAR, RANGE], [0, 1]))
def _(n, seed, mode=2):
    # the streamed int32 join is a hash table (keys over the whole int32 range): the tests kernel's generic test
    return make_case(seed, n, mode, [J(0.05, kind="spread", nb=3000), J(0.5, TOP, 2999, pays=["g7"])], [(21, INT, G7, False)],
                     [SUM(6, INT, 40), STAR], facts=[6])


@case("stream_narrow_keys", 120_007, _pass(1, 1, "generic", [1, 0, 0], True, [DIRECT, DIRECT, RANGE], [0, 1, 2]))
def _(n, seed, mode=2):
    # SMALLINT and TINYINT probe keys: the generic streaming kernel; a RANGE join tested inline by the generic final pass
    return make_case(seed, n, mode, [J(0.05, typ=SMALL, kind="spread", nb=1000), J(0.5, typ=TINY, kind="spread", nb=100),
                                     J(0.95, BOT, 2999, pays=["g7"])], [(31, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("stream_seven_tests", 120_007, _pass(2, 0, "dense-batched", [1, 1, 0], True, [RANGE] * 3, [0, 1, 2]))
def _(n, seed, mode=2):
    # five range conjuncts and two streamed joins: 7 tests > SR_MAX_STREAM_TESTS, so the generic streaming kernel
    preds = [(50 + k, abi.PRED_BETWEEN, 0, 899, ()) for k in range(5)]
    return make_case(seed, n, mode, [J(0.2, 0, 2999), J(0.5, -2999, 2999), J(0.95, 0, 4999, nb=4500, pays=["g7"])],
                     [(31, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6, 50, 51, 52, 53, 54], preds=preds)


@case("stream_exprs_and_joins", 120_007, _pass(1, 1, "generic", [1, 0, 0], True, [RANGE] * 3, [0, 1, 2]))
def _(n, seed, mode=2):
    # filter expressions (a wrapping BIGINT product, a comparison) with a conjunct and joins
    exprs = [[("col", 70), ("col", 6), "*", ("i", 0), "<"], [("col", 51), ("i", 100), ">="]]
    return make_case(seed, n, mode, [J(0.1, 0, 2999), J(0.4, TOP, 2999), J(0.92, BOT, 2999)], [(60, INT, G7, False)],
                     [SUM(70, BIG, 40), STAR, SUM(71, DBL, 41)], facts=[6, 50, 51, 60, 70, 71],
                     preds=[(50, abi.PRED_BETWEEN, 0, 799, ())], exprs=exprs)


@case("stream_bitmap_750k", 120_007, _pass(1, 0, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]))
def _(n, seed, mode=2):
    # a 750 K-key bitmap (between the carry and no-carry budgets of frag_plan_stream_smem): shared memory without a carry
    return make_case(seed, n, mode, [J(0.05, -750_000, 750_000, nb=4000), J(0.95, 0, 2999, pays=["g7"])], [(21, INT, G7, False)],
                     [SUM(6, INT, 40), STAR], facts=[6])


@case("stream_bitmap_750k_carry", 120_007, _pass(1, 0, "dense-batched", [0, 0], True, [RANGE] * 2, [0, 1]))
def _(n, seed, mode=2):
    # the same bitmap when the streamed join carries its key (its payload is the group key): global memory
    return make_case(seed, n, mode, [J(0.05, -750_000, 750_000, nb=4000, pays=["g7"]), J(0.95, 0, 2999)], [(11, INT, G7, False)],
                     [SUM(6, INT, 40), STAR], facts=[6])


# -- gather passes --
@case("gather4_six_joins", 300_007, _pass(1, 4, "generic", [1, 0, 0, 0, 0, 0], True, [RANGE, RANGE, LINEAR, RANGE, RANGE, LINEAR],
                                          [0, 1, 2, 3, 4, 5]))
def _(n, seed, mode=2):
    # six joins, four gather passes (the selection vectors ping-pong twice); hash tables in a gather pass (INT) and tested
    # inline by the final pass (BIGINT keys at both int64 extremes); a nullable probe key
    return make_case(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.3, TOP - 7000, 9999, nb=8000),
                                     J(0.45, kind="spread", nb=3000), J(0.62, 0, 20_000, nb=15_000, fnull=0.02),
                                     J(0.8, BOT, 999), J(0.97, typ=BIG, kind="spread", nb=3000)],
                     [(11, INT, G7, False)], [STAR, SUM(70, BIG, 40), MAX(6, INT, 41)], facts=[6, 70])


@case("gather3_six_joins_hash_agg", 300_007, _pass(2, 3, "generic", [1, 1, 0, 0, 0, 0], False, [RANGE, RANGE, RANGE, LINEAR, RANGE, RANGE],
                                                  [0, 1, 2, 3, 4, 5]))
def _(n, seed, mode=2):
    # six joins, two streamed (the second carries its key), three gather passes, a LEFT SEMI join with duplicates inline;
    # a hash aggregate on (BIGINT payload, fact INT) over INT, DOUBLE, nullable DECIMAL64 and BIGINT payloads
    return make_case(seed, n, mode, [J(0.1, 0, 2999), J(0.3, -4999, 4999, pays=["gbig", "int"]), J(0.45, TOP, 2999, pays=["dbl"]),
                                     J(0.62, kind="spread", nb=3000, pays=["dec"]), J(0.8, 0, 999, pays=["big"]),
                                     J(0.97, BOT, 1999, dup=True, semi=True, nb=3000)],
                     [(21, BIG, None, False), (60, INT, None, False)],
                     [STAR, SUM(22, INT, 40), SUM(31, DBL, 41), SUM(41, DEC, 42), MIN(51, BIG, 43), SUM(6, INT, 44)], facts=[6, 60])


@case("gather2_expand", 150_001, _pass(1, 2, "expand", [1, 0, 0, 0, 0], True, [RANGE, RANGE, RANGE, RANGE, LINEAR]))
def _(n, seed, mode=0):
    # an INNER join with duplicate build keys in a gather pass: the expand final pass, which also tests a bitmap join and
    # a LEFT SEMI hash join (duplicates) inline; payloads INT / DOUBLE as aggregate inputs
    return make_case(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.4, TOP + 1000, 1999, dup=True, pays=["int", "dbl"]),
                                     J(0.6, BOT, 2999), J(0.93, -5999, 5999, nb=5000),J(0.96, kind="spread", nb=2000, dup=True, semi=True)],
                     [(11, INT, G7, False)], [STAR, SUM(21, INT, 40), SUM(22, DBL, 41), MAX(70, BIG, 42)], facts=[70])


# -- the batched final pass (k_frag_final_dense) at and one past each limit of frag_plan_final_dense --
def _dense(seed, n, mode, joins, keys, fns, facts):
    return make_case(seed, n, mode, joins, keys, fns, facts=facts)


@case("dense_at_limits", 100_003, _pass(1, 0, "dense-batched", [1, 0, 0, 0], True, [RANGE] * 4), {"vals": 6, "look": 2, "test": 2, "fns": 4})
def _(n, seed, mode=2):
    # two directory lookups (streamed and inline), two inline bitmap tests over 64 keys each, one range ending at
    # INT32_MAX: ~1/64 of the surviving rows carry the last key of a range (bit `span` of its bitmap); four functions:
    # six fact values
    return _dense(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.95, 0, 1999, pays=["g4"]), J(0.93, I32[1] - 63, 63),
                                  J(0.97, BOT, 63)],
                  [(11, INT, G7, False), (21, INT, G4, False)], [SUM(6, INT, 40), MAX(7, INT, 41), COUNT(6, INT, 42), MIN(7, INT, 43), STAR],
                  [6, 7])


@case("dense_past_vals", 100_003, _pass(1, 0, "generic", [1, 0, 0, 0], True, [RANGE] * 4), {"vals": 7})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.95, 0, 1999, pays=["g4"]), J(0.93, TOP, 2999), J(0.97, BOT, 2999)],
                  [(11, INT, G7, False), (21, INT, G4, False)], [SUM(6, INT, 40), MAX(7, INT, 41), SUM(8, INT, 42), STAR], [6, 7, 8])


@case("dense_past_tests", 100_003, _pass(1, 0, "generic", [1, 0, 0, 0], True, [RANGE] * 4), {"test": 3})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.95, 0, 1999), J(0.93, TOP, 2999), J(0.97, BOT, 2999)],
                  [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], [6])


@case("dense_past_look", 100_003, _pass(1, 0, "generic", [1, 0, 0], True, [RANGE] * 3), {"look": 3})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, 0, 2999, pays=["g7"]), J(0.95, 0, 1999, pays=["g4"]), J(0.93, TOP, 2999, pays=["g4"])],
                  [(11, INT, G7, False), (21, INT, G4, False), (31, INT, G4, False)], [SUM(6, INT, 40), STAR], [6])


@case("dense_fact_keys_at_limits", 100_003, _pass(1, 0, "dense-batched", [1], True, [RANGE]), {"fkeys": 2, "fns": 4, "vals": 6})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, BOT, 2999)], [(60, INT, G7, False), (61, INT, G4, False)],
                  [SUM(6, INT, 40), MIN(7, INT, 41), MAX(8, INT, 42), COUNT(9, INT, 43), STAR], [6, 7, 8, 9, 60, 61])


@case("dense_past_fact_keys", 100_003, _pass(1, 0, "generic", [1], True, [RANGE]), {"fkeys": 3})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, BOT, 2999)], [(60, INT, G7, False), (61, INT, G4, False), (62, INT, (0, 2), False)],
                  [SUM(6, INT, 40), STAR], [6, 60, 61, 62])


@case("dense_past_fns", 100_003, _pass(1, 0, "generic", [1], True, [RANGE]), {"fns": 5})
def _(n, seed, mode=2):
    return _dense(seed, n, mode, [J(0.05, BOT, 2999)], [(60, INT, G7, False)],
                  [SUM(6, INT, 40), MIN(7, INT, 41), MAX(8, INT, 42), COUNT(9, INT, 43), SUM(7, INT, 44), STAR], [6, 7, 8, 9, 60])


# -- the hash-table retry loop of frag_push: the sampled first 65 536 rows promise few survivors, the rest all pass, and
# more than the table's 2^20 admission limit of groups arrive in one push --
@case("retry_after_1_gather", 1_250_003, _pass(2, 1, "generic", [1, 1, 0], False, [RANGE] * 3))
def _(n, seed, mode=2):
    return make_case(seed, n, mode, [J(1.0, 0, 2999, rate0=0.1), J(1.0, TOP, 2999, rate0=0.5), J(0.92, BOT, 2999, rate0=0.5)],
                     [(63, INT, None, False)], [STAR], facts=[63])


@case("retry_after_2_gathers", 1_250_003, _pass(2, 2, "generic", [1, 1, 0, 0], False, [RANGE] * 4))
def _(n, seed, mode=2):
    return make_case(seed, n, mode, [J(1.0, 0, 2999, rate0=0.1), J(1.0, TOP, 2999, rate0=0.5), J(0.96, BOT, 2999, rate0=0.5),
                                     J(0.96, -1499, 2999, rate0=0.5)],
                     [(63, INT, None, False)], [STAR], facts=[63])


@case("retry_expand_payload_key", 700_001, _pass(2, 1, "expand", [1, 1, 0], False, [RANGE] * 3))
def _(n, seed, mode=2):
    # each surviving row expands to ~2 build rows of join 2, whose payload is a group key beside a unique fact key
    return make_case(seed, n, mode, [J(1.0, 0, 2999, rate0=0.1), J(1.0, TOP, 2999, rate0=0.5),
                                     J(0.92, BOT, 1499, nb=3000, dup=True, pays=["int"], rate0=0.5)],
                     [(31, INT, None, False), (63, INT, None, False)], [STAR], facts=[63])


REDUCED_N = 6000


def build_case(name, n=None, mode=None):
    e = CASES[name]
    seed = 5000 + sorted(CASES).index(name)
    return e.build(n or e.n, seed) if mode is None else e.build(n or e.n, seed, mode)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the reference against the oracle, and the coverage of the table
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_run(oracle, c, fact_chunk=None):
    joins = []
    for j in c.joins:
        oj = oracle.Join(abi.make_join_desc(abi.JOIN_LEFT_SEMI if j["semi"] else abi.JOIN_INNER, [j["key_slot"]], [j["probe"]], [j["typ"]]))
        oj.append_build(_build_chunk(j))
        oj.build()
        joins.append((oj, j["probe"], [s for s, _, _, _ in j["pay"]]))
    res, passed = oracle.fragment_run(c.scan_desc(), joins, c.agg_desc(), fact_chunk or Chunk(c.fact_cols), num_threads=2)
    return res.output(), passed


@pytest.mark.parametrize("name", list(CASES))
def test_reference_agrees_with_the_oracle(oracle, name):
    c = build_case(name, REDUCED_N)
    cols, types, passed = c.reference()
    out, opassed = _oracle_run(oracle, c)
    assert opassed == passed, f"{name}: oracle passed {opassed}, reference {passed}"
    check_agg(out, cols, types, c.key_slots(), c.fns, f"oracle {name}")


def _positions(plan):
    """(position name, hint join index) of every join of a selection-vector plan"""
    ns, gp = plan["num_stream_joins"], plan["num_gather_passes"]
    return [("streamed" if q < ns else "gather" if q < ns + gp else "inline", j) for q, j in enumerate(plan["order"])]


def test_plan_table_covers_the_plan_space():
    plans = {name: e.plan for name, e in CASES.items()}
    small = {name: build_case(name, 200) for name in CASES}
    for name, p in plans.items():      # every declared plan names every field it is written for
        want = {"mode", "num_stream_joins", "num_gather_passes", "final_pass", "bitmap_in_smem", "agg_in_smem", "method"}
        assert want <= set(p), f"{name}: declares {sorted(set(p))}"
        assert len(p["method"]) == len(p["bitmap_in_smem"]) == len(small[name].joins), name
        assert p["method"] == [j["method"] for j in small[name].joins], name
    modes = {(small[n_].mode, p["mode"], CASES[n_].n) for n_, p in plans.items()}
    assert {m for _, m, _ in modes} == {CASCADE, PASSES}
    assert (0, CASCADE, SAMPLE - 1) in modes                                              # low rate, first push too small
    assert any(m == 0 and mode == PASSES and n_ >= SAMPLE for m, mode, n_ in modes)       # low rate, large first push
    assert any(m == 0 and mode == CASCADE and n_ >= SAMPLE for m, mode, n_ in modes)      # high rate, large first push
    sel = {n_: p for n_, p in plans.items() if p["mode"] == PASSES}
    assert {p["num_stream_joins"] for p in sel.values()} >= {1, 2}
    assert any(p["num_stream_joins"] == 1 and len(p["method"]) > 1 for p in sel.values())  # below the 8 % rule
    assert {p["num_gather_passes"] for p in sel.values()} >= {0, 1, 2, 3, 4}
    assert {p["final_pass"] for p in sel.values()} == {"generic", "expand", "dense-batched"}
    for k, at in (("vals", 6), ("look", 2), ("test", 2), ("fkeys", 2), ("fns", 4)):
        finals = {e.limits[k]: e.plan["final_pass"] for e in CASES.values() if k in e.limits}
        assert finals.get(at) == "dense-batched" and finals.get(at + 1) == "generic", (k, finals)
    for mode in (CASCADE, PASSES):
        ps = [p for p in plans.values() if p["mode"] == mode]
        assert any(0 in p["bitmap_in_smem"] and 1 in p["bitmap_in_smem"] for p in ps), mode
        assert {p["agg_in_smem"] for p in ps} == {True, False}, mode
    placed = {(pos, p["method"][j]) for p in sel.values() if "order" in p for pos, j in _positions(p)}
    for m in (RANGE, LINEAR):
        for pos in ("streamed", "gather", "inline"):
            assert (pos, m) in placed, (pos, m)
    assert any(p["num_gather_passes"] >= 3 and len(p["method"]) == 6 and not p["agg_in_smem"] for p in sel.values())
    dups = {(j["semi"], len(np.unique(j["keys"])) < len(j["keys"])) for c in small.values() for j in c.joins}
    assert (False, True) in dups and (True, True) in dups       # INNER and LEFT SEMI joins with duplicate build keys
    # payloads as group keys (INT, BIGINT) and as aggregate inputs (INT, BIGINT, DOUBLE, nullable DECIMAL64)
    pay_types = {}
    for c in small.values():
        for j in c.joins:
            for s, _, nl, t in j["pay"]:
                role = "key" if s in c.key_slots() else "input" if s in _used_slots(([], c.fns)) else None
                if role:
                    pay_types.setdefault(role, set()).add((t, nl is not None))
    assert {(INT, False), (BIG, False)} <= pay_types["key"]
    assert {(INT, False), (BIG, False), (DBL, False), (DEC, True)} <= pay_types["input"]


# ---------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------
def _build_chunk(j):
    return Chunk([(j["key_slot"], j["keys"], j["knulls"], j["typ"])] + j["pay"])


def _gpu_joins(gpu, ctx, c):
    joins = []
    try:
        for j in c.joins:
            g = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_LEFT_SEMI if j["semi"] else abi.JOIN_INNER, [j["key_slot"]], [j["probe"]], [j["typ"]]))
            joins.append(g)
            g.append_build(_build_chunk(j))
            g.build_finish()
    except Exception:
        for g in joins:
            g.close()
        raise
    return joins


MEMS = ("host", "pinned", "device", "device_off4")


def _morsel(cols, a, b, mem, keep):
    """rows [a, b) of the fact columns as a chunk in memory kind `mem`; device_off4: each column one element into its
    allocation (4 bytes off 16-byte alignment for int32 columns).  Buffers the push reads go to `keep`."""
    if mem == "host":
        return Chunk([(s, d[a:b].copy(), None if nl is None else nl[a:b].copy(), t) for s, d, nl, t in cols])
    import torch
    out = []
    for s, d, nl, t in cols:
        if mem == "pinned":
            dd = torch.from_numpy(d[a:b].copy()).pin_memory()
            nn = None if nl is None else torch.from_numpy(nl[a:b].copy()).pin_memory()
        else:
            pad = 1 if mem == "device_off4" else 0
            dd = torch.from_numpy(np.concatenate([d[a:a + 1] if b > a else d[:0], d[a:b]]) if pad else d[a:b].copy()).cuda()[pad:]
            nn = None if nl is None else torch.from_numpy(nl[a:b].copy()).cuda()
        keep.append((dd, nn))
        out.append((s, dd, nn, t))
    return Chunk(out, num_rows=b - a, mem=abi.MEM_HOST_PINNED if mem == "pinned" else abi.MEM_DEVICE if mem.startswith("device") else abi.MEM_HOST)


class Run:
    """a fragment over a case's joins (closed by close())"""

    def __init__(self, gpu, ctx, c, mode=None):
        self.gpu, self.ctx, self.c = gpu, ctx, c
        self.joins = _gpu_joins(gpu, ctx, c)
        self.frag = None
        try:
            self.frag = gpu.Fragment(ctx, c.scan_desc(), [(g, j["probe"], [s for s, _, _, _ in j["pay"]]) for g, j in zip(self.joins, c.joins)],
                                     c.agg_desc(), mode=c.mode if mode is None else mode)
        except Exception:
            self.close()
            raise
        self.keep = []

    def push(self, cols, a, b, mem="host"):
        self.frag.push(_morsel(cols, a, b, mem, self.keep))

    def plan(self):
        p = self.frag.plan()
        p["method"] = [g.info().method for g in self.joins]
        return p

    def result(self):
        out = [(t, d, nl) for _, t, d, nl in self.frag.agg.result()]
        self.ctx.sync()
        self.keep.clear()
        return out

    def close(self):
        if self.frag:
            self.frag.close()
        for g in self.joins:
            g.close()


def _check(c, out, passed, fact_cols=None, label=""):
    cols, types, want = c.reference(fact_cols)
    assert passed == want, f"{label}: {passed} rows passed, want {want}"
    check_agg(out, cols, types, c.key_slots(), c.fns, label)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fragment_plan_case(gpu, ctx, name):
    c = build_case(name)
    r = Run(gpu, ctx, c)
    try:
        r.push(c.fact_cols, 0, c.n)
        plan = r.plan()
        passed = r.frag.rows_passed
        out = r.result()
    finally:
        r.close()
    _check_plan(plan, CASES[name].plan, name)
    _check(c, out, passed, label=name)


# ---------------------------------------------------------------------------------------------------------------------
# the push lifecycle
# ---------------------------------------------------------------------------------------------------------------------
def _slice(cols, a, b):
    return [(s, d[a:b], None if nl is None else nl[a:b], t) for s, d, nl, t in cols]


def _stream(gpu, ctx, c, cuts, mems=("host",), mode=None):
    """push rows [cuts[k], cuts[k + 1]) in turn, memory kinds cycling through `mems` -> (plan, rows_passed, result)"""
    r = Run(gpu, ctx, c, mode)
    try:
        for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            r.push(c.fact_cols, a, b, mems[k % len(mems)])
        return r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
def test_empty_first_push(gpu, ctx, mode):
    # planned on zero rows: every sampled rate is 1.0, so every join after the streamed ones is tested inline
    c = build_case("gather4_six_joins", 90_001)
    plan, passed, out = _stream(gpu, ctx, c, [0, 0, 40_000, c.n], mode=mode)
    if mode == 2:
        _check_plan(plan, {"mode": PASSES, "num_stream_joins": 2, "num_gather_passes": 0, "final_pass": "generic"}, "empty first")
    else:
        assert plan["mode"] == CASCADE
    _check(c, out, passed, label=f"empty first push, mode {mode}")


@pytest.mark.gpu
def test_unrepresentative_first_push_cascade_then_selective_rows(gpu, ctx):
    # the first push passes every join (cascade chosen), the later ones 1 %
    c = build_case("auto_cascade_high_rate", 200_000)
    for k, j in enumerate(c.joins):
        fk = c.fact_cols[k][1]
        valid = j["keys"]
        rng = np.random.default_rng(k)
        fk[:70_000] = valid[rng.integers(0, len(valid), 70_000)]
        fk[70_000:] = np.where(rng.random(130_000) < 0.1, valid[rng.integers(0, len(valid), 130_000)], I32[0] + 5000 + k)
    plan, passed, out = _stream(gpu, ctx, c, [0, 70_000, 140_000, c.n])
    assert plan["mode"] == CASCADE and plan["pass_rate"] == [1.0, 1.0]
    _check(c, out, passed, label="cascade then 1 %")


@pytest.mark.gpu
def test_unrepresentative_first_push_selective_then_new_groups(gpu, ctx):
    # the first push passes 0.5 % (a small hash table is planned), the next one passes everything with a new group per row
    c = build_case("retry_after_1_gather", 400_001)
    for k, j in enumerate(c.joins):
        fk = c.fact_cols[k][1]
        rng = np.random.default_rng(10 + k)
        valid = j["keys"]
        hit = np.concatenate([rng.random(80_000) < 0.17, np.ones(c.n - 80_000, bool)])
        fk[:] = np.where(hit, valid[rng.integers(0, len(valid), c.n)], I32[0] + 7000 + k)
    plan, passed, out = _stream(gpu, ctx, c, [0, 80_000, c.n], mode=2)
    assert plan["mode"] == PASSES and plan["agg_in_smem"] is False
    _check(c, out, passed, label="selective then new groups")


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode", [("auto_selective_first_push_65536", 1), ("auto_selective_first_push_65536", 2),
                                       ("gather2_expand", 0)])
def test_morsel_sizes(gpu, ctx, name, mode):
    c = build_case(name, 1 + 4095 + 4097 + 65_537 + 3)
    cuts = np.cumsum([0, 65_537, 1, 4095, 4097, 3]).tolist()
    plan, passed, out = _stream(gpu, ctx, c, cuts, mode=mode)
    assert plan["mode"] == (CASCADE if mode == 1 else PASSES)
    _check(c, out, passed, label=f"morsels {name} mode {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode", [("stream_bitmap_750k_carry", 2), ("cascade_eager1", 1), ("stream2_mixed_smem", 2)])
def test_memory_kinds_alternate(gpu, ctx, name, mode):
    c = build_case(name, 60_000)
    cuts = [0, 9001, 20_000, 31_003, 42_000, 50_001, 60_000]
    plan, passed, out = _stream(gpu, ctx, c, cuts, mems=("device_off4", "host", "pinned", "device"), mode=mode)
    _check(c, out, passed, label=f"memory kinds {name}")
    if name == "stream_bitmap_750k_carry":
        assert plan["final_pass"] == "dense-batched"


def _with_nulls(cols, slot, a, frac, seed, set_to=None):
    """a copy of the fact columns where `slot` is NULL on `frac` of the rows from `a` on (data bytes set_to[...] when given)"""
    rng = np.random.default_rng(seed)
    out = []
    for s, d, nl, t in cols:
        if s == slot:
            d = d.copy()
            nl = np.zeros(len(d), np.uint8) if nl is None else nl.copy()
            m = np.zeros(len(d), bool)
            m[a:] = rng.random(len(d) - a) < frac
            nl[m] = 1
            if set_to is not None:
                d[m] = set_to[rng.integers(0, len(set_to), int(m.sum()))]
        out.append((s, d, nl, t))
    return out


def _two_pushes(gpu, ctx, c, cols, cut):
    """rows [0, cut) from the case's own columns (no NULL mask where it has none), the rest from `cols`"""
    r = Run(gpu, ctx, c)
    try:
        r.push(c.fact_cols, 0, cut)
        first = r.plan()
        r.push(cols, cut, c.n)
        return first, r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()


@pytest.mark.gpu
def test_aggregate_input_turns_nullable(gpu, ctx):
    # a later push makes the SUM input nullable: global accumulation and the generic final pass from then on
    c = build_case("dense_at_limits", 120_001)
    cols = _with_nulls(c.fact_cols, 6, 70_000, 0.3, 1)
    first, last, passed, out = _two_pushes(gpu, ctx, c, cols, 70_000)
    assert first["final_pass"] == "dense-batched" and first["agg_in_smem"]
    assert last["final_pass"] == "generic" and not last["agg_in_smem"] and last["order"] == first["order"]
    _check(c, out, passed, cols, "aggregate input turns nullable")


@pytest.mark.gpu
def test_streamed_probe_key_turns_nullable(gpu, ctx):
    # the streamed join's key turns nullable (data bytes of its NULL rows are build keys): the generic streaming kernel
    c = build_case("stream_bitmap_750k_carry", 120_001)
    cols = _with_nulls(c.fact_cols, 0, 65_536, 0.2, 2, set_to=c.joins[0]["keys"])
    first, last, passed, out = _two_pushes(gpu, ctx, c, cols, 65_536)
    assert first["final_pass"] == "dense-batched"
    _check(c, out, passed, cols, "streamed key turns nullable")


@pytest.mark.gpu
def test_inline_tested_key_turns_nullable(gpu, ctx):
    # the key of a join the final pass tests inline turns nullable, with build keys in the data bytes of its NULL rows;
    # the aggregate stays in shared memory, so only the nullable column rules out the batched final pass
    c = build_case("dense_at_limits", 120_001)
    cols = _with_nulls(c.fact_cols, 2, 65_536, 0.3, 3, set_to=c.joins[2]["keys"])
    first, last, passed, out = _two_pushes(gpu, ctx, c, cols, 65_536)
    assert first["final_pass"] == "dense-batched"
    assert last["final_pass"] == "generic" and last["agg_in_smem"]
    _check(c, out, passed, cols, "inline key turns nullable")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_group_key_turns_nullable_fails(gpu, ctx, mode):
    c = build_case("dense_fact_keys_at_limits", 20_000)
    cols = _with_nulls(c.fact_cols, 60, 10_000, 0.5, 4)
    r = Run(gpu, ctx, c, mode)
    try:
        r.push(c.fact_cols, 0, 10_000)
        with pytest.raises(gpu.GpuError) as ei:
            r.push(cols, 10_000, c.n)
        assert ei.value.code == abi.SR_ERR_INVALID_ARGUMENT and "nullable" in str(ei.value)
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cascade_eager1", "gather4_six_joins", "gather2_expand"])
def test_reset_then_second_stream(gpu, ctx, name):
    c = build_case(name, 100_001)
    d = build_case(name, 100_001)
    rng = np.random.default_rng(9)
    second = [(s, np.ascontiguousarray(dd[rng.permutation(len(dd))]), nl, t) if s >= 6 else (s, dd, nl, t) for s, dd, nl, t in d.fact_cols]
    r = Run(gpu, ctx, c)
    try:
        r.push(c.fact_cols, 0, 60_000)
        r.push(c.fact_cols, 60_000, c.n)
        order = r.plan()["order"]
        _check(c, r.result(), r.frag.rows_passed, label=f"{name} first stream")
        r.frag.reset()
        r.push(second, 0, 30_001)
        r.push(second, 30_001, c.n)
        assert r.plan()["order"] == order
        passed = r.frag.rows_passed
        out = r.result()
    finally:
        r.close()
    _check(c, out, passed, second, f"{name} second stream")


@pytest.mark.gpu
def test_last_pass_ms_and_push_after_finish(gpu, ctx):
    for name, mode in (("cascade_eager1", 1), ("stream1_pred_below_8pct", 2)):
        c = build_case(name, 70_000)
        r = Run(gpu, ctx, c, mode)
        try:
            r.push(c.fact_cols, 0, c.n)
            ms = r.frag.last_pass_ms()
            if mode == 1:
                assert ms is None
            else:
                assert len(ms) == 3 and all(x >= 0.0 for x in ms), ms
            r.result()
            with pytest.raises(gpu.GpuError) as ei:
                r.push(c.fact_cols, 0, 100)
            assert ei.value.code == abi.SR_ERR_STATE
        finally:
            r.close()


# ---------------------------------------------------------------------------------------------------------------------
# refusals of sr_fragment_create / frag_compile
# ---------------------------------------------------------------------------------------------------------------------
def _refusal(gpu, ctx, fact, joins, scan, agg, at_create=False):
    """-> the error code of the fragment's creation (at_create) or first push"""
    gj = []
    frag = None
    try:
        for jt, ktype, keys, pays in joins:
            g = gpu.Join(ctx, abi.make_join_desc(jt, [10], [0], [ktype]))
            gj.append(g)
            g.append_build(Chunk([(10, keys, None, ktype)] + pays))
            g.build_finish()
        fjoins = [(g, 0, [s for s, _, _, _ in pays]) for g, (_, _, _, pays) in zip(gj, joins)]
        with pytest.raises(gpu.GpuError) as ei:
            frag = gpu.Fragment(ctx, scan, fjoins, agg, mode=2)
            frag.push(Chunk(fact))
        assert (frag is None) == at_create
        return ei.value.code
    finally:
        if frag:
            frag.close()
        for g in gj:
            g.close()


@pytest.mark.gpu
def test_refusals(gpu, ctx):
    n = 1000
    rng = np.random.default_rng(1)
    cols = [(s, rng.integers(0, 100, n, dtype=np.int32), None, INT) for s in range(1, 26)]
    key32 = (0, rng.integers(0, 100, n, dtype=np.int32), None, INT)
    keys = np.arange(100, dtype=np.int32)
    inner = [(abi.JOIN_INNER, INT, keys, [])]
    count = abi.make_agg_desc(fns=[STAR])
    pred = abi.make_pred(1, abi.PRED_GE, 0)
    expr = abi.make_expr([("col", 2), ("i", 0), ">="])
    code = _refusal(gpu, ctx, [key32] + cols, inner, abi.ScanDesc([pred] * 9), count)
    assert code == abi.SR_ERR_NOT_SUPPORTED, "9 scan conjuncts"
    code = _refusal(gpu, ctx, [key32] + cols, inner, abi.ScanDesc([], [expr] * 5), count)
    assert code == abi.SR_ERR_NOT_SUPPORTED, "5 filter expressions"
    many = abi.make_agg_desc(fns=[SUM(s, INT, 40 + s) for s in range(1, 8)])
    preds = [abi.make_pred(s, abi.PRED_GE, 0) for s in range(8, 16)]
    exprs = [abi.make_expr([("col", s), ("col", s + 1), "+", ("i", 0), ">="]) for s in (16, 18, 20, 22)]
    code = _refusal(gpu, ctx, [key32] + cols, inner, abi.ScanDesc(preds, exprs), many)
    assert code == abi.SR_ERR_NOT_SUPPORTED, "more than SR_MAX_VALUES distinct columns"
    semi_pay = [(abi.JOIN_LEFT_SEMI, INT, keys, [(11, keys.copy(), None, INT)])]
    code = _refusal(gpu, ctx, [key32] + cols, semi_pay, abi.ScanDesc(), count, at_create=True)
    assert code == abi.SR_ERR_INVALID_ARGUMENT, "payload on a LEFT SEMI join"
    code = _refusal(gpu, ctx, [(0, key32[1].astype(np.int64), None, BIG)] + cols, inner, abi.ScanDesc(), count)
    assert code == abi.SR_ERR_INVALID_ARGUMENT, "BIGINT probe key on an INT join"
    code = _refusal(gpu, ctx, [(0, key32[1].astype(np.float64), None, DBL)] + cols,
                    [(abi.JOIN_INNER, BIG, keys.astype(np.int64), [])], abi.ScanDesc(), count)
    assert code == abi.SR_ERR_INVALID_ARGUMENT, "DOUBLE probe key"
