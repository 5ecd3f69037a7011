"""Other-join conjuncts on INNER and LEFT SEMI joins inside the fused fragment, against an exact star-join reference.

A join's other-join conjunct is a boolean expression over the fact row and the join's build row; NULL counts as false.
An INNER join emits a (fact row, build row) combination only when the conjunct holds for it; a LEFT SEMI join passes the
row once when the conjunct holds for some build row with its key.  The fragment must feed the aggregate exactly the
combinations `sr_join_probe` (with the conjunct) followed by `sr_agg_push` would, and count them in rows_passed.
`star_conj` restates that chain over Python values; `test_reference_agrees_with_the_oracle` checks it against the
oracle's per-operator chain (oracle.Join with the conjunct, then oracle.Agg) on every case.

`CASES` puts a conjunct join at every planner position (streamed first or second, a gather pass, inline in the final
pass), with unique and duplicate build keys, range-mapped and hash tables, INT and BIGINT keys, conjuncts over fact
columns, build columns that are not payloads, or both, with NULLs under each, in interpreted and simple form, and with
no GROUP BY, a dense shared-memory aggregate and a hash aggregate that refuses and retries rows.  The Q95 / Q94 tests
check the self join with `wh1 <> wh2` against closed forms of the generator.
"""
import collections

import numpy as np
import pytest

from starrocks_b200 import abi, tpcds
from starrocks_b200.abi import Chunk
from tests.test_gpu_frag_outer_anti import JT, KJ, make_kcase
from tests.test_gpu_frag_plans import BIG, BOT, INT, PASSES, STAR, SUM, TOP, G4, G7, _morsel, _used_slots
from tests.test_gpu_join_edges import LINEAR, RANGE, _check_plan
from tests.test_gpu_value_edges import check_agg, col_values, ref_agg, ref_expr, ref_pred

TAG = 80                 # nullable fact column 0..4 that conjuncts read
REDUCED_N = 6000


def tag_slot(k):
    """the build column of join k that only its conjunct reads (never a payload)"""
    return 10 * (k + 1) + 5


# conjunct shapes over fact TAG and join k's build tag
def c_both(k):          # interpreted: C_NE_I
    return [("col", TAG), ("col", tag_slot(k)), "!="]


def c_fact(k):          # interpreted, fact columns only
    return [("col", TAG), ("i", 2), "<"]


def c_build(k):         # interpreted, build column only
    return [("col", tag_slot(k)), ("i", 1), ">"]


def c_simple(k):        # F_BIN_CC: TAG - tag, true when nonzero (the same rows as !=)
    return [("col", TAG), ("col", tag_slot(k)), "-"]


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
CJoin = collections.namedtuple("CJoin", "kind probe keys payload build conj")   # build: {slot: (values, type)} of every build column


class _Const:
    """a build value seen by ref_expr at any row index"""
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = v

    def __getitem__(self, i):
        return self.v


def star_conj(scan, joins, agg, fact_cols):
    """the combinations that reach the aggregate -> ({slot: Python values}, {slot: type}, rows_passed), joins in hint
    order.  A NULL key never matches.  A join's conjunct (an RPN over fact slots and its build slots, or None) filters
    its candidate build rows first; NULL is false.  inner: one combination per passing build row; semi: the row once
    when one passes; anti: the row once when none matches; outer: as inner, or one with NULL payloads."""
    fc = {s: col_values(d, nl) for s, d, nl, _ in fact_cols}
    types = {s: t for s, _, _, t in fact_cols}
    for rj in joins:
        types.update({s: t for s, (_, t) in rj.build.items()})
    n = len(next(iter(fc.values())))
    preds, exprs = scan
    rows = range(n)
    for slot, op, lo, hi, ins in preds:
        rows = [i for i in rows if ref_pred(op, fc[slot][i], lo, hi, ins)]
    for rpn in exprs:
        rows = [i for i in rows if (lambda r: not r[1] and r[0] != 0)(ref_expr(rpn, fc, types, i))]
    combos = [(i,) for i in rows]
    for rj in joins:
        index = {}
        for b, k in enumerate(rj.keys):
            if k is not None:
                index.setdefault(k, []).append(b)

        def holds(i, b):
            env = collections.ChainMap({s: _Const(v[b]) for s, (v, _) in rj.build.items() if s not in fc}, fc)
            v, nl = ref_expr(rj.conj, env, types, i)
            return not nl and v != 0

        col = fc[rj.probe]
        nxt = []
        for c in combos:
            k = col[c[0]]
            m = index.get(k, []) if k is not None else []
            if rj.conj is not None:
                m = [b for b in m if holds(c[0], b)]
            if rj.kind == "semi":
                if m:
                    nxt.append(c + (None,))
            elif rj.kind == "anti":
                if not m:
                    nxt.append(c + (None,))
            elif m:
                nxt.extend(c + (b,) for b in m)
            elif rj.kind == "outer":
                nxt.append(c + (None,))
        combos = nxt
    cols = {}
    for s in _used_slots(agg):
        if s in fc:
            cols[s] = [fc[s][c[0]] for c in combos]
            continue
        for j, rj in enumerate(joins):
            if s in rj.payload:
                v, types[s] = rj.payload[s]
                cols[s] = [None if c[1 + j] is None else v[c[1 + j]] for c in combos]
                break
        else:
            raise KeyError(f"slot {s} is neither a fact column nor a payload")
    return cols, types, len(combos)


def test_reference_known_answers():
    # fact rows 0..4 probe join A (INNER, duplicate key 1, conjunct TAG != tag) and join B (LEFT SEMI, duplicate key 5,
    # conjunct tag > 1, a NULL tag)
    fact = [(0, np.array([1, 1, 2, 1, 3], np.int32), None, INT), (1, np.array([5, 5, 5, 6, 5], np.int32), None, INT),
            (TAG, np.array([0, 1, 2, 0, 3], np.int32), np.array([0, 0, 0, 1, 0], np.uint8), INT),
            (6, np.array([10, 20, 30, 40, 50], np.int32), None, INT)]
    a = CJoin("inner", 0, [1, 1, 2, 3], {11: ([100, 101, 200, 300], INT)},
              {15: ([0, 1, 2, 3], INT), 11: ([100, 101, 200, 300], INT)}, c_both(0))
    b = CJoin("semi", 1, [5, 5, 6], {}, {25: ([1, None, 2], INT)}, c_build(1))
    fns = [STAR, SUM(6, INT, 40)]
    cols, types, passed = star_conj(([], []), [a, b], ([11], fns), fact)
    # row 0 (TAG 0): A rows 100 (tag 0: fails), 101 (tag 1) -> 1; B: key 5, tags 1 (fails) / NULL (fails) -> row dropped
    # row 3 (TAG NULL): every A conjunct NULL -> dropped.  B only passes key 6 (tag 2): row 3, which A already dropped
    assert passed == 0 and ref_agg(cols, types, [11], fns) == {}
    b2 = b._replace(conj=[("col", 25), "isnull"])
    cols, types, passed = star_conj(([], []), [a, b2], ([11], fns), fact)
    # B now passes key 5 (a NULL tag); row 0 -> A 101; row 1 (TAG 1) -> A 100 (tag 0 != 1) only; row 2 key 2 tag 2 == 2
    # fails; row 4 (key 3, TAG 3 == tag 3) fails
    assert passed == 2 and ref_agg(cols, types, [11], fns) == {(101,): [1, 10], (100,): [1, 20]}


# ---------------------------------------------------------------------------------------------------------------------
# cases.  Fact slot k probes join k, TAG is read by conjuncts; join k's build keys are at 10 (k + 1), its payloads at
# 10 (k + 1) + 1 and + 2, its conjunct-only column at tag_slot(k)
# ---------------------------------------------------------------------------------------------------------------------
Entry = collections.namedtuple("Entry", "build n plan")
CASES = {}


def case(name, n, plan):
    def deco(fn):
        CASES[name] = Entry(fn, n, plan)
        return fn
    return deco


def _pass(ns, gp, final, order, methods, agg_smem=None):
    p = {"mode": PASSES, "num_stream_joins": ns, "num_gather_passes": gp, "final_pass": final, "order": order, "method": methods}
    if agg_smem is not None:
        p["agg_in_smem"] = agg_smem
    return p


def make_ccase(seed, n, mode, joins, conjs, agg_keys, fns, facts=(), tag_null=0.0, btag_null=0.0, preds=()):
    """make_kcase plus the TAG fact column and, for every join with a conjunct (conjs[k] a c_* shape or None), its
    conjunct-only build column tag_slot(k) of values 0..4"""
    c = make_kcase(seed, n, mode, joins, agg_keys, fns, facts=facts, preds=preds)
    rng = np.random.default_rng(seed + 1)
    c.fact_cols.append((TAG, rng.integers(0, 5, n, dtype=np.int32), (rng.random(n) < tag_null).astype(np.uint8) if tag_null else None, INT))
    for k, (j, cf) in enumerate(zip(c.joins, conjs)):
        j["conj"] = cf(k) if cf else None
        nb = len(j["keys"])
        j["extra"] = [(tag_slot(k), rng.integers(0, 5, nb, dtype=np.int32), (rng.random(nb) < btag_null).astype(np.uint8) if btag_null else None, INT)] if cf else []
    return c


@case("inner_unique_stream0_both", 120_007, _pass(1, 1, "generic", [0, 1], [RANGE, RANGE], True))
def _(n, seed, mode=2):
    # the conjunct join is the most selective: streamed first; TAG != tag over a dense shared-memory aggregate
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("inner", 0.5, TOP, 2999)], [c_both, None],
                      [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("semi_dup_stream1_build", 120_007, _pass(2, 0, "generic", [0, 1], [RANGE, RANGE], True))
def _(n, seed, mode=2):
    # a LEFT SEMI join with duplicate keys streamed second; its conjunct reads only a build column with NULLs
    return make_ccase(seed, n, mode, [KJ("inner", 0.3, 0, 1999, pays=["g7"]), KJ("semi", 0.5, TOP, 2999, nb=3000, dup=True)],
                      [None, c_build], [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6], btag_null=0.2)


@case("inner_dup_gather_hash_big", 120_007, _pass(1, 1, "expand", [0, 1], [RANGE, LINEAR]))
def _(n, seed, mode=2):
    # an expanding INNER hash join on BIGINT keys in a gather pass; TAG != tag with NULLs under the fact column; its
    # INT payload is a SUM input
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("inner", 0.5, typ=BIG, kind="spread", nb=3000, dup=True, pays=["int"])],
                      [None, c_both], [(11, INT, G7, False)], [SUM(21, INT, 40), STAR, SUM(6, INT, 41)], facts=[6], tag_null=0.1)


@case("semi_linear_inline_fact_single", 120_007, _pass(1, 0, "generic", [0, 1], [RANGE, LINEAR]))
def _(n, seed, mode=2):
    # a LEFT SEMI hash join that passes 95 % is tested inline by the final pass; its conjunct reads only the nullable
    # fact column; no GROUP BY
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999), KJ("semi", 0.95, kind="spread", nb=3000)], [None, c_fact],
                      [], [STAR, SUM(6, INT, 40)], facts=[6], tag_null=0.1)


@case("inner_dup_inline_simple", 120_007, _pass(1, 0, "expand", [0, 1], [RANGE, RANGE], False))
def _(n, seed, mode=2):
    # an expanding INNER join inline in the final pass with the simple form TAG - tag (NULLs under both columns); its
    # payload is a group key without a range: a hash aggregate
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999), KJ("inner", 0.95, BOT, 999, nb=3000, dup=True, pays=["big"])],
                      [None, c_simple], [(21, BIG, None, False)], [STAR, SUM(6, INT, 40)], facts=[6], tag_null=0.1, btag_null=0.1)


@case("inner_expand_hash_retry", 1_250_003, _pass(1, 1, "expand", [0, 1, 2], [RANGE, RANGE, RANGE], False))
def _(n, seed, mode=2):
    # the sample promises few survivors, then every row passes with a new group (fact slot 63 is a permutation): the hash
    # table refuses rows, and the final pass runs again over them, each with all its passing combinations
    return make_ccase(seed, n, mode, [KJ("inner", 1.0, 0, 2999, rate0=0.02), KJ("inner", 1.0, TOP, 2999, rate0=0.5),
                                      KJ("inner", 0.95, BOT, 999, nb=3000, dup=True)], [None, None, c_both],
                      [(63, INT, None, False)], [STAR], facts=[63])


@case("semi_and_inner_conjuncts_expand", 120_007, _pass(1, 2, "expand", [0, 1, 2, 3], [RANGE] * 4))
def _(n, seed, mode=2):
    # two conjunct joins in one fragment, a LEFT SEMI and an expanding INNER one, ahead of an expanding join without a
    # conjunct: when that join's chain ends, the odometer carries into the conjunct join, which moves to its next passing
    # entry, and back to its first passing entry when it ends
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("semi", 0.45, TOP, 2999, nb=3000, dup=True),
                                      KJ("inner", 0.65, BOT, 999, nb=3000, dup=True, pays=["int"]), KJ("inner", 0.97, 5000, 999, nb=3000, dup=True)],
                      [None, c_build, c_both, None], [(11, INT, G7, False)], [STAR, SUM(31, INT, 40)], facts=[], btag_null=0.1)


@case("expand_then_conjunct_last", 120_007, _pass(1, 1, "expand", [0, 1, 2], [RANGE] * 3))
def _(n, seed, mode=2):
    # the expanding conjunct join is the odometer's last (fastest) join: when its chain ends it starts again from its
    # first passing entry, not the chain head, while the join before it advances
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("inner", 0.6, TOP, 2999, nb=3000, dup=True, pays=["int"]),
                                      KJ("inner", 0.97, BOT, 999, nb=3000, dup=True)], [None, None, c_simple],
                      [(11, INT, G7, False)], [STAR, SUM(21, INT, 40)], facts=[], tag_null=0.05)


@case("mixed_outer_anti_big", 120_007, _pass(1, 1, "generic", [0, 1, 2], [RANGE, RANGE, RANGE], True))
def _(n, seed, mode=2):
    # a conjunct join on BIGINT range-mapped keys next to a LEFT ANTI join and a LEFT OUTER payload group key
    return make_ccase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, typ=BIG, pays=["g7"]), KJ("anti", 0.5, TOP, 2999), KJ("outer", 0.6, BOT, 999, pays=["g4"])],
                      [c_simple, None, None], [(11, INT, G7, False), (31, INT, G4, True)], [SUM(6, INT, 40), STAR], facts=[6])


def build_case(name, n=None, mode=None):
    e = CASES[name]
    seed = 9000 + sorted(CASES).index(name)
    return e.build(n or e.n, seed) if mode is None else e.build(n or e.n, seed, mode)


def cref_joins(c):
    out = []
    for j in c.joins:
        build = {s: (col_values(d, nl), t) for s, d, nl, t in j["pay"] + j["extra"]}
        out.append(CJoin(j["kind"], j["probe"], col_values(j["keys"], j["knulls"]), {s: (col_values(d, nl), t) for s, d, nl, t in j["pay"]},
                         build, j["conj"]))
    return out


def creference(c, fact_cols=None):
    return star_conj((c.preds, c.exprs), cref_joins(c), (c.key_slots(), c.fns), fact_cols or c.fact_cols)


def _join_desc(j, probe_out=(), probe_out_types=()):
    """the join's descriptor: its payloads and conjunct columns are declared as build outputs with their types (what a
    build side that never receives a chunk is probed with)"""
    outs = j["pay"] + j["extra"]
    return abi.make_join_desc(JT[j["kind"]], [j["key_slot"]], [j["probe"]], [j["typ"]], build_out=[s for s, _, _, _ in outs],
                              build_out_types=[t for _, _, _, t in outs], probe_out=probe_out, probe_out_types=probe_out_types,
                              other_conjunct=j["conj"])


def _build_chunk(j):
    return Chunk([(j["key_slot"], j["keys"], j["knulls"], j["typ"])] + j["pay"] + j["extra"])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the reference against the oracle's per-operator chain
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_chain(oracle, c):
    """sr_join_probe per join (with its conjunct), then the aggregate, on the oracle -> (output columns, rows reaching it)"""
    cur = [(s, d, nl, t) for s, d, nl, t in c.fact_cols]
    for p in c.preds:
        keep = np.array([ref_pred(p[1], v, p[2], p[3], p[4]) for v in col_values(*[(d, nl) for s, d, nl, _ in cur if s == p[0]][0])], bool)
        cur = [(s, d[keep], None if nl is None else nl[keep], t) for s, d, nl, t in cur]
    for j in c.joins:
        slots = [s for s, _, _, _ in cur]
        oj = oracle.Join(_join_desc(j, probe_out=slots, probe_out_types=[t for _, _, _, t in cur]))
        oj.append_build(_build_chunk(j))
        oj.build()
        chunk = Chunk(cur)
        pi, bi = oj.probe_all(chunk, cap=max(1024, chunk.num_rows * 8))
        types = {s: t for s, _, _, t in cur}
        types.update({s: t for s, _, _, t in j["pay"] + j["extra"]})
        pays = {s for s, _, _, _ in j["pay"]}
        cur = [(s, d, nl if nl.any() else None, types[s]) for s, d, nl in oj.output(chunk, pi, bi) if s in slots or s in pays]
    a = oracle.Agg(c.agg_desc())
    n = len(cur[0][1])
    if n:
        a.push(Chunk(cur))
    return a.output(), n


@pytest.mark.parametrize("name", list(CASES))
def test_reference_agrees_with_the_oracle(oracle, name):
    c = build_case(name, REDUCED_N)
    cols, types, passed = creference(c)
    out, opassed = _oracle_chain(oracle, c)
    assert opassed == passed, f"{name}: the oracle chain passed {opassed}, the reference {passed}"
    check_agg(out, cols, types, c.key_slots(), c.fns, f"oracle {name}")


# ---------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------
class Run:
    def __init__(self, gpu, ctx, c, mode=None):
        self.ctx = ctx
        self.joins, self.frag, self.keep = [], None, []
        try:
            for j in c.joins:
                g = gpu.Join(ctx, _join_desc(j))
                self.joins.append(g)
                if len(j["keys"]) or j.get("zero_row_chunk"):   # an empty build side gets no chunk unless asked for one of no rows
                    g.append_build(_build_chunk(j))
                g.build_finish()
            self.frag = gpu.Fragment(ctx, c.scan_desc(), [(g, j["probe"], [s for s, _, _, _ in j["pay"]]) for g, j in zip(self.joins, c.joins)],
                                     c.agg_desc(), mode=c.mode if mode is None else mode)
        except Exception:
            self.close()
            raise

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
    cols, types, want = creference(c, fact_cols)
    assert passed == want, f"{label}: {passed} rows passed, want {want}"
    check_agg(out, cols, types, c.key_slots(), c.fns, label)


def _run_all(gpu, ctx, c, mode=None):
    r = Run(gpu, ctx, c, mode)
    try:
        r.push(c.fact_cols, 0, c.n)
        return r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conjunct_case(gpu, ctx, name):
    c = build_case(name)
    plan, passed, out = _run_all(gpu, ctx, c)
    _check_plan(plan, CASES[name].plan, name)
    _check(c, out, passed, label=name)
    if name == "inner_expand_hash_retry":
        # the push sizes the table for twice the sampled survivor estimate + 2^16 and grows it by 4x steps until that
        # fills at most half of it: at most 8x that many slots, fewer than the groups, so rows were refused and retried
        est = plan["pred_rate"] * float(np.prod(plan["pass_rate"]))
        assert len(out[0][1]) > 8 * (c.n * est * 2 + (1 << 16)), (len(out[0][1]), est)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["inner_unique_stream0_both", "semi_dup_stream1_build", "inner_dup_gather_hash_big"])
def test_mode_hints_agree(gpu, ctx, name):
    # a conjunct forces the selection-vector passes: mode_hint 0, 1 and 2 plan and compute the same
    c = build_case(name, 90_001)
    got = []
    for mode in (0, 1, 2):
        plan, passed, out = _run_all(gpu, ctx, c, mode)
        assert plan["mode"] == PASSES, (name, mode)
        _check(c, out, passed, label=f"{name} mode_hint {mode}")
        got.append(passed)
    assert len(set(got)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["inner_unique_stream0_both", "inner_dup_gather_hash_big", "semi_linear_inline_fact_single"])
def test_multi_push_ragged_last_morsel(gpu, ctx, name):
    c = build_case(name, 1 + 4095 + 4097 + 65_537 + 3)
    cuts = np.cumsum([0, 65_537, 1, 4095, 4097, 3]).tolist()
    r = Run(gpu, ctx, c)
    try:
        for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            r.push(c.fact_cols, a, b, ("host", "device", "pinned", "device_off4")[k % 4])
        passed = r.frag.rows_passed
        out = r.result()
    finally:
        r.close()
    _check(c, out, passed, label=f"morsels {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["semi_linear_inline_fact_single", "inner_dup_gather_hash_big"])
def test_push_chunks_pinned_conjunct_only_column(gpu, ctx, name):
    # TAG is read by the conjunct alone: push_chunks must still gather it
    c = build_case(name, 90_001)
    assert TAG not in _used_slots((c.key_slots(), c.fns)) and TAG not in [s for s, *_ in c.preds]
    cuts = [0, 30_000, 30_001, 65_536, c.n]
    r = Run(gpu, ctx, c)
    try:
        chunks = [_morsel(c.fact_cols, a, b, "pinned", r.keep) for a, b in zip(cuts[:-1], cuts[1:])]
        r.frag.push_chunks(chunks)
        passed = r.frag.rows_passed
        out = r.result()
    finally:
        r.close()
    _check(c, out, passed, label=f"push_chunks {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", ["none", "zero_rows"])
@pytest.mark.parametrize("kind", ["inner", "semi"])
def test_empty_build_side(gpu, ctx, kind, chunk):
    # the conjunct join's build side is empty: without any chunk (its conjunct column's type comes from build_out_types)
    # or with one chunk of no rows.  It passes nothing
    c = make_ccase(5, 70_001, 2, [KJ("inner", 0.3, 0, 2999, pays=["g7"]), KJ(kind, 0.5, TOP, 2999)], [None, c_both],
                   [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])
    j = c.joins[1]
    j["keys"] = j["keys"][:0]
    j["knulls"] = None
    j["extra"] = [(s, d[:0], None, t) for s, d, _, t in j["extra"]]
    j["zero_row_chunk"] = chunk == "zero_rows"
    plan, passed, out = _run_all(gpu, ctx, c)
    assert passed == 0
    _check(c, out, passed, label=f"empty build {kind} chunk {chunk}")


# -- the Q95 / Q94 self join against closed forms of the generator --
def _q95_data(sf):
    gen = tpcds.Q95Gen(sf)
    ws = gen.web_sales_of_orders(0, gen.n_orders)
    return gen, ws


def _fact(ws, slots):
    cols = {tpcds.WS_ORDER: "ws_order_number", tpcds.WS_WH: "ws_warehouse_sk", tpcds.WS_SHIP_DATE: "ws_ship_date_sk", tpcds.WS_ADDR: "ws_ship_addr_sk",
            tpcds.WS_SITE: "ws_web_site_sk", tpcds.WS_COST: "ws_ext_ship_cost", tpcds.WS_PROFIT: "ws_net_profit"}
    typ = {name: t for name, _, t in tpcds.WS_COLS}
    return [(s, np.ascontiguousarray(ws[cols[s]]), None, typ[cols[s]]) for s in slots]


def _self_build(ws):
    return Chunk([(tpcds.WS2_ORDER, np.ascontiguousarray(ws["ws_order_number"]), None, abi.TYPE_BIGINT),
                  (tpcds.WS2_WH, np.ascontiguousarray(ws["ws_warehouse_sk"]), None, abi.TYPE_INT)])


def _closed_joins(gpu, ctx, specs):
    out = []
    try:
        for desc, chunk, probe in specs:
            g = gpu.Join(ctx, desc)
            out.append((g, probe, []))
            g.append_build(chunk)
            g.build_finish()
    except Exception:
        for g, _, _ in out:
            g.close()
        raise
    return out


@pytest.mark.gpu
def test_q95_ws_wh_closed_form(gpu, ctx):
    # ws_wh: the orders whose lines ship from more than one warehouse (mn != mx of Q95Gen.expected)
    gen, ws = _q95_data(0.5)
    d = tpcds.fused_conj_descs()
    o = np.arange(gen.n_orders)
    rep, _ = gen._expand(gen.lines_per_order(o))
    wh = ws["ws_warehouse_sk"]
    mn, mx = np.full(gen.n_orders, 1 << 30), np.zeros(gen.n_orders, np.int64)
    np.minimum.at(mn, rep, wh)
    np.maximum.at(mx, rep, wh)
    want_orders = np.flatnonzero(mn != mx) + 1
    per = np.bincount(rep, minlength=gen.n_orders)
    same = np.zeros(gen.n_orders, np.int64)     # (line, line) pairs of an order on the same warehouse
    for w in np.unique(wh):
        same += np.bincount(rep[wh == w], minlength=gen.n_orders) ** 2
    want_pairs = int((per ** 2 - same).sum())
    fact = _fact(ws, [tpcds.WS_ORDER, tpcds.WS_WH])
    joins = _closed_joins(gpu, ctx, [(d["ws_wh_join"], _self_build(ws), tpcds.WS_ORDER)])
    try:
        f = gpu.Fragment(ctx, abi.ScanDesc(), joins, d["ws_wh_agg"](len(want_orders)))
        try:
            keep = []
            n = len(fact[0][1])
            for lo in range(0, n, 1 << 20):
                f.push(_morsel(fact, lo, min(n, lo + (1 << 20)), "device", keep))
            assert f.plan()["final_pass"] == "expand"
            passed = f.rows_passed
            (_, t, keys, _), = f.agg.result()
            ctx.sync()
        finally:
            f.close()
    finally:
        for g, _, _ in joins:
            g.close()
    assert passed == want_pairs
    assert np.array_equal(np.sort(np.asarray(keys)), want_orders)


@pytest.mark.gpu
def test_q94_body_closed_form(gpu, ctx):
    gen, ws = _q95_data(0.5)
    d = tpcds.fused_conj_descs()
    wr = gen.web_returns_of_orders(0, gen.n_orders)["wr_order_number"]
    one = lambda slot, keys, t=abi.TYPE_INT: Chunk([(slot, np.ascontiguousarray(keys), None, t)])  # noqa: E731
    fact = _fact(ws, [tpcds.WS_ORDER, tpcds.WS_WH, tpcds.WS_SHIP_DATE, tpcds.WS_ADDR, tpcds.WS_SITE, tpcds.WS_COST, tpcds.WS_PROFIT])
    joins = _closed_joins(gpu, ctx, [(d["q94_semi_date"], one(tpcds.D_DATE_SK, gen.date_keys()), tpcds.WS_SHIP_DATE),
                                     (d["q94_semi_addr"], one(tpcds.CA_ADDRESS_SK, gen.address_keys()), tpcds.WS_ADDR),
                                     (d["q94_semi_site"], one(tpcds.WEB_SITE_SK, gen.site_keys()), tpcds.WS_SITE),
                                     (d["q94_exists"], _self_build(ws), tpcds.WS_ORDER),
                                     (d["q94_not_returned"], one(tpcds.WR_ORDER, wr, abi.TYPE_BIGINT), tpcds.WS_ORDER)])
    try:
        f = gpu.Fragment(ctx, d["q94_scan"], joins, d["q94_agg"])
        try:
            keep = []
            f.push(_morsel(fact, 0, len(fact[0][1]), "device", keep))
            passed = f.rows_passed
            res = f.agg.result()
            ctx.sync()
        finally:
            f.close()
    finally:
        for g, _, _ in joins:
            g.close()
    want = tpcds.q94_expected(gen, 0, gen.n_orders)
    got = tuple(int(np.asarray(dd)[0]) for _, _, dd, _ in res)
    assert want[0] > 0 and passed == want[0] and got == want


# -- refusals: on the first push, before any launch --
@pytest.mark.gpu
def test_refusals(gpu, ctx):
    keys = np.arange(100, dtype=np.int32)
    fact = Chunk([(0, keys.copy(), None, INT), (1, keys.copy(), None, INT), (2, keys.astype(np.float64), None, abi.TYPE_DOUBLE)] +
                 [(50 + k, keys.copy(), None, INT) for k in range(16)])

    def refused(conj0=None, conj1=None, pays0=(), fns=(STAR,)):
        gs = []
        try:
            for k, (conj, pays) in enumerate(((conj0, list(pays0)), (conj1, []))):
                g = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [10 * (k + 1)], [k], [INT], other_conjunct=conj))
                gs.append(g)
                g.append_build(Chunk([(10 * (k + 1), keys, None, INT), (10 * (k + 1) + 1, keys.copy(), None, INT), (10 * (k + 1) + 5, keys.copy(), None, INT)]))
                g.build_finish()
            f = gpu.Fragment(ctx, abi.ScanDesc(), [(gs[0], 0, list(pays0)), (gs[1], 1, [])], abi.make_agg_desc(fns=list(fns)), mode=2)
            try:
                with pytest.raises(gpu.GpuError) as ei:
                    f.push(fact)
                assert f.rows_passed == 0
                return ei.value.code, str(ei.value)
            finally:
                f.close()
        finally:
            for g in gs:
                g.close()

    # join 1's conjunct reads a payload of join 0
    code, msg = refused(conj1=[("col", 11), ("col", 1), "<"], pays0=[11])
    assert code == abi.SR_ERR_NOT_SUPPORTED and "slot 11" in msg and "join 1" in msg and "join 0" in msg, msg
    # ... or any other build column of join 0, or one join 0's conjunct reads
    code, msg = refused(conj1=[("col", 11), ("col", 1), "<"])
    assert code == abi.SR_ERR_NOT_SUPPORTED and "slot 11" in msg and "join 0" in msg, msg
    code, msg = refused(conj0=[("col", 15), ("col", 0), "<"], conj1=[("col", 15), ("col", 1), "<"])
    assert code == abi.SR_ERR_NOT_SUPPORTED and "slot 15" in msg, msg
    # a slot on neither side
    code, msg = refused(conj0=[("col", 77), ("col", 0), "<"])
    assert code == abi.SR_ERR_INVALID_ARGUMENT, msg
    # a double-valued conjunct
    code, msg = refused(conj0=[("col", 2), ("col", 15), "+"])
    assert code == abi.SR_ERR_INVALID_ARGUMENT and "not boolean" in msg, msg
    # more than SR_MAX_VALUES (20) distinct columns: 2 keys + 11 + 8 conjunct columns

    def chain(slots):
        rpn = [("col", slots[0])]
        for s in slots[1:]:
            rpn += [("col", s), "+"]
        return rpn + [("i", 0), "!="]
    code, msg = refused(conj0=chain([50 + k for k in range(10)] + [15]), conj1=chain([60 + k for k in range(6)] + [25, 21]))
    assert code == abi.SR_ERR_NOT_SUPPORTED and "too many" in msg, msg
    # a conjunct stays refused on LEFT ANTI and LEFT OUTER joins (test_gpu_frag_outer_anti.test_refusals), and an empty
    # build side whose conjunct column's type is not declared
    g = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [10], [0], [INT], other_conjunct=[("col", 15), ("col", 1), "<"]))
    try:
        g.build_finish()
        f = gpu.Fragment(ctx, abi.ScanDesc(), [(g, 0, [])], abi.make_agg_desc(fns=[STAR]), mode=2)
        try:
            with pytest.raises(gpu.GpuError) as ei:
                f.push(fact)
            assert ei.value.code == abi.SR_ERR_STATE and "build_out_types" in str(ei.value)
        finally:
            f.close()
    finally:
        g.close()
