"""LEFT ANTI and LEFT OUTER joins inside the fused fragment, against an exact star-join reference in plain Python.

A LEFT ANTI join (not null-aware) lets a fact row through when its key is NULL or no build row has it.  A LEFT OUTER
join never drops a row: it emits one combination per matching build row, or one whose payloads are all NULL.  The
fragment must produce exactly the combinations the per-operator chain (sr_join_probe per join, then sr_agg_push) feeds
the aggregate, so `star_kinds` restates that chain over Python values, `test_reference_known_answers_per_join_type`
pins it against `ref_join`'s pairs, and `test_reference_agrees_with_the_oracle` checks it against the oracle's
per-operator `orc_fragment_run` on every case.

`CASES` puts an anti join at every position the planner has (streamed with a shared or global bitmap or in the general
form, a gather pass, inline in the generic or the batched final pass, a cascade stage) and an outer join at every way
the final passes handle it (a looked-up payload, a directory with the all-NULL digit, an expanding chain, an unread join
with unique or duplicate keys, the cascade, the hash-aggregate retry).  `test_plan_table_covers_every_cell` checks on
the CPU that the table reaches every cell; `test_outer_anti_case` checks each case's plan and result on the device.
"""
import collections

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from tests.test_gpu_frag_plans import (BIG, BOT, CASCADE, COUNT, G4, G7, INT, MAX, PASSES, SAMPLE, STAR, SUM, TOP, J, _morsel, _used_slots,
                                       _with_nulls, make_case)
from tests.test_gpu_join_edges import LINEAR, RANGE, _check_plan, ref_join
from tests.test_gpu_value_edges import check_agg, col_values, ref_agg, ref_expr, ref_pred

JT = {"inner": abi.JOIN_INNER, "semi": abi.JOIN_LEFT_SEMI, "anti": abi.JOIN_LEFT_ANTI, "outer": abi.JOIN_LEFT_OUTER}


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
KJoin = collections.namedtuple("KJoin", "kind probe keys payload")   # kind: a JT key; payload: {build slot: (values, type)}


def star_kinds(scan, joins, agg, fact_cols):
    """the combinations that reach the aggregate -> ({slot: Python values}, {slot: type}, rows_passed), joins in hint
    order.  A NULL key never matches.  inner: one combination per matching build row; semi: the row once when one
    matches; anti: the row once when none matches (NULL keys included); outer: as inner, or one combination with NULL
    payloads when none matches."""
    fc = {s: col_values(d, nl) for s, d, nl, _ in fact_cols}
    types = {s: t for s, _, _, t in fact_cols}
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
        col = fc[rj.probe]
        nxt = []
        for c in combos:
            k = col[c[0]]
            m = index.get(k) if k is not None else None
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


def test_reference_known_answers_per_join_type():
    # every join type of the fragment against ref_join's (probe row, build row) pairs on its edge cases: duplicate and
    # NULL build keys, NULL probe keys, keys outside the build range on both sides, an empty build side
    builds = {"dup_and_null": [1, 1, 2, None, 5], "unique": [3, 1, 2], "empty": []}
    probe = [1, 2, None, 0, 6, 5, 1, 4]
    fact = [(0, np.array([0 if k is None else k for k in probe], np.int32), np.array([k is None for k in probe], np.uint8), INT)]
    for bname, bkeys in builds.items():
        pay = [100 + b for b in range(len(bkeys))]
        for kind, jt in JT.items():
            pairs, _ = ref_join([(k,) for k in bkeys], [(k,) for k in probe], jt)
            # ref_join's build indexes are 1-based, 0 = none; the payload of "none" is NULL
            want = sorted((i, None if b == 0 or kind in ("semi", "anti") else 100 + b - 1) for i, b in pairs)
            rj = KJoin(kind, 0, bkeys, {11: (pay, INT)} if kind in ("inner", "outer") else {})
            agg = ([], [(abi.AGG_COUNT_STAR, 0, 40, None)] + ([(abi.AGG_SUM, INT, 41, [("col", 11)])] if rj.payload else []))
            cols, _, passed = star_kinds(([], []), [rj], agg, fact)
            assert passed == len(pairs), (bname, kind)
            if rj.payload:
                assert sorted(cols[11], key=repr) == sorted([p for _, p in want], key=repr), (bname, kind)
    # a hand-made star: A outer with a duplicate key and a NULL payload, B anti, C inner; group by A's payload
    fact = [(0, np.array([1, 2, 7, 1, 0, 3], np.int32), np.array([0, 0, 0, 0, 1, 0], np.uint8), INT),
            (1, np.array([5, 6, 5, 9, 5, 5], np.int32), np.array([0, 0, 0, 0, 0, 1], np.uint8), INT),
            (2, np.array([8, 8, 8, 8, 8, 8], np.int32), None, INT),
            (6, np.array([10, 20, 30, 40, 50, 60], np.int32), None, INT)]
    a = KJoin("outer", 0, [1, 1, 3], {11: ([100, 101, None], INT)})
    b = KJoin("anti", 1, [6, 6, 7], {})
    c = KJoin("inner", 2, [8], {})
    fns = [(abi.AGG_COUNT_STAR, 0, 40, None), (abi.AGG_SUM, INT, 41, [("col", 6)])]
    cols, types, passed = star_kinds(([], []), [a, b, c], ([11], fns), fact)
    # row 0: two A rows x B passes (5) -> 2; row 1: B fails (6); row 2: A misses 7 -> NULL; row 3: two A rows, 9 passes
    # B -> 2; row 4: NULL A key -> NULL; row 5: A payload NULL, B key NULL passes
    assert passed == 7
    assert ref_agg(cols, types, [11], fns) == {(100,): [2, 50], (101,): [2, 50], (None,): [3, 140]}


# ---------------------------------------------------------------------------------------------------------------------
# cases: test_gpu_frag_plans.make_case with a join type per join.  Fact slot k probes join k; join k's build keys are
# at slot 10 (k + 1), its payloads at 10 (k + 1) + 1 and + 2.
# ---------------------------------------------------------------------------------------------------------------------
class KJ(J):
    """a J of join type `jt` (a JT key)"""

    def __init__(self, jt, rate, *a, **kw):
        super().__init__(rate, *a, semi=jt == "semi", **kw)
        self.jkind = jt


def make_kcase(seed, n, mode, joins, agg_keys, fns, facts=(), preds=()):
    c = make_case(seed, n, mode, joins, agg_keys, fns, facts=facts, preds=preds)
    for b, j in zip(c.joins, joins):
        b["kind"] = j.jkind
    return c


def kref_joins(c):
    return [KJoin(j["kind"], j["probe"], col_values(j["keys"], j["knulls"]), {s: (col_values(d, nl), t) for s, d, nl, t in j["pay"]})
            for j in c.joins]


def kreference(c, fact_cols=None):
    return star_kinds((c.preds, c.exprs), kref_joins(c), (c.key_slots(), c.fns), fact_cols or c.fact_cols)


Entry = collections.namedtuple("Entry", "build n plan cells")
CASES = {}


def case(name, n, plan, cells):
    def deco(fn):
        CASES[name] = Entry(fn, n, plan, set(cells))
        return fn
    return deco


def _casc(order, smem, agg_smem, methods):
    return {"mode": CASCADE, "order": order, "bitmap_in_smem": smem, "agg_in_smem": agg_smem, "num_stream_joins": 0,
            "num_gather_passes": 0, "method": methods}


def _pass(ns, gp, final, smem, agg_smem, methods, order):
    return {"mode": PASSES, "num_stream_joins": ns, "num_gather_passes": gp, "final_pass": final, "bitmap_in_smem": smem,
            "agg_in_smem": agg_smem, "method": methods, "order": order}


# -- anti joins --
@case("anti_stream_smem", 120_007, _pass(1, 1, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]), {("anti", "stream-smem")})
def _(n, seed, mode=2):
    # the anti join passes 5 %: streamed first, its bitmap in shared memory (tests kernel, VecTest kind 1)
    return make_kcase(seed, n, mode, [KJ("anti", 0.95, 0, 2999), KJ("inner", 0.5, TOP, 2999, pays=["g7"])], [(21, INT, G7, False)],
                      [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_stream_global_outer_input", 120_007, _pass(2, 0, "generic", [1, 0, 0], True, [RANGE] * 3, [0, 1, 2]),
      {("anti", "stream-global"), ("outer", "generic-input")})
def _(n, seed, mode=2):
    # the second streamed join is an anti join whose 400 K-key bitmap stays in global memory (VecTest kind 2); an outer
    # join's INT payload is a SUM input of the generic final pass
    return make_kcase(seed, n, mode, [KJ("inner", 0.12, 0, 700_000), KJ("anti", 0.6, -200_000, 200_000),
                                      KJ("outer", 0.7, BOT, 2999, pays=["int"])],
                      [(60, INT, G7, False)], [STAR, SUM(31, INT, 40), SUM(6, INT, 41)], facts=[6, 60])


@case("anti_stream_hash", 120_007, _pass(2, 0, "dense-batched", [0, 1], True, [LINEAR, RANGE], [0, 1]), {("anti", "stream-general")})
def _(n, seed, mode=2):
    # the streamed anti join is a hash table: the tests kernel's generic test, inverted
    return make_kcase(seed, n, mode, [KJ("anti", 0.9, kind="spread", nb=3000), KJ("inner", 0.5, TOP, 2999, pays=["g7"])],
                      [(21, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_stream_nullable", 120_007, _pass(1, 1, "generic", [1, 0], True, [RANGE] * 2, [0, 1]), {("anti", "stream-general")})
def _(n, seed, mode=2):
    # a nullable streamed anti key: the generic streaming kernel, where a NULL key passes
    return make_kcase(seed, n, mode, [KJ("anti", 0.97, 0, 2999, fnull=0.02), KJ("inner", 0.5, TOP, 2999, pays=["g7"])],
                      [(21, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_gather", 120_007, _pass(1, 1, "generic", [1, 0], True, [RANGE] * 2, [0, 1]), {("anti", "gather")})
def _(n, seed, mode=2):
    # an anti join with NULL probe keys in a gather pass
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("anti", 0.5, TOP, 2999, fnull=0.05)],
                      [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_inline_dense", 120_007, _pass(1, 0, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]), {("anti", "dense-test")})
def _(n, seed, mode=2):
    # an anti join passing 95 % is tested inline by the batched final pass: an inverted bitmap test
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("anti", 0.05, TOP, 2999)],
                      [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_inline_generic_hash", 120_007, _pass(1, 0, "generic", [1, 0], True, [RANGE, LINEAR], [0, 1]), {("anti", "inline-generic")})
def _(n, seed, mode=2):
    # an anti hash join with duplicate build keys tested inline by the generic final pass
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["int"]), KJ("anti", 0.04, kind="spread", nb=2000, dup=True)],
                      [(60, INT, G7, False)], [SUM(11, INT, 40), STAR], facts=[60])


@case("anti_cascade_first_outer_key", 100_003, _casc([0, 1, 2], [1, 1, 0], True, [RANGE] * 3),
      {("anti", "cascade-first"), ("outer", "cascade")})
def _(n, seed, mode=1):
    # the cascade's first stage is an anti join on the streamed key; an outer join's payload is a nullable group key
    return make_kcase(seed, n, mode, [KJ("anti", 0.7, 0, 1999), KJ("inner", 0.5, TOP, 2999, pays=["g7"]), KJ("outer", 0.6, BOT, 999, pays=["g4"])],
                      [(21, INT, G7, False), (31, INT, G4, True)], [SUM(6, INT, 40), STAR], facts=[6])


@case("anti_cascade_stage", 100_003, _casc([0, 1, 2], [1, 1, 0], False, [RANGE] * 3), {("anti", "cascade-stage"), ("outer", "unique-unread")})
def _(n, seed, mode=1):
    # an anti join with NULL probe keys as the cascade's second stage; an outer join nothing reads; a hash aggregate
    return make_kcase(seed, n, mode, [KJ("inner", 0.3, 0, 1999, pays=["big"]), KJ("anti", 0.5, TOP, 2999, fnull=0.05), KJ("outer", 0.5, BOT, 999)],
                      [(11, BIG, None, False)], [STAR, SUM(6, INT, 40)], facts=[6])


# -- outer joins --
@case("outer_dense_directory", 120_007, _pass(1, 0, "dense-batched", [1, 0], True, [RANGE] * 2, [0, 1]), {("outer", "dense-directory")})
def _(n, seed, mode=2):
    # the outer join's payload is a nullable group key: its directory holds digit 0 (NULL) for missing keys, and the
    # pass reads that digit for keys outside the range
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("outer", 0.6, 0, 1999, nb=1500, pays=["g4"])],
                      [(11, INT, G7, False), (21, INT, G4, True)], [SUM(6, INT, 40), MAX(7, INT, 41), STAR], facts=[6, 7])


@case("outer_expand", 120_007, _pass(1, 0, "expand", [1, 0], True, [RANGE] * 2, [0, 1]), {("outer", "expand")})
def _(n, seed, mode=2):
    # duplicate build keys and misses: one combination per chain entry, one all-NULL combination for a miss
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999), KJ("outer", 0.6, TOP + 1000, 1999, dup=True, pays=["int", "g7"])],
                      [(22, INT, G7, True)], [STAR, SUM(21, INT, 40), COUNT(21, INT, 41)], facts=[])


@case("outer_dup_unread", 120_007, _pass(1, 0, "expand", [1, 0], True, [RANGE] * 2, [0, 1]), {("outer", "dup-unread")})
def _(n, seed, mode=2):
    # nothing reads the outer join, but its duplicate keys multiply the rows
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ("outer", 0.5, BOT, 1499, nb=3000, dup=True)],
                      [(11, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("outer_unique_unread", 120_007, _pass(1, 0, "dense-batched", [1, 0], True, [RANGE] * 2, [1, 0]), {("outer", "unique-unread")})
def _(n, seed, mode=2):
    return make_kcase(seed, n, mode, [KJ("outer", 0.5, TOP, 2999), KJ("inner", 0.05, 0, 2999, pays=["g7"])],
                      [(21, INT, G7, False)], [SUM(6, INT, 40), STAR], facts=[6])


@case("outer_hash_retry", 1_250_003, _pass(2, 0, "generic", [1, 1, 0], False, [RANGE] * 3, [0, 1, 2]), {("outer", "hash-retry")})
def _(n, seed, mode=2):
    # the sampled first 65 536 rows promise few survivors, the rest all pass with a new group per row: the hash table
    # refuses rows and the final pass runs again over them; an outer payload is the second group key
    return make_kcase(seed, n, mode, [KJ("inner", 1.0, 0, 2999, rate0=0.1), KJ("inner", 1.0, TOP, 2999, rate0=0.5),
                                      KJ("outer", 0.7, BOT, 2999, pays=["int"])],
                      [(63, INT, None, False), (31, INT, None, True)], [STAR], facts=[63])


@case("all_outer_pred", 120_007, _pass(0, 0, "dense-batched", [0, 0], True, [RANGE] * 2, [1, 0]), {("outer", "all-outer")})
def _(n, seed, mode=2):
    # no filtering join: the streaming pass tests the scan conjunct only
    return make_kcase(seed, n, mode, [KJ("outer", 0.6, 0, 2999, pays=["g7"]), KJ("outer", 0.3, TOP, 999)],
                      [(11, INT, G7, True)], [SUM(6, INT, 40), STAR], facts=[6, 50], preds=[(50, abi.PRED_BETWEEN, 0, 99, ())])


@case("all_outer_cascade", 100_003, _casc([0], [0], True, [RANGE]), {("outer", "all-outer"), ("outer", "cascade")})
def _(n, seed, mode=1):
    return make_kcase(seed, n, mode, [KJ("outer", 0.6, 0, 2999, pays=["g7", "dbl"])], [(11, INT, G7, True)],
                      [SUM(6, INT, 40), STAR, SUM(12, abi.TYPE_DOUBLE, 41)], facts=[6])


CELLS = {("anti", p) for p in ("stream-smem", "stream-global", "stream-general", "gather", "inline-generic", "dense-test",
                               "cascade-first", "cascade-stage")} | \
        {("outer", p) for p in ("generic-input", "dense-directory", "expand", "unique-unread", "dup-unread", "cascade",
                                "hash-retry", "all-outer")}
REDUCED_N = 6000


def build_case(name, n=None, mode=None):
    e = CASES[name]
    seed = 7000 + sorted(CASES).index(name)
    return e.build(n or e.n, seed) if mode is None else e.build(n or e.n, seed, mode)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the reference against the oracle, and the coverage of the table
# ---------------------------------------------------------------------------------------------------------------------
def _join_desc(j):
    """the join's descriptor; its payloads are declared as build outputs with their types, as a plan's join node declares
    them (what a build side that never receives a chunk is probed with)"""
    return abi.make_join_desc(JT[j["kind"]], [j["key_slot"]], [j["probe"]], [j["typ"]], build_out=[s for s, _, _, _ in j["pay"]],
                              build_out_types=[t for _, _, _, t in j["pay"]])


def _build_chunk(j):
    return Chunk([(j["key_slot"], j["keys"], j["knulls"], j["typ"])] + j["pay"])


def _oracle_run(oracle, c):
    joins = []
    for j in c.joins:
        oj = oracle.Join(_join_desc(j))
        if len(j["keys"]):
            oj.append_build(_build_chunk(j))
        oj.build()
        joins.append((oj, j["probe"], [s for s, _, _, _ in j["pay"]]))
    res, passed = oracle.fragment_run(c.scan_desc(), joins, c.agg_desc(), Chunk(c.fact_cols), num_threads=2)
    return res.output(), passed


@pytest.mark.parametrize("name", list(CASES))
def test_reference_agrees_with_the_oracle(oracle, name):
    c = build_case(name, REDUCED_N)
    cols, types, passed = kreference(c)
    out, opassed = _oracle_run(oracle, c)
    assert opassed == passed, f"{name}: oracle passed {opassed}, reference {passed}"
    check_agg(out, cols, types, c.key_slots(), c.fns, f"oracle {name}")


def test_plan_table_covers_every_cell():
    """Checks the table, not the planner: each case's cells must follow from its joins and its DECLARED plan.  That the
    planner makes the declared plan is asserted on the device, by `test_outer_anti_case` (_check_plan: mode, order, stream
    and gather counts, final pass, bitmap_in_smem, method).  So the streamed anti cells rest on these declared fields: a
    shared-memory bitmap (VecTest kind 1) is bitmap_in_smem 1 on a RANGE join; a global bitmap (kind 2) bitmap_in_smem 0
    on a RANGE join streamed second; the general form a LINEAR join (kind 3 through stream_test) or a nullable probe key
    (the generic streaming kernel)."""
    assert set().union(*(e.cells for e in CASES.values())) == CELLS
    for name, e in CASES.items():
        c = build_case(name, 200)
        kinds = [j["kind"] for j in c.joins]
        p = e.plan
        assert len(p["method"]) == len(p["bitmap_in_smem"]) == len(kinds) and p["method"] == [j["method"] for j in c.joins], name
        assert sorted(p["order"]) == list(range(len(kinds))), name
        order_kinds = [kinds[j] for j in p["order"]]
        nf = sum(k != "outer" for k in kinds)
        assert all(k == "outer" for k in order_kinds[nf:]) and "outer" not in order_kinds[:nf], f"{name}: outer joins go last"
        dup = {j["kind"]: len(np.unique(j["keys"])) < len(j["keys"]) for j in c.joins}
        read = _used_slots((c.key_slots(), c.fns))
        for kind, pos in e.cells:
            assert kind in kinds, (name, kind)
            if p["mode"] == CASCADE:
                assert pos.startswith("cascade") or pos in ("unique-unread", "all-outer"), (name, pos)
                if pos == "cascade-first":
                    assert order_kinds[0] == "anti", name
                if pos == "cascade-stage":
                    assert "anti" in order_kinds[1:nf], name
                continue
            ns, gp = p["num_stream_joins"], p["num_gather_passes"]
            place = {"stream-smem": order_kinds[:ns], "stream-global": order_kinds[:ns], "stream-general": order_kinds[:ns],
                     "gather": order_kinds[ns:ns + gp], "inline-generic": order_kinds[ns + gp:nf], "dense-test": order_kinds[ns + gp:nf]}
            if kind == "anti":
                assert "anti" in place[pos], (name, pos)
                q = order_kinds.index("anti")            # probe position of the (only) anti join
                aj = c.joins[p["order"][q]]
                if pos == "stream-smem":
                    assert p["bitmap_in_smem"][q] == 1 and aj["method"] == RANGE, name
                if pos == "stream-global":
                    assert p["bitmap_in_smem"][q] == 0 and aj["method"] == RANGE and q == 1, name
                if pos == "stream-general":
                    nullable_key = any(s == aj["probe"] and nl is not None for s, _, nl, _ in c.fact_cols)
                    assert aj["method"] == LINEAR or nullable_key, name
                if pos == "dense-test":
                    assert p["final_pass"] == "dense-batched", name
                if pos == "inline-generic":
                    assert p["final_pass"] == "generic", name
            else:
                outer = [j for j in c.joins if j["kind"] == "outer"]
                pays_read = any(s in read for j in outer for s, _, _, _ in j["pay"])
                want = {"generic-input": p["final_pass"] == "generic" and pays_read,
                        "dense-directory": p["final_pass"] == "dense-batched" and pays_read,
                        "expand": p["final_pass"] == "expand" and dup["outer"] and pays_read,
                        "unique-unread": not dup["outer"] and not pays_read,
                        "dup-unread": p["final_pass"] == "expand" and dup["outer"] and not pays_read,
                        "hash-retry": not p["agg_in_smem"] and e.n > 1 << 20 and pays_read,   # more groups than the 2^20 admission limit
                        "all-outer": nf == 0}[pos]
                assert want, (name, pos)


# ---------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_joins(gpu, ctx, c):
    joins = []
    try:
        for j in c.joins:
            g = gpu.Join(ctx, _join_desc(j))
            joins.append(g)
            if len(j["keys"]) or j.get("zero_row_chunk"):   # an empty build side gets no chunk unless asked for one of no rows
                g.append_build(_build_chunk(j))
            g.build_finish()
    except Exception:
        for g in joins:
            g.close()
        raise
    return joins


class Run:
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
    cols, types, want = kreference(c, fact_cols)
    assert passed == want, f"{label}: {passed} rows passed, want {want}"
    check_agg(out, cols, types, c.key_slots(), c.fns, label)


def sampled_pass_rate(c, j, fact_cols=None):
    """the fraction of the first push's sampled rows that join j (hint order) lets through, as k_frag_sample counts it"""
    fact = {s: (d, nl) for s, d, nl, _ in fact_cols or c.fact_cols}
    jd = c.joins[j]
    if jd["kind"] == "outer":
        return 1.0
    d, nl = fact[jd["probe"]]
    m = min(len(d), SAMPLE)
    valid = jd["keys"] if jd["knulls"] is None else jd["keys"][jd["knulls"] == 0]
    hit = np.isin(d[:m], valid)
    if nl is not None:
        hit &= nl[:m] == 0
    passing = ~hit if jd["kind"] == "anti" else hit
    return round(float(passing.sum()) / m, 4) if m else 1.0


def _check_rates(c, plan, label):
    for j, jd in enumerate(c.joins):
        if jd["kind"] in ("anti", "outer"):
            assert plan["pass_rate"][j] == pytest.approx(sampled_pass_rate(c, j), abs=1e-4), f"{label}: pass_rate[{j}]"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_outer_anti_case(gpu, ctx, name):
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
    _check_rates(c, plan, name)
    _check(c, out, passed, label=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["anti_cascade_first_outer_key", "anti_stream_global_outer_input", "outer_dense_directory"])
def test_cascade_and_passes_agree(gpu, ctx, name):
    # the same fragment forced into each mode: identical results
    c = build_case(name, 90_001)
    got = {}
    for mode in (1, 2):
        r = Run(gpu, ctx, c, mode)
        try:
            r.push(c.fact_cols, 0, c.n)
            assert r.plan()["mode"] == (CASCADE if mode == 1 else PASSES)
            got[mode] = (r.frag.rows_passed, r.result())
        finally:
            r.close()
        _check(c, got[mode][1], got[mode][0], label=f"{name} mode {mode}")
    assert got[1][0] == got[2][0]


# -- edges, for each kind --
def _edge_case(kind, mode, n=70_001, seed=1):
    """join 0 (inner, 5 %, its payload the group key) then join 1 of `kind`; outer joins carry a nullable group key"""
    pays = ["g4"] if kind == "outer" else []
    keys = [(11, INT, G7, False)] + ([(21, INT, G4, True)] if kind == "outer" else [])
    return make_kcase(seed, n, mode, [KJ("inner", 0.05, 0, 2999, pays=["g7"]), KJ(kind, 0.5, -100, 1999, pays=pays)], keys,
                      [SUM(6, INT, 40), STAR], facts=[6])


def _run_all(gpu, ctx, c, cols=None, mode=None):
    cols = cols or c.fact_cols
    r = Run(gpu, ctx, c, mode)
    try:
        r.push(cols, 0, c.n)
        return r.plan(), r.frag.rows_passed, r.result()
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", ["none", "zero_rows"])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["anti", "outer"])
def test_empty_build_side(gpu, ctx, kind, mode, chunk):
    # chunk "none": build_finish() without any append_build, what a dimension scan that filters every row out hands the
    # build (the outer payload's type then comes from the join's build_out_types); "zero_rows": one chunk of no rows.
    # The anti join passes every row; the outer join puts every row in the NULL group of its payload
    c = _edge_case(kind, mode)
    j = c.joins[1]
    j["keys"] = j["keys"][:0]
    j["knulls"] = None
    j["pay"] = [(s, d[:0], None, t) for s, d, _, t in j["pay"]]
    j["zero_row_chunk"] = chunk == "zero_rows"
    plan, passed, out = _run_all(gpu, ctx, c)
    assert plan["pass_rate"][1] == 1.0
    cols, _, want = kreference(c)
    assert want > 0 and (kind == "anti" or set(cols[21]) == {None})
    _check(c, out, passed, label=f"empty build {kind} mode {mode} chunk {chunk}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["anti", "outer"])
def test_null_probe_keys(gpu, ctx, kind, mode):
    # NULL probe keys whose data bytes are build keys: they pass an anti join and miss an outer join
    c = _edge_case(kind, mode)
    cols = _with_nulls(c.fact_cols, 1, 0, 0.2, 5, set_to=c.joins[1]["keys"])
    plan, passed, out = _run_all(gpu, ctx, c, cols)
    _check(c, out, passed, cols, f"NULL probe keys {kind} mode {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["anti", "outer"])
def test_keys_just_outside_the_range(gpu, ctx, kind, mode):
    # every probe key of the join is one of lo - 1, lo, hi, hi + 1 (and the type's extremes)
    c = _edge_case(kind, mode)
    lo, hi = -100, -100 + 1999
    rng = np.random.default_rng(6)
    pool = np.array([lo - 1, lo, hi, hi + 1, -(2**31), 2**31 - 1], np.int32)
    cols = [(s, pool[rng.integers(0, len(pool), c.n)] if s == 1 else d, nl, t) for s, d, nl, t in c.fact_cols]
    plan, passed, out = _run_all(gpu, ctx, c, cols)
    _check(c, out, passed, cols, f"keys outside {kind} mode {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("nullable", [False, True])
def test_outer_payload_with_and_without_null_column(gpu, ctx, nullable, mode):
    # the outer payload group key's build column with or without NULLs of its own: both NULLs fall into one group
    c = _edge_case("outer", mode)
    s, d, _, t = c.joins[1]["pay"][0]
    nl = (np.random.default_rng(7).random(len(d)) < 0.3).astype(np.uint8) if nullable else None
    c.joins[1]["pay"][0] = (s, d, nl, t)
    plan, passed, out = _run_all(gpu, ctx, c)
    if mode == 2:
        assert plan["final_pass"] == "dense-batched"
    _check(c, out, passed, label=f"outer payload nulls={nullable} mode {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["anti_stream_global_outer_input", "outer_expand", "anti_cascade_first_outer_key", "all_outer_pred"])
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
@pytest.mark.parametrize("name", ["anti_stream_smem", "outer_dense_directory"])
def test_push_chunks_pinned(gpu, ctx, name):
    c = build_case(name, 90_001)
    cuts = [0, 30_000, 30_001, 65_536, c.n]
    r = Run(gpu, ctx, c)
    try:
        chunks = [_morsel(c.fact_cols, a, b, "pinned", r.keep) for a, b in zip(cuts[:-1], cuts[1:])]
        r.frag.push_chunks(chunks)
        plan = r.plan()
        passed = r.frag.rows_passed
        out = r.result()
    finally:
        r.close()
    _check_plan(plan, {k: v for k, v in CASES[name].plan.items() if k != "final_pass"}, name)
    _check(c, out, passed, label=f"push_chunks {name}")


# -- refusals --
def _refuse(gpu, ctx, desc, build, pays):
    g = gpu.Join(ctx, desc)
    try:
        g.append_build(Chunk(build))
        g.build_finish()
        with pytest.raises(gpu.GpuError) as ei:
            f = gpu.Fragment(ctx, abi.ScanDesc(), [(g, 0, pays)], abi.make_agg_desc(fns=[STAR]), mode=2)
            f.close()
        return ei.value.code
    finally:
        g.close()


@pytest.mark.gpu
def test_refusals(gpu, ctx):
    keys = np.arange(100, dtype=np.int32)
    build = [(10, keys, None, INT), (11, keys.copy(), None, INT)]
    for jt in (abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
        assert _refuse(gpu, ctx, abi.make_join_desc(jt, [10], [0], [INT]), build, []) == abi.SR_ERR_NOT_SUPPORTED, jt
    for jt in (abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT_OUTER):
        conj = abi.make_join_desc(jt, [10], [0], [INT], other_conjunct=[("col", 11), ("col", 1), "<"])
        assert _refuse(gpu, ctx, conj, build, []) == abi.SR_ERR_NOT_SUPPORTED, ("conjunct", jt)
        multi = abi.make_join_desc(jt, [10, 11], [0, 1], [INT, INT])
        assert _refuse(gpu, ctx, multi, build, []) == abi.SR_ERR_NOT_SUPPORTED, ("two keys", jt)
    for jt in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
        assert _refuse(gpu, ctx, abi.make_join_desc(jt, [10], [0], [INT]), build, [11]) == abi.SR_ERR_INVALID_ARGUMENT, ("payload", jt)
    # a payload missing from a build side that has columns
    assert _refuse(gpu, ctx, abi.make_join_desc(abi.JOIN_LEFT_OUTER, [10], [0], [INT]), build, [12]) == abi.SR_ERR_INVALID_ARGUMENT
    # a build side that never received a chunk, with a payload whose type the descriptor does not declare
    g = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_LEFT_OUTER, [10], [0], [INT], build_out=[11]))
    try:
        g.build_finish()
        with pytest.raises(gpu.GpuError) as ei:
            gpu.Fragment(ctx, abi.ScanDesc(), [(g, 0, [11])], abi.make_agg_desc(fns=[STAR]), mode=2).close()
        assert ei.value.code == abi.SR_ERR_STATE and "build_out_types" in str(ei.value)
    finally:
        g.close()
