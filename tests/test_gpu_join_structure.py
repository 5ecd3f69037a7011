"""The per-operator hash join's structure against an exact pair-sequence reference: the chains a build produces, the open
addressing table of LINEAR_CHAINED where it wraps from its last slot to slot 0, the tile geometry of the two probe passes,
the ordered merge of the other-join conjunct, the POST_PROBE scan over the build rows and the gathered output columns.

test_gpu_join_edges.py covers the join's key domain; here the keys are ordinary and the shapes are not: chains longer
than a sort tile (up to ~300 000 rows of one key) whose duplicates arrive over many build chunks (empty ones, 1-row ones,
all-NULL ones), probe lengths at every residue of the 4-row thread group and around the 1024-row block with the key column
at each 4-byte device offset, conjuncts that keep all, none, only the first or only the last candidate of a probe row,
1 to 4 probers feeding the POST_PROBE marks, and payloads of every fixed width.

The reference is `ref_join` / `ref_conjunct` of test_gpu_join_edges.py (plain Python, checked against the oracle there)
and `np_join` below, its vectorised restatement for one integer key, which `test_np_join_is_ref_join` pins to it on the
CPU before it judges outputs of millions of pairs.  `ref_tables` restates the sequential build (`next[i] = first[b];
first[b] = i`) so that sr_join_copy_table can be compared exactly, and `join_key_hash64` / `join_key_unhash64` restate the
table's hash and its inverse so that keys can be placed on a chosen slot.  Tests that need the device are marked `gpu`.
"""
import collections
import functools

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk
from starrocks_b200.rows import col_to_py
from tests.test_gpu_join_edges import (DIRECT, JOIN_TYPES, JT_NAME, LINEAR, M64, PAIR_TYPES, POST_PROBE, RANGE, ref_conjunct,
                                       ref_join)
from tests.test_gpu_value_edges import I16, I32, I64, wrap

METHODS = (DIRECT, RANGE, LINEAR)
M_NAME = {DIRECT: "direct", RANGE: "range", LINEAR: "linear"}
B_KEY, B_ROW, B_TAG = 10, 20, 21          # build slots: key, 1-based row number (= build index), conjunct tag
P_KEY, P_KEY2, P_ROW, P_TAG = 0, 1, 5, 6  # probe slots
B_KEY2 = 11
RIGHT_ONLY = (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI)
SEMI = (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI)
OUTER = (abi.JOIN_LEFT_OUTER, abi.JOIN_FULL_OUTER)
PROBE_ROWS, PROBE_TILE, REMAIN_BLOCK, CONJ_BLOCK = 4, 1024, 256, 256   # sr_join.cuh: PROBE_ROWS, PROBE_TILE, REMAIN_BLOCK, k_conj_*
SCAN_ONE_LEVEL = 16 * 1024              # scan_counts (sr_scan.cuh) scans more block counts than this in two levels


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
HASH_MUL = 11400714819323198485         # join_key_hash64, csrc/sr_device.cuh


def join_key_hash64(v, log):
    """the home slot of 64-bit key v in a table of 2^log slots (JoinKeyHash<T, 8>)"""
    v &= M64
    v ^= v >> (64 - log)
    return ((v * HASH_MUL) & M64) >> (64 - log)


def join_key_unhash64(slot, log, low=0):
    """a key (signed 64-bit) whose home slot is `slot`: the multiply by the odd constant is undone by its inverse modulo
    2^64 (`low` picks the product's bits below the slot), the xorshift by applying it until it is a fixed point"""
    r = 64 - log
    x = ((((slot << r) | (low & ((1 << r) - 1))) & M64) * pow(HASH_MUL, -1, 1 << 64)) & M64
    v = x
    for _ in range(64 // r + 1):
        v = x ^ (v >> r)
    return wrap(v, 64)


def table_log(valid_rows):
    """log2 of LINEAR_CHAINED's slot count: the smallest power of two >= max(1024, 2 x non-NULL build rows)"""
    cap = 1024
    while cap < 2 * valid_rows:
        cap <<= 1
    return cap.bit_length() - 1


def ref_tables(build_keys, method, min_value=0):
    """the reference's sequential build over table keys in build order (None = NULL): `next[i] = first[b]; first[b] = i`
    with b = key - min_value for the range methods and b = the key itself for LINEAR_CHAINED (one key per slot, so its
    chain is the key's).  -> (first {bucket: head row}, next list of build_rows + 1)"""
    first, nxt = {}, [0] * (len(build_keys) + 1)
    for i, k in enumerate(build_keys, 1):
        if k is None:
            continue
        b = k if method == LINEAR else k - min_value
        nxt[i] = first.get(b, 0)
        first[b] = i
    return first, nxt


def linear_slots(build_keys, log):
    """slots of the distinct keys under sequential linear probing, INT64_MIN in the extra slot 2^log.  Which key of a
    cluster lands where depends on the arrival order; the SET of occupied slots does not."""
    cap, occ, slot = 1 << log, set(), {}
    for k in build_keys:
        if k is None or k in slot:
            continue
        if k == I64[0]:
            slot[k] = cap
            continue
        s = join_key_hash64(k, log)
        while s in occ:
            s = (s + 1) & (cap - 1)
        occ.add(s)
        slot[k] = s
    return slot


def np_join(bk, bn, pk, pn, jt):
    """ref_join for one integer key, vectorised.  bk / pk: int64 keys, bn / pn: bool NULL masks -> (pi, bi, remain)"""
    bk, pk = np.asarray(bk, dtype=np.int64), np.asarray(pk, dtype=np.int64)
    bidx = np.flatnonzero(~bn).astype(np.int64) + 1
    bkv = bk[bidx - 1]
    order = np.lexsort((-bidx, bkv))                         # by key, a key's rows by descending build index
    sk, sb = bkv[order], bidx[order]
    lo, hi = np.searchsorted(sk, pk, "left"), np.searchsorted(sk, pk, "right")
    cnt = np.where(pn, 0, hi - lo)
    if jt in (abi.JOIN_INNER, abi.JOIN_RIGHT_OUTER):
        emit = cnt
    elif jt in OUTER:
        emit = np.maximum(cnt, 1)
    elif jt == abi.JOIN_LEFT_SEMI:
        emit = (cnt > 0).astype(np.int64)
    elif jt == abi.JOIN_LEFT_ANTI:
        emit = (cnt == 0).astype(np.int64)
    else:
        emit = np.zeros(len(pk), dtype=np.int64)
    total = int(emit.sum())
    pi = np.repeat(np.arange(len(pk), dtype=np.int64), emit)
    off = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(emit) - emit, emit)
    has = np.repeat(cnt > 0, emit) & (jt in PAIR_TYPES)
    src = np.minimum(np.repeat(lo, emit) + off, max(len(sb) - 1, 0))
    bi = np.where(has, sb[src] if len(sb) else 0, 0)
    matched = np.zeros(len(bk) + 1, dtype=bool)
    matched[bidx[np.isin(bkv, pk[~pn])]] = True
    if jt == abi.JOIN_RIGHT_SEMI:
        remain = np.flatnonzero(matched[1:]) + 1
    elif jt in POST_PROBE:
        remain = np.flatnonzero(~matched[1:]) + 1
    else:
        remain = np.empty(0, dtype=np.int64)
    return pi.astype(np.uint32), bi.astype(np.uint32), remain.astype(np.uint32)


def ref_rows(jt, pairs, probe_vals, build_vals):
    """the output columns of the probe-phase pairs as Python values: probe_out (not for RIGHT SEMI / ANTI), then build_out
    (not for LEFT SEMI / ANTI), NULL where the build index is 0 or the source value is NULL"""
    cols = [] if jt in RIGHT_ONLY else [[v[i] for i, _ in pairs] for v in probe_vals]
    if jt not in SEMI:
        cols += [[v[b - 1] if b else None for _, b in pairs] for v in build_vals]
    return cols


def ref_remain_rows(jt, remain, n_probe_out, build_vals):
    """the POST_PROBE output columns: NULL probe_out columns (RIGHT / FULL OUTER), then build_out of the remain rows"""
    cols = [[None] * len(remain) for _ in range(n_probe_out)] if jt in (abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER) else []
    return cols + [[v[b - 1] for b in remain] for v in build_vals]


def _pairs(pi, bi):
    return list(zip(np.asarray(pi).tolist(), np.asarray(bi).tolist()))


# ---------------------------------------------------------------------------------------------------------------------
# the corpus: builds are (keys int64, NULL mask, chunk boundaries, key type, method); probes are (keys, NULL mask)
# ---------------------------------------------------------------------------------------------------------------------
KEY_TYPE = {DIRECT: abi.TYPE_SMALLINT, RANGE: abi.TYPE_INT, LINEAR: abi.TYPE_BIGINT}
CHAIN_LENGTHS = [1, 2, 31, 32, 33, 255, 256, 257, 65_535, 65_537, 300_001]
CHAIN_SINGLES = 300                     # keys with one build row besides the lengths above
CHAIN_SHAPES = ["one_chunk", "many_chunks"]
PROBE_SIZES = list(range(10)) + [1023, 1024, 1025, 4097, 4098, 4099]
TWO_LEVEL_N = (SCAN_ONE_LEVEL + 4) * PROBE_TILE + 3
GEOMETRY_LAYOUTS = ["host", "dev0", "dev4", "dev8", "dev12", "nullable", "packed"]
CONJ_COUNTS = [255, 256, 257, 3001]
CONJ_PATTERNS = ["all", "none", "first", "last", "mixed"]
REMAIN_SIZES = [255, 256, 257, 10 * REMAIN_BLOCK + 77]


class Build:
    def __init__(self, method, keys, nulls, cuts, label):
        self.method, self.keys, self.nulls, self.cuts, self.label = method, np.asarray(keys, dtype=np.int64), nulls, cuts, label
        self.ktype = KEY_TYPE[method]

    @property
    def n(self):
        return len(self.keys)

    @functools.cached_property
    def table_keys(self):
        return [None if nl else k for k, nl in zip(self.keys.tolist(), self.nulls.tolist())]

    @functools.cached_property
    def has_dup(self):
        v = self.keys[~self.nulls]
        return len(np.unique(v)) < len(v)

    def chunks(self, payload=()):
        """the build chunks; a chunk without NULL keys carries no NULL column (the join turns the key nullable later)"""
        out = []
        dt = abi.TYPE_NUMPY[self.ktype]
        for lo, hi in zip(self.cuts[:-1], self.cuts[1:]):
            nl = self.nulls[lo:hi]
            cols = [(B_KEY, self.keys[lo:hi].astype(dt), nl.astype(np.uint8) if nl.any() else None, self.ktype),
                    (B_ROW, np.arange(lo + 1, hi + 1, dtype=np.int32), None)]
            cols += [(s, d[lo:hi].copy(), None if m is None else m[lo:hi].copy(), t) for s, d, m, t in payload]
            out.append(Chunk(cols))
        return out

    def desc(self, jt, **kw):
        return abi.make_join_desc(jt, [B_KEY], [P_KEY], [self.ktype], enable_rdm=self.method != LINEAR, **kw)


def _domain(method, rng, n):
    """n distinct keys of the method's key type"""
    if method == DIRECT:
        pool = np.concatenate([[I16[0], I16[1], -1, 0], rng.choice(np.arange(I16[0] + 1, I16[1] - 1), n, replace=False)])
    elif method == RANGE:
        pool = np.concatenate([[I32[1] - 9999, I32[1]], I32[1] - 9998 + rng.choice(9998, n, replace=False)])
    else:
        pool = np.concatenate([[I64[1], -1, 0], rng.integers(I64[0] + 1, I64[1], n, dtype=np.int64)])
    return np.unique(pool)[rng.permutation(len(np.unique(pool)))][:n].astype(np.int64)


def _pieces(rng, n):
    """chunk boundaries over n rows: 1-row and empty chunks among chunks of 2..20 000 rows"""
    cuts, p = [0], 0
    while p < n:
        step = int(rng.choice([0, 1, 1, 3, 1000, 4096, 20_000]))
        p = min(n, p + step)
        cuts.append(p)
    return cuts + [n]


def _with_null_runs(rng, keys, nulls, cuts, runs=6):
    """insert all-NULL chunks (their key bytes copy real keys) at some chunk boundaries"""
    ks, ns, nc = [], [], [0]
    for c, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
        ks.append(keys[lo:hi])
        ns.append(nulls[lo:hi])
        nc.append(nc[-1] + hi - lo)
        if c % max(1, (len(cuts) - 1) // runs) == 0:
            m = int(rng.integers(1, 40))
            ks.append(keys[rng.integers(0, len(keys), m)])
            ns.append(np.ones(m, dtype=bool))
            nc.append(nc[-1] + m)
    return np.concatenate(ks), np.concatenate(ns), nc


@functools.lru_cache(maxsize=None)
def chain_build(method, shape):
    """one key per length of CHAIN_LENGTHS (INT64_MIN takes the 257 chain under LINEAR_CHAINED), CHAIN_SINGLES unique
    keys, 3 % NULL rows whose key bytes are real keys; rows shuffled so that each chain is spread over the build"""
    rng = np.random.default_rng(10 + METHODS.index(method))
    dom = _domain(method, rng, len(CHAIN_LENGTHS) + CHAIN_SINGLES + 50)
    chain_keys = dom[:len(CHAIN_LENGTHS)].copy()
    if method == LINEAR:
        chain_keys[CHAIN_LENGTHS.index(257)] = I64[0]
    lengths = CHAIN_LENGTHS + [1] * CHAIN_SINGLES
    keys = np.repeat(np.concatenate([chain_keys, dom[len(CHAIN_LENGTHS):len(lengths)]]), lengths)
    nulls = np.zeros(len(keys), dtype=bool)
    nn = len(keys) * 3 // 100
    keys = np.concatenate([keys, keys[rng.integers(0, len(keys), nn)]])
    nulls = np.concatenate([nulls, np.ones(nn, dtype=bool)])
    perm = rng.permutation(len(keys))
    keys, nulls = keys[perm], nulls[perm]
    if shape == "one_chunk":
        return Build(method, keys, nulls, [0, len(keys)], f"{M_NAME[method]}/{shape}")
    keys, nulls, cuts = _with_null_runs(rng, keys, nulls, _pieces(rng, len(keys)))
    return Build(method, keys, nulls, cuts, f"{M_NAME[method]}/{shape}")


@functools.lru_cache(maxsize=None)
def chain_probe(method):
    """every chain key: the three longest chains 3 / 2 / 2 times, the rest 1-4 times; absent keys and NULL rows"""
    rng = np.random.default_rng(20 + METHODS.index(method))
    b = chain_build(method, "one_chunk")
    cnt = collections.Counter(b.keys[~b.nulls].tolist())
    rows = []
    for k, c in cnt.items():
        rows += [k] * (3 if c > 100_000 else 2 if c > 60_000 else int(rng.integers(1, 5)))
    absent = _domain(method, np.random.default_rng(99), len(cnt) + 200)
    absent = [int(a) for a in absent if int(a) not in cnt][:150]
    rows += absent
    keys = np.array(rows, dtype=np.int64)[rng.permutation(len(rows))]
    nulls = rng.random(len(keys)) < 0.03
    return keys, nulls


@functools.lru_cache(maxsize=None)
def unique_build(method):
    rng = np.random.default_rng(30 + METHODS.index(method))
    keys = _domain(method, rng, 3000)
    nulls = rng.random(len(keys)) < 0.05
    keys, nulls, cuts = _with_null_runs(rng, keys, nulls, [0, 1, 1, 700, 701, 2000, 3000], runs=2)
    return Build(method, keys, nulls, cuts, f"{M_NAME[method]}/unique")


def unique_probe(method):
    rng = np.random.default_rng(40 + METHODS.index(method))
    b = unique_build(method)
    keys = np.concatenate([b.keys[rng.integers(0, b.n, 4000)], _domain(method, np.random.default_rng(41), 300)])
    return keys[rng.permutation(len(keys))], rng.random(len(keys)) < 0.04


@functools.lru_cache(maxsize=None)
def dup_in_last_chunk_build(method):
    """unique keys over ten chunks; the last chunk brings the first duplicate (of a key of the first chunk)"""
    rng = np.random.default_rng(50 + METHODS.index(method))
    keys = _domain(method, rng, 2000)
    keys = np.concatenate([keys, keys[[3, 3]], keys[-1:]])
    nulls = np.zeros(len(keys), dtype=bool)
    nulls[rng.integers(0, 2000, 40)] = True
    nulls[3] = False
    cuts = list(range(0, 2001, 200)) + [len(keys)]
    b = Build(method, keys, nulls, cuts, f"{M_NAME[method]}/dup_in_last_chunk")
    assert not Build(method, keys[:2000], nulls[:2000], [0, 2000], "").has_dup and b.has_dup
    return b


WRAP_LOG = 10


@functools.lru_cache(maxsize=None)
def wrap_case(dups):
    """BIGINT keys crafted for a 1024-slot LINEAR_CHAINED table: 16 keys homed on slots 1020..1023 and 0 whose cluster
    runs past the last slot into slot 0 and on, 200 keys homed in [100, 900); with `dups` the cluster keys repeat up to
    5 times.  Probe: every build key, absent keys homed inside the cluster and just after it, NULL rows."""
    rng = np.random.default_rng(60 + dups)
    homes = [1020] * 6 + [1022] * 3 + [1023] * 4 + [0] * 2 + [3]
    lows = rng.integers(0, 1 << 53, 400).tolist()
    cluster = [join_key_unhash64(h, WRAP_LOG, lows[i]) for i, h in enumerate(homes)]
    others = [join_key_unhash64(int(h), WRAP_LOG, lows[100 + i]) for i, h in enumerate(rng.integers(100, 900, 200))]
    reps = rng.integers(1, 6, len(cluster)) if dups else np.ones(len(cluster), dtype=np.int64)
    keys = np.concatenate([np.repeat(np.array(cluster, dtype=np.int64), reps), np.array(others, dtype=np.int64)])
    nulls = np.zeros(len(keys), dtype=bool)
    keys = np.concatenate([keys, keys[:20]])
    nulls = np.concatenate([nulls, np.ones(20, dtype=bool)])
    perm = rng.permutation(len(keys))
    keys, nulls = keys[perm], nulls[perm]
    b = Build(LINEAR, keys, nulls, [0, len(keys) // 2, len(keys)], f"wrap/{'dup' if dups else 'unique'}")
    slots = linear_slots(b.table_keys, WRAP_LOG)
    occ = set(slots.values())
    end = 0
    while end in occ:
        end += 1
    inside = [1021, 1023, 0, 2, end - 1]
    absent_in = [join_key_unhash64(h, WRAP_LOG, lows[300 + i]) for i, h in enumerate(inside)]
    absent_after = [join_key_unhash64(end, WRAP_LOG, lows[350 + i]) for i in range(3)]
    pk = np.array(cluster + others + absent_in + absent_after, dtype=np.int64)
    pk = np.concatenate([pk, pk[:5]])
    pn = np.zeros(len(pk), dtype=bool)
    pn[-5:] = True
    perm = rng.permutation(len(pk))
    return b, pk[perm], pn[perm], {"end": end, "absent_in": absent_in, "absent_after": absent_after, "homes": homes}


def geometry_build(packed):
    rng = np.random.default_rng(70 + packed)
    keys = I32[1] - 2999 + rng.integers(0, 2000, 3000)
    nulls = rng.random(3000) < 0.04
    return Build(RANGE, keys, nulls, [0, 1000, 3000], "geometry")


def geometry_probe(layout):
    rng = np.random.default_rng(80 + GEOMETRY_LAYOUTS.index(layout))
    n = max(PROBE_SIZES)
    k = (I32[1] - 3010 + rng.integers(0, 3011, n)).astype(np.int64)      # ~ half hit; out-of-range keys below the build
    k[rng.random(n) < 0.05] = I32[0]
    nulls = (rng.random(n) < 0.1) if layout == "nullable" else np.zeros(n, dtype=bool)
    k2 = rng.integers(-3, 3, n).astype(np.int64) if layout == "packed" else None
    return k, nulls, k2


def vec_keys(layout):
    """whether k_probe_count's 128-bit key load applies (sr_join.cuh join_probe: one non-nullable 4-byte key column, 16-byte
    aligned); host columns are staged into fresh device buffers"""
    return layout in ("host", "dev0")


def conj_case(count, pattern):
    """RANGE build of 600 keys with chains of 1..4 rows; a probe whose candidates (key matches) total exactly `count`,
    with rows without candidates before the first candidate, in runs between candidates and after the last.  The
    conjunct is B_TAG + P_TAG > 0: tags pick which candidates pass."""
    rng = np.random.default_rng(90 + CONJ_COUNTS.index(count) * 10 + CONJ_PATTERNS.index(pattern))
    bkeys = np.repeat(np.arange(600, dtype=np.int64), rng.integers(1, 5, 600))
    bkeys = bkeys[rng.permutation(len(bkeys))]
    bnulls = rng.random(len(bkeys)) < 0.03
    b = Build(RANGE, bkeys, bnulls, [0, len(bkeys) // 2, len(bkeys)], f"conj/{count}/{pattern}")
    chain = collections.Counter(bkeys[~bnulls].tolist())
    by_len = collections.defaultdict(list)
    for k, c in chain.items():
        by_len[c].append(k)
    pk, pn = [-5, -4, -3], [False, False, True]
    cand = 0
    while cand < count:
        left = count - cand
        ls = [L for L in by_len if L <= left]
        L = int(rng.choice(ls))
        pk.append(int(rng.choice(by_len[L])))
        pn.append(False)
        cand += L
        if rng.random() < 0.3:
            for _ in range(int(rng.integers(1, 4))):
                pk.append(int(rng.integers(700, 800)))
                pn.append(bool(rng.random() < 0.3))
    pk += [-1, 1000, 7]
    pn += [False, False, True]
    pk, pn = np.array(pk, dtype=np.int64), np.array(pn, dtype=bool)
    idx = np.arange(1, b.n + 1)
    if pattern == "all":
        btag, ptag = np.ones(b.n), np.zeros(len(pk))
    elif pattern == "none":
        btag, ptag = np.zeros(b.n), np.zeros(len(pk))
    elif pattern in ("first", "last"):
        btag = np.zeros(b.n)
        best = {}
        for i, k, nl in zip(idx.tolist(), bkeys.tolist(), bnulls.tolist()):
            if not nl and (k not in best or pattern == "first"):
                best[k] = i
        btag[np.array(list(best.values())) - 1] = 1
        ptag = np.zeros(len(pk))
    else:
        btag, ptag = rng.integers(0, 2, b.n), rng.integers(-1, 2, len(pk))
    return b, pk, pn, btag.astype(np.int32), ptag.astype(np.int32)


CONJ = [("col", B_TAG), ("col", P_TAG), "+", ("i", 0), ">"]


def conj_holds(btag, ptag):
    """the conjunct of (probe row i, build row b) through ref_expr"""
    return ref_conjunct(CONJ, {B_TAG: abi.TYPE_INT, P_TAG: abi.TYPE_INT}, {P_TAG: ptag.tolist()}, {B_TAG: btag.tolist()})


def remain_build(nb):
    """nb rows, keys in [0, nb // 2) with duplicates, 6 % NULL keys; key K_LAST = nb (rows 1 and nb) is probed only by
    the last probe"""
    rng = np.random.default_rng(100 + nb)
    keys = rng.integers(0, max(nb // 2, 1), nb).astype(np.int64)
    nulls = rng.random(nb) < 0.06
    keys[[0, nb - 1]] = nb
    nulls[[0, nb - 1]] = False
    return Build(RANGE, keys, nulls, [0, nb // 3, nb // 3, nb], f"remain/{nb}")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the reference's known answers, the hash against the oracle, ref_tables against the oracle, np_join against
# ref_join, and the corpus' coverage
# ---------------------------------------------------------------------------------------------------------------------
def test_reference_known_answers():
    first, nxt = ref_tables([5, 7, None, 5, 5, 7], RANGE, 5)
    assert first == {0: 5, 2: 6} and nxt == [0, 0, 0, 0, 1, 4, 2]
    first, nxt = ref_tables([I64[0], 3, I64[0]], LINEAR)
    assert first == {I64[0]: 3, 3: 2} and nxt == [0, 0, 0, 1]
    assert table_log(0) == 10 and table_log(512) == 10 and table_log(513) == 11 and table_log(1 << 20) == 21
    assert join_key_hash64(0, 10) == 0 and join_key_hash64(1, 64 - 54) == (HASH_MUL >> 54)
    for log in (10, 11, 17, 20, 31):
        for slot in (0, 1, (1 << log) - 1, (1 << log) // 3):
            for low in (0, 1, (1 << (64 - log)) - 1, 0x5A5A5A5A5A5A5):
                assert join_key_hash64(join_key_unhash64(slot, log, low), log) == slot
    bk, bn = np.array([4, 2, 4, 9, 4]), np.array([False, False, False, False, True])
    pk, pn = np.array([4, 3, 9, 2]), np.array([False, False, False, True])
    pi, bi, rem = np_join(bk, bn, pk, pn, abi.JOIN_LEFT_OUTER)
    assert _pairs(pi, bi) == [(0, 3), (0, 1), (1, 0), (2, 4), (3, 0)]
    assert np_join(bk, bn, pk, pn, abi.JOIN_RIGHT_ANTI)[2].tolist() == [2, 5]
    assert np_join(bk, bn, pk, pn, abi.JOIN_RIGHT_SEMI)[2].tolist() == [1, 3, 4]
    assert ref_rows(abi.JOIN_LEFT_OUTER, [(0, 3), (1, 0)], [[10, None]], [[1, 2, None]]) == [[10, None], [None, None]]
    assert ref_remain_rows(abi.JOIN_FULL_OUTER, [2], 1, [[1, 2, 3]]) == [[None], [2]]


def test_hash_matches_oracle(oracle):
    rng = np.random.default_rng(1)
    keys = [0, 1, -1, I64[0], I64[1]] + [int(v) for v in rng.integers(I64[0], I64[1], 300, dtype=np.int64)]
    for log in (10, 12, 20, 24, 31):
        for k in keys:
            assert join_key_hash64(k, log) == oracle.lib().orc_join_key_hash64(k & M64, log), (k, log)


def _small_builds():
    return [unique_build(m) for m in METHODS] + [dup_in_last_chunk_build(m) for m in METHODS] + \
           [wrap_case(d)[0] for d in (0, 1)] + [remain_build(n) for n in REMAIN_SIZES] + [conj_case(257, "mixed")[0]]


def test_ref_tables_match_oracle(oracle):
    # the oracle under the forced method: DIRECT / RANGE tables exactly; LINEAR_CHAINED (fingerprint-packed slots, a
    # quadratic probe) through its next[] and the set of chain heads
    for b in _small_builds() + [chain_build(DIRECT, "many_chunks")]:
        m = {DIRECT: oracle.DIRECT_MAPPING, RANGE: oracle.RANGE_DIRECT_MAPPING, LINEAR: oracle.LINEAR_CHAINED}[b.method]
        oj = oracle.Join(b.desc(abi.JOIN_INNER), force_method=m)
        for ch in b.chunks():
            oj.append_build(ch)
        oj.build()
        first, nxt = ref_tables(b.table_keys, b.method, oj.min_value)
        assert oj.next().tolist() == nxt, b.label
        if b.method == LINEAR:
            of = oj.first()
            assert sorted((of[of != 0] & 0xFFFFFF).tolist()) == sorted(first.values()), b.label
        else:
            dense = np.zeros(oj.bucket_size, dtype=np.uint32)
            dense[list(first)] = list(first.values())
            assert np.array_equal(oj.first(), dense), b.label


def test_np_join_is_ref_join():
    cases = [(b, b.keys[np.random.default_rng(3).integers(0, b.n, 3000)], np.random.default_rng(4).random(3000) < 0.05)
             for b in _small_builds()]
    b = chain_build(DIRECT, "one_chunk")
    small = Build(DIRECT, b.keys[:5000], b.nulls[:5000], [0, 5000], "")
    pk = np.concatenate([np.unique(small.keys), [I16[0] - 1, I16[1] + 1]])[::-1].copy()  # each key once: long chains
    cases.append((small, pk, np.arange(len(pk)) % 17 == 3))
    for b, pk, pn in cases:
        brows = [(k,) for k in b.table_keys]
        prows = [(None,) if nl else (k,) for k, nl in zip(pk.tolist(), pn.tolist())]
        for jt in JOIN_TYPES:
            pairs, remain = ref_join(brows, prows, jt)
            pi, bi, rem = np_join(b.keys, b.nulls, pk, pn, jt)
            assert _pairs(pi, bi) == pairs, (b.label, JT_NAME[jt])
            assert rem.tolist() == remain, (b.label, JT_NAME[jt])


def test_corpus_covers_the_structure():
    # every join type x method x (unique, duplicate) build keys
    seen = set()
    for m in METHODS:
        for b in [unique_build(m), dup_in_last_chunk_build(m)] + [chain_build(m, s) for s in CHAIN_SHAPES]:
            seen |= {(jt, b.method, b.has_dup) for jt in JOIN_TYPES}
    assert seen == {(jt, m, d) for jt in JOIN_TYPES for m in METHODS for d in (False, True)}
    # probe lengths: every residue mod 4 at 0..9, 1023..1025 and 4097..4099; one probe past the one-level scan
    for group in (range(10), range(1023, 1026), range(4097, 4100)):
        assert set(group) <= set(PROBE_SIZES)
    assert {n % PROBE_ROWS for n in range(10)} == set(range(PROBE_ROWS))
    assert (TWO_LEVEL_N + PROBE_TILE - 1) // PROBE_TILE > SCAN_ONE_LEVEL
    assert any(vec_keys(x) for x in GEOMETRY_LAYOUTS) and not all(vec_keys(x) for x in GEOMETRY_LAYOUTS)
    # chains: the lengths asked for, spread over many chunks with 1-row, empty and all-NULL chunks; INT64_MIN duplicates
    for m in METHODS:
        for s in CHAIN_SHAPES:
            b = chain_build(m, s)
            lengths = collections.Counter(collections.Counter(b.keys[~b.nulls].tolist()).values())
            assert set(CHAIN_LENGTHS) <= set(lengths) and max(lengths) >= 300_000, b.label
            if s == "many_chunks":
                sizes = np.diff(b.cuts)
                assert (sizes == 0).any() and (sizes == 1).any() and len(sizes) > 50
                assert any(b.nulls[lo:hi].all() for lo, hi in zip(b.cuts[:-1], b.cuts[1:]) if hi > lo)
        pk, pn = chain_probe(m)
        big = chain_build(m, "one_chunk").keys
        top = collections.Counter(big.tolist()).most_common(1)[0][0]
        assert 0 < ((pk == top) & ~pn).sum() <= 4                           # the 300 000-row chain, hit by few rows
    assert (chain_build(LINEAR, "one_chunk").keys == I64[0]).sum() >= 2
    # a cluster that wraps from the last slot to slot 0, with absent keys homed inside and just after it
    for d in (0, 1):
        b, pk, pn, info = wrap_case(d)
        assert table_log(int((~b.nulls).sum())) == WRAP_LOG
        slots = linear_slots(b.table_keys, WRAP_LOG)
        home = {k: join_key_hash64(k, WRAP_LOG) for k in slots}
        assert any(slots[k] < home[k] for k in slots), "no key wrapped past the last slot"
        occ = set(slots.values())
        assert {1020, 1021, 1022, 1023, 0} <= occ and info["end"] not in occ and info["end"] > 2
        assert all(join_key_hash64(k, WRAP_LOG) in occ for k in info["absent_in"])
        assert all(k not in slots for k in info["absent_in"] + info["absent_after"])
    # conjunct assembly: candidate counts at the 256-thread block edges, every pass pattern, stand-alone rows before the
    # first candidate, between candidates and after the last
    assert {255, 256, 257} <= set(CONJ_COUNTS) and max(CONJ_COUNTS) > 10 * CONJ_BLOCK
    for count in CONJ_COUNTS:
        for pattern in CONJ_PATTERNS:
            b, pk, pn, btag, ptag = conj_case(count, pattern)
            brows = [(k,) for k in b.table_keys]
            prows = [(None,) if nl else (k,) for k, nl in zip(pk.tolist(), pn.tolist())]
            cands, _ = ref_join(brows, prows, abi.JOIN_INNER)
            assert len(cands) == count
            kept = set(ref_join(brows, prows, abi.JOIN_INNER, conj_holds(btag, ptag))[0])
            cand_rows = [i for i, _ in cands]
            assert min(cand_rows) > 0 and max(cand_rows) < len(pk) - 1
            assert any(b2 - a > 1 for a, b2 in zip(cand_rows, cand_rows[1:])), "no run of rows without candidates"
            by_row = collections.defaultdict(list)
            for p in cands:
                by_row[p[0]].append(p)
            want = {"all": lambda ps: set(ps), "none": lambda ps: set(), "first": lambda ps: {ps[0]},
                    "last": lambda ps: {ps[-1]}}.get(pattern)
            if want:
                assert all(kept & set(ps) == want(ps) for ps in by_row.values()), pattern
            else:
                assert 0 < len(kept) < count and any(not (kept & set(ps)) for ps in by_row.values())
    # POST_PROBE: build sizes around one 256-row block and over ten blocks
    assert {255, 256, 257} <= set(REMAIN_SIZES) and max(REMAIN_SIZES) >= 10 * REMAIN_BLOCK


# ---------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------
def _raw(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), -1)


def check_cols(got, idx_sources, label):
    """got: chunk_out_to_host columns; idx_sources: per column (index array, data, nulls or None, build side).  A build
    column's index is 1-based with 0 = no row (NULL).  Null flags compared everywhere, data where not NULL."""
    assert len(got) == len(idx_sources), f"{label}: {len(got)} columns, want {len(idx_sources)}"
    for c, ((_, _, d, nl), (idx, src, snl, build)) in enumerate(zip(got, idx_sources)):
        idx = np.asarray(idx, dtype=np.int64)
        sn = np.zeros(len(src), dtype=bool) if snl is None else np.asarray(snl, dtype=bool)
        if build:
            src = np.concatenate([np.zeros(1, dtype=src.dtype), src])
            sn = np.concatenate([[True], sn])
        en = sn[idx] if len(idx) else np.zeros(0, dtype=bool)
        gn = np.zeros(len(d), dtype=bool) if nl is None else nl.astype(bool)
        assert len(d) == len(idx), f"{label}: column {c} has {len(d)} rows, want {len(idx)}"
        bad = np.flatnonzero(gn != en)
        assert not len(bad), f"{label}: column {c} row {bad[0]}: NULL flag {gn[bad[0]]}, want {en[bad[0]]}"
        if len(idx):
            diff = (_raw(d) != _raw(src)[idx]).any(axis=1) & ~en
            bad = np.flatnonzero(diff)
            assert not len(bad), f"{label}: column {c} row {bad[0]} differs ({len(bad)} rows)"


def check_pairs(pi, bi, epi, ebi, label):
    assert len(pi) == len(epi), f"{label}: {len(pi)} pairs, want {len(epi)}"
    bad = np.flatnonzero((pi != epi) | (bi != ebi))
    assert not len(bad), f"{label}: pair {bad[0]} is {(int(pi[bad[0]]), int(bi[bad[0]]))}, want {(int(epi[bad[0]]), int(ebi[bad[0]]))} ({len(bad)} differ)"


def _keycols(b):
    """the build's output columns B_ROW, B_KEY as (data, nulls) in build order"""
    return [(np.arange(1, b.n + 1, dtype=np.int32), None), (b.keys.astype(abi.TYPE_NUMPY[b.ktype]), b.nulls)]


def check_table(j, b, label):
    """sr_join_get_info and sr_join_copy_table against ref_tables"""
    info = j.info()
    assert info.method == b.method, f"{label}: method {info.method}"
    assert info.has_duplicates == int(b.has_dup), f"{label}: has_duplicates {info.has_duplicates}"
    assert info.build_rows == b.n, f"{label}: build_rows {info.build_rows}"
    first, nxt = j.copy_table()
    rfirst, rnext = ref_tables(b.table_keys, b.method, info.min_value)
    bad = np.flatnonzero(nxt != np.array(rnext, dtype=np.uint32))
    assert not len(bad), f"{label}: next[{bad[0]}] = {nxt[bad[0]]}, want {rnext[bad[0]]} ({len(bad)} differ)"
    if b.method != LINEAR:
        dense = np.zeros(info.bucket_size, dtype=np.uint32)
        dense[list(rfirst)] = list(rfirst.values())
        bad = np.flatnonzero(first != dense)
        assert not len(bad), f"{label}: first[{bad[0]}] = {first[bad[0]]}, want {dense[bad[0]]}"
        return
    # LINEAR_CHAINED: the chain reached from each occupied slot is a key's whole chain, every key has one slot, it sits
    # on its home slot or behind a run of occupied slots, and the occupied slots are those of sequential linear probing
    log = table_log(int((~b.nulls).sum()))
    cap = 1 << log
    assert info.bucket_size == cap + 1, f"{label}: {info.bucket_size} slots, want {cap + 1}"
    keys = b.keys.tolist()
    occ = set(np.flatnonzero(first[:cap]).tolist())
    want = linear_slots(b.table_keys, log)
    assert occ == {s for s in want.values() if s < cap}, f"{label}: occupied slots differ from linear probing"
    heads = {}
    for s in sorted(occ) + ([cap] if first[cap] else []):
        k = keys[int(first[s]) - 1]
        assert k not in heads, f"{label}: key {k} in slots {heads.get(k)} and {s}"
        heads[k] = s
        assert int(first[s]) == rfirst[k], f"{label}: slot {s} heads row {first[s]}, key {k}'s chain starts at {rfirst[k]}"
        if s == cap:
            assert k == I64[0], f"{label}: the extra slot holds {k}"
        else:
            h = join_key_hash64(k, log)
            assert all(((h + d) & (cap - 1)) in occ for d in range(((s - h) & (cap - 1)) + 1)), f"{label}: key {k} unreachable"
    assert set(heads) == set(rfirst), f"{label}: {len(heads)} keys in the table, want {len(rfirst)}"


def probe_chunk(pk, pn, ktype, extra=(), layout="host", pk2=None):
    """probe chunk: key P_KEY (and P_KEY2), row number P_ROW, extra (slot, data, nulls, type) columns"""
    import torch
    n = len(pk)
    dt = abi.TYPE_NUMPY[ktype]
    keys = pk.astype(dt)
    nl = pn.astype(np.uint8) if pn.any() or layout == "nullable" else None
    cols = [(P_KEY, keys, nl, ktype), (P_ROW, np.arange(n, dtype=np.int32), None, abi.TYPE_INT)]
    if pk2 is not None:
        cols.append((P_KEY2, pk2.astype(dt), None, ktype))
    cols += list(extra)
    if layout in ("host", "packed"):
        return Chunk(cols, num_rows=n)
    off = int(layout[3:]) if layout.startswith("dev") else 0
    dev = []
    for s, d, m, t in cols:
        raw = d.view(np.uint8)
        o = off if s == P_KEY else 0
        buf = torch.zeros(len(raw) + 64, dtype=torch.uint8, device="cuda")
        buf[o:o + len(raw)] = torch.from_numpy(raw.copy()).cuda()
        assert (buf.data_ptr() + o) % 16 == o
        mb = torch.from_numpy(m.copy()).cuda() if m is not None else None
        dev.append((s, buf[o:], mb, t))
    return Chunk(dev, num_rows=n, mem=abi.MEM_DEVICE)


def probe_and_check(gpu, ctx, j, b, jt, pk, pn, chunk, label, prober=0, table_keys=None):
    """probe, then the pair sequence and the P_ROW / B_ROW / B_KEY output columns against np_join.  table_keys: the
    (build, probe) keys np_join compares when they are not the key columns themselves (packed keys)"""
    out = j.probe(chunk, prober)
    n = out.num_rows
    got = gpu.chunk_out_to_host(ctx, out)
    pi, bi = j.probe_indexes(n, prober)
    bt, pt = table_keys or (b.keys, pk)
    epi, ebi, _ = np_join(bt, b.nulls, pt, pn, jt)
    check_pairs(pi, bi, epi, ebi, label)
    srcs = [] if jt in RIGHT_ONLY else [(epi, np.arange(len(pk), dtype=np.int32), None, False)]
    if jt not in SEMI:
        srcs += [(ebi, d, m, True) for d, m in _keycols(b)]
    check_cols(got, srcs, label)
    return len(pi)


def check_remain(gpu, ctx, j, b, jt, all_pk, all_pn, label, n_probe_out=1):
    got = gpu.chunk_out_to_host(ctx, j.probe_remain())
    _, _, erem = np_join(b.keys, b.nulls, all_pk, all_pn, jt)
    with_probe = jt in (abi.JOIN_RIGHT_OUTER, abi.JOIN_FULL_OUTER)
    srcs = [(np.zeros(len(erem), dtype=np.int64), np.zeros(1, dtype=np.int32), None, True)] * (n_probe_out if with_probe else 0)
    srcs += [(erem, d, m, True) for d, m in _keycols(b)]
    check_cols(got, srcs, f"{label}: POST_PROBE")


def _run(gpu, ctx, b, jt, probes, label, check_tab=True):
    """build b, check its table, probe each (pk, pn, chunk) on prober 0 and check, then POST_PROBE over all of them"""
    j = gpu.Join(ctx, b.desc(jt, build_out=[B_ROW, B_KEY], probe_out=[P_ROW]))
    try:
        for ch in b.chunks():
            j.append_build(ch)
        j.build_finish()
        if check_tab:
            check_table(j, b, label)
        total = 0
        for pk, pn, chunk, tag in probes:
            total += probe_and_check(gpu, ctx, j, b, jt, pk, pn, chunk, f"{label}/{tag}")
        if jt in POST_PROBE:
            all_pk = np.concatenate([p[0] for p in probes]) if probes else np.empty(0, dtype=np.int64)
            all_pn = np.concatenate([p[1] for p in probes]) if probes else np.empty(0, dtype=bool)
            check_remain(gpu, ctx, j, b, jt, all_pk, all_pn, label)
        return total
    finally:
        j.close()


@pytest.mark.gpu
def test_key_hash_matches_device(gpu, ctx):
    rng = np.random.default_rng(2)
    keys = np.concatenate([[0, 1, -1, I64[0], I64[1]], rng.integers(I64[0], I64[1], 5000, dtype=np.int64)]).astype(np.int64)
    crafted = np.array([join_key_unhash64(s, 10, int(lo)) for s, lo in zip(range(1024), rng.integers(0, 1 << 53, 1024))], dtype=np.int64)
    for log in (1, 10, 11, 16, 20, 24, 31):
        got = ctx.join_key_hash(keys, log)
        assert got.tolist() == [join_key_hash64(k, log) for k in keys.tolist()], log
    assert ctx.join_key_hash(crafted, 10).tolist() == list(range(1024))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", CHAIN_SHAPES + ["dup_in_last_chunk", "unique"])
@pytest.mark.parametrize("method", METHODS, ids=[M_NAME[m] for m in METHODS])
def test_chains(gpu, ctx, method, shape):
    # the relinked chains (descending build index) of every length in CHAIN_LENGTHS, the build appended as one chunk or
    # as many, and builds whose duplicates only arrive in the last chunk or never; every join type
    if shape in CHAIN_SHAPES:
        b, (pk, pn) = chain_build(method, shape), chain_probe(method)
    elif shape == "unique":
        b, (pk, pn) = unique_build(method), unique_probe(method)
    else:
        b = dup_in_last_chunk_build(method)
        pk = np.concatenate([b.keys[:2000:3], b.keys[[3, 2002]]])
        pn = np.zeros(len(pk), dtype=bool)
    chunk = probe_chunk(pk, pn, b.ktype)
    for jt in JOIN_TYPES:
        _run(gpu, ctx, b, jt, [(pk, pn, chunk, "probe")], f"{b.label}/{JT_NAME[jt]}")


@pytest.mark.gpu
@pytest.mark.parametrize("dups", [0, 1], ids=["unique", "dup"])
def test_linear_cluster_wraps_to_slot_zero(gpu, ctx, dups):
    b, pk, pn, _ = wrap_case(dups)
    chunk = probe_chunk(pk, pn, b.ktype)
    for jt in JOIN_TYPES:
        _run(gpu, ctx, b, jt, [(pk, pn, chunk, "probe")], f"{b.label}/{JT_NAME[jt]}")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", GEOMETRY_LAYOUTS)
def test_probe_tile_geometry(gpu, ctx, layout):
    # every probe length of PROBE_SIZES through one join per type (prober 0 re-used, so its buffers shrink and grow), the
    # key host-side, on the device at byte offsets 0 / 4 / 8 / 12, nullable, or packed from two columns
    packed = layout == "packed"
    b = geometry_build(packed)
    k, nulls, k2 = geometry_probe(layout)
    if packed:   # (INT key, INT key2) packs into 8 bytes: LINEAR_CHAINED over (key2 << 32) | key
        rng = np.random.default_rng(5)
        bk2 = rng.integers(-3, 3, b.n).astype(np.int64)
        table = (bk2 << 32) | (b.keys & 0xFFFFFFFF)
        pb = Build(LINEAR, table, b.nulls, b.cuts, "geometry/packed")
    for jt in JOIN_TYPES:
        label = f"{layout}/{JT_NAME[jt]}"
        if not packed:
            probes = [(k[:n], nulls[:n], probe_chunk(k[:n], nulls[:n], abi.TYPE_INT, layout=layout), f"n={n}") for n in PROBE_SIZES]
            _run(gpu, ctx, b, jt, probes, label)
            continue
        desc = abi.make_join_desc(jt, [B_KEY, B_KEY2], [P_KEY, P_KEY2], [abi.TYPE_INT, abi.TYPE_INT], build_out=[B_ROW, B_KEY],
                                  probe_out=[P_ROW])
        j = gpu.Join(ctx, desc)
        try:
            for lo, hi in zip(b.cuts[:-1], b.cuts[1:]):
                nl = b.nulls[lo:hi].astype(np.uint8)
                j.append_build(Chunk([(B_KEY, b.keys[lo:hi].astype(np.int32), nl), (B_KEY2, bk2[lo:hi].astype(np.int32), None),
                                      (B_ROW, np.arange(lo + 1, hi + 1, dtype=np.int32), None)]))
            j.build_finish()
            assert j.info().method == LINEAR and j.info().has_duplicates == int(pb.has_dup)
            ptable = (k2 << 32) | (k & 0xFFFFFFFF)
            for n in PROBE_SIZES:
                ch = probe_chunk(k[:n], nulls[:n], abi.TYPE_INT, layout=layout, pk2=k2[:n])
                probe_and_check(gpu, ctx, j, b, jt, k[:n], nulls[:n], ch, f"{label}/n={n}", table_keys=(table, ptable[:n]))
        finally:
            j.close()


@pytest.mark.gpu
def test_probe_past_the_one_level_scan(gpu, ctx):
    # more than 16 K probe blocks: scan_counts takes its two-level path; the key on the device, 128-bit loads.  Unique
    # build keys, so the reference is a lookup table: the probe row's build index or 0
    import torch
    rng = np.random.default_rng(6)
    span = 1 << 20
    keys = rng.permutation(span)[:700_000].astype(np.int32) - span // 2
    pos = np.zeros(span, dtype=np.uint32)
    pos[keys + span // 2] = np.arange(1, len(keys) + 1, dtype=np.uint32)
    pk = rng.integers(-span // 2, span // 2, TWO_LEVEL_N).astype(np.int32)
    hit = pos[pk + span // 2]
    dk = torch.from_numpy(pk).cuda()
    assert dk.data_ptr() % 16 == 0
    chunk = Chunk([(P_KEY, dk, None), (P_ROW, torch.arange(TWO_LEVEL_N, dtype=torch.int32, device="cuda"), None)], mem=abi.MEM_DEVICE)
    j = gpu.Join(ctx, abi.make_join_desc(abi.JOIN_INNER, [B_KEY], [P_KEY], [abi.TYPE_INT], build_out=[B_ROW], probe_out=[P_ROW]))
    try:
        j.append_build(Chunk([(B_KEY, keys, None), (B_ROW, np.arange(1, len(keys) + 1, dtype=np.int32), None)]))
        j.build_finish()
        assert j.info().method == RANGE and j.info().has_duplicates == 0
        out = j.probe(chunk)
        (_, _, prow, _), (_, _, brow, _) = gpu.chunk_out_to_host(ctx, out)
        pi, bi = j.probe_indexes(out.num_rows)
        epi = np.flatnonzero(hit).astype(np.uint32)
        check_pairs(pi, bi, epi, hit[epi], "two_level")
        assert np.array_equal(prow, epi.astype(np.int32)) and np.array_equal(brow, hit[epi].astype(np.int32))
    finally:
        j.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", CONJ_COUNTS)
def test_conjunct_assembly(gpu, ctx, count):
    # candidates (key matches) totalling `count`, every pass pattern, every join type: the merge of kept candidates and
    # stand-alone probe rows (k_conj_emit), and the POST_PROBE marks of passing pairs
    for pattern in CONJ_PATTERNS:
        b, pk, pn, btag, ptag = conj_case(count, pattern)
        brows = [(k,) for k in b.table_keys]
        prows = [(None,) if nl else (k,) for k, nl in zip(pk.tolist(), pn.tolist())]
        holds = conj_holds(btag, ptag)
        payload = [(B_TAG, btag, None, abi.TYPE_INT)]
        chunk = probe_chunk(pk, pn, b.ktype, extra=[(P_TAG, ptag, None, abi.TYPE_INT)])
        for jt in JOIN_TYPES:
            label = f"{count}/{pattern}/{JT_NAME[jt]}"
            pairs, remain = ref_join(brows, prows, jt, holds)
            j = gpu.Join(ctx, b.desc(jt, build_out=[B_ROW, B_TAG], probe_out=[P_ROW, P_TAG], other_conjunct=CONJ))
            try:
                for ch in b.chunks(payload):
                    j.append_build(ch)
                j.build_finish()
                out = j.probe(chunk)
                got = [col_to_py(t, d, nl) for _, t, d, nl in gpu.chunk_out_to_host(ctx, out)]
                pi, bi = j.probe_indexes(out.num_rows)
                assert _pairs(pi, bi) == pairs, f"{label}: pairs differ ({len(pi)} vs {len(pairs)})"
                bvals = [list(range(1, b.n + 1)), btag.tolist()]
                assert got == ref_rows(jt, pairs, [list(range(len(pk))), ptag.tolist()], bvals), f"{label}: output columns"
                if jt in POST_PROBE:
                    rem = [col_to_py(t, d, nl) for _, t, d, nl in gpu.chunk_out_to_host(ctx, j.probe_remain())]
                    assert rem == ref_remain_rows(jt, remain, 2, bvals), f"{label}: POST_PROBE rows"
            finally:
                j.close()


@pytest.mark.gpu
@pytest.mark.parametrize("probers", [1, 2, 3, 4])
@pytest.mark.parametrize("nb", REMAIN_SIZES)
def test_post_probe_over_probers(gpu, ctx, nb, probers):
    # probers take turns with changing batch sizes; with 3 or more, prober 1 only ever probes zero rows; key K_LAST is
    # only in the last batch of the last prober.  The POST_PROBE rows are those of the union of all batches.
    b = remain_build(nb)
    rng = np.random.default_rng(nb * 10 + probers)
    sizes = [0, 1, 5, 1023, 4099, 300, 2]
    for jt in POST_PROBE:
        label = f"{nb}/{probers}p/{JT_NAME[jt]}"
        j = gpu.Join(ctx, b.desc(jt, build_out=[B_ROW, B_KEY], probe_out=[P_ROW]))
        try:
            for ch in b.chunks():
                j.append_build(ch)
            j.build_finish()
            check_table(j, b, label)
            all_pk, all_pn, step = [], [], 0
            for rnd in range(3):
                for p in range(probers):
                    n = 0 if (probers >= 3 and p == 1) else sizes[step % len(sizes)]
                    step += 1
                    pk = rng.integers(0, max(nb // 8, 1) + 3, n).astype(np.int64)
                    pn = rng.random(n) < 0.05
                    if rnd == 2 and p == probers - 1:
                        pk = np.concatenate([pk, [nb]])
                        pn = np.concatenate([pn, [False]])
                    probe_and_check(gpu, ctx, j, b, jt, pk, pn, probe_chunk(pk, pn, b.ktype), f"{label}/round {rnd} prober {p}", prober=p)
                    all_pk.append(pk)
                    all_pn.append(pn)
            check_remain(gpu, ctx, j, b, jt, np.concatenate(all_pk), np.concatenate(all_pn), label)
        finally:
            j.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nb", REMAIN_SIZES)
def test_post_probe_without_a_probe(gpu, ctx, nb):
    # no probe at all: the probe_out types come from the desc; every build row (NULL keys too) is unmatched
    b = remain_build(nb)
    for jt in POST_PROBE:
        j = gpu.Join(ctx, b.desc(jt, build_out=[B_ROW, B_KEY], probe_out=[P_ROW], probe_out_types=[abi.TYPE_INT]))
        try:
            for ch in b.chunks():
                j.append_build(ch)
            j.build_finish()
            check_remain(gpu, ctx, j, b, jt, np.empty(0, dtype=np.int64), np.empty(0, dtype=bool), f"{nb}/{JT_NAME[jt]}")
        finally:
            j.close()


PAYLOAD_TYPES = [abi.TYPE_TINYINT, abi.TYPE_SMALLINT, abi.TYPE_INT, abi.TYPE_BIGINT, abi.TYPE_LARGEINT]


def _payload(rng, n, typ, nullable):
    if abi.TYPE_WIDTH[typ] == 16:
        d = rng.integers(0, 256, 16 * n, dtype=np.uint8).view(np.dtype((np.void, 16)))
    else:
        info = np.iinfo(abi.TYPE_NUMPY[typ])
        d = rng.integers(info.min, info.max, n, dtype=abi.TYPE_NUMPY[typ], endpoint=True)
    return d, ((rng.random(n) < 0.2).astype(np.uint8) if nullable else None)


@pytest.mark.gpu
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("jt", [abi.JOIN_LEFT_OUTER, abi.JOIN_FULL_OUTER, abi.JOIN_RIGHT_OUTER],
                         ids=[JT_NAME[t] for t in (abi.JOIN_LEFT_OUTER, abi.JOIN_FULL_OUTER, abi.JOIN_RIGHT_OUTER)])
def test_payload_widths(gpu, ctx, jt, mem):
    # build_out and probe_out columns of 1, 2, 4, 8 and 16 bytes, nullable and not, through the NULL padding of outer
    # rows (build index 0) and of POST_PROBE rows (probe columns NULL); on the device the 16-byte probe column sits 8
    # bytes off a 16-byte boundary
    import torch
    rng = np.random.default_rng(7 + jt)
    nb, npr = 1500, 2501
    bk = rng.integers(0, 900, nb).astype(np.int64)
    bn = rng.random(nb) < 0.05
    b = Build(RANGE, bk, bn, [0, 700, nb], "payload")
    pk = rng.integers(-50, 1000, npr).astype(np.int64)
    pn = rng.random(npr) < 0.05
    bpay = [(30 + 2 * c + nl, typ) + _payload(rng, nb, typ, nl) for c, typ in enumerate(PAYLOAD_TYPES) for nl in (0, 1)]
    ppay = [(50 + 2 * c + nl, typ) + _payload(rng, npr, typ, nl) for c, typ in enumerate(PAYLOAD_TYPES) for nl in (0, 1)]
    extra = [(s, d, m, t) for s, t, d, m in ppay]
    if mem == "host":
        chunk = probe_chunk(pk, pn, b.ktype, extra=extra)
    else:
        dev = [(P_KEY, torch.from_numpy(pk.astype(np.int32)).cuda(), torch.from_numpy(pn.astype(np.uint8)).cuda(), abi.TYPE_INT)]
        for s, d, m, t in extra:
            raw = d.view(np.uint8)
            o = 8 if abi.TYPE_WIDTH[t] == 16 else 0
            buf = torch.zeros(len(raw) + 32, dtype=torch.uint8, device="cuda")
            buf[o:o + len(raw)] = torch.from_numpy(raw.copy()).cuda()
            dev.append((s, buf[o:], torch.from_numpy(m).cuda() if m is not None else None, t))
        chunk = Chunk(dev, num_rows=npr, mem=abi.MEM_DEVICE)
    desc = b.desc(jt, build_out=[s for s, *_ in bpay], probe_out=[s for s, *_ in ppay])
    j = gpu.Join(ctx, desc)
    try:
        for ch in b.chunks([(s, d, m, t) for s, t, d, m in bpay]):
            j.append_build(ch)
        j.build_finish()
        out = j.probe(chunk)
        got = [col_to_py(t, d, nl) for _, t, d, nl in gpu.chunk_out_to_host(ctx, out)]
        pi, bi = j.probe_indexes(out.num_rows)
        pairs, remain = ref_join([(k,) for k in b.table_keys], [(None,) if x else (k,) for k, x in zip(pk.tolist(), pn.tolist())], jt)
        assert _pairs(pi, bi) == pairs
        pvals = [col_to_py(t, d, m) for _, t, d, m in ppay]
        bvals = [col_to_py(t, d, m) for _, t, d, m in bpay]
        exp = ref_rows(jt, pairs, pvals, bvals)
        for c, (g, e) in enumerate(zip(got, exp)):
            assert g == e, f"output column {c} (slot {out.cols[c].slot_id}) differs"
        assert len(got) == len(exp) == 20
        rem = [col_to_py(t, d, nl) for _, t, d, nl in gpu.chunk_out_to_host(ctx, j.probe_remain())] if jt in POST_PROBE else None
        if rem is not None:
            assert rem == ref_remain_rows(jt, remain, len(ppay), bvals), "POST_PROBE rows"
    finally:
        j.close()
