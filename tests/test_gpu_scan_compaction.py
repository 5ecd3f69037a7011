"""The scan's order-preserving compaction (sr_scan_filter: k_scan_mask -> k_scan_lvl1 / k_scan_counts -> k_scan_compact)
at every form its kernels take, against an exact row selection.

k_scan_compact picks its code path per batch, per tile and per column from facts no predicate test controls: how many
rows survive in the batch and in each 256-row tile, whether the tile is the ragged last one, each column's width and
address, and whether a tile lies past the first 1024 tiles of the two-level scan.  A wrong offset or staging index in
one of these forms drops, duplicates or reorders rows without any error.  Uniform random selections almost never reach
some of the forms (a dense tile in the direct kernel is ~6 standard deviations out at p = 1/8), while real scans are
clustered (sorted date ranges, keys loaded in order), so the selections here are built tile by tile.

The model below restates the dispatch rules; the CPU tests check it on hand-built masks and assert that this file's
case table reaches every form, and one GPU test ties the model to the kernels the device launched.  Every GPU case is
compared byte for byte with numpy: raw.reshape(-1, width)[mask] for data, nulls[mask] for null columns (the
reference's Chunk::filter, in row order), and the selection vector must equal the mask.
"""
import collections
import functools
import re

import numpy as np
import pytest

from starrocks_b200 import abi
from starrocks_b200.abi import Chunk

LANE_ROWS = 8                            # SCANW_ROWS: consecutive rows per lane (sr_scan.cuh:83)
TILE = 32 * LANE_ROWS                    # SCANW_TILE: one warp's rows
TILES_PER_BLOCK = 1024                   # k_scan_lvl1's block of tile counts: block_offsets[tile >> 10] (sr_scan.cuh:299)
BLOCK_ROWS = TILE * TILES_PER_BLOCK      # 262,144 rows

STAGED_KERNEL, DIRECT_KERNEL = "k_scan_compact<true>", "k_scan_compact<false>"
FAST_MASK, GENERIC_MASK = "k_scan_mask<true, false>", "k_scan_mask<false, false>"
COUNT_CLASSES = ("0", "1-31", "32-63", "64-256")


# =====================================================================================================================
# the model of the dispatch
# =====================================================================================================================
def count_class(c):
    return COUNT_CLASSES[0 if c == 0 else 1 if c < 32 else 2 if c < 64 else 3]


def compact_kernel(n, total):
    """sr_gpu.cu:440-448: no launch without survivors; the staged instantiation when at least 1/8 of the rows survive"""
    if n == 0 or total == 0:
        return None
    return STAGED_KERNEL if total * 8 >= n else DIRECT_KERNEL


def tile_form(kernel, tile_total, full):
    """k_scan_compact's form of one tile (sr_scan.cuh:297-302): dense = a quarter of the rows survive in a full tile;
    staged = the staged instantiation and at least 32 survivors.  "sparse direct" is every other non-empty tile."""
    if tile_total == 0:
        return "empty"                                                  # :297
    dense = tile_total >= TILE // 4 and full                            # :301
    if kernel == STAGED_KERNEL and tile_total >= 32:                    # :302
        return "staged dense" if dense else "staged"
    return "direct dense" if dense else "sparse direct"


def column_path(form, width, addr):
    """how k_scan_compact moves one column's values in a tile of `form`.  addr: the column's device address modulo 256
    (a host column's is its staging buffer's: 0); the output columns are always 256-byte aligned."""
    dense = form in ("staged dense", "direct dense")
    vec32 = width == 4 and dense and addr % 32 == 0                    # sr_scan.cuh:311 (`vec`), :334 (compact_rows_vec32)
    if form in ("staged", "staged dense") and width in (1, 4, 8):      # :310-319: widths 2 and 16 take the direct path
        return "staged vec32" if vec32 else "staged"
    if width == 16:
        return "int4" if addr % 16 == 0 else "words16"                  # sr_gpu.cu:435
    return "direct vec32" if vec32 else "direct"


Forms = collections.namedtuple("Forms", "mask_kernel lane_forms compact_kernel tiles columns blocks total")


def dispatch(mask, cols, ctl_nullable, ctl_addr):
    """the forms the kernels take for one sr_scan_filter call whose one conjunct is a range test on the control column.
    mask: bool per row; cols: [(width, nullable, data_addr, null_addr)], addresses modulo 256.
      mask_kernel   k_scan_mask<FAST, false>: a nullable control column in this batch downgrades FAST (sr_scan.cuh:546-549)
      lane_forms    per lane of k_scan_mask: "vec0" (FAST, control column 32-byte aligned (:550), all 8 rows inside the
                    batch (:118-126)); "predicated: misaligned" / "predicated: ragged lane" (FAST otherwise); "generic"
      tiles         {(kernel, form, full or ragged, survivor count class): tiles}
      columns       {(width, nullable, kernel, form, data path, null path or None)}
      blocks        the 1024-tile blocks of the tile scan that hold survivors"""
    n = len(mask)
    total = int(np.count_nonzero(mask))
    fast = not ctl_nullable
    vec0 = fast and ctl_addr % 32 == 0
    lane_forms = set()
    if n:
        if not fast:
            lane_forms.add("generic")
        else:
            if n >= LANE_ROWS:
                lane_forms.add("vec0" if vec0 else "predicated: misaligned")
            if n % LANE_ROWS:
                lane_forms.add("predicated: ragged lane")
    kernel = compact_kernel(n, total)
    ntiles = -(-n // TILE)
    padded = np.zeros(ntiles * TILE, dtype=bool)
    padded[:n] = mask
    counts = np.count_nonzero(padded.reshape(ntiles, TILE), axis=1)
    tiles, columns = collections.Counter(), set()
    if kernel is not None:
        for t, c in enumerate(counts.tolist()):
            full = (t + 1) * TILE <= n
            form = tile_form(kernel, c, full)
            tiles[(kernel, form, "full" if full else "ragged", count_class(c))] += 1
        for form in {k[1] for k in tiles} - {"empty"}:
            for width, nullable, addr, null_addr in cols:
                columns.add((width, nullable, kernel, form, column_path(form, width, addr),
                             column_path(form, 1, null_addr) if nullable else None))
    blocks = {int(b) for b in np.flatnonzero(counts) // TILES_PER_BLOCK}
    return Forms(FAST_MASK if fast else GENERIC_MASK, frozenset(lane_forms), kernel, tiles, columns, blocks, total)


def reachable_tiles():
    out = set()
    for kernel in (STAGED_KERNEL, DIRECT_KERNEL):
        for full in ("full", "ragged"):
            for c, cls in zip((0, 1, 32, 64), COUNT_CLASSES):
                out.add((kernel, tile_form(kernel, c, full == "full"), full, cls))
    return out


def reachable_columns(nullable):
    """every (width, nullable, kernel, form, data path, null path) a column at a 256-byte aligned address or one value
    into its allocation can take"""
    out = set()
    for kernel, forms in ((STAGED_KERNEL, ("sparse direct", "staged", "staged dense")), (DIRECT_KERNEL, ("sparse direct", "direct dense"))):
        for form in forms:
            for w in (1, 2, 4, 8, 16):
                for addr in (0, 8 if w == 16 else w):
                    out.add((w, nullable, kernel, form, column_path(form, w, addr), column_path(form, 1, 1) if nullable else None))
    return out


# =====================================================================================================================
# columns, selections and placements
# =====================================================================================================================
CTL_SLOT, ROWID_SLOT = 0, 31
PAYLOAD = [(1, abi.TYPE_BOOLEAN, False), (2, abi.TYPE_TINYINT, False), (3, abi.TYPE_SMALLINT, False), (4, abi.TYPE_INT, False),
           (5, abi.TYPE_BIGINT, False), (6, abi.TYPE_LARGEINT, False), (7, abi.TYPE_FLOAT, False), (8, abi.TYPE_DOUBLE, False),
           (9, abi.TYPE_DATE, False), (10, abi.TYPE_DATETIME, False), (11, abi.TYPE_DECIMAL32, False),
           (12, abi.TYPE_DECIMAL64, False), (13, abi.TYPE_DECIMAL128, False),
           (21, abi.TYPE_TINYINT, True), (22, abi.TYPE_SMALLINT, True), (23, abi.TYPE_FLOAT, True), (24, abi.TYPE_DATETIME, True),
           (25, abi.TYPE_LARGEINT, True), (ROWID_SLOT, abi.TYPE_INT, False)]
OUT_SLOTS = [s for s, _, _ in PAYLOAD]
assert len(OUT_SLOTS) <= abi.SR_MAX_OUT_COLS and {abi.TYPE_WIDTH[t] for _, t, nl in PAYLOAD if nl} == {1, 2, 4, 8, 16}
assert {t for _, t, _ in PAYLOAD} == set(abi.TYPE_WIDTH)

# +-0.0, +-inf, subnormals, NaNs of several payloads and signs: compaction moves bits, not values
FLOAT_BITS = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x7FC00000,
              0xFFC00000, 0x7F800001, 0x7FC00001, 0xFFBFFFFF, 0x7FFFFFFF, 0xFFFFFFFF]
DOUBLE_BITS = [0x0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x1, 0x8000000000000001, 0x000FFFFFFFFFFFFF,
               0x800FFFFFFFFFFFFF, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8000000000001,
               0x7FF4000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF]


@functools.lru_cache(maxsize=1)
def payload(n):
    """slot -> (data as n * width bytes, null bytes or None): random bytes, float columns with every third value an
    edge bit pattern, ~30% NULLs with garbage under them, and the INT row id"""
    rng = np.random.default_rng(1000 + n)
    cols = {}
    for slot, typ, nullable in PAYLOAD:
        w = abi.TYPE_WIDTH[typ]
        if slot == ROWID_SLOT:
            raw = np.arange(n, dtype=np.int32).view(np.uint8)
        else:
            raw = np.frombuffer(bytearray(rng.bytes(n * w)), dtype=np.uint8)
        if typ in (abi.TYPE_FLOAT, abi.TYPE_DOUBLE) and n:
            bits = np.array(FLOAT_BITS if w == 4 else DOUBLE_BITS, dtype=np.uint32 if w == 4 else np.uint64)
            v = raw.view(bits.dtype)
            v[::3] = np.resize(bits, len(v[::3]))
        nulls = (rng.random(n) < 0.3).astype(np.uint8) if nullable else None
        cols[slot] = (raw, nulls)
    return cols


COUNTS = (0, 1, 31, 32, 63, 64, 255, 256)
# per-tile survivor shapes: (shape, survivors); "lane 0" / "lane 31" keep rows of that lane only, "even lanes" the
# first rows of lanes 0, 2, 4, ..., "one lane" all of lane 17, "spread" evenly spaced rows
PATTERNS = ([("first", c) for c in COUNTS] + [("last", c) for c in COUNTS[1:]] +
            [("lane 0", 1), ("lane 0", 8), ("lane 31", 1), ("lane 31", 8), ("one lane", 8)] +
            [("even lanes", c) for c in (31, 32, 63, 64, 128)] + [("spread", c) for c in (31, 32, 63, 64, 255)])


def tile_rows(shape, count, rows=TILE):
    """the survivors of one tile of `rows` rows (fewer than TILE: the ragged last tile; shapes are clipped to it)"""
    m = np.zeros(TILE, dtype=bool)
    if shape == "first":
        m[:min(count, rows)] = True
    elif shape == "last":
        m[rows - min(count, rows):rows] = True
    elif shape == "lane 0":
        m[LANE_ROWS - count:LANE_ROWS] = True
    elif shape == "lane 31":
        m[TILE - LANE_ROWS:TILE - LANE_ROWS + count] = True
    elif shape == "one lane":
        m[17 * LANE_ROWS:18 * LANE_ROWS] = True
    elif shape == "even lanes":
        even = np.flatnonzero((np.arange(TILE) // LANE_ROWS) % 2 == 0)
        m[even[:count]] = True
    elif shape == "spread":
        m[(np.arange(count) * TILE) // count] = True
    else:
        raise ValueError(shape)
    return m[:rows]


def shaped(n, gap=0, at=None):
    """tile t takes PATTERNS[t // (gap + 1)] (cycled) when t % (gap + 1) == 0 and no survivors otherwise; `at`:
    {tile: (shape, count)} placed on purpose (a negative tile counts from the end)"""
    ntiles = -(-n // TILE)
    m = np.zeros(n, dtype=bool)
    fixed = {(t + ntiles if t < 0 else t): p for t, p in (at or {}).items()}
    for t in range(ntiles):
        rows = min(TILE, n - t * TILE)
        p = fixed.get(t)
        if p is None and t % (gap + 1) == 0:
            p = PATTERNS[(t // (gap + 1)) % len(PATTERNS)]
        if p is not None:
            m[t * TILE:t * TILE + rows] = tile_rows(*p, rows=rows)
    return m


def ranges(n, spans):
    m = np.zeros(n, dtype=bool)
    for lo, hi in spans:
        m[lo:hi] = True
    return m


def clustered(n):
    """survivors in a few clustered regions, ~3.5% of the rows: a sorted date range inside block 0, one across the
    tile 1023 / 1024 boundary, one in block 2, a short run, single rows every 4099, and the last rows of the batch"""
    m = ranges(n, [(1001, 41003), (BLOCK_ROWS - 2500, BLOCK_ROWS + 2501), (2 * BLOCK_ROWS + 3, 2 * BLOCK_ROWS + 100_003),
                   (3_000_000, 3_000_050), (n - 300, n)])
    m[::4099] = True
    return m


def first(n, k):
    return ranges(n, [(0, k)])


# survivors at the tile 1023 / 1024 boundary and in the last (ragged) tile, placed on purpose
EDGES_DENSE = {TILES_PER_BLOCK - 1: ("last", 256), TILES_PER_BLOCK: ("first", 256), -1: ("last", 255)}
EDGES_SPARSE = {TILES_PER_BLOCK - 1: ("last", 64), TILES_PER_BLOCK: ("lane 0", 1), -1: ("last", 64)}
EDGES_EMPTY_TAIL = {TILES_PER_BLOCK - 1: ("lane 31", 8), TILES_PER_BLOCK: ("first", 63), -1: ("first", 0)}

CASES = {
    "empty batch": (0, lambda n: np.zeros(0, dtype=bool)),
    "1 row kept": (1, lambda n: np.ones(n, dtype=bool)),
    "1 row dropped": (1, lambda n: np.zeros(n, dtype=bool)),
    "255 all": (255, lambda n: np.ones(n, dtype=bool)),
    "255 last 31": (255, lambda n: shaped(n, at={0: ("last", 31)})),
    "255 even lanes 64": (255, lambda n: shaped(n, at={0: ("even lanes", 64)})),
    "255 spread 32": (255, lambda n: shaped(n, at={0: ("spread", 32)})),
    "256 all": (256, lambda n: np.ones(n, dtype=bool)),
    "256 first 32 (total * 8 == n)": (256, lambda n: first(n, 32)),
    "256 first 31": (256, lambda n: first(n, 31)),
    "256 lane 31": (256, lambda n: shaped(n, at={0: ("lane 31", 8)})),
    "256 spread 64": (256, lambda n: shaped(n, at={0: ("spread", 64)})),
    "257 all": (257, lambda n: np.ones(n, dtype=bool)),
    "257 last 33": (257, lambda n: ranges(n, [(n - 33, n)])),
    "257 last 32": (257, lambda n: ranges(n, [(n - 32, n)])),
    "2048 one full tile (total * 8 == n)": (2048, lambda n: ranges(n, [(768, 1024)])),
    "2048 255 in one tile": (2048, lambda n: ranges(n, [(769, 1024)])),
    "2049 total 257 (ceil(n / 8))": (2049, lambda n: ranges(n, [(512, 768), (2048, 2049)])),
    "2049 total 256 (ceil(n / 8) - 1)": (2049, lambda n: ranges(n, [(513, 768), (2048, 2049)])),
    "262143 mixed": (262_143, lambda n: shaped(n, 0, EDGES_DENSE)),
    "262143 selective": (262_143, lambda n: shaped(n, 3, EDGES_SPARSE)),
    "262144 mixed": (262_144, lambda n: shaped(n, 0, EDGES_DENSE)),
    "262144 selective": (262_144, lambda n: shaped(n, 3, EDGES_EMPTY_TAIL)),
    "262145 mixed": (262_145, lambda n: shaped(n, 0, EDGES_EMPTY_TAIL)),
    "262145 selective": (262_145, lambda n: shaped(n, 3, EDGES_SPARSE)),
    "786509 mixed": (3 * BLOCK_ROWS + 77, lambda n: shaped(n, 0, EDGES_DENSE)),
    "786509 selective": (3 * BLOCK_ROWS + 77, lambda n: shaped(n, 3, {**EDGES_SPARSE, -1: ("first", 40)})),
    "786509 selective, empty tail": (3 * BLOCK_ROWS + 77, lambda n: shaped(n, 5, EDGES_EMPTY_TAIL)),
    "4195538 clustered": ((1 << 22) + 1234, clustered),
}


@functools.lru_cache(maxsize=4)
def case_mask(name):
    n, fn = CASES[name]
    m = fn(n)
    assert m.dtype == bool and len(m) == n
    return m


# placement -> (memory kind, data offset of a payload column of width w, null offset, control column offset).
# Host columns are staged into 256-byte aligned buffers; device columns are read in place at these offsets from a
# 256-byte aligned address.
PLACEMENTS = {
    "host": (abi.MEM_HOST, lambda w: 0, 0, 0),
    "device aligned": (abi.MEM_DEVICE, lambda w: 0, 0, 0),
    "device one value in": (abi.MEM_DEVICE, lambda w: 8 if w == 16 else w, 1, 4),
    "device control misaligned": (abi.MEM_DEVICE, lambda w: 0, 0, 4),
}
FORMS = {"fast": False, "generic": True}   # form -> the control column has a null column (with no NULL in it)


def column_addrs(placement, drop_nulls=False):
    """-> [(width, nullable, data_addr, null_addr)] of the output columns, and the control column's address (mod 256)"""
    _, off, noff, ctl = PLACEMENTS[placement]
    cols = [(abi.TYPE_WIDTH[t], nl and not drop_nulls, off(abi.TYPE_WIDTH[t]), noff) for _, t, nl in PAYLOAD]
    return cols, ctl


def model(name, placement, form, drop_nulls=False):
    cols, ctl = column_addrs(placement, drop_nulls)
    return dispatch(case_mask(name), cols, FORMS[form], ctl)


RUNS = [(c, p, f) for c in CASES for p in PLACEMENTS for f in FORMS]


# =====================================================================================================================
# CPU: the model on hand-built masks
# =====================================================================================================================
ALIGNED4, OFFSET4 = [(4, False, 0, 0)], [(4, False, 4, 0)]


def test_model_64_survivors_in_the_last_full_tile():
    n = 2 * TILE + 100
    f = dispatch(ranges(n, [(TILE, TILE + 64)]), ALIGNED4, False, 0)
    assert f.compact_kernel == DIRECT_KERNEL and f.total == 64
    assert f.tiles == {(DIRECT_KERNEL, "empty", "full", "0"): 1, (DIRECT_KERNEL, "direct dense", "full", "64-256"): 1,
                       (DIRECT_KERNEL, "empty", "ragged", "0"): 1}
    assert f.columns == {(4, False, DIRECT_KERNEL, "direct dense", "direct vec32", None)}
    assert dispatch(ranges(n, [(TILE, TILE + 64)]), OFFSET4, False, 0).columns == {(4, False, DIRECT_KERNEL, "direct dense", "direct", None)}
    # 63 survivors: not dense
    assert dispatch(ranges(n, [(TILE, TILE + 63)]), ALIGNED4, False, 0).columns == {(4, False, DIRECT_KERNEL, "sparse direct", "direct", None)}


def test_model_64_survivors_in_the_ragged_tail():
    n = 2 * TILE + 100
    f = dispatch(ranges(n, [(n - 64, n)]), ALIGNED4 + [(16, True, 0, 0)], False, 0)
    assert f.compact_kernel == DIRECT_KERNEL
    assert f.tiles[(DIRECT_KERNEL, "sparse direct", "ragged", "64-256")] == 1
    assert f.columns == {(4, False, DIRECT_KERNEL, "sparse direct", "direct", None),
                         (16, True, DIRECT_KERNEL, "sparse direct", "int4", "direct")}
    # the same rows with enough survivors elsewhere: the staged kernel stages the ragged tile, not densely
    g = dispatch(ranges(n, [(0, 2 * TILE - 200), (n - 64, n)]), ALIGNED4 + [(2, False, 0, 0)], False, 0)
    assert g.compact_kernel == STAGED_KERNEL
    assert g.tiles[(STAGED_KERNEL, "staged", "ragged", "64-256")] == 1
    assert (2, False, STAGED_KERNEL, "staged", "direct", None) in g.columns


@pytest.mark.parametrize("n", [256, 2048, 2049, 262_145])
def test_model_switches_kernels_at_an_eighth_of_the_rows(n):
    need = -(-n // 8)                                      # ceil(n / 8): the fewest survivors the staged kernel takes
    assert dispatch(first(n, need), ALIGNED4, False, 0).compact_kernel == STAGED_KERNEL
    assert dispatch(first(n, need - 1), ALIGNED4, False, 0).compact_kernel == DIRECT_KERNEL
    assert dispatch(first(n, 0), ALIGNED4, False, 0).compact_kernel is None


def test_model_tile_forms_at_32_and_64_survivors():
    n = 64 * TILE
    for c, want in ((31, "sparse direct"), (32, "staged"), (63, "staged"), (64, "staged dense")):
        m = np.zeros(n, dtype=bool)
        m[:n // 2] = True                                   # the staged kernel
        m[-TILE:] = tile_rows("spread", c)
        f = dispatch(m, [(16, False, 8, 0), (1, False, 1, 0), (8, True, 0, 0)], False, 0)
        assert f.tiles[(STAGED_KERNEL, want, "full", count_class(c))] == (33 if c == 64 else 1)   # + the 32 whole tiles
        staged = want.startswith("staged")
        assert (16, False, STAGED_KERNEL, want, "words16", None) in f.columns
        assert (1, False, STAGED_KERNEL, want, "staged" if staged else "direct", None) in f.columns
        assert (8, True, STAGED_KERNEL, want, "staged" if staged else "direct", "staged" if staged else "direct") in f.columns


def test_model_mask_forms():
    n = 3 * TILE
    m = first(n, 10)
    assert dispatch(m, ALIGNED4, False, 0).lane_forms == {"vec0"}
    assert dispatch(m, ALIGNED4, False, 4).lane_forms == {"predicated: misaligned"}
    assert dispatch(m, ALIGNED4, True, 0).lane_forms == {"generic"} and dispatch(m, ALIGNED4, True, 0).mask_kernel == GENERIC_MASK
    assert dispatch(first(n + 3, 10), ALIGNED4, False, 0).lane_forms == {"vec0", "predicated: ragged lane"}
    assert dispatch(first(7, 1), ALIGNED4, False, 0).lane_forms == {"predicated: ragged lane"}
    assert dispatch(first(0, 0), ALIGNED4, False, 0).lane_forms == frozenset()


def test_model_blocks_of_the_tile_scan():
    n = 3 * BLOCK_ROWS + 77
    assert dispatch(ranges(n, [(BLOCK_ROWS - 1, BLOCK_ROWS)]), ALIGNED4, False, 0).blocks == {0}
    assert dispatch(ranges(n, [(BLOCK_ROWS, BLOCK_ROWS + 1)]), ALIGNED4, False, 0).blocks == {1}
    assert dispatch(ranges(n, [(n - 1, n)]), ALIGNED4, False, 0).blocks == {3}


def test_patterns_have_their_survivor_counts():
    for shape, c in PATTERNS:
        m = tile_rows(shape, c)
        assert np.count_nonzero(m) == c, (shape, c)
        lanes = set(np.flatnonzero(m) // LANE_ROWS)
        if shape.startswith("lane"):
            assert lanes == {int(shape.split()[1])}
        if shape == "even lanes":
            assert all(ln % 2 == 0 for ln in lanes)
    assert np.count_nonzero(tile_rows("last", 64, rows=77)) == 64 and tile_rows("last", 64, rows=77)[-1]
    assert tile_rows("first", 255, rows=1).tolist() == [True]


# =====================================================================================================================
# CPU: the case table reaches every form
# =====================================================================================================================
def test_case_table_coverage():
    """asserts, over CASES x PLACEMENTS x FORMS:
      - both compaction instantiations, and both k_scan_mask forms without a runtime filter
      - per lane of k_scan_mask: vec0, predicated (misaligned control column), predicated (ragged lane), generic
      - per tile: every (instantiation, form, full / ragged tile, survivor class 0 / 1-31 / 32-63 / 64-256) there is
      - per column, for widths 1 / 2 / 4 / 8 / 16, nullable and not: every (instantiation, tile form, data path, null
        path) there is: staged or direct, vec32 or not, int4 or Words16
      - survivors in block 0 and in later blocks of the tile scan, and in tiles 1023 and 1024 of one batch in each
        instantiation
      - the switch at total * 8 == n taken both ways"""
    kernels, masks, lanes, tiles, columns, blocks = set(), set(), set(), set(), set(), set()
    for name, placement, form in RUNS:
        f = model(name, placement, form)
        kernels.add(f.compact_kernel)
        masks.add(f.mask_kernel)
        lanes |= f.lane_forms
        tiles |= set(f.tiles)
        columns |= f.columns
        blocks |= f.blocks
    assert kernels == {None, STAGED_KERNEL, DIRECT_KERNEL}
    assert masks == {FAST_MASK, GENERIC_MASK}
    assert lanes == {"vec0", "predicated: misaligned", "predicated: ragged lane", "generic"}
    assert tiles == reachable_tiles(), sorted(reachable_tiles() - tiles)
    for nullable in (False, True):
        want = reachable_columns(nullable)
        got = {c for c in columns if c[1] == nullable}
        assert got == want, f"nullable={nullable}: missing {sorted(want - got)}"
    assert {0, 1, 2, 3, 15} <= blocks
    boundary = [name for name in CASES if len(case_mask(name)) > BLOCK_ROWS
                and case_mask(name)[BLOCK_ROWS - TILE:BLOCK_ROWS].any() and case_mask(name)[BLOCK_ROWS:BLOCK_ROWS + TILE].any()]
    assert {model(name, "host", "fast").compact_kernel for name in boundary} == {STAGED_KERNEL, DIRECT_KERNEL}, boundary
    exact = [name for name in CASES if len(case_mask(name)) and np.count_nonzero(case_mask(name)) * 8 == len(case_mask(name))]
    below = [name for name in CASES if len(case_mask(name)) and np.count_nonzero(case_mask(name)) == -(-len(case_mask(name)) // 8) - 1]
    assert exact and below, (exact, below)


def reference(name, drop_nulls=False):
    """slot -> (expected data bytes, expected null bytes or None): numpy's row selection, in row order"""
    m = case_mask(name)
    out = {}
    for slot, typ, nullable in PAYLOAD:
        raw, nulls = payload(len(m))[slot]
        w = abi.TYPE_WIDTH[typ]
        out[slot] = (raw.reshape(-1, w)[m].tobytes(), nulls[m].tobytes() if nullable and not drop_nulls else None)
    return out


def control(m, generic):
    return (~m).astype(np.int32), (np.zeros(len(m), dtype=np.uint8) if generic else None)


def scan_desc():
    return abi.ScanDesc([abi.make_pred(CTL_SLOT, abi.PRED_EQ, 0)], out_slots=OUT_SLOTS)


def test_reference_agrees_with_the_oracle(oracle):
    # the numpy row selection the GPU tests assert against, and the oracle's Chunk::filter, on one small case each form
    for name in ("257 last 33", "262145 selective"):
        m = case_mask(name)
        n = len(m)
        want = reference(name)
        for generic in (False, True):
            ctl, ctl_nulls = control(m, generic)
            spec = [(CTL_SLOT, ctl, ctl_nulls)]
            for slot, typ, _ in PAYLOAD:
                raw, nulls = payload(n)[slot]
                spec.append((slot, raw.ctypes.data, nulls, typ))
            chunk = Chunk(spec, num_rows=n)
            assert np.array_equal(oracle.scan_evaluate(scan_desc(), chunk), m.astype(np.uint8))
            rows, got = oracle.scan_filter(scan_desc(), chunk)
            assert rows == np.count_nonzero(m)
            for slot, (data, nulls) in got.items():
                assert data.view(np.uint8).tobytes() == want[slot][0], f"{name}: slot {slot}"
                assert (None if nulls is None else nulls.tobytes()) == want[slot][1], f"{name}: slot {slot} nulls"


# =====================================================================================================================
# GPU: every case, placement and form, byte for byte
# =====================================================================================================================
class Batch:
    """the control column and the payload of case `name` as one chunk in `placement`; generic: the control column has a
    null column with no NULL in it (FAST downgrades to generic evaluation, the selection stays the same)"""

    def __init__(self, name, placement, generic, drop_nulls=False):
        m = case_mask(name)
        n = len(m)
        mem, off, noff, ctl_off = PLACEMENTS[placement]
        ctl, ctl_nulls = control(m, generic)
        cols = [(CTL_SLOT, abi.TYPE_INT, ctl.view(np.uint8), ctl_nulls, ctl_off, 0)]
        for slot, typ, nullable in PAYLOAD:
            raw, nulls = payload(n)[slot]
            cols.append((slot, typ, raw, None if drop_nulls else nulls, off(abi.TYPE_WIDTH[typ]), noff))
        self.keep = []
        spec = []
        if mem == abi.MEM_HOST:
            for slot, typ, raw, nulls, _, _ in cols:
                self.keep.append(raw)
                spec.append((slot, raw.ctypes.data, nulls, typ))
        else:
            spec = self._on_device(cols)
        self.chunk = Chunk(spec, num_rows=n, mem=mem)

    def _on_device(self, cols):
        import torch
        pieces, pos = [], 0
        for slot, typ, raw, nulls, off, noff in cols:
            for buf, o in ((raw, off), (nulls, noff)):
                if buf is None:
                    continue
                start = pos + o
                pieces.append((start, buf))
                pos = (start + len(buf) + 32 + 255) // 256 * 256
        image = np.zeros(max(pos, 256), dtype=np.uint8)
        for start, buf in pieces:
            image[start:start + len(buf)] = buf
        dev = torch.empty(len(image) + 256, dtype=torch.uint8, device="cuda")
        shift = -dev.data_ptr() % 256
        dev[shift:shift + len(image)].copy_(torch.from_numpy(image))
        self.keep.append(dev)
        base = dev.data_ptr() + shift
        spec, k = [], 0
        for slot, typ, raw, nulls, off, noff in cols:
            dp = base + pieces[k][0]
            k += 1
            np_ = None
            if nulls is not None:
                np_ = base + pieces[k][0]
                k += 1
            spec.append((slot, dp, np_, typ))
        return spec


def first_difference(got, want, w):
    g = np.frombuffer(got, dtype=np.uint8)
    e = np.frombuffer(want, dtype=np.uint8)
    k = min(len(g), len(e))
    bad = np.flatnonzero(g[:k] != e[:k])
    return f"{len(g) // w} rows vs {len(e) // w}, first difference at output row {int(bad[0]) // w if len(bad) else k // w}"


def check_selection(sel, m, label):
    bad = np.flatnonzero(sel != m.astype(np.uint8))
    assert len(bad) == 0, f"{label}: selection differs at {len(bad)} rows, first {int(bad[0])}: {int(sel[bad[0]])}"


def check_filter(gpu, ctx, out, name, label, drop_nulls=False):
    m = case_mask(name)
    want = reference(name, drop_nulls)
    got = gpu.chunk_out_to_host(ctx, out)
    assert out.num_rows == np.count_nonzero(m), label
    assert [g[0] for g in got] == OUT_SLOTS, label
    for (slot, typ, data, nulls), (_, t, _) in zip(got, PAYLOAD):
        w = abi.TYPE_WIDTH[t]
        assert typ == t, label
        raw = data.view(np.uint8).tobytes()
        assert raw == want[slot][0], f"{label}: slot {slot} (width {w}): {first_difference(raw, want[slot][0], w)}"
        if want[slot][1] is None:
            assert nulls is None, f"{label}: slot {slot} has a null column"
        else:
            assert nulls is not None and nulls.tobytes() == want[slot][1], \
                f"{label}: slot {slot} nulls: {first_difference(b'' if nulls is None else nulls.tobytes(), want[slot][1], 1)}"


@pytest.mark.gpu
@pytest.mark.parametrize("name,placement,form", RUNS, ids=[f"{c}-{p}-{f}".replace(" ", "_") for c, p, f in RUNS])
def test_compaction_matches_row_selection(gpu, ctx, name, placement, form):
    b = Batch(name, placement, FORMS[form])
    label = f"{name} / {placement} / {form}"
    sc = gpu.Scan(ctx, scan_desc())
    try:
        check_selection(sc.evaluate(b.chunk), case_mask(name), label)
        check_filter(gpu, ctx, sc.filter(b.chunk), name, label)
    finally:
        sc.close()


# =====================================================================================================================
# GPU: one handle across batches that change size, form, memory kind and alignment
# =====================================================================================================================
# (case, placement, form, calls, payload without null columns): sizes grow and shrink across the 262,144-row block
# boundary with empty batches in between; FAST, then generic, then FAST again; every memory kind and alignment
SEQUENCE = [
    ("786509 mixed", "host", "fast", "filter", False),
    ("257 last 33", "device one value in", "generic", "evaluate filter", False),
    ("empty batch", "host", "fast", "filter evaluate", False),
    ("262145 selective", "device control misaligned", "fast", "filter", True),
    ("1 row kept", "device aligned", "generic", "filter", False),
    ("262144 mixed", "device one value in", "generic", "evaluate", False),
    ("262143 selective", "host", "fast", "filter evaluate filter", False),
    ("empty batch", "device aligned", "generic", "filter", True),
    ("2049 total 256 (ceil(n / 8) - 1)", "device aligned", "fast", "filter", False),
    ("786509 selective, empty tail", "device one value in", "fast", "evaluate filter", True),
    ("256 lane 31", "host", "generic", "filter", False),
    ("262145 mixed", "device aligned", "fast", "filter", False),
    ("255 all", "device control misaligned", "fast", "evaluate filter", False),
]


@pytest.mark.gpu
def test_one_handle_across_changing_batches(gpu, ctx):
    # the grow-only scratch (mask_bits, tile_counts, local_excl, block_offsets, the selection bytes and the output column
    # set) must carry nothing stale into a smaller or differently shaped batch; each output is read before the next call
    sc = gpu.Scan(ctx, scan_desc())
    try:
        for step, (name, placement, form, calls, drop_nulls) in enumerate(SEQUENCE):
            b = Batch(name, placement, FORMS[form], drop_nulls)
            label = f"step {step}: {name} / {placement} / {form}"
            for call in calls.split():
                if call == "evaluate":
                    check_selection(sc.evaluate(b.chunk), case_mask(name), label)
                else:
                    check_filter(gpu, ctx, sc.filter(b.chunk), name, label, drop_nulls)
    finally:
        sc.close()


# =====================================================================================================================
# GPU: the model against the kernels the device launched
# =====================================================================================================================
PROFILED = [("256 first 32 (total * 8 == n)", "host", "fast"), ("256 first 31", "device aligned", "fast"),
            ("256 first 32 (total * 8 == n)", "device one value in", "generic"), ("2049 total 256 (ceil(n / 8) - 1)", "host", "generic"),
            ("1 row dropped", "host", "fast"), ("262145 selective", "device control misaligned", "fast"),
            ("262145 mixed", "host", "generic")]
DEMANGLED = re.compile(r"k_scan_(mask|compact)<([^>]*)>")
MANGLED = re.compile(r"k_scan_(mask|compact)I((?:Lb[01]E)+)E")


def scan_kernel_name(name):
    """the k_scan_mask / k_scan_compact instantiation a profiler event names (demangled or mangled), else None"""
    d = DEMANGLED.search(name)
    if d:
        return f"k_scan_{d.group(1)}<{', '.join(a.strip() for a in d.group(2).split(','))}>"
    mg = MANGLED.search(name)
    if mg:
        args = ["true" if b == "1" else "false" for b in re.findall(r"Lb([01])E", mg.group(2))]
        return f"k_scan_{mg.group(1)}<{', '.join(args)}>"
    return None


def test_scan_kernel_names_parse():
    assert scan_kernel_name("void srd::k_scan_compact<true>(unsigned char const*, unsigned int const*)") == STAGED_KERNEL
    assert scan_kernel_name("void srd::k_scan_mask<false, false>(srd::ScanProg const*, srd::ScanTests)") == GENERIC_MASK
    assert scan_kernel_name("_ZN3srd11k_scan_maskILb1ELb0EEEvPKNS_8ScanProgE") == FAST_MASK
    assert scan_kernel_name("_ZN3srd14k_scan_compactILb0EEEvPKhPKjPKmNS_11CompactArgsEl") == DIRECT_KERNEL
    assert scan_kernel_name("void srd::k_scan_lvl1<false>(unsigned int const*, long)") is None


PROFILED_CALLS = 3


@pytest.mark.gpu
def test_model_predicts_the_launched_kernels(gpu, ctx):
    # A trace has been seen to miss the first launch of its window, so the window opens with a kernel of its own, each batch is
    # filtered PROFILED_CALLS times, and the instantiations the trace holds are compared with the model's as a set.
    import torch
    from torch.profiler import ProfilerActivity, profile

    seen = set()
    for name, placement, form in PROFILED:
        b = Batch(name, placement, FORMS[form])
        f = model(name, placement, form)
        sc = gpu.Scan(ctx, scan_desc())
        try:
            sc.evaluate(b.chunk)   # compiles the scan outside the profiled window
            ctx.sync()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                torch.ones(1, device="cuda").add_(1)
                torch.cuda.synchronize()
                for _ in range(PROFILED_CALLS):
                    out = sc.filter(b.chunk)
                ctx.sync()
            check_filter(gpu, ctx, out, name, name)
        finally:
            sc.close()
        kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        scan_kernels = [k for k in kernels if "k_scan" in k]
        assert scan_kernels, f"{name}: the profile holds no k_scan kernel event (CUDA events: {kernels})"
        launched = collections.Counter(k for k in map(scan_kernel_name, scan_kernels) if k is not None)
        predicted = {f.mask_kernel} | ({f.compact_kernel} if f.compact_kernel else set())
        assert set(launched) == predicted and max(launched.values()) <= PROFILED_CALLS, \
            f"{name} / {placement} / {form}: launched {dict(launched)}, the model predicts {sorted(predicted)}"
        seen |= set(launched)
    assert seen == {FAST_MASK, GENERIC_MASK, STAGED_KERNEL, DIRECT_KERNEL}
