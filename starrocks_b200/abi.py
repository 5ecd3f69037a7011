"""ctypes mirror of include/sr_gpu_ops.h (struct layouts + small builders).

Pure declarations: importing this module loads no native library.  Both the product binding
(starrocks_b200/gpu.py -> libsr_gpu.so) and the test-only oracle binding (oracle/oracle.py)
use these definitions so that the same descriptors drive both implementations.
"""
import ctypes as C

import numpy as np

SR_ABI_VERSION = 1

# sr_status
SR_OK = 0
SR_ERR_INVALID_ARGUMENT = -1
SR_ERR_NOT_SUPPORTED = -2
SR_ERR_OUT_OF_MEMORY = -3
SR_ERR_CUDA = -4
SR_ERR_STATE = -5
SR_ERR_NO_DEVICE = -6

# sr_type (be/src/types/logical_type.h subset)
TYPE_BOOLEAN, TYPE_TINYINT, TYPE_SMALLINT, TYPE_INT, TYPE_BIGINT, TYPE_LARGEINT = 1, 2, 3, 4, 5, 6
TYPE_FLOAT, TYPE_DOUBLE, TYPE_DATE, TYPE_DATETIME = 7, 8, 9, 10
TYPE_DECIMAL32, TYPE_DECIMAL64, TYPE_DECIMAL128 = 11, 12, 13

TYPE_WIDTH = {
    TYPE_BOOLEAN: 1, TYPE_TINYINT: 1, TYPE_SMALLINT: 2, TYPE_INT: 4, TYPE_BIGINT: 8, TYPE_LARGEINT: 16,
    TYPE_FLOAT: 4, TYPE_DOUBLE: 8, TYPE_DATE: 4, TYPE_DATETIME: 8, TYPE_DECIMAL32: 4, TYPE_DECIMAL64: 8,
    TYPE_DECIMAL128: 16,
}
TYPE_NUMPY = {
    TYPE_BOOLEAN: np.uint8, TYPE_TINYINT: np.int8, TYPE_SMALLINT: np.int16, TYPE_INT: np.int32,
    TYPE_BIGINT: np.int64, TYPE_FLOAT: np.float32, TYPE_DOUBLE: np.float64, TYPE_DATE: np.int32,
    TYPE_DATETIME: np.int64, TYPE_DECIMAL32: np.int32, TYPE_DECIMAL64: np.int64,
}
NUMPY_TYPE = {
    np.dtype(np.uint8): TYPE_BOOLEAN, np.dtype(np.int8): TYPE_TINYINT, np.dtype(np.int16): TYPE_SMALLINT,
    np.dtype(np.int32): TYPE_INT, np.dtype(np.int64): TYPE_BIGINT, np.dtype(np.float32): TYPE_FLOAT,
    np.dtype(np.float64): TYPE_DOUBLE,
}

MEM_HOST, MEM_DEVICE, MEM_HOST_PINNED = 0, 1, 2

# sr_pred_op
PRED_EQ, PRED_NE, PRED_LT, PRED_LE, PRED_GT, PRED_GE, PRED_BETWEEN, PRED_IN, PRED_NOT_IN = 1, 2, 3, 4, 5, 6, 7, 8, 9
PRED_IS_NULL, PRED_IS_NOT_NULL = 10, 11

# sr_expr_op
EX_COL, EX_ICONST, EX_DCONST, EX_ADD, EX_SUB, EX_MUL, EX_TO_DOUBLE = 1, 2, 3, 4, 5, 6, 7
EX_EQ, EX_NE, EX_LT, EX_LE, EX_GT, EX_GE, EX_AND, EX_OR, EX_NOT, EX_IS_NULL, EX_DIV = 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18

JOIN_INNER, JOIN_LEFT_OUTER, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI = 0, 1, 2, 3
JOIN_RIGHT_OUTER, JOIN_RIGHT_SEMI, JOIN_RIGHT_ANTI, JOIN_FULL_OUTER = 4, 5, 6, 7
JOIN_METHOD_NONE, JOIN_METHOD_DIRECT_MAPPING, JOIN_METHOD_RANGE_DIRECT_MAPPING, JOIN_METHOD_LINEAR_CHAINED = 0, 1, 2, 3

AGG_SUM, AGG_COUNT, AGG_COUNT_STAR, AGG_AVG, AGG_MIN, AGG_MAX, AGG_AVG_MERGE, AGG_COUNT_DISTINCT = 1, 2, 3, 4, 5, 6, 7, 8

HASH_FNV, HASH_CRC32, HASH_XXH3 = 0, 1, 2
REDUCE_MULHI, REDUCE_MODULO = 0, 1

SR_MAX_OUT_COLS = 32
SR_MAX_IN_LIST = 16
SR_MAX_EXPR_NODES = 24
SR_MAX_JOIN_KEYS = 4
SR_MAX_JOIN_OUT = 16
SR_MAX_GROUP_KEYS = 4
SR_MAX_AGG_FNS = 8
SR_MAX_FRAG_JOINS = 6
SR_MAX_FRAG_PAYLOAD = 2
SR_MAX_PART_KEYS = 4


class sr_col_view(C.Structure):
    _fields_ = [("data", C.c_void_p), ("nulls", C.c_void_p), ("type", C.c_int32), ("slot_id", C.c_int32)]


class sr_chunk_view(C.Structure):
    _fields_ = [("cols", C.POINTER(sr_col_view)), ("num_cols", C.c_int32), ("mem", C.c_int32),
                ("num_rows", C.c_int64)]


class sr_col_out(C.Structure):
    _fields_ = [("data", C.c_void_p), ("nulls", C.c_void_p), ("type", C.c_int32), ("slot_id", C.c_int32)]


class sr_chunk_out(C.Structure):
    _fields_ = [("cols", sr_col_out * SR_MAX_OUT_COLS), ("num_cols", C.c_int32), ("mem", C.c_int32),
                ("num_rows", C.c_int64)]


class sr_pred(C.Structure):
    _fields_ = [("slot_id", C.c_int32), ("op", C.c_int32), ("ilo", C.c_int64), ("ihi", C.c_int64),
                ("dlo", C.c_double), ("dhi", C.c_double), ("in_list", C.c_int64 * SR_MAX_IN_LIST),
                ("in_count", C.c_int32), ("reserved", C.c_int32)]


class sr_expr_node(C.Structure):
    _fields_ = [("op", C.c_int32), ("slot_id", C.c_int32), ("ival", C.c_int64), ("dval", C.c_double)]


class sr_expr(C.Structure):
    _fields_ = [("nodes", sr_expr_node * SR_MAX_EXPR_NODES), ("num_nodes", C.c_int32), ("reserved", C.c_int32)]


class sr_scan_desc(C.Structure):
    _fields_ = [("preds", C.POINTER(sr_pred)), ("num_preds", C.c_int32), ("num_filter_exprs", C.c_int32),
                ("filter_exprs", C.POINTER(sr_expr)), ("out_slots", C.POINTER(C.c_int32)),
                ("num_out_slots", C.c_int32), ("reserved", C.c_int32)]


class sr_join_desc(C.Structure):
    _fields_ = [("join_type", C.c_int32), ("num_keys", C.c_int32),
                ("build_key_slots", C.c_int32 * SR_MAX_JOIN_KEYS), ("probe_key_slots", C.c_int32 * SR_MAX_JOIN_KEYS),
                ("key_types", C.c_int32 * SR_MAX_JOIN_KEYS),
                ("num_build_out", C.c_int32), ("build_out_slots", C.c_int32 * SR_MAX_JOIN_OUT),
                ("num_probe_out", C.c_int32), ("probe_out_slots", C.c_int32 * SR_MAX_JOIN_OUT),
                ("enable_range_direct_mapping", C.c_int32), ("reserved", C.c_int32),
                ("build_out_types", C.c_int32 * SR_MAX_JOIN_OUT), ("probe_out_types", C.c_int32 * SR_MAX_JOIN_OUT),
                ("other_conjunct", sr_expr)]


PAGE_PLAIN, PAGE_FOR, PAGE_BITSHUFFLE, PAGE_DICT, PAGE_RLE = 0, 1, 2, 3, 4
NULL_BITSHUFFLE, NULL_RLE = 0, 1


class sr_page_view(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size", C.c_int64)]


class sr_null_map_view(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size", C.c_int64), ("num_rows", C.c_int64)]


class sr_chunk_pb_meta(C.Structure):
    _fields_ = [("serialized_size", C.c_int64), ("num_rows", C.c_int64), ("num_cols", C.c_int32), ("reserved", C.c_int32),
                ("slot_ids", C.c_int32 * SR_MAX_OUT_COLS), ("types", C.c_int32 * SR_MAX_OUT_COLS),
                ("is_nulls", C.c_uint8 * SR_MAX_OUT_COLS), ("is_consts", C.c_uint8 * SR_MAX_OUT_COLS)]


class sr_join_info(C.Structure):
    _fields_ = [("method", C.c_int32), ("has_duplicates", C.c_int32), ("build_rows", C.c_int64),
                ("bucket_size", C.c_int64), ("min_value", C.c_int64), ("max_value", C.c_int64)]


class sr_agg_fn(C.Structure):
    _fields_ = [("kind", C.c_int32), ("input_type", C.c_int32), ("out_slot", C.c_int32), ("reserved", C.c_int32),
                ("input", sr_expr)]


class sr_agg_desc(C.Structure):
    _fields_ = [("num_group_keys", C.c_int32), ("group_slots", C.c_int32 * SR_MAX_GROUP_KEYS),
                ("group_types", C.c_int32 * SR_MAX_GROUP_KEYS), ("has_ranges", C.c_int32),
                ("group_nullable", C.c_int32 * SR_MAX_GROUP_KEYS),
                ("group_min", C.c_int64 * SR_MAX_GROUP_KEYS), ("group_max", C.c_int64 * SR_MAX_GROUP_KEYS),
                ("num_fns", C.c_int32), ("reserved", C.c_int32), ("fns", sr_agg_fn * SR_MAX_AGG_FNS),
                ("expected_groups", C.c_int64)]


class sr_frag_join(C.Structure):
    _fields_ = [("join", C.c_void_p), ("probe_key_slot", C.c_int32), ("num_payload", C.c_int32),
                ("payload_build_slots", C.c_int32 * SR_MAX_FRAG_PAYLOAD)]


class sr_fragment_desc(C.Structure):
    _fields_ = [("scan", sr_scan_desc), ("num_joins", C.c_int32), ("mode_hint", C.c_int32),
                ("joins", sr_frag_join * SR_MAX_FRAG_JOINS), ("agg", sr_agg_desc)]


class sr_fragment_plan(C.Structure):
    _fields_ = [("num_joins", C.c_int32), ("order", C.c_int32 * SR_MAX_FRAG_JOINS),
                ("bitmap_in_smem", C.c_int32 * SR_MAX_FRAG_JOINS), ("pass_rate", C.c_double * SR_MAX_FRAG_JOINS),
                ("smem_bytes", C.c_int32), ("grid", C.c_int32), ("block", C.c_int32), ("agg_in_smem", C.c_int32),
                ("mode", C.c_int32), ("num_stream_joins", C.c_int32), ("num_gather_passes", C.c_int32),
                ("final_pass", C.c_int32), ("pred_rate", C.c_double)]


FINAL_PASS_NAMES = {0: None, 1: "generic", 2: "expand", 3: "dense-batched"}   # sr_fragment_plan.final_pass (SR_FINAL_PASS_*)


class sr_part_desc(C.Structure):
    _fields_ = [("hash_fn", C.c_int32), ("reduce_op", C.c_int32), ("num_channels", C.c_int32),
                ("num_part_slots", C.c_int32), ("part_slots", C.c_int32 * SR_MAX_PART_KEYS)]


class sr_rf_info(C.Structure):
    _fields_ = [("min_value", C.c_int64), ("max_value", C.c_int64), ("num_inserted", C.c_int64), ("has_null", C.c_int32),
                ("log_num_buckets", C.c_int32), ("key_type", C.c_int32), ("num_in_values", C.c_int32)]


class sr_scan_rf_stats(C.Structure):
    _fields_ = [("rows_tested", C.c_int64), ("rows_passed", C.c_int64), ("batches_skipped", C.c_int64), ("last_selectivity", C.c_double)]


RF_IN_FILTER_ROW_LIMIT = 1024


STATE_REDUCE_SUM, STATE_REDUCE_MIN, STATE_REDUCE_MAX = 0, 1, 2


class sr_agg_state_array(C.Structure):
    _fields_ = [("data", C.c_void_p), ("count", C.c_int64), ("elem_type", C.c_int32), ("reduce", C.c_int32)]


# ---------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------
class Chunk:
    """Owns the ctypes arrays of a sr_chunk_view and keeps the column buffers alive.

    columns: list of (slot_id, data, nulls_or_None[, sr_type]).  `data`/`nulls` are numpy arrays
    (host) or objects with .data_ptr() (torch CUDA tensors, device) or raw ints (pointers).
    """

    def __init__(self, columns, num_rows=None, mem=MEM_HOST):
        self._keep = []
        self.slots = []
        self.types = []
        cols = (sr_col_view * max(1, len(columns)))()
        n = num_rows
        for k, col in enumerate(columns):
            slot, data, nulls = col[0], col[1], col[2]
            typ = col[3] if len(col) > 3 else None
            dptr, dn, dtyp = _ptr_of(data)
            nptr, _, _ = _ptr_of(nulls) if nulls is not None else (None, None, None)
            if typ is None:
                typ = dtyp
            if typ is None:
                raise ValueError("column type required for raw pointers")
            if n is None:
                n = dn
            cols[k].data = dptr
            cols[k].nulls = nptr
            cols[k].type = typ
            cols[k].slot_id = slot
            self._keep.append((data, nulls))
            self.slots.append(slot)
            self.types.append(typ)
        self._cols = cols
        self.view = sr_chunk_view(C.cast(cols, C.POINTER(sr_col_view)), len(columns), mem, 0 if n is None else n)
        self.num_rows = self.view.num_rows
        self.mem = mem

    def ref(self):
        return C.byref(self.view)

    def columns(self):
        """-> [(slot_id, data, nulls_or_None)] as passed to the constructor"""
        return [(s, d, nl) for s, (d, nl) in zip(self.slots, self._keep)]


def _ptr_of(x):
    """-> (pointer int, num elements or None, sr_type or None)"""
    if x is None:
        return None, None, None
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise ValueError("column arrays must be contiguous")
        if x.dtype.kind == "V" and x.dtype.itemsize == 16:
            return x.ctypes.data, x.shape[0], None
        return x.ctypes.data, x.shape[0], NUMPY_TYPE.get(x.dtype)
    if hasattr(x, "data_ptr"):  # torch tensor
        import torch
        tmap = {torch.uint8: TYPE_BOOLEAN, torch.int8: TYPE_TINYINT, torch.int16: TYPE_SMALLINT,
                torch.int32: TYPE_INT, torch.int64: TYPE_BIGINT, torch.float32: TYPE_FLOAT,
                torch.float64: TYPE_DOUBLE}
        return x.data_ptr(), x.numel(), tmap.get(x.dtype)
    if isinstance(x, int):
        return x, None, None
    raise TypeError(f"unsupported column buffer {type(x)}")


def make_pred(slot, op, lo=0, hi=0, in_list=None, is_double=False):
    p = sr_pred()
    p.slot_id = slot
    p.op = op
    if is_double:
        p.dlo, p.dhi = float(lo), float(hi)
    else:
        p.ilo, p.ihi = int(lo), int(hi)
    if in_list is not None:
        if len(in_list) > SR_MAX_IN_LIST:
            raise ValueError("IN list too long")
        for k, v in enumerate(in_list):
            p.in_list[k] = int(v)
        p.in_count = len(in_list)
    return p


def make_expr(rpn):
    """rpn: list of tokens: ('col', slot) | ('i', int) | ('d', float) | one of
    '+','-','*','/','todouble','==','!=','<','<=','>','>=','and','or','not','isnull'."""
    ops = {"+": EX_ADD, "-": EX_SUB, "*": EX_MUL, "/": EX_DIV, "todouble": EX_TO_DOUBLE, "==": EX_EQ, "!=": EX_NE,
           "<": EX_LT, "<=": EX_LE, ">": EX_GT, ">=": EX_GE, "and": EX_AND, "or": EX_OR, "not": EX_NOT,
           "isnull": EX_IS_NULL}
    e = sr_expr()
    if len(rpn) > SR_MAX_EXPR_NODES:
        raise ValueError("expression too long")
    for k, tok in enumerate(rpn):
        nd = e.nodes[k]
        if isinstance(tok, tuple):
            kind, val = tok
            if kind == "col":
                nd.op, nd.slot_id = EX_COL, int(val)
            elif kind == "i":
                nd.op, nd.ival = EX_ICONST, int(val)
            elif kind == "d":
                nd.op, nd.dval = EX_DCONST, float(val)
            else:
                raise ValueError(tok)
        else:
            nd.op = ops[tok]
    e.num_nodes = len(rpn)
    return e


class ScanDesc:
    def __init__(self, preds=(), filter_exprs=(), out_slots=()):
        self._preds = (sr_pred * max(1, len(preds)))(*preds)
        self._exprs = (sr_expr * max(1, len(filter_exprs)))(*filter_exprs)
        self._slots = (C.c_int32 * max(1, len(out_slots)))(*out_slots)
        self.out_slots = list(out_slots)
        self.desc = sr_scan_desc(C.cast(self._preds, C.POINTER(sr_pred)), len(preds), len(filter_exprs),
                                 C.cast(self._exprs, C.POINTER(sr_expr)), C.cast(self._slots, C.POINTER(C.c_int32)),
                                 len(out_slots), 0)

    def ref(self):
        return C.byref(self.desc)


def make_join_desc(join_type, build_keys, probe_keys, key_types, build_out=(), probe_out=(), enable_rdm=True, build_out_types=(), probe_out_types=(),
                   other_conjunct=None):
    d = sr_join_desc()
    d.join_type = join_type
    d.num_keys = len(build_keys)
    for k in range(len(build_keys)):
        d.build_key_slots[k] = build_keys[k]
        d.probe_key_slots[k] = probe_keys[k]
        d.key_types[k] = key_types[k]
    d.num_build_out = len(build_out)
    for k, s in enumerate(build_out):
        d.build_out_slots[k] = s
    d.num_probe_out = len(probe_out)
    for k, s in enumerate(probe_out):
        d.probe_out_slots[k] = s
    d.enable_range_direct_mapping = 1 if enable_rdm else 0
    for k, t in enumerate(build_out_types):
        d.build_out_types[k] = t
    for k, t in enumerate(probe_out_types):
        d.probe_out_types[k] = t
    if other_conjunct is not None:
        d.other_conjunct = make_expr(other_conjunct)
    return d


def make_agg_desc(group_slots=(), group_types=(), fns=(), ranges=None, group_nullable=None, expected_groups=0):
    """fns: list of (kind, input_type, out_slot, rpn_or_None)."""
    d = sr_agg_desc()
    d.num_group_keys = len(group_slots)
    for k in range(len(group_slots)):
        d.group_slots[k] = group_slots[k]
        d.group_types[k] = group_types[k]
        d.group_nullable[k] = int(group_nullable[k]) if group_nullable else 0
    if ranges is not None:
        d.has_ranges = 1
        for k, (lo, hi) in enumerate(ranges):
            d.group_min[k], d.group_max[k] = int(lo), int(hi)
    d.num_fns = len(fns)
    for k, (kind, ityp, out_slot, rpn) in enumerate(fns):
        d.fns[k].kind = kind
        d.fns[k].input_type = ityp
        d.fns[k].out_slot = out_slot
        if rpn is not None:
            d.fns[k].input = make_expr(rpn)
    d.expected_groups = expected_groups
    return d


def make_part_desc(part_slots, num_channels, hash_fn=HASH_FNV, reduce_op=REDUCE_MULHI):
    d = sr_part_desc()
    d.hash_fn, d.reduce_op, d.num_channels, d.num_part_slots = hash_fn, reduce_op, num_channels, len(part_slots)
    for k, s in enumerate(part_slots):
        d.part_slots[k] = s
    return d


def agg_state_slot(out_slot):
    """SR_AGG_STATE_SLOT: slot of the second state column of a function (AVG: the count)"""
    return out_slot | 0x40000000


def two_phase_descs(desc):
    """Python statement of sr_agg_two_phase_descs (include/sr_gpu_ops.h): single-phase desc -> (first phase, merge phase).
    AVG(x) becomes SUM(double(x)) + COUNT(x) in the first phase and AVG_MERGE(sum, count) in the merge phase; counts are
    summed, sums summed, MIN / MAX re-applied.  Raises NotImplementedError where the C function returns
    SR_ERR_NOT_SUPPORTED (128-bit states, more than SR_MAX_AGG_FNS first-phase functions)."""
    p1, p2 = sr_agg_desc(), sr_agg_desc()
    C.memmove(C.byref(p1), C.byref(desc), C.sizeof(sr_agg_desc))
    C.memmove(C.byref(p2), C.byref(desc), C.sizeof(sr_agg_desc))
    for f in range(SR_MAX_AGG_FNS):
        C.memset(C.byref(p1.fns[f]), 0, C.sizeof(sr_agg_fn))
    n1 = 0

    def state_col(slot):
        e = sr_expr()
        e.nodes[0].op, e.nodes[0].slot_id, e.num_nodes = EX_COL, slot, 1
        return e
    float_class = (TYPE_FLOAT, TYPE_DOUBLE)
    for f in range(desc.num_fns):
        fn = desc.fns[f]
        m = sr_agg_fn()
        m.out_slot = fn.out_slot
        if fn.kind == AGG_AVG_MERGE:
            raise ValueError("already a merge phase")
        if fn.kind == AGG_COUNT_DISTINCT:
            raise NotImplementedError("COUNT(DISTINCT) is single-phase: shuffle on the group keys")
        if fn.kind not in (AGG_COUNT, AGG_COUNT_STAR, AGG_AVG) and TYPE_WIDTH[agg_result_type(fn.kind, fn.input_type)] > 8:
            raise NotImplementedError("128-bit states")
        if n1 + (2 if fn.kind == AGG_AVG else 1) > SR_MAX_AGG_FNS:
            raise NotImplementedError("too many first-phase functions")
        if fn.kind == AGG_AVG:
            C.memmove(C.byref(p1.fns[n1]), C.byref(fn), C.sizeof(sr_agg_fn))
            s1 = p1.fns[n1]
            s1.kind, s1.reserved = AGG_SUM, 0
            if fn.input_type not in float_class:
                s1.input.nodes[s1.input.num_nodes].op = EX_TO_DOUBLE
                s1.input.num_nodes += 1
                s1.input_type = TYPE_DOUBLE
            C.memmove(C.byref(p1.fns[n1 + 1]), C.byref(fn), C.sizeof(sr_agg_fn))
            c1 = p1.fns[n1 + 1]
            c1.kind, c1.reserved, c1.out_slot = AGG_COUNT, 0, agg_state_slot(fn.out_slot)
            n1 += 2
            m.kind, m.input_type, m.input, m.reserved = AGG_AVG_MERGE, TYPE_DOUBLE, state_col(fn.out_slot), agg_state_slot(fn.out_slot)
        else:
            C.memmove(C.byref(p1.fns[n1]), C.byref(fn), C.sizeof(sr_agg_fn))
            n1 += 1
            m.input = state_col(fn.out_slot)
            if fn.kind in (AGG_COUNT, AGG_COUNT_STAR):
                m.kind, m.input_type = AGG_SUM, TYPE_BIGINT
            elif fn.kind == AGG_SUM:
                m.kind, m.input_type = AGG_SUM, agg_result_type(fn.kind, fn.input_type)
            else:
                m.kind, m.input_type = fn.kind, fn.input_type
        C.memmove(C.byref(p2.fns[f]), C.byref(m), C.sizeof(sr_agg_fn))
    p1.num_fns = n1
    return p1, p2


def agg_result_type(kind, input_type):
    """SumResultLT / AvgResultLT (be/src/exprs/agg/sum.h:24-34, avg.h:27-47)."""
    if kind in (AGG_COUNT, AGG_COUNT_STAR, AGG_COUNT_DISTINCT):
        return TYPE_BIGINT
    if kind in (AGG_AVG, AGG_AVG_MERGE):
        return TYPE_DOUBLE
    if kind == AGG_SUM:
        if input_type in (TYPE_FLOAT, TYPE_DOUBLE):
            return TYPE_DOUBLE
        if input_type in (TYPE_DECIMAL32, TYPE_DECIMAL64, TYPE_DECIMAL128):
            return TYPE_DECIMAL128
        if input_type == TYPE_LARGEINT:
            return TYPE_LARGEINT
        return TYPE_BIGINT
    return input_type  # MIN / MAX keep the input type
