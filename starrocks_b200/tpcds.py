"""TPC-DS Q95-shaped workload (BASELINE.json config 4): synthetic shardable generator, operator descriptors and ONE plan
function that runs on either engine -- the CUDA operators through the C-ABI or the CPU oracle -- so that parity means "the
same plan over the same chunks gives the same three numbers".

    with ws_wh as (select ws1.ws_order_number from web_sales ws1, web_sales ws2
                   where ws1.ws_order_number = ws2.ws_order_number and ws1.ws_warehouse_sk <> ws2.ws_warehouse_sk)
    select count(distinct ws_order_number), sum(ws_ext_ship_cost), sum(ws_net_profit)
    from web_sales ws1, date_dim, customer_address, web_site
    where d_date between D and D + 60 days and ws1.ws_ship_date_sk = d_date_sk
      and ws1.ws_ship_addr_sk = ca_address_sk and ca_state = 'IL'
      and ws1.ws_web_site_sk = web_site_sk and web_company_name = 'pri'
      and ws1.ws_order_number in (select ws_order_number from ws_wh)
      and ws1.ws_order_number in (select wr_order_number from web_returns, ws_wh where wr_order_number = ws_wh.ws_order_number)

Plan of one fragment instance (web_sales / web_returns HASH_PARTITIONED on the order number, dimensions broadcast):
    web_sales SELF JOIN on ws_order_number (one-to-many: JoinHashMap's chain walk, join_hash_map.hpp:718-795),
        other conjunct wh1 <> wh2 as a filter over the join output                 -> ws_wh
    ws_wh  GROUP BY ws_order_number (duplicate-free build side of the IN-subqueries) -> LEFT SEMI builds S1, S1r
    web_returns LEFT SEMI S1r                                                        -> LEFT SEMI build S2
    web_sales: date range, LEFT SEMI date_dim / customer_address / web_site / S1 / S2
        -> COUNT(DISTINCT ws_order_number), SUM(ws_ext_ship_cost), SUM(ws_net_profit)  (distinct.h:48-62, sum.h)
Row counts follow TPC-DS (per unit of SF: 60 K orders, 720 K web_sales rows -- 1..23 lines per order --, 12 K web_returns
rows, 6 K addresses; 54 sites); values are counter-based hashes of (order, line) like tpch.HashGen.
"""
import numpy as np

from . import abi
from .tpch import HashGen

# slots
WS_ORDER, WS_WH, WS_SHIP_DATE, WS_ADDR, WS_SITE, WS_COST, WS_PROFIT = 0, 1, 2, 3, 4, 5, 6
WS2_ORDER, WS2_WH = 10, 11          # the build side of the self join: the same columns under other slot ids
D_DATE_SK, CA_ADDRESS_SK, WEB_SITE_SK = 20, 21, 22
OUT_DISTINCT, OUT_COST, OUT_PROFIT = 30, 31, 32

DATE_LO = 2451211                    # d_date_sk of the first day of the 60-day window
DATE_SPAN = 1823                     # ship dates cover five years from DATE0
DATE0 = 2450815
NUM_SITES = 54
MAX_LINES = 32                       # lines per order < 32: row key = order * 32 + line

WS_COLS = [("ws_order_number", WS_ORDER, abi.TYPE_BIGINT), ("ws_warehouse_sk", WS_WH, abi.TYPE_INT), ("ws_ship_date_sk", WS_SHIP_DATE, abi.TYPE_INT),
           ("ws_ship_addr_sk", WS_ADDR, abi.TYPE_INT), ("ws_web_site_sk", WS_SITE, abi.TYPE_INT), ("ws_ext_ship_cost", WS_COST, abi.TYPE_BIGINT),
           ("ws_net_profit", WS_PROFIT, abi.TYPE_BIGINT)]


class Q95Gen(HashGen):
    """every column a pure function of (order index, line): any rank generates any block of orders on its own device"""

    def __init__(self, sf, device=None):
        super().__init__(1.0, device)
        self.n_orders = max(16, int(60_000 * sf))
        self.n_addr = max(50, int(6_000 * sf))

    def _where(self, c, a, b):
        if self.dev is None:
            return np.where(c, a, b)
        import torch
        return torch.where(c, a, b)

    def _expand(self, per):
        """(order position of every line, line number inside its order)"""
        if self.dev is None:
            rep = np.repeat(np.arange(len(per), dtype=np.int64), per)
            first = np.cumsum(per) - per
            return rep, np.arange(len(rep), dtype=np.int64) - first[rep]
        import torch
        rep = torch.repeat_interleave(torch.arange(per.numel(), dtype=torch.int64, device=self.dev), per)
        first = torch.cumsum(per, 0) - per
        return rep, torch.arange(rep.numel(), dtype=torch.int64, device=self.dev) - first[rep]

    def lines_per_order(self, o):
        return 1 + self._h(1, o) % 23

    def web_sales_of_orders(self, lo, hi):
        o = self._arange(lo, hi)
        rep, line = self._expand(self.lines_per_order(o))
        orow = o[rep]
        key = orow * MAX_LINES + line
        # most lines of an order ship from its home warehouse, so a share of the orders never meets wh1 <> wh2
        home = self._h(2, orow) % 15
        wh = 1 + self._where(self._h(3, key) % 10 < 8, home, self._h(4, key) % 15)
        return {"ws_order_number": orow + 1, "ws_warehouse_sk": self._i32(wh), "ws_ship_date_sk": self._i32(DATE0 + self._h(5, key) % DATE_SPAN),
                "ws_ship_addr_sk": self._i32(1 + self._h(6, key) % self.n_addr), "ws_web_site_sk": self._i32(1 + self._h(7, key) % NUM_SITES),
                "ws_ext_ship_cost": self._h(8, key) % 100_000, "ws_net_profit": self._h(9, key) % 200_001 - 100_000}

    def returns_per_order(self, o):
        r = 1 + self._h(11, o) % 3
        return self._where(self._h(10, o) % 10 == 0, r, r * 0)

    def web_returns_of_orders(self, lo, hi):
        o = self._arange(lo, hi)
        rep, _ = self._expand(self.returns_per_order(o))
        return {"wr_order_number": o[rep] + 1}

    # dimensions after their scan predicates (the broadcast build sides)
    def date_keys(self):
        return self._i32(self._arange(DATE_LO, DATE_LO + 61))

    def address_ok(self, a):
        return self._h(12, a) % 8 == 7           # ca_state = 'IL'

    def address_keys(self):
        a = self._arange(1, self.n_addr + 1)
        return self._i32(a[self.address_ok(a)])

    def site_ok(self, s):
        return s % 3 == 1                        # web_company_name = 'pri'

    def site_keys(self):
        s = self._arange(1, NUM_SITES + 1)
        return self._i32(s[self.site_ok(s)])

    def expected(self, lo, hi):
        """the query over the generator functions, join-free, for the orders [lo, hi) -> (distinct orders, cost, profit)"""
        ws = self.web_sales_of_orders(lo, hi)
        o = self._arange(lo, hi)
        per = self.lines_per_order(o)
        rep, _ = self._expand(per)
        wh = ws["ws_warehouse_sk"]
        n = hi - lo
        if self.dev is None:
            mn = np.full(n, 1 << 30, dtype=np.int64)
            mx = np.zeros(n, dtype=np.int64)
            np.minimum.at(mn, rep, wh)
            np.maximum.at(mx, rep, wh)
        else:
            import torch
            mn = torch.full((n,), 1 << 30, dtype=torch.int64, device=self.dev).scatter_reduce(0, rep, wh.to(torch.int64), "amin")
            mx = torch.zeros(n, dtype=torch.int64, device=self.dev).scatter_reduce(0, rep, wh.to(torch.int64), "amax")
        order_ok = (mn != mx) & (self.returns_per_order(o) > 0)
        d = ws["ws_ship_date_sk"]
        row_ok = order_ok[rep] & (d >= DATE_LO) & (d <= DATE_LO + 60) & self.address_ok(ws["ws_ship_addr_sk"].astype(np.int64) if self.dev is None else ws["ws_ship_addr_sk"].to(dtype=mn.dtype)) \
            & self.site_ok(ws["ws_web_site_sk"])
        if self.dev is None:
            hit = np.zeros(n, dtype=bool)
            hit[rep[row_ok]] = True
        else:
            import torch
            hit = torch.zeros(n, dtype=torch.bool, device=self.dev)
            hit[rep[row_ok]] = True
        return int(hit.sum()), int(ws["ws_ext_ship_cost"][row_ok].sum()), int(ws["ws_net_profit"][row_ok].sum())


# ---------------------------------------------------------------------------------------------------------------------
# descriptors
# ---------------------------------------------------------------------------------------------------------------------
def q95_descs():
    d = {}
    d["self_join"] = abi.make_join_desc(abi.JOIN_INNER, [WS2_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], build_out=[WS2_WH], probe_out=[WS_ORDER, WS_WH])
    d["wh_differs"] = abi.ScanDesc(filter_exprs=[abi.make_expr([("col", WS_WH), ("col", WS2_WH), "!="])], out_slots=[WS_ORDER])
    d["ws_wh_distinct"] = lambda expected: abi.make_agg_desc([WS_ORDER], [abi.TYPE_BIGINT], expected_groups=expected)
    main_out = [WS_ORDER, WS_ADDR, WS_SITE, WS_COST, WS_PROFIT]
    d["date_scan"] = abi.ScanDesc(preds=[abi.make_pred(WS_SHIP_DATE, abi.PRED_BETWEEN, DATE_LO, DATE_LO + 60)], out_slots=[WS_SHIP_DATE] + main_out)
    d["semi_date"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [D_DATE_SK], [WS_SHIP_DATE], [abi.TYPE_INT], probe_out=main_out)
    d["semi_addr"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [CA_ADDRESS_SK], [WS_ADDR], [abi.TYPE_INT], probe_out=[WS_ORDER, WS_SITE, WS_COST, WS_PROFIT])
    d["semi_site"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [WEB_SITE_SK], [WS_SITE], [abi.TYPE_INT], probe_out=[WS_ORDER, WS_COST, WS_PROFIT])
    d["semi_order"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [WS_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], probe_out=[WS_ORDER, WS_COST, WS_PROFIT])
    d["semi_returns"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [WS_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], probe_out=[WS_ORDER])
    d["final_agg"] = abi.make_agg_desc(fns=[(abi.AGG_COUNT_DISTINCT, abi.TYPE_BIGINT, OUT_DISTINCT, [("col", WS_ORDER)]),
                                            (abi.AGG_SUM, abi.TYPE_BIGINT, OUT_COST, [("col", WS_COST)]),
                                            (abi.AGG_SUM, abi.TYPE_BIGINT, OUT_PROFIT, [("col", WS_PROFIT)])])
    return d


WR_ORDER = 40                        # web_returns' order number as a build key


def fused_conj_descs():
    """The self join with wh1 <> wh2 as its other-join conjunct, in the two shapes the fused fragment runs:
      ws_wh  web_sales ws1 JOIN web_sales ws2 ON order AND wh1 <> wh2, GROUP BY ws1.ws_order_number (Q95's CTE);
      q94    the Q94 body: ship date BETWEEN, LEFT SEMI date / address / site, EXISTS (ws2: same order, other warehouse)
             as a LEFT SEMI self join with the conjunct, NOT EXISTS web_returns as a LEFT ANTI join, then COUNT(*),
             SUM(ws_ext_ship_cost), SUM(ws_net_profit).
    -> {name: join descriptor or (scan, agg) descriptors}; the self joins' build side is web_sales as (WS2_ORDER, WS2_WH)"""
    wh_differs = [("col", WS_WH), ("col", WS2_WH), "!="]
    d = {}
    d["ws_wh_join"] = abi.make_join_desc(abi.JOIN_INNER, [WS2_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], probe_out=[WS_ORDER], other_conjunct=wh_differs)
    d["ws_wh_agg"] = lambda expected: abi.make_agg_desc([WS_ORDER], [abi.TYPE_BIGINT], expected_groups=expected)
    body = [WS_ORDER, WS_WH, WS_COST, WS_PROFIT]
    d["q94_scan"] = abi.ScanDesc(preds=[abi.make_pred(WS_SHIP_DATE, abi.PRED_BETWEEN, DATE_LO, DATE_LO + 60)], out_slots=[WS_SHIP_DATE, WS_ADDR, WS_SITE] + body)
    d["q94_semi_date"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [D_DATE_SK], [WS_SHIP_DATE], [abi.TYPE_INT], probe_out=[WS_ADDR, WS_SITE] + body)
    d["q94_semi_addr"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [CA_ADDRESS_SK], [WS_ADDR], [abi.TYPE_INT], probe_out=[WS_SITE] + body)
    d["q94_semi_site"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [WEB_SITE_SK], [WS_SITE], [abi.TYPE_INT], probe_out=body)
    d["q94_exists"] = abi.make_join_desc(abi.JOIN_LEFT_SEMI, [WS2_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], probe_out=body, other_conjunct=wh_differs)
    d["q94_not_returned"] = abi.make_join_desc(abi.JOIN_LEFT_ANTI, [WR_ORDER], [WS_ORDER], [abi.TYPE_BIGINT], probe_out=[WS_COST, WS_PROFIT])
    d["q94_agg"] = abi.make_agg_desc(fns=[(abi.AGG_COUNT_STAR, 0, OUT_DISTINCT, None), (abi.AGG_SUM, abi.TYPE_BIGINT, OUT_COST, [("col", WS_COST)]),
                                          (abi.AGG_SUM, abi.TYPE_BIGINT, OUT_PROFIT, [("col", WS_PROFIT)])])
    return d


def q94_expected(gen, lo, hi):
    """the q94 body of fused_conj_descs over the generator functions, join-free, for the orders [lo, hi) -> (count, cost,
    profit); numpy generator only"""
    ws = gen.web_sales_of_orders(lo, hi)
    o = gen._arange(lo, hi)
    rep, _ = gen._expand(gen.lines_per_order(o))
    wh = ws["ws_warehouse_sk"]
    mn = np.full(hi - lo, 1 << 30, dtype=np.int64)
    mx = np.zeros(hi - lo, dtype=np.int64)
    np.minimum.at(mn, rep, wh)
    np.maximum.at(mx, rep, wh)
    order_ok = (mn != mx) & (gen.returns_per_order(o) == 0)
    d = ws["ws_ship_date_sk"]
    ok = order_ok[rep] & (d >= DATE_LO) & (d <= DATE_LO + 60) & gen.address_ok(ws["ws_ship_addr_sk"].astype(np.int64)) & gen.site_ok(ws["ws_web_site_sk"])
    return int(ok.sum()), int(ws["ws_ext_ship_cost"][ok].sum()), int(ws["ws_net_profit"][ok].sum())


# ---------------------------------------------------------------------------------------------------------------------
# engines: the same four verbs over the CUDA operators and over the oracle
# ---------------------------------------------------------------------------------------------------------------------
class GpuEngine:
    mem = abi.MEM_DEVICE

    def __init__(self, gpu, ctx):
        self.gpu, self.ctx, self.handles = gpu, ctx, []

    def _dev(self, out):
        return abi.Chunk([(out.cols[k].slot_id, out.cols[k].data, out.cols[k].nulls, out.cols[k].type) for k in range(out.num_cols)],
                         num_rows=out.num_rows, mem=abi.MEM_DEVICE)

    def scan(self, desc):
        s = self.gpu.Scan(self.ctx, desc)
        self.handles.append(s)
        return lambda chunk: self._dev(s.filter(chunk))

    def join(self, desc, build_chunks):
        j = self.gpu.Join(self.ctx, desc)
        self.handles.append(j)
        for ch in build_chunks:
            j.append_build(ch)
        j.build_finish()
        return lambda chunk: self._dev(j.probe(chunk))

    def agg(self, desc):
        a = self.gpu.Agg(self.ctx, desc)
        self.handles.append(a)

        def finish():
            a.finish()
            return self._dev(a.pull(mem=abi.MEM_DEVICE))
        return a.push, finish

    def rows(self, chunk):
        out = []
        for s, d, nl in chunk.columns():
            k = chunk.slots.index(s)
            w = abi.TYPE_WIDTH[chunk.types[k]]
            raw = self.gpu._copy_dev_to_host(self.ctx, d, w * chunk.num_rows)
            out.append(raw.view({4: np.int32, 8: np.int64}[w]))
        return out

    def close(self):
        for h in reversed(self.handles):
            h.close()
        self.handles = []


class OracleEngine:
    mem = abi.MEM_HOST

    def __init__(self, oracle):
        self.oracle = oracle

    def scan(self, desc):
        def run(chunk):
            _, res = self.oracle.scan_filter(desc, chunk)
            return abi.Chunk([(s, res[s][0], res[s][1], chunk.types[chunk.slots.index(s)]) for s in desc.out_slots])
        return run

    def join(self, desc, build_chunks):
        j = self.oracle.Join(desc)
        for ch in build_chunks:
            j.append_build(ch)
        j.build()

        def probe(chunk):
            pi, bi = j.probe_all(chunk, cap=max(1024, chunk.num_rows * 16))
            cols = j.output(chunk, pi, bi)
            types = {s: t for s, t in zip(chunk.slots, chunk.types)}
            types.update(j.build_types)
            return abi.Chunk([(s, d, None, types[s]) for s, d, _ in cols], num_rows=len(pi))
        return probe

    def agg(self, desc):
        a = self.oracle.Agg(desc)

        slots = [desc.group_slots[k] for k in range(desc.num_group_keys)] + [desc.fns[f].out_slot for f in range(desc.num_fns)]

        def finish():
            out = a.output()                                  # (type, data, nulls) per column, keys first
            return abi.Chunk([(s, dt, None, t) for s, (t, dt, _) in zip(slots, out)], num_rows=len(out[0][1]) if out else 0)
        return a.push, finish

    def rows(self, chunk):
        return [d for _, d, _ in chunk.columns()]

    def close(self):
        pass


def q95_local_plan(eng, ws, wr, dims, morsel_rows=4_000_000, expected_orders=0):
    """the fragment instance over its (complete-orders) shard.  ws: chunk with WS_COLS; wr: chunk [(WS_ORDER, wr_order_number)];
    dims: {"date","addr","site"} -> single-column chunks.  -> ((distinct, cost, profit), {"pairs": self-join output rows, ...})"""
    d = q95_descs()
    stats = {}
    cols = {s: (data, nl) for s, data, nl in ws.columns()}
    n = ws.num_rows

    def ws_slice(lo, hi, slots, rename=None):
        out = []
        for s in slots:
            data = cols[s][0]
            w = abi.TYPE_WIDTH[ws.types[ws.slots.index(s)]]
            piece = data[lo:hi] if hasattr(data, "__getitem__") else data + lo * w
            out.append(((rename or {}).get(s, s), piece, None, ws.types[ws.slots.index(s)]))
        return abi.Chunk(out, num_rows=hi - lo, mem=eng.mem)

    # ws_wh: one-to-many self join, other conjunct, duplicate-free order numbers
    probe_self = eng.join(d["self_join"], [ws_slice(0, n, [WS_ORDER, WS_WH], {WS_ORDER: WS2_ORDER, WS_WH: WS2_WH})])
    differs = eng.scan(d["wh_differs"])
    push_wswh, finish_wswh = eng.agg(d["ws_wh_distinct"](expected_orders))
    pairs = 0
    for lo in range(0, n, morsel_rows):
        joined = probe_self(ws_slice(lo, min(n, lo + morsel_rows), [WS_ORDER, WS_WH]))
        pairs += joined.num_rows
        if joined.num_rows:
            push_wswh(differs(joined))
    ws_wh = finish_wswh()
    stats["self_join_rows"] = pairs
    stats["ws_wh_orders"] = ws_wh.num_rows
    # IN (select wr_order_number from web_returns, ws_wh ...)
    returned = eng.join(d["semi_returns"], [ws_wh])(wr)
    stats["returned_orders_rows"] = returned.num_rows
    in_ws_wh = eng.join(d["semi_order"], [ws_wh])
    in_returns = eng.join(d["semi_order"], [returned])
    on_date = eng.join(d["semi_date"], [dims["date"]])
    on_addr = eng.join(d["semi_addr"], [dims["addr"]])
    on_site = eng.join(d["semi_site"], [dims["site"]])
    date_scan = eng.scan(d["date_scan"])
    push_final, finish_final = eng.agg(d["final_agg"])
    reach = 0
    for lo in range(0, n, morsel_rows):
        x = date_scan(ws_slice(lo, min(n, lo + morsel_rows), [WS_ORDER, WS_SHIP_DATE, WS_ADDR, WS_SITE, WS_COST, WS_PROFIT]))
        for step in (on_date, on_addr, on_site, in_ws_wh, in_returns):
            if x.num_rows == 0:
                break
            x = step(x)
        if x.num_rows:
            reach += x.num_rows
            push_final(x)
    stats["rows_aggregated"] = reach
    out = finish_final()
    r = eng.rows(out)
    return (int(r[0][0]), int(r[1][0]) if reach else 0, int(r[2][0]) if reach else 0), stats


def table_chunk(table, cols, mem=abi.MEM_HOST):
    return abi.Chunk([(slot, table[name], None, typ) for name, slot, typ in cols], mem=mem)
