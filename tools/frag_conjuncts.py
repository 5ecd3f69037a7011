"""The fused fragment against the per-operator chain on the TPC-DS Q95 / Q94 self join with `wh1 <> wh2`, one H100:

    python tools/frag_conjuncts.py [--sf 125] [--steps 5] [--warmup 1] [--out results.json]

Two variants over the same HBM-resident web_sales shard (tpcds.Q95Gen; SF125 is the per-GPU share of SF1000 on eight
GPUs), pushed in 4 M-row morsels as tpcds.q95_local_plan pushes them:
  ws_wh  web_sales ws1 JOIN web_sales ws2 ON order AND wh1 <> wh2, GROUP BY ws1.ws_order_number;
         per-operator: the first loop of tpcds.q95_local_plan (sr_join_probe, a filter on wh1 <> wh2, sr_agg_push);
  q94    the Q94 body (tpcds.fused_conj_descs): ship date BETWEEN, LEFT SEMI date / address / site, LEFT SEMI self join
         with the conjunct, LEFT ANTI web_returns, COUNT(*) and two SUMs;
         per-operator: sr_scan_filter, sr_join_probe per join (the self join evaluates its conjunct), sr_agg_push.
Each step runs the whole variant, fused and per-operator alternately; the outputs are pulled to the host and must be
equal (ws_wh: the group count and the sorted keys; q94: all three numbers).  Times are device events around one step;
the card's name and power limit are read in the same call.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, tpcds  # noqa: E402
from tools.frag_join_kinds import card, timed  # noqa: E402

MORSEL = 4_000_000


def dev_chunk(cols):
    """[(slot, tensor)] -> device chunk (the tensors' own types)"""
    t = {torch.int32: abi.TYPE_INT, torch.int64: abi.TYPE_BIGINT}
    return abi.Chunk([(s, x, None, t[x.dtype]) for s, x in cols], num_rows=cols[0][1].numel(), mem=abi.MEM_DEVICE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=125.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--variants", default="ws_wh,q94")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frag_conjuncts.py: no CUDA device")
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    gen = tpcds.Q95Gen(args.sf, device=dev)
    ws = {k: v.contiguous() for k, v in gen.web_sales_of_orders(0, gen.n_orders).items()}
    wr = gen.web_returns_of_orders(0, gen.n_orders)["wr_order_number"].contiguous()
    torch.cuda.synchronize()
    n = ws["ws_order_number"].numel()
    col = {tpcds.WS_ORDER: ws["ws_order_number"], tpcds.WS_WH: ws["ws_warehouse_sk"], tpcds.WS_SHIP_DATE: ws["ws_ship_date_sk"],
           tpcds.WS_ADDR: ws["ws_ship_addr_sk"], tpcds.WS_SITE: ws["ws_web_site_sk"], tpcds.WS_COST: ws["ws_ext_ship_cost"], tpcds.WS_PROFIT: ws["ws_net_profit"]}
    morsels = [(lo, min(n, lo + MORSEL)) for lo in range(0, n, MORSEL)]

    def slices(slots):
        return [dev_chunk([(s, col[s][lo:hi]) for s in slots]) for lo, hi in morsels]

    report = {"card": card(), "sf": args.sf, "rows": n, "orders": gen.n_orders, "morsel_rows": MORSEL, "steps": args.steps,
              "warmup": args.warmup, "variants": {}}
    print(f"card: {report['card']}  Q95Gen SF{args.sf:g}: {n} web_sales rows in HBM, {len(morsels)} morsels, {args.steps} timed steps")
    fd, qd = tpcds.fused_conj_descs(), tpcds.q95_descs()
    self_build = dev_chunk([(tpcds.WS2_ORDER, ws["ws_order_number"]), (tpcds.WS2_WH, ws["ws_warehouse_sk"])])
    eng = tpcds.GpuEngine(gpu, ctx)
    handles = []

    def join(desc, chunk):
        j = gpu.Join(ctx, desc)
        handles.append(j)
        j.append_build(chunk)
        j.build_finish()
        return j

    expected_orders = gen.n_orders
    for name in args.variants.split(","):
        if name == "ws_wh":
            fact = slices([tpcds.WS_ORDER, tpcds.WS_WH])
            frag = gpu.Fragment(ctx, abi.ScanDesc(), [(join(fd["ws_wh_join"], self_build), tpcds.WS_ORDER, [])], fd["ws_wh_agg"](expected_orders))
            # per-operator: tpcds.q95_local_plan's first loop
            probe_self = eng.join(qd["self_join"], [dev_chunk([(tpcds.WS2_ORDER, ws["ws_order_number"]), (tpcds.WS2_WH, ws["ws_warehouse_sk"])])])
            differs = eng.scan(qd["wh_differs"])
            op_agg = gpu.Agg(ctx, qd["ws_wh_distinct"](expected_orders))
            handles.append(op_agg)
            fact_op = fact

            def operators():
                op_agg.reset()
                pairs = 0
                for m in fact_op:
                    joined = probe_self(m)
                    pairs += joined.num_rows
                    if joined.num_rows:
                        op_agg.push(differs(joined))
                op_agg.finish()
                return gpu.chunk_out_to_host(ctx, op_agg.pull(mem=abi.MEM_HOST)), pairs

            def compare(f, o):
                fk, ok = np.sort(np.asarray(f[0][2])), np.sort(np.asarray(o[0][2]))
                return {"groups": int(fk.size)}, fk.size == ok.size and bool(np.array_equal(fk, ok))
        else:
            fact = slices([tpcds.WS_ORDER, tpcds.WS_WH, tpcds.WS_SHIP_DATE, tpcds.WS_ADDR, tpcds.WS_SITE, tpcds.WS_COST, tpcds.WS_PROFIT])
            specs = [("q94_semi_date", dev_chunk([(tpcds.D_DATE_SK, gen.date_keys())]), tpcds.WS_SHIP_DATE),
                     ("q94_semi_addr", dev_chunk([(tpcds.CA_ADDRESS_SK, gen.address_keys())]), tpcds.WS_ADDR),
                     ("q94_semi_site", dev_chunk([(tpcds.WEB_SITE_SK, gen.site_keys())]), tpcds.WS_SITE),
                     ("q94_exists", self_build, tpcds.WS_ORDER),
                     ("q94_not_returned", dev_chunk([(tpcds.WR_ORDER, wr)]), tpcds.WS_ORDER)]
            joins = [(join(fd[k], ch), probe) for k, ch, probe in specs]
            frag = gpu.Fragment(ctx, fd["q94_scan"], [(j, p, []) for j, p in joins], fd["q94_agg"])
            scan = gpu.Scan(ctx, fd["q94_scan"])
            handles.append(scan)
            op_agg = gpu.Agg(ctx, fd["q94_agg"])
            handles.append(op_agg)
            fact_op = fact

            def operators():
                op_agg.reset()
                reach = 0
                for m in fact_op:
                    x = gpu.chunk_out_as_view(scan.filter(m))
                    for j, _ in joins:
                        if x.num_rows == 0:
                            break
                        x = gpu.chunk_out_as_view(j.probe(x))
                    if x.num_rows:
                        reach += x.num_rows
                        op_agg.push(x)
                op_agg.finish()
                return gpu.chunk_out_to_host(ctx, op_agg.pull(mem=abi.MEM_HOST)), reach

            def compare(f, o):
                fv = [int(np.asarray(c[2])[0]) for c in f]
                ov = [int(np.asarray(c[2])[0]) for c in o]
                return {"count": fv[0], "cost": fv[1], "profit": fv[2]}, fv == ov

        def fused():
            frag.reset()
            for m in fact:
                frag.push(m)
            frag.agg.finish()
            return gpu.chunk_out_to_host(ctx, frag.agg.pull(mem=abi.MEM_HOST))

        for _ in range(args.warmup):
            fused()
            operators()
        fms, oms = [], []
        for _ in range(args.steps):          # alternated, so both forms see the same state of the machine
            fres, t = timed(fused, stream, 1, 0)
            fms += t
            passed = frag.rows_passed
            (ores, op_rows), t = timed(operators, stream, 1, 0)
            oms += t
        result, equal = compare(fres, ores)
        plan = frag.plan()
        r = {"fused_ms": {"best": min(fms), "median": float(np.median(fms))}, "operators_ms": {"best": min(oms), "median": float(np.median(oms))},
             "speedup_median": float(np.median(oms) / np.median(fms)), "rows_passed": passed, "operator_rows": op_rows, "equal": equal,
             "result": result, "plan": {k: plan[k] for k in ("mode", "order", "pass_rate", "num_stream_joins", "num_gather_passes", "final_pass")}}
        report["variants"][name] = r
        print(f"{name:6s} fused {r['fused_ms']['median']:8.2f} ms (best {r['fused_ms']['best']:.2f})  operators {r['operators_ms']['median']:8.2f} ms "
              f"(best {r['operators_ms']['best']:.2f})  x{r['speedup_median']:.2f}  {passed} rows passed (per-operator: {op_rows} rows "
              f"{'self-joined' if name == 'ws_wh' else 'aggregated'})  {result}  outputs {'equal' if equal else 'DIFFER'}  plan {r['plan']}")
        frag.close()
    eng.close()
    for h in reversed(handles):
        h.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)
    if not all(v["equal"] for v in report["variants"].values()):
        raise SystemExit("frag_conjuncts.py: the fused fragment and the per-operator chain disagree")


if __name__ == "__main__":
    main()
