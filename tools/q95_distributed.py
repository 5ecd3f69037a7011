"""TPC-DS Q95 shape across the N GPUs of one box (BASELINE.json config 4: SF1000 on 8 GPUs, ExchangeSink all-to-all).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/q95_distributed.py --sf 1000 [--check oracle|invariants|none]

Every rank generates the web_sales / web_returns rows of ITS block of orders on its own device (tpcds.Q95Gen), the
ExchangeSink step (sr_xchg_partition: FNV + ReduceOp, exchange_sink_operator.cpp:586-637) re-partitions both tables on the
order number and one grouped NCCL send/recv moves all columns; after it every order lives on exactly one rank, so the
self join, the IN-subqueries and COUNT(DISTINCT ws_order_number) are local (starrocks_b200.tpcds.q95_local_plan) and the
three results are summed over the ranks.  Checks: `invariants` -- the join-free evaluation of the query over the generator
functions, per block, all-reduced; `oracle` (small SF) -- the same plan run by the CPU oracle over the host-generated tables.
Rank 0 prints one JSON line (bench.py format); rows/s counts web_sales rows.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, tpcds  # noqa: E402
from starrocks_b200.distributed import device_view, exchange_partitions  # noqa: E402


def shuffle(xchg, chunk, dev, keep):
    out, offs = xchg.partition(chunk)
    cols = [device_view(out.cols[k].data, out.num_rows, abi.TYPE_WIDTH[out.cols[k].type], dev) for k in range(out.num_cols)]
    meta = [(out.cols[k].slot_id, out.cols[k].type) for k in range(out.num_cols)]
    recv = exchange_partitions(cols, offs.tolist())
    rank = dist.get_rank()
    sent_rows = int(out.num_rows - (offs[rank + 1] - offs[rank]))
    keep.append(recv)
    return abi.Chunk([(meta[k][0], recv[k], None, meta[k][1]) for k in range(len(meta))], num_rows=int(recv[0].numel()),
                     mem=abi.MEM_DEVICE), sent_rows * sum(abi.TYPE_WIDTH[t] for _, t in meta)


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--check", choices=["oracle", "invariants", "none"], default="invariants")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--morsel-rows", type=int, default=4_000_000)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write the last timed step's result as DIR/<name>.npy (float64)")
    return ap.parse_args(argv)


def main(args=None):
    args = args or parse()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(local, stream=stream.cuda_stream)

    g = tpcds.Q95Gen(args.sf, device=dev)
    blk = (g.n_orders + world - 1) // world
    lo, hi = min(g.n_orders, rank * blk), min(g.n_orders, (rank + 1) * blk)
    step = 2_000_000                                                             # orders per generator call (bounded temporaries)
    parts = [g.web_sales_of_orders(a, min(hi, a + step)) for a in range(lo, hi, step)]
    ws = {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
    del parts
    wr = g.web_returns_of_orders(lo, hi)
    dims = {"date": abi.Chunk([(tpcds.D_DATE_SK, g.date_keys(), None)], mem=abi.MEM_DEVICE),
            "addr": abi.Chunk([(tpcds.CA_ADDRESS_SK, g.address_keys(), None)], mem=abi.MEM_DEVICE),
            "site": abi.Chunk([(tpcds.WEB_SITE_SK, g.site_keys(), None)], mem=abi.MEM_DEVICE)}
    ws_chunk = tpcds.table_chunk(ws, tpcds.WS_COLS, mem=abi.MEM_DEVICE)
    wr_chunk = abi.Chunk([(tpcds.WS_ORDER, wr["wr_order_number"], None)], mem=abi.MEM_DEVICE)
    n_ws, n_wr = int(ws["ws_order_number"].numel()), int(wr["wr_order_number"].numel())
    torch.cuda.synchronize()

    def run_plan():
        keep = []
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        x_ws = gpu.Xchg(ctx, abi.make_part_desc([tpcds.WS_ORDER], world))
        ws_local, b1 = shuffle(x_ws, ws_chunk, dev, keep)
        x_wr = gpu.Xchg(ctx, abi.make_part_desc([tpcds.WS_ORDER], world))
        wr_local, b2 = shuffle(x_wr, wr_chunk, dev, keep)
        eng = tpcds.GpuEngine(gpu, ctx)
        res, st = tpcds.q95_local_plan(eng, ws_local, wr_local, dims, morsel_rows=args.morsel_rows, expected_orders=int(blk * 1.2) + 1024)
        e1.record(stream)
        dist.barrier()
        torch.cuda.synchronize()
        eng.close()
        x_ws.close()
        x_wr.close()
        st["bytes_sent"] = b1 + b2
        st["rows_local"] = ws_local.num_rows
        return res, st, e0.elapsed_time(e1)

    for _ in range(max(1, args.warmup)):
        res, st, ms = run_plan()
    times = []
    for _ in range(args.steps):
        res, st, ms = run_plan()
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        times.append(float(t[0]))
    ms_per_step = sum(times) / len(times)

    exp = g.expected(lo, hi) if args.check == "invariants" else (0, 0, 0)
    tot = torch.tensor(list(res) + list(exp) + [n_ws, n_wr, st["bytes_sent"], st["self_join_rows"], st["ws_wh_orders"], st["rows_aggregated"]],
                       dtype=torch.int64, device=dev)
    dist.all_reduce(tot)
    tot = [int(x) for x in tot.tolist()]
    checks = {}
    if args.check == "invariants":
        checks = {"equals_join_free_evaluation": tot[0:3] == tot[3:6]}
    if args.check == "oracle" and rank == 0:
        import numpy as np
        from oracle import oracle
        hg = tpcds.Q95Gen(args.sf)
        hws, hwr = hg.web_sales_of_orders(0, hg.n_orders), hg.web_returns_of_orders(0, hg.n_orders)
        hd = {"date": abi.Chunk([(tpcds.D_DATE_SK, hg.date_keys(), None)]), "addr": abi.Chunk([(tpcds.CA_ADDRESS_SK, hg.address_keys(), None)]),
              "site": abi.Chunk([(tpcds.WEB_SITE_SK, hg.site_keys(), None)])}
        ores, ost = tpcds.q95_local_plan(tpcds.OracleEngine(oracle), tpcds.table_chunk(hws, tpcds.WS_COLS),
                                         abi.Chunk([(tpcds.WS_ORDER, hwr["wr_order_number"], None)]), hd, morsel_rows=1_000_000)
        checks = {"bit_exact_vs_oracle": list(ores) == tot[0:3], "self_join_rows_equal": ost["self_join_rows"] == tot[9],
                  "ws_wh_orders_equal": ost["ws_wh_orders"] == tot[10]}
    if rank == 0:
        line = {"metric": "web_sales rows/sec for TPC-DS Q95 shape (one-to-many self join + IN-subqueries + COUNT DISTINCT, NCCL shuffle)",
                "value": tot[6] / (ms_per_step / 1000.0), "unit": "rows/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "int64 keys / int64 sums", "data": "synthetic",
                "config": {"workload": f"TPC-DS SF{args.sf:g} Q95 shape", "web_sales_rows": tot[6], "web_returns_rows": tot[7], "orders": g.n_orders,
                           "parallelism": f"hash-partitioned on ws_order_number over {world} GPUs", "morsel_rows": args.morsel_rows},
                "result": {"count_distinct_orders": tot[0], "sum_ext_ship_cost": tot[1], "sum_net_profit": tot[2]},
                "plan_rows": {"self_join_output": tot[9], "ws_wh_orders": tot[10], "rows_aggregated": tot[11]},
                "exchange_bytes": tot[8], "checks": checks, "check_mode": args.check}
        print(json.dumps(line))
        if args.dump_outputs:
            # the query's three numbers from the last timed step
            import numpy as np
            os.makedirs(args.dump_outputs, exist_ok=True)
            for nm, v in zip(("count_distinct_orders", "sum_ext_ship_cost", "sum_net_profit"), tot[0:3]):
                np.save(os.path.join(args.dump_outputs, nm + ".npy"), np.array([v], dtype=np.float64))
    ok = all(checks.values()) if checks else True
    flag = torch.tensor([0 if ok else 1], device=dev)
    dist.broadcast(flag, 0)
    return line if rank == 0 else None, int(flag[0]) == 0


if __name__ == "__main__":
    _, good = main()
    dist.destroy_process_group()
    sys.exit(0 if good else 1)
