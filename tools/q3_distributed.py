"""TPC-H Q3 across the N GPUs of one box with an NCCL hash shuffle (BASELINE.json config 3: SF300 on 8 GPUs; SURVEY.md 8e).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/q3_distributed.py --sf 300 [--check oracle|invariants|none]          (also: bench.py --workload q3)

Plan per rank (one process per GPU; the fragment instances of the reference's distributed plan, fe .../tpch/q3.sql):
    customer (replicated, broadcast join)     -> J1
    orders shard   -- o_orderdate < D, SEMI J1 -> HASH_PARTITIONED exchange on o_orderkey  -> local build of J2
    lineitem shard -- l_shipdate  > D          -> HASH_PARTITIONED exchange on l_orderkey  -> probe J2 + aggregate
The exchange is the reference's ExchangeSink hash step (FNV + ReduceOp, exchange_sink_operator.cpp:586-637, shuffler.h:72-89)
done by sr_xchg_partition on the device, followed by one grouped NCCL send/recv of all columns (starrocks_b200.distributed).
The group key contains the shuffle key, so the groups of different ranks are disjoint after the shuffle: the aggregate is
single-phase, the result is the union of the per-rank results.

No rank ever holds a whole table: every rank generates ITS shard on its own device from the counter-based generator
(tpch.HashGen) -- the orders with index = rank (mod N), the line items of the orders in block rank, i.e. of orders that live
on other ranks.  Checks: `oracle` (small SF): the union is compared bit for bit with the CPU oracle run on the host-generated
whole tables; `invariants` (any SF): number of groups and the exact 128-bit total of the revenue column against a join-free
evaluation of the query over the generator functions, computed per rank and all-reduced.
Rank 0 prints one JSON line (bench.py format).
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, tpch  # noqa: E402
from starrocks_b200.distributed import device_view, exchange_partitions  # noqa: E402


def shuffle(xchg, chunk, dev, keep):
    """partition `chunk` (device) by the xchg's key and exchange -> (received chunk, bytes sent to other ranks)"""
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
    ap.add_argument("--sf", type=float, default=1.0)
    ap.add_argument("--check", choices=["oracle", "invariants", "none"], default="invariants")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
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

    # ---- this rank's shards, generated on its own device ----
    g = tpch.HashGen(args.sf, device=dev)
    blk = (g.no + world - 1) // world
    lo, hi = min(g.no, rank * blk), min(g.no, (rank + 1) * blk)
    customer = g.customer()                                                      # replicated (broadcast join)
    orders = g.orders(torch.arange(rank, g.no, world, dtype=torch.int64, device=dev))
    lineitem = {}
    step = 16_000_000                                                            # bounded temporaries of the generator
    parts = [g.lineitem_of_orders(a, min(hi, a + step)) for a in range(lo, hi, step)]
    for k in parts[0]:
        lineitem[k] = torch.cat([p[k] for p in parts])
    del parts
    n_li, n_ord = int(lineitem["l_orderkey"].numel()), int(orders["o_orderkey"].numel())
    torch.cuda.synchronize()

    cust_scan, j1d, ord_scan, j2d, _ = tpch.q3_descs()
    li_scan = abi.ScanDesc(preds=[abi.make_pred(tpch.L_SHIPDATE, abi.PRED_GT, tpch.CUTOFF)],
                           out_slots=[tpch.L_ORDERKEY, tpch.L_EXTENDEDPRICE, tpch.L_DISCOUNT])
    payload = [tpch.O_ORDERDATE, tpch.O_SHIPPRIORITY]
    cust_chunk = tpch.table_chunk(customer, tpch.CUSTOMER_COLS, mem=abi.MEM_DEVICE)
    ord_chunk = tpch.table_chunk(orders, tpch.ORDERS_COLS, mem=abi.MEM_DEVICE)
    li_chunk = tpch.table_chunk(lineitem, tpch.LINEITEM_COLS, mem=abi.MEM_DEVICE)
    expected_groups = int(g.no * 0.1 / world * 1.3) + 1024

    def run_plan(want_result):
        """one execution of the plan with fresh operator handles; -> (result, stats, device ms, phase seconds)"""
        keep = []
        phases = {}
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        mark = [time.perf_counter()]
        e0.record(stream)

        def phase(name):
            if not want_result:        # the timed runs are not interrupted by host synchronisations of their own
                return
            torch.cuda.synchronize()
            now = time.perf_counter()
            phases[name] = phases.get(name, 0.0) + now - mark[0]
            mark[0] = now

        # --- build side ---
        s1 = gpu.Scan(ctx, cust_scan)
        j1 = gpu.Join(ctx, j1d)
        j1.append_build(tpch._dev_chunk(s1.filter(cust_chunk)))
        j1.build_finish()
        phase("customer scan + J1 build")
        s2 = gpu.Scan(ctx, ord_scan)
        o_j = tpch._dev_chunk(j1.probe(tpch._dev_chunk(s2.filter(ord_chunk))))
        phase("orders scan + semi-join probe")
        x_ord = gpu.Xchg(ctx, abi.make_part_desc([tpch.O_ORDERKEY], world))
        o_local, bytes_o = shuffle(x_ord, o_j, dev, keep)
        phase("orders partition + all-to-all")
        j2 = gpu.Join(ctx, j2d)
        j2.append_build(o_local)
        j2.build_finish()
        phase("J2 build")
        # --- probe side ---
        s3 = gpu.Scan(ctx, li_scan)
        l_f = tpch._dev_chunk(s3.filter(li_chunk))
        phase("lineitem scan")
        x_li = gpu.Xchg(ctx, abi.make_part_desc([tpch.L_ORDERKEY], world))
        l_local, bytes_l = shuffle(x_li, l_f, dev, keep)
        phase("lineitem partition + all-to-all")
        frag = gpu.Fragment(ctx, abi.ScanDesc(), [(j2, tpch.L_ORDERKEY, payload)], tpch.q3_agg_desc(expected_groups))
        if l_local.num_rows > 0:
            frag.push(l_local)
        frag.agg.finish()
        out = frag.agg.pull(mem=abi.MEM_DEVICE)
        groups = int(out.num_rows)
        phase("probe J2 + aggregate + result")
        e1.record(stream)
        dist.barrier()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        res = None
        if want_result:   # copy the (small) result out before the handles go away
            res = {"n": groups, "cols": [device_view(out.cols[k].data, groups * (2 if abi.TYPE_WIDTH[out.cols[k].type] == 16 else 1),
                                                     8 if abi.TYPE_WIDTH[out.cols[k].type] >= 8 else 4, dev).clone() for k in range(out.num_cols)],
                   "types": [out.cols[k].type for k in range(out.num_cols)], "host": gpu.chunk_out_to_host(ctx, out) if args.check == "oracle" else None}
        st = (bytes_o + bytes_l, j2.info().build_rows, l_local.num_rows, groups)
        frag.close()
        for h in (s1, s2, s3, j1, j2, x_ord, x_li):
            h.close()
        return res, st, ms, phases

    for _ in range(max(1, args.warmup)):
        res, st, ms, phases = run_plan(True)         # warm-up: NCCL channels, allocator, kernel modules; also the checked result
    times = []
    for i in range(args.steps):
        r, st, ms, _ = run_plan(i == args.steps - 1)   # the last timed step's result is checked (the copy is outside its timing)
        res = r if r is not None else res
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        times.append(float(t[0]))
    ms_per_step = sum(times) / len(times)
    bytes_total, j2_rows, probe_rows, groups = st

    # ---- checks ----
    checks = {}
    rev = res["cols"][3].view(-1, 2)                                           # decimal128 sums as (lo, hi) int64 pairs
    my_total = int(rev[:, 0].sum().item()) + (int(rev[:, 1].sum().item()) << 64)   # every group's sum is far below 2^63: exact
    stats = torch.tensor([groups, bytes_total, j2_rows, probe_rows, n_li, n_ord], dtype=torch.int64, device=dev)
    dist.all_reduce(stats)
    totals = [None] * world
    dist.all_gather_object(totals, my_total)
    if args.check == "invariants":
        # the query without joins: a line item counts iff its ship date and ITS ORDER's generator-defined date / customer
        # segment qualify; groups = orders with at least one such line item
        oi = torch.arange(lo, hi, dtype=torch.int64, device=dev)
        per = 1 + g._h(4, oi) % 7
        rep = torch.repeat_interleave(torch.arange(hi - lo, dtype=torch.int64, device=dev), per)
        ok = g.order_qualifies(oi)[rep] & (lineitem["l_shipdate"] > tpch.CUTOFF)
        val = lineitem["l_extendedprice"] * (100 - lineitem["l_discount"])
        exp_total = int(val[ok].sum().item())                                  # < 2^63 per rank (values < 2^30, < 2^28 rows)
        hit = torch.zeros(hi - lo, dtype=torch.bool, device=dev)
        hit[rep[ok]] = True
        exp = torch.tensor([int(hit.sum().item())], dtype=torch.int64, device=dev)
        dist.all_reduce(exp)
        exp_totals = [None] * world
        dist.all_gather_object(exp_totals, exp_total)
        checks = {"groups_equal_join_free_count": int(exp[0]) == int(stats[0]), "revenue_total_equals_join_free_total": sum(exp_totals) == sum(totals)}
    gathered = [None] * world if rank == 0 else None
    if args.check == "oracle":
        from starrocks_b200.rows import gpu_rows
        dist.gather_object(gpu_rows(res["host"]), gathered, dst=0)
    if rank == 0:
        n_li_total = int(stats[4])
        line = {"metric": "lineitem rows/sec for TPC-H Q3 (hash join + aggregate, NCCL shuffle)", "value": n_li_total / (ms_per_step / 1000.0), "unit": "rows/s",
                "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong",
                "vs_baseline": None, "dtype": "int32 keys / decimal64 inputs / decimal128 sums", "data": "synthetic",
                "config": {"workload": f"TPC-H SF{args.sf:g} Q3 (lineitem JOIN orders JOIN customer) hash join + aggregate, NCCL shuffle",
                           "lineitem_rows": n_li_total, "orders_rows": int(stats[5]), "customer_rows": g.nc,
                           "parallelism": f"dp{world}: orders and lineitem sharded and HASH_PARTITIONED on the order key (FNV + ReduceOp), customer replicated"},
                "groups": int(stats[0]), "shuffled_bytes_per_step": int(stats[1]), "j2_build_rows": int(stats[2]), "probe_rows_after_shuffle": int(stats[3]),
                "algorithmic_bytes": n_li_total * 24 + int(stats[5]) * 16 + g.nc * 8,
                "phase_ms_rank0_warmup_run": {k: round(v * 1e3, 3) for k, v in phases.items()}, "all_ms": times, "checks": checks}
        if args.check == "oracle":
            from oracle import oracle
            from starrocks_b200.rows import oracle_rows
            t = tpch.gen_tables_hashed(args.sf)
            oj2, okeep = tpch.q3_build_oracle(oracle, t)
            _, _, _, _, full_scan = tpch.q3_descs()
            ores, _ = oracle.fragment_run(full_scan, [(oj2, tpch.L_ORDERKEY, payload)], tpch.q3_agg_desc(),
                                          tpch.table_chunk(t["lineitem"], tpch.LINEITEM_COLS), num_threads=os.cpu_count() or 1)
            union = sorted(r for part in gathered for r in part)
            exp = oracle_rows(ores)
            line["checks"] = {"bit_exact_vs_oracle": union == exp, "oracle_groups": len(exp)}
        print(json.dumps(line), flush=True)
        if args.dump_outputs:
            # the group count and the exact revenue total, split into 32-bit halves so that float64 holds them exactly
            import numpy as np
            os.makedirs(args.dump_outputs, exist_ok=True)
            total = sum(totals)
            for nm, v in (("groups", int(stats[0])), ("revenue_total_hi32", total >> 32), ("revenue_total_lo32", total & 0xFFFFFFFF)):
                np.save(os.path.join(args.dump_outputs, nm + ".npy"), np.array([v], dtype=np.float64))
    dist.barrier()
    ctx.close()
    return 0


if __name__ == "__main__":
    main()
    if dist.is_initialized():
        dist.destroy_process_group()
