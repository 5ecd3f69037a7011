"""The fused fragment against the per-operator chain on SSB Q4.1 shapes with LEFT OUTER and LEFT ANTI joins, one H100:

    python tools/frag_join_kinds.py [--sf 100] [--steps 5] [--warmup 2] [--out results.json]

Three variants of SSB Q4.1 (GROUP BY d_year, c_nation; SUM(lo_revenue), SUM(lo_supplycost)):
  q41        as is: four INNER joins;
  q41_outer  the customer join as LEFT OUTER: fact rows whose customer is not in AMERICA (80 %) keep their row and
             group under a NULL c_nation;
  q41_anti   plus a LEFT ANTI join on lo_partkey against an exclusion set of parts (every tenth part key).
Each runs on the same HBM-resident lineorder shard two ways:
  fused      sr_fragment_push (scan -> probe x N -> aggregate in one set of passes), then sink_finish + pull;
  operators  sr_join_probe per join, each materialising its output chunk on the device, then sr_agg_push, sink_finish
             + pull -- the path such a plan takes when the fragment refuses it.
Both results are pulled to the host and must be equal group for group (integer sums: exactly).  Times are device
events around one whole step after warm-up, best and median of --steps; the card's name and power limit are printed
with them.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, ssb  # noqa: E402

S = ssb.LO_SLOTS
EXCL_PARTKEY = 60   # build key slot of the exclusion set


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def gen_lineorder(dev, n, sz, seed):
    """the Q4.1 fact columns on the device (distributions of ssb.gen_lineorder)"""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    ri = lambda lo, hi: torch.randint(lo, hi, (n,), dtype=torch.int32, device=dev, generator=g)  # noqa: E731
    datekey = torch.from_numpy(ssb.gen_dates()["d_datekey"]).to(dev)
    return {"lo_orderdate": datekey[torch.randint(0, datekey.numel(), (n,), device=dev, generator=g)].contiguous(),
            "lo_custkey": ri(1, sz["customer"] + 1), "lo_suppkey": ri(1, sz["supplier"] + 1), "lo_partkey": ri(1, sz["part"] + 1),
            "lo_revenue": ri(81_000, 10_400_001), "lo_supplycost": ri(54_000, 125_001)}


def variant_joins(name, dims):
    """(join type, table, build columns, key slot, probe slot, payload slots, dimension predicates) in probe order"""
    plans = {p[0]: p for p in ssb.dim_plans_q41()}
    out = []
    for table in ("supplier", "customer", "part", "dates"):
        _, key_col, key_slot, probe_slot, payload, preds, slotmap = plans[table]
        jt = abi.JOIN_LEFT_OUTER if (name == "q41_outer" and table == "customer") else abi.JOIN_INNER
        cols = [(slotmap[c], dims[table][c]) for c in dims[table]]
        out.append((jt, cols, key_slot, probe_slot, [s for _, s in payload], preds))
        if name == "q41_anti" and table == "part":
            excl = dims["part"]["p_partkey"][dims["part"]["p_partkey"] % 10 == 3]
            out.append((abi.JOIN_LEFT_ANTI, [(EXCL_PARTKEY, excl)], EXCL_PARTKEY, S["lo_partkey"], [], []))
    return out


def build(ctx, joins):
    """dimension scan + filter on the device, then the join build.  Each join's probe_out lists the columns the joins
    after it and the aggregate read, so the same built joins serve the fragment and the per-operator chain."""
    need = [S["lo_revenue"], S["lo_supplycost"], ssb.D_YEAR, ssb.C_NATION]
    later = [[p for _, _, _, p, _, _ in joins[k + 1:]] for k in range(len(joins))]
    built, keep = [], []
    avail = [S[c] for c in ssb.Q41_FACT_COLS]
    for k, (jt, cols, key_slot, probe_slot, pays, preds) in enumerate(joins):
        chunk = abi.Chunk([(s, d, None, abi.TYPE_INT) for s, d in cols])
        scan = gpu.Scan(ctx, abi.ScanDesc(preds=preds, out_slots=[key_slot] + pays))
        o = scan.filter(chunk)
        bchunk = abi.Chunk([(o.cols[q].slot_id, o.cols[q].data, o.cols[q].nulls, o.cols[q].type) for q in range(o.num_cols)],
                           num_rows=o.num_rows, mem=abi.MEM_DEVICE)
        probe_out = [s for s in avail if s in need or s in later[k]]
        j = gpu.Join(ctx, abi.make_join_desc(jt, [key_slot], [probe_slot], [abi.TYPE_INT], build_out=pays, probe_out=probe_out,
                                             probe_out_types=[abi.TYPE_INT] * len(probe_out)))
        j.append_build(bchunk)
        j.build_finish()
        built.append((j, probe_slot, pays))
        keep.append((scan, chunk, bchunk))
        avail = probe_out + pays
    return built, keep


def agg_desc():
    return abi.make_agg_desc([ssb.D_YEAR, ssb.C_NATION], [abi.TYPE_INT, abi.TYPE_INT],
                             fns=[(abi.AGG_SUM, abi.TYPE_BIGINT, ssb.OUT_SUM_REVENUE, [("col", S["lo_revenue"])]),
                                  (abi.AGG_SUM, abi.TYPE_BIGINT, ssb.OUT_SUM_SUPPLYCOST, [("col", S["lo_supplycost"])])],
                             ranges=[(1992, 1998), (0, 24)], group_nullable=[False, True])


def groups(res):
    """(slot, type, data, nulls) columns of an aggregate result -> {(d_year, c_nation or None): (revenue, supplycost)}"""
    (_, _, y, yn), (_, _, nat, nn), (_, _, rev, _), (_, _, cost, _) = res
    nat = [None if nn is not None and nn[i] else int(nat[i]) for i in range(len(nat))]
    return {(int(y[i]), nat[i]): (int(rev[i]), int(cost[i])) for i in range(len(y))}


def timed(fn, stream, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return out, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--variants", default="q41,q41_outer,q41_anti")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frag_join_kinds.py: no CUDA device")
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    sz = ssb.sizes(args.sf)
    n = sz["lineorder"]
    dims = ssb.gen_dims(args.sf)
    cols = gen_lineorder(dev, n, sz, ssb.SEED)
    torch.cuda.synchronize()
    fact = ssb.fact_chunk(cols, ssb.Q41_FACT_COLS, mem=abi.MEM_DEVICE)
    report = {"card": card(), "sf": args.sf, "rows": n, "steps": args.steps, "warmup": args.warmup, "variants": {}}
    print(f"card: {report['card']}  SSB SF{args.sf:g}: {n} lineorder rows in HBM, {args.steps} timed steps after {args.warmup} warm-up")
    for name in args.variants.split(","):
        joins, keep = build(ctx, variant_joins(name, dims))
        frag = gpu.Fragment(ctx, abi.ScanDesc(), joins, agg_desc())
        chain_agg = gpu.Agg(ctx, agg_desc())

        def fused():
            frag.reset()
            frag.push(fact)
            frag.agg.finish()
            return gpu.chunk_out_to_host(ctx, frag.agg.pull(mem=abi.MEM_HOST))

        def operators():
            chunk = fact
            for j, _, _ in joins:
                chunk = gpu.chunk_out_as_view(j.probe(chunk))
            chain_agg.reset()
            chain_agg.push(chunk)
            chain_agg.finish()
            return gpu.chunk_out_to_host(ctx, chain_agg.pull(mem=abi.MEM_HOST))

        fres, fms = timed(fused, stream, args.steps, args.warmup)
        plan = frag.plan()
        passed = frag.rows_passed
        ores, oms = timed(operators, stream, args.steps, args.warmup)
        fg, og = groups(fres), groups(ores)
        equal = fg == og
        r = {"fused_ms": {"best": min(fms), "median": float(np.median(fms))}, "operators_ms": {"best": min(oms), "median": float(np.median(oms))},
             "speedup_median": float(np.median(oms) / np.median(fms)), "groups": len(fg), "rows_passed": passed, "equal": equal,
             "plan": {k: plan[k] for k in ("mode", "order", "pass_rate", "num_stream_joins", "num_gather_passes", "final_pass")}}
        report["variants"][name] = r
        print(f"{name:10s} fused {r['fused_ms']['median']:8.2f} ms (best {r['fused_ms']['best']:.2f})  operators "
              f"{r['operators_ms']['median']:8.2f} ms (best {r['operators_ms']['best']:.2f})  x{r['speedup_median']:.2f}  "
              f"{len(fg)} groups, {passed} rows passed, outputs {'equal' if equal else 'DIFFER'}  plan {r['plan']}")
        frag.close()
        chain_agg.close()
        for j, _, _ in joins:
            j.close()
        del keep
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)
    if not all(v["equal"] for v in report["variants"].values()):
        raise SystemExit("frag_join_kinds.py: the fused fragment and the per-operator chain disagree")


if __name__ == "__main__":
    main()
