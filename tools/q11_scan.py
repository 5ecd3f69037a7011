"""SSB Q1.1 (flat form: scan + 3 predicates + SUM(lo_extendedprice * lo_discount), no join) on one H100 -- BASELINE.json
config 0 at SF100 size, through (a) the fused fragment and (b) the separate operators (sr_scan_filter -> sr_agg_push).

    python tools/q11_scan.py [--rows 600000000]

Algorithmic bytes (SURVEY.md 8d): 4 int32 columns = 16 B/row.  Prints one JSON line; the result is checked against a
torch restatement on the same columns (and against the oracle at small sizes in tests/test_gpu_parity.py).
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, ssb  # noqa: E402


def timed(fn, stream, reps):
    fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    n = args.rows
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    g = torch.Generator(device=dev)
    g.manual_seed(ssb.SEED)
    cols = {
        "lo_orderdate": (19920101 + torch.randint(0, 7, (n,), device=dev, generator=g, dtype=torch.int32) * 10000
                         + torch.randint(0, 12, (n,), device=dev, generator=g, dtype=torch.int32) * 100
                         + torch.randint(0, 28, (n,), device=dev, generator=g, dtype=torch.int32)),
        "lo_discount": torch.randint(0, 11, (n,), device=dev, generator=g, dtype=torch.int32),
        "lo_quantity": torch.randint(1, 51, (n,), device=dev, generator=g, dtype=torch.int32),
        "lo_extendedprice": torch.randint(90_000, 10_494_951, (n,), device=dev, generator=g, dtype=torch.int32),
    }
    torch.cuda.synchronize()
    chunk = ssb.fact_chunk(cols, ssb.Q11_FACT_COLS, mem=abi.MEM_DEVICE)
    sd = abi.ScanDesc(preds=ssb.q11_scan_preds())
    frag = gpu.Fragment(ctx, sd, [], ssb.q11_agg_desc())

    def run_fused():
        frag.reset()
        frag.push(chunk)
        return frag.agg.result()

    ms_fused, res = timed(run_fused, stream, args.reps)
    passes = frag.last_pass_ms()
    got = int(res[0][2][0])
    m = ((cols["lo_orderdate"] >= 19930101) & (cols["lo_orderdate"] <= 19931231) & (cols["lo_discount"] >= 1)
         & (cols["lo_discount"] <= 3) & (cols["lo_quantity"] < 25))
    exp = int((cols["lo_extendedprice"][m].to(torch.int64) * cols["lo_discount"][m].to(torch.int64)).sum().item())
    passed = int(m.sum().item())
    del m

    # separate operators: filter materialises the two surviving columns, the aggregate consumes them
    sd2 = abi.ScanDesc(preds=ssb.q11_scan_preds(), out_slots=[ssb.LO_SLOTS["lo_extendedprice"], ssb.LO_SLOTS["lo_discount"]])
    scan = gpu.Scan(ctx, sd2)
    agg = gpu.Agg(ctx, ssb.q11_agg_desc())

    def run_ops():
        agg.reset()
        out = scan.filter(chunk)
        agg.push(abi.Chunk([(out.cols[k].slot_id, out.cols[k].data, out.cols[k].nulls, out.cols[k].type) for k in range(out.num_cols)],
                           num_rows=out.num_rows, mem=abi.MEM_DEVICE))
        return agg.result()

    ms_ops, res2 = timed(run_ops, stream, args.reps)
    got2 = int(res2[0][2][0])
    line = {"query": "SSB Q1.1 (flat)", "rows": n, "rows_passed": passed, "algorithmic_bytes": n * 16,
            "fused_fragment": {"ms": ms_fused, "rows_per_s": n / ms_fused * 1e3, "algorithmic_gbs": n * 16 / ms_fused / 1e6, "pass_ms": passes,
                               "plan": frag.plan()},
            "separate_operators": {"ms": ms_ops, "rows_per_s": n / ms_ops * 1e3, "algorithmic_gbs": n * 16 / ms_ops / 1e6},
            "result_matches_torch_restatement": got == exp and got2 == exp, "sum": got}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
