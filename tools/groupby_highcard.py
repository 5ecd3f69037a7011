"""High-cardinality group-by on one H100 (BASELINE.json config 5 at half size, which fits 80 GB; SURVEY.md section 8d):
5e8 rows, key int64 = splitmix64(i) mod 5e7, value int64 U[0, 1000]; SELECT key, SUM(v), COUNT(*) GROUP BY key.

    python tools/groupby_highcard.py [--rows 500000000] [--keys 50000000] [--morsel 100000000]

The table is the sr_agg hash table (open addressing, 64-bit CAS claim, SoA accumulators); rows are pushed in morsels
through the C-ABI (sr_agg_push) from HBM-resident columns.  Size-independent checks (the CPU oracle would need minutes
at this size; parity against it is pinned at small sizes in tests/test_gpu_parity.py):
  * sum over groups of COUNT(*) == rows,  sum over groups of SUM(v) == sum(v),
  * number of groups == number of distinct keys (counted independently with torch.unique on a sample-free pass).
Prints one JSON line with rows/s and the algorithmic bandwidth (16 B/row in + 24 B/group out, SURVEY 8d).
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu  # noqa: E402
from starrocks_b200.distributed import device_view  # noqa: E402


def splitmix64(x):
    """torch int64 implementation (wrapping arithmetic) of splitmix64's output function"""
    x = x + (-7046029254386353131)          # 0x9E3779B97F4A7C15 as signed
    z = x
    z = (z ^ ((z >> 30) & ((1 << 34) - 1))) * (-4658895280553007687)   # 0xBF58476D1CE4E5B9
    z = (z ^ ((z >> 27) & ((1 << 37) - 1))) * (-7723592293110705685)   # 0x94D049BB133111EB
    return z ^ ((z >> 31) & ((1 << 33) - 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--keys", type=int, default=50_000_000)
    ap.add_argument("--morsel", type=int, default=500_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    n, nk = args.rows, args.keys
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    vals = torch.empty(n, dtype=torch.int64, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(20240921)
    step = 50_000_000
    for lo in range(0, n, step):
        hi = min(n, lo + step)
        i = torch.arange(lo, hi, dtype=torch.int64, device=dev)
        h = splitmix64(i)
        keys[lo:hi] = torch.remainder(h & ((1 << 62) - 1), nk)
        vals[lo:hi] = torch.randint(0, 1001, (hi - lo,), dtype=torch.int64, device=dev, generator=g)
        del i, h
    total_v = int(vals.sum().item())
    torch.cuda.synchronize()

    d = abi.make_agg_desc([0], [abi.TYPE_BIGINT], fns=[(abi.AGG_SUM, abi.TYPE_BIGINT, 10, [("col", 1)]), (abi.AGG_COUNT_STAR, 0, 11, None)],
                          expected_groups=nk)
    agg = gpu.Agg(ctx, d)
    times = []
    for rep in range(args.reps + 1):
        agg.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for lo in range(0, n, args.morsel):
            hi = min(n, lo + args.morsel)
            agg.push(abi.Chunk([(0, keys[lo:hi], None, abi.TYPE_BIGINT), (1, vals[lo:hi], None, abi.TYPE_BIGINT)], mem=abi.MEM_DEVICE))
        agg.finish()
        groups = agg.num_groups          # materialises the output columns on the device
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if rep > 0:
            times.append(dt)
    out = agg.pull(mem=abi.MEM_DEVICE)
    gk = device_view(out.cols[0].data, out.num_rows, 8, dev)
    gs = device_view(out.cols[1].data, out.num_rows, 8, dev)
    gc = device_view(out.cols[2].data, out.num_rows, 8, dev)
    checks = {"count_sum_equals_rows": int(gc.sum().item()) == n, "sum_sum_equals_total": int(gs.sum().item()) == total_v,
              "groups": int(groups), "group_keys_unique": int(torch.unique(gk).numel()) == int(groups)}
    distinct = 0
    # independent distinct count: per-key-range unique (bounded memory)
    present = torch.zeros(nk, dtype=torch.bool, device=dev)
    for lo in range(0, n, step):
        present[keys[lo:min(n, lo + step)]] = True
    distinct = int(present.sum().item())
    checks["groups_equal_distinct_keys"] = distinct == int(groups)
    best = min(times)
    line = {"workload": f"group-by {n} rows, {nk} distinct int64 keys, SUM + COUNT", "rows": n, "seconds": best,
            "rows_per_s": n / best, "algorithmic_bytes": n * 16 + int(groups) * 24,
            "algorithmic_gbs": (n * 16 + int(groups) * 24) / best / 1e9, "all_times": times, "checks": checks}
    print(json.dumps(line))
    agg.close()


if __name__ == "__main__":
    main()
