"""Time of sr_xchg_partition (hash + channel histogram, scan, stable scatter, gather of every column) on HBM-resident
columns, one GPU:

    python tools/xchg_partition_bench.py [--rows 50000000] [--channels 8 256] [--reps 5]

Four columns: the INT partition key, a BIGINT, a DOUBLE and a DECIMAL128 payload (the 16-byte gather), FNV / MULHI.
Prints one JSON line: the card, its power limit, and per channel count the best and median milliseconds of `reps` calls
(each call ends in a device synchronise: sr_xchg_partition returns the channel offsets on the host) and the algorithmic
GB/s (input columns read once, output columns written once).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--channels", type=int, nargs="+", default=[8, 256])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    n = args.rows
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    key = torch.randint(-(1 << 31), (1 << 31) - 1, (n,), device=dev, generator=g, dtype=torch.int32)
    big = torch.randint(-(1 << 62), 1 << 62, (n,), device=dev, generator=g, dtype=torch.int64)
    dbl = torch.randn(n, device=dev, generator=g, dtype=torch.float64)
    dec = torch.randint(-(1 << 62), 1 << 62, (2 * n,), device=dev, generator=g, dtype=torch.int64)
    torch.cuda.synchronize()
    chunk = abi.Chunk([(0, key, None), (1, big, None), (2, dbl, None), (3, dec.data_ptr(), None, abi.TYPE_DECIMAL128)],
                      num_rows=n, mem=abi.MEM_DEVICE)
    moved = n * (4 + 8 + 8 + 16)
    ctx = gpu.Context(0)
    res = {"card": card(), "rows": n, "columns": "INT key, BIGINT, DOUBLE, DECIMAL128", "library": gpu.LIB_PATH, "channels": {}}
    for nch in args.channels:
        x = gpu.Xchg(ctx, abi.make_part_desc([0], nch))
        try:
            x.partition(chunk)                       # warm-up: buffers allocated, module loaded
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                x.partition(chunk)                   # synchronises before it returns
                times.append((time.perf_counter() - t0) * 1e3)
        finally:
            x.close()
        best = min(times)
        res["channels"][str(nch)] = {"best_ms": round(best, 3), "median_ms": round(float(np.median(times)), 3),
                                     "algorithmic_GBps": round(2 * moved / best / 1e6, 1)}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
