"""The fused fragment (SSB Q4.1, SF100 dimensions) fed three ways, in one process, the variants alternating:
  (a) sr_fragment_push of contiguous page-locked 4M-row morsels, read in place over PCIe (sector-selective);
  (b) sr_fragment_push_chunks of the same rows as 4096-row chunks laid out chunk after chunk in one registered arena
      (sr_host_register), in lists of 4M rows: k_chunk_gather moves every read column in full;
  (c) the C++ operator path (starrocks_b200/host/bench/operator_e2e_bench) with --pool pinned against its default.
Prints one JSON line: ms per step, rows/s, the bytes that cross PCIe, the card and its power limit, and whether every
variant computed the same groups.
  python tools/frag_chunk_list_bench.py [--rows 600000000] [--steps 3] [--op-rows 200000000] [--dop 8]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from starrocks_b200 import abi, gpu, ssb  # noqa: E402
from starrocks_b200.rows import gpu_rows  # noqa: E402

MORSEL = 1 << 22
CHUNK = 4096


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--op-rows", type=int, default=200_000_000)
    ap.add_argument("--dop", type=int, default=8)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    sz = ssb.sizes(100.0)
    dims = ssb.gen_dims(100.0)
    gjoins, gkeep = ssb.build_dims(gpu, dims, ssb.dim_plans_q41(), ctx=ctx)
    n = a.rows
    names = ssb.Q41_FACT_COLS
    slots = [ssb.LO_SLOTS[nm] for nm in names]
    cols = bench.gen_lineorder_device(torch, dev, n, sz, ssb.SEED)
    # (a): one page-locked array per column
    host = {nm: torch.empty(n, dtype=torch.int32, pin_memory=True) for nm in names}
    for nm in names:
        host[nm].copy_(cols[nm])
    # (b): one registered arena, the 4096-row chunks one after another, each chunk's columns back to back
    arena = np.empty(n * 4 * len(names) + 4096, np.uint8)
    base = (-arena.ctypes.data) % 4096
    view = arena[base:base + n * 4 * len(names)]
    chunk_starts = list(range(0, n, CHUNK))
    for nm_k, nm in enumerate(names):
        h = host[nm].numpy()
        for lo in chunk_starts:
            hi = min(n, lo + CHUNK)
            off = lo * 4 * len(names) + nm_k * (hi - lo) * 4
            view[off:off + (hi - lo) * 4] = h[lo:hi].view(np.uint8)
    del cols
    torch.cuda.synchronize()
    ctx.host_register(view.ctypes.data, view.nbytes)
    ptr0 = view.ctypes.data

    def chunk_view(lo):
        hi = min(n, lo + CHUNK)
        return abi.Chunk([(s, ptr0 + lo * 4 * len(names) + k * (hi - lo) * 4, None, abi.TYPE_INT) for k, s in enumerate(slots)], num_rows=hi - lo,
                         mem=abi.MEM_HOST_PINNED)

    frag = gpu.Fragment(ctx, abi.ScanDesc(), gjoins, ssb.q41_agg_desc())
    # the lists are built once, outside the timed steps: the step times the library call, not the Python that builds views
    lists = []
    for lo in range(0, n, MORSEL):
        chunks = [chunk_view(c) for c in range(lo, min(n, lo + MORSEL), CHUNK)]
        lists.append((chunks, (abi.sr_chunk_view * len(chunks))(*[c.view for c in chunks])))
    morsels = [abi.Chunk([(s, host[nm][lo:min(n, lo + MORSEL)].data_ptr(), None, abi.TYPE_INT) for s, nm in zip(slots, names)],
                         num_rows=min(n, lo + MORSEL) - lo, mem=abi.MEM_HOST_PINNED) for lo in range(0, n, MORSEL)]

    def run(variant):
        frag.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(len(morsels)):
            if variant == "a":
                frag.push(morsels[k])
            else:
                ctx.check(gpu.lib().sr_fragment_push_chunks(frag.h, lists[k][1], len(lists[k][0])))
        passed = frag.rows_passed          # synchronises
        secs = time.perf_counter() - t0
        return secs, passed, sorted(map(tuple, gpu_rows(frag.agg.result())))

    out = {"card": card(), "rows": n, "morsel_rows": MORSEL, "chunk_rows": CHUNK}
    results = {"a": [], "b": []}
    answers = {}
    for v in ("a", "b"):
        run(v)                              # warm-up of both shapes
    for _ in range(a.steps):
        for v in ("a", "b"):
            secs, passed, rows = run(v)
            results[v].append(secs)
            answers.setdefault(v, (passed, rows))
            assert answers[v] == (passed, rows)
    for v, label in (("a", "push_contiguous_pinned_in_place"), ("b", "push_chunks_registered_pool")):
        best = min(results[v])
        out[label] = {"ms_per_step": [round(1e3 * s, 2) for s in results[v]], "rows_per_s_best": n / best,
                      "pcie_bytes": None if v == "a" else n * 4 * len(names)}
    out["push_contiguous_pinned_in_place"]["pcie_bytes_note"] = "sector-selective in-place reads: at most the offered bytes"
    out["offered_bytes"] = n * 4 * len(names)
    out["a_equals_b"] = answers["a"] == answers["b"]
    frag.close()
    ctx.sync()
    ctx.host_unregister(view.ctypes.data)
    # (c): the operator path, default pageable chunks against chunks in a registered pool
    binary = os.path.join(ROOT, "starrocks_b200", "host", "bench", "operator_e2e_bench")
    ops = {}
    for rep in range(2):
        for pool in ("pageable", "pinned"):
            r = subprocess.run([binary, str(a.op_rows), str(a.dop), str(MORSEL), "--pool", pool], capture_output=True, text=True, timeout=3600)
            if r.returncode != 0:
                raise SystemExit(f"operator_e2e_bench --pool {pool} failed: {r.stdout}{r.stderr}")
            line = json.loads(r.stdout.strip().splitlines()[-1])
            ops.setdefault(pool, []).append({k: line[k] for k in ("seconds", "rows_per_s", "groups", "matches_row_at_a_time_evaluation",
                                                                   "h2d_bytes_offered", "forwarded_chunks", "fragment_batches")})
    out["operator_api"] = {"rows": a.op_rows, "dop": a.dop, **ops}
    out["operator_outputs_identical"] = all(x["matches_row_at_a_time_evaluation"] and x["groups"] == 35 for v in ops.values() for x in v)
    out["card_after"] = card()
    print(json.dumps(out))
    for j, _, _ in gjoins:
        j.close()
    for item in gkeep:
        item[0].close()
    ctx.close()


if __name__ == "__main__":
    main()
