"""Segment page decode on the device (SURVEY.md 8f-4): throughput of sr_pages_decode on SSB-shaped key columns.

    python tools/page_decode_bench.py [--rows 50000000] [--page-rows 65536] [--encoding for|bitshuffle|both|dict|nulls|rle]

Encodes synthetic lineorder key columns on the host -- frame-of-reference pages with the (reference-pinned) oracle encoder,
BIT_SHUFFLE pages (bitshuffle + LZ4, StarRocks' default for these types) with the CPU codec in bshuf_oracle -- then times
the decode of the resident pages (device memory) and of pages in page-locked host memory (the decode is the PCIe transfer:
only the encoded bytes cross the bus), and checks every decoded column against the raw values.  Prints one JSON line.

--encoding dict: low-cardinality string columns (7, 25 and 256 words, codes drawn uniformly) written as dictionary data
pages (mode word + bitshuffle page of int32 codes) and decoded into global ids through a per-segment table, timed next to
BIT_SHUFFLE pages of the same codes decoded as plain int32 -- the difference is the mode word and the translation.

--encoding nulls: the null maps of nullable columns (0 %, 0.1 %, 1 %, 10 %, 50 % random NULLs and runs of ~1000, as
BITSHUFFLE_NULL and RLE_NULL maps; a page without NULL has no map) decoded by sr_null_maps_decode from device and from
page-locked host memory, timed next to the H2D copy of the decoded uint8 null column from page-locked memory -- what a
caller that decodes the maps on the CPU moves instead.

--encoding rle: BOOLEAN columns as RLE pages -- random, runs of ~5000, and alternating runs of 8 (the worst case of the
serial run-header walk: one header per two bytes of page).
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bshuf_oracle  # noqa: E402  (encoders only: test infrastructure building the input)
from oracle import oracle  # noqa: E402
from starrocks_b200 import abi, gpu  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--page-rows", type=int, default=65_536)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--repeat", type=int, default=8, help="decode the encoded pages this many times over into one column (amortises the per-call costs without more host encoding)")
    ap.add_argument("--encoding", choices=["for", "bitshuffle", "both", "dict", "nulls", "rle"], default="for")
    args = ap.parse_args()
    if args.encoding == "dict":
        return dict_bench(args)
    if args.encoding in ("nulls", "rle"):
        return bool_bench(args)
    n = args.rows
    rng = np.random.default_rng(1)
    cols = {"lo_custkey (22 bits)": rng.integers(1, 3_000_000, n, dtype=np.int32), "lo_suppkey (18 bits)": rng.integers(1, 200_000, n, dtype=np.int32),
            "lo_orderdate (sorted runs)": np.sort(rng.integers(19920101, 19981231, (n + 4095) // 4096 * 4096, dtype=np.int32).reshape(-1, 4096), axis=1).reshape(-1)[:n].copy(),
            "lo_revenue int64 (24 bits)": rng.integers(1, 10_000_000, n, dtype=np.int64)}
    ctx = gpu.Context(0)
    dec = gpu.PageDecoder(ctx)
    encodings = {"for": (abi.PAGE_FOR, oracle.for_encode), "bitshuffle": (abi.PAGE_BITSHUFFLE, bshuf_oracle.bitshuffle_encode)}
    res = []
    for (name, v), enc in ((c, e) for c in cols.items() for e in (["for", "bitshuffle"] if args.encoding == "both" else [args.encoding])):
        code, encode = encodings[enc]
        t0 = time.perf_counter()
        pages = [encode(v[lo:lo + args.page_rows]) for lo in range(0, n, args.page_rows)]
        enc_s = time.perf_counter() - t0
        total = sum(len(p) for p in pages)
        typ = abi.TYPE_INT if v.dtype == np.int32 else abi.TYPE_BIGINT
        R = args.repeat
        out = torch.empty(n * R, dtype=torch.int32 if v.dtype == np.int32 else torch.int64, device="cuda")
        blob = torch.from_numpy(np.concatenate([np.pad(p, (0, (-len(p)) % 16)) for p in pages]))
        offs = np.cumsum([0] + [len(p) + (-len(p)) % 16 for p in pages])
        dblob = blob.cuda()
        pblob = blob.pin_memory()
        line = {"column": name, "encoding": enc, "rows": n * R, "pages": len(pages) * R, "page_bytes": total * R, "bits_per_value": 8.0 * total / n}
        for label, base, mem in (("device", dblob.data_ptr(), abi.MEM_DEVICE), ("pinned_host", pblob.data_ptr(), abi.MEM_HOST_PINNED)):
            views = [(base + int(offs[k]), len(p)) for k, p in enumerate(pages)] * R
            best = 1e9
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                rows = dec.decode(code, typ, views, out.data_ptr(), n * R, mem=mem)
                e1.record()
                torch.cuda.synchronize()
                best = min(best, e0.elapsed_time(e1))
            assert rows == n * R
            ok = bool((out.view(R, n).cpu().numpy() == v[None, :]).all())
            line[label] = {"ms": best, "values_per_s": n * R / best * 1e3, "page_gbs": total * R / best / 1e6, "output_gbs": n * R * v.dtype.itemsize / best / 1e6,
                           "bit_exact": ok}
        line["host_encode_s"] = enc_s
        res.append(line)
    dec.close()
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"workload": "segment page decode (sr_pages_decode)", "device": props.name, "page_rows": args.page_rows,
                      "columns": res}))


def _time(dec, code, views, out, rows, mem, reps):
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        got = dec.decode(code, abi.TYPE_INT, views, out.data_ptr(), rows, mem=mem)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    assert got == rows
    return best


def _power_limit():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return "unknown"


def _best_ms(fn, reps):
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def bool_bench(args):
    """--encoding nulls / rle: one byte per row out, a fraction of a bit per row in"""
    n, R, P = args.rows, args.repeat, args.page_rows
    rng = np.random.default_rng(3)
    ctx = gpu.Context(0)
    dec = gpu.PageDecoder(ctx)
    out = torch.empty(n * R, dtype=torch.uint8, device="cuda")
    parts = [(lo, min(lo + P, n)) for lo in range(0, n, P)]
    res = []
    if args.encoding == "nulls":
        host_col = torch.empty(n * R, dtype=torch.uint8).pin_memory()
        h2d_ms = _best_ms(lambda: out.copy_(host_col, non_blocking=True), args.reps)
        clustered = np.zeros(n, np.uint8)
        for st in rng.integers(0, n, n // 10_000):
            clustered[st:st + 1000] = 1
        columns = [("%g%% random" % (100 * f), (rng.random(n) < f).astype(np.uint8)) for f in (0.0, 0.001, 0.01, 0.1, 0.5)]
        columns.append(("runs of ~1000 (%.1f%%)" % (100 * clustered.mean()), clustered))
        cases = [(name, f, label, enc) for name, f in columns for label, enc in (("bitshuffle", bshuf_oracle.NULL_BITSHUFFLE), ("rle", bshuf_oracle.NULL_RLE))]
    else:
        columns = [("random", rng.integers(0, 2, n).astype(np.uint8)), ("runs of ~5000", np.repeat(rng.integers(0, 2, n // 5000 + 1), 5000)[:n].astype(np.uint8)),
                   ("alternating runs of 8", np.repeat(np.arange(n // 8 + 1) % 2, 8)[:n].astype(np.uint8))]
        cases = [(name, f, "rle_page", None) for name, f in columns]
    for name, f, label, enc in cases:
        t0 = time.perf_counter()
        if enc is None:
            bufs = [bshuf_oracle.rle_bool_page_encode(f[a:b]) for a, b in parts]
        else:
            bufs = [bshuf_oracle.null_map_encode(f[a:b], enc) for a, b in parts]
        enc_s = time.perf_counter() - t0
        total = sum(len(b) for b in bufs)
        blob = torch.from_numpy(np.concatenate([np.pad(b, (0, (-len(b)) % 16)) for b in bufs] + [np.zeros(16, np.uint8)]))
        offs = np.cumsum([0] + [len(b) + (-len(b)) % 16 for b in bufs])
        dblob, pblob = blob.cuda(), blob.pin_memory()
        line = {"column": name, "encoding": label, "rows": n * R, "pages": len(bufs) * R, "bits_per_row": 8.0 * total / n}
        want = int(f.sum()) * R
        for where, base, mem in (("device", dblob.data_ptr(), abi.MEM_DEVICE), ("pinned_host", pblob.data_ptr(), abi.MEM_HOST_PINNED)):
            out.fill_(0xA5)
            # the view array is built once, outside the timed window: the window holds the library call alone
            rows, nulls = C.c_int64(0), C.c_int64(0)
            if enc is None:
                views = (abi.sr_page_view * (len(bufs) * R))(*[abi.sr_page_view(base + int(offs[k]), len(b)) for k, b in enumerate(bufs)] * R)
                def call():
                    ctx.check(gpu.lib().sr_pages_decode(dec.h, abi.PAGE_RLE, abi.TYPE_BOOLEAN, views, len(views), mem, out.data_ptr(), n * R, C.byref(rows)))
            else:
                views = (abi.sr_null_map_view * (len(bufs) * R))(*[abi.sr_null_map_view(base + int(offs[k]), len(b), b1 - a1)
                                                                  for k, (b, (a1, b1)) in enumerate(zip(bufs, parts))] * R)
                def call():
                    ctx.check(gpu.lib().sr_null_maps_decode(dec.h, enc, views, len(views), mem, out.data_ptr(), n * R, C.byref(rows), C.byref(nulls)))
            ms = _best_ms(call, args.reps)
            ok = rows.value == n * R and (enc is None or nulls.value == want) and bool((out.view(R, n).cpu().numpy() == f[None, :]).all())
            line[where] = {"ms": ms, "g_rows_per_s": n * R / ms / 1e6, "page_gbs": total * R / ms / 1e6, "bit_exact": ok}
        if enc is not None:
            line["vs_h2d_copy_of_null_column"] = {lbl: h2d_ms / line[lbl]["ms"] for lbl in ("device", "pinned_host")}
        line["host_encode_s"] = enc_s
        res.append(line)
        del dblob, pblob
    dec.close()
    head = {"workload": "null map decode (sr_null_maps_decode)" if args.encoding == "nulls" else "BOOLEAN RLE page decode (sr_pages_decode, SR_PAGE_RLE)",
            "device": torch.cuda.get_device_properties(0).name, "power_limit": _power_limit(), "page_rows": P}
    if args.encoding == "nulls":
        head["h2d_copy_of_uint8_null_column"] = {"ms": h2d_ms, "g_rows_per_s": n * R / h2d_ms / 1e6, "gbs": n * R / h2d_ms / 1e6}
    head["columns"] = res
    print(json.dumps(head))


def dict_bench(args):
    import subprocess
    n, R = args.rows, args.repeat
    rng = np.random.default_rng(2)
    ctx = gpu.Context(0)
    dec = gpu.PageDecoder(ctx)
    out = torch.empty(n * R, dtype=torch.int32, device="cuda")
    res = []
    for words in (7, 25, 256):
        codes = rng.integers(0, words, n, dtype=np.int32)
        ids = (rng.permutation(words) + 1).astype(np.int32)            # a segment's local -> global id table
        dec.set_dict(ids)
        want = {"dict": ids[codes], "bitshuffle": codes}
        line = {"column": "%d words" % words, "rows": n * R}
        for enc, code, encode in (("dict", abi.PAGE_DICT, bshuf_oracle.dict_page_encode), ("bitshuffle", abi.PAGE_BITSHUFFLE, bshuf_oracle.bitshuffle_encode)):
            pages = [encode(codes[lo:lo + args.page_rows]) for lo in range(0, n, args.page_rows)]
            total = sum(len(p) for p in pages)
            blob = torch.from_numpy(np.concatenate([np.pad(p, (0, (-len(p)) % 16)) for p in pages]))
            offs = np.cumsum([0] + [len(p) + (-len(p)) % 16 for p in pages])
            dblob, pblob = blob.cuda(), blob.pin_memory()
            e = {"pages": len(pages) * R, "page_bytes": total * R, "bits_per_value": 8.0 * total / n}
            for label, base, mem in (("device", dblob.data_ptr(), abi.MEM_DEVICE), ("pinned_host", pblob.data_ptr(), abi.MEM_HOST_PINNED)):
                views = [(base + int(offs[k]), len(p)) for k, p in enumerate(pages)] * R
                out.fill_(-1)
                ms = _time(dec, code, views, out, n * R, mem, args.reps)
                ok = bool((out.view(R, n).cpu().numpy() == want[enc][None, :]).all())
                e[label] = {"ms": ms, "g_values_per_s": n * R / ms / 1e6, "page_gbs": total * R / ms / 1e6, "bit_exact": ok}
            line[enc] = e
            del dblob, pblob
        res.append(line)
    dec.close()
    props = torch.cuda.get_device_properties(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        power = "unknown"
    print(json.dumps({"workload": "dictionary page decode into global ids (sr_pages_decode, SR_PAGE_DICT)", "device": props.name,
                      "power_limit": power, "page_rows": args.page_rows, "columns": res}))


if __name__ == "__main__":
    main()
