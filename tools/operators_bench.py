"""Throughput of the separate operator entry points (the non-fused path a BE pipeline takes when a plan shape is not
covered by the fused fragment) on HBM-resident chunks, one H100:

    python tools/operators_bench.py [--rows 200000000]

  sr_scan_evaluate / sr_scan_filter   SSB Q1.1 conjuncts; filter materialises two surviving columns
  sr_join_probe                       INNER join against a 3 M-row dense-key build side, one payload column, 20 % match
  runtime filter                      the same join with its build-side filter (min/max + bloom) attached to the scan:
                                      scan_filter(+filter) then join_probe on the survivors
  sr_agg_push                         no GROUP BY / dense (7 x 25 groups) / hash (1 M groups)
  two-phase aggregate                 sr_agg_convert_to_states (the streaming first phase's pass-through leg) and first-phase
                                      push + pull of the intermediate rows + merge-phase push
Each line: milliseconds (best of N), rows/s and algorithmic GB/s (input columns read + output written).
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from starrocks_b200 import abi, gpu, ssb  # noqa: E402


def best_ms(fn, stream, reps):
    fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only-agg", action="store_true")
    args = ap.parse_args()
    n = args.rows
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = gpu.Context(0, stream=stream.cuda_stream)
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    ri = lambda lo, hi: torch.randint(lo, hi, (n,), device=dev, generator=g, dtype=torch.int32)  # noqa: E731
    cols = {"lo_orderdate": 19920101 + ri(0, 7) * 10000 + ri(0, 12) * 100 + ri(0, 28), "lo_discount": ri(0, 11),
            "lo_quantity": ri(1, 51), "lo_extendedprice": ri(90_000, 10_494_951), "lo_custkey": ri(1, 3_000_001),
            "lo_revenue": ri(81_000, 10_400_000), "g1": ri(1992, 1999), "g2": ri(0, 25), "gk": ri(0, 1_000_000)}
    torch.cuda.synchronize()
    out = {}

    def report(name, ms, bytes_):
        out[name] = {"ms": round(ms, 3), "rows_per_s": n / ms * 1e3, "algorithmic_gbs": bytes_ / ms / 1e6}

    if not args.only_agg:
        # ---- scan ----
        q11 = ssb.fact_chunk(cols, ssb.Q11_FACT_COLS, mem=abi.MEM_DEVICE)
        scan_all = gpu.Scan(ctx, abi.ScanDesc(preds=ssb.q11_scan_preds()))
        sel = torch.empty(n, dtype=torch.uint8, device=dev)
        L = gpu.lib()
        report("scan_evaluate (3 conjuncts -> uint8 selection)",
               best_ms(lambda: ctx.check(L.sr_scan_evaluate(scan_all.h, q11.ref(), sel.data_ptr(), abi.MEM_DEVICE)), stream, args.reps), n * (12 + 1))
        scan2 = gpu.Scan(ctx, abi.ScanDesc(preds=ssb.q11_scan_preds(), out_slots=[ssb.LO_SLOTS["lo_extendedprice"], ssb.LO_SLOTS["lo_discount"]]))
        passed = scan2.filter(q11).num_rows
        report("scan_filter (3 conjuncts, 2 columns out, %.1f %% pass)" % (100.0 * passed / n), best_ms(lambda: scan2.filter(q11), stream, args.reps), n * 16)
        scan_half = gpu.Scan(ctx, abi.ScanDesc(preds=[abi.make_pred(ssb.LO_SLOTS["lo_quantity"], abi.PRED_LE, 25)],
                                               out_slots=[ssb.LO_SLOTS[c] for c in ssb.Q11_FACT_COLS]))
        passed = scan_half.filter(q11).num_rows
        report("scan_filter (1 conjunct, 4 columns out, %.1f %% pass)" % (100.0 * passed / n), best_ms(lambda: scan_half.filter(q11), stream, args.reps),
               n * 16 + passed * 16)

        # ---- join probe ----
        nb = 3_000_000
        rng = np.random.default_rng(3)
        keep = np.sort(rng.choice(np.arange(1, nb + 1, dtype=np.int32), size=nb // 5, replace=False))
        build = abi.Chunk([(100, keep, None), (101, (keep % 25).astype(np.int32), None)])
        jd = abi.make_join_desc(abi.JOIN_INNER, [100], [ssb.LO_SLOTS["lo_custkey"]], [abi.TYPE_INT], build_out=[101],
                                probe_out=[ssb.LO_SLOTS["lo_custkey"], ssb.LO_SLOTS["lo_revenue"]])
        j = gpu.Join(ctx, jd)
        j.append_build(build)
        j.build_finish()
        probe = abi.Chunk([(ssb.LO_SLOTS["lo_custkey"], cols["lo_custkey"], None, abi.TYPE_INT), (ssb.LO_SLOTS["lo_revenue"], cols["lo_revenue"], None, abi.TYPE_INT)],
                          mem=abi.MEM_DEVICE)
        matched = j.probe(probe).num_rows
        report("join_probe INNER (%.1f %% match, 2 probe + 1 build column out)" % (100.0 * matched / n), best_ms(lambda: j.probe(probe), stream, args.reps),
               n * 4 + matched * (8 + 12))

        # ---- runtime filter: the join's build-side filter on the scan, then the probe on what survives ----
        rf = gpu.RuntimeFilter.from_join(j, 0, True, False)
        scan_rf = gpu.Scan(ctx, abi.ScanDesc(preds=[], out_slots=[ssb.LO_SLOTS["lo_custkey"], ssb.LO_SLOTS["lo_revenue"]]))
        scan_rf.add_runtime_filter(rf, ssb.LO_SLOTS["lo_custkey"])
        kept = scan_rf.filter(probe)
        survivors = kept.num_rows
        report("scan_filter + runtime filter (bloom of %d keys, %.1f %% pass, 2 columns out)" % (len(keep), 100.0 * survivors / n),
               best_ms(lambda: scan_rf.filter(probe), stream, args.reps), n * 8 + survivors * 8)

        def scan_then_probe():
            o = scan_rf.filter(probe)
            v = abi.sr_chunk_view(C.cast(o.cols, C.POINTER(abi.sr_col_view)), o.num_cols, abi.MEM_DEVICE, o.num_rows)  # same column layout
            ctx.check(L.sr_join_probe(j.h, 0, C.byref(v), C.byref(abi.sr_chunk_out())))
        report("scan_filter + runtime filter -> join_probe (vs join_probe on every row above)", best_ms(scan_then_probe, stream, args.reps),
               n * 8 + survivors * 8 + survivors * 4 + matched * 20)

    # ---- aggregate ----
    def agg_case(name, desc, columns, bytes_):
        a = gpu.Agg(ctx, desc)
        ch = abi.Chunk([(s, cols[c], None, abi.TYPE_INT) for s, c in columns], mem=abi.MEM_DEVICE)

        def run():
            a.reset()
            a.push(ch)
        report(name, best_ms(run, stream, args.reps), bytes_)
        a.close()

    agg_case("agg_push no GROUP BY: SUM(a*b), COUNT(*)",
             abi.make_agg_desc(fns=[(abi.AGG_SUM, abi.TYPE_BIGINT, 10, [("col", 1), ("col", 2), "*"]), (abi.AGG_COUNT_STAR, 0, 11, None)]),
             [(1, "lo_extendedprice"), (2, "lo_discount")], n * 8)
    agg_case("agg_push dense 7 x 25 groups: 2 x SUM",
             abi.make_agg_desc([1, 2], [abi.TYPE_INT, abi.TYPE_INT], fns=[(abi.AGG_SUM, abi.TYPE_INT, 10, [("col", 3)]), (abi.AGG_SUM, abi.TYPE_INT, 11, [("col", 4)])],
                               ranges=[(1992, 1998), (0, 24)]),
             [(1, "g1"), (2, "g2"), (3, "lo_revenue"), (4, "lo_extendedprice")], n * 16)
    agg_case("agg_push hash 1 M groups: SUM, COUNT(*)",
             abi.make_agg_desc([1], [abi.TYPE_INT], fns=[(abi.AGG_SUM, abi.TYPE_INT, 10, [("col", 3)]), (abi.AGG_COUNT_STAR, 0, 11, None)]),
             [(1, "gk"), (3, "lo_revenue")], n * 8)
    # ---- two-phase aggregate: pass-through leg and the merge of pre-aggregated states ----
    d1 = abi.make_agg_desc([1], [abi.TYPE_INT], fns=[(abi.AGG_SUM, abi.TYPE_INT, 10, [("col", 3)]), (abi.AGG_AVG, abi.TYPE_INT, 11, [("col", 3)]),
                                                     (abi.AGG_COUNT_STAR, 0, 12, None)])
    p1, p2 = gpu.two_phase_descs(d1)
    first, final = gpu.Agg(ctx, p1), gpu.Agg(ctx, p2)
    ch = abi.Chunk([(1, cols["gk"], None, abi.TYPE_INT), (3, cols["lo_revenue"], None, abi.TYPE_INT)], mem=abi.MEM_DEVICE)
    report("agg_convert_to_states (pass-through leg): key + SUM, AVG, COUNT(*) states",
           best_ms(lambda: first.convert_to_states(ch), stream, args.reps), n * 8 + n * (8 + 8 + 8 + 8))

    def first_phase_then_merge():
        first.reset()
        first.push(ch)
        first.finish()
        final.reset()
        final.push(gpu.chunk_out_as_view(first.pull(mem=abi.MEM_DEVICE)))
    report("two-phase hash aggregate, 1 M groups: first-phase push + pull states + merge push", best_ms(first_phase_then_merge, stream, args.reps), n * 8)
    first.close()
    final.close()
    print(json.dumps({"rows": n, "operators": out}, indent=1))


if __name__ == "__main__":
    main()
