"""Turn an `ncu --set full` report into a text summary + traffic.json (bench.py reads profiles/traffic.json when it exists).
  mkdir -p profiles && python scripts/ncu_summary.py report.ncu-rep profiles/frag_full_summary.txt profiles/traffic.json
"""
import csv
import json
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor", "smsp__inst_executed.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
]
UNIT_SCALE = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}


def main():
    rep, out_txt, out_json = sys.argv[1:4]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    head, units = rows[0], rows[1]
    idx = {k: i for i, k in enumerate(head)}
    lines = ["# ncu --set full --clock-control none --import-source on, k_frag_* kernels of `python bench.py --steps 2 --warmup 1`",
             "# (SSB SF100 Q4.1, 600 M rows, one GPU); per-launch values; one launch of each kernel = one fragment push over the shard", ""]
    traffic = {}
    for r in rows[2:]:
        name = r[idx["Kernel Name"]].split("(")[0].replace("void ", "").replace("srd::", "")
        lines.append(f"## {name}")
        for m in METRICS:
            if m in idx:
                lines.append(f"{m:<100s} {r[idx[m]]:>16s} {units[idx[m]]}")
        lines.append("")
        rd = float(r[idx["dram__bytes_read.sum"]]) * UNIT_SCALE.get(units[idx["dram__bytes_read.sum"]], 1.0)
        wr = float(r[idx["dram__bytes_write.sum"]]) * UNIT_SCALE.get(units[idx["dram__bytes_write.sum"]], 1.0)
        traffic[name.split("<")[0]] = int(rd + wr)
    open(out_txt, "w").write("\n".join(lines))
    json.dump({"kernels": traffic, "dram_bytes_per_launch": sum(traffic.values()),
               "source": f"{out_txt} (ncu --set full, dram__bytes_read.sum + dram__bytes_write.sum per launch; one fragment push = one launch of each kernel)"},
              open(out_json, "w"), indent=1)
    print(json.dumps(traffic))


if __name__ == "__main__":
    main()
