"""Summarise an .ncu-rep (one or more kernels) into a small markdown/JSON file.

    python scripts/ncu_summary.py st_fast_v1.ncu-rep profiles/st_fast_v1

Reads the report with `ncu -i ... --page raw --csv` (works without a GPU).
"""
import csv
import io
import json
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size", "launch__waves_per_multiprocessor",
    "sm__inst_executed.sum", "smsp__inst_executed.avg.per_cycle_active", "sm__inst_executed.avg.per_cycle_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_fma.sum",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.sum", "sm__inst_executed_pipe_lsu.sum",
    "sm__inst_executed_pipe_xu.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "smsp__average_warp_latency_issue_stalled_barrier.pct", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__warps_eligible.avg.per_cycle_active", "smsp__warps_active.avg.per_cycle_active",
    "lts__t_bytes.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_st.sum",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    idx = {h: i for i, h in enumerate(hdr)}
    res = []
    for r in data:
        d = {"kernel": r[idx["Kernel Name"]]}
        for k in KEYS:
            if k in idx:
                d[k] = r[idx[k]] + " " + units[idx[k]]
        stalls = {h: r[i] for h, i in idx.items() if "issue_stalled" in h and h.endswith("per_issue_active.ratio")}
        d["stall_ratios_top"] = sorted(((float(v.replace(",", "")), k.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""))
                                        for k, v in stalls.items() if v), reverse=True)[:8]
        res.append(d)
    with open(out + ".json", "w") as f:
        json.dump(res, f, indent=1)
    with open(out + ".md", "w") as f:
        for d in res:
            f.write("## %s\n\n| metric | value |\n|---|---|\n" % d["kernel"])
            for k, v in d.items():
                if k not in ("kernel",):
                    f.write("| %s | %s |\n" % (k, v))
            f.write("\n")
    print(open(out + ".md").read())


if __name__ == "__main__":
    main()
