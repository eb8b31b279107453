"""Summarise .ncu-rep captures (ncu --set full) into a few numbers per kernel.

usage: python tools/ncu_summary.py prof_x.ncu-rep [...] > prof_x_ncu_summary.txt
"""
import csv, io, subprocess, sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "smsp__inst_executed.sum", "smsp__thread_inst_executed.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__inst_executed_op_shared_atom.sum", "smsp__inst_executed_op_shared_ld.sum", "smsp__inst_executed_op_shared_st.sum",
    "smsp__inst_executed_op_global_ld.sum", "smsp__inst_executed_op_global_st.sum", "smsp__inst_executed_op_global_atom.sum",
    "smsp__inst_executed_op_global_red.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum",
    "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
]


def main():
    for path in sys.argv[1:]:
        raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(raw)))
        if len(rows) < 3:
            print("!! no data in", path)
            continue
        hdr, units = rows[0], rows[1]
        col = {h: i for i, h in enumerate(hdr)}
        for r in rows[2:]:
            print("--- %s   [%s]" % (r[col["Kernel Name"]][:90], path.split("/")[-1]))
            for k in KEYS:
                if k in col:
                    print("  %-78s %s %s" % (k, r[col[k]], units[col[k]]))
            stalls = []
            for h, i in col.items():
                if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio") or \
                   h.startswith("smsp__average_warp_latency_issue_stalled_") and h.endswith(".ratio"):
                    try:
                        stalls.append((float(r[i]), h.split("stalled_")[1].split("_per_")[0].replace(".ratio", "")))
                    except ValueError:
                        pass
            stalls.sort(reverse=True)
            print("  stalls: " + ", ".join("%s=%.2f" % (n, v) for v, n in stalls[:8]))


if __name__ == "__main__":
    main()
