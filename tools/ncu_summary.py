"""Extracts the judged subset of an .ncu-rep (ncu -i ... --page raw --csv) into a small CSV."""
import csv
import subprocess
import sys

KEEP = ['Kernel Name', 'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'launch__registers_per_thread',
        'launch__grid_size', 'launch__block_size', 'launch__occupancy_limit_registers', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'smsp__inst_executed.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct', 'smsp__thread_inst_executed_per_inst_executed.ratio',
        'sass__inst_executed_local_loads', 'sass__inst_executed_local_stores', 'sass__inst_executed_shared_loads', 'sass__inst_executed_shared_stores',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'launch__shared_mem_per_block_dynamic']


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write("launch,metric,unit,value\n")
        for li, vals in enumerate(rows[2:]):
            for h, u, v in zip(hdr, units, vals):
                if h in KEEP or (h.startswith('smsp__average_warps_issue_stalled') and h.endswith('per_issue_active.ratio')):
                    f.write('%d,%s,%s,"%s"\n' % (li, h, u, v))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
