"""Exports the key metrics of an .ncu-rep (ncu -i ... --page raw --csv) to a compact CSV."""
import csv
import subprocess
import sys

KEYS = ["Kernel Name", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "gpu__time_duration.sum", "sm__cycles_elapsed.max",
        "sm__cycles_active.avg", "smsp__cycles_active.avg", "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__m_xbar2l1tex_read_bytes.sum",
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_writes.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_reads.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_math_pipe_throttle_per_warp_active.pct",
        "smsp__warp_issue_stalled_barrier_per_warp_active.pct", "smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct"]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr = rows[0]
    idx = [hdr.index(k) for k in KEYS if k in hdr]
    with open(out, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow([hdr[i] for i in idx])
        w.writerow([rows[1][i] for i in idx])
        for r in rows[2:]:
            w.writerow([r[i] for i in idx])
    print(out, len(rows) - 2, "kernels")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
