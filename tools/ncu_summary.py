"""Summarise an .ncu-rep (ncu --set full) into the handful of numbers DESIGN.md / bench.py quote.

usage: python tools/ncu_summary.py x.ncu-rep [more.ncu-rep ...] > summary.md
"""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "registers/thread"),
    ("launch__occupancy_limit_shared_mem", "occupancy limit (smem), CTAs/SM"),
    ("launch__occupancy_limit_registers", "occupancy limit (regs), CTAs/SM"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
    ("lts__t_bytes.sum", "L2 bytes"),
    ("l1tex__t_sector_hit_rate.pct", "L1 hit rate %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("sm__inst_executed.avg.per_cycle_active", "IPC (active)"),
    ("smsp__issue_active.avg.pct", "issue active %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "FMA pipe %"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU pipe %"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor-pipe instructions"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe %"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "shared-memory wavefronts"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared-memory bank conflicts"),
    ("sm__cycles_elapsed.max", "SM cycles elapsed"),
]
STALLS = "smsp__average_warps_issue_stalled_%s_per_issue_active.ratio"
STALL_NAMES = ["long_scoreboard", "short_scoreboard", "wait", "barrier", "branch_resolving", "not_selected",
               "math_pipe_throttle", "mio_throttle", "lg_throttle", "membar", "no_instruction", "dispatch_stall",
               "sleeping", "tex_throttle", "drain", "imc_miss"]


def rows_of(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    r = list(csv.reader(io.StringIO(out)))
    hdr, units = r[0], r[1]
    return hdr, units, r[2:]


def main():
    for path in sys.argv[1:]:
        hdr, units, rows = rows_of(path)
        print(f"## `{path.split('/')[-1]}`\n")
        for row in rows:
            get = lambda k: (row[hdr.index(k)], units[hdr.index(k)]) if k in hdr else (None, None)  # noqa: E731
            print(f"### {get('Kernel Name')[0]}  (launch id {get('ID')[0]})\n")
            print("| metric | value |\n|---|---:|")
            for k, label in KEYS:
                v, u = get(k)
                if v is not None:
                    print(f"| {label} (`{k}`) | {v} {u} |")
            st = []
            for s in STALL_NAMES:
                v, _ = get(STALLS % s)
                if v is not None:
                    st.append((float(v), s))
            st.sort(reverse=True)
            print("\nwarp stall reasons (warps per issue-active cycle): " +
                  ", ".join(f"{s} {v:.2f}" for v, s in st if v >= 0.02) + "\n")


if __name__ == "__main__":
    main()
