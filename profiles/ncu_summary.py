"""ncu report (.ncu-rep, --set full) -> one markdown table per kernel launch with the metrics the roofline argument uses.
    python profiles/ncu_summary.py gpurun_out/rNN_hot.ncu-rep > profiles/rNN_hot_ncu.md"""
import csv
import io
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"), ("launch__registers_per_thread", "regs/thread"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1/TEX throughput %"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput %"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
    ("dram__bytes_read.sum", "dram read"), ("dram__bytes_write.sum", "dram write"),
    ("lts__t_sector_hit_rate.pct", "L2 hit %"), ("l1tex__t_sector_hit_rate.pct", "L1 hit %"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "global load requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "global load sectors"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_red.sum", "global red requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum", "global red sectors"),
    ("lts__t_sectors_op_red.sum", "L2 red sectors"), ("lts__t_sectors_op_atom.sum", "L2 atom sectors"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe % (MMAs; sm__pipe_tensor_cycles_active)"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe % (hmma)"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall lg_throttle"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math_pipe"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
    ("smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "stall no_instruction"),
    ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall not_selected"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall mio_throttle"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard"),
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    print(f"# {path}\n")
    for r in rows[2:]:
        name = r[col["Kernel Name"]].split("(")[0]
        print(f"## {name}   (launch id {r[col['ID']]})\n")
        print("| metric | value | unit |\n|---|---:|---|")
        for key, label in WANT:
            if key in col:
                print(f"| {label} (`{key}`) | {r[col[key]]} | {units[col[key]]} |")
        print()


if __name__ == "__main__":
    main(sys.argv[1])
