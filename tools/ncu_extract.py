"""Key metrics of an .ncu-rep (one kernel launch) as a markdown table: python tools/ncu_extract.py rep [out.md]"""
import csv, io, subprocess, sys

WANT = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.max",
    "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tensor.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed_pipe_uniform.sum",
    "l1tex__m_xbar2l1tex_read_bytes.sum",
    "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_barrier_per_warp_active.pct",
    "smsp__warp_issue_stalled_wait_per_warp_active.pct", "smsp__warp_issue_stalled_sleeping_per_warp_active.pct",
]


def main(rep, out=None):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rows[0], rows[1], rows[-1]
    name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
    lines = [f"kernel: `{name[:120]}`", "", "| metric | unit | value |", "|---|---|---:|"]
    for w in WANT:
        for h, u, v in zip(hdr, units, vals):
            if h.endswith(w) or h == w:
                lines.append(f"| {w} | {u} | {v} |")
                break
    text = "\n".join(lines) + "\n"
    if out:
        open(out, "w").write(text)
    print(text)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else None)
