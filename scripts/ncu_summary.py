"""Summarise an .ncu-rep (read here, no GPU): key raw metrics per kernel launch + top stall reasons.
usage: python scripts/ncu_summary.py prof.ncu-rep [out.txt]"""
import csv, io, subprocess, sys
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
KEYS = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__thread_inst_executed.sum",
        "sm__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_alu.sum", "sm__inst_executed_pipe_xu.sum", "sm__inst_executed_pipe_lsu.sum",
        "sm__inst_executed_pipe_fmaheavy.sum", "sm__inst_executed_pipe_fmalite.sum",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed", "smsp__inst_executed_op_shared_ld.sum", "smsp__inst_executed_op_shared_st.sum",
        "smsp__inst_executed_op_global_red.sum", "smsp__inst_executed_op_global_ld.sum", "smsp__inst_executed_op_global_st.sum",
        "smsp__sass_inst_executed_op_shuffle.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"]
out = []
for r in rows[2:]:
    d = dict(zip(hdr, r))
    out.append("=" * 100)
    for k in KEYS:
        if k in d: out.append(f"{k:85s} {d[k]:>18s} {units[hdr.index(k)]}")
    st = [(h, float(d[h].replace(',', ''))) for h in hdr if h.startswith("smsp__average_warp") and h.endswith("_per_issue_active.ratio") and d[h] not in ("", "n/a")]
    st.sort(key=lambda x: -x[1])
    out.append("-- warp-cycles per issued instruction by stall reason (top 8):")
    for h, v in st[:8]: out.append(f"   {h:90s} {v:8.3f}")
txt = "\n".join(out)
print(txt)
if len(sys.argv) > 2: open(sys.argv[2], "w").write(txt + "\n")
