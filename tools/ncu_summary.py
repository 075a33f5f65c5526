"""Text summary of one kernel of an ncu report (headline raw metrics + hottest source lines).
usage: python tools/ncu_summary.py <report.ncu-rep> <lib.so> <kernel-substring> <title> [mangled-substring]
The optional mangled substring (e.g. ILi0ELb1ELb1E for sim_topk_kernel<0, true, true>) picks ONE template instantiation for
the SASS-offset -> source-line mapping; without it the first instantiation in the cubin is used, which is wrong for the others."""
import csv, io, subprocess, sys
rep, lib, kern, title = sys.argv[1:5]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
row = next(r for r in rows[2:] if any(kern in c for c in r[:8]))
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct",
        "l1tex__t_sector_hit_rate.pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.avg",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]
print("# %s" % title)
print("# source: %s (ncu --set full --clock-control none --import-source on; numbers under the profiler are not bench values)" % rep.split("/")[-1])
vals = {}
for h, u, v in zip(hdr, units, row):
    if h in want or h.startswith("smsp__average_warps_issue_stalled") and h.endswith("per_issue_active.ratio"):
        vals[h] = (v, u)
for h in want:
    if h in vals:
        print("%-70s %s %s" % (h, vals[h][0], vals[h][1]))
st = sorted(((float(v[0]), h) for h, v in vals.items() if h.startswith("smsp__average_warps_issue_stalled")), reverse=True)[:6]
print("top stall reasons (warps per issue-active cycle): " + ", ".join("%s=%.2f" % (h.split("stalled_")[1].split("_per_")[0], x) for x, h in st))
try:
    rd = float(vals["dram__bytes_read.sum"][0]); wr = float(vals["dram__bytes_write.sum"][0])
    scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}
    tot = rd * scale[vals["dram__bytes_read.sum"][1]] + wr * scale[vals["dram__bytes_write.sum"][1]]
    print("dram traffic per launch (read+write): %.4g bytes" % tot)
except Exception as ex:
    print("traffic: n/a (%r)" % ex)
print()
print(subprocess.run([sys.executable, "tools/ncu_lines.py", rep, lib, kern, "22"] + sys.argv[5:6], capture_output=True, text=True).stdout)
