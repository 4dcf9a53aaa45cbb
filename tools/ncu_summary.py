"""Summarise an .ncu-rep (ncu --set full) into the metrics the roofline discussion uses.  usage: ncu_summary.py rep [out.txt]"""
import csv
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr = rows[0]
KEYS = ["Kernel Name", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]
out = []
for r in rows[2:]:
    d = dict(zip(hdr, r))
    out.append("-" * 100)
    for k in KEYS:
        if k in d and d[k] != "":
            out.append(f"{k} = {d[k]}  [{dict(zip(hdr, rows[1])).get(k, '')}]")
    st = sorted(((float(v), k) for k, v in d.items() if k.startswith("smsp__average_warps_issue_stalled_") and
                 k.endswith("_per_issue_active.ratio") and v not in ("", "n/a")), reverse=True)[:8]
    out.append("top stall reasons (warps per issue-active cycle): " + ", ".join(
        f"{k[len('smsp__average_warps_issue_stalled_'):-len('_per_issue_active.ratio')]} {v:.2f}" for v, k in st))
    tensor = [f"{k} = {v}" for k, v in d.items() if "tensor" in k and "pct_of_peak_sustained_active" in k and v not in ("", "0", "n/a")]
    out.append("tensor pipes: " + "; ".join(tensor[:6]))
text = "\n".join(out)
if len(sys.argv) > 2:
    open(sys.argv[2], "w").write(f"# {rep} (ncu --set full --clock-control none)\n" + text + "\n")
print(text[:3000])
