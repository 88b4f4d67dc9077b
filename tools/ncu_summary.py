"""Write a text summary of an ncu report: per-kernel metrics + top stall lines per CUDA source line.
   python tools/ncu_summary.py <report>.ncu-rep <summary>.txt ["header line"]"""
import csv, io, subprocess, sys
rep, dst = sys.argv[1], sys.argv[2]
hdr = sys.argv[3] if len(sys.argv) > 3 else ""
M = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
     "launch__registers_per_thread", "sm__inst_issued.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
     "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
     "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__grid_size"]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--metrics", ",".join(M)], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
h = rows[0]; ki = h.index("Kernel Name"); cols = [h.index(m) for m in M]
out = [f"# ncu --set full summary ({rep.split('/')[-1]}): {hdr}",
       "# columns: kernel | ms | dram read GB | dram write GB | warps active % | regs | issue active % | warp instr | threads/instr | L1 hit % | L2 hit % | CTAs/SM limit smem | regs | grid"]
names = []
for r in rows[2:]:
    if float(r[cols[0]]) < 0.05: continue            # the optimistic first pass of a retried decode launches empty kernels
    nm = r[ki].split("(")[0]; names.append(nm)
    vals = []
    for c, m in zip(cols, M):
        v = r[c]
        try: v = f"{float(v):.3f}" if "." in v else v
        except ValueError: pass
        vals.append(v)
    out.append(f"{nm} | " + " | ".join(vals))
out.append("")
out.append("## top stall lines (CUDA source) per kernel")
for nm in dict.fromkeys(names):
    top = subprocess.run([sys.executable, __file__.replace("ncu_summary.py", "ncu_top.py"), rep, nm, "12"], capture_output=True, text=True).stdout
    out.append(top.rstrip()); out.append("")
open(dst, "w").write("\n".join(l[:260] for l in "\n".join(out).split("\n")) + "\n")
print("wrote", dst)
