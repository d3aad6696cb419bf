"""Text summary of an .ncu-rep (run where ncu is installed; no GPU needed): headline metrics per sample, the
instruction / stall-sample split between barriers, and the hottest stall sites.

  python tools/ncu_summary.py prof_X.ncu-rep <samples in the profiled launch> > prof_X.summary.txt
"""
import csv, subprocess, sys

rep, nsamp = sys.argv[1], float(sys.argv[2])
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, vals = rows[0], rows[1], rows[2]
get = lambda name: next((vals[i] for i, h in enumerate(hdr) if h == name), None)
unit = lambda name: next((units[i] for i, h in enumerate(hdr) if h == name), "")
print("kernel:", get("Kernel Name"))
print("grid", get("launch__grid_size"), "block", get("launch__block_size"), "registers/thread", get("launch__registers_per_thread"),
      "dynamic smem/block", get("launch__shared_mem_per_block_dynamic"))
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sectors_srcunit_tex_op_red.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__cycles_elapsed.max"]
for w in want:
    v = get(w)
    if v is not None:
        print("%-70s %s %s" % (w, v, unit(w)))
ns = lambda name: float(get(name) or 0)
t_ms = ns("gpu__time_duration.sum") * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit("gpu__time_duration.sum"), 1.0)
gb = lambda name: ns(name) * {"byte": 1e-9, "Kbyte": 1e-6, "Mbyte": 1e-3, "Gbyte": 1.0}.get(unit(name), 1.0)
print("per sample: %.2f thread-instructions, %.2f B DRAM read, %.2f B DRAM written; %.1f G samples/s under ncu"
      % (ns("smsp__inst_executed.sum") * 32 / nsamp, gb("dram__bytes_read.sum") * 1e9 / nsamp, gb("dram__bytes_write.sum") * 1e9 / nsamp,
         nsamp / t_ms / 1e6))
print("stall reasons (warps per issue-active cycle):")
for i, h in enumerate(hdr):
    if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio"):
        if float(vals[i]) >= 0.05:
            print("   %-28s %.2f" % (h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")], float(vals[i])))
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(src.splitlines()))
h2 = rows[1]
ia, isrc, iall, iex = h2.index("Address"), h2.index("Source"), h2.index("Warp Stall Sampling (All Samples)"), h2.index("Instructions Executed")
data = []
for r in rows[2:]:
    try:
        data.append((int(r[iall]), int(r[iex]), r[ia][-5:], r[isrc]))
    except Exception:
        pass
tot, totex = sum(d[0] for d in data) or 1, sum(d[1] for d in data) or 1
print("regions between barriers / votes (share of executed instructions, thread-instructions per sample, share of stall samples):")
ci = cs = li = ls = 0
for d in data:
    ci += d[1]; cs += d[0]
    if "BAR.SYNC" in d[3] or "VOTE.ANY" in d[3]:
        print("   up to %s %-24s inst %5.1f%% (%5.1f/sample)  stalls %5.1f%%" % (d[2], d[3][:24], 100 * (ci - li) / totex, (ci - li) * 32 / nsamp, 100 * (cs - ls) / tot))
        li, ls = ci, cs
print("   tail inst %.1f%% stalls %.1f%%" % (100 * (totex - li) / totex, 100 * (tot - ls) / tot))
print("hottest stall sites:")
for d in sorted(data, reverse=True)[:12]:
    print("   %5.1f%%  executed %9d  %s  %s" % (100 * d[0] / tot, d[1], d[2], d[3][:80]))
