#!/usr/bin/env python
"""Summarise ncu captures into small text files under profiles/ (git-ignored: local notes, never committed).
usage: python scripts/summarize_ncu.py r01"""
import csv, io, os, subprocess, sys, collections
tag = sys.argv[1] if len(sys.argv) > 1 else "r01"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
out_dir = os.path.join(ROOT, "profiles"); os.makedirs(out_dir, exist_ok=True)
WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "lts__t_sector_hit_rate.pct", "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "launch__occupancy_limit_registers",
        "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static"]
for f in sorted(os.listdir(os.path.join(ROOT, "gpurun_out"))):
    if not f.endswith(".ncu-rep"):
        continue
    r = subprocess.run(["ncu", "-i", os.path.join(ROOT, "gpurun_out", f), "--page", "raw", "--csv"], capture_output=True, text=True)
    rows = list(csv.reader(io.StringIO(r.stdout)))
    if len(rows) < 3:
        continue
    hdr, units = rows[0], rows[1]
    if f.startswith("prof_multi"):
        # one capture of several kernels (ncu -k regex:"a|b|c"): one summary file per kernel, the same format as the single-kernel captures
        seen = set()
        for vals in rows[2:]:
            name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
            base = name.split("(")[0].split("<")[0].split("::")[-1]
            if base in seen:
                continue
            seen.add(base)
            with open(os.path.join(out_dir, f"{tag}_prof_{base}.txt"), "w") as o:
                o.write(f"# ncu --set full --clock-control none, {f} (multi-kernel capture of one frame of bench.py); one launch per row block\n")
                o.write(f"kernel: {name[:160]}\n")
                for w in WANT:
                    if w in hdr:
                        i = hdr.index(w)
                        o.write(f"  {w} = {vals[i]} {units[i]}\n")
        print("wrote", f, sorted(seen))
        continue
    with open(os.path.join(out_dir, f"{tag}_{f.replace('.ncu-rep', '')}.txt"), "w") as o:
        o.write(f"# ncu --set full --clock-control none, {f}; one launch per row block\n")
        for vals in rows[2:]:
            name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
            o.write(f"kernel: {name[:160]}\n")
            for w in WANT:
                if w in hdr:
                    i = hdr.index(w)
                    o.write(f"  {w} = {vals[i]} {units[i]}\n")
    print("wrote", f)
lc = os.path.join(ROOT, "gpurun_out", "launches.csv")
if os.path.exists(lc):
    agg = collections.OrderedDict()
    txt = open(lc).read()
    start = txt.find('"ID"')
    rows = list(csv.reader(io.StringIO(txt[start:]))) if start >= 0 else []
    if rows:
        hdr = rows[0]
        ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
        for r in rows[1:]:
            if len(r) <= vi: continue
            k = r[ki].split("(")[0]
            try: v = float(r[vi].replace(",", ""))
            except ValueError: continue
            a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += v
        tot = sum(v[1] for v in agg.values())
        with open(os.path.join(out_dir, f"{tag}_launch_list.txt"), "w") as o:
            o.write("# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised: compare SHARES)\n# kernel  launches  total_ns  share\n")
            for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
                o.write(f"{k:40s} {n:6d} {t:14.0f} {t / tot:7.4f}\n")
        print("wrote launch list", len(agg))
