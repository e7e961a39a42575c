#!/usr/bin/env python
"""Turns an ncu capture (*.ncu-rep) into the small text summary that
is committed under profiles/: launch configuration, time, pipe utilisation, DRAM traffic, stall reasons and the
executed-instruction mix by opcode and by loop level.  Usage: python profiles/summarize.py <rep | stem of exported csv pages> <units> > out.txt
`units` = how many work units (warp-generations for k_evolve_fast, warps for k_serial) the capture covers."""
import collections
import csv
import re
import subprocess
import sys

rep, units = sys.argv[1], float(sys.argv[2])
if rep.endswith(".ncu-rep"):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
else:  # <stem>: the two pages exported on the GPU box as <stem>.raw.csv and <stem>.source.csv.gz (the report itself embeds the whole library)
    import gzip
    raw = open(rep + ".raw.csv").read()
    src = gzip.open(rep + ".source.csv.gz", "rt").read()
rows = list(csv.reader(raw.splitlines()))
hdr, unitrow, d = rows[0], rows[1], dict(zip(rows[0], rows[2]))
print("kernel:", d.get("Kernel Name"))
want = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__cycles_elapsed.max", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__warps_eligible.avg.per_cycle_active"]
for w in want:
    if w in d:
        print(f"  {w:72s} {d[w]:>16s} {unitrow[hdr.index(w)]}")
print("stalls (warps stalled per issue-active cycle):")
st = [(h, float(d[h])) for h in hdr if "issue_stalled" in h and h.endswith("per_issue_active.ratio")]
for h, v in sorted(st, key=lambda x: -x[1])[:8]:
    print(f"  {h.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', ''):28s} {v:6.3f}")
k, hdr2 = [], None
for r in csv.reader(src.splitlines()):
    if r and r[0] == "Address":
        hdr2 = r
    elif len(r) > 6 and r[0].startswith("0x"):
        k.append(r)
iex, isrc, isamp = hdr2.index("Instructions Executed"), hdr2.index("Source"), hdr2.index("# Samples")
tot = sum(int(r[iex]) for r in k)
print(f"SASS lines {len(k)}, warp-instructions executed {tot} = {tot / units:.1f} per unit ({units:.0f} units)")
ops, samp = collections.Counter(), collections.Counter()
for r in k:
    m = re.match(r"\s*(@!?U?P\d+\s+)?([A-Z0-9_.]+)", r[isrc])
    op = m.group(2).split(".")[0] if m else "?"
    ops[op] += int(r[iex])
    samp[op] += int(r[isamp])
ts = max(sum(samp.values()), 1)
print("opcode mix (per unit, share of instructions, share of stall samples):")
for op, c in ops.most_common(18):
    print(f"  {op:10s} {c / units:9.1f} {100 * c / tot:5.1f}% {100 * samp[op] / ts:5.1f}%")
cls = collections.Counter()
for r in k:
    cls[int(r[iex])] += 1
print("loop levels (SASS lines sharing an execution count):")
for c, nl in sorted(cls.items(), key=lambda x: -x[0] * x[1])[:6]:
    print(f"  executed {c / units:8.2f}x per unit: {nl:5d} lines -> {c * nl / units:8.1f} instr per unit")
