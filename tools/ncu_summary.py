#!/usr/bin/env python
"""Summarise an .ncu-rep (read with `ncu -i`): headline metrics, opcode mix, stall reasons per opcode class.
    python tools/ncu_summary.py prof.ncu-rep [kernel-index]
"""
import csv, subprocess, sys, io
from collections import Counter

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
kidx = int(sys.argv[2]) if len(sys.argv) > 2 else 0
vals = rows[2 + kidx]
m = dict(zip(hdr, vals)); u = dict(zip(hdr, units))
keys = ["Kernel Name", "gpu__time_duration.sum", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "sm__icc_request_hit_rate.pct", "smsp__sass_inst_executed_op_local_ld.sum",
        "smsp__sass_inst_executed_op_local_st.sum", "smsp__sass_inst_executed_op_shared_ld.sum", "smsp__sass_inst_executed_op_shared_st.sum",
        "smsp__sass_inst_executed_op_global_ld.sum", "smsp__sass_inst_executed_op_global_st.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__thread_inst_executed_per_inst_executed.ratio"]
for k in keys:
    if k in m: print(f"{k:75s} {m[k]} {u.get(k,'')}")
print("-- stall reasons (warps per issue-active cycle) --")
st = {k: float(v) for k, v in m.items() if k.startswith("smsp__average_warps_issue_stalled_") and k.endswith("_per_issue_active.ratio")}
for k, v in sorted(st.items(), key=lambda kv: -kv[1])[:10]:
    print(f"   {k.replace('smsp__average_warps_issue_stalled_','').replace('_per_issue_active.ratio',''):24s} {v:.3f}")

src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
# find the header row
hi = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
hdr = rows[hi]; data = [r for r in rows[hi + 1:] if len(r) == len(hdr)]
isrc, iex, ism = hdr.index("Source"), hdr.index("Instructions Executed"), hdr.index("# Samples")
stall_cols = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
tot_ex = sum(int(r[iex]) for r in data); tot_s = sum(int(r[ism]) for r in data)
print(f"-- SASS: {len(data)} instructions, {tot_ex} executed warp-instructions, {tot_s} samples --")
c, cs = Counter(), Counter()
stall_by_op = {}
for r in data:
    toks = r[isrc].split()
    op = toks[1] if toks[0].startswith("@") else toks[0]
    op = op.split(".")[0]
    c[op] += int(r[iex]); cs[op] += int(r[ism])
    d = stall_by_op.setdefault(op, Counter())
    for i in stall_cols:
        d[hdr[i]] += int(r[i] or 0)
for op, n in cs.most_common(18):
    top = ", ".join(f"{k.replace('stall_','')}:{v}" for k, v in stall_by_op[op].most_common(3))
    print(f"   {op:8s} exec {c[op]/tot_ex*100:5.1f}%  samples {n/tot_s*100:5.1f}%   [{top}]")
print("-- hottest instructions by samples --")
for r in sorted(data, key=lambda r: -int(r[ism]))[:25]:
    d = {hdr[i]: int(r[i] or 0) for i in stall_cols}
    top = ", ".join(f"{k.replace('stall_','')}:{v}" for k, v in sorted(d.items(), key=lambda kv: -kv[1])[:2])
    print(f"   {int(r[ism]):6d}  {r[isrc].strip()[:70]:70s} [{top}]")
