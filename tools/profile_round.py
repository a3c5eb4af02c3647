#!/usr/bin/env python3
"""Turn one round's ncu artefacts into summaries under profiles/ (local output, not committed).

usage: tools/profile_round.py <tag> <launches.csv> <full.ncu-rep> <streams-per-launch> [libsolo_b200.so]
  <launches.csv>  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file <launches.csv> python tools/ncu_target.py N T dec
  <full.ncu-rep>  ncu --set full --clock-control none --import-source on -k regex:^sb_|sb_enc -o ... python tools/ncu_target.py N T dec
                  (every codec kernel once; the LAST captured launch of a kernel is used)
writes profiles/<tag>_launches.txt, profiles/<tag>_full.txt, profiles/<tag>_sass.txt and profiles/ncu_summary.json
(per kernel DRAM traffic, issue utilisation, warp instructions).  ncu launch times are cold-cache and serialised: compare SHARES."""
import collections
import csv
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag, launches, rep, spl = sys.argv[1], sys.argv[2], sys.argv[3], int(sys.argv[4])
so = sys.argv[5] if len(sys.argv) > 5 else os.path.join(ROOT, "solo_b200", "libsolo_b200.so")
P = os.path.join(ROOT, "profiles")
os.makedirs(P, exist_ok=True)


def short(name):
    return re.sub(r"\(.*", "", name).replace("<unnamed>::", "")


# ---- launch list ----
rows = [r for r in csv.reader(l for l in open(launches) if l.startswith('"'))]
hdr = rows[0]
ki, vi, gi, bi = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Grid Size"), hdr.index("Block Size")
per = collections.OrderedDict()
for r in rows[1:]:
    per.setdefault(short(r[ki]), []).append((float(r[vi].replace(",", "")), r[gi], r[bi]))
codec = {k: v for k, v in per.items() if k.startswith("sb_") and "init" not in k}
tot = sum(sum(t for t, _, _ in v) for v in codec.values())
with open(os.path.join(P, tag + "_launches.txt"), "w") as f:
    f.write("# %s: ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised launches), %d streams per launch\n" % (tag, spl))
    f.write("# share = kernel's part of the codec kernels' total\n")
    f.write("%-32s %8s %12s %8s  %s\n" % ("kernel", "launches", "avg_us", "share", "grid x block"))
    for k, v in codec.items():
        t = sum(x for x, _, _ in v)
        f.write("%-32s %8d %12.1f %7.1f%%  %s x %s\n" % (k, len(v), t / len(v) / 1e3, 100 * t / tot, v[0][1], v[0][2]))
    f.write("%-32s %8s %12.1f\n" % ("sum of the averages", "", sum(sum(x for x, _, _ in v) / len(v) for v in codec.values()) / 1e3))
print(open(os.path.join(P, tag + "_launches.txt")).read())

# ---- full capture ----
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rr = list(csv.reader(raw.splitlines()))
h, units = rr[0], rr[1]
col = {n: i for i, n in enumerate(h)}
want = [
    ("gpu__time_duration.sum", "duration"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
    ("launch__registers_per_thread", "registers/thread"), ("launch__shared_mem_per_block_dynamic", "dynamic smem/block"),
    ("launch__shared_mem_per_block_static", "static smem/block"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots used % (active cycles)"),
    ("sm__issue_active.avg.pct_of_peak_sustained_elapsed", "issue slots used % (elapsed)"),
    ("smsp__inst_executed.sum", "warp instructions"), ("smsp__thread_inst_executed_per_inst_executed.ratio", "active lanes / instruction"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM written"),
    ("sass__inst_executed_local_loads", "local loads (warp inst)"), ("sass__inst_executed_local_stores", "local stores (warp inst)"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared-memory bank conflicts"),
]
stalls = ["barrier", "wait", "short_scoreboard", "long_scoreboard", "no_instruction", "math_pipe_throttle", "branch_resolving", "not_selected",
          "mio_throttle", "lg_throttle", "dispatch_stall"]
last = collections.OrderedDict()
for r in rr[2:]:
    last[short(r[col["Kernel Name"]])] = r


def val(r, n):
    if n not in col or r[col[n]] == "":
        return None
    try:
        return float(r[col[n]].replace(",", ""))
    except ValueError:
        return None


def in_bytes(r, n):
    v = val(r, n)
    if v is None:
        return None
    u = units[col[n]].lower()
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)


def in_ns(r, n):
    v = val(r, n)
    u = units[col[n]].lower()
    return None if v is None else v * {"ns": 1, "us": 1e3, "usecond": 1e3, "ms": 1e6, "msecond": 1e6, "s": 1e9, "second": 1e9, "nsecond": 1}.get(u, 1)


summary = {}
with open(os.path.join(P, tag + "_full.txt"), "w") as f:
    f.write("# %s: ncu --set full --clock-control none, one launch per kernel, %d streams per launch\n" % (tag, spl))
    for k, r in last.items():
        if not k.startswith("sb_") or "init" in k:
            continue
        f.write("\n== %s ==\n" % k)
        for n, label in want:
            if n in col:
                f.write("  %-38s %s %s\n" % (label, r[col[n]], units[col[n]]))
        mix = []
        for s_ in stalls:
            n = "smsp__average_warps_issue_stalled_%s_per_issue_active.ratio" % s_
            v = val(r, n)
            if v is not None:
                mix.append((v, s_))
        f.write("  stall cycles per issued instruction:   " + ", ".join("%s %.2f" % (s_, v) for v, s_ in sorted(mix, reverse=True)[:7]) + "\n")
        dr, dw = in_bytes(r, "dram__bytes_read.sum") or 0, in_bytes(r, "dram__bytes_write.sum") or 0
        inst = val(r, "smsp__inst_executed.sum") or 0
        f.write("  per stream:                            %.0f warp instructions, %.1f KB DRAM traffic\n" % (inst / spl, (dr + dw) / spl / 1e3))
        summary[k] = {"duration_ns": in_ns(r, "gpu__time_duration.sum"), "dram_bytes_per_launch": dr + dw, "streams_per_launch": spl,
                      "issue_active_pct": val(r, "smsp__issue_active.avg.pct_of_peak_sustained_active"),
                      "warp_inst_per_stream": inst / spl, "active_lanes_per_inst": val(r, "smsp__thread_inst_executed_per_inst_executed.ratio"),
                      "registers": val(r, "launch__registers_per_thread")}
print(open(os.path.join(P, tag + "_full.txt")).read())

# ---- static SASS ----
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
cnt, fn = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        d = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        fn = short(d.replace("(anonymous namespace)::", ""))
        cnt[fn] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and fn:
        op = m.group(1)
        cnt[fn]["total"] += 1
        base = op.split(".")[0]
        for key in ("LDL", "STL", "LDS", "STS", "SHFL", "BAR", "UBLKCP", "LDG", "STG", "VOTE", "MUFU"):
            if base == key:
                cnt[fn][key] += 1
        if op.startswith("IMAD.HI"):
            cnt[fn]["IMAD.HI"] += 1
        elif base == "IMAD":
            cnt[fn]["IMAD"] += 1
keys = ["total", "IMAD", "IMAD.HI", "SHFL", "VOTE", "BAR", "LDS", "STS", "LDG", "STG", "LDL", "STL", "UBLKCP", "MUFU"]
with open(os.path.join(P, tag + "_sass.txt"), "w") as f:
    f.write("# %s: static SASS instruction counts per kernel (cuobjdump -sass %s)\n" % (tag, os.path.relpath(so, ROOT)))
    f.write("%-34s " % "kernel" + " ".join("%8s" % k for k in keys) + "\n")
    for fn, c in cnt.items():
        if c["total"]:
            f.write("%-34s " % fn[:34] + " ".join("%8d" % c[k] for k in keys) + "\n")
            if fn in summary:
                summary[fn]["sass_instructions"] = c["total"]
                summary[fn]["sass_local_ld_st"] = c["LDL"] + c["STL"]
print(open(os.path.join(P, tag + "_sass.txt")).read())

out = {"from": tag, "kernels": summary}
dom = max(summary, key=lambda k: summary[k]["duration_ns"] or 0)
out["dominant_kernel"] = dom
out["dram_bytes_per_packet"] = sum(v["dram_bytes_per_launch"] for v in summary.values()) / spl
tsum = sum(v["duration_ns"] or 0 for v in summary.values())
out["issue_util_time_weighted_pct"] = sum((v["issue_active_pct"] or 0) * (v["duration_ns"] or 0) for v in summary.values()) / max(tsum, 1)
out["warp_inst_per_packet"] = sum(v["warp_inst_per_stream"] for v in summary.values())
json.dump(out, open(os.path.join(P, "ncu_summary.json"), "w"), indent=1)
print("ncu_summary.json: dominant", dom, " DRAM bytes/packet %.0f  issue util %.1f%%  warp inst/packet %.0f" % (
    out["dram_bytes_per_packet"], out["issue_util_time_weighted_pct"], out["warp_inst_per_packet"]))
