#!/usr/bin/env python3
"""Turn the ncu reports of profiles/run_ncu.sh (<output directory>/prof_<workload>[_src|_frame|_frame8]_<tag>.ncu-rep) into the committed
evidence: profiles/<tag>_<workload>_summary.txt (per-launch metrics + hottest source lines) and profiles/traffic.json — the
per-frame instruction and DRAM counters of every kernel class that bench.py's roofline divides by its own CUDA-event times.
usage: profiles/make_summaries.py <tag> [output directory of run_ncu.sh, default ncu_out]"""
import csv
import glob
import json
import os
import re
import subprocess
import sys

tag = sys.argv[1]
src = sys.argv[2] if len(sys.argv) > 2 else "ncu_out"
HERE = os.path.dirname(os.path.abspath(__file__))
CLASSES = {"k_trace_closest": "trace_closest", "k_shadow_accumulate": "shadow_accumulate", "k_shade_queues": "shade_queues",
           "k_trace_both": "trace_both", "k_frame": "frame"}
SCALE = {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1.0, "us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1.0, "msecond": 1e-3, "usecond": 1e-6,
         "nsecond": 1e-9, "second": 1.0}


def raw(rep):
    """raw page of a report: a .csv exported on the GPU box (ncu -i rep --page raw --csv) or the .ncu-rep itself"""
    if rep.endswith(".csv"):
        out = open(rep).read()
    else:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = [r for r in csv.reader(out.splitlines()) if r and not r[0].startswith("==")]
    return rows[0], rows[1], rows[2:]


def fnum(x):
    try:
        return float(x.replace(",", ""))
    except ValueError:
        return 0.0


def aggregate(rep):
    """-> {class: counters summed over the launches in the report}"""
    hdr, units, rows = raw(rep)
    col = {n: i for i, n in enumerate(hdr)}

    def val(r, name):
        if name not in col:
            return None
        return fnum(r[col[name]]) * SCALE.get(units[col[name]], 1.0)
    agg = {}
    for r in rows:
        kname = r[col["Kernel Name"]]
        cls = next((c for k, c in CLASSES.items() if k in kname), None)
        if cls is None:
            continue
        a = agg.setdefault(cls, {"launches": 0, "inst": 0.0, "thread_inst": 0.0, "dram_bytes": 0.0, "seconds": 0.0, "issue_active_x_s": 0.0,
                                 "warps_active_x_s": 0.0, "regs": None, "durations_us": []})
        inst = val(r, "smsp__inst_executed.sum") or 0.0
        tinst = val(r, "smsp__thread_inst_executed.sum")
        if tinst is None:
            tinst = inst * (val(r, "smsp__thread_inst_executed_per_inst_executed.ratio") or 0.0)
        sec = val(r, "gpu__time_duration.sum") or 0.0
        a["launches"] += 1; a["inst"] += inst; a["thread_inst"] += tinst; a["seconds"] += sec
        a["dram_bytes"] += (val(r, "dram__bytes_read.sum") or 0.0) + (val(r, "dram__bytes_write.sum") or 0.0)
        a["issue_active_x_s"] += (val(r, "smsp__issue_active.avg.pct_of_peak_sustained_active") or 0.0) * sec
        a["warps_active_x_s"] += (val(r, "sm__warps_active.avg.pct_of_peak_sustained_active") or 0.0) * sec
        a["regs"] = val(r, "launch__registers_per_thread")
        a["durations_us"].append(round(sec * 1e6, 1))
    return agg


def kernel_entry(a, frames=1):
    return {"launches_per_frame": a["launches"] / frames, "inst_per_frame": a["inst"] / frames, "thread_inst_per_frame": a["thread_inst"] / frames,
            "dram_bytes_per_frame": a["dram_bytes"] / frames, "ms_under_ncu_per_frame": a["seconds"] * 1e3 / frames,
            "lane_occupancy": a["thread_inst"] / (32.0 * a["inst"]) if a["inst"] else None,
            "issue_active_pct": a["issue_active_x_s"] / a["seconds"] if a["seconds"] else None,
            "warps_active_pct": a["warps_active_x_s"] / a["seconds"] if a["seconds"] else None,
            "dram_GBs_under_ncu": a["dram_bytes"] / a["seconds"] / 1e9 if a["seconds"] else None,
            "registers": a["regs"], "duration_us_under_ncu": a["durations_us"]}


tj_path = os.path.join(HERE, "traffic.json")
try:
    tj = json.load(open(tj_path))
    if "workloads" not in tj:
        tj = {"workloads": {}}
except Exception:
    tj = {"workloads": {}}
tj["schema"] = ("workloads[name].kernels[class]: counters of ONE frame of the per-phase schedule with the shadow pass as its own kernel "
                "(ncu --set full --clock-control none, profiles/run_ncu.sh); frame_kernel / frame_kernel_world8: the one-kernel frame (k_frame) on the "
                "whole image and on rank 0 of an 8-way scanline partition")

for rep in sorted(glob.glob(os.path.join(src, f"prof_*_{tag}.csv")) + glob.glob(os.path.join(src, f"prof_*_{tag}.ncu-rep"))):
    m = re.match(rf"prof_(.+?)(_src|_frame8|_frame)?_{re.escape(tag)}\.(csv|ncu-rep)$", os.path.basename(rep))
    if not m or m.group(2):
        continue
    w = m.group(1)
    entry = {"tag": tag, "kernels": {c: kernel_entry(a) for c, a in aggregate(rep).items()}}
    for suffix, key in (("_frame", "frame_kernel"), ("_frame8", "frame_kernel_world8")):
        rp = next((q for q in (os.path.join(src, f"prof_{w}{suffix}_{tag}.csv"), os.path.join(src, f"prof_{w}{suffix}_{tag}.ncu-rep")) if os.path.exists(q)), None)
        if rp:
            a = aggregate(rp).get("frame")
            if a:
                entry[key] = kernel_entry(a)
    tj["workloads"][w] = entry
    s1 = subprocess.run([sys.executable, os.path.join(HERE, "ncu_summary.py"), rep], capture_output=True, text=True).stdout
    with open(os.path.join(HERE, f"{tag}_{w}_summary.txt"), "w") as f:
        f.write(f"# ncu --set full --clock-control none, workload {w} (bench.py WORKLOADS), per-phase schedule with the shadow pass as its own kernel\n"
                f"# (tools/render_frames.py {w} 2 0 1 <copies> 0), all launches of the second frame in launch order, tag {tag}\n"
                "# one column per launch (cold-cache, serialised by the profiler: compare shares, not absolutes)\n")
        f.write("\n".join(l[:600] for l in s1.splitlines()) + "\n\n")
        for c, k in entry["kernels"].items():
            f.write(f"{c:18s}: {k['launches_per_frame']:.0f} launches/frame, {k['inst_per_frame'] / 1e6:9.1f} M warp instructions, lane occupancy "
                    f"{k['lane_occupancy'] * 32:.1f}/32, issue active {k['issue_active_pct']:.1f} %, warps active {k['warps_active_pct']:.1f} %, "
                    f"DRAM {k['dram_bytes_per_frame'] / 1e6:8.1f} MB/frame = {k['dram_GBs_under_ncu']:.0f} GB/s under ncu, {k['registers']:.0f} registers\n")
        for key in ("frame_kernel", "frame_kernel_world8"):
            if key in entry:
                k = entry[key]
                f.write(f"{key:18s}: {k['ms_under_ncu_per_frame']:.3f} ms under ncu, {k['inst_per_frame'] / 1e6:9.1f} M warp instructions, lane occupancy "
                        f"{k['lane_occupancy'] * 32:.1f}/32, issue active {k['issue_active_pct']:.1f} %, warps active {k['warps_active_pct']:.1f} %, "
                        f"DRAM {k['dram_bytes_per_frame'] / 1e6:8.1f} MB = {k['dram_GBs_under_ncu']:.0f} GB/s, {k['registers']:.0f} registers\n")
        srep = os.path.join(src, f"prof_{w}_src_{tag}.ncu-rep")
        if os.path.exists(srep):
            for kid, label in ((":::1", "k_trace_closest, bounce 1"), (":::2", "k_shade_queues, bounce 1")):
                s2 = subprocess.run([sys.executable, os.path.join(HERE, "ncu_lines.py"), srep, kid, "22"], capture_output=True, text=True).stdout
                f.write(f"\n## per source line: {label}\n" + "\n".join(l[:170] for l in s2.splitlines()) + "\n")
    print(w, json.dumps({c: {"Minst": round(k["inst_per_frame"] / 1e6, 1), "lanes": round(k["lane_occupancy"] * 32, 1), "dramMB": round(k["dram_bytes_per_frame"] / 1e6, 1)}
                         for c, k in entry["kernels"].items()}))

# launch list of the bench command itself (ncu --metrics gpu__time_duration.sum, profiles/run_ncu.sh launches): per-kernel shares
import collections
lc = os.path.join(src, f"launches_{tag}.csv")
if os.path.exists(lc):
    lines = [l for l in open(lc) if not l.startswith("==")]
    agg = collections.OrderedDict()
    for row in csv.DictReader(lines):
        v = fnum(row["Metric Value"]); u = row["Metric Unit"]
        v = v / 1e3 if u in ("ns", "nsecond") else (v * 1e3 if u in ("ms", "msecond") else v)
        agg.setdefault(row["Kernel Name"].split("(")[0][-44:], []).append(v)
    tot = sum(sum(v) for v in agg.values()) or 1.0
    with open(os.path.join(HERE, f"{tag}_launch_shares.txt"), "w") as f:
        f.write(f"# ncu --metrics gpu__time_duration.sum --clock-control none, python bench.py --steps 2 --warmup 3 --no-cpu-baseline --secondary none --no-host-e2e, tag {tag}\n")
        f.write("# (counter frame + warm-up + 2 timed steps + per-kernel-timing steps + e2e frames); per-launch times are cold-cache and serialised:\n"
                "# the SHARES are what must agree with bench.py's CUDA-event split\n")
        for k, v in agg.items():
            f.write(f"{k:46s} launches {len(v):4d}  total {sum(v):10.1f} us  share {100 * sum(v) / tot:5.1f}%\n")
    with open(os.path.join(HERE, f"{tag}_launches.csv"), "w") as f:
        f.writelines(lines)

json.dump(tj, open(tj_path, "w"), indent=1)
