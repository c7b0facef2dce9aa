#!/usr/bin/env python3
"""Turn the `ncu --set full` captures of tools/profile_all.sh into
  profiles/ncu_traffic.json   -- DRAM bytes per launch for every kernel of every workload (bench.py's roofline.traffic)
  profiles/<tag>_ncu_summary.md -- the metrics the write-ups quote, one table per kernel, with the binding unit named.
usage: python tools/ncu_traffic.py <dir with *.csv (ncu --page raw --csv) or *.ncu-rep> [tag]"""
import csv
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ncu_pick import WANT  # noqa: E402

UNITS = [  # (metric, label) candidates for "what binds"
    ("l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "LSU / shared-memory data pipe"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM"),
    ("sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "FMA-heavy pipe (IMAD)"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe"),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "XU pipe (POPC)"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU instruction pipe"),
]
CHUNK = 8192


def short(name):
    return name.split("(")[0].replace("void ", "").replace("rb200::", "").strip()


def to_bytes(v, unit):
    scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}
    return float(v.replace(",", "")) * scale.get(unit, 1)


def main():
    d = sys.argv[1]
    tag = sys.argv[2] if len(sys.argv) > 2 else "r2"
    traffic = {"source": "ncu --set full --clock-control none, one capture per kernel per workload (tools/profile_all.sh)",
               "workloads": {}}
    md = [f"# {tag}: `ncu --set full --clock-control none` of every hot kernel on every BASELINE workload (1 GPU)", "",
          "Command: `tools/profile_all.sh` (bench.py --workload W --steps 1, chunk 8192).  The LAST captured launch of each kernel is "
          "shown.  `binds` = the busiest unit among LSU data pipe / issue slots / DRAM / FMA-heavy / ALU / XU.", ""]
    for rep in sorted(f for f in os.listdir(d) if f.endswith(".ncu-rep") or f.endswith(".csv")):
        w = rep.rsplit(".", 1)[0]
        if rep.endswith(".csv"):
            out = open(os.path.join(d, rep)).read()
        else:
            out = subprocess.run(["ncu", "-i", os.path.join(d, rep), "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(l for l in out.splitlines() if l.startswith('"')))
        if len(rows) < 3:
            continue
        hdr, units = rows[0], rows[1]
        last = {}
        for vals in rows[2:]:
            last[short(vals[hdr.index("Kernel Name")])] = vals
        per = {}
        md += [f"## workload `{w}`", ""]
        enc_call = 0.0
        for k, vals in last.items():
            get = lambda m: vals[hdr.index(m)] if m in hdr else None  # noqa: E731
            rd = to_bytes(get("dram__bytes_read.sum"), units[hdr.index("dram__bytes_read.sum")])
            wr = to_bytes(get("dram__bytes_write.sum"), units[hdr.index("dram__bytes_write.sum")])
            per[k.split("<")[0]] = rd + wr
            if "decode" not in k:
                enc_call += rd + wr
            busy = [(float(get(m)), lab) for m, lab in UNITS if get(m) not in (None, "")]
            top = max(busy) if busy else (0, "?")
            md += [f"### `{k}` -- binds: **{top[1]} {top[0]:.0f} %**", "", "| metric | value | unit |", "|---|---|---|"]
            for m in WANT:
                if m in hdr:
                    md.append(f"| {m} | {vals[hdr.index(m)]} | {units[hdr.index(m)]} |")
            md.append("")
        per["encode_call"] = enc_call          # every kernel of one encode call (model / encode / scan / compaction)
        traffic["workloads"][w] = {"chunk_syms": CHUNK, "dram_bytes_per_launch": per}
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)      # git-ignored: captures are machine-specific records
    with open(os.path.join(ROOT, "profiles", "ncu_traffic.json"), "w") as f:
        json.dump(traffic, f, indent=1)
    with open(os.path.join(ROOT, "profiles", f"{tag}_ncu_summary.md"), "w") as f:
        f.write("\n".join(md) + "\n")
    print(json.dumps(traffic["workloads"], indent=1))


if __name__ == "__main__":
    main()
