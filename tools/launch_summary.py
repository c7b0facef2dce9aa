#!/usr/bin/env python3
"""Summarise an ncu launch list (`--metrics gpu__time_duration.sum --csv`) of `bench.py`.

Launches are grouped by kernel name and by size class: the full-workload launches of the device-resident steps and the
slice launches of the pipelined HOST path (the e2e leg) have the same kernel names but durations two orders of magnitude
apart, so each name is split at a third of its longest launch.  Output: a markdown table on stdout.

usage: tools/launch_summary.py launches.csv
"""
import collections
import csv
import re
import sys


def short(name: str) -> str:
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    name = re.sub(r"rb200::DecPolicy<([^>]*)>", lambda m: "DecPolicy<" + m.group(1).replace(" ", "") + ">", name)
    return name if len(name) <= 96 else name[:93] + "..."


def main(path: str) -> None:
    rows = [r for r in csv.reader(open(path, newline="")) if len(r) > 10 and r[0].isdigit()]
    by_name = collections.OrderedDict()
    for r in rows:
        by_name.setdefault(short(r[4]), []).append(float(r[-1]) / 1e6)
    ours = {k: v for k, v in by_name.items() if k.startswith("rb200::")}
    other = {k: v for k, v in by_name.items() if not k.startswith("rb200::")}
    print(f"{len(rows)} launches, {sum(len(v) for v in ours.values())} of them repo kernels\n")
    print("| kernel | class | launches | mean ms | min ms | max ms |")
    print("|---|---|---|---|---|---|")
    for name, ms in ours.items():
        cut = max(ms) / 3
        for label, part in (("full workload", [m for m in ms if m >= cut]), ("host-path slices", [m for m in ms if m < cut])):
            if part:
                print(f"| `{name}` | {label} | {len(part)} | {sum(part) / len(part):.4f} | {min(part):.4f} | {max(part):.4f} |")
    n_other = sum(len(v) for v in other.values())
    t_other = sum(sum(v) for v in other.values())
    print(f"\ntorch kernels (synthetic input generation and the round-trip comparison, outside every timed region): "
          f"{n_other} launches, {t_other:.1f} ms in total")


if __name__ == "__main__":
    main(sys.argv[1])
