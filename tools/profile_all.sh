#!/bin/bash
# ncu --set full captures of every hot kernel on every BASELINE workload (1 GPU).  Run from the repo root on the GPU machine:
#   tools/profile_all.sh <output dir>
# then: python tools/ncu_traffic.py <output dir>  (writes profiles/ncu_traffic.json and a summary)
# (reads the .csv tables this script leaves; the multi-hundred-MB .ncu-rep files are deleted on the box)
# One bench.py process per workload (--steps 1: warm-up launches + one timed step); ncu keeps the matching launches.
set -u
OUT=${1:?usage: tools/profile_all.sh <output dir>}
mkdir -p "$OUT"
for W in uniform_1GiB_word32 zipf1.1_1GiB_alias32 text_1GiB_word32 blocks_64KiB_word32 uniform_1GiB_rans64; do
    timeout 900 ncu --set full --clock-control none --import-source on \
        -k 'regex:decode|encode|block_model|histogram|compact|scan_tiles' --launch-skip 4 -c 10 \
        -o "$OUT/$W" -f python bench.py --workload "$W" --steps 1 --warmup 1 --configs none --e2e-steps 0 --no-cpu-baseline \
        > "$OUT/$W.log" 2>&1
    echo "$W: ncu exit $?" >> "$OUT/status.txt"
    # the reports run to hundreds of MB: keep the raw-metric table (what tools/ncu_traffic.py reads), drop the report
    ncu -i "$OUT/$W.ncu-rep" --page raw --csv > "$OUT/$W.csv" 2>> "$OUT/status.txt" && rm -f "$OUT/$W.ncu-rep"
done
