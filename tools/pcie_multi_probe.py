"""Host-path scaling probe (VERDICT r1 item 8): how much pinned-copy bandwidth do K GPUs get when they copy at the same
time?  One child process per GPU (CUDA_VISIBLE_DEVICES), bidirectional 64 MiB pinned copies (H2D on one stream, D2H on
another -- what a host-mode rb200_encode / rb200_decode call does) for about a second after a common start time.
Placements: `local` = every GPU's buffers first-touched on its own NUMA node; `alt` = odd GPUs use the OTHER node.
Run on the GPU box with all GPUs visible:  python tools/pcie_multi_probe.py  > pcie_multi_probe.jsonl"""
import json
import os
import subprocess
import sys
import time

CHILD = r'''
import json, os, sys, time
import torch
sys.path.insert(0, %(root)r)
from tools.pcie_probe import node_cpus
gpu, node, t_start, secs = int(sys.argv[1]), int(sys.argv[2]), float(sys.argv[3]), float(sys.argv[4])
nodes = node_cpus()
if node in nodes:
    os.sched_setaffinity(0, nodes[node] & os.sched_getaffinity(0) or os.sched_getaffinity(0))
n = 64 << 20
h_in = torch.empty(n, dtype=torch.uint8).pin_memory(); h_in.fill_(1)        # first touch on `node`
h_out = torch.empty(n, dtype=torch.uint8).pin_memory(); h_out.fill_(2)
dev = torch.device("cuda:0")
d_a = torch.empty(n, dtype=torch.uint8, device=dev); d_b = torch.ones(n, dtype=torch.uint8, device=dev)
s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
for _ in range(3):
    with torch.cuda.stream(s1): d_a.copy_(h_in, non_blocking=True)
    with torch.cuda.stream(s2): h_out.copy_(d_b, non_blocking=True)
torch.cuda.synchronize()
while time.time() < t_start: pass
t0 = time.perf_counter(); reps = 0
while time.perf_counter() - t0 < secs:
    for _ in range(4):
        with torch.cuda.stream(s1): d_a.copy_(h_in, non_blocking=True)
        with torch.cuda.stream(s2): h_out.copy_(d_b, non_blocking=True)
    torch.cuda.synchronize(); reps += 4
dt = time.perf_counter() - t0
print(json.dumps({"gpu": gpu, "buffer_node": node, "gbs_per_direction": n * reps / dt / 1e9}))
'''


def gpu_nodes():
    out = subprocess.run(["nvidia-smi", "--query-gpu=index,pci.bus_id", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = {}
    for line in out.strip().splitlines():
        idx, bus = [x.strip() for x in line.split(",")]
        bus = bus.lower()
        bus = bus[4:] if len(bus) > 12 else bus
        try:
            res[int(idx)] = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read())
        except Exception:  # noqa: BLE001
            res[int(idx)] = 0
    return res


def main():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    nodes = gpu_nodes()
    n_nodes = len([d for d in os.listdir("/sys/devices/system/node") if d.startswith("node") and d[4:].isdigit()])
    print(json.dumps({"gpu_numa_nodes": nodes, "numa_nodes": n_nodes}), flush=True)
    for k in (1, 2, 4, 8):
        if k > len(nodes):
            break
        for placement in ("local", "alt"):
            if placement == "alt" and (k == 1 or n_nodes < 2):
                continue
            t_start = time.time() + 25.0          # children need ~20 s to import torch on a fresh box
            procs = []
            for g in range(k):
                node = nodes[g] if placement == "local" or g % 2 == 0 else (nodes[g] + 1) % n_nodes
                env = dict(os.environ, CUDA_VISIBLE_DEVICES=str(g))
                procs.append(subprocess.Popen([sys.executable, "-c", CHILD % {"root": root}, str(g), str(node), str(t_start), "1.5"],
                                              stdout=subprocess.PIPE, text=True, env=env))
            rows = []
            for p in procs:
                out, _ = p.communicate(timeout=300)
                rows += [json.loads(l) for l in out.splitlines() if l.startswith("{")]
            tot = sum(r["gbs_per_direction"] for r in rows)
            print(json.dumps({"gpus": k, "placement": placement, "aggregate_gbs_per_direction": round(tot, 1),
                              "per_gpu": [round(r["gbs_per_direction"], 1) for r in sorted(rows, key=lambda r: r["gpu"])],
                              "buffer_nodes": [r["buffer_node"] for r in sorted(rows, key=lambda r: r["gpu"])]}), flush=True)


if __name__ == "__main__":
    main()
