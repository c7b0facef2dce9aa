#!/usr/bin/env python3
"""Record the kernel launches of the encode calls: for each call, every kernel as (name, grid, block, shared memory)
from torch.profiler's CUDA activity trace, and the context's launch count.  Two builds that must not differ in launch
geometry (the encoder's path, grid and workspace planning) give identical files:

    RB200_LIB=a/librans_b200.so python tools/encode_launches.py a.json
    RB200_LIB=b/librans_b200.so python tools/encode_launches.py b.json && cmp a.json b.json

Covers word, alias, byte and rans64 at chunks from 32 to 131072 and the per-block encoder with and without the model
build, in device and host memory.  Run it once per RB200_ENCODE_PATH value (the path is read once per process); with
RB200_SLICE_MIB=1 the host calls run several pipeline slices.  All calls run in ONE profiler session (many short
sessions lose kernel records), separated by a torch kernel; a call whose recorded kernels do not add up to the
context's launch count makes the script fail.  Needs a GPU.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ryg_rans_b200 as rb  # noqa: E402

N = 6_000_017                      # symbols per single-model call: a ragged last chunk at every chunk size
BLOCKS, BLOCK_SIZE = 64, 65536      # 4 MiB: within the N symbols


def trace_kernels(prof):
    """The kernels of a finished profiler session, in launch order."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    return [[e["name"], e["args"].get("grid"), e["args"].get("block"), e["args"].get("shared memory")] for e in ks]


def main(out_path):
    ctx = rb.Context(0)
    rng = np.random.default_rng(11)
    p = 1.0 / np.arange(1, 257) ** 1.1
    data = rng.choice(256, N, p=p / p.sum()).astype(np.uint8)
    d_data = torch.from_numpy(data).cuda()
    blocks = data[:BLOCKS * BLOCK_SIZE]
    d_blocks = d_data[:BLOCKS * BLOCK_SIZE]
    freqs = ctx.blocks_build_models(blocks, BLOCKS, BLOCK_SIZE)       # before the session: not an encode call
    d_freqs = torch.from_numpy(freqs.view(np.int16)).cuda()
    records = []

    def record(label, call):
        before = ctx.launches
        call()
        ctx.sync()
        torch.cuda._sleep(1000)                # the separator: the only kernel that is not the library's
        records.append({"call": label, "launches": ctx.launches - before})

    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
    prof.start()
    torch.cuda._sleep(1000)

    for coder, name, sb in ((rb.CODER_WORD, "word", 12), (rb.CODER_ALIAS, "alias", 16), (rb.CODER_BYTE, "byte", 14),
                            (rb.CODER_RANS64, "rans64", 14)):
        model = ctx.model(coder, sb, rb.SymbolStats().count_freqs(data).normalize_freqs(1 << sb).freqs)
        for chunk in (32, 2048, 4096, 8192, 65536, 131072):
            cap = ctx.encode_bound(N, chunk)
            blob = torch.empty(cap, dtype=torch.uint8, device="cuda")
            offs = torch.empty(ctx.chunk_count(N, chunk) + 1, dtype=torch.int64, device="cuda")
            record(f"{name} chunk {chunk} device",
                   lambda: ctx.encode_device(model, d_data.data_ptr(), N, chunk, blob.data_ptr(), cap, offs.data_ptr()))
            record(f"{name} chunk {chunk} host", lambda: ctx.encode_host(model, data, chunk))
        model.close()

    for chunk in (2048, 8192):
        cap = ctx.encode_bound(blocks.size, chunk)
        blob = torch.empty(cap, dtype=torch.uint8, device="cuda")
        offs = torch.empty(BLOCKS * (BLOCK_SIZE // chunk) + 1, dtype=torch.int64, device="cuda")
        built = torch.empty_like(d_freqs)
        record(f"blocks chunk {chunk} device",
               lambda: ctx.blocks_encode_device(d_blocks.data_ptr(), BLOCKS, BLOCK_SIZE, d_freqs.data_ptr(), chunk, blob.data_ptr(), cap,
                                                offs.data_ptr()))
        record(f"blocks+models chunk {chunk} device",
               lambda: ctx.blocks_model_encode_device(d_blocks.data_ptr(), BLOCKS, BLOCK_SIZE, built.data_ptr(), chunk, blob.data_ptr(),
                                                      cap, offs.data_ptr()))
        record(f"blocks chunk {chunk} host", lambda: ctx.blocks_encode_host(blocks, BLOCKS, BLOCK_SIZE, freqs, chunk))
        record(f"blocks+models chunk {chunk} host", lambda: ctx.blocks_model_encode_host(blocks, BLOCKS, BLOCK_SIZE, chunk))
    torch.cuda.synchronize()
    prof.stop()
    ctx.close()
    calls = [[]]
    for k in trace_kernels(prof):
        if "rb200::" in k[0]:
            calls[-1].append(k)
        else:
            calls.append([])
    calls = calls[1:-1]               # nothing runs before the first separator or after the last
    if len(calls) != len(records):
        raise SystemExit(f"{len(calls)} separated calls recorded for {len(records)} calls")
    for r, ks in zip(records, calls):
        if len(ks) != r["launches"]:
            raise SystemExit(f"{r['call']}: {len(ks)} kernels recorded for {r['launches']} launches")
        r["kernels"] = ks
    with open(out_path, "w") as f:
        json.dump(records, f, indent=0)
    print(f"{len(records)} calls, {sum(len(r['kernels']) for r in records)} kernel launches -> {out_path}")


if __name__ == "__main__":
    main(sys.argv[1])
