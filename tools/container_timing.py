"""What the container costs on the GPU, on the headline workload (1 GiB of uniform bytes, word coder, chunks of 8192,
device buffers):

  rb200_crc32 over 1 GiB of device memory (ms, and the share of 3.35 TB/s, the H100 SXM data-sheet bandwidth);
  rb200_encode against rb200_container_encode with flags 0 and RB200_CONTAINER_CRC_BLOB, alternated;
  rb200_decode against rb200_container_decode;
  host rb200_container_pack with RB200_CONTAINER_CRC_BLOB against rb200_crc32 in HOST mode, on the same blob.

With --blocks, the per-block container on the per-GPU blocks workload (8192 blocks of 64 KiB, chunks of 8192, device
buffers, per-block Zipf data with a permuted alphabet per block):

  rb200_blocks_model_encode against rb200_container_blocks_encode (models built) with flags 0 and
  RB200_CONTAINER_CRC_BLOB, alternated;
  rb200_blocks_decode against rb200_container_blocks_decode and rb200_container_blocks_decode_async, each container
  call with flags 0 and RB200_CONTAINER_CRC_BLOB, alternated; and the host time each container decode call takes to
  return.

With --single, the single-model container's decode calls on three workloads of 1 GiB in device memory, chunks of 8192:
the headline one (uniform, word), Zipf 1.1 with the alias coder at scale_bits 16, and uniform with rans64 at 14:

  rb200_decode against rb200_container_decode and rb200_container_decode_async, each container call with flags 0 and
  RB200_CONTAINER_CRC_BLOB, alternated; the host time each container decode call takes to return; and a torch.profiler
  list of the kernels of rb200_decode and of the async call (median device time per kernel), which shows the planned
  decoder against the shipped one and the launches the verdict gated out.

With --model, the single-model container's encode on the same three workloads, each with flags 0 and
RB200_CONTAINER_CRC_BLOB, alternated:

  rb200_container_encode with a prebuilt model; rb200_model_from_data + rb200_container_encode + rb200_model_destroy
  (what a caller without a model does); rb200_container_model_encode_async (the model built on the GPU); the host time
  each call takes to return; and a torch.profiler list of the async call's kernels (histogram, model kernel, encoder,
  the gated-out word encoder instance, CRCs, header).  The varlen arm: rb200_container_model_encode_varlen_async at
  *d_n = n_max = 1 GiB against the fixed async call, and at *d_n = 64 MiB with n_max = 1 GiB against the fixed call at
  64 MiB (the cost of launch shapes sized for n_max), with a torch.profiler list of the varlen call's kernels.

With --blocks-coder, per-block models for the byte and rans64 coders on 8192 blocks of 64 KiB, chunks of 8192, device
buffers, on two data sets: "skewed" (per block one symbol at p = 0.90..0.99 and a Zipf-1.1 tail over the other 255,
alphabet permuted per block) and "zipf" (the --blocks data):

  rb200_blocks_coder_model_encode (byte and rans64 at scale_bits 14) against rb200_blocks_model_encode (word), alternated;
  rb200_blocks_coder_decode against rb200_blocks_decode and against the single-model decoders of the byte and rans64
  coders (K8 / K9) on the same number of bytes, alternated; the size of each output in bytes per symbol (512 B of model
  per block included; single models at 1024 B) with byte and rans64 also at scale_bits 15 and every coder's single model
  from the whole data; and a torch.profiler list of each per-block call's kernels.
  The version 3 container of the same blocks (byte and rans64 at 14, models built, flags 0 and RB200_CONTAINER_CRC_BLOB):
  rb200_blocks_coder_decode against rb200_container_blocks_coder_decode and rb200_container_blocks_coder_decode_async,
  alternated; the host time each container call takes to return; and a torch.profiler list of the async call's kernels.

With --blocks-alias, per-block models for the alias coder on the --blocks-coder workloads (8192 blocks of 64 KiB, chunks
of 8192, device buffers, "skewed" and "zipf"): rb200_blocks_alias_model_encode against rb200_blocks_coder_model_encode
(byte) and rb200_blocks_alias_decode against rb200_blocks_coder_decode (byte), at scale_bits 14 and 15, all four in one
alternated run; the size of each output in bytes per symbol (512 B of model per block included); and a torch.profiler
list of each call's kernels.  Then the --blocks-coder container rows for the version 4 (alias) and version 3 (byte)
containers of the same blocks at 14 and 15, in one alternated run: rb200_blocks_{alias,coder}_decode against
rb200_container_blocks_{alias,coder}_decode (DEVICE) and the async call, flags 0 and RB200_CONTAINER_CRC_BLOB; the
host time each container call takes to return; and a torch.profiler list of each async call's kernels.

With --auto, rb200_container_model_encode_auto_async over {word 12, alias 16, byte 14} with a 2 % tolerance, on 1 GiB of
uniform bytes and of p = 0.99 data (symbol 0, a Zipf-1.1 tail over the rest), chunks of 8192: against the fixed call
for the pair it chose, flags 0 and RB200_CONTAINER_CRC_BLOB, alternated; the costs, the bytes per symbol against the
word coder's; and a torch.profiler list of the auto call's kernels (the choice kernel, the gated-out launches).

With --blocks-auto, rb200_container_blocks_model_encode_auto_async over {word 12, byte 14, alias 14} with a 2 %
tolerance on the --blocks-coder workloads (8192 blocks of 64 KiB, chunks of 8192, "skewed" and "zipf"): against the
fixed model-building container call for the pair it chose, flags 0 and RB200_CONTAINER_CRC_BLOB, alternated; the
device costs against rb200_choose_blocks_coder's; every candidate's blob in bytes per symbol; a torch.profiler list of
the auto call's kernels and the fixed call's; and rb200_container_blocks_any_decode_async against the chosen version's
own async decode, alternated, with its kernel list.

With --blocks-varlen, rb200_container_blocks_model_encode_varlen_async on the --blocks-auto workloads with n_blocks_max =
8192, flags 0, alternated: at *d_n_blocks = 8192 against the fixed auto call, at *d_n_blocks = 1024 against the fixed
auto call at 1024 blocks, and with the chosen pair as its one candidate against the fixed model-building container call
of that pair; a torch.profiler list of the varlen calls' kernels and their fixed twins'.

With --blocks-stored, rb200_container_blocks_stored_encode_async (version 5, incompressible blocks stored) over the
--blocks-auto candidates against rb200_container_blocks_model_encode_auto_async on uniform, Zipf, skewed and half-uniform
/ half-Zipf blocks, flags 0, alternated: bytes per symbol of both containers, encode times, and
rb200_container_blocks_stored_decode_async against rb200_container_blocks_any_decode_async on the auto container; a
torch.profiler list of the version 5 calls' kernels.

With --stored, rb200_container_stored_encode_async (version 6, incompressible chunks stored) over the --auto candidates
against rb200_container_model_encode_auto_async on 1 GiB of uniform, p = 0.99 skewed and half-uniform / half-Zipf data,
chunks of 8192, flags 0, alternated: bytes per symbol of both containers and the bytes after the header, encode times,
and rb200_container_stored_decode_async against rb200_container_decode_async on the auto container; a torch.profiler
list of the four calls' kernels.

With --stored-varlen, rb200_container_stored_encode_varlen_async (n_max = 1 GiB) on the --stored workloads, flags 0 and
RB200_CONTAINER_CRC_BLOB, alternated: at *d_n = n_max against the fixed stored call, with the candidates and with the
chosen pair alone, and at *d_n = n_max / 16 against the fixed call at that length; a torch.profiler list of both calls'
kernels.  With --blocks-stored-varlen, the same for rb200_container_blocks_stored_encode_varlen_async (n_blocks_max =
8192 blocks of 64 KiB, the sixteenth at 512 blocks) on the --blocks-stored workloads.

With --planes, rb200_container_planes_encode_async and rb200_container_planes_decode_async (version 7, one version 6
container per byte plane) against rb200_container_stored_encode_async and rb200_container_stored_decode_async (version 6)
on the same 1 GiB of bf16 and of fp32 N(0, 0.02) data in device memory, chunks of 8192, {word 12, alias 16, byte 14} at
2 %, flags 0, alternated: bytes per input byte, encode and decode times, the version 7 minus version 6 time per GiB, a
torch.profiler list of the version 7 calls' kernels, and the split and interleave kernels' rate (2n bytes moved each)
against 3.35 TB/s.

With --planes-varlen, rb200_container_planes_encode_varlen_async (n_max = 1 GiB) against rb200_container_planes_encode_async
on the --planes data, flags 0 and RB200_CONTAINER_CRC_BLOB, alternated: at *d_n = n_max and at *d_n = n_max / 16, each
against the fixed call at that length, after checking that both wrote the same bytes; varlen minus fixed in total and
per plane, and a torch.profiler list of both calls' kernels.

With --delta, rb200_container_delta_encode_async and rb200_container_delta_decode_async (version 8, the difference from a
base tensor) against the version 7 calls on the same tensor: 1 GiB of bf16 and of fp32, base = fp32 master weights of
N(0, 0.02), in = the same after one step of 1e-4 * sign * U(0, 1), as the kind; chunks of 8192, {byte 14, word 12,
alias 16} at 2 %, flags 0, alternated.  Sizes of both, encode and decode times and the version 8 minus version 7 time
per GiB, a torch.profiler list of the version 8 calls' kernels, and the delta split and interleave kernels' rate (3n
bytes moved each) beside the version 7 interleave's (2n bytes) in the same run.  The decodes write to a separate
output, so every repetition sees the same base.

Device calls are timed with CUDA events after a warm-up; the card's name and power limit are printed with the
numbers.  Every output is checked against the plain calls plus rb200_container_pack / rb200_container_blocks_pack.
    python tools/container_timing.py [--blocks | --blocks-coder | --blocks-alias | --single | --model | --auto | --blocks-auto
                                      | --blocks-varlen | --blocks-stored | --stored | --stored-varlen
                                      | --blocks-stored-varlen | --planes | --planes-varlen | --delta] [--reps 10]
                                     [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ryg_rans_b200 as rb  # noqa: E402
from ryg_rans_b200 import api  # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    import torch
    return q or torch.cuda.get_device_name(0)


def timed(fn, sync):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    sync()
    b.synchronize()
    return a.elapsed_time(b)


def stats(ts):
    ts = np.asarray(ts)
    return {"median_ms": float(np.median(ts)), "min_ms": float(ts.min()), "max_ms": float(ts.max()), "n": int(ts.size)}


def alternate(calls, sync, warmup, reps):
    """times every call `reps` times after `warmup` rounds, in alternation"""
    times = {k: [] for k in calls}
    for _ in range(warmup):
        for f in calls.values():
            timed(f, sync)
    for _ in range(reps):
        for k, f in calls.items():
            times[k].append(timed(f, sync))
    return {k: stats(v) for k, v in times.items()}


def blocks_data(n_blocks, block_size, seed):
    """per-block Zipf(0.6 + 0.1 (b % 9)) over a permuted alphabet per block, generated on the GPU"""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ranks = torch.arange(1, 257, device="cuda", dtype=torch.float64)
    probs = torch.stack([1.0 / ranks ** (0.6 + 0.1 * e) for e in range(9)])
    out = torch.empty(n_blocks * block_size, dtype=torch.uint8, device="cuda")
    step = 256
    for b0 in range(0, n_blocks, step):
        nb = min(step, n_blocks - b0)
        p = probs[torch.arange(b0, b0 + nb, device="cuda") % 9]
        r = torch.multinomial(p, block_size, replacement=True, generator=g)
        perm = torch.argsort(torch.rand(nb, 256, device="cuda", generator=g), dim=1)
        out[b0 * block_size:(b0 + nb) * block_size] = torch.gather(perm, 1, r).to(torch.uint8).reshape(-1)
    return out


def blocks(args):
    import torch
    n_blocks, block_size, chunk = 8192, 65536, 8192
    n = n_blocks * block_size
    d_in = blocks_data(n_blocks, block_size, 1234)
    ctx = rb.Context(0)
    n_chunks = n // chunk
    bound = ctx.encode_bound(n, chunk)
    cap = ctx.container_blocks_capacity(n_blocks, block_size, chunk)
    d_blob = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_offs = torch.empty(n_chunks + 1, dtype=torch.int64, device="cuda")
    d_freqs = torch.empty(n_blocks * 256, dtype=torch.int16, device="cuda")
    d_cont = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    sync = ctx.sync
    calls = {
        "blocks_model_encode": lambda: ctx.blocks_model_encode_device(d_in.data_ptr(), n_blocks, block_size, d_freqs.data_ptr(), chunk,
                                                                      d_blob.data_ptr(), bound, d_offs.data_ptr()),
        "container_blocks_encode": lambda: ctx.container_blocks_encode_device(d_in.data_ptr(), n_blocks, block_size, None, chunk, 0,
                                                                              d_cont.data_ptr(), cap),
        "container_blocks_encode_crc": lambda: ctx.container_blocks_encode_device(d_in.data_ptr(), n_blocks, block_size, None, chunk,
                                                                                  api.CONTAINER_CRC_BLOB, d_cont.data_ptr(), cap),
    }
    enc = alternate(calls, sync, args.warmup, args.reps)

    # outputs: both containers equal pack of the plain call's blob, directory and models
    calls["blocks_model_encode"]()
    sync()
    blob_bytes = int(d_offs[n_chunks].item())
    h_blob = d_blob[:blob_bytes].cpu().numpy()
    h_offs = d_offs.cpu().numpy().view(np.uint64)
    h_freqs = d_freqs.cpu().numpy().view(np.uint16).reshape(n_blocks, 256)
    identical = {}
    d_want = {}                                                       # flags -> the container in device memory
    for flags, key in ((0, "container_blocks_encode"), (api.CONTAINER_CRC_BLOB, "container_blocks_encode_crc")):
        want = api.container_blocks_pack(n_blocks, block_size, chunk, h_freqs, h_offs, h_blob, flags)
        calls[key]()
        sync()
        identical[key + "_equals_pack"] = bool(np.array_equal(d_cont[:want.size].cpu().numpy(), want))
        d_want[flags] = torch.from_numpy(want).cuda()
    size = want.size                                                  # both flags give the same size
    crc = api.CONTAINER_CRC_BLOB

    dec = {
        "blocks_decode": lambda: ctx.blocks_decode_device(d_blob.data_ptr(), blob_bytes, d_offs.data_ptr(), d_freqs.data_ptr(), n_blocks,
                                                          block_size, chunk, d_out.data_ptr()),
        "container_blocks_decode": lambda: ctx.container_blocks_decode_device(d_want[0].data_ptr(), size, d_out.data_ptr(), n),
        "container_blocks_decode_crc": lambda: ctx.container_blocks_decode_device(d_want[crc].data_ptr(), size, d_out.data_ptr(), n),
        "container_blocks_decode_async": lambda: ctx.container_blocks_decode_async(d_want[0].data_ptr(), size, d_out.data_ptr(), n),
        "container_blocks_decode_async_crc": lambda: ctx.container_blocks_decode_async(d_want[crc].data_ptr(), size, d_out.data_ptr(), n),
    }
    dtimes = alternate(dec, sync, args.warmup, args.reps)
    # host time until each container decode call returns (the synchronous call waits for the GPU; the async one enqueues)
    host = {k: [] for k in dec if k != "blocks_decode"}
    for _ in range(args.reps):
        for k in host:
            t0 = time.perf_counter()
            dec[k]()
            host[k].append((time.perf_counter() - t0) * 1e3)
            sync()
    decode_ok = {}
    for k in dec:
        d_out.zero_()
        dec[k]()
        sync()
        decode_ok[k + "_equals_input"] = bool(torch.equal(d_out[:n], d_in))

    res = {
        "card": card(),
        "workload": {"n_blocks": n_blocks, "block_size": block_size, "chunk_syms": chunk, "n": n, "blob_bytes": blob_bytes,
                     "container_bytes": size, "prefix_bytes": size - blob_bytes},
        "encode": enc,
        "decode": dtimes,
        "decode_call_host_ms": {k: stats(v) for k, v in host.items()},
        "checks": {**identical, **decode_ok},
    }
    ctx.close()
    return res


def skewed_blocks_data(n_blocks, block_size, seed):
    """per block one symbol at p = 0.90 + 0.01 (b % 10) and a Zipf-1.1 tail over the other 255, alphabet permuted per
    block, generated on the GPU"""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    tail = 1.0 / torch.arange(1, 256, device="cuda", dtype=torch.float64) ** 1.1
    tail = tail / tail.sum()
    probs = torch.stack([torch.cat([torch.tensor([0.90 + 0.01 * e], device="cuda", dtype=torch.float64), (0.10 - 0.01 * e) * tail])
                         for e in range(10)])
    out = torch.empty(n_blocks * block_size, dtype=torch.uint8, device="cuda")
    step = 256
    for b0 in range(0, n_blocks, step):
        nb = min(step, n_blocks - b0)
        p = probs[torch.arange(b0, b0 + nb, device="cuda") % 10]
        r = torch.multinomial(p, block_size, replacement=True, generator=g)
        perm = torch.argsort(torch.rand(nb, 256, device="cuda", generator=g), dim=1)
        out[b0 * block_size:(b0 + nb) * block_size] = torch.gather(perm, 1, r).to(torch.uint8).reshape(-1)
    return out


def blocks_coder(args):
    import torch
    n_blocks, block_size, chunk, sb = 8192, 65536, 8192, 14
    n = n_blocks * block_size
    n_chunks = n // chunk
    ctx = rb.Context(0)
    bound = ctx.encode_bound(n, chunk)
    sync = ctx.sync
    res = {"card": card(), "workload": {"n_blocks": n_blocks, "block_size": block_size, "chunk_syms": chunk, "n": n, "scale_bits": sb},
           "checks": {}}
    coders = {"byte": rb.CODER_BYTE, "rans64": rb.CODER_RANS64}
    for name, make in (("skewed", skewed_blocks_data), ("zipf", blocks_data)):
        d_in = make(n_blocks, block_size, 1234)
        bufs = {k: (torch.empty(bound + 16, dtype=torch.uint8, device="cuda"), torch.empty(n_chunks + 1, dtype=torch.int64, device="cuda"),
                    torch.empty(n_blocks * 256, dtype=torch.int16, device="cuda")) for k in ("word", *coders)}
        d_out = torch.empty(n + 16, dtype=torch.uint8, device="cuda")

        def menc(k, s=sb):
            b, o, f = bufs[k]
            if k == "word":
                return lambda: ctx.blocks_model_encode_device(d_in.data_ptr(), n_blocks, block_size, f.data_ptr(), chunk, b.data_ptr(), bound,
                                                              o.data_ptr())
            return lambda: ctx.blocks_coder_model_encode_device(coders[k], s, d_in.data_ptr(), n_blocks, block_size, f.data_ptr(), chunk,
                                                                b.data_ptr(), bound, o.data_ptr())
        enc = {f"{k}_blocks_model_encode": menc(k) for k in ("byte", "rans64", "word")}
        etimes = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        blob_bytes = {k: int(bufs[k][1][n_chunks].item()) for k in bufs}
        sizes = {f"{k}_per_block_sb{12 if k == 'word' else sb}": (blob_bytes[k] + 512 * n_blocks) / n for k in bufs}

        def dec_blocks(k):
            b, o, f = bufs[k]
            if k == "word":
                return lambda: ctx.blocks_decode_device(b.data_ptr(), blob_bytes[k], o.data_ptr(), f.data_ptr(), n_blocks, block_size, chunk,
                                                        d_out.data_ptr())
            return lambda: ctx.blocks_coder_decode_device(coders[k], sb, b.data_ptr(), blob_bytes[k], o.data_ptr(), f.data_ptr(), n_blocks,
                                                          block_size, chunk, d_out.data_ptr())
        dec = {f"{k}_blocks_decode": dec_blocks(k) for k in ("byte", "rans64", "word")}
        # single models from the whole data (K8 / K9 and the word decoder), on the same bytes
        single = {}
        for k, coder, s in (("byte", rb.CODER_BYTE, sb), ("rans64", rb.CODER_RANS64, sb), ("word", rb.CODER_WORD, 12)):
            m = rb.Model.from_data(ctx, coder, s, device_ptr=d_in.data_ptr(), n=n)
            b = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
            o = torch.empty(n_chunks + 1, dtype=torch.int64, device="cuda")
            ctx.encode_device(m, d_in.data_ptr(), n, chunk, b.data_ptr(), bound, o.data_ptr())
            sync()
            single[k] = (m, b, o, int(o[n_chunks].item()))
            sizes[f"{k}_single_model_sb{s}"] = (single[k][3] + 1024) / n
        for k in ("byte", "rans64"):
            m, b, o, bb = single[k]
            dec[f"{k}_single_model_decode"] = (lambda m=m, b=b, o=o, bb=bb:
                                               ctx.decode_device(m, b.data_ptr(), bb, o.data_ptr(), chunk, d_out.data_ptr(), n))
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_out.zero_()
            f()
            sync()
            res["checks"][f"{name}_{k}_equals_input"] = bool(torch.equal(d_out[:n], d_in))
        for k in coders:                                               # sizes at scale_bits 15
            menc(k, 15)()
            sync()
            sizes[f"{k}_per_block_sb15"] = (int(bufs[k][1][n_chunks].item()) + 512 * n_blocks) / n
        profile = {k: kernel_times(f, sync, args.reps) for k, f in (("byte_blocks_model_encode", menc("byte")),
                                                                     ("rans64_blocks_model_encode", menc("rans64")))}
        for k in ("byte", "rans64"):                                   # the blobs at 14 again for the decode profile
            menc(k)()
            sync()
        profile.update({k: kernel_times(dec[k], sync, args.reps) for k in ("byte_blocks_decode", "rans64_blocks_decode")})
        for m, *_ in single.values():
            m.close()
        res[name] = {"encode": etimes, "decode": dtimes, "bytes_per_symbol": sizes, "kernels": profile}
        arms = {k: (lambda flags, p, cap, c=c: ctx.container_blocks_coder_encode_device(c, sb, d_in.data_ptr(), n_blocks, block_size, None,
                                                                                        chunk, flags, p, cap),
                    ctx.container_blocks_coder_decode_device, ctx.container_blocks_coder_decode_async) for k, c in coders.items()}
        res[name].update(blocks_coder_containers(ctx, args, name, arms, d_in, d_out, dec, res["checks"]))
    ctx.close()
    return res


def blocks_alias(args):
    import torch
    n_blocks, block_size, chunk = 8192, 65536, 8192
    n = n_blocks * block_size
    n_chunks = n // chunk
    ctx = rb.Context(0)
    bound = ctx.encode_bound(n, chunk)
    sync = ctx.sync
    res = {"card": card(), "workload": {"n_blocks": n_blocks, "block_size": block_size, "chunk_syms": chunk, "n": n}, "checks": {}}
    arms = [(c, sb) for sb in (14, 15) for c in ("alias", "byte")]
    for name, make in (("skewed", skewed_blocks_data), ("zipf", blocks_data)):
        d_in = make(n_blocks, block_size, 1234)
        d_out = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        bufs = {a: (torch.empty(bound + 16, dtype=torch.uint8, device="cuda"), torch.empty(n_chunks + 1, dtype=torch.int64, device="cuda"),
                    torch.empty(n_blocks * 256, dtype=torch.int16, device="cuda")) for a in arms}

        def menc(a):
            (c, sb), (b, o, f) = a, bufs[a]
            if c == "alias":
                return lambda: ctx.blocks_alias_model_encode_device(sb, d_in.data_ptr(), n_blocks, block_size, f.data_ptr(), chunk, b.data_ptr(),
                                                                    bound, o.data_ptr())
            return lambda: ctx.blocks_coder_model_encode_device(rb.CODER_BYTE, sb, d_in.data_ptr(), n_blocks, block_size, f.data_ptr(), chunk,
                                                                b.data_ptr(), bound, o.data_ptr())

        def dec(a, bb):
            (c, sb), (b, o, f) = a, bufs[a]
            if c == "alias":
                return lambda: ctx.blocks_alias_decode_device(sb, b.data_ptr(), bb, o.data_ptr(), f.data_ptr(), n_blocks, block_size, chunk,
                                                              d_out.data_ptr())
            return lambda: ctx.blocks_coder_decode_device(rb.CODER_BYTE, sb, b.data_ptr(), bb, o.data_ptr(), f.data_ptr(), n_blocks,
                                                          block_size, chunk, d_out.data_ptr())
        enc = {f"{c}_sb{sb}_blocks_model_encode": menc((c, sb)) for c, sb in arms}
        etimes = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        blob_bytes = {a: int(bufs[a][1][n_chunks].item()) for a in arms}
        sizes = {f"{c}_sb{sb}_per_block": (blob_bytes[(c, sb)] + 512 * n_blocks) / n for c, sb in arms}
        for sb in (14, 15):                                            # both coders normalise every block the same way
            res["checks"][f"{name}_sb{sb}_models_equal_byte"] = bool(torch.equal(bufs[("alias", sb)][2], bufs[("byte", sb)][2]))
        decs = {f"{c}_sb{sb}_blocks_decode": dec((c, sb), blob_bytes[(c, sb)]) for c, sb in arms}
        dtimes = alternate(decs, sync, args.warmup, args.reps)
        for k, f in decs.items():
            d_out.zero_()
            f()
            sync()
            res["checks"][f"{name}_{k}_equals_input"] = bool(torch.equal(d_out[:n], d_in))
        profile = {k: kernel_times(f, sync, args.reps) for k, f in {**enc, **decs}.items()}
        res[name] = {"encode": etimes, "decode": dtimes, "bytes_per_symbol": sizes, "kernels": profile}

        def cenc(c, sb):
            """the encode of the version 4 (alias) or version 3 (byte) container of the same blocks, so that both planned
            decoders run side by side"""
            if c == "alias":
                return lambda flags, p, cap: ctx.container_blocks_alias_encode_device(sb, d_in.data_ptr(), n_blocks, block_size, None, chunk,
                                                                                      flags, p, cap)
            return lambda flags, p, cap: ctx.container_blocks_coder_encode_device(rb.CODER_BYTE, sb, d_in.data_ptr(), n_blocks, block_size,
                                                                                  None, chunk, flags, p, cap)
        decodes = {"alias": (ctx.container_blocks_alias_decode_device, ctx.container_blocks_alias_decode_async),
                   "byte": (ctx.container_blocks_coder_decode_device, ctx.container_blocks_coder_decode_async)}
        carms = {f"{c}_sb{sb}": (cenc(c, sb), *decodes[c]) for c, sb in arms}
        res[name].update(blocks_coder_containers(ctx, args, name, carms, d_in, d_out, decs, res["checks"]))
    ctx.close()
    return res


def blocks_coder_containers(ctx, args, name, arms, d_in, d_out, dec, checks):
    """The per-block container (version 3 or 4) of the same blocks, models built on the GPU, each arm with flags 0 and
    RB200_CONTAINER_CRC_BLOB: the plain per-block decode dec[f"{arm}_blocks_decode"] against the container's DEVICE
    decode and its async decode, alternated; the host time each container call takes to return; and a torch.profiler
    list of the async call's kernels (the planned decoder and the gated-out launches).  arms: {arm: (encode, decode,
    decode_async)}, encode(flags, out_ptr, out_cap) writes the container of d_in, decode and decode_async take
    (buf_ptr, size, out_ptr, out_cap)."""
    import torch
    n = d_in.numel()
    n_blocks, block_size, chunk = 8192, 65536, 8192
    cap = ctx.container_blocks_capacity(n_blocks, block_size, chunk)
    sync = ctx.sync
    conts = {}
    for k, (encode, _, _) in arms.items():
        for flags, tag in ((0, ""), (api.CONTAINER_CRC_BLOB, "_crc")):
            d = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
            encode(flags, d.data_ptr(), cap)
            sync()
            blob_bytes = int(d[32:40].cpu().numpy().view(np.uint64)[0])
            conts[k + tag] = (d, int(ctx.lib.dll.rb200_container_blocks_size(n_blocks, n // chunk, blob_bytes)))
    calls = {}
    for k, (_, decode, decode_async) in arms.items():
        calls[f"{k}_blocks_decode"] = dec[f"{k}_blocks_decode"]
        for tag in ("", "_crc"):
            d, size = conts[k + tag]
            calls[f"{k}_container_decode{tag}"] = lambda d=d, size=size, f=decode: f(d.data_ptr(), size, d_out.data_ptr(), n)
            calls[f"{k}_container_decode_async{tag}"] = lambda d=d, size=size, f=decode_async: f(d.data_ptr(), size, d_out.data_ptr(), n)
    times = alternate(calls, sync, args.warmup, args.reps)
    host = {k: [] for k in calls if "container" in k}
    for _ in range(args.reps):
        for k in host:
            t0 = time.perf_counter()
            calls[k]()
            host[k].append((time.perf_counter() - t0) * 1e3)
            sync()
    for k, f in calls.items():
        d_out.zero_()
        f()
        sync()
        checks[f"{name}_{k}_equals_input"] = bool(torch.equal(d_out[:n], d_in))
    profile = {f"{k}_container_decode_async": kernel_times(calls[f"{k}_container_decode_async"], sync, args.reps) for k in arms}
    return {"container_decode": times, "container_decode_call_host_ms": {k: stats(v) for k, v in host.items()},
            "container_kernels": profile}


def headline(args):
    import torch
    n, chunk = 1 << 30, 8192
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    d_in = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
    ctx = rb.Context(0)
    model = rb.Model.from_data(ctx, rb.CODER_WORD, 12, device_ptr=d_in.data_ptr(), n=n)
    n_chunks = ctx.chunk_count(n, chunk)
    bound = ctx.encode_bound(n, chunk)
    cap = ctx.container_capacity(n, chunk)
    d_blob = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_offs = torch.empty(n_chunks + 1, dtype=torch.int64, device="cuda")
    d_cont = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    sync = ctx.sync

    calls = {
        "encode": lambda: ctx.encode_device(model, d_in.data_ptr(), n, chunk, d_blob.data_ptr(), bound, d_offs.data_ptr()),
        "container_encode": lambda: ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, 0, d_cont.data_ptr(), cap),
        "container_encode_crc": lambda: ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, api.CONTAINER_CRC_BLOB,
                                                                    d_cont.data_ptr(), cap),
    }
    enc = alternate(calls, sync, args.warmup, args.reps)

    # outputs: the CRC_BLOB container (last call) equals pack of the plain encode's blob and directory
    calls["encode"]()
    sync()
    blob_bytes = int(d_offs[n_chunks].item())
    h_blob = d_blob[:blob_bytes].cpu().numpy()
    h_offs = d_offs.cpu().numpy().view(np.uint64)
    t0 = time.perf_counter()
    want = api.container_pack(rb.CODER_WORD, 12, chunk, n, model.freqs, h_offs, h_blob, api.CONTAINER_CRC_BLOB)
    t_pack = time.perf_counter() - t0
    calls["container_encode_crc"]()
    sync()
    size = want.size
    identical_encode = bool(np.array_equal(d_cont[:size].cpu().numpy(), want))
    d_want = torch.from_numpy(want).cuda()

    # rb200_crc32 over 1 GiB of device memory
    crc_times = []
    for i in range(args.warmup + args.reps):
        t = timed(lambda: ctx.crc32_device(d_in.data_ptr(), n), sync)
        if i >= args.warmup:
            crc_times.append(t)
    crc_ok = ctx.crc32_device(d_blob.data_ptr(), blob_bytes) == int(np.frombuffer(want[48:52].tobytes(), np.uint32)[0])

    # decode: plain against container (the CRC_BLOB container, both checks on the GPU)
    dec = {
        "decode": lambda: ctx.decode_device(model, d_blob.data_ptr(), blob_bytes, d_offs.data_ptr(), chunk, d_out.data_ptr(), n),
        "container_decode": lambda: ctx.container_decode_device(d_want.data_ptr(), size, d_out.data_ptr(), n),
    }
    dtimes = alternate(dec, sync, args.warmup, args.reps)
    d_out.zero_()
    dec["container_decode"]()
    identical_decode = bool(torch.equal(d_out[:n], d_in))

    # host: pack with the blob CRC (one core) against rb200_crc32 in HOST mode, same blob
    host_crc = []
    for i in range(1 + args.reps):
        t0 = time.perf_counter()
        c = ctx.crc32(h_blob)
        if i:
            host_crc.append((time.perf_counter() - t0) * 1e3)
    host_crc_ok = c == int(np.frombuffer(want[48:52].tobytes(), np.uint32)[0])

    res = {
        "card": card(),
        "workload": {"n": n, "coder": "word", "chunk_syms": chunk, "blob_bytes": blob_bytes, "container_bytes": size},
        "crc32_device_1GiB": {**stats(crc_times), "share_of_3.35TBps": n / HBM_BPS * 1e3 / float(np.median(crc_times))},
        "encode": enc,
        "decode": dtimes,
        "host_blob": {"container_pack_crc_blob_ms": t_pack * 1e3, "rb200_crc32_host_mode": stats(host_crc)},
        "checks": {"container_encode_equals_pack": identical_encode, "container_decode_equals_input": identical_decode,
                   "crc32_device_equals_header": bool(crc_ok), "crc32_host_equals_header": bool(host_crc_ok)},
    }
    model.close()
    ctx.close()
    return res


def zipf_data(n, seed, s=1.1):
    """p(r) ~ r^-s over 256 symbols, generated on the GPU in pieces"""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    p = 1.0 / torch.arange(1, 257, device="cuda", dtype=torch.float64) ** s
    cdf = (torch.cumsum(p, 0) / p.sum()).to(torch.float32)
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    step = 1 << 26
    for lo in range(0, n, step):
        u = torch.rand(min(step, n - lo), device="cuda", generator=g)
        out[lo:lo + u.numel()] = torch.searchsorted(cdf, u).clamp_(max=255).to(torch.uint8)
    return out


def kernel_times(fn, sync, reps):
    """torch.profiler over `reps` calls of fn: {kernel name: median device time in us per call, launches per call}"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
            sync()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Memcpy") and not e.name.startswith("Memset"):
            per.setdefault(e.name, []).append(e.time_range.elapsed_us())
    return {k: {"median_us": float(np.median(v)), "launches_per_call": len(v) / reps} for k, v in per.items()}


def single(args):
    import torch
    n, chunk = 1 << 30, 8192
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    workloads = (("uniform word", rb.CODER_WORD, 12, lambda: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)),
                 ("Zipf 1.1 alias 16", rb.CODER_ALIAS, 16, lambda: zipf_data(n, 1235)),
                 ("uniform rans64 14", rb.CODER_RANS64, 14, lambda: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)))
    ctx = rb.Context(0)
    sync = ctx.sync
    crc = api.CONTAINER_CRC_BLOB
    cap = ctx.container_capacity(n, chunk)
    n_chunks = ctx.chunk_count(n, chunk)
    dir_off = 64 + 1024
    boff = (dir_off + 8 * (n_chunks + 1) + 15) & ~15
    d_out = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    d_cont = {0: torch.empty(cap + 16, dtype=torch.uint8, device="cuda"), crc: torch.empty(cap + 16, dtype=torch.uint8, device="cuda")}
    res = {"card": card(), "workloads": {}, "checks": {}}
    for name, coder, sb, make in workloads:
        d_in = make()
        model = rb.Model.from_data(ctx, coder, sb, device_ptr=d_in.data_ptr(), n=n)
        for flags, d in d_cont.items():
            ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, flags, d.data_ptr(), cap)
        sync()
        head = d_cont[0][:64].cpu().numpy()
        blob_bytes = int(head[32:40].view(np.uint64)[0])
        size = boff + blob_bytes
        b0, bc = d_cont[0].data_ptr(), d_cont[crc].data_ptr()
        dec = {
            "decode": lambda: ctx.decode_device(model, b0 + boff, blob_bytes, b0 + dir_off, chunk, d_out.data_ptr(), n),
            "container_decode": lambda: ctx.container_decode_device(b0, size, d_out.data_ptr(), n),
            "container_decode_crc": lambda: ctx.container_decode_device(bc, size, d_out.data_ptr(), n),
            "container_decode_async": lambda: ctx.container_decode_async(b0, size, d_out.data_ptr(), n),
            "container_decode_async_crc": lambda: ctx.container_decode_async(bc, size, d_out.data_ptr(), n),
        }
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        host = {k: [] for k in dec if k != "decode"}
        for _ in range(args.reps):
            for k in host:
                t0 = time.perf_counter()
                dec[k]()
                host[k].append((time.perf_counter() - t0) * 1e3)
                sync()
        for k in dec:
            d_out.zero_()
            dec[k]()
            sync()
            res["checks"][f"{name}: {k}_equals_input"] = bool(torch.equal(d_out[:n], d_in))
        kernels = {k: kernel_times(dec[k], sync, args.reps) for k in ("decode", "container_decode_async", "container_decode_async_crc")}
        planned = {k: v for k, v in kernels["container_decode_async"].items() if "decode_planned_kernel" in k}
        ran = max(planned, key=lambda k: planned[k]["median_us"])
        res["workloads"][name] = {
            "n": n, "chunk_syms": chunk, "blob_bytes": blob_bytes, "container_bytes": size,
            "decode": dtimes,
            "decode_call_host_ms": {k: stats(v) for k, v in host.items()},
            "kernels": kernels,
            "planned_decoder": ran,
            "gated_out_launches": {"count": len(planned) - 1, "sum_us": sum(v["median_us"] for k, v in planned.items() if k != ran)},
        }
        model.close()
        del d_in
    ctx.close()
    return res


def model_encode(args):
    import torch
    n, chunk = 1 << 30, 8192
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    workloads = (("uniform word", rb.CODER_WORD, 12, lambda: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)),
                 ("Zipf 1.1 alias 16", rb.CODER_ALIAS, 16, lambda: zipf_data(n, 1235)),
                 ("uniform rans64 14", rb.CODER_RANS64, 14, lambda: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)))
    ctx = rb.Context(0)
    sync = ctx.sync
    crc = api.CONTAINER_CRC_BLOB
    cap = ctx.container_capacity(n, chunk)
    d_ref = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    small = 64 << 20
    d_n = torch.tensor([n, small], dtype=torch.int64, device="cuda")
    n_full, n_small = d_n.data_ptr(), d_n[1:].data_ptr()
    res = {"card": card(), "workloads": {}, "checks": {}}
    for name, coder, sb, make in workloads:
        d_in = make()
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        model = rb.Model.from_data(ctx, coder, sb, device_ptr=i, n=n)

        def from_data(flags):
            m = rb.Model.from_data(ctx, coder, sb, device_ptr=i, n=n)
            ctx.container_encode_device(m, i, n, chunk, flags, r, cap)
            m.close()

        calls = {}
        for tag, flags in (("", 0), ("_crc", crc)):
            calls["encode_prebuilt" + tag] = lambda flags=flags: ctx.container_encode_device(model, i, n, chunk, flags, r, cap)
            calls["from_data_encode" + tag] = lambda flags=flags: from_data(flags)
            calls["model_encode_async" + tag] = lambda flags=flags: ctx.container_model_encode_async(coder, sb, i, n, chunk, flags, o, cap)
            calls["varlen_n_max" + tag] = lambda flags=flags: ctx.container_model_encode_varlen_async(coder, sb, i, n_full, n, chunk, flags, o,
                                                                                                      cap)
            calls["model_encode_async_64m" + tag] = lambda flags=flags: ctx.container_model_encode_async(coder, sb, i, small, chunk, flags, r,
                                                                                                        cap)
            calls["varlen_64m_of_n_max" + tag] = lambda flags=flags: ctx.container_model_encode_varlen_async(coder, sb, i, n_small, n, chunk,
                                                                                                             flags, o, cap)
        times = alternate(calls, sync, args.warmup, args.reps)
        host = {k: [] for k in calls if not k.startswith("encode_prebuilt")}
        for _ in range(args.reps):
            for k in host:
                t0 = time.perf_counter()
                calls[k]()
                host[k].append((time.perf_counter() - t0) * 1e3)
                sync()
        for tag in ("", "_crc"):
            calls["encode_prebuilt" + tag]()
            calls["model_encode_async" + tag]()
            sync()
            head = d_out[:64].cpu().numpy()
            size = int(ctx.lib.dll.rb200_container_size(int(head[24:32].view(np.uint64)[0]), int(head[32:40].view(np.uint64)[0])))
            res["checks"][f"{name}: model_encode_async{tag}_equals_prebuilt"] = bool(torch.equal(d_out[:size], d_ref[:size]))
            for nn, varlen in ((n, "varlen_n_max"), (small, "varlen_64m_of_n_max")):
                d_out.zero_()
                ctx.container_model_encode_async(coder, sb, i, nn, chunk, 0 if not tag else crc, r, cap)
                calls[varlen + tag]()
                sync()
                head = d_out[:64].cpu().numpy()
                size = int(ctx.lib.dll.rb200_container_size(int(head[24:32].view(np.uint64)[0]), int(head[32:40].view(np.uint64)[0])))
                res["checks"][f"{name}: {varlen}{tag}_equals_fixed_call"] = bool(torch.equal(d_out[:size], d_ref[:size]))
        res["workloads"][name] = {
            "n": n, "chunk_syms": chunk,
            "encode": times,
            "call_host_ms": {k: stats(v) for k, v in host.items()},
            "kernels": {k: kernel_times(calls[k], sync, args.reps) for k in ("model_encode_async", "model_encode_async_crc", "varlen_n_max_crc",
                                                                             "varlen_64m_of_n_max_crc")},
        }
        model.close()
        del d_in
    ctx.close()
    return res


def skewed_data(n, seed, p_top=0.99):
    """symbol 0 at p_top, a Zipf-1.1 tail over symbols 1..255, generated on the GPU in pieces"""
    import torch
    tail = zipf_data(n, seed + 1)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    step = 1 << 26
    for lo in range(0, n, step):
        part = tail[lo:lo + step]
        u = torch.rand(part.numel(), device="cuda", generator=g)
        part.copy_(torch.where(u < p_top, torch.zeros_like(part), part % 255 + 1))
    return tail


def auto_encode(args):
    """rb200_container_model_encode_auto_async over {word 12, alias 16, byte 14} (2 % tolerance) against the fixed call
    for the pair it chose, on uniform bytes and on p = 0.99 data"""
    import torch
    n, chunk, tol = 1 << 30, 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    workloads = (("uniform", lambda: torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)),
                 ("p = 0.99", lambda: skewed_data(n, 1236)))
    ctx = rb.Context(0)
    sync = ctx.sync
    crc = api.CONTAINER_CRC_BLOB
    cap = ctx.container_capacity(n, chunk)
    d_ref = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "candidates": ["word 12", "alias 16", "byte 14"], "tolerance_ppm": tol, "workloads": {}, "checks": {}}

    def container_size(d):
        head = d[:64].cpu().numpy()
        return int(ctx.lib.dll.rb200_container_size(int(head[24:32].view(np.uint64)[0]), int(head[32:40].view(np.uint64)[0])))

    for name, make in workloads:
        d_in = make()
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        ctx.container_model_encode_auto_async(cands, tol, i, n, chunk, 0, o, cap)
        sync()
        head = d_out[:64].cpu().numpy()
        coder, sb = int(head[6]), int(head[7])
        blob_auto = int(head[32:40].view(np.uint64)[0])
        k, costs = api.choose_coder(ctx.histogram_device(i, n), n, chunk, cands, tol)
        res["checks"][f"{name}: header_is_the_rule's_choice"] = cands[k] == api.CANDIDATE(coder, sb)
        calls = {}
        for tag, flags in (("", 0), ("_crc", crc)):
            calls["auto" + tag] = lambda flags=flags: ctx.container_model_encode_auto_async(cands, tol, i, n, chunk, flags, o, cap)
            calls["fixed_chosen" + tag] = lambda flags=flags: ctx.container_model_encode_async(coder, sb, i, n, chunk, flags, r, cap)
        times = alternate(calls, sync, args.warmup, args.reps)
        for tag in ("", "_crc"):
            calls["auto" + tag]()
            calls["fixed_chosen" + tag]()
            sync()
            size = container_size(d_out)
            res["checks"][f"{name}: auto{tag}_equals_fixed_call"] = bool(torch.equal(d_out[:size], d_ref[:size]))
        ctx.container_model_encode_async(rb.CODER_WORD, 12, i, n, chunk, 0, r, cap)
        sync()
        blob_word = int(d_ref[32:40].cpu().numpy().view(np.uint64)[0])
        kernels = {k: kernel_times(calls[k], sync, args.reps) for k in ("auto_crc", "fixed_chosen_crc")}
        res["workloads"][name] = {
            "n": n, "chunk_syms": chunk, "chosen": {"coder": coder, "scale_bits": sb},
            "costs": [int(c) for c in costs], "blob_bytes": blob_auto,
            "bytes_per_symbol": blob_auto / n, "word12_bytes_per_symbol": blob_word / n,
            "encode": times,
            "auto_minus_fixed_median_us": {tag or "flags 0": 1e3 * (times["auto" + tag]["median_ms"] - times["fixed_chosen" + tag]["median_ms"])
                                           for tag in ("", "_crc")},
            "kernels": kernels,
        }
        del d_in
    ctx.close()
    return res


def blocks_auto(args):
    """rb200_container_blocks_model_encode_auto_async over {word 12, byte 14, alias 14} (2 % tolerance) against the fixed
    model-building call for the pair it chose, on the --blocks-coder workloads; every candidate's bytes per symbol; a
    kernel split of the auto call; rb200_container_blocks_any_decode_async against the version's own async decode"""
    import torch
    n_blocks, block_size, chunk, tol = 8192, 65536, 8192, 20000
    n = n_blocks * block_size
    W, B, A = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS
    cands = [api.CANDIDATE(W, 12), api.CANDIDATE(B, 14), api.CANDIDATE(A, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    crc = api.CONTAINER_CRC_BLOB
    cap = ctx.container_blocks_capacity(n_blocks, block_size, chunk)
    d_ref = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "workload": {"n_blocks": n_blocks, "block_size": block_size, "chunk_syms": chunk, "n": n},
           "candidates": ["word 12", "byte 14", "alias 14"], "tolerance_ppm": tol, "workloads": {}, "checks": {}}

    def fixed(coder, sb, i, o, flags):
        if coder == W:
            return lambda: ctx.container_blocks_encode_device(i, n_blocks, block_size, None, chunk, flags, o, cap)
        if coder == A:
            return lambda: ctx.container_blocks_alias_encode_device(sb, i, n_blocks, block_size, None, chunk, flags, o, cap)
        return lambda: ctx.container_blocks_coder_encode_device(coder, sb, i, n_blocks, block_size, None, chunk, flags, o, cap)

    def head(d):
        h = d[:64].cpu().numpy()
        return int(h[4:6].view(np.uint16)[0]), int(h[6]), int(h[7]), int(h[32:40].view(np.uint64)[0])

    boff = (64 + 512 * n_blocks + 8 * (n // chunk + 1) + 15) & ~15
    for name, make in (("skewed", skewed_blocks_data), ("zipf", blocks_data)):
        d_in = make(n_blocks, block_size, 4321)
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        ctx.container_blocks_model_encode_auto_async(cands, tol, i, n_blocks, block_size, chunk, 0, o, cap)
        sync()
        version, coder, sb, blob_auto = head(d_out)
        costs = [int(c) for c in ctx.container_blocks_auto_costs(len(cands))]
        counts = torch.stack([torch.bincount(d_in[b * block_size:(b + 1) * block_size].long(), minlength=256) for b in range(n_blocks)])
        k, host_costs = api.choose_blocks_coder(counts.cpu().numpy().astype(np.uint32), block_size, chunk, cands, tol)
        res["checks"][f"{name}: choice_and_costs_are_the_host_rule's"] = cands[k] == api.CANDIDATE(coder, sb) and costs == [int(c) for c in host_costs]
        calls = {}
        for tag, flags in (("", 0), ("_crc", crc)):
            calls["auto" + tag] = lambda flags=flags: ctx.container_blocks_model_encode_auto_async(cands, tol, i, n_blocks, block_size, chunk,
                                                                                                  flags, o, cap)
            calls["fixed_chosen" + tag] = fixed(coder, sb, i, r, flags)
        times = alternate(calls, sync, args.warmup, args.reps)
        for tag in ("", "_crc"):
            calls["auto" + tag]()
            calls["fixed_chosen" + tag]()
            sync()
            size = boff + head(d_out)[3]
            res["checks"][f"{name}: auto{tag}_equals_fixed_call"] = bool(torch.equal(d_out[:size], d_ref[:size]))
        per_candidate = {}
        for c, cost in zip(cands, costs):
            fixed(c >> 8, c & 0xFF, i, r, 0)()
            sync()
            per_candidate[f"{c >> 8}/{c & 0xFF}"] = {"bytes_per_symbol": head(d_ref)[3] / n, "cost_per_symbol": cost / n}
        kernels = kernel_times(calls["auto_crc"], sync, args.reps)
        kernels_fixed = kernel_times(calls["fixed_chosen_crc"], sync, args.reps)
        # decode: the container of the chosen version, by the any call and by the version's own async decode
        calls["auto_crc"]()
        sync()
        own = {2: ctx.container_blocks_decode_async, 3: ctx.container_blocks_coder_decode_async, 4: ctx.container_blocks_alias_decode_async}[version]
        dec = {"any_decode_async": lambda: ctx.container_blocks_any_decode_async(o, cap, d_dec.data_ptr(), n),
               "own_decode_async": lambda: own(o, cap, d_dec.data_ptr(), n)}
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_dec.zero_()
            f()
            sync()
            res["checks"][f"{name}: {k}_round_trip"] = bool(torch.equal(d_dec[:n], d_in[:n]))
        dkernels = kernel_times(dec["any_decode_async"], sync, args.reps)
        res["workloads"][name] = {
            "chosen": {"version": version, "coder": coder, "scale_bits": sb}, "costs": costs,
            "bytes_per_symbol": blob_auto / n, "candidates": per_candidate,
            "encode": times,
            "auto_minus_fixed_median_us": {tag or "flags 0": 1e3 * (times["auto" + tag]["median_ms"] - times["fixed_chosen" + tag]["median_ms"])
                                           for tag in ("", "_crc")},
            "auto_crc_kernels": kernels, "fixed_chosen_crc_kernels": kernels_fixed,
            "decode": dtimes,
            "any_minus_own_median_us": 1e3 * (dtimes["any_decode_async"]["median_ms"] - dtimes["own_decode_async"]["median_ms"]),
            "any_decode_kernels": dkernels,
        }
        del d_in
    ctx.close()
    return res


def blocks_varlen(args):
    """rb200_container_blocks_model_encode_varlen_async (n_blocks_max 8192) against the fixed calls: the auto call at 8192
    and at 1024 blocks, and, with one candidate, the fixed model-building call of the pair the auto call chose"""
    import torch
    nb_max, block_size, chunk, tol = 8192, 65536, 8192, 20000
    W, B, A = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS
    cands = [api.CANDIDATE(W, 12), api.CANDIDATE(B, 14), api.CANDIDATE(A, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    cap = ctx.container_blocks_capacity(nb_max, block_size, chunk)
    d_ref = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_nb = torch.tensor([nb_max, 1024], dtype=torch.int32, device="cuda")
    res = {"card": card(), "workload": {"n_blocks_max": nb_max, "block_size": block_size, "chunk_syms": chunk},
           "candidates": ["word 12", "byte 14", "alias 14"], "tolerance_ppm": tol, "workloads": {}, "checks": {}}

    def size(d):
        h = d[:64].cpu().numpy()
        nb, blob = int(h[56:60].view(np.uint32)[0]), int(h[32:40].view(np.uint64)[0])
        return ((64 + 512 * nb + 8 * (nb * block_size // chunk + 1) + 15) & ~15) + blob

    for name, make in (("skewed", skewed_blocks_data), ("zipf", blocks_data)):
        d_in = make(nb_max, block_size, 4321)
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        ctx.container_blocks_model_encode_auto_async(cands, tol, i, nb_max, block_size, chunk, 0, r, cap)
        sync()
        h = d_ref[:8].cpu().numpy()
        coder, sb = int(h[6]), int(h[7])
        fixed_pair = {W: lambda: ctx.container_blocks_encode_device(i, nb_max, block_size, None, chunk, 0, r, cap),
                      A: lambda: ctx.container_blocks_alias_encode_device(sb, i, nb_max, block_size, None, chunk, 0, r, cap)}.get(
            coder, lambda: ctx.container_blocks_coder_encode_device(coder, sb, i, nb_max, block_size, None, chunk, 0, r, cap))
        arms = {  # (varlen call, fixed call)
            "max": (lambda: ctx.container_blocks_model_encode_varlen_async(cands, tol, i, d_nb.data_ptr(), nb_max, block_size, chunk, 0, o, cap),
                    lambda: ctx.container_blocks_model_encode_auto_async(cands, tol, i, nb_max, block_size, chunk, 0, r, cap)),
            "1024": (lambda: ctx.container_blocks_model_encode_varlen_async(cands, tol, i, d_nb[1:].data_ptr(), nb_max, block_size, chunk, 0, o,
                                                                            cap),
                     lambda: ctx.container_blocks_model_encode_auto_async(cands, tol, i, 1024, block_size, chunk, 0, r, cap)),
            "one_candidate": (lambda: ctx.container_blocks_model_encode_varlen_async([api.CANDIDATE(coder, sb)], 0, i, d_nb.data_ptr(), nb_max,
                                                                                     block_size, chunk, 0, o, cap),
                              fixed_pair),
        }
        out = {"chosen": {"coder": coder, "scale_bits": sb}}
        for arm, (varlen, fixed) in arms.items():
            times = alternate({"varlen": varlen, "fixed": fixed}, sync, args.warmup, args.reps)
            varlen()
            fixed()
            sync()
            n = size(d_ref)
            res["checks"][f"{name} {arm}: varlen_equals_fixed_call"] = size(d_out) == n and bool(torch.equal(d_out[:n], d_ref[:n]))
            out[arm] = {"encode": times, "varlen_minus_fixed_median_us": 1e3 * (times["varlen"]["median_ms"] - times["fixed"]["median_ms"]),
                        "varlen_kernels": kernel_times(varlen, sync, args.reps), "fixed_kernels": kernel_times(fixed, sync, args.reps)}
        res["workloads"][name] = out
        del d_in
    ctx.close()
    return res


def uniform_blocks(nb, bs, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randint(0, 256, (nb * bs,), dtype=torch.uint8, device="cuda", generator=g)


def half_blocks(nb, bs, seed):
    """uniform blocks between per-block Zipf ones"""
    d = blocks_data(nb, bs, seed).view(nb, bs)
    d[0::2] = uniform_blocks(nb // 2, bs, seed + 1).view(nb // 2, bs)
    return d.reshape(-1)


def half_data(n, chunk, seed):
    """runs of 3 chunks + 1000 symbols, uniform and Zipf in turn: every boundary falls inside a chunk"""
    import torch
    run = 3 * chunk + 1000
    m = -(-n // (2 * run)) * 2 * run
    d = zipf_data(m, seed).view(-1, 2, run)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed + 1)
    d[:, 0, :] = torch.randint(0, 256, (d.shape[0], run), dtype=torch.uint8, device="cuda", generator=g)
    return d.reshape(-1)[:n]


# the stored encodes' workloads: (name, make(n_blocks, block_size, seed)) and (name, make(n, chunk_syms, seed))
STORED_BLOCKS_WORKLOADS = (("uniform", uniform_blocks), ("zipf", blocks_data), ("skewed", skewed_blocks_data), ("half_uniform_zipf", half_blocks))
STORED_WORKLOADS = (("uniform", lambda n, chunk, seed: uniform_blocks(1, n, seed)), ("p = 0.99", lambda n, chunk, seed: skewed_data(n, seed)),
                    ("half_uniform_zipf", half_data))


def blocks_stored(args):
    """rb200_container_blocks_stored_encode_async (version 5) over {word 12, byte 14, alias 14} (2 % tolerance) against
    rb200_container_blocks_model_encode_auto_async, on uniform, Zipf, skewed and half-uniform / half-Zipf blocks: bytes
    per symbol of both containers, encode times, the version 5 decode against rb200_container_blocks_any_decode_async on
    the auto container, and a kernel split of both version 5 calls"""
    import torch
    n_blocks, block_size, chunk, tol = 8192, 65536, 8192, 20000
    n = n_blocks * block_size
    W, B, A = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS
    cands = [api.CANDIDATE(W, 12), api.CANDIDATE(B, 14), api.CANDIDATE(A, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    cap = ctx.container_blocks_capacity(n_blocks, block_size, chunk)
    bound = api.container_blocks_stored_bound(n_blocks, block_size, chunk)
    d_auto = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_st = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "workload": {"n_blocks": n_blocks, "block_size": block_size, "chunk_syms": chunk, "n": n},
           "candidates": ["word 12", "byte 14", "alias 14"], "tolerance_ppm": tol, "bound_bytes_per_symbol": bound / n,
           "workloads": {}, "checks": {}}

    def size(d):
        h = d[:64].cpu().numpy()
        return ((64 + 512 * n_blocks + 8 * (n // chunk + 1) + 15) & ~15) + int(h[32:40].view(np.uint64)[0]), int(h[6]), int(h[7])

    for name, make in STORED_BLOCKS_WORKLOADS:
        d_in = make(n_blocks, block_size, 4321)
        i, a, o = d_in.data_ptr(), d_auto.data_ptr(), d_st.data_ptr()
        enc = {"stored_encode": lambda: ctx.container_blocks_stored_encode_async(cands, tol, i, n_blocks, block_size, chunk, 0, o, bound),
               "auto_encode": lambda: ctx.container_blocks_model_encode_auto_async(cands, tol, i, n_blocks, block_size, chunk, 0, a, cap)}
        times = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        st_size, coder, sb = size(d_st)
        auto_size = size(d_auto)[0]
        rows = d_st[64:64 + 512 * n_blocks].view(torch.int16).view(n_blocks, 256)
        stored = int((rows == 0).all(dim=1).sum().item())
        res["checks"][f"{name}: stored_container_within_bound"] = st_size <= bound
        dec = {"stored_decode_async": lambda: ctx.container_blocks_stored_decode_async(o, bound, d_dec.data_ptr(), n),
               "any_decode_async_on_auto": lambda: ctx.container_blocks_any_decode_async(a, cap, d_dec.data_ptr(), n)}
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_dec.zero_()
            f()
            sync()
            res["checks"][f"{name}: {k}_round_trip"] = bool(torch.equal(d_dec[:n], d_in[:n]))
        res["workloads"][name] = {
            "chosen": {"coder": coder, "scale_bits": sb}, "stored_blocks": stored,
            "bytes_per_symbol": {"stored": st_size / n, "auto": auto_size / n},
            "encode": times, "stored_minus_auto_encode_median_us": 1e3 * (times["stored_encode"]["median_ms"] - times["auto_encode"]["median_ms"]),
            "decode": dtimes,
            "stored_minus_any_decode_median_us": 1e3 * (dtimes["stored_decode_async"]["median_ms"] - dtimes["any_decode_async_on_auto"]["median_ms"]),
            "stored_encode_kernels": kernel_times(enc["stored_encode"], sync, args.reps),
            "auto_encode_kernels": kernel_times(enc["auto_encode"], sync, args.reps),
            "stored_decode_kernels": kernel_times(dec["stored_decode_async"], sync, args.reps),
            "any_decode_kernels": kernel_times(dec["any_decode_async_on_auto"], sync, args.reps),
        }
        del d_in
    ctx.close()
    return res


def stored(args):
    """rb200_container_stored_encode_async (version 6) over {word 12, alias 16, byte 14} (2 % tolerance) against
    rb200_container_model_encode_auto_async, on uniform, p = 0.99 skewed and half-uniform / half-Zipf data: bytes per
    symbol of both containers, encode times, the version 6 decode against rb200_container_decode_async on the auto
    container, and a kernel split of all four calls"""
    import torch
    n, chunk, tol = 1 << 30, 8192, 20000
    n_chunks = n // chunk
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    cap = ctx.container_capacity(n, chunk)
    bound = api.container_stored_bound(n, chunk)
    d_auto = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_st = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    bitmap = (1088 + 8 * (n_chunks + 1) + 15) & ~15
    v6_boff, v1_boff = bitmap + 16 * ((n_chunks + 127) // 128), bitmap
    res = {"card": card(), "workload": {"n": n, "chunk_syms": chunk}, "candidates": ["word 12", "alias 16", "byte 14"], "tolerance_ppm": tol,
           "bound_bytes_per_symbol": bound / n, "workloads": {}, "checks": {}}

    def blob_bytes(d):
        h = d[:64].cpu().numpy()
        return int(h[32:40].view(np.uint64)[0]), int(h[6]), int(h[7])

    for name, make in STORED_WORKLOADS:
        d_in = make(n, chunk, 4321)[:n].contiguous()
        i, a, o = d_in.data_ptr(), d_auto.data_ptr(), d_st.data_ptr()
        enc = {"stored_encode": lambda: ctx.container_stored_encode_async(cands, tol, i, n, chunk, 0, o, bound),
               "auto_encode": lambda: ctx.container_model_encode_auto_async(cands, tol, i, n, chunk, 0, a, cap)}
        times = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        st_blob, coder, sb = blob_bytes(d_st)
        auto_blob = blob_bytes(d_auto)[0]
        bits = d_st[bitmap:bitmap + 4 * ((n_chunks + 31) // 32)].cpu().numpy().view(np.uint32)
        stored_chunks = int(sum(bin(int(w)).count("1") for w in bits))
        res["checks"][f"{name}: stored_container_within_bound"] = v6_boff + st_blob <= bound
        if stored_chunks == 0:
            res["checks"][f"{name}: nothing_stored_blob_equals_auto"] = bool(
                torch.equal(d_st[v6_boff:v6_boff + st_blob], d_auto[v1_boff:v1_boff + auto_blob]))
        dec = {"stored_decode_async": lambda: ctx.container_stored_decode_async(o, bound, d_dec.data_ptr(), n),
               "decode_async_on_auto": lambda: ctx.container_decode_async(a, cap, d_dec.data_ptr(), n)}
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_dec.zero_()
            f()
            sync()
            res["checks"][f"{name}: {k}_round_trip"] = bool(torch.equal(d_dec[:n], d_in[:n]))
        res["workloads"][name] = {
            "chosen": {"coder": coder, "scale_bits": sb}, "stored_chunks": stored_chunks, "n_chunks": n_chunks,
            "bytes_per_symbol": {"stored": (v6_boff + st_blob) / n, "auto": (v1_boff + auto_blob) / n},
            "bytes_after_header": {"stored": v6_boff + st_blob - 64, "auto": v1_boff + auto_blob - 64},
            "encode": times, "stored_minus_auto_encode_median_us": 1e3 * (times["stored_encode"]["median_ms"] - times["auto_encode"]["median_ms"]),
            "decode": dtimes,
            "stored_minus_v1_decode_median_us": 1e3 * (dtimes["stored_decode_async"]["median_ms"] - dtimes["decode_async_on_auto"]["median_ms"]),
            "stored_encode_kernels": kernel_times(enc["stored_encode"], sync, args.reps),
            "auto_encode_kernels": kernel_times(enc["auto_encode"], sync, args.reps),
            "stored_decode_kernels": kernel_times(dec["stored_decode_async"], sync, args.reps),
            "v1_decode_kernels": kernel_times(dec["decode_async_on_auto"], sync, args.reps),
        }
        del d_in
    ctx.close()
    return res


def varlen_arms(res, name, arms, sync, args, same):
    """times every arm's (varlen, fixed) pair, alternated, at flags 0 and with the blob CRC; checks that the varlen
    call wrote the fixed call's container (same()) and profiles both calls of every flags-0 arm"""
    out = {}
    for arm, (varlen, fixed) in arms.items():
        for tag, flags in (("", 0), ("_crc", api.CONTAINER_CRC_BLOB)):
            v, f = (lambda v=varlen, flags=flags: v(flags)), (lambda f=fixed, flags=flags: f(flags))
            times = alternate({"varlen": v, "fixed": f}, sync, args.warmup, args.reps)
            v()
            f()
            sync()
            res["checks"][f"{name} {arm}{tag}: varlen_equals_fixed_call"] = same()
            out[arm + tag] = {"encode": times, "varlen_minus_fixed_median_us": 1e3 * (times["varlen"]["median_ms"] - times["fixed"]["median_ms"])}
            if not tag:
                out[arm]["varlen_kernels"] = kernel_times(v, sync, args.reps)
                out[arm]["fixed_kernels"] = kernel_times(f, sync, args.reps)
    return out


def stored_varlen(args):
    """rb200_container_stored_encode_varlen_async (n_max = 1 GiB, chunks of 8192) against the fixed stored call on the
    --stored workloads: at *d_n = n_max with the list and with the pair it chose as the one candidate, and at
    *d_n = n_max / 16 against the fixed call at that length"""
    import torch
    n_max, chunk, tol = 1 << 30, 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    bound = api.container_stored_bound(n_max, chunk)
    d_ref = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n_max, n_max // 16], dtype=torch.int64, device="cuda")
    res = {"card": card(), "workload": {"n_max": n_max, "chunk_syms": chunk}, "candidates": ["word 12", "alias 16", "byte 14"],
           "tolerance_ppm": tol, "workloads": {}, "checks": {}}

    def size(d):
        h = d[:64].cpu().numpy()
        n_chunks = int(h[24:32].view(np.uint64)[0])
        bitmap = (1088 + 8 * (n_chunks + 1) + 15) & ~15
        return bitmap + 16 * ((n_chunks + 127) // 128) + int(h[32:40].view(np.uint64)[0])

    def same():
        n = size(d_ref)
        return size(d_out) == n and bool(torch.equal(d_out[:n], d_ref[:n]))

    for name, make in STORED_WORKLOADS:
        d_in = make(n_max, chunk, 4321)[:n_max].contiguous()
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        ctx.container_stored_encode_async(cands, tol, i, n_max, chunk, 0, r, bound)
        sync()
        one = [api.CANDIDATE(int(d_ref[6].item()), int(d_ref[7].item()))]
        arms = {  # (varlen call, fixed call), each taking flags
            "bound": (lambda fl: ctx.container_stored_encode_varlen_async(cands, tol, i, d_n.data_ptr(), n_max, chunk, fl, o, bound),
                      lambda fl: ctx.container_stored_encode_async(cands, tol, i, n_max, chunk, fl, r, bound)),
            "bound_one_candidate": (lambda fl: ctx.container_stored_encode_varlen_async(one, 0, i, d_n.data_ptr(), n_max, chunk, fl, o, bound),
                                    lambda fl: ctx.container_stored_encode_async(one, 0, i, n_max, chunk, fl, r, bound)),
            "sixteenth": (lambda fl: ctx.container_stored_encode_varlen_async(cands, tol, i, d_n[1:].data_ptr(), n_max, chunk, fl, o, bound),
                          lambda fl: ctx.container_stored_encode_async(cands, tol, i, n_max // 16, chunk, fl, r, bound)),
        }
        res["workloads"][name] = {"chosen": {"coder": one[0] >> 8, "scale_bits": one[0] & 0xFF},
                                  **varlen_arms(res, name, arms, sync, args, same)}
        del d_in
    ctx.close()
    return res


def blocks_stored_varlen(args):
    """rb200_container_blocks_stored_encode_varlen_async (n_blocks_max = 8192 blocks of 64 KiB, chunks of 8192) against
    the fixed stored call on the --blocks-stored workloads: at *d_n_blocks = 8192 with the list and with the pair it
    chose as the one candidate, and at *d_n_blocks = 512 against the fixed call at 512 blocks"""
    import torch
    nb_max, block_size, chunk, tol = 8192, 65536, 8192, 20000
    W, B, A = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS
    cands = [api.CANDIDATE(W, 12), api.CANDIDATE(B, 14), api.CANDIDATE(A, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    bound = api.container_blocks_stored_bound(nb_max, block_size, chunk)
    d_ref = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
    d_nb = torch.tensor([nb_max, nb_max // 16], dtype=torch.int32, device="cuda")
    res = {"card": card(), "workload": {"n_blocks_max": nb_max, "block_size": block_size, "chunk_syms": chunk},
           "candidates": ["word 12", "byte 14", "alias 14"], "tolerance_ppm": tol, "workloads": {}, "checks": {}}

    def size(d):
        h = d[:64].cpu().numpy()
        nb, blob = int(h[56:60].view(np.uint32)[0]), int(h[32:40].view(np.uint64)[0])
        return ((64 + 512 * nb + 8 * (nb * block_size // chunk + 1) + 15) & ~15) + blob

    def same():
        n = size(d_ref)
        return size(d_out) == n and bool(torch.equal(d_out[:n], d_ref[:n]))

    for name, make in STORED_BLOCKS_WORKLOADS:
        d_in = make(nb_max, block_size, 4321)
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()
        ctx.container_blocks_stored_encode_async(cands, tol, i, nb_max, block_size, chunk, 0, r, bound)
        sync()
        one = [api.CANDIDATE(int(d_ref[6].item()), int(d_ref[7].item()))]
        arms = {
            "bound": (lambda fl: ctx.container_blocks_stored_encode_varlen_async(cands, tol, i, d_nb.data_ptr(), nb_max, block_size, chunk, fl,
                                                                                 o, bound),
                      lambda fl: ctx.container_blocks_stored_encode_async(cands, tol, i, nb_max, block_size, chunk, fl, r, bound)),
            "bound_one_candidate": (lambda fl: ctx.container_blocks_stored_encode_varlen_async(one, 0, i, d_nb.data_ptr(), nb_max, block_size,
                                                                                               chunk, fl, o, bound),
                                    lambda fl: ctx.container_blocks_stored_encode_async(one, 0, i, nb_max, block_size, chunk, fl, r, bound)),
            "sixteenth": (lambda fl: ctx.container_blocks_stored_encode_varlen_async(cands, tol, i, d_nb[1:].data_ptr(), nb_max, block_size,
                                                                                     chunk, fl, o, bound),
                          lambda fl: ctx.container_blocks_stored_encode_async(cands, tol, i, nb_max // 16, block_size, chunk, fl, r, bound)),
        }
        res["workloads"][name] = {"chosen": {"coder": one[0] >> 8, "scale_bits": one[0] & 0xFF},
                                  **varlen_arms(res, name, arms, sync, args, same)}
        del d_in
    ctx.close()
    return res


def planes(args):
    """version 7 against version 6 on the same bytes: bf16 and fp32 N(0, 0.02), 1 GiB each"""
    import torch
    n, chunk, tol = 1 << 30, 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    v6_bound = api.container_stored_bound(n, chunk)
    d_v6 = torch.empty(v6_bound + 16, dtype=torch.uint8, device="cuda")
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "workload": {"n": n, "chunk_syms": chunk}, "candidates": ["word 12", "alias 16", "byte 14"], "tolerance_ppm": tol,
           "workloads": {}, "checks": {}}
    gen = torch.Generator(device="cuda").manual_seed(4321)
    for name, dtype, w in (("bf16", torch.bfloat16, 2), ("fp32", torch.float32, 4)):
        d_in = (torch.randn(n // w, device="cuda", generator=gen) * 0.02).to(dtype).view(torch.uint8)
        bound = api.container_planes_bound(n, w, chunk)
        d_v7 = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
        i, o6, o7, dd = d_in.data_ptr(), d_v6.data_ptr(), d_v7.data_ptr(), d_dec.data_ptr()
        enc = {"v7_encode": lambda: ctx.container_planes_encode_async(cands, tol, w, i, n, chunk, 0, o7, bound),
               "v6_encode": lambda: ctx.container_stored_encode_async(cands, tol, i, n, chunk, 0, o6, v6_bound)}
        times = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        h7, h6 = d_v7[:64 + 16 * w].cpu().numpy(), d_v6[:64].cpu().numpy()
        size7 = 64 + 16 * w + int(h7[32:40].view(np.uint64)[0])
        n_chunks = int(h6[24:32].view(np.uint64)[0])
        size6 = ((1088 + 8 * (n_chunks + 1) + 15) & ~15) + 16 * ((n_chunks + 127) // 128) + int(h6[32:40].view(np.uint64)[0])
        table = h7[64:].view(np.uint64).reshape(w, 2)
        res["checks"][f"{name}: v7_within_bound"] = size7 <= bound
        dec = {"v7_decode": lambda: ctx.container_planes_decode_async(w, o7, size7, dd, n),
               "v6_decode": lambda: ctx.container_stored_decode_async(o6, size6, dd, n)}
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_dec.zero_()
            f()
            sync()
            res["checks"][f"{name}: {k}_round_trip"] = bool(torch.equal(d_dec[:n], d_in))
        ek = kernel_times(enc["v7_encode"], sync, args.reps)
        dk = kernel_times(dec["v7_decode"], sync, args.reps)

        def rate(kernels, part):
            us = sum(v["median_us"] * v["launches_per_call"] for k, v in kernels.items() if part in k)
            return {"us": us, "TB_per_s": 2 * n / us / 1e6 if us else None, "share_of_3.35_TB_per_s": 2 * n / us / 1e6 / 3.35 if us else None}

        res["workloads"][name] = {
            "bytes_per_input_byte": {"v7": size7 / n, "v6": size6 / n},
            "plane_bytes_per_symbol": [int(table[p, 1]) / (n // w) for p in range(w)],
            "plane_coders": [int(h) for h in (d_v7[int(table[p, 0]) + 6].item() for p in range(w))],
            "encode": times, "decode": dtimes,
            "v7_minus_v6_encode_ms_per_GiB": times["v7_encode"]["median_ms"] - times["v6_encode"]["median_ms"],
            "v7_minus_v6_decode_ms_per_GiB": dtimes["v7_decode"]["median_ms"] - dtimes["v6_decode"]["median_ms"],
            "split_kernel": rate(ek, "planes_split_kernel"), "interleave_kernel": rate(dk, "planes_interleave_kernel"),
            "v7_encode_kernels": ek, "v7_decode_kernels": dk,
        }
        del d_in, d_v7
    ctx.close()
    return res


def planes_varlen(args):
    """rb200_container_planes_encode_varlen_async (n_max = 1 GiB, chunks of 8192) against the fixed plane call on bf16
    and fp32 N(0, 0.02): at *d_n = n_max and at *d_n = n_max / 16 against the fixed call at that length"""
    import torch
    n_max, chunk, tol = 1 << 30, 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    ctx = rb.Context(0)
    sync = ctx.sync
    d_n = torch.tensor([n_max, n_max // 16], dtype=torch.int64, device="cuda")
    res = {"card": card(), "workload": {"n_max": n_max, "chunk_syms": chunk}, "candidates": ["word 12", "alias 16", "byte 14"],
           "tolerance_ppm": tol, "workloads": {}, "checks": {}}
    gen = torch.Generator(device="cuda").manual_seed(4321)
    for name, dtype, w in (("bf16", torch.bfloat16, 2), ("fp32", torch.float32, 4)):
        d_in = (torch.randn(n_max // w, device="cuda", generator=gen) * 0.02).to(dtype).view(torch.uint8)
        bound = api.container_planes_bound(n_max, w, chunk)
        d_ref = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
        d_out = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
        i, r, o = d_in.data_ptr(), d_ref.data_ptr(), d_out.data_ptr()

        def size(d, w=w):
            return 64 + 16 * w + int(d[32:40].cpu().numpy().view(np.uint64)[0])

        def same(d_ref=d_ref, d_out=d_out):
            n = size(d_ref)
            return size(d_out) == n and bool(torch.equal(d_out[:n], d_ref[:n]))

        arms = {  # (varlen call, fixed call), each taking flags
            "bound": (lambda fl: ctx.container_planes_encode_varlen_async(cands, tol, w, i, d_n.data_ptr(), n_max, chunk, fl, o, bound),
                      lambda fl: ctx.container_planes_encode_async(cands, tol, w, i, n_max, chunk, fl, r, bound)),
            "sixteenth": (lambda fl: ctx.container_planes_encode_varlen_async(cands, tol, w, i, d_n[1:].data_ptr(), n_max, chunk, fl, o, bound),
                          lambda fl: ctx.container_planes_encode_async(cands, tol, w, i, n_max // 16, chunk, fl, r, bound)),
        }
        for arm, (varlen, fixed) in arms.items():                     # equal bytes before anything is timed
            for tag, flags in (("", 0), ("_crc", api.CONTAINER_CRC_BLOB)):
                d_out.fill_(0x5C)
                torch.cuda.synchronize()
                varlen(flags)
                fixed(flags)
                sync()
                res["checks"][f"{name} {arm}{tag}: varlen_equals_fixed_call_before_timing"] = same()
        res["workloads"][name] = varlen_arms(res, name, arms, sync, args, same)
        for arm in arms:
            for tag in ("", "_crc"):
                res["workloads"][name][arm + tag]["varlen_minus_fixed_per_plane_us"] = (
                    res["workloads"][name][arm + tag]["varlen_minus_fixed_median_us"] / w)
        del d_in, d_ref, d_out
        torch.cuda.empty_cache()
    ctx.close()
    return res


def delta(args):
    """version 8 against version 7 on the same tensor: bf16 and fp32 after one synthetic training step, 1 GiB each"""
    import torch
    n, chunk, tol = 1 << 30, 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_BYTE, 14), api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16)]
    ctx = rb.Context(0)
    sync = ctx.sync
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "workload": {"n": n, "chunk_syms": chunk, "step": "lr 1e-4, one step"},
           "candidates": ["byte 14", "word 12", "alias 16"], "tolerance_ppm": tol, "workloads": {}, "checks": {}}
    gen = torch.Generator(device="cuda").manual_seed(4321)
    for name, dtype, w in (("bf16", torch.bfloat16, 2), ("fp32", torch.float32, 4)):
        master = torch.randn(n // w, device="cuda", generator=gen) * 0.02
        d_base = master.to(dtype, copy=True).view(torch.uint8)        # a copy also for fp32: the step below moves master
        sign = torch.randint(0, 2, (n // w,), device="cuda", generator=gen, dtype=torch.int8).float() * 2 - 1
        master += 1e-4 * sign * torch.rand(n // w, device="cuda", generator=gen)
        d_in = master.to(dtype, copy=True).view(torch.uint8)
        del master, sign
        torch.cuda.empty_cache()
        bound = api.container_planes_bound(n, w, chunk)
        d_v7 = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
        d_v8 = torch.empty(bound + 16, dtype=torch.uint8, device="cuda")
        i, b, o7, o8, dd = d_in.data_ptr(), d_base.data_ptr(), d_v7.data_ptr(), d_v8.data_ptr(), d_dec.data_ptr()
        enc = {"v8_encode": lambda: ctx.container_delta_encode_async(cands, tol, w, i, b, n, chunk, 0, o8, bound),
               "v7_encode": lambda: ctx.container_planes_encode_async(cands, tol, w, i, n, chunk, 0, o7, bound)}
        times = alternate(enc, sync, args.warmup, args.reps)
        for f in enc.values():
            f()
        sync()
        h7, h8 = d_v7[:64].cpu().numpy(), d_v8[:64].cpu().numpy()
        size7 = 64 + 16 * w + int(h7[32:40].view(np.uint64)[0])
        size8 = 64 + 16 * w + int(h8[32:40].view(np.uint64)[0])
        res["checks"][f"{name}: v8_within_bound"] = size8 <= bound
        dec = {"v8_decode": lambda: ctx.container_delta_decode_async(w, o8, size8, b, dd, n),
               "v7_decode": lambda: ctx.container_planes_decode_async(w, o7, size7, dd, n)}
        dtimes = alternate(dec, sync, args.warmup, args.reps)
        for k, f in dec.items():
            d_dec.zero_()
            f()
            sync()
            res["checks"][f"{name}: {k}_round_trip"] = bool(torch.equal(d_dec[:n], d_in))
        ek = kernel_times(enc["v8_encode"], sync, args.reps)
        dk = kernel_times(dec["v8_decode"], sync, args.reps)
        dk7 = kernel_times(dec["v7_decode"], sync, args.reps)

        def rate(kernels, part, moved):
            us = sum(v["median_us"] * v["launches_per_call"] for k, v in kernels.items() if part in k)
            return {"us": us, "TB_per_s": moved / us / 1e6 if us else None}

        res["workloads"][name] = {
            "bytes_per_input_byte": {"v8": size8 / n, "v7": size7 / n},
            "encode": times, "decode": dtimes,
            "v8_minus_v7_encode_ms_per_GiB": times["v8_encode"]["median_ms"] - times["v7_encode"]["median_ms"],
            "v8_minus_v7_decode_ms_per_GiB": dtimes["v8_decode"]["median_ms"] - dtimes["v7_decode"]["median_ms"],
            "delta_split_kernel": rate(ek, "delta_split_kernel", 3 * n),
            "delta_interleave_kernel": rate(dk, "delta_interleave_kernel", 3 * n),
            "v7_interleave_kernel": rate(dk7, "planes_interleave_kernel", 2 * n),
            "v8_encode_kernels": ek, "v8_decode_kernels": dk,
        }
        del d_in, d_base, d_v7, d_v8
        torch.cuda.empty_cache()
    ctx.close()
    return res


def tensor_list_shapes(name):
    """(a) 8 transformer layers at hidden size 2048 (q, k, v, o 2048 x 2048; gate, up, down 2048 x 8192; two norms of
    2048): 72 tensors, 1 GiB in bf16; (b) a LoRA-like list of 448 tensors of 64 Ki elements (128 KiB in bf16)"""
    if name == "lora":
        return [1 << 16] * 448
    layer = [2048 * 2048] * 4 + [2048 * 8192] * 3 + [2048, 2048]
    return layer * 8


def tensors(args):
    """version 9 on three lists -- (a) 8 layers at hidden 2048 in bf16, (b) 448 LoRA-like bf16 tensors of 128 KiB, (c)
    list (a) in fp32 -- against T version 7 calls (looped, and as one captured graph) and one version 7 call on the
    already-concatenated bytes (the floor)"""
    import torch
    chunk, tol = 8192, 20000
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 14)]
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    sync = ctx.sync
    res = {"card": card(), "workload": {"chunk_syms": chunk, "data": "N(0, 0.02) per tensor"}, "candidates": ["word 12", "alias 16", "byte 14"],
           "tolerance_ppm": tol, "workloads": {}, "checks": {}}
    gen = torch.Generator(device="cuda").manual_seed(99)
    for name, shape, dtype, w in (("a_layers_bf16", "layers", torch.bfloat16, 2), ("b_lora_bf16", "lora", torch.bfloat16, 2),
                                  ("c_layers_fp32", "layers", torch.float32, 4)):
        counts = tensor_list_shapes(shape)
        t_count = len(counts)
        ts = [(torch.randn(c, device="cuda", generator=gen) * 0.02).to(dtype).view(torch.uint8) for c in counts]
        lengths = [t.numel() for t in ts]
        n = sum(lengths)
        cat = torch.cat(ts)
        refs = torch.tensor([[t.data_ptr(), t.numel()] for t in ts], dtype=torch.int64, device="cuda")
        bound9 = api.container_tensors_bound(n, t_count, w, chunk)
        bound7 = api.container_planes_bound(n, w, chunk)
        d_v9 = torch.empty(bound9, dtype=torch.uint8, device="cuda")
        d_v7 = torch.empty(bound7, dtype=torch.uint8, device="cuda")
        b7 = [api.container_planes_bound(b, w, chunk) for b in lengths]
        offs = np.concatenate([[0], np.cumsum([(b + 15) // 16 * 16 for b in b7])]).astype(np.int64)
        d_each = torch.empty(int(offs[-1]), dtype=torch.uint8, device="cuda")
        outs = [torch.empty_like(t) for t in ts]
        orefs = torch.tensor([[o.data_ptr(), o.numel()] for o in outs], dtype=torch.int64, device="cuda")
        d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        o9, o7, oe, dd = d_v9.data_ptr(), d_v7.data_ptr(), d_each.data_ptr(), d_dec.data_ptr()

        def enc_each():
            for t, o, b in zip(ts, offs, b7):
                ctx.container_planes_encode_async(cands, tol, w, t.data_ptr(), t.numel(), chunk, 0, oe + int(o), b)

        with torch.cuda.stream(stream):
            ctx.container_tensors_encode_async(cands, tol, w, refs.data_ptr(), t_count, n, chunk, 0, o9, bound9)
            ctx.container_planes_encode_async(cands, tol, w, cat.data_ptr(), n, chunk, 0, o7, bound7)
            enc_each()
            sync()
            size9 = 64 + 16 * w + (8 * t_count + 15) // 16 * 16 + int(d_v9[:64].cpu().numpy()[32:40].view(np.uint64)[0])
            size7 = 64 + 16 * w + int(d_v7[:64].cpu().numpy()[32:40].view(np.uint64)[0])
            sizes_each = []
            for o in offs[:-1]:
                h = d_each[int(o):int(o) + 64].cpu().numpy()
                sizes_each.append(64 + 16 * w + int(h[32:40].view(np.uint64)[0]))
            # the version 9 planes are the concatenation's version 7 planes
            res["checks"][f"{name}: v9_planes_equal_v7_of_concatenation"] = bool(torch.equal(
                d_v9[64 + 16 * w + (8 * t_count + 15) // 16 * 16:size9], d_v7[64 + 16 * w:size7]))

            def dec_each():
                at = 0
                for o, s_, b in zip(offs, sizes_each, lengths):
                    ctx.container_planes_decode_async(w, oe + int(o), s_, dd + at, b)
                    at += b

            dec_each()
            ctx.container_tensors_decode_async(w, o9, size9, orefs.data_ptr(), t_count, n)
            ctx.container_planes_decode_async(w, o7, size7, dd, n)
            sync()
            g_enc, g_dec = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(g_enc, stream=stream):
                enc_each()
            with torch.cuda.graph(g_dec, stream=stream):
                dec_each()
            enc = {"v9_one_call": lambda: ctx.container_tensors_encode_async(cands, tol, w, refs.data_ptr(), t_count, n, chunk, 0, o9, bound9),
                   "v7_T_calls_looped": enc_each,
                   "v7_T_calls_graph": g_enc.replay,
                   "v7_concatenated_floor": lambda: ctx.container_planes_encode_async(cands, tol, w, cat.data_ptr(), n, chunk, 0, o7, bound7)}
            dec = {"v9_one_call": lambda: ctx.container_tensors_decode_async(w, o9, size9, orefs.data_ptr(), t_count, n),
                   "v7_T_calls_looped": dec_each,
                   "v7_T_calls_graph": g_dec.replay,
                   "v7_concatenated_floor": lambda: ctx.container_planes_decode_async(w, o7, size7, dd, n)}
            etimes = alternate(enc, sync, args.warmup, args.reps)
            dtimes = alternate(dec, sync, args.warmup, args.reps)
            for o in outs:
                o.zero_()
            dec["v9_one_call"]()
            sync()
            res["checks"][f"{name}: v9_round_trip"] = all(bool(torch.equal(o, t)) for o, t in zip(outs, ts))
            ek9 = kernel_times(enc["v9_one_call"], sync, args.reps)
            ek7 = kernel_times(enc["v7_concatenated_floor"], sync, args.reps)
            dk9 = kernel_times(dec["v9_one_call"], sync, args.reps)
            dk7 = kernel_times(dec["v7_concatenated_floor"], sync, args.reps)
            del g_enc, g_dec

        def rate(kernels, part):
            us = sum(v["median_us"] * v["launches_per_call"] for k, v in kernels.items() if part in k)
            return {"us": us, "TB_per_s": 2 * n / us / 1e6 if us else None}

        res["workloads"][name] = {
            "tensors": t_count, "n": n,
            "bytes_per_input_byte": {"v9": size9 / n, "v7_T_containers": sum(sizes_each) / n, "v7_concatenated": size7 / n},
            "encode": etimes, "decode": dtimes,
            "v9_minus_floor_encode_ms": etimes["v9_one_call"]["median_ms"] - etimes["v7_concatenated_floor"]["median_ms"],
            "v9_minus_floor_decode_ms": dtimes["v9_one_call"]["median_ms"] - dtimes["v7_concatenated_floor"]["median_ms"],
            "tensors_split_kernel": rate(ek9, "tensors_split_kernel"), "planes_split_kernel": rate(ek7, "planes_split_kernel"),
            "tensors_interleave_kernel": rate(dk9, "tensors_interleave_kernel"),
            "planes_interleave_kernel": rate(dk7, "planes_interleave_kernel"),
            "launches_per_call": {"v9_encode": sum(v["launches_per_call"] for v in ek9.values()),
                                  "v9_decode": sum(v["launches_per_call"] for v in dk9.values())},
        }
        del ts, cat, refs, d_v9, d_v7, d_each, outs, orefs, d_dec
        torch.cuda.empty_cache()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", action="store_true", help="the per-block container on 8192 blocks of 64 KiB")
    ap.add_argument("--blocks-coder", action="store_true", help="per-block models for the byte and rans64 coders, 8192 blocks of 64 KiB")
    ap.add_argument("--blocks-alias", action="store_true", help="per-block models for the alias coder against byte, 8192 blocks of 64 KiB")
    ap.add_argument("--single", action="store_true", help="the single-model container's decode calls on three workloads")
    ap.add_argument("--model", action="store_true", help="the single-model container's encode with the model built from the data")
    ap.add_argument("--auto", action="store_true", help="the model-building encode with the coder chosen on the GPU")
    ap.add_argument("--blocks-auto", action="store_true", help="the per-block model-building encode with the coder chosen on the GPU")
    ap.add_argument("--blocks-varlen", action="store_true", help="the per-block auto encode with the block count in device memory")
    ap.add_argument("--blocks-stored", action="store_true", help="the per-block encode and decode with incompressible blocks stored (version 5)")
    ap.add_argument("--stored", action="store_true", help="the single-model encode and decode with incompressible chunks stored (version 6)")
    ap.add_argument("--stored-varlen", action="store_true", help="the version 6 encode with the length in device memory")
    ap.add_argument("--blocks-stored-varlen", action="store_true", help="the version 5 encode with the block count in device memory")
    ap.add_argument("--planes", action="store_true", help="the byte-plane container (version 7) against version 6 on bf16 and fp32")
    ap.add_argument("--planes-varlen", action="store_true", help="the byte-plane encode with the length in device memory, on bf16 and fp32")
    ap.add_argument("--delta", action="store_true", help="the delta byte-plane container (version 8) against version 7 on bf16 and fp32")
    ap.add_argument("--tensors", action="store_true", help="the tensor-list container (version 9) against T version 7 calls and the concatenation")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = blocks(args) if args.blocks else blocks_coder(args) if args.blocks_coder else blocks_alias(args) if args.blocks_alias else single(args) if args.single else model_encode(args) if args.model else auto_encode(args) if args.auto else blocks_auto(args) if args.blocks_auto else blocks_varlen(args) if args.blocks_varlen else blocks_stored(args) if args.blocks_stored else stored(args) if args.stored else stored_varlen(args) if args.stored_varlen else blocks_stored_varlen(args) if args.blocks_stored_varlen else planes(args) if args.planes else planes_varlen(args) if args.planes_varlen else delta(args) if args.delta else tensors(args) if args.tensors else headline(args)
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    sys.exit(0 if all(res["checks"].values()) else 1)


if __name__ == "__main__":
    main()
