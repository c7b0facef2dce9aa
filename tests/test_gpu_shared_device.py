"""Every coder's encode paths and decoders on a shared device: contexts running at once in threads, host pipelines in
parallel, a device whose SMs are partly taken by a neighbour, two processes time-sliced on one GPU, and work queued with
no synchronisation between calls (CUDA graph replays, a rejected decode between good ones, encodes of different paths).

The context's contract is one context per (device, stream, calling thread), so contexts run at the same time, and on a
shared GPU they always do.  What can go wrong there and nowhere else: a fused or ring encoder whose grid is only partly
resident (its scanner and workers poll each other with bounded waits), K2r's spill tier taking the branch a lagging
scan front forces, self-re-arming device state (the persistent decoders' DecodeWork, the CRC accumulator, the async
container decoders' `go` grids) left dirty for the next launch, and per-context host pipelines interleaving.

Ground truth: every case runs first alone on an idle device and is checked against the oracle; that result is the
baseline, and every concurrent, busy or queued run of the case must equal it byte for byte, whole output buffers with
their sentinel-filled tails included, with rb200_sync returning 0 (never RB200_E_STALL).  Encodes are deterministic, so
anything else is a bug.  Each encode case names the path plan_encode / plan_blocks_encode picks for it (encode_path,
the library's rule restated, checked against the case table without a GPU), pinned on the GPU by the launch count --
a fused path is one launch, a split one more -- and, for the word coder's one-launch paths (K2r, K2f, K5f), by the
name of the kernel its baseline run launched, read with torch.profiler.

  A. K contexts created at once from K threads, each on its own non-blocking stream (one variant with a context on the
     legacy default stream), running the case list in K rotations and in lockstep for several rounds;
  B. the host-buffer calls (flat, per-block and container with CRC_BLOB) on K threads in a child process with 1 MiB
     slices, pageable numpy buffers and growing sizes;
  C. every case enqueued while tests/shared_device/hold.cu holds all SMs but 1, all but 8, and half of them;
  D. two child processes running halves of the case list in a loop at once;
  E. graphs of varlen encode + async decode (versions 1, 5, 6) replayed R times back to back with stream-ordered input
     updates and output copies and one sync, on one context and on two at once; [good, corrupt, good] rb200_decode
     queues per coder with one sync; encodes of four paths queued on one context with one sync.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import threading
import time
import zlib

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, TESTS)
import conftest  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402
import test_container_stored as cs  # noqa: E402
import test_gpu_blocks_geometry as gbg  # noqa: E402
import test_gpu_container_blocks_stored as gbs  # noqa: E402
import test_gpu_container_stored as gs  # noqa: E402
import test_word_encode_ring_spill as spill  # noqa: E402

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = api.CONTAINER_CRC_BLOB
SENTINEL = 0x5C
E_STREAM, E_STALL = -4, -9
K = 4                                   # contexts / threads at once
ROUNDS = 4                              # rounds of the whole case list per thread (A)
LOCKSTEP = 3                            # calls of the same case each thread queues at once in A's lockstep rounds
HOLD_US = 250_000                       # one neighbour hold (C): far below the kernels' 8 s stall limit
N_FLAT = (24 << 20) + 777               # symbols of a flat case (ragged last chunk)
PB = (768, 32768, 4096)                 # (n_blocks, block_size, chunk_syms) of the per-block cases: 24 MiB
V5 = (384, 65536, 8192)                 # the version 5 cases: 24 MiB
N6, CH6 = (24 << 20) + 4097, 8192       # the version 6 cases

# ---------------------------------------------------------------------------------------------------- the path rule

FUSED_MIN_CHUNK, FUSED_MAX_CHUNK = 4096, 65536      # use_fused_encode: chunks in this range run fused
RING_MAX_CHUNK = 8192                               # kEncRingMaxChunk
WORD_SLOTS = 4096                                   # a word symbol of this frequency keeps a model off K2r


def encode_path(coder, chunk_syms, freqs=None, per_block=False, build=False):
    """The encode path plan_encode (flat) or plan_blocks_encode (per_block) picks, RB200_ENCODE_PATH unset: K2r / K2f
    (word, fused), fused (alias and byte), K5f (word, per-block) or split."""
    fusable = FUSED_MIN_CHUNK <= chunk_syms <= FUSED_MAX_CHUNK
    if per_block:
        return "K5f" if coder == WORD and (build or fusable) else "split"
    if coder == RANS64 or not fusable:
        return "split"
    if coder == WORD:
        return "K2r" if chunk_syms <= RING_MAX_CHUNK and int(np.max(freqs)) < WORD_SLOTS else "K2f"
    return "fused"


# (name, coder, scale_bits, data kind, chunk_syms, path): the flat encodes; "spill" is test_word_encode_ring_spill's
# alternating data under its {4095, 1} model, every other kind is coded with the model of its data
FLAT_ENCODES = [
    ("word-K2r", WORD, 12, "zipf", 8192, "K2r"),
    ("word-K2r-spill", WORD, 12, "spill", 8192, "K2r"),
    ("word-K2f", WORD, 12, "const", 8192, "K2f"),            # one symbol of frequency 4096
    ("word-split", WORD, 12, "text", 2048, "split"),
    ("alias-fused", ALIAS, 16, "zipf", 4096, "fused"),
    ("alias-split", ALIAS, 14, "skew", 2048, "split"),
    ("byte-fused", BYTE, 14, "text", 8192, "fused"),
    ("byte-split", BYTE, 12, "zipf", 1024, "split"),
    ("rans64-split", RANS64, 15, "zipf", 4096, "split"),
]
# (name, per-block instance, path): the per-block model-building encodes of PB
BLOCK_ENCODES = [("blocks-word-K5f", gbg.WORD, "K5f"), ("blocks-byte", gbg.BYTE[14], "split"),
                 ("blocks-rans64", gbg.RANS64[12], "split"), ("blocks-alias", gbg.ALIAS[11], "split")]
# (name, coder, scale_bits, data kind, chunk_syms): the flat rb200_decode cases
FLAT_DECODES = [("word", WORD, 12, "zipf", 8192), ("byte", BYTE, 14, "text", 4096), ("alias", ALIAS, 16, "zipf", 4096),
                ("rans64", RANS64, 15, "zipf", 2048)]


def flat_data(kind, n, seed):
    return spill._alternating(n, seed) if kind == "spill" else conftest._gen(kind, n, seed)


def flat_model(oracle_lib, kind, data, sb):
    """(freqs, cum) of a flat case"""
    if kind == "spill":
        return spill._rare_model()
    return oracle_lib.model(data, sb)


def test_case_table_follows_the_path_rule(oracle_lib):
    """Each encode case is on the path it names, by the library's rule, and the table covers every path of every
    coder: K2r (with and without spills), K2f, word split, alias and byte fused and split, rans64 split, K5f and the
    split per-block encoders."""
    for name, coder, sb, kind, ch, path in FLAT_ENCODES:
        data = flat_data(kind, 1 << 20, 1)
        freqs, _ = flat_model(oracle_lib, kind, data, sb)
        assert encode_path(coder, ch, freqs) == path, name
    for name, inst, path in BLOCK_ENCODES:
        assert encode_path(inst.coder, PB[2], per_block=True, build=True) == path, name
    seen = {(c, p) for _, c, _, _, _, p in FLAT_ENCODES} | {(i.coder, p) for _, i, p in BLOCK_ENCODES}
    assert seen >= {(WORD, "K2r"), (WORD, "K2f"), (WORD, "split"), (ALIAS, "fused"), (ALIAS, "split"), (BYTE, "fused"),
                    (BYTE, "split"), (RANS64, "split"), (WORD, "K5f")}
    assert {i.coder for _, i, _ in BLOCK_ENCODES} == {WORD, BYTE, ALIAS, RANS64}
    assert {c for _, c, _, _, _ in FLAT_DECODES} == {WORD, BYTE, ALIAS, RANS64}
    # the rule at its edges
    f_ring, f_wide = np.full(256, 16, np.uint32), np.zeros(256, np.uint32)
    f_wide[7] = 4096
    assert [encode_path(WORD, ch, f_ring) for ch in (4095, 4096, 8192, 8193, 65536, 65537)] == \
        ["split", "K2r", "K2r", "K2f", "K2f", "split"]
    assert encode_path(WORD, 4096, f_wide) == "K2f"
    assert [encode_path(c, 4096) for c in (BYTE, ALIAS, RANS64)] == ["fused", "fused", "split"]
    assert encode_path(WORD, 2048, per_block=True, build=True) == "K5f"
    assert encode_path(WORD, 2048, per_block=True) == "split"


def test_holder_compiles_for_sm90a(tmp_path):
    """tests/shared_device/hold.cu builds with the library's flags, and its host entry points are exported."""
    lib = build_holder(str(tmp_path))
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    for name in ("hold_sms", "hold_end", "hold_smem_bytes"):
        assert f" T {name}" in syms, name
    sass = subprocess.run([os.path.join(os.path.dirname(_nvcc()), "cuobjdump"), "-sass", lib], capture_output=True, text=True).stdout
    assert "sm_90a" in sass and "NANOSLEEP" in sass


def _nvcc():
    from ryg_rans_b200.build import _nvcc as nvcc
    return nvcc()


def build_holder(out_dir):
    from ryg_rans_b200.build import NVCC_FLAGS
    out = os.path.join(out_dir, "libhold.so")
    subprocess.check_call([_nvcc(), *NVCC_FLAGS, "-shared", "-o", out, os.path.join(TESTS, "shared_device", "hold.cu")])
    return out


# ---------------------------------------------------------------------------------------------------- the cases

def _torch():
    import torch
    return torch


def _dev(a):
    torch = _torch()
    a = np.array(a, copy=True).view(np.uint8).reshape(-1)          # writable, as torch.from_numpy wants
    t = torch.zeros(a.size + 16, dtype=torch.uint8, device="cuda")
    t[:a.size] = torch.from_numpy(a)
    return t


def _tail(a, size):
    """a's bytes and then the sentinel up to size bytes"""
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    assert a.size <= size
    return np.concatenate([a, np.full(size - a.size, SENTINEL, np.uint8)])


class Case:
    """One library call on device memory.  make(oracle_lib) builds it: `d` the shared device inputs, `models` the
    (coder, scale_bits, freqs) each context creates, `sizes` the output buffers (sentinel-filled before every call),
    `call(ctx, models, outs)` the enqueue (it may return a host value, e.g. a CRC), `want` the oracle's whole output
    buffers and host value.  `path`: the encode path it pins (launches: 1 fused, more split)."""

    def __init__(self, name, make, path=None, dir_of=None):
        self.name, self._make, self.path, self.dir_of = name, make, path, dir_of
        self.built = False

    def make(self, oracle_lib):
        if not self.built:
            self.d, self.models, self.sizes, self.call, self.want = self._make(oracle_lib)
            self.built = True
        return self

    def __repr__(self):
        return self.name


def _flat_encode_case(name, coder, sb, kind, ch, path):
    def make(orl):
        data = flat_data(kind, N_FLAT, 11 + coder)
        freqs, cum = flat_model(orl, kind, data, sb)
        assert encode_path(coder, ch, freqs) == path, name
        blob, offs = orl.chunked_encode(coder, data, freqs, cum, ch, scale_bits=sb)
        cap = api.load().dll.rb200_encode_bound(data.size, ch)
        sizes = [cap + 64, offs.nbytes + 64]
        d = {"in": _dev(data)}

        def call(ctx, models, outs):
            ctx.encode_device(models[0], d["in"].data_ptr(), data.size, ch, outs[0].data_ptr(), cap, outs[1].data_ptr())
        return d, [(coder, sb, freqs)], sizes, call, ([_tail(blob, sizes[0]), _tail(offs, sizes[1])], None)
    return Case(name, make, path, dir_of=(0, 1))


def _block_encode_case(name, inst, path):
    nb, bs, ch = PB

    def make(orl):
        data = gbg.block_data(PB)
        freqs, offs, blob = gbg.oracle_streams(orl, inst, PB)
        cap = api.load().dll.rb200_encode_bound(data.size, ch)
        sizes = [cap + 64, offs.nbytes + 64, freqs.nbytes + 64]
        d = {"in": _dev(data)}

        def call(ctx, models, outs):
            args = (d["in"].data_ptr(), nb, bs, outs[2].data_ptr(), ch, outs[0].data_ptr(), cap, outs[1].data_ptr())
            if inst.coder == WORD:
                ctx.blocks_model_encode_device(*args)
            elif inst.coder == ALIAS:
                ctx.blocks_alias_model_encode_device(inst.sb, *args)
            else:
                ctx.blocks_coder_model_encode_device(inst.coder, inst.sb, *args)
        return d, [], sizes, call, ([_tail(blob, sizes[0]), _tail(offs, sizes[1]), _tail(freqs, sizes[2])], None)
    return Case(name, make, path, dir_of=(0, 1))


def _v6_data():
    return cs.mixed_data(N6 + 100_003, CH6, 61)


def _v5_data():
    nb, bs, _ = V5
    return gbs.block_data("halfuniform", nb + 16, bs, 51)


def _v6_encode_case(varlen):
    def make(orl):
        full = _v6_data()
        n = N6 if varlen else full.size
        want = gs.expected(orl, gs.THREE, 20000, full[:n], CH6, CRC_BLOB)[0]
        n_max = full.size
        cap = api.container_stored_bound(n_max if varlen else n, CH6)
        d = {"in": _dev(full), "n": _dev(np.array([n], np.uint64))}

        def call(ctx, models, outs):
            if varlen:
                ctx.container_stored_encode_varlen_async(gs.THREE, 20000, d["in"].data_ptr(), d["n"].data_ptr(), n_max, CH6, CRC_BLOB,
                                                         outs[0].data_ptr(), cap)
            else:
                ctx.container_stored_encode_async(gs.THREE, 20000, d["in"].data_ptr(), n, CH6, CRC_BLOB, outs[0].data_ptr(), cap)
        return d, [], [cap + 64], call, ([_tail(want, cap + 64)], None)
    return Case("v6-encode-varlen" if varlen else "v6-encode", make)


def _v5_encode_case(varlen):
    nb, bs, ch = V5

    def make(orl):
        full = _v5_data()
        nb_max = nb + 16
        count = nb if varlen else nb_max
        want = gbs.expected(orl, gbs.THREE, 20000, full[:count * bs], count, bs, ch, CRC_BLOB)[0]
        cap = api.container_blocks_stored_bound(nb_max if varlen else count, bs, ch)
        d = {"in": _dev(full), "nb": _dev(np.array([count], np.uint32))}

        def call(ctx, models, outs):
            if varlen:
                ctx.container_blocks_stored_encode_varlen_async(gbs.THREE, 20000, d["in"].data_ptr(), d["nb"].data_ptr(), nb_max, bs, ch,
                                                                CRC_BLOB, outs[0].data_ptr(), cap)
            else:
                ctx.container_blocks_stored_encode_async(gbs.THREE, 20000, d["in"].data_ptr(), count, bs, ch, CRC_BLOB,
                                                         outs[0].data_ptr(), cap)
        return d, [], [cap + 64], call, ([_tail(want, cap + 64)], None)
    return Case("v5-encode-varlen" if varlen else "v5-encode", make)


_FLAT_STREAMS = {}


def flat_streams(orl, coder, sb, kind, ch):
    """(data, freqs, cum, blob, offsets) by the oracle for a flat decode case (cached)"""
    key = (coder, sb, kind, ch)
    if key not in _FLAT_STREAMS:
        data = flat_data(kind, N_FLAT, 31 + coder)
        freqs, cum = orl.model(data, sb)
        blob, offs = orl.chunked_encode(coder, data, freqs, cum, ch, scale_bits=sb)
        _FLAT_STREAMS[key] = (data, freqs, cum, blob, offs)
    return _FLAT_STREAMS[key]


def _flat_decode_case(name, coder, sb, kind, ch):
    def make(orl):
        data, freqs, cum, blob, offs = flat_streams(orl, coder, sb, kind, ch)
        assert np.array_equal(orl.chunked_decode(coder, blob, offs, data.size, freqs, cum, ch, scale_bits=sb), data)
        d = {"blob": _dev(blob), "offs": _dev(offs)}

        def call(ctx, models, outs):
            ctx.decode_device(models[0], d["blob"].data_ptr(), blob.size, d["offs"].data_ptr(), ch, outs[0].data_ptr(), data.size)
        return d, [(coder, sb, freqs)], [data.size + 64], call, ([_tail(data, data.size + 64)], None)
    return Case(f"decode-{name}", make)


def _block_decode_case(inst):
    nb, bs, ch = PB

    def make(orl):
        data = gbg.block_data(PB)
        freqs, offs, blob = gbg.oracle_streams(orl, inst, PB)
        d = {"blob": _dev(blob), "offs": _dev(offs), "freqs": _dev(freqs)}

        def call(ctx, models, outs):
            args = (d["blob"].data_ptr(), blob.size, d["offs"].data_ptr(), d["freqs"].data_ptr(), nb, bs, ch, outs[0].data_ptr())
            if inst.coder == WORD:
                ctx.blocks_decode_device(*args)
            elif inst.coder == ALIAS:
                ctx.blocks_alias_decode_device(inst.sb, *args)
            else:
                ctx.blocks_coder_decode_device(inst.coder, inst.sb, *args)
        return d, [], [data.size + 64], call, ([_tail(data, data.size + 64)], None)
    return Case(f"blocks-decode-{inst.name}", make)


def _container_of(orl, version):
    """(container, symbols) of one version, from the oracle's streams (5 and 6: the oracle-packed stored containers)"""
    nb, bs, ch = PB
    if version == 1:
        data, freqs, _, blob, offs = flat_streams(orl, WORD, 12, "zipf", 8192)
        return api.container_pack(WORD, 12, 8192, data.size, freqs, offs, blob, CRC_BLOB), data
    if version == 5:
        full = _v5_data()
        return gbs.expected(orl, gbs.THREE, 20000, full, V5[0] + 16, V5[1], V5[2], CRC_BLOB)[0], full
    if version == 6:
        full = _v6_data()
        return gs.expected(orl, gs.THREE, 20000, full, CH6, CRC_BLOB)[0], full
    data = gbg.block_data(PB)
    inst = {2: gbg.WORD, 3: gbg.BYTE[14], 4: gbg.ALIAS[11], "any": gbg.RANS64[12]}[version]
    freqs, offs, blob = gbg.oracle_streams(orl, inst, PB)
    return inst.pack(nb, bs, ch, freqs, offs, blob, CRC_BLOB), data


ASYNC_DECODES = {1: "container_decode_async", 2: "container_blocks_decode_async", 3: "container_blocks_coder_decode_async",
                 4: "container_blocks_alias_decode_async", 5: "container_blocks_stored_decode_async",
                 6: "container_stored_decode_async", "any": "container_blocks_any_decode_async"}


def _async_decode_case(version):
    def make(orl):
        buf, data = _container_of(orl, version)
        d = {"buf": _dev(buf)}

        def call(ctx, models, outs):
            getattr(ctx, ASYNC_DECODES[version])(d["buf"].data_ptr(), buf.size, outs[0].data_ptr(), data.size, outs[1].data_ptr())
        return d, [], [data.size + 64, 8], call, ([_tail(data, data.size + 64), np.array([data.size], np.uint64).view(np.uint8)], None)
    return Case(f"async-decode-v{version}", make)


def _crc_case():
    def make(orl):
        data = flat_data("zipf", N_FLAT, 71)
        d = {"in": _dev(data)}

        def call(ctx, models, outs):
            return ctx.crc32_device(d["in"].data_ptr(), data.size)
        return d, [], [], call, ([], zlib.crc32(data.tobytes()))
    return Case("crc32", make)


def all_cases():
    """every case, in one fixed order (a thread runs a rotation of it)"""
    return ([_flat_encode_case(*e) for e in FLAT_ENCODES]
            + [_block_encode_case(*e) for e in BLOCK_ENCODES]
            + [_v6_encode_case(False), _v6_encode_case(True), _v5_encode_case(False), _v5_encode_case(True)]
            + [_flat_decode_case(*e) for e in FLAT_DECODES]
            + [_block_decode_case(i) for i in (gbg.WORD, gbg.BYTE[14], gbg.RANS64[12], gbg.ALIAS[11])]
            + [_async_decode_case(v) for v in (1, 2, 3, 4, 5, 6, "any")]
            + [_crc_case()])


# ---------------------------------------------------------------------------------------------------- running them

class Runner:
    """One context on one stream (a torch stream; the legacy default stream for stream 0), with its models and output
    buffers for every case, allocated once and refilled with the sentinel before every call."""

    def __init__(self, ctx, stream):
        self.ctx, self.stream = ctx, stream
        self.models, self.outs = {}, {}

    def enqueue(self, case):
        """sentinel fill + the call on this context's stream; returns the call's host value"""
        torch = _torch()
        with torch.cuda.stream(self.stream):
            if case.name not in self.outs:
                self.models[case.name] = [self.ctx.model(*m) for m in case.models]
                self.outs[case.name] = [torch.empty(s, dtype=torch.uint8, device="cuda") for s in case.sizes]
            for o in self.outs[case.name]:
                o.fill_(SENTINEL)
            return case.call(self.ctx, self.models[case.name], self.outs[case.name])

    def sync(self):
        return self.ctx.lib.dll.rb200_sync(self.ctx.h)

    def run(self, case):
        """(sync code, outputs, host value, launches) of one call"""
        before = self.ctx.launches
        value = self.enqueue(case)
        rc = self.sync()
        return rc, self.outs[case.name], value, self.ctx.launches - before

    def close(self):
        self.stream.synchronize()
        for ms in self.models.values():
            for m in ms:
                m.close()
        self.models, self.outs = {}, {}
        self.ctx.close()


def _first_diff(case, i, got, want, base_outs):
    bad = (got != want).nonzero()
    at = int(bad[0, 0])
    msg = f"{case.name}: output {i} differs in {bad.shape[0]} bytes, first at byte {at} ({int(got[at]):#x} != {int(want[at]):#x})"
    if case.dir_of and i == case.dir_of[0]:
        offs = base_outs[case.dir_of[1]].cpu().numpy()
        offs = offs[:offs.size - 64].view(np.uint64)
        msg += f", chunk {int(np.searchsorted(offs, at, side='right')) - 1} of {offs.size - 1}"
    return msg


def check(case, base, rc, outs, value, ctx):
    """None when a run equals the baseline, else what differs"""
    torch = _torch()
    if rc != 0:
        stall = " (RB200_E_STALL: a bounded wait expired)" if rc == E_STALL else ""
        return f"{case.name}: rb200_sync returned {rc}{stall}; last CUDA error '{ctx.lib.dll.rb200_last_cuda_error(ctx.h).decode()}'"
    for i, (got, want) in enumerate(zip(outs, base.outs)):
        if not torch.equal(got, want):
            return _first_diff(case, i, got, want, base.outs)
    if value != base.value:
        return f"{case.name}: host value {value!r} != {base.value!r}"
    return None


class Baseline:
    def __init__(self, outs, value):
        self.outs, self.value = outs, value


# the word coder's one-launch paths, by the kernel each launches: the launch count tells fused from split, not K2r from
# K2f, so the baseline run of such a case is profiled and the kernel it ran is named
WORD_KERNELS = {"K2r": "word_encode_ring_kernel", "K2f": "word_encode_fused_kernel", "K5f": "block_encode_fused_kernel"}


def _run_profiled(runner, case):
    """runner.run(case) under torch.profiler: (its result, the names of the kernels that ran)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        result = runner.run(case)
    return result, {e.name for e in prof.events()}


def take_baseline(case, runner):
    """the case alone on an idle device, checked against the oracle, with its path pinned: fused or split by the launch
    count, and the word coder's fused paths (K2r, K2f, K5f) by the kernel that ran"""
    torch = _torch()
    word_fused = case.path in WORD_KERNELS
    (rc, outs, value, launches), kernels = _run_profiled(runner, case) if word_fused else (runner.run(case), set())
    assert rc == 0, (case.name, rc)
    want, want_value = case.want
    for i, (got, w) in enumerate(zip(outs, want)):
        g = got.cpu().numpy()
        if not np.array_equal(g, w):
            at = int(np.flatnonzero(g != w)[0])
            pytest.fail(f"{case.name}: output {i} differs from the oracle at byte {at} of {g.size}")
    assert value == want_value, case.name
    if case.path is not None:
        assert (launches == 1) == (case.path != "split") and launches >= 1, (case.name, case.path, launches)
    if word_fused:
        ran = {p for p, k in WORD_KERNELS.items() if any(k in name for name in kernels)}
        assert ran == {case.path}, (case.name, case.path, sorted(n for n in kernels if "kernel" in n))
    with torch.cuda.stream(runner.stream):
        return Baseline([o.clone() for o in outs], value)


class World:
    def __init__(self, oracle_lib):
        torch = _torch()
        self.cases = [c.make(oracle_lib) for c in all_cases()]
        stream = torch.cuda.Stream()
        runner = Runner(rb.Context(0, stream=stream.cuda_stream), stream)
        self.base = {c.name: take_baseline(c, runner) for c in self.cases}
        runner.close()
        torch.cuda.synchronize()


@pytest.fixture(scope="module")
def world(oracle_lib):
    torch = _torch()
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    w = World(oracle_lib)
    yield w
    del w
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _threads(body, n, timeout=900):
    errors = []

    def wrap(t):
        try:
            body(t, errors)
        except Exception as e:          # a failed call inside a thread is a finding, reported by the test
            errors.append(f"thread {t}: {type(e).__name__}: {e}")

    ts = [threading.Thread(target=wrap, args=(t,)) for t in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout)
    assert not any(t.is_alive() for t in ts), "a thread did not finish"
    return errors


# ---------------------------------------------------------------------------------------------------- A

@pytest.mark.gpu
@pytest.mark.parametrize("legacy", [False, True], ids=["own-streams", "one-on-legacy-stream"])
def test_concurrent_contexts_in_threads(world, legacy):
    """K contexts created at the same moment from K threads, each on its own stream (with `legacy`, thread 0's context
    on the legacy default stream), running the case list for ROUNDS rounds: in its own rotation (different kernels at
    once) and in lockstep (every thread queues the same case LOCKSTEP times at once: the same kernels, on per-context
    state, at once).  ctypes releases the GIL, so the library calls overlap.  Every output equals the baseline."""
    torch = _torch()
    cases = world.cases
    created = threading.Barrier(K)

    def body(t, errors):
        stream = torch.cuda.default_stream() if legacy and t == 0 else torch.cuda.Stream()
        try:
            created.wait(timeout=300)
            ctx = rb.Context(0, stream=stream.cuda_stream)          # rb200_ctx_create from K threads at once
            created.wait(timeout=300)
        except Exception:
            created.abort()
            raise
        runner = Runner(ctx, stream)
        shift = t * len(cases) // K
        try:
            for rnd in range(ROUNDS):
                # even rounds: this thread's rotation, so different kernels overlap; odd rounds: every thread starts the
                # same case at once and enqueues it LOCKSTEP times before its sync, so the same kernels overlap
                lockstep = rnd % 2 == 1
                for case in cases if lockstep else cases[shift:] + cases[:shift]:
                    if lockstep:
                        created.wait(timeout=300)
                        values = [runner.enqueue(case) for _ in range(LOCKSTEP)]
                        rc, outs, value = runner.sync(), runner.outs[case.name], values[-1]
                        if values.count(value) != LOCKSTEP:
                            errors.append(f"thread {t} round {rnd}: {case.name}: host values {values}")
                    else:
                        rc, outs, value, _ = runner.run(case)
                    msg = check(case, world.base[case.name], rc, outs, value, ctx)
                    if msg:
                        errors.append(f"thread {t} round {rnd} ({'legacy stream' if legacy and t == 0 else 'own stream'}): {msg}")
        except Exception:
            created.abort()
            raise
        finally:
            runner.close()

    errors = _threads(body, K)
    assert not errors, "\n".join(errors[:20])


# ---------------------------------------------------------------------------------------------------- B

HOST_SIZES = [300_007, (3 << 20) + 5, (9 << 20) + 3]          # per thread, in this order: every workspace grows mid-run
HOST_FLAT = [(WORD, 12, "zipf", 8192), (ALIAS, 16, "text", 4096), (BYTE, 13, "zipf", 2048), (RANS64, 14, "skew", 4096)]


def _host_cases(orl):
    """[(name, fn(ctx) -> tuple of arrays, want tuple)] of the host-buffer calls, every size"""
    out = []
    for n in HOST_SIZES:
        for coder, sb, kind, ch in HOST_FLAT:
            data = conftest._gen(kind, n, n + coder)
            freqs, cum = orl.model(data, sb)
            blob, offs = orl.chunked_encode(coder, data, freqs, cum, ch, scale_bits=sb)

            def enc(ctx, data=data, coder=coder, sb=sb, freqs=freqs, ch=ch):
                m = ctx.model(coder, sb, freqs)
                try:
                    return ctx.encode_host(m, data, ch)
                finally:
                    m.close()

            def dec(ctx, data=data, coder=coder, sb=sb, freqs=freqs, ch=ch, blob=blob, offs=offs):
                m = ctx.model(coder, sb, freqs)
                try:
                    return (ctx.decode_host(m, blob, offs, data.size, ch),)
                finally:
                    m.close()

            def cont(ctx, data=data, coder=coder, sb=sb, freqs=freqs, ch=ch):
                m = ctx.model(coder, sb, freqs)
                try:
                    buf = ctx.container_encode_host(m, data, ch, CRC_BLOB)
                finally:
                    m.close()
                return buf, ctx.container_decode_host(buf)

            want_c = api.container_pack(coder, sb, ch, n, freqs, offs, blob, CRC_BLOB)
            out += [(f"encode-{coder}-{n}", enc, (blob, offs)), (f"decode-{coder}-{n}", dec, (data,)),
                    (f"container-{coder}-{n}", cont, (want_c, data))]
        bs, ch = 32768, 4096
        nb = n // bs
        data = conftest._gen("text", nb * bs, n + 7)
        for coder, sb in ((BYTE, 12), (RANS64, 13), (ALIAS, 14)):
            freqs, offs, blob = cc.oracle_blocks_encode(orl, coder, sb, data, nb, bs, ch)

            def benc(ctx, data=data, coder=coder, sb=sb, nb=nb):
                if coder == ALIAS:
                    return ctx.blocks_alias_model_encode_host(sb, data, nb, bs, ch)
                return ctx.blocks_coder_model_encode_host(coder, sb, data, nb, bs, ch)

            def bdec(ctx, data=data, coder=coder, sb=sb, nb=nb, freqs=freqs, offs=offs, blob=blob):
                if coder == ALIAS:
                    return (ctx.blocks_alias_decode_host(sb, blob, offs, freqs, nb, bs, ch),)
                return (ctx.blocks_coder_decode_host(coder, sb, blob, offs, freqs, nb, bs, ch),)

            out += [(f"blocks-encode-{coder}-{n}", benc, (blob, offs, freqs)), (f"blocks-decode-{coder}-{n}", bdec, (data,))]
    return out


def _same(got, want):
    return len(got) == len(want) and all(np.array_equal(np.asarray(g), np.asarray(w)) for g, w in zip(got, want))


def child_host_pipelines():
    """(child process, RB200_SLICE_MIB=1) the host-buffer calls alone, against the oracle, then on K threads at once"""
    import oracle
    orl = oracle.Oracle()
    cases = _host_cases(orl)
    ctx = rb.Context(0)
    for name, fn, want in cases:                   # the baseline: alone, on an idle device
        assert _same(fn(ctx), want), f"{name}: differs from the oracle"
    ctx.close()
    per_size = len(cases) // len(HOST_SIZES)
    start = threading.Barrier(K)

    def body(t, errors):
        ctx = rb.Context(0)
        start.wait(timeout=300)
        try:
            for s in range(len(HOST_SIZES)):        # sizes grow: staging, directories and workspaces grow mid-run
                group = cases[s * per_size:(s + 1) * per_size]
                shift = t * len(group) // K
                for name, fn, want in group[shift:] + group[:shift]:
                    try:
                        got = fn(ctx)
                    except rb.RansError as e:
                        errors.append(f"thread {t}: {name}: {e}")
                        continue
                    if not _same(got, want):
                        errors.append(f"thread {t}: {name}: differs from the baseline")
        finally:
            ctx.close()

    errors = _threads(body, K)
    if errors:
        print("\n".join(errors[:20]))
        sys.exit(1)
    print(f"host pipelines: {len(cases)} calls x {K} threads ok")


def _child(fn, env=None, timeout=900, args=()):
    code = f"import sys; sys.path.insert(0, {TESTS!r}); sys.path.insert(0, {ROOT!r}); import test_gpu_shared_device as t; t.{fn}(*sys.argv[1:])"
    return subprocess.run([sys.executable, "-c", code, *args], env=dict(os.environ, **(env or {})), capture_output=True, text=True,
                          timeout=timeout)


@pytest.mark.gpu
def test_host_pipelines_on_parallel_threads(cuda_box):
    out = _child("child_host_pipelines", {"RB200_SLICE_MIB": "1"})
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]


# ---------------------------------------------------------------------------------------------------- C

class Holder:
    def __init__(self, path):
        self.dll = C.CDLL(path)
        self.dll.hold_sms.argtypes = [C.c_int, C.c_uint, C.c_uint, C.POINTER(C.c_int)]
        self.dll.hold_sms.restype = C.c_int
        self.dll.hold_end.restype = C.c_int
        self.dll.hold_smem_bytes.restype = C.c_int

    def hold(self, ctas, hold_us=HOLD_US, wait_ms=5000):
        resident = C.c_int(0)
        rc = self.dll.hold_sms(ctas, hold_us, wait_ms, C.byref(resident))
        assert rc == 0, f"hold_sms: CUDA error {rc}"
        return resident.value

    def end(self):
        assert self.dll.hold_end() == 0


@pytest.fixture(scope="module")
def holder(tmp_path_factory):
    h = Holder(build_holder(str(tmp_path_factory.mktemp("shared_device"))))
    yield h
    h.end()


@pytest.mark.gpu
@pytest.mark.parametrize("share", ["all-but-1", "all-but-8", "half"])
def test_busy_device(world, holder, share):
    """Every case enqueued while a neighbour's CTAs take whole SMs (the neighbour reports itself resident first), so
    the fused, ring and K5f encoders and the persistent and planned decoders run with part of their grid resident and
    K2r's scan front lags.  The holds end by themselves after HOLD_US."""
    torch = _torch()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = {"all-but-1": sms - 1, "all-but-8": sms - 8, "half": sms // 2}[share]
    assert holder.dll.hold_smem_bytes() > 0
    stream = torch.cuda.Stream()
    runner = Runner(rb.Context(0, stream=stream.cuda_stream), stream)
    errors, seen = [], []
    try:
        for case in world.cases:                  # outputs, models and workspaces first: no allocation under a hold
            msg = check(case, world.base[case.name], *runner.run(case)[:3], runner.ctx)
            assert msg is None, msg
        for case in world.cases:
            seen.append(holder.hold(ctas))
            rc, outs, value, _ = runner.run(case)
            msg = check(case, world.base[case.name], rc, outs, value, runner.ctx)
            if msg:
                errors.append(f"{ctas} of {sms} SMs held ({seen[-1]} resident): {msg}")
        holder.end()
    finally:
        runner.close()
    print(f"{sms} SMs; {ctas} held; resident per hold: min {min(seen)}, max {max(seen)}")
    assert not errors, "\n".join(errors)
    assert max(seen) == ctas, f"the neighbour never had all {ctas} CTAs resident: {seen}"


# ---------------------------------------------------------------------------------------------------- D

def _digests(outs, value):
    return [hashlib.sha256(o.cpu().numpy().tobytes()).hexdigest() for o in outs] + [repr(value)]


def child_case_loop(part, parts, seconds, digest_file):
    """(child process) cases part::parts in a loop for `seconds`, each output against the baseline's digests"""
    import oracle
    torch = _torch()
    want = json.load(open(digest_file))
    cases = [c.make(oracle.Oracle()) for c in all_cases()[int(part)::int(parts)]]
    stream = torch.cuda.Stream()
    runner = Runner(rb.Context(0, stream=stream.cuda_stream), stream)
    errors, loops, end = [], 0, time.monotonic() + float(seconds)
    while (loops == 0 or time.monotonic() < end) and not errors:
        for case in cases:
            rc, outs, value, _ = runner.run(case)
            if rc != 0:
                errors.append(f"{case.name}: rb200_sync returned {rc}")
            elif _digests(outs, value) != want[case.name]:
                errors.append(f"{case.name}: differs from the baseline (loop {loops})")
        loops += 1
    runner.close()
    if errors:
        print("\n".join(errors))
        sys.exit(1)
    print(f"part {part}: {loops} loops of {len(cases)} cases ok")


@pytest.mark.gpu
def test_two_processes_at_once(world, tmp_path):
    """Two processes, time-sliced on the device, each running half the case list in a loop for a few seconds."""
    digests = {c.name: _digests(world.base[c.name].outs, world.base[c.name].value) for c in world.cases}
    path = str(tmp_path / "digests.json")
    json.dump(digests, open(path, "w"))
    results = [None, None]

    def run(part):
        results[part] = _child("child_case_loop", timeout=900, args=(str(part), "2", "6", path))

    ts = [threading.Thread(target=run, args=(p,)) for p in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for part, out in enumerate(results):
        assert out is not None and out.returncode == 0, (part, out.stdout[-3000:] + out.stderr[-3000:])


# ---------------------------------------------------------------------------------------------------- E

R = 8


class GraphKit:
    """varlen encode + async decode of one version captured in one CUDA graph on ctx's stream.  The three versions share
    their context's encode workspace, which each one's eager round trip grows to its own plan, so every kit of a context
    is built (and has grown the workspace) before any of them is captured."""

    def __init__(self, ctx, stream, version):
        torch = _torch()
        self.ctx, self.stream, self.version = ctx, stream, version
        if version == 5:
            self.nb_max, self.bs, self.ch = 40, 65536, 8192
            self.n_max = self.nb_max * self.bs
            self.cap = api.container_blocks_stored_bound(self.nb_max, self.bs, self.ch)
        else:
            self.ch = 8192 if version == 1 else 4096
            self.n_max = (5 << 20) + 333
            self.cap = ctx.container_capacity(self.n_max, self.ch) if version == 1 else api.container_stored_bound(self.n_max, self.ch)
        with torch.cuda.stream(stream):
            self.d_in = torch.zeros(self.n_max + 16, dtype=torch.uint8, device="cuda")
            self.d_len = torch.zeros(1, dtype=torch.int32 if version == 5 else torch.int64, device="cuda")
            self.d_buf = torch.full((self.cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
            self.d_out = torch.full((self.n_max + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
            self.d_nsym = torch.zeros(1, dtype=torch.int64, device="cuda")
            self.d_len.fill_(self.nb_max if version == 5 else self.n_max)
            self.round_trip()                           # grows the workspace outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        self.graph = None

    def capture(self):
        """Only once every kit of this context has run its eager round trip: a graph holds the context's workspace
        pointers, and an eager call that grows the workspace afterwards frees what the graph would write."""
        torch = _torch()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(self.stream):
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.round_trip()

    def round_trip(self):
        c, v = self.ctx, self.version
        if v == 1:
            c.container_model_encode_varlen_async(WORD, 12, self.d_in.data_ptr(), self.d_len.data_ptr(), self.n_max, self.ch, CRC_BLOB,
                                                  self.d_buf.data_ptr(), self.cap)
            c.container_decode_async(self.d_buf.data_ptr(), self.cap, self.d_out.data_ptr(), self.n_max, self.d_nsym.data_ptr())
        elif v == 5:
            c.container_blocks_stored_encode_varlen_async(gbs.THREE, 20000, self.d_in.data_ptr(), self.d_len.data_ptr(), self.nb_max, self.bs,
                                                          self.ch, CRC_BLOB, self.d_buf.data_ptr(), self.cap)
            c.container_blocks_stored_decode_async(self.d_buf.data_ptr(), self.cap, self.d_out.data_ptr(), self.n_max, self.d_nsym.data_ptr())
        else:
            c.container_stored_encode_varlen_async(gs.THREE, 20000, self.d_in.data_ptr(), self.d_len.data_ptr(), self.n_max, self.ch, CRC_BLOB,
                                                   self.d_buf.data_ptr(), self.cap)
            c.container_stored_decode_async(self.d_buf.data_ptr(), self.cap, self.d_out.data_ptr(), self.n_max, self.d_nsym.data_ptr())

    def inputs(self, seed):
        """R (length value, symbols) pairs: lengths (block counts for version 5) and data kinds that change what is stored"""
        out = []
        for i in range(R):
            if self.version == 5:
                count = [1, 40, 7, 23, 40, 2, 31, 16][i]
                kind = ["uniform", "halfuniform", "zipf", "halfuniform", "zipf", "uniform", "halfuniform", "zipf"][i]
                out.append((count, gbs.block_data(kind, count, self.bs, seed + i)))
            else:
                n = [1, self.n_max, 77_777, 3 * self.ch + 1, self.n_max - 1, self.ch, (2 << 20) + 9, 1_000_003][i]
                kind = ["zipf", "mixed", "uniform", "text", "mixed", "const", "zipf", "skew"][i]
                out.append((n, gs.data_of(kind, n, self.ch, seed + i)))
        return out

    def want(self, orl, value, data):
        if self.version == 5:
            return gbs.expected(orl, gbs.THREE, 20000, data, value, self.bs, self.ch, CRC_BLOB)[0]
        if self.version == 6:
            return gs.expected(orl, gs.THREE, 20000, data, self.ch, CRC_BLOB)[0]
        freqs, cum = orl.model(data, 12)
        blob, offs = orl.chunked_encode(WORD, data, freqs, cum, self.ch, scale_bits=12)
        return api.container_pack(WORD, 12, self.ch, data.size, freqs, offs, blob, CRC_BLOB)


@pytest.mark.gpu
@pytest.mark.parametrize("contexts", [1, 2])
def test_graph_replays_queued_without_sync(oracle_lib, contexts):
    """Each context's graphs of versions 1, 5 and 6, captured only after every kit's eager warm-up has grown the
    workspaces the graphs point into, replayed R times back to back on its stream: before each replay a stream-ordered
    update of the length and the input, after it a stream-ordered copy of the container and the decoded symbols into
    slot i; with two contexts both streams are fed at once.  One sync at the end; every slot equals the oracle's
    container and the input."""
    torch = _torch()
    kits = []
    for c in range(contexts):
        stream = torch.cuda.Stream()
        ctx = rb.Context(0, stream=stream.cuda_stream)
        kits += [GraphKit(ctx, stream, v) for v in (1, 5, 6)]
    for kit in kits:                        # every eager call is behind us: the captured workspaces stay allocated
        kit.capture()
    feeds = []
    for k, kit in enumerate(kits):
        ins = kit.inputs(100 * k + 7)
        with torch.cuda.stream(kit.stream):
            src = [torch.from_numpy(d).to("cuda", non_blocking=False) for _, d in ins]
            bufs = torch.empty((R, kit.cap + 64), dtype=torch.uint8, device="cuda")
            outs = torch.empty((R, kit.n_max + 64), dtype=torch.uint8, device="cuda")
            nsyms = torch.empty((R,), dtype=torch.int64, device="cuda")
        feeds.append((ins, src, bufs, outs, nsyms))
    torch.cuda.synchronize()
    for i in range(R):                      # no host synchronisation from here to the end
        for kit, (ins, src, bufs, outs, nsyms) in zip(kits, feeds):
            with torch.cuda.stream(kit.stream):
                value, data = ins[i]
                kit.d_len.fill_(value)
                kit.d_in[:data.size].copy_(src[i])
                kit.d_buf.fill_(SENTINEL)
                kit.d_out.fill_(SENTINEL)
                kit.d_nsym.fill_(-1)
                kit.graph.replay()
                bufs[i].copy_(kit.d_buf)
                outs[i].copy_(kit.d_out)
                nsyms[i:i + 1].copy_(kit.d_nsym)
    for kit in kits[::3]:
        assert kit.ctx.lib.dll.rb200_sync(kit.ctx.h) == 0
    for kit, (ins, src, bufs, outs, nsyms) in zip(kits, feeds):
        got_b, got_o, got_n = bufs.cpu().numpy(), outs.cpu().numpy(), nsyms.cpu().numpy()
        for i, (value, data) in enumerate(ins):
            case = f"context {kits.index(kit) // 3}, version {kit.version}, replay {i}"
            want = kit.want(oracle_lib, value, data)
            assert np.array_equal(got_b[i][:want.size], want), case
            assert (got_b[i][want.size:] == SENTINEL).all(), case
            assert int(got_n[i]) == data.size, case
            assert np.array_equal(got_o[i][:data.size], data) and (got_o[i][data.size:] == SENTINEL).all(), case
    for kit in kits:
        del kit.graph
    for kit in kits[::3]:
        kit.ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,coder,sb,kind,ch", FLAT_DECODES, ids=[d[0] for d in FLAT_DECODES])
def test_decode_queue_with_a_rejected_call(oracle_lib, name, coder, sb, kind, ch):
    """[good, corrupt, good] rb200_decode calls queued with one sync: RB200_E_STREAM, and both good outputs complete --
    the persistent decoders' DecodeWork is re-armed after a rejected chunk with no sync to reset it.  The context then
    decodes again with a clean status."""
    torch = _torch()
    data, freqs, cum, blob, offs = flat_streams(oracle_lib, coder, sb, kind, ch)
    bad = blob.copy()
    mid = (int(offs[1]) + int(offs[2])) // 2
    bad[mid] ^= 0x5A                                    # inside chunk 1's stream
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    model = ctx.model(coder, sb, freqs)
    with torch.cuda.stream(stream):
        d_good, d_bad, d_offs = _dev(blob), _dev(bad), _dev(offs)
        outs = [torch.full((data.size + 64,), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(4)]
        for d_blob, out in zip((d_good, d_bad, d_good), outs):
            ctx.decode_device(model, d_blob.data_ptr(), blob.size, d_offs.data_ptr(), ch, out.data_ptr(), data.size)
    assert ctx.lib.dll.rb200_sync(ctx.h) == E_STREAM
    want = _tail(data, data.size + 64)
    for k in (0, 2):
        got = outs[k].cpu().numpy()
        assert np.array_equal(got, want), (name, k, int(np.flatnonzero(got != want)[0]) if got.size == want.size else None)
    with torch.cuda.stream(stream):
        ctx.decode_device(model, d_good.data_ptr(), blob.size, d_offs.data_ptr(), ch, outs[3].data_ptr(), data.size)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    assert np.array_equal(outs[3].cpu().numpy(), want), name
    model.close()
    ctx.close()


@pytest.mark.gpu
def test_encodes_of_four_paths_queued_without_sync(world):
    """K2r, alias fused, rans64 split and per-block K5f enqueued back to back on one context (they share its scratch
    and sizes workspaces), then one sync: each output equals its baseline."""
    torch = _torch()
    names = ["word-K2r-spill", "alias-fused", "rans64-split", "blocks-word-K5f", "word-K2r", "byte-split"]
    cases = [c for n in names for c in world.cases if c.name == n]
    stream = torch.cuda.Stream()
    runner = Runner(rb.Context(0, stream=stream.cuda_stream), stream)
    for case in cases:                                  # workspaces grown, buffers allocated
        assert check(case, world.base[case.name], *runner.run(case)[:3], runner.ctx) is None
    for rnd in range(2):
        order = cases if rnd == 0 else cases[::-1]
        values = [runner.enqueue(case) for case in order]
        rc = runner.sync()
        for case, value in zip(order, values):
            msg = check(case, world.base[case.name], rc, runner.outs[case.name], value, runner.ctx)
            assert msg is None, f"round {rnd}: {msg}"
    runner.close()
