"""Per-block coders at the geometries the format allows beyond multiples of 1024: ragged chunks (chunk_syms % 32 != 0),
blocks that do not start 16-byte aligned, 2-3 and 9-16 chunks per block (the 4-warp CTA with idle warps, the 512-thread
CTA), 32-symbol chunks, tens of thousands of 32-symbol blocks, chunks above 64 Ki and the largest legal chunk, 2^24.

For every instance of RB200_BLOCK_DISPATCH (the word coder's included), against the
oracle: the models built on the GPU, blob and directory with built and with caller models in both memory kinds, decode
of the oracle's streams and of the GPU's own, the plain DEVICE-mode calls on input and output pointers that are not
16-byte aligned (nothing written outside the output, past blob_bytes or past the last directory entry), the containers
of versions 2, 3 and 4 (device encode against a packer written from the format, open, sync and async decode, a CUDA
graph of encode + async decode), the HOST-mode slice pipeline with slice boundaries off 16 bytes, the word coder's split
and fused encode paths, and the version 3 and 4 block decoders' rejects.  The host-only part packs and opens the same
geometries from oracle streams and checks the geometry rules at their boundaries, without a GPU."""
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, TESTS)
import test_container_blocks as cb2  # noqa: E402
import test_container_blocks_alias as ca  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402

HOST = 0
CRC_BLOB = api.CONTAINER_CRC_BLOB
SENTINEL = 0x5C

# (n_blocks, block_size, chunk_syms)
RAGGED_UNALIGNED = (7, 99, 33)        # 3 chunks of one full step + 1 ragged symbol; blocks at every alignment mod 16
NINE = (5, 9000, 1000)                # 9 chunks per block: 512-thread CTAs; ragged step of 8; blocks 8-byte aligned
SIXTEEN = (6, 16 * 1000, 1000)        # 16 chunks per block: the full 16-warp CTA
TWO = (4, 8194, 4097)                 # 2 chunks per block (idle warps in a 4-warp CTA); ragged by 1; chunk above K2f's 4096
SMALLEST = (3, 1024, 32)              # 32 chunks of the minimum 32 symbols: the smallest streams
TINY = (16384, 32, 32)                # many tiny blocks: model section 8 MiB against 512 KiB of data
ABOVE_64K = (3, 3 << 17, 1 << 17)     # chunks above 64 Ki through K5f (word, models built) and the split per-block encoders
LARGEST = (1, 1 << 24, 1 << 24)       # the largest legal chunk, one block
GEOMETRIES = [RAGGED_UNALIGNED, NINE, SIXTEEN, TWO, SMALLEST, TINY, ABOVE_64K, LARGEST]

# one kind per block, in this order: a const block (word frequency 4096, byte / rans64 at 32768 for scale_bits 15, a full
# alias bucket) from two blocks on, a uniform block (at scale_bits 8 normalize_freqs steals slots) from three on
KINDS = ["zipf", "const", "uniform", "text", "two", "skew"]


class Inst:
    """One coder at one scale_bits: the per-block and container calls of its container version, (coder, scale_bits)
    bound as each call family takes them."""

    def __init__(self, name, coder, sb):
        self.name, self.coder, self.sb = name, coder, sb
        if coder == rb.CODER_WORD:
            self.version, self.stem, self.pre, self.py_pack, self.ocoder = 2, "blocks", (), cb2.py_pack, orc.CODER_WORD
        elif coder == rb.CODER_ALIAS:
            self.version, self.stem, self.pre, self.py_pack, self.ocoder = 4, "blocks_alias", (sb,), ca.py_pack, orc.CODER_ALIAS
        else:
            self.version, self.stem, self.pre, self.py_pack = 3, "blocks_coder", (coder, sb), cc.py_pack
            self.ocoder = {rb.CODER_BYTE: orc.CODER_BYTE, rb.CODER_RANS64: orc.CODER_RANS64}[coder]
        self.unit = 4 if coder == rb.CODER_RANS64 else (2 if coder == rb.CODER_WORD else 1)   # stream renormalisation bytes
        self.state_bytes = 8 if coder == rb.CODER_RANS64 else 4                              # one lane's state in the header

    def __repr__(self):
        return self.name

    def ctx(self, ctx, what):
        """ctx.<stem>_<what>, or ctx.container_<stem>_<...> for what = 'container_...', with (coder, sb) bound where the
        call takes them (the container decodes read them from the header)"""
        name = f"container_{self.stem}_{what[10:]}" if what.startswith("container_") else f"{self.stem}_{what}"
        return getattr(ctx, name) if what.startswith("container_decode") else functools.partial(getattr(ctx, name), *self.pre)

    def pack(self, *a):
        return getattr(api, f"container_{self.stem}_pack")(*self.pre, *a)

    def open(self, buf):
        return getattr(api, f"container_{self.stem}_open")(buf)

    def dll(self, lib, what):
        """the C call rb200_<stem>_<what> (or rb200_container_<stem>_<...>) as fn(ctx handle, *rest)"""
        fn = getattr(lib, f"rb200_container_{self.stem}_{what[10:]}" if what.startswith("container_") else f"rb200_{self.stem}_{what}")
        return lambda h, *a: fn(h, *self.pre, *a)


WORD = Inst("word", rb.CODER_WORD, 12)
BYTE = {sb: Inst(f"byte{sb}", rb.CODER_BYTE, sb) for sb in (14, 12, 8, 11, 15)}
RANS64 = {sb: Inst(f"rans64-{sb}", rb.CODER_RANS64, sb) for sb in (14, 12, 11, 15)}
ALIAS = {sb: Inst(f"alias{sb}", rb.CODER_ALIAS, sb) for sb in (14, 12, 8, 11, 15)}
# every dispatch instance: word; byte at 14, 12 and generic (8, 11, 15); rans64 (one instance) at 14, 12, 11; alias at
# 14, 12 and generic (8, 11, 15)
INSTANCES = [WORD, *BYTE.values(), RANS64[14], RANS64[12], RANS64[11], *ALIAS.values()]

# The ragged and unaligned geometries run every instance; the others one instance of each coder, scale_bits rotated
# (LARGEST only the word coder and the byte coder, to bound the time).
CASES = ([(i, g) for g in (RAGGED_UNALIGNED, NINE, TWO) for i in INSTANCES]
         + [(i, SIXTEEN) for i in (WORD, BYTE[15], RANS64[14], ALIAS[11])]
         + [(i, SMALLEST) for i in (WORD, BYTE[12], RANS64[11], ALIAS[15])]
         + [(i, TINY) for i in (WORD, BYTE[14], RANS64[12], ALIAS[8])]
         + [(i, ABOVE_64K) for i in (WORD, BYTE[8], RANS64[15], ALIAS[12])]
         + [(i, LARGEST) for i in (WORD, BYTE[14])])


def _gid(g):
    return f"{g[0]}x{g[1]}-by-{g[2]}"


def _cid(c):
    return f"{c[0].name}-{_gid(c[1])}"


@functools.lru_cache(maxsize=None)
def block_data(geo):
    """The blocks of `geo`, kind KINDS[b % 6] and seed 500 + b per block (read-only: shared between tests)"""
    import conftest
    nb, bs, _ = geo
    out = np.concatenate([conftest._gen(KINDS[b % len(KINDS)], bs, 500 + b) for b in range(nb)])
    out.flags.writeable = False
    return out


_ORACLE = {}


def oracle_streams(oracle_lib, inst, geo):
    """(block_freqs, offsets, blob) by the oracle: every block's normalize_freqs(count_freqs(block), 1 << sb) and its
    chunked encode, directories rebased (cached for the largest geometries)"""
    key = (inst.ocoder, inst.sb, geo)
    if key not in _ORACLE:
        if len(_ORACLE) > 8:
            _ORACLE.clear()
        _ORACLE[key] = cc.oracle_blocks_encode(oracle_lib, inst.ocoder, inst.sb, block_data(geo), *geo)
    return _ORACLE[key]


def _where(inst, geo, offs, pos):
    """block, chunk, lane (within the stream header) or byte of blob position `pos`, by the oracle's directory"""
    per = geo[1] // geo[2]
    c = int(np.searchsorted(offs, pos, side="right")) - 1
    c = min(max(c, 0), offs.size - 2)
    at = pos - int(offs[c])
    where = f"lane {at // inst.state_bytes} of the header" if 0 <= at < 32 * inst.state_bytes else f"byte {at} of the stream"
    return f"block {c // per}, chunk {c % per}, {where}"


def same(what, inst, geo, got, want, offs=None):
    """assert_equal with the first difference mapped back to block, chunk and lane: models [n_blocks, 256] (what
    'models'), directories (what 'directory'), blobs (offs: the oracle's directory) or decoded symbols"""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape == want.shape and np.array_equal(got, want):
        return
    ctx = f"{inst.name} at {geo}: {what}"
    if got.shape != want.shape:
        pytest.fail(f"{ctx}: shape {got.shape} != {want.shape}")
    i = int(np.flatnonzero((got != want).reshape(-1))[0])
    per = geo[1] // geo[2]
    if what.startswith("models"):
        msg = f"block {i // 256} symbol {i % 256}: {got.reshape(-1)[i]} != {want.reshape(-1)[i]}"
    elif what.startswith("directory"):
        msg = f"entry {i} (block {i // per}, chunk {i % per}): {got[i]} != {want[i]}"
    elif offs is not None:
        msg = f"byte {i} ({_where(inst, geo, offs, i)}): {got[i]:#x} != {want[i]:#x}"
    else:
        msg = f"symbol {i} (block {i // geo[1]}, chunk {i % geo[1] // geo[2]}, step {i % geo[1] % geo[2] // 32})"
    pytest.fail(f"{ctx}: {int((got != want).sum())} differ, first at {msg}")


def _k(inst, geo):
    """the misalignment (1..15 bytes) of this case's input and output pointers"""
    return 1 + (geo[0] + geo[1] + geo[2] + inst.coder + inst.sb) % 15


# ---------------------------------------------------------------------------------------------------- host-only part

HOST_CASES = ([(i, g) for g in GEOMETRIES[:-1] for i in (WORD, BYTE[14], RANS64[11], ALIAS[15])]
              + [(i, LARGEST) for i in (WORD, BYTE[14])])


@pytest.mark.parametrize("inst,geo", HOST_CASES, ids=[_cid(c) for c in HOST_CASES])
def test_pack_open_and_oracle_decode(oracle_lib, inst, geo):
    """version 2/3/4 pack of oracle streams at the geometry equals the packer written from the format; open accepts it
    and returns the geometry; the oracle decodes the opened views back to the data"""
    nb, bs, ch = geo
    freqs, offs, blob = oracle_streams(oracle_lib, inst, geo)
    for flags in (0, CRC_BLOB):
        buf = inst.pack(nb, bs, ch, freqs, offs, blob, flags)
        same(f"pack, flags {flags}", inst, geo, buf, inst.py_pack(*inst.pre, nb, bs, ch, freqs, offs, blob, flags))
        meta, f2, o2, b2 = inst.open(buf)
        want = {"n_blocks": nb, "block_size": bs, "chunk_syms": ch, "flags": flags, "n_symbols": nb * bs,
                "n_chunks": nb * (bs // ch), "blob_bytes": blob.size}
        if inst.version > 2:
            want.update(coder=inst.coder, scale_bits=inst.sb)
        assert meta == want
        assert np.array_equal(f2, freqs) and np.array_equal(o2, offs) and np.array_equal(b2, blob)
    meta = dict(meta, scale_bits=inst.sb)
    same("oracle decode of the opened container", inst, geo, cc.oracle_decode_blocks(oracle_lib, inst.ocoder, meta, f2, o2, b2),
         block_data(geo))


# (n_blocks, block_size, chunk_syms) the format refuses: 33 chunks per block; chunk_syms 31; block_size % chunk_syms != 0
ILLEGAL = [(1, 33 * 32, 32), (1, 4 * 31, 31), (1, 100, 33)]
# and its edges, accepted: 32 chunks per block; chunk_syms 32 (one chunk per block)
EDGES = [(2, 32 * 32, 32), (3, 32, 32)]


def _illegal_streams(oracle_lib, inst, geo):
    """a container's arrays for a geometry the format refuses, consistent in every other way: each block's first
    (block_size // chunk_syms) * chunk_syms symbols encoded by the oracle in chunks of chunk_syms"""
    nb, bs, ch = geo
    data = block_data(geo)
    freqs, parts, offs, base = [], [], [], 0
    for b in range(nb):
        blk = data[b * bs:(b + 1) * bs]
        f, c = oracle_lib.model(blk, inst.sb)
        ob, oo = oracle_lib.chunked_encode(inst.ocoder, blk[:bs // ch * ch], f, c, ch, scale_bits=inst.sb)
        freqs.append(f)
        parts.append(ob)
        offs.append(oo[:-1] + base)
        base += ob.size
    return (np.stack(freqs).astype(np.uint16), np.concatenate(offs + [[base]]).astype(np.uint64),
            np.concatenate(parts).astype(np.uint8))


@pytest.mark.parametrize("inst", [WORD, BYTE[14], RANS64[12], ALIAS[11]], ids=repr)
def test_geometry_rules_at_their_boundaries(oracle_lib, inst):
    """33 chunks per block, chunk_syms 31 and block_size % chunk_syms != 0 are refused by pack (-1) and by open (-4, a
    container otherwise consistent and correctly checksummed); 32 chunks per block and chunk_syms 32 are accepted"""
    for geo in ILLEGAL:
        nb, bs, ch = geo
        freqs, offs, blob = _illegal_streams(oracle_lib, inst, geo)
        assert offs.size == nb * (bs // ch) + 1
        with pytest.raises(rb.RansError) as ei:
            inst.pack(nb, bs, ch, freqs, offs, blob, 0)
        assert ei.value.code == -1, geo
        for flags in (0, CRC_BLOB):
            with pytest.raises(rb.RansError) as ei:
                inst.open(inst.py_pack(*inst.pre, nb, bs, ch, freqs, offs, blob, flags))
            assert ei.value.code == -4, (geo, flags)
    for geo in EDGES:
        nb, bs, ch = geo
        freqs, offs, blob = oracle_streams(oracle_lib, inst, geo)
        meta = inst.open(inst.pack(nb, bs, ch, freqs, offs, blob, CRC_BLOB))[0]
        assert (meta["n_blocks"], meta["block_size"], meta["chunk_syms"]) == geo


# ---------------------------------------------------------------------------------------------------- GPU part

def _torch():
    import torch
    return torch


def _dev_at(a, k=0, pad=64, fill=SENTINEL):
    """a device copy of `a`'s bytes at byte offset k of a buffer filled with `fill`, `pad` bytes of it after the copy"""
    torch = _torch()
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    t = torch.full((k + a.size + pad,), fill, dtype=torch.uint8, device="cuda")
    if a.size:
        t[k:k + a.size] = torch.from_numpy(a.copy())
    return t


def _untouched(t):
    return bool((t == SENTINEL).all().item())


@pytest.fixture(scope="module")
def blocks_ctx(cuda_box):
    """this module's own context: the workspaces its largest geometries grow (K5f's scratch reaches 512 MiB at
    LARGEST) are freed when the module ends, rather than held by the session's context for every later module"""
    ctx = rb.Context(0)
    try:
        yield ctx
    finally:
        ctx.close()


def _device_encode(ctx, inst, geo, d_in, k, caller_freqs):
    """the plain DEVICE-mode model_encode (caller_freqs None) or encode on input d_in + k into sentinel-filled blob,
    directory and model buffers: (blob, offsets, models, d_blob, d_off, d_freqs), after checking that nothing was written
    past blob_bytes, past directory entry n_chunks or (model_encode) past the last model row"""
    torch = _torch()
    nb, bs, ch = geo
    n, n_chunks = nb * bs, nb * (bs // ch)
    cap = ctx.encode_bound(n, ch)
    d_freqs = _dev_at(np.full((nb, 256), 0x5C5C, np.uint16) if caller_freqs is None else caller_freqs, pad=512)
    d_blob = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_off = torch.full(((n_chunks + 5) * 8,), SENTINEL, dtype=torch.uint8, device="cuda")
    fn = inst.ctx(ctx, "model_encode_device" if caller_freqs is None else "encode_device")
    fn(d_in.data_ptr() + k, nb, bs, d_freqs.data_ptr(), ch, d_blob.data_ptr(), cap, d_off.data_ptr())
    ctx.sync()
    offs = d_off[:(n_chunks + 1) * 8].cpu().numpy().view(np.uint64)
    assert _untouched(d_off[(n_chunks + 1) * 8:]), "directory written past entry n_chunks"
    size = int(offs[-1])
    assert size <= cap
    assert _untouched(d_blob[size:]), "blob written past blob_bytes"
    assert _untouched(d_freqs[nb * 512:]), "models written past the last block"
    freqs = d_freqs[:nb * 512].cpu().numpy().view(np.uint16).reshape(nb, 256)
    return d_blob[:size].cpu().numpy(), offs, freqs, d_blob, d_off, d_freqs


def _device_decode(ctx, inst, geo, d_blob, blob_size, d_off, d_freqs, k):
    """the plain DEVICE-mode decode into out + k of a sentinel-filled buffer: the symbols, after checking that nothing
    before out or at or after out + n_blocks * block_size was written"""
    torch = _torch()
    nb, bs, ch = geo
    n = nb * bs
    d_out = torch.full((k + n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    inst.ctx(ctx, "decode_device")(d_blob.data_ptr(), blob_size, d_off.data_ptr(), d_freqs.data_ptr(), nb, bs, ch, d_out.data_ptr() + k)
    ctx.sync()
    assert _untouched(d_out[:k]) and _untouched(d_out[k + n:]), "decode wrote outside [out, out + n)"
    return d_out[k:k + n].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("inst,geo", CASES, ids=[_cid(c) for c in CASES])
def test_models_streams_and_decode(blocks_ctx, oracle_lib, inst, geo):
    nb, bs, ch = geo
    data = block_data(geo)
    want_f, want_o, want_b = oracle_streams(oracle_lib, inst, geo)
    k = _k(inst, geo)
    # HOST mode: models built on the GPU, then the caller's models
    blob, offs, freqs = inst.ctx(blocks_ctx, "model_encode_host")(data, nb, bs, ch)
    same("models (model_encode, HOST)", inst, geo, freqs, want_f)
    same("directory (model_encode, HOST)", inst, geo, offs, want_o)
    same("blob (model_encode, HOST)", inst, geo, blob, want_b, want_o)
    blob, offs = inst.ctx(blocks_ctx, "encode_host")(data, nb, bs, want_f, ch)
    same("directory (encode, HOST)", inst, geo, offs, want_o)
    same("blob (encode, HOST)", inst, geo, blob, want_b, want_o)
    # DEVICE mode on an input k bytes past 16-byte alignment
    d_in = _dev_at(data, k)
    if inst.coder == rb.CODER_WORD:
        same("models (blocks_build_models, HOST)", inst, geo, blocks_ctx.blocks_build_models(data, nb, bs), want_f)
        d_freqs = _dev_at(np.full((nb, 256), 0x5C5C, np.uint16), pad=512)
        blocks_ctx.blocks_build_models_device(d_in.data_ptr() + k, nb, bs, d_freqs.data_ptr())
        blocks_ctx.sync()
        assert _untouched(d_freqs[nb * 512:])
        same("models (blocks_build_models, DEVICE)", inst, geo, d_freqs[:nb * 512].cpu().numpy().view(np.uint16).reshape(nb, 256), want_f)
    blob, offs, freqs, d_blob, d_off, d_freqs = _device_encode(blocks_ctx, inst, geo, d_in, k, None)
    same("models (model_encode, DEVICE)", inst, geo, freqs, want_f)
    same("directory (model_encode, DEVICE)", inst, geo, offs, want_o)
    same("blob (model_encode, DEVICE)", inst, geo, blob, want_b, want_o)
    # decode of the GPU's own streams, where the encode left them; output k bytes past alignment
    same("decode of the GPU's streams (DEVICE)", inst, geo, _device_decode(blocks_ctx, inst, geo, d_blob, blob.size, d_off, d_freqs, k), data)
    blob, offs, _, _, _, _ = _device_encode(blocks_ctx, inst, geo, _dev_at(data, 16 - k), 16 - k, want_f)
    same("directory (encode, DEVICE)", inst, geo, offs, want_o)
    same("blob (encode, DEVICE)", inst, geo, blob, want_b, want_o)
    # decode of the oracle's streams
    same("decode of the oracle's streams (HOST)", inst, geo, inst.ctx(blocks_ctx, "decode_host")(want_b, want_o, want_f, nb, bs, ch), data)
    out = _device_decode(blocks_ctx, inst, geo, _dev_at(want_b), want_b.size, _dev_at(want_o), _dev_at(want_f), (k + 5) % 16)
    same("decode of the oracle's streams (DEVICE)", inst, geo, out, data)


@pytest.mark.gpu
@pytest.mark.parametrize("inst,geo", CASES, ids=[_cid(c) for c in CASES])
def test_containers(blocks_ctx, oracle_lib, inst, geo):
    """the device container encode (input k bytes past alignment, models built and the caller's) equals the packer
    written from the format over the oracle's streams, with and without CRC_BLOB; open accepts it; the sync decode in
    both memory kinds and the async decode return the data and the symbol count"""
    torch = _torch()
    nb, bs, ch = geo
    n = nb * bs
    data = block_data(geo)
    want_f, want_o, want_b = oracle_streams(oracle_lib, inst, geo)
    k = _k(inst, geo)
    d_in = _dev_at(data, k)
    d_freqs = _dev_at(want_f)
    cap = blocks_ctx.container_blocks_capacity(nb, bs, ch)
    for flags in (0, CRC_BLOB):
        want = inst.py_pack(*inst.pre, nb, bs, ch, want_f, want_o, want_b, flags)
        for name, fp in (("models built", None), ("caller models", d_freqs.data_ptr())):
            d_buf = torch.full((cap + 16,), 0xAA, dtype=torch.uint8, device="cuda")
            inst.ctx(blocks_ctx, "container_encode_device")(d_in.data_ptr() + k, nb, bs, fp, ch, flags, d_buf.data_ptr(), cap)
            blocks_ctx.sync()
            same(f"container (device encode, {name}, flags {flags})", inst, geo, d_buf[:want.size].cpu().numpy(), want)
        same(f"container (HOST encode, flags {flags})", inst, geo, inst.ctx(blocks_ctx, "container_encode_host")(data, nb, bs, ch, None, flags),
             want)
        meta = inst.open(want)[0]
        assert (meta["n_blocks"], meta["block_size"], meta["chunk_syms"], meta["n_symbols"]) == (nb, bs, ch, n)
        same(f"container decode (HOST, flags {flags})", inst, geo, inst.ctx(blocks_ctx, "container_decode_host")(want), data)
        d_out = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        assert inst.ctx(blocks_ctx, "container_decode_device")(d_buf.data_ptr(), want.size, d_out.data_ptr(), n) == n
        same(f"container decode (DEVICE, flags {flags})", inst, geo, d_out[:n].cpu().numpy(), data)
        assert _untouched(d_out[n:])
        d_out.fill_(SENTINEL)
        d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        inst.ctx(blocks_ctx, "container_decode_async")(d_buf.data_ptr(), want.size, d_out.data_ptr(), n, d_n.data_ptr())
        assert blocks_ctx.lib.dll.rb200_sync(blocks_ctx.h) == 0
        assert int(d_n.item()) == n
        same(f"container decode (async, flags {flags})", inst, geo, d_out[:n].cpu().numpy(), data)
        assert _untouched(d_out[n:])


GRAPH_CASES = [(WORD, NINE), (BYTE[12], RAGGED_UNALIGNED), (ALIAS[11], TWO)]


@pytest.mark.gpu
@pytest.mark.parametrize("inst,geo", GRAPH_CASES, ids=[_cid(c) for c in GRAPH_CASES])
def test_encode_and_async_decode_in_one_cuda_graph(gen, inst, geo):
    """container encode (models built, input off alignment) and the async decode captured together at a ragged
    geometry, replayed on new data of that geometry"""
    torch = _torch()
    nb, bs, ch = geo
    n, k = nb * bs, 3
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    g = None
    try:
        cap = ctx.container_blocks_capacity(nb, bs, ch)
        d_in = torch.zeros(n + k + 16, dtype=torch.uint8, device="cuda")
        d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
        d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
        d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

        def round_trip():
            inst.ctx(ctx, "container_encode_device")(d_in.data_ptr() + k, nb, bs, None, ch, CRC_BLOB, d_buf.data_ptr(), cap)
            inst.ctx(ctx, "container_decode_async")(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

        with torch.cuda.stream(stream):
            d_in[k:k + n].copy_(torch.from_numpy(block_data(geo).copy()))
            round_trip()                                             # grows the encoder's workspaces outside the capture
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                round_trip()
            for seed in (61, 62):
                data = np.concatenate([gen(KINDS[(b + seed) % len(KINDS)], bs, seed * 100 + b) for b in range(nb)])
                d_in[k:k + n].copy_(torch.from_numpy(data))
                d_out.zero_()
                d_n.zero_()
                g.replay()
                assert ctx.lib.dll.rb200_sync(ctx.h) == 0
                assert int(d_n.item()) == n
                same(f"graph replay {seed}", inst, geo, d_out[:n].cpu().numpy(), data)
    finally:
        stream.synchronize()
        del g
        ctx.close()


@pytest.mark.gpu
def test_fused_encode_scratch_is_capped(cuda_box, oracle_lib):
    """K5f (the word coder's model-building per-block encode) over 32 blocks of one 2^24-symbol chunk: plan_blocks_encode
    caps its worker CTAs so that their scratch stays within 2 GiB (uncapped, 33 CTAs x 4 warps x 2 slots of 32 MiB
    would take 8.25 GiB), and the capped grid, 6 workers for 32 blocks, still codes every block as the oracle does"""
    torch = _torch()
    nb, bs = 32, 1 << 24
    n = nb * bs
    g = torch.Generator(device="cuda").manual_seed(5)
    d_in = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    for b in range(nb):                                              # a different alphabet size, so a different model, per block
        d_in[b * bs:(b + 1) * bs] = torch.randint(0, 2 + 8 * b, (bs,), device="cuda", generator=g, dtype=torch.uint8)
    cap = int(rb.load().dll.rb200_encode_bound(n, bs))
    d_blob = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_off = torch.empty((nb + 1) * 8, dtype=torch.uint8, device="cuda")
    d_freqs = torch.empty(nb * 512, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    ctx = rb.Context(0)
    try:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        ctx.blocks_model_encode_device(d_in.data_ptr(), nb, bs, d_freqs.data_ptr(), bs, d_blob.data_ptr(), cap, d_off.data_ptr())
        ctx.sync()
        grown = free0 - torch.cuda.mem_get_info()[0]
        assert grown <= (2 << 30) + (128 << 20), f"the encode took {grown / 2**30:.2f} GiB of device memory"
        offs = d_off.cpu().numpy().view(np.uint64)
        freqs = d_freqs.cpu().numpy().view(np.uint16).reshape(nb, 256)
        for b in (0, 13, nb - 1):
            blk = d_in[b * bs:(b + 1) * bs].cpu().numpy()
            f, c = oracle_lib.model(blk, 12)
            assert np.array_equal(freqs[b], f), b
            ob, _ = oracle_lib.chunked_encode(orc.CODER_WORD, blk, f, c, bs)
            assert np.array_equal(d_blob[int(offs[b]) & ~15:int(offs[b + 1]) & ~15].cpu().numpy(), ob), b
        ctx.blocks_decode_device(d_blob.data_ptr(), int(offs[-1]), d_off.data_ptr(), d_freqs.data_ptr(), nb, bs, bs, d_out.data_ptr())
        ctx.sync()
        assert torch.equal(d_out, d_in[:n])
    finally:
        ctx.close()


# ---- the word coder's encode paths and the HOST-mode slice pipeline, each in a child process with its environment

def child_word_paths():
    """every geometry for the word coder, HOST and DEVICE mode, models built (always K5f) and the caller's (K5 or K5f,
    by RB200_ENCODE_PATH; K5 above 64 Ki): streams equal the oracle's"""
    oracle_lib, ctx = orc.Oracle(), rb.Context(0)
    for geo in GEOMETRIES:
        nb, bs, ch = geo
        data = block_data(geo)
        want_f, want_o, want_b = cc.oracle_blocks_encode(oracle_lib, orc.CODER_WORD, 12, data, *geo)
        blob, offs, freqs = ctx.blocks_model_encode_host(data, nb, bs, ch)
        same("models", WORD, geo, freqs, want_f)
        same("blob (model_encode)", WORD, geo, blob, want_b, want_o)
        same("directory (model_encode)", WORD, geo, offs, want_o)
        blob, offs = ctx.blocks_encode_host(data, nb, bs, want_f, ch)
        same("blob (encode)", WORD, geo, blob, want_b, want_o)
        same("directory (encode)", WORD, geo, offs, want_o)
        d_in = _dev_at(data, 7)
        for f in (None, want_f):
            blob, offs, _, _, _, _ = _device_encode(ctx, WORD, geo, d_in, 7, f)
            same(f"blob (DEVICE, {'built' if f is None else 'caller'} models)", WORD, geo, blob, want_b, want_o)
            same(f"directory (DEVICE, {'built' if f is None else 'caller'} models)", WORD, geo, offs, want_o)
        print("word paths ok", geo, flush=True)


# NINE: one 45000-byte slice; (50000, 99, 33): 4.7 MiB of 99-byte blocks, enough for plan_slices' ramp, so that slices
# start at byte offsets that are not multiples of 16 (slice_starts)
SLICED = [NINE, (50000, 99, 33)]
SLICE_MIB = 1


def slice_starts(n_units, unit_bytes, slice_mib):
    """the byte offsets at which the HOST-mode pipelines' slices of whole blocks start: plan_slices' rule (rans_b200.cu)
    for n_units blocks of unit_bytes symbols, RB200_SLICE_MIB=slice_mib, 256 slices at most"""
    tc = max(-(-(slice_mib << 20) // unit_bytes), 1)                  # blocks per steady-state slice
    room = 256 - 8
    if n_units // tc >= room:
        tc = n_units // room + 1
    ramp = [tc // 8, tc // 4, tc // 2]
    ramped = n_units >= 4 * tc and ramp[0] > 0
    tail = sum(ramp) if ramped else 0
    counts = list(ramp) if ramped else []
    c = sum(counts)
    while n_units - c > tail:
        counts.append(min(n_units - c - tail, tc))
        c += counts[-1]
    counts += ramp[::-1] if ramped else []
    assert sum(counts) == n_units
    return np.cumsum([0] + counts[:-1]) * unit_bytes


def test_sliced_geometry_puts_slice_starts_off_16_bytes():
    nb, bs, _ = SLICED[1]
    starts = slice_starts(nb, bs, SLICE_MIB)
    assert len(starts) > 4 and (starts % 16 != 0).sum() >= 4, starts


def child_slices():
    """RB200_SLICE_MIB=SLICE_MIB: the HOST-mode per-block and container calls of every coder over many slices"""
    oracle_lib, ctx = orc.Oracle(), rb.Context(0)
    for geo in SLICED:
        nb, bs, ch = geo
        data = block_data(geo)
        for inst in (WORD, BYTE[14], RANS64[11], ALIAS[12]):
            want_f, want_o, want_b = cc.oracle_blocks_encode(oracle_lib, inst.ocoder, inst.sb, data, *geo)
            blob, offs, freqs = inst.ctx(ctx, "model_encode_host")(data, nb, bs, ch)
            same("models", inst, geo, freqs, want_f)
            same("directory (model_encode)", inst, geo, offs, want_o)
            same("blob (model_encode)", inst, geo, blob, want_b, want_o)
            blob, offs = inst.ctx(ctx, "encode_host")(data, nb, bs, want_f, ch)
            same("directory (encode)", inst, geo, offs, want_o)
            same("blob (encode)", inst, geo, blob, want_b, want_o)
            same("decode", inst, geo, inst.ctx(ctx, "decode_host")(want_b, want_o, want_f, nb, bs, ch), data)
            want = inst.py_pack(*inst.pre, nb, bs, ch, want_f, want_o, want_b, CRC_BLOB)
            got = inst.ctx(ctx, "container_encode_host")(data, nb, bs, ch, None, CRC_BLOB)
            same("container (models built)", inst, geo, got, want)
            same("container (caller models)", inst, geo, inst.ctx(ctx, "container_encode_host")(data, nb, bs, ch, want_f, CRC_BLOB), want)
            same("container decode", inst, geo, inst.ctx(ctx, "container_decode_host")(want), data)
            print("slices ok", inst, geo, flush=True)


def _child(fn, env):
    code = f"import sys; sys.path.insert(0, {TESTS!r}); sys.path.insert(0, {ROOT!r}); import test_gpu_blocks_geometry as t; t.{fn}()"
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    return out.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["split", "fused"])
def test_word_encode_paths(cuda_box, path):
    assert _child("child_word_paths", {"RB200_ENCODE_PATH": path}).count("word paths ok") == len(GEOMETRIES)


@pytest.mark.gpu
def test_host_slice_pipeline(cuda_box):
    nb, bs, _ = SLICED[1]
    assert (slice_starts(nb, bs, SLICE_MIB) % 16 != 0).any()
    assert _child("child_slices", {"RB200_SLICE_MIB": str(SLICE_MIB)}).count("slices ok") == 4 * len(SLICED)


# ---- rejects of block_decode_kernel

def _bad_inputs(blob, offs, unit, flip_chunks):
    """(what, blob, offsets, chunk whose output must stay untouched or None): a flipped byte inside each chunk of
    flip_chunks' stream, a last entry past the blob, one ending before the stream header, and (unit > 1) a chunk start
    inside a renormalisation unit"""
    import test_decode_rejects as dr
    for c in flip_chunks:
        yield ("flip", c), dr._flipped(blob, offs, c), offs, None
    for c, o in dr._bad_directories(offs, blob.size, unit):
        yield ("directory", c), blob, o, c


@pytest.mark.gpu
@pytest.mark.parametrize("inst", [BYTE[14], BYTE[11], RANS64[12], ALIAS[15]], ids=repr)
def test_block_coder_decoder_rejects(blocks_ctx, oracle_lib, inst):
    """at NINE (ragged steps, 9 chunks per block): a corrupt stream or directory entry is -4, a rejected entry's chunk
    is left untouched, and the context then decodes the intact input correctly twice in a row"""
    geo = NINE
    nb, bs, ch = geo
    data = block_data(geo)
    freqs, offs, blob = oracle_streams(oracle_lib, inst, geo)
    d_freqs = _dev_at(freqs)

    def run(b, o):
        torch = _torch()
        d_out = torch.zeros(data.size, dtype=torch.uint8, device="cuda")
        err = None
        d_blob, d_off = _dev_at(b), _dev_at(o)                  # held until the decode has run
        try:
            inst.ctx(blocks_ctx, "decode_device")(d_blob.data_ptr(), b.size, d_off.data_ptr(), d_freqs.data_ptr(), nb, bs, ch, d_out.data_ptr())
            blocks_ctx.sync()
        except rb.RansError as e:
            err = e
        return d_out.cpu().numpy(), err

    def clean_twice(what):
        for rep in range(2):
            out, err = run(blob, offs)
            assert err is None, (what, rep)
            same(f"decode after {what}, {rep}", inst, geo, out, data)

    clean_twice("nothing")
    per = bs // ch
    for what, b, o, c in _bad_inputs(blob, offs, inst.unit, [1, 2 * per + 3]):   # block 0 (Zipf), block 2 (uniform)
        out, err = run(b, o)
        assert err is not None and err.code == -4, what
        if c is not None:
            lo, hi = c * ch, (c + 1) * ch
            assert data[lo:hi].any() and not out[lo:hi].any(), ("chunk decoded despite its directory entry", what)
        clean_twice(what)


@pytest.mark.gpu
def test_illegal_geometries_launch_nothing(blocks_ctx):
    """33 chunks per block, chunk_syms 31 and block_size % chunk_syms != 0 as arguments: -1 from every per-block and
    container call of every coder, nothing launched"""
    lib = blocks_ctx.lib.dll
    h = blocks_ctx.h
    n0 = blocks_ctx.launches
    for inst in (WORD, BYTE[14], RANS64[12], ALIAS[11]):
        for nb, bs, ch in ILLEGAL:
            data = np.zeros(nb * bs + 16, np.uint8)
            freqs = np.zeros((nb, 256), np.uint16)
            freqs[:, 0] = 1 << inst.sb if inst.sb < 16 else 0
            blob = np.zeros(1 << 16, np.uint8)
            offs = np.zeros(nb * 64, np.uint64)
            out = np.zeros(nb * bs + 16, np.uint8)
            size = C.c_size_t(0)
            p = (data.ctypes.data, nb, bs, freqs.ctypes.data, ch, blob.ctypes.data, blob.size, offs.ctypes.data, C.byref(size), HOST)
            assert inst.dll(lib, "encode")(h, *p) == -1, (inst, nb, bs, ch)
            assert inst.dll(lib, "model_encode")(h, *p) == -1, (inst, nb, bs, ch)
            assert inst.dll(lib, "decode")(h, blob.ctypes.data, blob.size, offs.ctypes.data, freqs.ctypes.data, nb, bs, ch, out.ctypes.data,
                                           HOST) == -1, (inst, nb, bs, ch)
            assert inst.dll(lib, "container_encode")(h, data.ctypes.data, nb, bs, None, ch, 0, blob.ctypes.data, blob.size, C.byref(size),
                                                     HOST) == -1, (inst, nb, bs, ch)
    assert blocks_ctx.launches == n0
