"""Every coder at its rate ceiling: caller models under which each encoder and decoder moves the most bytes a lane can
move in one step.

The rings, mirrors, slots and bounds of the library are sized from that one rate: 2 bytes per lane per step for the
word, byte and alias coders, 4 bytes (one u32, on average 2 bytes per symbol) for rans64.  A model built from its data
codes at the data's entropy, at most 8 bits per symbol, so those buffers are only filled to the brim by caller models
in which the data's symbols are rare.  Each model here has frequency-1 symbols (255 of them, or one) and a dominant
symbol that holds the rest of 1 << scale_bits:
  - "ceiling" data draws every symbol from the frequency-1 ones: scale_bits bits per symbol, so at scale_bits 16 the
    byte and alias streams are exactly 2 m + 128 bytes for a chunk of m symbols and rans64's 2 m + 256, and the word
    coder's chunks of 8192 make 12 416-byte streams, longer than K2r's 9 472-byte ring;
  - "floor" data is the dominant symbol alone, streams of little more than their header;
  - "regions" alternate the two in regions of one step to three chunks, not aligned to chunks, so neighbouring streams
    range from header-only to the ceiling (the scanner, placement, compaction, slot reuse and K2r's spill);
  - "mix50" / "mix97" are Bernoulli mixtures with 50 % / 97 % ceiling symbols, which leave the encoders' output rings
    a spread of pending byte counts just under their flush test.
Every encode is compared byte for byte (directory and blob) with the oracle's chunked encode, every decode with the
data, and device-memory decodes leave the sentinel bytes past n untouched.  The test without a GPU pins the oracle to
the reference's own code on every model here.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
WORD, BYTE, ALIAS, RANS64 = orc.CODER_WORD, orc.CODER_BYTE, orc.CODER_ALIAS, orc.CODER_RANS64   # the library's numbering too
CRC_BLOB = 1
E_SPACE = -3
SENTINEL = 0x5C
RING_BYTES = 9472            # K2r's per-warp stream ring (RB200_RING_BYTES in word_kernels.cuh)
RING_WARPS = 20              # K2r's warps per CTA, one CTA per SM (RB200_RING_WARPS)
FUSED_WORD_WARPS = 2 * 16    # K2f: 2 CTAs of 16 warps per SM (RB200_FUSED_MINBLOCKS x kEncWarps)
FUSED_ALIAS_WARPS = 32       # the fused alias / byte encoder: one CTA of 32 warps per SM (kAliasEncWarps)
SLOTS_PER_WARP = 2           # every fused encoder: two scratch / spill slots per worker warp
DOM, REM, ONE = 0x41, 0xC8, 0x07
SHAPES = ["ceiling", "floor", "regions", "mix50", "mix97"]


def _freqs(sb, kind):
    f = np.zeros(256, np.uint32)
    total = 1 << sb
    if kind == "ones":             # scale_bits 8: every symbol has frequency 1
        f[:] = 1
    elif kind == "dom":            # 255 x 1 + a dominant symbol
        f[:] = 1
        f[DOM] = total - 255
    elif kind == "pair":           # {total - 1, 1}: the largest frequency the coder takes next to one rare symbol
        f[DOM], f[ONE] = total - 1, 1
    else:                          # word: 254 x 1, a symbol with the remainder and a dominant symbol of `kind`
        f[:] = 1
        f[DOM] = int(kind)
        f[REM] = total - int(kind) - 254
    assert int(f.sum()) == total
    return f


# name -> (coder, scale_bits, model kind).  Word: 2963 keeps the 32-bit reciprocal exact, 2964 is the first frequency
# that needs the 33-bit one (test_device_tables.py), so both R32 instances of the word encoder run at the ceiling.
# Alias 10 and byte 15 / 8 are the generic (<0>) decoder instances, the others the specialised ones.
MODELS = {
    "word12-pair": (WORD, 12, "pair"), "word12-dom": (WORD, 12, "dom"),
    "word12-d2963": (WORD, 12, "2963"), "word12-d2964": (WORD, 12, "2964"),
    "byte8": (BYTE, 8, "ones"), "byte12": (BYTE, 12, "dom"), "byte14": (BYTE, 14, "dom"), "byte15": (BYTE, 15, "dom"),
    "byte16": (BYTE, 16, "dom"), "byte16-pair": (BYTE, 16, "pair"),
    "alias8": (ALIAS, 8, "ones"), "alias10": (ALIAS, 10, "dom"), "alias12": (ALIAS, 12, "dom"), "alias14": (ALIAS, 14, "dom"),
    "alias16": (ALIAS, 16, "dom"),
    "rans64-8": (RANS64, 8, "ones"), "rans64-14": (RANS64, 14, "dom"), "rans64-16": (RANS64, 16, "dom"),
}


def model(name):
    """(coder, scale_bits, freqs, cum) of a model in MODELS"""
    coder, sb, kind = MODELS[name]
    f = _freqs(sb, kind)
    return coder, sb, f, np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)


def rate_data(freqs, shape, n, seed, lo=32, hi=3 * 8192):
    """`shape` data (SHAPES) for a model: ceiling symbols are drawn uniformly from its frequency-1 symbols, floor symbols
    are its most frequent one; regions are lo..hi symbols long"""
    rng = np.random.default_rng(seed)
    ones = np.flatnonzero(freqs == 1).astype(np.uint8)
    top = np.uint8(np.argmax(freqs))
    if shape == "floor":
        return np.full(n, top, np.uint8)
    ceil = ones[rng.integers(0, ones.size, n)]
    if shape == "ceiling":
        return ceil
    if shape == "regions":
        ends = np.cumsum(rng.integers(lo, hi + 1, n // lo + 1))
        high = (np.searchsorted(ends, np.arange(n), side="right") + rng.integers(2)) % 2 == 0
    else:
        high = rng.random(n) < {"mix50": 0.5, "mix97": 0.97}[shape]
    return np.where(high, ceil, top).astype(np.uint8)


def stream_sizes(offs):
    """the exact length of every chunk stream of a directory (a stream ends where the next one's 16-byte padding starts)"""
    o = np.asarray(offs).astype(np.int64)
    return np.append(o[1:-1] & ~15, o[-1]) - o[:-1]


def check_ceiling_premise(coder, sb, chunk, n, offs):
    """ceiling streams really are at the rate the buffers are sized for"""
    sizes = stream_sizes(offs)
    full, tail = sizes[:n // chunk], n % chunk
    header = 256 if coder == RANS64 else 128
    assert full.size, "no full chunk"
    assert full.min() >= sb * chunk // 8 - header, "streams below the model's ceiling rate"
    if coder in (BYTE, ALIAS) and sb == 16:            # two bytes per lane every step
        assert (full == 2 * chunk + 128).all()
        assert not tail or sizes[-1] == 2 * tail + 128
    if coder == RANS64 and sb == 16 and chunk % 64 == 0:   # one u32 per lane every two steps
        assert (full == 2 * chunk + 256).all()
    if coder == WORD and chunk == 4096:                 # a pending stream and the current one exceed K2r's ring
        assert 2 * full.min() > RING_BYTES
    if coder == WORD and chunk == 8192:                 # every stream alone exceeds the ring: K2r spills each one
        assert (full > RING_BYTES).all()


def _ragged_n(chunk, i):
    """about 1 Mi symbols (8192 chunks of 32: the oracle's alias coder builds its tables once per chunk), never a
    multiple of the chunk; odd (so not a multiple of 32) for odd i"""
    return min(1 << 20, 8192 * chunk) + chunk // 2 + 32 * i + 17 * (i % 2)


def _dev(a, pad=0, fill=0):
    import torch
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    t = torch.full((a.size + pad,), fill, dtype=torch.uint8, device="cuda")
    if a.size:
        t[:a.size] = torch.from_numpy(a).cuda()
    return t


def device_round_trip(ctx, mdl, data, chunk, blob, offs):
    """encode_device / decode_device: the same container as the host call, and nothing written past n"""
    import torch
    n = data.size
    cap = ctx.encode_bound(n, chunk)
    d_in = _dev(data)
    d_blob = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_offs = torch.zeros(offs.size, dtype=torch.int64, device="cuda")
    ctx.encode_device(mdl, d_in.data_ptr(), n, chunk, d_blob.data_ptr(), cap, d_offs.data_ptr())
    ctx.sync()
    assert np.array_equal(d_offs.cpu().numpy().view(np.uint64), offs)
    assert np.array_equal(d_blob[:blob.size].cpu().numpy(), blob)
    d_out = torch.full((n + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.decode_device(mdl, d_blob.data_ptr(), blob.size, d_offs.data_ptr(), chunk, d_out.data_ptr(), n)
    ctx.sync()
    assert torch.equal(d_out[:n], d_in[:n])
    assert bool((d_out[n:] == SENTINEL).all())


def check_flat(ctx, oracle_lib, name, chunk, shapes=SHAPES, device=True):
    """encode_host / decode_host of every shape against the oracle; the ceiling also through device memory"""
    coder, sb, freqs, cum = model(name)
    mdl = ctx.model(coder, sb, freqs)
    for i, shape in enumerate(shapes):
        n = _ragged_n(chunk, i)
        data = rate_data(freqs, shape, n, seed=1000 * i + chunk + sb, hi=3 * chunk)
        blob, offs = ctx.encode_host(mdl, data, chunk)
        oblob, ooffs = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
        assert np.array_equal(offs, ooffs), (name, chunk, shape, "directory")
        assert np.array_equal(blob, oblob), (name, chunk, shape, "blob")
        assert np.array_equal(ctx.decode_host(mdl, blob, offs, n, chunk), data), (name, chunk, shape, "decode")
        if shape == "ceiling":
            check_ceiling_premise(coder, sb, chunk, n, offs)
            if device:
                device_round_trip(ctx, mdl, data, chunk, blob, offs)
        elif shape == "floor" and MODELS[name][2] != "ones":
            assert stream_sizes(offs).max() <= 256 + chunk // 8, (name, chunk)
    mdl.close()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's own code on these models
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(MODELS))
def test_oracle_matches_reference_at_the_ceiling(oracle_lib, ref_lib, name):
    coder, sb, freqs, cum = model(name)
    for shape in ("ceiling", "regions"):
        for nl in (1, 2, 32):
            n = 3 * 8192 + 4711 + nl
            data = rate_data(freqs, shape, n, seed=nl + sb, lo=1, hi=3000)
            so = oracle_lib.encode(coder, data, freqs, cum, nl, sb)
            sr = ref_lib.encode(coder, data, freqs, cum, nl, sb)
            assert np.array_equal(so, sr), (shape, nl, "oracle stream != reference stream")
            for lib in (oracle_lib, ref_lib):
                dec, used = lib.decode(coder, sr, n, freqs, cum, nl, sb)
                assert np.array_equal(dec, data) and used == sr.size, (shape, nl, lib.path)
        # the chunked container the GPU tests compare against: at the ceiling rate, and it decodes
        for chunk in (1000, 4096, 8192):
            n = 9 * chunk + chunk // 3 + 1
            data = rate_data(freqs, shape, n, seed=chunk, hi=3 * chunk)
            blob, offs = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
            if shape == "ceiling":
                check_ceiling_premise(coder, sb, chunk, n, offs)
            assert np.array_equal(oracle_lib.chunked_decode(coder, blob, offs, n, freqs, cum, chunk, nlanes=32, scale_bits=sb), data)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the flat calls
# ---------------------------------------------------------------------------------------------------------------------

CHUNKS = [32, 1000, 2048, 4096, 8192, 65536]        # split below 4096 symbols, fused (word: K2r to 8192, K2f above) from it
WORD_CHUNKS = [32, 1000, 2048, 4096, 8192, 16384, 65536]


def _flat_params():
    for name, (coder, _, _) in MODELS.items():
        for chunk in (WORD_CHUNKS if coder == WORD else CHUNKS):
            yield pytest.param(name, chunk, id=f"{name}-{chunk}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,chunk", list(_flat_params()))
def test_flat_matches_oracle(gpu_ctx, oracle_lib, name, chunk):
    check_flat(gpu_ctx, oracle_lib, name, chunk)


def forced_path_main():
    """RB200_ENCODE_PATH is read once per process, so the forced paths run here, in a child process."""
    import ryg_rans_b200 as rb
    path = os.environ["RB200_ENCODE_PATH"]
    ctx = rb.Context(0)
    oracle_lib = orc.Oracle()
    for name in ("word12-pair", "word12-dom", "word12-d2963", "word12-d2964"):
        for chunk in (4096, 8192):
            check_flat(ctx, oracle_lib, name, chunk)
    if path == "fused":                     # K2f where K2r is the default, over more chunks than it has worker warps
        check_slot_reuse(ctx, oracle_lib, "word12-dom", FUSED_WORD_WARPS)
    else:                                   # the split alias / byte encoders and the split per-block word encoder
        for name in ("byte16", "alias16", "byte16-pair"):
            check_flat(ctx, oracle_lib, name, 8192, shapes=("ceiling", "regions"))
        check_word_blocks(ctx, oracle_lib, 24, 65536, 8192)
    ctx.close()
    print("forced path ok")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fused", "split"])
def test_forced_encode_path(cuda_box, path):
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_rate_ceiling as t; t.forced_path_main()"
    env = dict(os.environ, RB200_ENCODE_PATH=path)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "forced path ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: slot reuse at the ceiling (data made on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def _gpu_rate_data(freqs, shape, n, chunk, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ones = torch.from_numpy(np.flatnonzero(freqs == 1).astype(np.uint8)).cuda()
    data = ones[torch.randint(0, ones.numel(), (n,), device="cuda", generator=g)]
    if shape == "regions":
        lens = torch.randint(32, 3 * chunk + 1, (n // (3 * chunk) * 2 + 64,), device="cuda", generator=g)
        ends = torch.cumsum(lens, 0)
        assert int(ends[-1]) >= n
        mark = torch.zeros(n, dtype=torch.uint8, device="cuda")
        mark[ends[ends < n]] = 1
        low = (torch.cumsum(mark, 0, dtype=torch.int32) & 1).bool()
        data[low] = int(np.argmax(freqs))
    return data


def check_slot_reuse(ctx, oracle_lib, name, warps_per_sm, chunk=4096):
    """Over more chunks than twice the encoder's worker warps, so every slot of a warp is reused: the ceiling and regions
    of ceiling and floor, through device memory, against the oracle."""
    import torch
    coder, sb, freqs, cum = model(name)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 32 * chunk + chunk // 2 + 7
    n_chunks = ctx.chunk_count(n, chunk)
    assert n_chunks > SLOTS_PER_WARP * sms * warps_per_sm
    mdl = ctx.model(coder, sb, freqs)
    cap = ctx.encode_bound(n, chunk)
    for shape in ("ceiling", "regions"):
        data = _gpu_rate_data(freqs, shape, n, chunk, seed=sb * 7 + len(shape))
        d_blob = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        d_offs = torch.zeros(n_chunks + 1, dtype=torch.int64, device="cuda")
        ctx.encode_device(mdl, data.data_ptr(), n, chunk, d_blob.data_ptr(), cap, d_offs.data_ptr())
        ctx.sync()
        h_data = data.cpu().numpy()
        offs = d_offs.cpu().numpy().view(np.uint64)
        oblob, ooffs = oracle_lib.chunked_encode(coder, h_data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
        assert np.array_equal(offs, ooffs), (name, shape, "directory")
        assert int(offs[-1]) == oblob.size and np.array_equal(d_blob[:oblob.size].cpu().numpy(), oblob), (name, shape, "blob")
        if shape == "ceiling":
            check_ceiling_premise(coder, sb, chunk, n, offs)
        del h_data, oblob
        d_out = torch.full((n + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
        ctx.decode_device(mdl, d_blob.data_ptr(), int(offs[-1]), d_offs.data_ptr(), chunk, d_out.data_ptr(), n)
        ctx.sync()
        assert torch.equal(d_out[:n], data) and bool((d_out[n:] == SENTINEL).all()), (name, shape, "decode")
        del data, d_blob, d_out
    mdl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,warps", [("word12-dom", RING_WARPS), ("byte16", FUSED_ALIAS_WARPS), ("alias16", FUSED_ALIAS_WARPS)],
                         ids=["K2r-word12", "fused-byte16", "fused-alias16"])
def test_slot_reuse_at_the_ceiling(gpu_ctx, oracle_lib, name, warps):
    check_slot_reuse(gpu_ctx, oracle_lib, name, warps)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: bounds, capacities and a blob one vector short
# ---------------------------------------------------------------------------------------------------------------------

BOUND_CASES = [("word12-dom", 8192, "K2r"), ("word12-d2964", 16384, "K2f"), ("word12-pair", 2048, "word-split"),
               ("byte16", 4096, "byte-fused"), ("alias16", 8192, "alias-fused"), ("byte16-pair", 2048, "byte-split"),
               ("alias16", 1000, "alias-split"), ("rans64-16", 4096, "rans64")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,chunk,path", BOUND_CASES, ids=[c[2] for c in BOUND_CASES])
def test_bounds_at_the_ceiling(gpu_ctx, oracle_lib, name, chunk, path):
    import torch
    import ryg_rans_b200 as rb
    coder, sb, freqs, cum = model(name)
    n = 64 * chunk + chunk // 2 + 5
    data = rate_data(freqs, "ceiling", n, seed=chunk + 3)
    mdl = gpu_ctx.model(coder, sb, freqs)
    blob, offs = gpu_ctx.encode_host(mdl, data, chunk)
    oblob, ooffs = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    check_ceiling_premise(coder, sb, chunk, n, offs)
    assert blob.size <= gpu_ctx.encode_bound(n, chunk)
    cont = gpu_ctx.container_encode_host(mdl, data, chunk)
    assert cont.size <= gpu_ctx.container_capacity(n, chunk)
    # a blob of exactly the container's size is enough
    b2, o2 = gpu_ctx.encode_host(mdl, data, chunk, blob_cap=blob.size)
    assert np.array_equal(o2, offs) and np.array_equal(b2, blob)
    # one vector less is RB200_E_SPACE, and nothing is written past the cap
    cap = blob.size - 16
    d_in = _dev(data)
    d_blob = torch.full((cap + 65536,), 0xAB, dtype=torch.uint8, device="cuda")
    d_offs = torch.zeros(offs.size, dtype=torch.int64, device="cuda")
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_device(mdl, d_in.data_ptr(), n, chunk, d_blob.data_ptr(), cap, d_offs.data_ptr())
        gpu_ctx.sync()
    assert ei.value.code == E_SPACE
    assert bool((d_blob[cap:] == 0xAB).all())
    # the context encodes again afterwards
    b3, o3 = gpu_ctx.encode_host(mdl, data, chunk)
    assert np.array_equal(o3, offs) and np.array_equal(b3, blob)
    mdl.close()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: single-model containers (version 1); the async decode runs C3's planned decoders
# ---------------------------------------------------------------------------------------------------------------------

V1_MODELS = ["word12-dom", "word12-d2964", "alias16", "alias14", "alias12", "alias10", "byte16", "byte14", "byte12", "byte8",
             "byte16-pair", "rans64-8", "rans64-14", "rans64-16"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", V1_MODELS)
def test_container_at_the_ceiling(gpu_ctx, oracle_lib, name):
    import torch
    from ryg_rans_b200 import api
    coder, sb, freqs, cum = model(name)
    mdl = gpu_ctx.model(coder, sb, freqs)
    for chunk, shape in ((8192, "ceiling"), (4096, "regions"), (65536, "ceiling"), (2048, "mix97")):
        n = 2 * (1 << 20) + chunk // 3 + 1
        data = rate_data(freqs, shape, n, seed=chunk + sb, hi=3 * chunk)
        oblob, ooffs = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
        if shape == "ceiling":
            check_ceiling_premise(coder, sb, chunk, n, ooffs)
        want = api.container_pack(coder, sb, chunk, n, freqs, ooffs, oblob, CRC_BLOB)
        cont = gpu_ctx.container_encode_host(mdl, data, chunk, flags=CRC_BLOB)
        assert cont.size == want.size and np.array_equal(cont, want), (chunk, shape)
        assert np.array_equal(gpu_ctx.container_decode_host(want), data), (chunk, shape)
        d_buf = _dev(want)
        d_out = torch.full((n + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        gpu_ctx.container_decode_async(d_buf.data_ptr(), want.size, d_out.data_ptr(), n, d_n.data_ptr())
        gpu_ctx.sync()
        assert int(d_n.item()) == n
        assert np.array_equal(d_out[:n].cpu().numpy(), data), (chunk, shape)
        assert bool((d_out[n:] == SENTINEL).all())
    mdl.close()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: per-block models, version 2 (word) and version 3 (byte, rans64)
# ---------------------------------------------------------------------------------------------------------------------

def _block_shape(b):
    """ceiling and floor blocks alternate; every fifth block holds regions"""
    return "regions" if b % 5 == 4 else ("ceiling", "floor")[b % 2]


def _oracle_blocks(oracle_lib, coder, sb, data, block_freqs, bs, ch):
    """every block its own oracle container, concatenated with its directory rebased"""
    parts, offs, base = [], [], 0
    for b, f in enumerate(block_freqs):
        f = f.astype(np.uint32)
        cum = np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)
        ob, oo = oracle_lib.chunked_encode(coder, data[b * bs:(b + 1) * bs], f, cum, ch, nlanes=32, scale_bits=sb)
        parts.append(ob)
        offs.append(oo[:-1] + np.uint64(base))
        base += ob.size
    return np.concatenate(offs + [np.array([base], np.uint64)]), np.concatenate(parts)


def _blocks_case(models, nb, bs, ch, seed):
    """block b: the frequencies models[b % len] with its symbols rotated by 37 b, and _block_shape(b) data"""
    freqs, data = [], []
    for b in range(nb):
        f = np.roll(models[b % len(models)], 37 * b)
        freqs.append(f.astype(np.uint16))
        data.append(rate_data(f, _block_shape(b), bs, seed=seed + b, hi=3 * ch))
    return np.stack(freqs), np.concatenate(data)


def _check_blocks_decode_async(ctx, fn, cont, data):
    import torch
    n = data.size
    d_buf = _dev(cont)
    d_out = torch.full((n + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    fn(d_buf.data_ptr(), cont.size, d_out.data_ptr(), n, d_n.data_ptr())
    ctx.sync()
    assert int(d_n.item()) == n
    assert np.array_equal(d_out[:n].cpu().numpy(), data)
    assert bool((d_out[n:] == SENTINEL).all())


def check_word_blocks(ctx, oracle_lib, nb, bs, ch):
    from ryg_rans_b200 import api
    word_models = [model(name)[2] for name in ("word12-pair", "word12-dom", "word12-d2963", "word12-d2964")]
    freqs, data = _blocks_case(word_models, nb, bs, ch, seed=ch)
    want_o, want_b = _oracle_blocks(oracle_lib, WORD, 12, data, freqs, bs, ch)
    blob, offs = ctx.blocks_encode_host(data, nb, bs, freqs, ch)
    assert np.array_equal(offs, want_o) and np.array_equal(blob, want_b)
    per = bs // ch
    ceil = stream_sizes(offs)[:per]                       # block 0 is a ceiling block
    assert ceil.min() >= 3 * ch // 2
    assert np.array_equal(ctx.blocks_decode_host(want_b, want_o, freqs, nb, bs, ch), data)
    cont = api.container_blocks_pack(nb, bs, ch, freqs, want_o, want_b, CRC_BLOB)
    assert np.array_equal(ctx.container_blocks_encode_host(data, nb, bs, ch, freqs, CRC_BLOB), cont)
    assert np.array_equal(ctx.container_blocks_decode_host(cont), data)
    _check_blocks_decode_async(ctx, ctx.container_blocks_decode_async, cont, data)


@pytest.mark.gpu
@pytest.mark.parametrize("nb,bs,ch", [(24, 65536, 8192), (10, 65536, 2048), (9, 17 * 1024, 1024)], ids=["K5f", "K5-32", "K5-17"])
def test_word_blocks_at_the_ceiling(gpu_ctx, oracle_lib, nb, bs, ch):
    check_word_blocks(gpu_ctx, oracle_lib, nb, bs, ch)


@pytest.mark.gpu
@pytest.mark.parametrize("nb,bs,ch", [(12, 65536, 8192), (9, 17 * 1024, 1024)], ids=["8-per-block", "17-per-block"])
@pytest.mark.parametrize("sb", [8, 12, 15])
@pytest.mark.parametrize("coder", [BYTE, RANS64], ids=["byte", "rans64"])
def test_coder_blocks_at_the_ceiling(gpu_ctx, oracle_lib, coder, sb, nb, bs, ch):
    from ryg_rans_b200 import api
    freqs, data = _blocks_case([_freqs(sb, "ones" if sb == 8 else "dom")], nb, bs, ch, seed=sb + ch)
    want_o, want_b = _oracle_blocks(oracle_lib, coder, sb, data, freqs, bs, ch)
    blob, offs = gpu_ctx.blocks_coder_encode_host(coder, sb, data, nb, bs, freqs, ch)
    assert np.array_equal(offs, want_o) and np.array_equal(blob, want_b)
    per = bs // ch
    assert stream_sizes(offs)[:per].min() >= sb * ch // 8 - 256     # block 0 is a ceiling block
    assert np.array_equal(gpu_ctx.blocks_coder_decode_host(coder, sb, want_b, want_o, freqs, nb, bs, ch), data)
    cont = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, want_o, want_b, CRC_BLOB)
    assert np.array_equal(gpu_ctx.container_blocks_coder_encode_host(coder, sb, data, nb, bs, ch, freqs, CRC_BLOB), cont)
    assert np.array_equal(gpu_ctx.container_blocks_coder_decode_host(cont), data)
    _check_blocks_decode_async(gpu_ctx, gpu_ctx.container_blocks_coder_decode_async, cont, data)
