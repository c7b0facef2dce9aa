"""Per-block models for the byte and rans64 coders on the GPU: every model the kernels build equals the oracle's
normalize_freqs(count_freqs(block), 1 << scale_bits), the blob and directory equal the oracle's per-block chunked
encodes concatenated, decode of the oracle's streams and of the GPU's own returns the data in both memory kinds, the
error codes, and the version 3 container against rb200_container_blocks_coder_pack."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks_coder as cc  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST, DEVICE = 0, 1
CRC_BLOB = 1
OCODER = {rb.CODER_BYTE: orc.CODER_BYTE, rb.CODER_RANS64: orc.CODER_RANS64}
# the geometries of the word coder's per-block test: 32 chunks per block, 17 chunks per block, chunk == block
GEOMETRIES = [(13, 65536, 8192), (7, 4096, 4096), (6, 16384, 2048), (12, 65536, 65536), (5, 65536, 2048), (5, 17 * 1024, 1024)]


def _block_data(gen, n_blocks, block_size):
    kinds = ["zipf", "uniform", "text", "two", "skew", "const"]
    return np.concatenate([gen(kinds[b % len(kinds)], block_size, seed=1000 + b) for b in range(n_blocks)])


def _dev(a, pad=16):
    import torch
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    t = torch.zeros(a.size + pad, dtype=torch.uint8, device="cuda")
    if a.size:
        t[:a.size] = torch.from_numpy(a)
    return t


def _oracle(oracle_lib, coder, sb, data, nb, bs, ch):
    return cc.oracle_blocks_encode(oracle_lib, OCODER[coder], sb, data, nb, bs, ch)


def _device_encode(ctx, coder, sb, data, nb, bs, ch, freqs=None):
    """DEVICE-mode model_encode (freqs None) or encode: (blob, offsets, block_freqs) on the host"""
    import torch
    cap = ctx.encode_bound(data.size, ch)
    d_in = _dev(data)
    d_freqs = _dev(np.zeros((nb, 256), np.uint16) if freqs is None else np.ascontiguousarray(freqs, np.uint16))
    d_blob = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros((nb * (bs // ch) + 1) * 8, dtype=torch.uint8, device="cuda")
    fn = ctx.blocks_coder_model_encode_device if freqs is None else ctx.blocks_coder_encode_device
    fn(coder, sb, d_in.data_ptr(), nb, bs, d_freqs.data_ptr(), ch, d_blob.data_ptr(), cap, d_off.data_ptr())
    ctx.sync()
    offs = d_off.cpu().numpy().view(np.uint64)
    return d_blob[:int(offs[-1])].cpu().numpy(), offs, d_freqs[:nb * 512].cpu().numpy().view(np.uint16).reshape(nb, 256)


def _device_decode(ctx, coder, sb, blob, offs, freqs, nb, bs, ch):
    import torch
    d_blob, d_off, d_freqs = _dev(blob), _dev(offs), _dev(np.ascontiguousarray(freqs, np.uint16))
    d_out = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
    ctx.blocks_coder_decode_device(coder, sb, d_blob.data_ptr(), blob.size, d_off.data_ptr(), d_freqs.data_ptr(), nb, bs, ch,
                                   d_out.data_ptr())
    ctx.sync()
    return d_out.cpu().numpy()


@pytest.mark.parametrize("n_blocks,block_size,chunk", GEOMETRIES)
@pytest.mark.parametrize("sb", [8, 12, 14, 15])
@pytest.mark.parametrize("coder", [rb.CODER_BYTE, rb.CODER_RANS64])
def test_block_coder_models_streams_and_roundtrip(gpu_ctx, oracle_lib, gen, coder, sb, n_blocks, block_size, chunk):
    nb, bs, ch = n_blocks, block_size, chunk
    data = _block_data(gen, nb, bs)
    want_f, want_o, want_b = _oracle(oracle_lib, coder, sb, data, nb, bs, ch)
    blob, offs, freqs = gpu_ctx.blocks_coder_model_encode_host(coder, sb, data, nb, bs, ch)
    assert np.array_equal(freqs, want_f)
    assert np.array_equal(offs, want_o) and np.array_equal(blob, want_b)
    blob2, offs2 = gpu_ctx.blocks_coder_encode_host(coder, sb, data, nb, bs, freqs, ch)
    assert np.array_equal(offs2, want_o) and np.array_equal(blob2, want_b)
    for f in (None, want_f):
        b3, o3, f3 = _device_encode(gpu_ctx, coder, sb, data, nb, bs, ch, f)
        assert np.array_equal(f3, want_f) and np.array_equal(o3, want_o) and np.array_equal(b3, want_b), f is None
    assert np.array_equal(gpu_ctx.blocks_coder_decode_host(coder, sb, want_b, want_o, want_f, nb, bs, ch), data)
    assert np.array_equal(_device_decode(gpu_ctx, coder, sb, want_b, want_o, want_f, nb, bs, ch), data)


@pytest.mark.parametrize("coder,sb", [(rb.CODER_BYTE, 14), (rb.CODER_RANS64, 14), (rb.CODER_BYTE, 11)])
def test_block_coder_errors(gpu_ctx, oracle_lib, gen, coder, sb):
    nb, bs, ch = 4, 16384, 4096
    data = _block_data(gen, nb, bs)
    freqs, offs, blob = _oracle(oracle_lib, coder, sb, data, nb, bs, ch)
    lib = gpu_ctx.lib.dll

    def code(fn, *a):
        with pytest.raises(rb.RansError) as ei:
            fn(*a)
        return ei.value.code

    # a caller table that does not sum: -2 from the HOST call, -7 from sync in DEVICE mode
    bad = freqs.copy()
    bad[1][int(np.flatnonzero(bad[1])[0])] += 1
    assert code(gpu_ctx.blocks_coder_encode_host, coder, sb, data, nb, bs, bad, ch) == -2
    assert code(_device_encode, gpu_ctx, coder, sb, data, nb, bs, ch, bad) == -7
    # a symbol outside its block's model (block 0 coded with block 3's table, which lacks some of its symbols): -7
    other = freqs.copy()
    other[0] = freqs[3]                                                  # block 3 holds two symbols, block 0 many
    assert (other[0][np.unique(data[:bs])] == 0).any()
    assert code(gpu_ctx.blocks_coder_encode_host, coder, sb, data, nb, bs, other, ch) == -7
    assert code(_device_encode, gpu_ctx, coder, sb, data, nb, bs, ch, other) == -7
    # a decode table that does not sum, a corrupt stream: -4
    assert code(gpu_ctx.blocks_coder_decode_host, coder, sb, blob, offs, bad, nb, bs, ch) == -4
    assert code(_device_decode, gpu_ctx, coder, sb, blob, offs, bad, nb, bs, ch) == -4
    corrupt = blob.copy()
    corrupt[int(offs[5]) + 3] ^= 0x10                                  # lane 0's final state in chunk 5
    assert code(gpu_ctx.blocks_coder_decode_host, coder, sb, corrupt, offs, freqs, nb, bs, ch) == -4
    assert code(_device_decode, gpu_ctx, coder, sb, corrupt, offs, freqs, nb, bs, ch) == -4
    assert np.array_equal(gpu_ctx.blocks_coder_decode_host(coder, sb, blob, offs, freqs, nb, bs, ch), data)   # the context recovers
    # argument errors: -1, nothing launched
    out = np.zeros(data.size, np.uint8)
    o = np.zeros(offs.size, np.uint64)
    b = np.zeros(blob.size + 4096, np.uint8)
    n0 = gpu_ctx.launches
    for c, s in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, sb), (4, sb), (-1, sb), (coder, 7), (coder, 16)):
        assert lib.rb200_blocks_coder_encode(gpu_ctx.h, c, s, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                             o.ctypes.data, None, HOST) == -1, (c, s)
        assert lib.rb200_blocks_coder_model_encode(gpu_ctx.h, c, s, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data,
                                                   b.size, o.ctypes.data, None, HOST) == -1, (c, s)
        assert lib.rb200_blocks_coder_decode(gpu_ctx.h, c, s, blob.ctypes.data, blob.size, offs.ctypes.data, freqs.ctypes.data, nb, bs,
                                             ch, out.ctypes.data, HOST) == -1, (c, s)
    for g_nb, g_bs, g_ch in ((0, bs, ch), (nb, bs, 3000), (nb, 33 * 512, 512), (nb, bs, 16), (nb, 0, ch)):
        assert lib.rb200_blocks_coder_encode(gpu_ctx.h, coder, sb, data.ctypes.data, g_nb, g_bs, freqs.ctypes.data, g_ch, b.ctypes.data,
                                             b.size, o.ctypes.data, None, HOST) == -1, (g_nb, g_bs, g_ch)
    assert lib.rb200_blocks_coder_encode(gpu_ctx.h, coder, sb, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                         o.ctypes.data, None, 2) == -1
    assert lib.rb200_blocks_coder_encode(gpu_ctx.h, coder, sb, None, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                         o.ctypes.data, None, HOST) == -1
    assert lib.rb200_blocks_coder_encode(gpu_ctx.h, coder, sb, data.ctypes.data, nb, bs, None, ch, b.ctypes.data, b.size,
                                         o.ctypes.data, None, HOST) == -1
    assert lib.rb200_blocks_coder_decode(gpu_ctx.h, coder, sb, blob.ctypes.data, blob.size, offs.ctypes.data, None, nb, bs, ch,
                                         out.ctypes.data, HOST) == -1
    # 2^31 chunks: 2^26 blocks of 32 chunks
    assert lib.rb200_blocks_coder_model_encode(gpu_ctx.h, coder, sb, data.ctypes.data, 1 << 26, 1024, freqs.ctypes.data, 32,
                                               b.ctypes.data, b.size, o.ctypes.data, None, DEVICE) == -1
    assert gpu_ctx.launches == n0


def _container_cases(gen):
    for coder, sb in ((rb.CODER_BYTE, 14), (rb.CODER_RANS64, 15), (rb.CODER_BYTE, 8), (rb.CODER_RANS64, 12)):
        for nb, bs, ch in ((3, 65536, 8192), (5, 17 * 1024, 1024), (2, 4096, 4096)):
            yield coder, sb, nb, bs, ch, _block_data(gen, nb, bs)


def _container_device_encode(ctx, coder, sb, data, nb, bs, ch, flags, freqs=None):
    import torch
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_in = _dev(data)
    d_freqs = None if freqs is None else _dev(np.ascontiguousarray(freqs, np.uint16))
    d_out = torch.full((cap + 16,), 0xAA, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_coder_encode_device(coder, sb, d_in.data_ptr(), nb, bs, None if d_freqs is None else d_freqs.data_ptr(), ch, flags,
                                             d_out.data_ptr(), cap)
    ctx.sync()
    return d_out


def _container_decode(ctx, buf, mode, sentinel=0x5C):
    """rb200_container_blocks_coder_decode of host bytes `buf`: (rc, n_symbols, out, out_untouched)"""
    import torch
    fn = ctx.lib.dll.rb200_container_blocks_coder_decode
    n = C.c_uint64(0)
    cap = 1 << 20
    if mode == HOST:
        b = np.zeros(buf.size + 16, np.uint8)[:buf.size]
        b[:] = buf
        out = np.full(cap, sentinel, np.uint8)
        rc = fn(ctx.h, b.ctypes.data, buf.size, out.ctypes.data, cap, C.byref(n), HOST)
        return rc, n.value, out, True
    d_buf = _dev(buf)
    d_out = torch.full((cap,), sentinel, dtype=torch.uint8, device="cuda")
    rc = fn(ctx.h, d_buf.data_ptr(), buf.size, d_out.data_ptr(), cap, C.byref(n), DEVICE)
    out = d_out.cpu().numpy()
    return rc, n.value, out, bool((out == sentinel).all())


def test_block_coder_container_encode_equals_pack_and_decodes(gpu_ctx, oracle_lib, gen):
    for coder, sb, nb, bs, ch, data in _container_cases(gen):
        blob, offs, freqs = gpu_ctx.blocks_coder_model_encode_host(coder, sb, data, nb, bs, ch)
        for flags in (0, CRC_BLOB):
            want = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, offs, blob, flags)
            got = {"host, built": gpu_ctx.container_blocks_coder_encode_host(coder, sb, data, nb, bs, ch, None, flags),
                   "host, tables": gpu_ctx.container_blocks_coder_encode_host(coder, sb, data, nb, bs, ch, freqs, flags)}
            for name, f in (("device, built", None), ("device, tables", freqs)):
                got[name] = _container_device_encode(gpu_ctx, coder, sb, data, nb, bs, ch, flags, f)[:want.size].cpu().numpy()
            for name, g in got.items():
                assert g.size == want.size and np.array_equal(g, want), (coder, sb, nb, bs, ch, flags, name)
            # a container packed from the oracle's streams decodes in both memory kinds
            of, oo, ob = _oracle(oracle_lib, coder, sb, data, nb, bs, ch)
            obuf = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, of, oo, ob, flags)
            assert np.array_equal(obuf, want)
            for mode in (HOST, DEVICE):
                rc, n, out, _ = _container_decode(gpu_ctx, obuf, mode)
                assert rc == 0 and n == data.size and np.array_equal(out[:n], data), (coder, sb, mode)
            assert np.array_equal(gpu_ctx.container_blocks_coder_decode_host(obuf), data)


def test_block_coder_container_rejections(gpu_ctx, oracle_lib, gen):
    coder, sb, nb, bs, ch = rb.CODER_RANS64, 14, 3, 16384, 4096
    data = _block_data(gen, nb, bs)
    freqs, offs, blob = _oracle(oracle_lib, coder, sb, data, nb, bs, ch)
    good = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    v2like = good.copy()
    v2like[4] = 2                                                       # another version
    bad_model = good.copy()
    bad_model[64 + 512 + 7] ^= 0x01                                     # CRC mismatch in the model section
    bad_blob = good.copy()
    bad_blob[-5] ^= 0x01                                                # blob CRC mismatch
    for name, buf in (("version", v2like), ("model", bad_model), ("blob", bad_blob), ("truncated", good[:100].copy())):
        for mode in (HOST, DEVICE):
            rc, _, _, untouched = _container_decode(gpu_ctx, buf, mode)
            assert rc == -4, (name, mode)
            if mode == DEVICE:
                assert untouched, name
    # the version 1 and 2 decoders reject version 3, and the version 3 decoder theirs
    for fn in (gpu_ctx.lib.dll.rb200_container_decode, gpu_ctx.lib.dll.rb200_container_blocks_decode):
        n = C.c_uint64(0)
        out = np.zeros(data.size, np.uint8)
        assert fn(gpu_ctx.h, good.ctypes.data, good.size, out.ctypes.data, out.size, C.byref(n), HOST) == -4
    wblob, woffs, wfreqs = gpu_ctx.blocks_model_encode_host(data, nb, bs, ch)
    v2 = api.container_blocks_pack(nb, bs, ch, wfreqs, woffs, wblob, 0)
    assert _container_decode(gpu_ctx, v2, HOST)[0] == -4
    # encode: a bad caller table is -2 (HOST) and -7 from sync with the header unwritten (DEVICE); arguments -1
    bad = freqs.copy()
    bad[2][int(np.flatnonzero(bad[2])[0])] -= 1
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.container_blocks_coder_encode_host(coder, sb, data, nb, bs, ch, bad, 0)
    assert ei.value.code == -2
    with pytest.raises(rb.RansError) as ei:
        _container_device_encode(gpu_ctx, coder, sb, data, nb, bs, ch, 0, bad)
    assert ei.value.code == -7
    out = np.zeros(gpu_ctx.container_blocks_capacity(nb, bs, ch), np.uint8)
    for c, s in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 14), (coder, 7), (coder, 16)):
        assert gpu_ctx.lib.dll.rb200_container_blocks_coder_encode(gpu_ctx.h, c, s, data.ctypes.data, nb, bs, None, ch, 0, out.ctypes.data,
                                                                   out.size, None, HOST) == -1, (c, s)


_MULTI_SLICE = r'''
import sys, hashlib, numpy as np
sys.path.insert(0, %r)
import oracle, ryg_rans_b200 as rb
from ryg_rans_b200 import api
rng = np.random.default_rng(9)
orc = oracle.Oracle()
ctx = rb.Context(0)
n_blocks, bs, ch = 300, 65536, 8192
blocks = []
for b in range(n_blocks):
    p = 1.0 / np.arange(1, 257) ** (0.6 + 0.1 * (b %% 9))
    blocks.append(rng.permutation(256).astype(np.uint8)[rng.choice(256, bs, p=p / p.sum())])
data = np.concatenate(blocks)
digest = hashlib.sha256()
for coder, ocoder, sb in ((rb.CODER_BYTE, oracle.CODER_BYTE, 14), (rb.CODER_RANS64, oracle.CODER_RANS64, 15)):
    blob, offs, freqs = ctx.blocks_coder_model_encode_host(coder, sb, data, n_blocks, bs, ch)
    per = bs // ch
    for b in range(0, n_blocks, 37):
        f, c = orc.model(blocks[b], sb)
        assert np.array_equal(f.astype(np.uint16), freqs[b])
        ob, oo = orc.chunked_encode(ocoder, blocks[b], f, c, ch, scale_bits=sb)
        lo, hi = int(offs[b * per]) & ~15, int(offs[(b + 1) * per]) & ~15
        assert np.array_equal(blob[lo:hi], ob), b
    want = api.container_blocks_coder_pack(coder, sb, n_blocks, bs, ch, freqs, offs, blob, api.CONTAINER_CRC_BLOB)
    got = ctx.container_blocks_coder_encode_host(coder, sb, data, n_blocks, bs, ch, None, api.CONTAINER_CRC_BLOB)
    assert np.array_equal(got, want), coder
    digest.update(got.tobytes())
    assert np.array_equal(ctx.blocks_coder_decode_host(coder, sb, blob, offs, freqs, n_blocks, bs, ch), data)
    assert np.array_equal(ctx.container_blocks_coder_decode_host(got), data)
    # 1 MiB slices of 16 blocks ramp 2, 4, 8 blocks: the third slice holds blocks [6, 14); corrupt a blob byte there
    boff = 64 + 512 * n_blocks + 8 * offs.size
    boff += -boff %% 16
    pos = (int(offs[6 * per]) + int(offs[14 * per])) // 2
    bad = got.copy()
    bad[boff + pos] ^= 0x01
    try:
        ctx.container_blocks_coder_decode_host(bad)
        raise SystemExit("corruption not reported")
    except rb.RansError as e:
        assert e.code == -4, e.code
    assert np.array_equal(ctx.container_blocks_coder_decode_host(got), data)
print("digest", digest.hexdigest())
print("slices ok", ctx.launches)
''' % ROOT


def test_block_coder_host_multi_slice(cuda_box):
    """RB200_SLICE_MIB=1 and ~19 MiB of 64 KiB blocks: the host calls run many pipeline slices of whole blocks, each
    slice's blob CRC taken on the device and joined on the host; the containers equal pack's, sampled blocks equal the
    oracle's, and a corrupted blob byte in the third slice is -4."""
    env = dict(os.environ, RB200_SLICE_MIB="1")
    out = subprocess.run([sys.executable, "-c", _MULTI_SLICE], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "slices ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
