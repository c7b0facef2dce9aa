"""Per-block models for the alias coder on the GPU: every model the kernels build equals the oracle's
normalize_freqs(count_freqs(block), 1 << scale_bits), the blob and directory equal the oracle's per-block alias
chunked encodes concatenated (the per-block alias tables are built by the CTAs), decode of the oracle's streams returns
the data in both memory kinds, the error codes, and the version 4 container against rb200_container_blocks_alias_pack."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks_coder as cc  # noqa: E402
import test_gpu_blocks_coder as gc  # noqa: E402

pytestmark = pytest.mark.gpu

HOST, DEVICE = 0, 1
CRC_BLOB = 1


def _block_data(gen, n_blocks, block_size):
    """Zipf, one symbol, two symbols, uniform, text, skewed, and a block whose counts fill every bucket exactly (every
    symbol block_size / 256 times: no pairing at all)"""
    rng = np.random.default_rng(block_size + n_blocks)
    blocks = []
    for b in range(n_blocks):
        k = b % 7
        if k == 6:
            blocks.append(rng.permutation(np.arange(block_size) % 256).astype(np.uint8))
        else:
            blocks.append(gen(["zipf", "const", "two", "uniform", "text", "skew"][k], block_size, seed=2000 + b))
    return np.concatenate(blocks)


def _oracle(oracle_lib, sb, data, nb, bs, ch):
    return cc.oracle_blocks_encode(oracle_lib, orc.CODER_ALIAS, sb, data, nb, bs, ch)


def _device_encode(ctx, sb, data, nb, bs, ch, freqs=None):
    """DEVICE-mode model_encode (freqs None) or encode: (blob, offsets, block_freqs) on the host"""
    import torch
    cap = ctx.encode_bound(data.size, ch)
    d_in = gc._dev(data)
    d_freqs = gc._dev(np.zeros((nb, 256), np.uint16) if freqs is None else np.ascontiguousarray(freqs, np.uint16))
    d_blob = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros((nb * (bs // ch) + 1) * 8, dtype=torch.uint8, device="cuda")
    fn = ctx.blocks_alias_model_encode_device if freqs is None else ctx.blocks_alias_encode_device
    fn(sb, d_in.data_ptr(), nb, bs, d_freqs.data_ptr(), ch, d_blob.data_ptr(), cap, d_off.data_ptr())
    ctx.sync()
    offs = d_off.cpu().numpy().view(np.uint64)
    return d_blob[:int(offs[-1])].cpu().numpy(), offs, d_freqs[:nb * 512].cpu().numpy().view(np.uint16).reshape(nb, 256)


def _device_decode(ctx, sb, blob, offs, freqs, nb, bs, ch):
    import torch
    d_blob, d_off, d_freqs = gc._dev(blob), gc._dev(offs), gc._dev(np.ascontiguousarray(freqs, np.uint16))
    d_out = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
    ctx.blocks_alias_decode_device(sb, d_blob.data_ptr(), blob.size, d_off.data_ptr(), d_freqs.data_ptr(), nb, bs, ch, d_out.data_ptr())
    ctx.sync()
    return d_out.cpu().numpy()


@pytest.mark.parametrize("n_blocks,block_size,chunk", gc.GEOMETRIES)
@pytest.mark.parametrize("sb", [8, 12, 14, 15])
def test_block_alias_models_streams_and_roundtrip(gpu_ctx, oracle_lib, gen, sb, n_blocks, block_size, chunk):
    nb, bs, ch = n_blocks, block_size, chunk
    data = _block_data(gen, nb, bs)
    want_f, want_o, want_b = _oracle(oracle_lib, sb, data, nb, bs, ch)
    blob, offs, freqs = gpu_ctx.blocks_alias_model_encode_host(sb, data, nb, bs, ch)
    assert np.array_equal(freqs, want_f)
    assert np.array_equal(offs, want_o) and np.array_equal(blob, want_b)
    blob2, offs2 = gpu_ctx.blocks_alias_encode_host(sb, data, nb, bs, freqs, ch)
    assert np.array_equal(offs2, want_o) and np.array_equal(blob2, want_b)
    for f in (None, want_f):
        b3, o3, f3 = _device_encode(gpu_ctx, sb, data, nb, bs, ch, f)
        assert np.array_equal(f3, want_f) and np.array_equal(o3, want_o) and np.array_equal(b3, want_b), f is None
    assert np.array_equal(gpu_ctx.blocks_alias_decode_host(sb, want_b, want_o, want_f, nb, bs, ch), data)
    assert np.array_equal(_device_decode(gpu_ctx, sb, want_b, want_o, want_f, nb, bs, ch), data)


@pytest.mark.parametrize("sb", [14, 11])
def test_block_alias_errors(gpu_ctx, oracle_lib, gen, sb):
    nb, bs, ch = 4, 16384, 4096
    data = _block_data(gen, nb, bs)
    freqs, offs, blob = _oracle(oracle_lib, sb, data, nb, bs, ch)
    lib = gpu_ctx.lib.dll

    def code(fn, *a):
        with pytest.raises(rb.RansError) as ei:
            fn(*a)
        return ei.value.code

    # a caller table that does not sum: -2 from the HOST call, -7 from sync in DEVICE mode
    bad = freqs.copy()
    bad[0][int(np.flatnonzero(bad[0])[0])] += 1
    assert code(gpu_ctx.blocks_alias_encode_host, sb, data, nb, bs, bad, ch) == -2
    assert code(_device_encode, gpu_ctx, sb, data, nb, bs, ch, bad) == -7
    # a symbol outside its block's model (block 0 coded with block 1's one-symbol table): -7
    other = freqs.copy()
    other[0] = freqs[1]
    assert (other[0][np.unique(data[:bs])] == 0).any()
    assert code(gpu_ctx.blocks_alias_encode_host, sb, data, nb, bs, other, ch) == -7
    assert code(_device_encode, gpu_ctx, sb, data, nb, bs, ch, other) == -7
    # a decode table that does not sum, a corrupt stream: -4, then the context recovers
    assert code(gpu_ctx.blocks_alias_decode_host, sb, blob, offs, bad, nb, bs, ch) == -4
    assert code(_device_decode, gpu_ctx, sb, blob, offs, bad, nb, bs, ch) == -4
    corrupt = blob.copy()
    corrupt[int(offs[1]) + 3] ^= 0x10                                  # lane 0's final state in chunk 1
    assert code(gpu_ctx.blocks_alias_decode_host, sb, corrupt, offs, freqs, nb, bs, ch) == -4
    assert code(_device_decode, gpu_ctx, sb, corrupt, offs, freqs, nb, bs, ch) == -4
    assert np.array_equal(gpu_ctx.blocks_alias_decode_host(sb, blob, offs, freqs, nb, bs, ch), data)
    # argument errors: -1, nothing launched
    out = np.zeros(data.size, np.uint8)
    o = np.zeros(offs.size, np.uint64)
    b = np.zeros(blob.size + 4096, np.uint8)
    n0 = gpu_ctx.launches
    for s in (7, 16, 0):
        assert lib.rb200_blocks_alias_encode(gpu_ctx.h, s, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                             o.ctypes.data, None, HOST) == -1, s
        assert lib.rb200_blocks_alias_model_encode(gpu_ctx.h, s, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                                   o.ctypes.data, None, HOST) == -1, s
        assert lib.rb200_blocks_alias_decode(gpu_ctx.h, s, blob.ctypes.data, blob.size, offs.ctypes.data, freqs.ctypes.data, nb, bs, ch,
                                             out.ctypes.data, HOST) == -1, s
    for g_nb, g_bs, g_ch in ((0, bs, ch), (nb, bs, 3000), (nb, 33 * 512, 512), (nb, bs, 16), (nb, 0, ch)):
        assert lib.rb200_blocks_alias_encode(gpu_ctx.h, sb, data.ctypes.data, g_nb, g_bs, freqs.ctypes.data, g_ch, b.ctypes.data, b.size,
                                             o.ctypes.data, None, HOST) == -1, (g_nb, g_bs, g_ch)
        assert lib.rb200_blocks_alias_decode(gpu_ctx.h, sb, blob.ctypes.data, blob.size, offs.ctypes.data, freqs.ctypes.data, g_nb, g_bs,
                                             g_ch, out.ctypes.data, HOST) == -1, (g_nb, g_bs, g_ch)
    assert lib.rb200_blocks_alias_encode(gpu_ctx.h, sb, data.ctypes.data, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size,
                                         o.ctypes.data, None, 2) == -1
    assert lib.rb200_blocks_alias_decode(gpu_ctx.h, sb, blob.ctypes.data, blob.size, offs.ctypes.data, freqs.ctypes.data, nb, bs, ch,
                                         out.ctypes.data, 5) == -1
    assert lib.rb200_blocks_alias_encode(gpu_ctx.h, sb, None, nb, bs, freqs.ctypes.data, ch, b.ctypes.data, b.size, o.ctypes.data, None,
                                         HOST) == -1
    assert lib.rb200_blocks_alias_encode(gpu_ctx.h, sb, data.ctypes.data, nb, bs, None, ch, b.ctypes.data, b.size, o.ctypes.data, None,
                                         HOST) == -1
    assert lib.rb200_blocks_alias_decode(gpu_ctx.h, sb, blob.ctypes.data, blob.size, offs.ctypes.data, None, nb, bs, ch, out.ctypes.data,
                                         HOST) == -1
    assert lib.rb200_blocks_alias_model_encode(gpu_ctx.h, sb, data.ctypes.data, 1 << 26, 1024, freqs.ctypes.data, 32, b.ctypes.data,
                                               b.size, o.ctypes.data, None, DEVICE) == -1
    assert gpu_ctx.launches == n0


def _container_device_encode(ctx, sb, data, nb, bs, ch, flags, freqs=None):
    import torch
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_in = gc._dev(data)
    d_freqs = None if freqs is None else gc._dev(np.ascontiguousarray(freqs, np.uint16))
    d_out = torch.full((cap + 16,), 0xAA, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_alias_encode_device(sb, d_in.data_ptr(), nb, bs, None if d_freqs is None else d_freqs.data_ptr(), ch, flags,
                                             d_out.data_ptr(), cap)
    ctx.sync()
    return d_out


def _container_decode(ctx, buf, mode, sentinel=0x5C):
    """rb200_container_blocks_alias_decode of host bytes `buf`: (rc, n_symbols, out, out_untouched)"""
    import torch
    fn = ctx.lib.dll.rb200_container_blocks_alias_decode
    n = C.c_uint64(0)
    cap = 1 << 20
    if mode == HOST:
        b = np.zeros(buf.size + 16, np.uint8)[:buf.size]
        b[:] = buf
        out = np.full(cap, sentinel, np.uint8)
        rc = fn(ctx.h, b.ctypes.data, buf.size, out.ctypes.data, cap, C.byref(n), HOST)
        return rc, n.value, out, True
    d_buf = gc._dev(buf)
    d_out = torch.full((cap,), sentinel, dtype=torch.uint8, device="cuda")
    rc = fn(ctx.h, d_buf.data_ptr(), buf.size, d_out.data_ptr(), cap, C.byref(n), DEVICE)
    out = d_out.cpu().numpy()
    return rc, n.value, out, bool((out == sentinel).all())


def test_block_alias_container_encode_equals_pack_and_decodes(gpu_ctx, oracle_lib, gen):
    for sb in (14, 15, 8, 12):
        for nb, bs, ch in ((3, 65536, 8192), (7, 17 * 1024, 1024), (2, 4096, 4096)):
            data = _block_data(gen, nb, bs)
            of, oo, ob = _oracle(oracle_lib, sb, data, nb, bs, ch)
            for flags in (0, CRC_BLOB):
                want = api.container_blocks_alias_pack(sb, nb, bs, ch, of, oo, ob, flags)
                got = {"host, built": gpu_ctx.container_blocks_alias_encode_host(sb, data, nb, bs, ch, None, flags),
                       "host, tables": gpu_ctx.container_blocks_alias_encode_host(sb, data, nb, bs, ch, of, flags)}
                for name, f in (("device, built", None), ("device, tables", of)):
                    got[name] = _container_device_encode(gpu_ctx, sb, data, nb, bs, ch, flags, f)[:want.size].cpu().numpy()
                for name, g in got.items():
                    assert g.size == want.size and np.array_equal(g, want), (sb, nb, bs, ch, flags, name)
                for mode in (HOST, DEVICE):
                    rc, n, out, _ = _container_decode(gpu_ctx, want, mode)
                    assert rc == 0 and n == data.size and np.array_equal(out[:n], data), (sb, mode)
                assert np.array_equal(gpu_ctx.container_blocks_alias_decode_host(want), data)


def test_block_alias_container_rejections(gpu_ctx, oracle_lib, gen):
    sb, nb, bs, ch = 14, 3, 16384, 4096
    data = _block_data(gen, nb, bs)
    freqs, offs, blob = _oracle(oracle_lib, sb, data, nb, bs, ch)
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    v3like = good.copy()
    v3like[4] = 3                                                       # another version
    bad_model = good.copy()
    bad_model[64 + 512 + 7] ^= 0x01                                     # CRC mismatch in the model section
    bad_blob = good.copy()
    bad_blob[-5] ^= 0x01                                                # blob CRC mismatch
    for name, buf in (("version", v3like), ("model", bad_model), ("blob", bad_blob), ("truncated", good[:100].copy())):
        for mode in (HOST, DEVICE):
            rc, _, _, untouched = _container_decode(gpu_ctx, buf, mode)
            assert rc == -4, (name, mode)
            if mode == DEVICE:
                assert untouched, name
    # the version 1, 2 and 3 decoders reject version 4, and the version 4 decoder a version 3 container
    for fn in (gpu_ctx.lib.dll.rb200_container_decode, gpu_ctx.lib.dll.rb200_container_blocks_decode,
               gpu_ctx.lib.dll.rb200_container_blocks_coder_decode):
        n = C.c_uint64(0)
        out = np.zeros(data.size, np.uint8)
        assert fn(gpu_ctx.h, good.ctypes.data, good.size, out.ctypes.data, out.size, C.byref(n), HOST) == -4
    bblob, boffs, bfreqs = gpu_ctx.blocks_coder_model_encode_host(rb.CODER_BYTE, sb, data, nb, bs, ch)
    v3 = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, bfreqs, boffs, bblob, 0)
    assert _container_decode(gpu_ctx, v3, HOST)[0] == -4
    # encode: a bad caller table is -2 (HOST) and -7 from sync (DEVICE); arguments -1
    bad = freqs.copy()
    bad[2][int(np.flatnonzero(bad[2])[0])] -= 1
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.container_blocks_alias_encode_host(sb, data, nb, bs, ch, bad, 0)
    assert ei.value.code == -2
    with pytest.raises(rb.RansError) as ei:
        _container_device_encode(gpu_ctx, sb, data, nb, bs, ch, 0, bad)
    assert ei.value.code == -7
    out = np.zeros(gpu_ctx.container_blocks_capacity(nb, bs, ch), np.uint8)
    for s in (7, 16):
        assert gpu_ctx.lib.dll.rb200_container_blocks_alias_encode(gpu_ctx.h, s, data.ctypes.data, nb, bs, None, ch, 0, out.ctypes.data,
                                                                   out.size, None, HOST) == -1, s
