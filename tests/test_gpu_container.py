"""The container in host and device memory through the C-ABI: rb200_crc32 against zlib, rb200_container_encode
against rb200_container_pack of rb200_encode's output (byte for byte), rb200_container_decode of containers packed
from oracle encodes, and every rejection rb200_container_open makes, in both memory kinds."""
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORD, BYTE, ALIAS, RANS64 = 0, 1, 2, 3
CODERS = [(WORD, 12), (BYTE, 14), (BYTE, 8), (ALIAS, 16), (ALIAS, 12), (RANS64, 14)]
HOST, DEVICE = 0, 1


def _torch():
    import torch
    return torch


def _to_dev(a, pad=16):
    """a copy of host bytes in a fresh (256-byte aligned) device buffer, with `pad` spare bytes"""
    torch = _torch()
    t = torch.zeros(a.size + pad, dtype=torch.uint8, device="cuda")
    if a.size:
        t[:a.size] = torch.from_numpy(np.ascontiguousarray(a))
    return t


def _model_for(oracle_lib, gen, data, sb):
    src = data if data.size else gen("zipf", 1000, 3)
    return oracle_lib.model(src, sb)


def _reseal(buf):
    """Recompute the container's meta CRC (IEEE CRC-32 = zlib's) after editing header / model / directory fields, so
    that the semantic checks behind the checksum are what rejects the container."""
    n_chunks = struct.unpack_from("<Q", buf, 24)[0]
    hdr = bytearray(buf[:64].tobytes())
    hdr[44:52] = b"\0" * 8                                   # meta_crc, blob_crc
    end = 64 + 1024 + 8 * (n_chunks + 1)
    if end > buf.size:
        return buf
    crc = zlib.crc32(bytes(hdr) + buf[64:end].tobytes()) & 0xffffffff
    struct.pack_into("<I", buf, 44, crc)
    return buf


def _container_size(buf_head, lib):
    n_chunks, blob_bytes = struct.unpack_from("<QQ", buf_head, 24)
    return int(lib.dll.rb200_container_size(n_chunks, blob_bytes))


def _encode_device(ctx, model, data, chunk, flags, out_cap=None, fill=0xAA):
    torch = _torch()
    cap = ctx.container_capacity(data.size, chunk) if out_cap is None else out_cap
    d_in = _to_dev(data)
    d_out = torch.full((cap + 16,), fill, dtype=torch.uint8, device="cuda")
    ctx.container_encode_device(model, d_in.data_ptr(), data.size, chunk, flags, d_out.data_ptr(), cap)
    return d_out


def _decode(ctx, buf, mode, out_cap=None, sentinel=0x5C):
    """rb200_container_decode of host bytes `buf` in either memory kind: (rc, n_symbols, out, out_untouched)"""
    import ctypes as C
    torch = _torch()
    lib = ctx.lib
    n = C.c_uint64(0)
    cap = out_cap if out_cap is not None else 1 << 20
    if mode == HOST:
        b = np.zeros(buf.size + 16, np.uint8)[:buf.size]
        b[:] = buf
        out = np.full(max(cap, 16), sentinel, np.uint8)
        rc = lib.dll.rb200_container_decode(ctx.h, b.ctypes.data, buf.size, out.ctypes.data, cap, C.byref(n), HOST)
        return rc, n.value, out, True
    d_buf = _to_dev(buf)
    d_out = torch.full((max(cap, 16),), sentinel, dtype=torch.uint8, device="cuda")
    rc = lib.dll.rb200_container_decode(ctx.h, d_buf.data_ptr(), buf.size, d_out.data_ptr(), cap, C.byref(n), DEVICE)
    out = d_out.cpu().numpy()
    return rc, n.value, out, bool((out == sentinel).all())


# ---------------------------------------------------------------------------------------------------- rb200_crc32

def test_crc32_matches_zlib(gpu_ctx):
    torch = _torch()
    rng = np.random.default_rng(11)
    big = rng.integers(0, 256, 100 * (1 << 20) + 77, dtype=np.uint8)
    d_big = torch.from_numpy(big).cuda()
    lengths = list(range(0, 66)) + [4095, 4096, 4097, (1 << 20) + 13]
    for start in range(16):
        for n in lengths:
            want = zlib.crc32(big[start:start + n].tobytes())
            assert gpu_ctx.crc32_device(d_big.data_ptr() + start, n) == want, (start, n)
    for n in lengths + [big.size]:
        want = zlib.crc32(big[:n].tobytes())
        assert gpu_ctx.crc32(big[:n]) == want, n
        assert gpu_ctx.crc32_device(d_big.data_ptr(), n) == want, n
    # chained crc_in, zlib's rule: crc(a || b) = crc32(b, crc32(a))
    whole = zlib.crc32(big[:(8 << 20) + 5].tobytes())
    for _ in range(6):
        cuts = np.sort(rng.integers(0, (8 << 20) + 6, 3))
        edges = [0, *map(int, cuts), (8 << 20) + 5]
        c_dev = c_host = 0
        for lo, hi in zip(edges[:-1], edges[1:]):
            c_dev = gpu_ctx.crc32_device(d_big.data_ptr() + lo, hi - lo, c_dev)
            c_host = gpu_ctx.crc32(big[lo:hi], c_host)
        assert c_dev == whole and c_host == whole, edges
    assert gpu_ctx.crc32(big[:0], 0x12345678) == 0x12345678


def test_crc32_past_4gib(gpu_ctx):
    """A buffer of 2^32 + 17 bytes: the segment lengths and the x^(8 len) powers take 64-bit lengths."""
    torch = _torch()
    n = (1 << 32) + 17
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    d = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
    got = gpu_ctx.crc32_device(d.data_ptr(), n)
    got_tail = gpu_ctx.crc32_device(d.data_ptr() + 3, n - 3)
    h = d.cpu().numpy()
    del d
    want, step = 0, 1 << 28
    for lo in range(0, n, step):
        want = zlib.crc32(memoryview(h[lo:lo + step]), want)
    want_tail = zlib.crc32(memoryview(h[3:]))
    assert got == want and got_tail == want_tail


# ---------------------------------------------------------------------------------------------------- encode == pack

@pytest.mark.parametrize("coder,sb", CODERS)
def test_container_encode_equals_pack(gpu_ctx, oracle_lib, gen, coder, sb):
    from ryg_rans_b200 import api
    for n in (0, 1, 31, 4097, 100003, 300000):
        data = gen("zipf", n, seed=n + sb)
        freqs, cum = _model_for(oracle_lib, gen, data, sb)
        model = gpu_ctx.model(coder, sb, freqs)
        for chunk in (32, 4096, 16384):
            blob, offs = gpu_ctx.encode_host(model, data, chunk)
            for flags in (0, api.CONTAINER_CRC_BLOB):
                want = api.container_pack(coder, sb, chunk, n, freqs, offs, blob, flags)
                got_host = gpu_ctx.container_encode_host(model, data, chunk, flags)
                d_out = _encode_device(gpu_ctx, model, data, chunk, flags)
                gpu_ctx.sync()
                head = d_out[:64].cpu().numpy()
                got_dev = d_out[:_container_size(head, gpu_ctx.lib)].cpu().numpy()
                for got in (got_host, got_dev):
                    assert got.size == want.size and np.array_equal(got, want), (n, chunk, flags)
                    meta, f2, o2, b2 = api.container_open(got)
                    assert meta["n_symbols"] == n and meta["flags"] == flags
                    out = oracle_lib.chunked_decode(coder, b2, o2, n, f2, cum, chunk, nlanes=32, scale_bits=sb)
                    assert np.array_equal(out, data)
        model.close()


# ---------------------------------------------------------------------------------------------------- decode

@pytest.mark.parametrize("coder,sb", CODERS)
def test_container_decode_of_oracle_containers(gpu_ctx, oracle_lib, gen, coder, sb):
    from ryg_rans_b200 import api
    for n, chunk, kind in ((0, 4096, "zipf"), (1, 32, "zipf"), (4097, 32, "text"), (100003, 4096, "zipf"), (300000, 16384, "uniform")):
        data = gen(kind, n, seed=n + 1)
        freqs, cum = _model_for(oracle_lib, gen, data, sb)
        ob, oo = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
        for flags in (0, api.CONTAINER_CRC_BLOB):
            buf = api.container_pack(coder, sb, chunk, n, freqs, oo, ob, flags)
            assert np.array_equal(gpu_ctx.container_decode_host(buf), data)
            for mode in (HOST, DEVICE):
                rc, got_n, out, _ = _decode(gpu_ctx, buf, mode, out_cap=max(n, 1))
                assert rc == 0 and got_n == n and np.array_equal(out[:n], data), (n, chunk, flags, mode)


# ---------------------------------------------------------------------------------------------------- rejection

def test_container_decode_rejects_what_open_rejects(gpu_ctx, oracle_lib, gen):
    from ryg_rans_b200 import api
    data = gen("text", 20000, 6)
    freqs, cum = oracle_lib.model(data, 12)
    blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 4096)
    good = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob, api.CONTAINER_CRC_BLOB)
    plain = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob, 0)
    for mode in (HOST, DEVICE):
        rc, n, out, _ = _decode(gpu_ctx, good, mode)
        assert rc == 0 and n == data.size and np.array_equal(out[:n], data)

    def rejected(buf, mode, code=-4):
        rc, _, _, untouched = _decode(gpu_ctx, buf, mode)
        assert rc == code, (rc, mode)
        if mode == DEVICE:
            assert untouched, "device output written for a rejected container"

    bad_bufs = []
    for base in (good, plain):
        for pos in (5, 70, 64 + 1024 + 9):                       # header, model, directory
            bad = base.copy()
            bad[pos] ^= 0x40
            bad_bufs.append(bad)
    bad = good.copy()
    bad[-7] ^= 0x40                                              # the blob, under its CRC
    bad_bufs.append(bad)
    for cut in list(range(0, 64 + 1024 + 8 * offs.size + 16, 7)) + [good.size - 16, good.size - 1]:
        bad_bufs.append(good[:cut].copy())
    edits = {
        "magic": (0, "<I", 0x12345678), "version": (4, "<H", 2), "coder": (6, "<B", 9), "scale_bits": (7, "<B", 3),
        "lanes": (8, "<I", 64), "chunk_syms zero": (12, "<I", 0), "chunk_syms other": (12, "<I", 2048),
        "n_symbols huge": (16, "<Q", 2 ** 64 - 1), "n_symbols + 1 chunk": (16, "<Q", data.size + 4096),
        "n_chunks huge": (24, "<Q", 2 ** 40), "n_chunks 2^31": (24, "<Q", 2 ** 31), "blob_bytes odd": (32, "<Q", blob.size + 8),
        "blob_bytes beyond the buffer": (32, "<Q", blob.size + 4096), "blob_bytes short": (32, "<Q", blob.size - 16),
        "freqs do not sum to 1 << scale_bits": (64 + 4 * 65, "<I", 7), "word coder with scale_bits 14": (7, "<B", 14),
        "first stream starts beyond the first vector": (64 + 1024, "<Q", 32),
        "directory not monotone": (64 + 1024 + 8, "<Q", int(offs[2]) + 16),
        "last entry != blob size": (64 + 1024 + 8 * (offs.size - 1), "<Q", int(offs[-1]) - 16),
    }
    for name, (off, fmt, val) in edits.items():
        bad = plain.copy()
        struct.pack_into(fmt, bad, off, val)
        bad_bufs.append(_reseal(bad))
    for bad in bad_bufs:
        with pytest.raises(Exception):
            api.container_open(bad)                               # the host parser agrees
        for mode in (HOST, DEVICE):
            rejected(bad, mode)
    # out_cap < n: -3 with *n_symbols set, output untouched
    for mode in (HOST, DEVICE):
        rc, n, _, untouched = _decode(gpu_ctx, good, mode, out_cap=data.size - 1)
        assert rc == -3 and n == data.size and untouched
    # misaligned buffers: -1
    torch = _torch()
    import ctypes as C
    n = C.c_uint64(0)
    d_buf, d_out = _to_dev(good, 64), torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    lib = gpu_ctx.lib.dll
    for db, do in ((8, 0), (0, 8), (4, 0)):
        assert lib.rb200_container_decode(gpu_ctx.h, d_buf.data_ptr() + db, good.size, d_out.data_ptr() + do, data.size, C.byref(n),
                                          DEVICE) == -1
    h_buf = np.zeros(good.size + 64, np.uint8)
    h_out = np.zeros(data.size + 64, np.uint8)
    for hb, ho in ((4, 0), (0, 4)):
        assert lib.rb200_container_decode(gpu_ctx.h, h_buf.ctypes.data + hb, good.size, h_out.ctypes.data + ho, data.size, C.byref(n),
                                          HOST) == -1
    model = gpu_ctx.model(WORD, 12, freqs)
    d_in = _to_dev(data)
    cap = gpu_ctx.container_capacity(data.size, 4096)
    assert lib.rb200_container_encode(gpu_ctx.h, model.h, d_in.data_ptr(), data.size, 4096, 0, d_out.data_ptr() + 8, cap, None,
                                      DEVICE) == -1
    h_enc = np.zeros(cap + 16, np.uint8)
    assert lib.rb200_container_encode(gpu_ctx.h, model.h, data.ctypes.data, data.size, 4096, 0, h_enc.ctypes.data + 4, cap, None,
                                      HOST) == -1
    model.close()
    # and the context still decodes the intact container
    for mode in (HOST, DEVICE):
        rc, n, out, _ = _decode(gpu_ctx, good, mode)
        assert rc == 0 and np.array_equal(out[:n], data)


def test_container_device_encode_space_is_reported(gpu_ctx, oracle_lib, gen):
    from ryg_rans_b200 import api
    data = gen("zipf", 300000, 9)
    freqs, cum = oracle_lib.model(data, 12)
    model = gpu_ctx.model(WORD, 12, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, 4096)
    want = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob, api.CONTAINER_CRC_BLOB)
    _encode_device(gpu_ctx, model, data, 4096, api.CONTAINER_CRC_BLOB, out_cap=want.size - 16)
    with pytest.raises(Exception) as ei:
        gpu_ctx.sync()
    assert ei.value.code == -3
    with pytest.raises(Exception) as ei:
        gpu_ctx.container_encode_host(model, data, 4096, api.CONTAINER_CRC_BLOB, out_cap=want.size - 16)
    assert ei.value.code == -3
    d_out = _encode_device(gpu_ctx, model, data, 4096, api.CONTAINER_CRC_BLOB, out_cap=want.size)
    gpu_ctx.sync()
    assert np.array_equal(d_out[:want.size].cpu().numpy(), want)
    model.close()


# ---------------------------------------------------------------------------------------------------- host pipeline

def test_container_host_multi_slice(cuda_box):
    """RB200_SLICE_MIB=1 and 9 MB of input: the host calls run many pipeline slices, each slice's blob CRC taken on
    the device and joined on the host.  The containers equal pack's; a byte corrupted inside the third slice's blob
    range is reported as -4; the same context then decodes the intact container."""
    code = r'''
import sys, numpy as np, zlib
sys.path.insert(0, %r)
import oracle, ryg_rans_b200 as rb
from ryg_rans_b200 import api
rng = np.random.default_rng(5)
p = 1.0 / np.arange(1, 257) ** 1.1
data = rng.choice(256, 9_000_017, p=p / p.sum()).astype(np.uint8)
orc = oracle.Oracle()
ctx = rb.Context(0)
for coder, sb in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 16), (rb.CODER_RANS64, 14)):
    f, c = orc.model(data, sb)
    m = ctx.model(coder, sb, f)
    chunk = 8192
    ob, oo = orc.chunked_encode(coder, data, f, c, chunk, scale_bits=sb)
    want = api.container_pack(coder, sb, chunk, data.size, f, oo, ob, api.CONTAINER_CRC_BLOB)
    got = ctx.container_encode_host(m, data, chunk, api.CONTAINER_CRC_BLOB)
    assert np.array_equal(got, want), coder
    assert ctx.crc32(ob) == zlib.crc32(ob.tobytes())
    # 1 MiB slices of 128 chunks ramp 16, 32, 64 chunks: the third slice holds chunks [48, 112)
    boff = 64 + 1024 + 8 * oo.size + (-(64 + 1024 + 8 * oo.size) %% 16)
    # a byte only the CRC sees: the zero pad in front of a stream that starts inside its vector
    pads = [int(oo[k]) & ~15 for k in range(49, 112) if int(oo[k]) & 15]
    pos = pads[len(pads) // 2] if pads else (int(oo[48]) + int(oo[112])) // 2
    assert (int(oo[48]) & ~15) <= pos < (int(oo[112]) & ~15)
    bad = got.copy()
    bad[boff + pos] ^= 0x01
    try:
        ctx.container_decode_host(bad)
        raise SystemExit("corruption not reported")
    except rb.RansError as e:
        assert e.code == -4, e.code
    assert np.array_equal(ctx.container_decode_host(got), data)
    m.close()
print("slices ok", ctx.launches)
''' % ROOT
    env = dict(os.environ, RB200_SLICE_MIB="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "slices ok" in out.stdout, out.stderr[-2000:]
