"""The per-block container (version 2) in host and device memory through the C-ABI: rb200_container_blocks_encode
against rb200_container_blocks_pack of rb200_blocks_model_encode's output (byte for byte), rb200_container_blocks_decode
of containers packed from oracle encodes, every rejection rb200_container_blocks_open makes, in both memory kinds."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks as cb  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST, DEVICE = 0, 1
CRC_BLOB = 1


def _torch():
    import torch
    return torch


def _to_dev(a, pad=16):
    """a copy of host bytes in a fresh (256-byte aligned) device buffer, with `pad` spare bytes"""
    torch = _torch()
    a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    t = torch.zeros(a.size + pad, dtype=torch.uint8, device="cuda")
    if a.size:
        t[:a.size] = torch.from_numpy(a)
    return t


def _fallback_data():
    """blocks whose model has a symbol of frequency 2964 (the 32-bit reciprocal is not exact: the 33-bit fallback)"""
    rng = np.random.default_rng(11)
    blocks = []
    for f0 in (2964, 16):
        b = np.concatenate([np.full(f0 * 16, 7, np.uint8), np.full((4096 - f0) * 16, 9, np.uint8)])
        rng.shuffle(b)
        blocks.append(b)
    return np.concatenate(blocks)


def _cases():
    yield from cb.cases()
    yield 2, 65536, 8192, _fallback_data()


def _encode_device(ctx, data, nb, bs, ch, flags, freqs=None, out_cap=None, fill=0xAA):
    torch = _torch()
    cap = ctx.container_blocks_capacity(nb, bs, ch) if out_cap is None else out_cap
    d_in = _to_dev(data)
    d_freqs = None if freqs is None else _to_dev(np.ascontiguousarray(freqs, np.uint16))
    d_out = torch.full((cap + 16,), fill, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_encode_device(d_in.data_ptr(), nb, bs, None if d_freqs is None else d_freqs.data_ptr(), ch, flags,
                                       d_out.data_ptr(), cap)
    return d_out


def _decode(ctx, buf, mode, out_cap=None, sentinel=0x5C, v1=False):
    """rb200_container_blocks_decode (or, with v1, rb200_container_decode) of host bytes `buf` in either memory kind:
    (rc, n_symbols, out, out_untouched)"""
    torch = _torch()
    fn = ctx.lib.dll.rb200_container_decode if v1 else ctx.lib.dll.rb200_container_blocks_decode
    n = C.c_uint64(0)
    cap = out_cap if out_cap is not None else 1 << 20
    if mode == HOST:
        b = np.zeros(buf.size + 16, np.uint8)[:buf.size]
        b[:] = buf
        out = np.full(max(cap, 16), sentinel, np.uint8)
        rc = fn(ctx.h, b.ctypes.data, buf.size, out.ctypes.data, cap, C.byref(n), HOST)
        return rc, n.value, out, True
    d_buf = _to_dev(buf)
    d_out = torch.full((max(cap, 16),), sentinel, dtype=torch.uint8, device="cuda")
    rc = fn(ctx.h, d_buf.data_ptr(), buf.size, d_out.data_ptr(), cap, C.byref(n), DEVICE)
    out = d_out.cpu().numpy()
    return rc, n.value, out, bool((out == sentinel).all())


def test_blocks_container_encode_equals_pack(gpu_ctx, oracle_lib):
    from ryg_rans_b200 import api
    for nb, bs, ch, data in _cases():
        blob, offs, freqs = gpu_ctx.blocks_model_encode_host(data, nb, bs, ch)
        for flags in (0, CRC_BLOB):
            want = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
            got = {
                "host, built": gpu_ctx.container_blocks_encode_host(data, nb, bs, ch, None, flags),
                "host, tables": gpu_ctx.container_blocks_encode_host(data, nb, bs, ch, freqs, flags),
            }
            for name, f in (("device, built", None), ("device, tables", freqs)):
                d_out = _encode_device(gpu_ctx, data, nb, bs, ch, flags, f)
                gpu_ctx.sync()
                got[name] = d_out[:want.size].cpu().numpy()
            for name, g in got.items():
                assert g.size == want.size and np.array_equal(g, want), (nb, bs, ch, flags, name)
            meta, f2, o2, b2 = api.container_blocks_open(want)
            assert meta["n_symbols"] == data.size and meta["flags"] == flags
            assert np.array_equal(cb.oracle_decode_blocks(oracle_lib, meta, f2, o2, b2), data), (nb, bs, ch)


def test_blocks_container_decode_of_oracle_containers(gpu_ctx, oracle_lib):
    from ryg_rans_b200 import api
    for nb, bs, ch, data in _cases():
        freqs, offs, blob = cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
        for flags in (0, CRC_BLOB):
            buf = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
            assert np.array_equal(gpu_ctx.container_blocks_decode_host(buf), data)
            for mode in (HOST, DEVICE):
                rc, n, out, _ = _decode(gpu_ctx, buf, mode, out_cap=data.size)
                assert rc == 0 and n == data.size and np.array_equal(out[:n], data), (nb, bs, ch, flags, mode)


@pytest.fixture(scope="module")
def base(oracle_lib):
    nb, bs, ch = 3, 16384, 4096
    data = cb.block_data(nb, bs, 7)
    freqs, offs, blob = cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
    return data, (nb, bs, ch, freqs, offs, blob)


def test_blocks_container_decode_rejects_what_open_rejects(gpu_ctx, base):
    from ryg_rans_b200 import api
    data, geo = base
    nb, bs, ch, freqs, offs, blob = geo
    good = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    for mode in (HOST, DEVICE):
        rc, n, out, _ = _decode(gpu_ctx, good, mode)
        assert rc == 0 and n == data.size and np.array_equal(out[:n], data)
    for name, bad in cb.rejected_containers(*geo):
        for mode in (HOST, DEVICE):
            rc, _, _, untouched = _decode(gpu_ctx, bad, mode)
            assert rc == -4, (name, mode, rc)
            if mode == DEVICE:
                assert untouched, f"device output written for a rejected container ({name})"
    # out_cap < n: -3 with *n_symbols set, output untouched
    for mode in (HOST, DEVICE):
        rc, n, _, untouched = _decode(gpu_ctx, good, mode, out_cap=data.size - 1)
        assert rc == -3 and n == data.size and untouched
    # misaligned buffers: -1
    torch = _torch()
    lib = gpu_ctx.lib.dll
    n = C.c_uint64(0)
    d_buf, d_out = _to_dev(good, 64), torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    for db, do in ((8, 0), (0, 8), (4, 0)):
        assert lib.rb200_container_blocks_decode(gpu_ctx.h, d_buf.data_ptr() + db, good.size, d_out.data_ptr() + do, data.size,
                                                 C.byref(n), DEVICE) == -1
    h_buf = np.zeros(good.size + 64, np.uint8)
    h_out = np.zeros(data.size + 64, np.uint8)
    for hb, ho in ((4, 0), (0, 4)):
        assert lib.rb200_container_blocks_decode(gpu_ctx.h, h_buf.ctypes.data + hb, good.size, h_out.ctypes.data + ho, data.size,
                                                 C.byref(n), HOST) == -1
    cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
    d_in = _to_dev(data)
    d_enc = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    assert lib.rb200_container_blocks_encode(gpu_ctx.h, d_in.data_ptr(), nb, bs, None, ch, 0, d_enc.data_ptr() + 8, cap, None, DEVICE) == -1
    h_enc = np.zeros(cap + 16, np.uint8)
    assert lib.rb200_container_blocks_encode(gpu_ctx.h, data.ctypes.data, nb, bs, None, ch, 0, h_enc.ctypes.data + 4, cap, None, HOST) == -1
    # out_cap below header, model and directory: -3 from the call
    for mode, ptr in ((DEVICE, d_enc.data_ptr()), (HOST, h_enc.ctypes.data)):
        src = d_in.data_ptr() if mode == DEVICE else data.ctypes.data
        assert lib.rb200_container_blocks_encode(gpu_ctx.h, src, nb, bs, None, ch, 0, ptr, 64 + 512 * nb, None, mode) == -3
    # a caller table that does not sum to 4096: -2 from the call in HOST mode
    bad = freqs.copy()
    bad[1][int(np.flatnonzero(bad[1])[0])] -= 1
    with pytest.raises(Exception) as ei:
        gpu_ctx.container_blocks_encode_host(data, nb, bs, ch, bad, 0)
    assert ei.value.code == -2
    # and the context still decodes the intact container
    for mode in (HOST, DEVICE):
        rc, n, out, _ = _decode(gpu_ctx, good, mode)
        assert rc == 0 and np.array_equal(out[:n], data)


def test_blocks_container_device_encode_errors_leave_the_header_unwritten(gpu_ctx, base):
    from ryg_rans_b200 import api
    data, (nb, bs, ch, freqs, offs, blob) = base
    gblob, goffs, gfreqs = gpu_ctx.blocks_model_encode_host(data, nb, bs, ch)
    want = api.container_blocks_pack(nb, bs, ch, gfreqs, goffs, gblob, CRC_BLOB)
    d_out = _encode_device(gpu_ctx, data, nb, bs, ch, CRC_BLOB, out_cap=want.size - 16)
    with pytest.raises(Exception) as ei:
        gpu_ctx.sync()
    assert ei.value.code == -3
    assert (d_out[:64].cpu().numpy() == 0xAA).all()
    with pytest.raises(Exception) as ei:
        gpu_ctx.container_blocks_encode_host(data, nb, bs, ch, None, CRC_BLOB, out_cap=want.size - 16)
    assert ei.value.code == -3
    d_out = _encode_device(gpu_ctx, data, nb, bs, ch, CRC_BLOB, out_cap=want.size)
    gpu_ctx.sync()
    assert np.array_equal(d_out[:want.size].cpu().numpy(), want)
    # one caller table summing to 4095 on the device: the block encoder codes that block with an empty model (-7)
    bad = gfreqs.copy()
    bad[1][int(np.flatnonzero(bad[1])[0])] -= 1
    d_out = _encode_device(gpu_ctx, data, nb, bs, ch, 0, freqs=bad)
    with pytest.raises(Exception) as ei:
        gpu_ctx.sync()
    assert ei.value.code == -7
    assert (d_out[:64].cpu().numpy() == 0xAA).all()
    d_out = _encode_device(gpu_ctx, data, nb, bs, ch, 0, freqs=gfreqs)              # the context recovers
    gpu_ctx.sync()
    assert np.array_equal(d_out[:want.size].cpu().numpy(), api.container_blocks_pack(nb, bs, ch, gfreqs, goffs, gblob, 0))


def test_blocks_and_single_model_containers_reject_each_other_on_the_gpu(gpu_ctx, oracle_lib, gen, base):
    from ryg_rans_b200 import api
    import oracle as orc
    data, (nb, bs, ch, freqs, offs, blob) = base
    d1 = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(d1, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, d1, f, c, 4096)
    for flags in (0, CRC_BLOB):
        v1 = api.container_pack(0, 12, 4096, d1.size, f, oo, ob, flags)
        v2 = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
        for mode in (HOST, DEVICE):
            rc, _, _, untouched = _decode(gpu_ctx, v1, mode)
            assert rc == -4 and untouched, (flags, mode)
            rc, _, _, untouched = _decode(gpu_ctx, v2, mode, v1=True)
            assert rc == -4 and untouched, (flags, mode)
            assert _decode(gpu_ctx, v1, mode, v1=True)[0] == 0 and _decode(gpu_ctx, v2, mode)[0] == 0


_MULTI_SLICE = r'''
import sys, hashlib, numpy as np
sys.path.insert(0, %r)
import ryg_rans_b200 as rb
from ryg_rans_b200 import api
rng = np.random.default_rng(21)
nb, bs, ch = 528, 65536, 8192                       # 33 MiB: 1 MiB slices of 16 blocks, ramped 2, 4, 8 blocks
blocks = []
for b in range(nb):
    p = 1.0 / np.arange(1, 257) ** (0.6 + 0.1 * (b %% 9))
    blocks.append(rng.permutation(256).astype(np.uint8)[rng.choice(256, bs, p=p / p.sum())])
data = np.concatenate(blocks)
ctx = rb.Context(0)
blob, offs, freqs = ctx.blocks_model_encode_host(data, nb, bs, ch)
want = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, api.CONTAINER_CRC_BLOB)
got = ctx.container_blocks_encode_host(data, nb, bs, ch, None, api.CONTAINER_CRC_BLOB)
assert np.array_equal(got, want)
assert np.array_equal(ctx.container_blocks_encode_host(data, nb, bs, ch, freqs, api.CONTAINER_CRC_BLOB), want)
assert np.array_equal(ctx.container_blocks_decode_host(got), data)
# the third slice holds blocks [6, 14) = chunks [48, 112); a byte inside its blob range is seen by its slice's CRC
boff = api.container_blocks_open(got)[2].ctypes.data - got.ctypes.data
bad = got.copy()
pos = boff + ((int(offs[48]) & ~15) + (int(offs[112]) & ~15)) // 2
bad[pos] ^= 0x01
try:
    ctx.container_blocks_decode_host(bad)
    raise SystemExit("corruption not reported")
except rb.RansError as e:
    assert e.code == -4, e.code
assert np.array_equal(ctx.container_blocks_decode_host(got), data)
print("digest", hashlib.sha256(got.tobytes()).hexdigest())
print("slices ok", ctx.launches)
''' % ROOT


def test_blocks_container_host_multi_slice(cuda_box):
    """RB200_SLICE_MIB=1 and 33 MiB of 64 KiB blocks: the host calls run many pipeline slices, each slice's blob CRC
    taken on the device and joined on the host.  The containers equal pack's, a corrupted byte in the third slice's
    blob range is -4, and the fused and split encode paths give the identical container."""
    digests = []
    for path in ("fused", "split"):
        env = dict(os.environ, RB200_SLICE_MIB="1", RB200_ENCODE_PATH=path)
        out = subprocess.run([sys.executable, "-c", _MULTI_SLICE], env=env, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and "slices ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
        digests.append([ln for ln in out.stdout.splitlines() if ln.startswith("digest")][0])
    assert digests[0] == digests[1]
