"""rb200_container_blocks_decode_async: the per-block (version 2) container checked and decoded in device memory with
nothing done on the host.  Oracle containers of every geometry decode to the data and to rb200_container_blocks_decode's
output; an encode and a decode round-trip with one synchronisation; everything rb200_container_blocks_open rejects is -4
from rb200_sync with the output untouched; out_cap < n is -3; the call captured in a CUDA graph decodes containers of
different geometry and flags on replay."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks as cb  # noqa: E402
import test_gpu_container_blocks as gcb  # noqa: E402

pytestmark = pytest.mark.gpu

CRC_BLOB = 1
SENTINEL = 0x5C


def _torch():
    import torch
    return torch


def _async(ctx, d_buf, size, n, out_cap=None):
    """the async decode of d_buf[0, size) into a sentinel-filled buffer, then one rb200_sync: (rc, *d_n_symbols or -1, out)"""
    torch = _torch()
    cap = n if out_cap is None else out_cap
    d_out = torch.full((max(n, cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    ctx.container_blocks_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())
    rc = ctx.lib.dll.rb200_sync(ctx.h)
    return rc, int(d_n.item()), d_out


def _untouched(d_out):
    return bool((d_out == SENTINEL).all().item())


def _extra_cases():
    """1 chunk per block, with more blocks than the decoder's grid has CTAs; 32 chunks per block"""
    yield 4096, 4096, 4096, cb.block_data(4096, 4096, 31)
    yield 2, 65536, 2048, cb.block_data(2, 65536, 32)


@pytest.fixture(scope="module")
def base(oracle_lib):
    nb, bs, ch = 3, 16384, 4096
    data = cb.block_data(nb, bs, 7)
    return data, (nb, bs, ch, *cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch))


def test_async_decode_of_oracle_containers(gpu_ctx, oracle_lib):
    from ryg_rans_b200 import api
    for nb, bs, ch, data in list(gcb._cases()) + list(_extra_cases()):
        freqs, offs, blob = cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
        for flags in (0, CRC_BLOB):
            buf = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
            rc, n, d_out = _async(gpu_ctx, gcb._to_dev(buf), buf.size, data.size)
            assert rc == 0 and n == data.size, (nb, bs, ch, flags, rc, n)
            out = d_out[:n].cpu().numpy()
            assert np.array_equal(out, data), (nb, bs, ch, flags)
            assert _untouched(d_out[n:])
            rc, n2, sync_out, _ = gcb._decode(gpu_ctx, buf, gcb.DEVICE, out_cap=data.size)
            assert rc == 0 and n2 == n and np.array_equal(sync_out[:n], out)


def test_async_round_trip_without_host_sync(gpu_ctx):
    torch = _torch()
    for nb, bs, ch in ((8, 65536, 8192), (64, 4096, 1024), (2, 32768, 1024)):
        data = cb.block_data(nb, bs, 40 + nb)
        cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
        d_in = gcb._to_dev(data)
        for flags in (0, CRC_BLOB):
            d_cont = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
            d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
            d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
            gpu_ctx.container_blocks_encode_device(d_in.data_ptr(), nb, bs, None, ch, flags, d_cont.data_ptr(), cap)
            gpu_ctx.container_blocks_decode_async(d_cont.data_ptr(), cap, d_out.data_ptr(), data.size, d_n.data_ptr())
            gpu_ctx.sync()
            assert int(d_n.item()) == data.size
            assert torch.equal(d_out[:data.size], d_in[:data.size]), (nb, bs, ch, flags)
            assert _untouched(d_out[data.size:])


def _junk():
    """the seeded junk of test_blocks_open_rejects_flips_truncations_and_each_rule: random bytes with a valid magic and
    version, resealed"""
    rng = np.random.default_rng(0)
    for i in range(200):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        struct.pack_into("<IH", junk, 0, cb.MAGIC, 2)
        yield f"junk {i}", cb.reseal(junk)


def test_async_rejects_what_open_rejects(gpu_ctx, base):
    import ryg_rans_b200 as rb
    from ryg_rans_b200 import api
    data, geo = base
    for name, bad in list(cb.rejected_containers(*geo)) + list(_junk()):
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_open(bad)
        assert ei.value.code == -4, name
        rc, _, d_out = _async(gpu_ctx, gcb._to_dev(bad), bad.size, data.size)
        assert rc == -4, (name, rc)
        assert _untouched(d_out), f"output written for a rejected container ({name})"
    good = api.container_blocks_pack(*geo, CRC_BLOB)
    rc, n, d_out = _async(gpu_ctx, gcb._to_dev(good), good.size, data.size)
    assert rc == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_out_cap_too_small(gpu_ctx, base):
    from ryg_rans_b200 import api
    data, geo = base
    good = api.container_blocks_pack(*geo, CRC_BLOB)
    rc, n, d_out = _async(gpu_ctx, gcb._to_dev(good), good.size, data.size, out_cap=data.size - 1)
    assert rc == -3 and n == data.size and _untouched(d_out)
    # a content error comes before the space check: a blob CRC mismatch with out_cap too small is -4
    bad = good.copy()
    bad[-7] ^= 0x40
    rc, n, d_out = _async(gpu_ctx, gcb._to_dev(bad), bad.size, data.size, out_cap=data.size - 1)
    assert rc == -4 and n == data.size and _untouched(d_out)
    rc, n, d_out = _async(gpu_ctx, gcb._to_dev(good), good.size, data.size)
    assert rc == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_rejects_version_1(gpu_ctx, oracle_lib, gen):
    import oracle as orc
    from ryg_rans_b200 import api
    d1 = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(d1, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, d1, f, c, 4096)
    for flags in (0, CRC_BLOB):
        v1 = api.container_pack(0, 12, 4096, d1.size, f, oo, ob, flags)
        rc, n, d_out = _async(gpu_ctx, gcb._to_dev(v1), v1.size, d1.size)
        assert rc == -4 and n == -1 and _untouched(d_out), flags


def test_async_argument_errors_launch_nothing(gpu_ctx, base):
    from ryg_rans_b200 import api
    torch = _torch()
    data, geo = base
    good = api.container_blocks_pack(*geo, 0)
    lib = gpu_ctx.lib.dll
    d_buf = gcb._to_dev(good, 64)
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2, dtype=torch.int64, device="cuda")
    b, o, n = d_buf.data_ptr(), d_out.data_ptr(), d_n.data_ptr()
    before = gpu_ctx.launches
    calls = [(None, b, o, n), (gpu_ctx.h, None, o, n), (gpu_ctx.h, b, None, n), (gpu_ctx.h, b + 8, o, n), (gpu_ctx.h, b, o + 8, n),
             (gpu_ctx.h, b + 4, o, n), (gpu_ctx.h, b, o + 1, n), (gpu_ctx.h, b, o, n + 4)]
    for ctx, bp, op, np_ in calls:
        assert lib.rb200_container_blocks_decode_async(ctx, bp, good.size, op, data.size, np_) == -1, (bp, op, np_)
    assert gpu_ctx.launches == before
    gpu_ctx.container_blocks_decode_async(b, good.size, o, data.size, n)
    gpu_ctx.sync()
    assert torch.equal(d_out[:data.size].cpu(), torch.from_numpy(data))


def test_async_decode_in_a_cuda_graph(oracle_lib):
    import ryg_rans_b200 as rb
    from ryg_rans_b200 import api
    torch = _torch()
    conts = []
    for nb, bs, ch, flags, seed in ((3, 65536, 8192, CRC_BLOB, 51), (40, 4096, 1024, 0, 52), (5, 32768, 1024, CRC_BLOB, 53)):
        data = cb.block_data(nb, bs, seed)
        freqs, offs, blob = cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
        conts.append((api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags), data))
    corrupt = conts[0][0].copy()
    corrupt[-20] ^= 0x01                                             # inside the blob: only the blob CRC sees it
    size = max(c.size for c, _ in conts) + 256                       # fixed for the graph: the containers are shorter
    cap = max(d.size for _, d in conts)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    d_buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
    d_out = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    decode = lambda: ctx.container_blocks_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())  # noqa: E731
    with torch.cuda.stream(stream):
        def load(buf):
            d_buf.zero_()
            d_buf[:buf.size].copy_(torch.from_numpy(buf))
            d_out.fill_(SENTINEL)
            d_n.fill_(-1)
        load(conts[1][0])                                            # one call outside the graph first
        decode()
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            decode()
        launches = ctx.launches
        for buf, data, want in [(c, d, 0) for c, d in conts] + [(corrupt, None, -4), (conts[1][0], conts[1][1], 0)]:
            load(buf)
            g.replay()
            rc = ctx.lib.dll.rb200_sync(ctx.h)
            assert rc == want, (buf.size, rc)
            if data is None:
                assert _untouched(d_out)
            else:
                assert int(d_n.item()) == data.size
                assert np.array_equal(d_out[:data.size].cpu().numpy(), data), buf.size
                assert _untouched(d_out[data.size:])
        assert ctx.launches == launches                              # replays do not go through the library
    del g
    ctx.close()


def test_encode_and_async_decode_in_one_cuda_graph():
    """INTEGRATION.md's device-resident round trip: rb200_container_blocks_encode (models built) and the async decode
    captured together, replayed on new data of the same geometry"""
    import ryg_rans_b200 as rb
    torch = _torch()
    nb, bs, ch = 16, 65536, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_in = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nb * bs + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_blocks_encode_device(d_in.data_ptr(), nb, bs, None, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_blocks_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb * bs, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(cb.block_data(nb, bs, 60)))
        round_trip()                                                 # grows the encoder's workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for seed in (61, 62):
            data = cb.block_data(nb, bs, seed)
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            assert int(d_n.item()) == data.size and np.array_equal(d_out[:data.size].cpu().numpy(), data), seed
    del g
    ctx.close()
