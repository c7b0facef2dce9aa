"""rb200_container_blocks_coder_decode_async: the version 3 container (per-block models of the byte and rans64 coders)
checked and decoded in device memory with nothing done on the host.  Oracle containers of both coders, four scale_bits
and every geometry decode to the data and to rb200_container_blocks_coder_decode's output; an encode and a decode
round-trip with one synchronisation; everything rb200_container_blocks_coder_open rejects is -4 from rb200_sync with the
output untouched; out_cap < n is -3; a corrupt stream is -4 and does not disturb a call queued behind it; one captured
call picks the decoder on the GPU at every replay."""
import os
import struct
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks as cb2  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402

pytestmark = pytest.mark.gpu

CRC_BLOB = 1
SENTINEL = 0x5C
CODERS = [rb.CODER_BYTE, rb.CODER_RANS64]
# 32 chunks per block; 17 chunks per block; chunk == block; 1 chunk per block, more blocks than any decoder grid has
# CTAs (at most 8 per SM)
GEOMETRIES = [(3, 65536, 2048), (4, 17 * 1024, 1024), (4, 65536, 65536), (1536, 1024, 1024)]


def _torch():
    import torch
    return torch


def _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags):
    freqs, offs, blob = gbc._oracle(oracle_lib, coder, sb, data, nb, bs, ch)
    return api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, offs, blob, flags)


def _async(ctx, d_buf, size, n, out_cap=None):
    """the async decode of d_buf[0, size) into a sentinel-filled buffer, then one rb200_sync: (rc, *d_n_symbols or -1, out)"""
    torch = _torch()
    cap = n if out_cap is None else out_cap
    d_out = torch.full((max(n, cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    ctx.container_blocks_coder_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())
    rc = ctx.lib.dll.rb200_sync(ctx.h)
    return rc, int(d_n.item()), d_out


def _untouched(d_out):
    return bool((d_out == SENTINEL).all().item())


@pytest.mark.parametrize("sb", [8, 12, 14, 15])
@pytest.mark.parametrize("coder", CODERS)
def test_async_decode_of_oracle_containers(gpu_ctx, oracle_lib, coder, sb):
    torch = _torch()
    for i, (nb, bs, ch) in enumerate(GEOMETRIES):
        data = cc.block_data(nb, bs, 70 + i)
        for flags in (0, CRC_BLOB):
            buf = _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags)
            d_buf = gbc._dev(buf)
            rc, n, d_out = _async(gpu_ctx, d_buf, buf.size, data.size)
            assert rc == 0 and n == data.size, (nb, bs, ch, flags, rc, n)
            out = d_out[:n].cpu().numpy()
            assert np.array_equal(out, data), (nb, bs, ch, flags)
            assert _untouched(d_out[n:])
            d_sync = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
            assert gpu_ctx.container_blocks_coder_decode_device(d_buf.data_ptr(), buf.size, d_sync.data_ptr(), data.size) == n
            assert torch.equal(d_sync[:n], d_out[:n]), (nb, bs, ch, flags)


def test_async_round_trip_without_host_sync(gpu_ctx, gen):
    torch = _torch()
    for coder, sb in ((rb.CODER_BYTE, 14), (rb.CODER_BYTE, 11), (rb.CODER_RANS64, 15)):
        for nb, bs, ch in ((8, 65536, 8192), (64, 4096, 1024), (5, 17 * 1024, 1024)):
            data = gbc._block_data(gen, nb, bs)
            cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
            d_in = gbc._dev(data)
            for flags in (0, CRC_BLOB):
                d_cont = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
                d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
                d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
                gpu_ctx.container_blocks_coder_encode_device(coder, sb, d_in.data_ptr(), nb, bs, None, ch, flags, d_cont.data_ptr(), cap)
                gpu_ctx.container_blocks_coder_decode_async(d_cont.data_ptr(), cap, d_out.data_ptr(), data.size, d_n.data_ptr())
                gpu_ctx.sync()
                assert int(d_n.item()) == data.size
                assert torch.equal(d_out[:data.size], d_in[:data.size]), (coder, sb, nb, bs, ch, flags)
                assert _untouched(d_out[data.size:])


@pytest.fixture(scope="module")
def base(oracle_lib):
    """test_coder_open_rejects_each_rule's container: byte coder at 14, 3 blocks of 16 KiB in chunks of 4096"""
    nb, bs, ch, sb = 3, 16384, 4096, 14
    data = cc.block_data(nb, bs, 7)
    freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, cc.orc.CODER_BYTE, sb, data, nb, bs, ch)
    return data, (nb, bs, ch, sb, freqs, offs, blob)


def _rejected_containers(nb, bs, ch, sb, freqs, offs, blob):
    """every container test_coder_open_rejects_each_rule builds: field edits resealed, CRC flips in every section,
    truncations, a blob CRC that does not match"""
    dir_off = 64 + 512 * nb
    good = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, 0)
    nz = int(np.flatnonzero(freqs[1])[0])
    edits = {
        "coder word": [(6, "<B", 0)], "coder alias": [(6, "<B", 2)], "coder 4": [(6, "<B", 4)],
        "scale_bits 7": [(7, "<B", 7)], "scale_bits 16": [(7, "<B", 16)],
        "version 2": [(4, "<H", 2)], "version 1": [(4, "<H", 1)], "version 4": [(4, "<H", 4)], "magic": [(0, "<I", 0x12345678)],
        "lanes 64": [(8, "<I", 64)], "33 chunks per block": [(12, "<I", 512), (52, "<I", 33 * 512), (16, "<Q", nb * 33 * 512),
                                                             (24, "<Q", nb * 33)],
        "n_blocks 0": [(56, "<I", 0)], "n_symbols != n_blocks * block_size": [(16, "<Q", nb * bs + ch)],
        "n_chunks + 1": [(24, "<Q", offs.size)], "blob_bytes odd": [(32, "<Q", blob.size + 8)],
        "reserved nonzero": [(60, "<I", 1)], "unknown flag bit": [(40, "<I", 2)], "unknown flag bit with CRC_BLOB": [(40, "<I", 3)],
        "block 1 sums to 2^14 - 1": [(64 + 512 + 2 * nz, "<H", int(freqs[1][nz]) - 1)],
        "block 2 sums to 2^14 + 1": [(64 + 1024 + 2 * nz, "<H", int(freqs[2][nz]) + 1)],
        "block 0 sums to 4096": [(64 + 2 * s, "<H", int(v)) for s, v in enumerate(np.bincount(np.arange(4096) % 256, minlength=256))],
        "scale_bits 13 (the blocks sum to 2^14)": [(7, "<B", 13)],
        "first stream starts beyond the first vector": [(dir_off, "<Q", 32)],
        "directory not monotone": [(dir_off + 8, "<Q", int(offs[2]) + 16)],
        "last entry != blob size": [(dir_off + 8 * (offs.size - 1), "<Q", int(offs[-1]) - 16)],
    }
    for name, fields in edits.items():
        bad = good.copy()
        for off, fmt, val in fields:
            struct.pack_into(fmt, bad, off, val)
        yield name, cc.reseal(bad)
    for flags in (0, CRC_BLOB):
        g = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, flags)
        for pos in (5, 6, 7, 53, 70, 64 + 512 * 2 + 3, dir_off + 9) + ((g.size - 7,) if flags else ()):
            bad = g.copy()
            bad[pos] ^= 0x40
            yield f"flip {pos}, flags {flags}", bad
        for cut in list(range(0, dir_off + 8 * offs.size + 16, 13)) + [g.size - 16, g.size - 1]:
            yield f"cut {cut}, flags {flags}", g[:cut].copy()
    crc = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    struct.pack_into("<I", crc, 48, struct.unpack_from("<I", crc, 48)[0] ^ 1)
    yield "blob CRC", crc


def _junk():
    """random bytes with a valid magic and version 3, resealed"""
    rng = np.random.default_rng(3)
    for i in range(200):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        struct.pack_into("<IH", junk, 0, cc.MAGIC, 3)
        yield f"junk {i}", cc.reseal(junk)


def _other_versions(oracle_lib, gen):
    """version 1 and version 2 containers of both flag settings"""
    import oracle as orc
    d1 = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(d1, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, d1, f, c, 4096)
    nb, bs, ch = 3, 16384, 4096
    d2 = cb2.block_data(nb, bs, 8)
    wf, wo, wb = cb2.oracle_blocks_encode(oracle_lib, d2, nb, bs, ch)
    for flags in (0, CRC_BLOB):
        yield f"version 1, flags {flags}", api.container_pack(rb.CODER_WORD, 12, 4096, d1.size, f, oo, ob, flags)
        yield f"version 2, flags {flags}", api.container_blocks_pack(nb, bs, ch, wf, wo, wb, flags)


def test_async_rejects_what_open_rejects(gpu_ctx, oracle_lib, gen, base):
    data, geo = base
    cases = list(_rejected_containers(*geo)) + list(_junk()) + list(_other_versions(oracle_lib, gen))
    for name, bad in cases:
        cc.rejected(api.container_blocks_coder_open, bad)
        rc, _, d_out = _async(gpu_ctx, gbc._dev(bad), bad.size, data.size)
        assert rc == -4, (name, rc)
        assert _untouched(d_out), f"output written for a rejected container ({name})"
    nb, bs, ch, sb, freqs, offs, blob = geo
    good = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    rc, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size)
    assert rc == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_other_async_decodes_reject_version_3(gpu_ctx, base):
    torch = _torch()
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    for flags in (0, CRC_BLOB):
        v3 = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, flags)
        d_buf = gbc._dev(v3)
        for call in (gpu_ctx.container_decode_async, gpu_ctx.container_blocks_decode_async):
            d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
            d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
            call(d_buf.data_ptr(), v3.size, d_out.data_ptr(), data.size, d_n.data_ptr())
            assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4
            assert int(d_n.item()) == -1 and _untouched(d_out)


def test_async_out_cap_too_small(gpu_ctx, base):
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    good = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    rc, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size, out_cap=data.size - 1)
    assert rc == -3 and n == data.size and _untouched(d_out)
    # a content error comes before the space check: a blob CRC mismatch with out_cap too small is -4
    bad = good.copy()
    bad[-7] ^= 0x40
    rc, n, d_out = _async(gpu_ctx, gbc._dev(bad), bad.size, data.size, out_cap=data.size - 1)
    assert rc == -4 and n == data.size and _untouched(d_out)
    rc, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size)
    assert rc == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_argument_errors_launch_nothing(gpu_ctx, base):
    torch = _torch()
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    good = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, 0)
    lib = gpu_ctx.lib.dll
    d_buf = gbc._dev(good, 64)
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2, dtype=torch.int64, device="cuda")
    b, o, n = d_buf.data_ptr(), d_out.data_ptr(), d_n.data_ptr()
    before = gpu_ctx.launches
    calls = [(None, b, o, n), (gpu_ctx.h, None, o, n), (gpu_ctx.h, b, None, n), (gpu_ctx.h, b + 8, o, n), (gpu_ctx.h, b, o + 8, n),
             (gpu_ctx.h, b + 4, o, n), (gpu_ctx.h, b, o + 1, n), (gpu_ctx.h, b, o, n + 4)]
    for ctx, bp, op, np_ in calls:
        assert lib.rb200_container_blocks_coder_decode_async(ctx, bp, good.size, op, data.size, np_) == -1, (bp, op, np_)
    assert gpu_ctx.launches == before
    gpu_ctx.container_blocks_coder_decode_async(b, good.size, o, data.size, n)
    gpu_ctx.sync()
    assert torch.equal(d_out[:data.size].cpu(), torch.from_numpy(data))


@pytest.mark.parametrize("coder,sb", [(rb.CODER_BYTE, 14), (rb.CODER_RANS64, 14), (rb.CODER_BYTE, 11)])
def test_async_corrupt_stream_then_a_valid_container(gpu_ctx, oracle_lib, gen, coder, sb):
    """test_block_coder_errors' corrupt stream in a container with flags 0: every check passes and the decoder reports
    it.  A valid call queued right behind it, no rb200_sync in between, decodes completely although the status word
    already holds the first call's error; the sync reports that error."""
    torch = _torch()
    nb, bs, ch = 4, 16384, 4096
    data = gbc._block_data(gen, nb, bs)
    freqs, offs, blob = gbc._oracle(oracle_lib, coder, sb, data, nb, bs, ch)
    good = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, offs, blob, 0)
    bad = good.copy()
    bad[good.size - blob.size + int(offs[5]) + 3] ^= 0x10               # lane 0's final state in chunk 5
    d_bad, d_good = gbc._dev(bad), gbc._dev(good)
    rc, n, _ = _async(gpu_ctx, d_bad, bad.size, data.size)
    assert rc == -4 and n == data.size, rc
    d_out0 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    d_out1 = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_blocks_coder_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), data.size)
    gpu_ctx.container_blocks_coder_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), data.size)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4
    assert np.array_equal(d_out1[:data.size].cpu().numpy(), data)
    assert _untouched(d_out1[data.size:])
    rc, n, d_out = _async(gpu_ctx, d_good, good.size, data.size)
    assert rc == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_decoder_picked_on_the_device_in_a_cuda_graph(oracle_lib, gen):
    """ONE captured call, replayed over containers of every decoder variant (byte at 14, 12 and generic, rans64) of
    several geometries and both flag settings copied into the same buffer, a blob-corrupted one and a valid one again"""
    torch = _torch()
    conts = []
    for coder, sb, nb, bs, ch, flags in ((rb.CODER_BYTE, 14, 3, 65536, 8192, CRC_BLOB), (rb.CODER_BYTE, 12, 40, 4096, 1024, 0),
                                         (rb.CODER_BYTE, 9, 5, 17 * 1024, 1024, CRC_BLOB), (rb.CODER_BYTE, 15, 2, 65536, 65536, 0),
                                         (rb.CODER_RANS64, 15, 6, 32768, 1024, CRC_BLOB), (rb.CODER_RANS64, 12, 600, 1024, 1024, 0)):
        data = gbc._block_data(gen, nb, bs)
        conts.append((_oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags), data))
    corrupt = conts[0][0].copy()
    corrupt[-20] ^= 0x01                                             # inside the blob: only the blob CRC sees it
    size = max(c.size for c, _ in conts) + 256                       # fixed for the graph: the containers are shorter
    cap = max(d.size for _, d in conts)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    d_buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
    d_out = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    decode = lambda: ctx.container_blocks_coder_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())  # noqa: E731
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


@pytest.mark.parametrize("coder,sb", [(rb.CODER_BYTE, 14), (rb.CODER_RANS64, 15)])
def test_encode_and_async_decode_in_one_cuda_graph(gen, coder, sb):
    """INTEGRATION.md's device-resident round trip: rb200_container_blocks_coder_encode (models built) and the async
    decode captured together, replayed on new data of the same geometry"""
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
        ctx.container_blocks_coder_encode_device(coder, sb, d_in.data_ptr(), nb, bs, None, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_blocks_coder_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb * bs, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(cc.block_data(nb, bs, 60)))
        round_trip()                                                 # grows the encoder's workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for seed in (61, 62):
            data = np.concatenate([cc.block_data(nb // 2, bs, seed), gbc._block_data(gen, nb // 2, bs)])
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            assert int(d_n.item()) == data.size and np.array_equal(d_out[:data.size].cpu().numpy(), data), seed
    del g
    ctx.close()
