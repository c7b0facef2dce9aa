"""rb200_container_blocks_alias_decode_async: the version 4 container (per-block models of the alias coder) checked and
decoded in device memory with nothing done on the host, each block's alias table built by the decoding CTA.  Oracle
containers at five scale_bits and every geometry decode to the data and to rb200_container_blocks_alias_decode's
output, with neighbouring blocks on very different tables, so that a CTA which keeps or overwrites a table too early
writes wrong bytes; caller models at the rate ceiling; an encode and a decode round-trip with one synchronisation;
everything rb200_container_blocks_alias_open rejects is -4 from rb200_sync with the output untouched; the four async
calls reject each other's versions; eight launches per call, the 2^36-byte blob, out_cap < n and the argument errors;
a corrupt stream does not disturb a call queued behind it; one captured call picks the decoder on the GPU at every
replay, and an encode and the decode share one CUDA graph."""
import os
import struct
import sys

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks_coder as cc  # noqa: E402
import test_gpu_blocks_alias as gba  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_blocks_coder_async as gca  # noqa: E402
import test_rate_ceiling as rc  # noqa: E402

pytestmark = pytest.mark.gpu

CRC_BLOB = gca.CRC_BLOB
SENTINEL = gca.SENTINEL
_untouched = gca._untouched
_torch = gca._torch


def _oracle_container(oracle_lib, sb, data, nb, bs, ch, flags):
    freqs, offs, blob = gba._oracle(oracle_lib, sb, data, nb, bs, ch)
    return api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)


def _async(ctx, d_buf, size, n, out_cap=None, call=None):
    """an async decode (the version 4 one unless `call`) of d_buf[0, size) into a sentinel-filled buffer, then one
    rb200_sync: (rc, *d_n_symbols or -1, out)"""
    torch = _torch()
    cap = n if out_cap is None else out_cap
    d_out = torch.full((max(n, cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    (call or ctx.container_blocks_alias_decode_async)(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out


@pytest.mark.parametrize("sb", [8, 11, 12, 14, 15])
def test_async_decode_of_oracle_containers(gpu_ctx, oracle_lib, gen, sb):
    """gba._block_data cycles zipf, one symbol, two symbols, uniform, text, skewed and exact bucket multiples block by
    block; the last geometry has more blocks than the decoder grid has CTAs, so every CTA rebuilds its table"""
    torch = _torch()
    for nb, bs, ch in gca.GEOMETRIES:
        data = gba._block_data(gen, nb, bs)
        for flags in (0, CRC_BLOB):
            buf = _oracle_container(oracle_lib, sb, data, nb, bs, ch, flags)
            d_buf = gbc._dev(buf)
            rc_, n, d_out = _async(gpu_ctx, d_buf, buf.size, data.size)
            assert rc_ == 0 and n == data.size, (nb, bs, ch, flags, rc_, n)
            assert np.array_equal(d_out[:n].cpu().numpy(), data), (nb, bs, ch, flags)
            assert _untouched(d_out[n:])
            d_sync = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
            assert gpu_ctx.container_blocks_alias_decode_device(d_buf.data_ptr(), buf.size, d_sync.data_ptr(), data.size) == n
            assert torch.equal(d_sync[:n], d_out[:n]), (nb, bs, ch, flags)


@pytest.mark.parametrize("nb,bs,ch", [(12, 65536, 8192), (9, 17 * 1024, 1024)], ids=["8-per-block", "17-per-block"])
@pytest.mark.parametrize("sb", [14, 15])
def test_async_decode_at_the_ceiling(gpu_ctx, oracle_lib, sb, nb, bs, ch):
    """caller models of 255 frequency-1 symbols and a dominant one (rotated per block), ceiling and floor blocks: at 15,
    1.875 bytes per lane-step, the most the alias decoder's stream window is asked to move"""
    freqs, data = rc._blocks_case([rc._freqs(sb, "dom")], nb, bs, ch, seed=sb + ch)
    want_o, want_b = rc._oracle_blocks(oracle_lib, orc.CODER_ALIAS, sb, data, freqs, bs, ch)
    assert rc.stream_sizes(want_o)[:bs // ch].min() >= sb * ch // 8 - 128      # block 0 is a ceiling block
    cont = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, want_o, want_b, CRC_BLOB)
    got = gba._container_device_encode(gpu_ctx, sb, data, nb, bs, ch, CRC_BLOB, freqs)[:cont.size].cpu().numpy()
    assert np.array_equal(got, cont)
    rc._check_blocks_decode_async(gpu_ctx, gpu_ctx.container_blocks_alias_decode_async, cont, data)


def test_async_round_trip_without_host_sync(gpu_ctx, gen):
    torch = _torch()
    for sb in (14, 11, 15):
        for nb, bs, ch in ((8, 65536, 8192), (64, 4096, 1024), (5, 17 * 1024, 1024)):
            data = gba._block_data(gen, nb, bs)
            cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
            d_in = gbc._dev(data)
            for flags in (0, CRC_BLOB):
                d_cont = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
                d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
                d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
                gpu_ctx.container_blocks_alias_encode_device(sb, d_in.data_ptr(), nb, bs, None, ch, flags, d_cont.data_ptr(), cap)
                gpu_ctx.container_blocks_alias_decode_async(d_cont.data_ptr(), cap, d_out.data_ptr(), data.size, d_n.data_ptr())
                gpu_ctx.sync()
                assert int(d_n.item()) == data.size
                assert torch.equal(d_out[:data.size], d_in[:data.size]), (sb, nb, bs, ch, flags)
                assert _untouched(d_out[data.size:])


@pytest.fixture(scope="module")
def base(oracle_lib):
    """test_alias_open_rejects_each_rule's container: alias coder at 14, 3 blocks of 16 KiB in chunks of 4096"""
    nb, bs, ch, sb = 3, 16384, 4096, 14
    data = cc.block_data(nb, bs, 9)
    freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_ALIAS, sb, data, nb, bs, ch)
    return data, (nb, bs, ch, sb, freqs, offs, blob)


def _rejected_containers(nb, bs, ch, sb, freqs, offs, blob):
    """every container test_alias_open_rejects_each_rule builds: field edits resealed, CRC flips in every section,
    truncations, a blob CRC that does not match"""
    dir_off = 64 + 512 * nb
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    nz = int(np.flatnonzero(freqs[1])[0])
    edits = {
        "coder word": [(6, "<B", 0)], "coder byte": [(6, "<B", 1)], "coder rans64": [(6, "<B", 3)], "coder 4": [(6, "<B", 4)],
        "scale_bits 7": [(7, "<B", 7)], "scale_bits 16": [(7, "<B", 16)],
        "version 3": [(4, "<H", 3)], "version 2": [(4, "<H", 2)], "version 1": [(4, "<H", 1)], "version 5": [(4, "<H", 5)],
        "magic": [(0, "<I", 0x12345678)],
        "lanes 64": [(8, "<I", 64)], "33 chunks per block": [(12, "<I", 512), (52, "<I", 33 * 512), (16, "<Q", nb * 33 * 512),
                                                             (24, "<Q", nb * 33)],
        "n_blocks 0": [(56, "<I", 0)], "n_symbols != n_blocks * block_size": [(16, "<Q", nb * bs + ch)],
        "n_chunks + 1": [(24, "<Q", offs.size)], "blob_bytes odd": [(32, "<Q", blob.size + 8)],
        "reserved nonzero": [(60, "<I", 1)], "unknown flag bit": [(40, "<I", 2)], "unknown flag bit with CRC_BLOB": [(40, "<I", 3)],
        "block 1 sums to 2^14 - 1": [(64 + 512 + 2 * nz, "<H", int(freqs[1][nz]) - 1)],
        "block 2 sums to 2^14 + 1": [(64 + 1024 + 2 * nz, "<H", int(freqs[2][nz]) + 1)],
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
        g = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        for pos in (5, 6, 7, 53, 70, 64 + 512 * 2 + 3, dir_off + 9) + ((g.size - 7,) if flags else ()):
            bad = g.copy()
            bad[pos] ^= 0x40
            yield f"flip {pos}, flags {flags}", bad
        for cut in list(range(0, dir_off + 8 * offs.size + 16, 13)) + [g.size - 16, g.size - 1]:
            yield f"cut {cut}, flags {flags}", g[:cut].copy()
    crc = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    struct.pack_into("<I", crc, 48, struct.unpack_from("<I", crc, 48)[0] ^ 1)
    yield "blob CRC", crc


def _junk():
    """random bytes with a valid magic and version 4, resealed"""
    rng = np.random.default_rng(4)
    for i in range(100):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        struct.pack_into("<IH", junk, 0, cc.MAGIC, 4)
        yield f"junk {i}", cc.reseal(junk)


def test_async_rejects_what_open_rejects(gpu_ctx, base):
    data, geo = base
    for name, bad in list(_rejected_containers(*geo)) + list(_junk()):
        cc.rejected(api.container_blocks_alias_open, bad)
        rc_, _, d_out = _async(gpu_ctx, gbc._dev(bad), bad.size, data.size)
        assert rc_ == -4, (name, rc_)
        assert _untouched(d_out), f"output written for a rejected container ({name})"
    nb, bs, ch, sb, freqs, offs, blob = geo
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    rc_, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size)
    assert rc_ == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_calls_reject_each_others_versions(gpu_ctx, oracle_lib, gen, base):
    """the version 4 call rejects valid version 1, 2 and 3 containers; the version 1, 2 and 3 calls reject a valid
    version 4 container: -4, output and *d_n_symbols untouched"""
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    bf, bo, bb = cc.oracle_blocks_encode(oracle_lib, orc.CODER_BYTE, sb, data, nb, bs, ch)
    others = list(gca._other_versions(oracle_lib, gen))
    others += [(f"version 3, flags {flags}", api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, bf, bo, bb, flags))
               for flags in (0, CRC_BLOB)]
    for name, buf in others:
        rc_, n, d_out = _async(gpu_ctx, gbc._dev(buf), buf.size, data.size)
        assert rc_ == -4 and n == -1, (name, rc_, n)
        assert _untouched(d_out), name
    for flags in (0, CRC_BLOB):
        v4 = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        d_buf = gbc._dev(v4)
        for call in (gpu_ctx.container_decode_async, gpu_ctx.container_blocks_decode_async, gpu_ctx.container_blocks_coder_decode_async):
            rc_, n, d_out = _async(gpu_ctx, d_buf, v4.size, data.size, call=call)
            assert rc_ == -4 and n == -1, (call.__name__, flags, rc_, n)
            assert _untouched(d_out), call.__name__
        rc_, n, d_out = _async(gpu_ctx, d_buf, v4.size, data.size)
        assert rc_ == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_launches_per_call(gpu_ctx, base):
    """plan, meta CRC, blob CRC, prefix check, verdict and the three decoders of RB200_BLOCK_ALIAS_DISPATCH"""
    torch = _torch()
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    d_buf = gbc._dev(good)
    d_out = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launches
    gpu_ctx.container_blocks_alias_decode_async(d_buf.data_ptr(), good.size, d_out.data_ptr(), data.size)
    assert gpu_ctx.launches - before == 8
    gpu_ctx.sync()
    assert np.array_equal(d_out[:data.size].cpu().numpy(), data)


def test_blob_of_2_36_bytes_is_refused(gpu_ctx, base):
    """header and last directory entry claim a blob of 2^36 bytes, with a size that covers it (nothing is read past the
    directory without the blob CRC): open's rules hold, the verdict refuses it"""
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    buf = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    boff = buf.size - blob.size
    struct.pack_into("<Q", buf, 32, 1 << 36)
    struct.pack_into("<Q", buf, 64 + 512 * nb + 8 * (offs.size - 1), 1 << 36)
    rc_, n, d_out = _async(gpu_ctx, gbc._dev(cc.reseal(buf)), boff + (1 << 36), data.size)
    assert rc_ == -4 and n == data.size, (rc_, n)
    assert _untouched(d_out)


def test_async_out_cap_too_small(gpu_ctx, base):
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)
    rc_, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size, out_cap=data.size - 1)
    assert rc_ == -3 and n == data.size and _untouched(d_out)
    bad = good.copy()                                                # a content error comes before the space check
    bad[-7] ^= 0x40
    rc_, n, d_out = _async(gpu_ctx, gbc._dev(bad), bad.size, data.size, out_cap=data.size - 1)
    assert rc_ == -4 and n == data.size and _untouched(d_out)
    rc_, n, d_out = _async(gpu_ctx, gbc._dev(good), good.size, data.size)
    assert rc_ == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_argument_errors_launch_nothing(gpu_ctx, base):
    torch = _torch()
    data, (nb, bs, ch, sb, freqs, offs, blob) = base
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    lib = gpu_ctx.lib.dll
    d_buf = gbc._dev(good, 64)
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2, dtype=torch.int64, device="cuda")
    b, o, n = d_buf.data_ptr(), d_out.data_ptr(), d_n.data_ptr()
    before = gpu_ctx.launches
    calls = [(None, b, o, n), (gpu_ctx.h, None, o, n), (gpu_ctx.h, b, None, n), (gpu_ctx.h, b + 8, o, n), (gpu_ctx.h, b, o + 8, n),
             (gpu_ctx.h, b + 4, o, n), (gpu_ctx.h, b, o + 1, n), (gpu_ctx.h, b, o, n + 4)]
    for ctx, bp, op, np_ in calls:
        assert lib.rb200_container_blocks_alias_decode_async(ctx, bp, good.size, op, data.size, np_) == -1, (bp, op, np_)
    assert gpu_ctx.launches == before
    gpu_ctx.container_blocks_alias_decode_async(b, good.size, o, data.size, n)
    gpu_ctx.sync()
    assert torch.equal(d_out[:data.size].cpu(), torch.from_numpy(data))


@pytest.mark.parametrize("sb", [14, 12, 11])
def test_async_corrupt_stream_then_a_valid_container(gpu_ctx, oracle_lib, gen, sb):
    """a corrupt stream in a container with flags 0: every check passes and the decoder reports it.  A valid call
    queued right behind it, no rb200_sync in between, decodes completely (the block counter re-armed itself); the sync
    reports the first call's error"""
    torch = _torch()
    nb, bs, ch = 4, 16384, 4096
    data = gba._block_data(gen, nb, bs)
    freqs, offs, blob = gba._oracle(oracle_lib, sb, data, nb, bs, ch)
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    bad = good.copy()
    bad[good.size - blob.size + int(offs[5]) + 3] ^= 0x10               # lane 0's final state in chunk 5
    d_bad, d_good = gbc._dev(bad), gbc._dev(good)
    rc_, n, _ = _async(gpu_ctx, d_bad, bad.size, data.size)
    assert rc_ == -4 and n == data.size, rc_
    d_out0 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    d_out1 = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_blocks_alias_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), data.size)
    gpu_ctx.container_blocks_alias_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), data.size)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4
    assert np.array_equal(d_out1[:data.size].cpu().numpy(), data)
    assert _untouched(d_out1[data.size:])
    rc_, n, d_out = _async(gpu_ctx, d_good, good.size, data.size)
    assert rc_ == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def test_async_decoder_picked_on_the_device_in_a_cuda_graph(oracle_lib, gen):
    """ONE captured call, replayed over containers of one geometry at scale_bits 14, 12 and 11 (each its own decoder)
    copied into the same buffer, with a rejected one between them"""
    torch = _torch()
    nb, bs, ch = 40, 8192, 2048
    data = gba._block_data(gen, nb, bs)
    conts = [(_oracle_container(oracle_lib, sb, data, nb, bs, ch, flags), data) for sb, flags in ((14, CRC_BLOB), (12, 0), (11, CRC_BLOB))]
    rejected = conts[1][0].copy()
    rejected[64 + 512 * 7 + 9] ^= 0x01                               # block 7's model: meta_crc
    size = max(c.size for c, _ in conts) + 256                       # fixed for the graph: the containers are shorter
    cap = nb * bs
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    d_buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
    d_out = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    decode = lambda: ctx.container_blocks_alias_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())  # noqa: E731
    with torch.cuda.stream(stream):
        def load(buf):
            d_buf.zero_()
            d_buf[:buf.size].copy_(torch.from_numpy(buf))
            d_out.fill_(SENTINEL)
            d_n.fill_(-1)
        load(conts[0][0])                                            # one call outside the graph first
        decode()
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            decode()
        launches = ctx.launches
        seq = [conts[0] + (0,), conts[1] + (0,), (rejected, None, -4), conts[2] + (0,), conts[0] + (0,)]
        for buf, data, want in seq:
            load(buf)
            g.replay()
            rc_ = ctx.lib.dll.rb200_sync(ctx.h)
            assert rc_ == want, (buf.size, rc_)
            if data is None:
                assert _untouched(d_out)
            else:
                assert int(d_n.item()) == data.size
                assert np.array_equal(d_out[:data.size].cpu().numpy(), data), buf.size
                assert _untouched(d_out[data.size:])
        assert ctx.launches == launches                              # replays do not go through the library
    del g
    ctx.close()


@pytest.mark.parametrize("sb", [14, 15])
def test_encode_and_async_decode_in_one_cuda_graph(gen, sb):
    """rb200_container_blocks_alias_encode (models built on the GPU) and the async decode captured together, replayed on
    new data of the same geometry"""
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
        ctx.container_blocks_alias_encode_device(sb, d_in.data_ptr(), nb, bs, None, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_blocks_alias_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb * bs, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(cc.block_data(nb, bs, 60)))
        round_trip()                                                 # grows the encoder's workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for seed in (61, 62):
            data = np.concatenate([cc.block_data(nb // 2, bs, seed), gba._block_data(gen, nb // 2, bs)])
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            assert int(d_n.item()) == data.size and np.array_equal(d_out[:data.size].cpu().numpy(), data), seed
    del g
    ctx.close()
