"""The three enqueue-only container decodes share one check stage (container_decode.cuh), which is given the version of
the call: each call rejects a valid container of either other version (-4 from rb200_sync, output and *d_n_symbols
untouched), enqueues a fixed number of launches (17 for version 1, 6 for version 2, 9 for version 3), and refuses a
container that open accepts but the decoders do not take, a blob of 2^36 bytes or more (-4, output untouched,
*d_n_symbols written)."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks as cb2  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402

pytestmark = pytest.mark.gpu

CRC_BLOB = 1
SENTINEL = 0x5C
NB, BS, CH = 3, 16384, 4096                                          # every version: 3 x 16 KiB in chunks of 4096
LAUNCHES = {1: 17, 2: 6, 3: 9}


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def containers(oracle_lib):
    """one data set in a valid container of each version and both flag settings: {(version, flags): container}"""
    data = cb2.block_data(NB, BS, 11)
    f, c = oracle_lib.model(data, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data, f, c, CH)
    wf, wo, wb = cb2.oracle_blocks_encode(oracle_lib, data, NB, BS, CH)
    bf, bo, bb = cc.oracle_blocks_encode(oracle_lib, orc.CODER_BYTE, 14, data, NB, BS, CH)
    out = {}
    for flags in (0, CRC_BLOB):
        out[1, flags] = api.container_pack(rb.CODER_WORD, 12, CH, data.size, f, oo, ob, flags)
        out[2, flags] = api.container_blocks_pack(NB, BS, CH, wf, wo, wb, flags)
        out[3, flags] = api.container_blocks_coder_pack(rb.CODER_BYTE, 14, NB, BS, CH, bf, bo, bb, flags)
    return data, out


def _call(ctx, version):
    return {1: ctx.container_decode_async, 2: ctx.container_blocks_decode_async, 3: ctx.container_blocks_coder_decode_async}[version]


def _async(ctx, version, d_buf, size, n):
    """the version's async decode of d_buf[0, size) into a sentinel-filled buffer, then one rb200_sync:
    (rc, *d_n_symbols or -1, out)"""
    torch = _torch()
    d_out = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    _call(ctx, version)(d_buf.data_ptr(), size, d_out.data_ptr(), n, d_n.data_ptr())
    rc = ctx.lib.dll.rb200_sync(ctx.h)
    return rc, int(d_n.item()), d_out


def _untouched(d_out):
    return bool((d_out == SENTINEL).all().item())


@pytest.mark.parametrize("version", [1, 2, 3])
def test_each_call_rejects_the_other_versions(gpu_ctx, containers, version):
    data, conts = containers
    for flags in (0, CRC_BLOB):
        rc, n, d_out = _async(gpu_ctx, version, gbc._dev(conts[version, flags]), conts[version, flags].size, data.size)
        assert rc == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data), (version, flags)
        for other in {1, 2, 3} - {version}:
            buf = conts[other, flags]
            rc, n, d_out = _async(gpu_ctx, version, gbc._dev(buf), buf.size, data.size)
            assert rc == -4 and n == -1, (version, other, flags, rc, n)
            assert _untouched(d_out), f"version {version} call wrote output for a version {other} container"


@pytest.mark.parametrize("version", [1, 2, 3])
def test_launches_per_call(gpu_ctx, containers, version):
    torch = _torch()
    data, conts = containers
    buf = conts[version, CRC_BLOB]
    d_buf = gbc._dev(buf)
    d_out = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launches
    _call(gpu_ctx, version)(d_buf.data_ptr(), buf.size, d_out.data_ptr(), data.size)
    assert gpu_ctx.launches - before == LAUNCHES[version]
    gpu_ctx.sync()
    assert np.array_equal(d_out[:data.size].cpu().numpy(), data)


def _reseal(buf):
    """meta_crc recomputed after editing header or directory fields, with the model section of the header's version"""
    n_chunks, = struct.unpack_from("<Q", buf, 24)
    version, = struct.unpack_from("<H", buf, 4)
    model_bytes = 1024 if version == 1 else 512 * struct.unpack_from("<I", buf, 56)[0]
    hdr = bytearray(buf[:64].tobytes())
    hdr[44:52] = b"\0" * 8
    end = 64 + model_bytes + 8 * (n_chunks + 1)
    struct.pack_into("<I", buf, 44, zlib.crc32(bytes(hdr) + buf[64:end].tobytes()))
    return buf


@pytest.mark.parametrize("version", [1, 2, 3])
def test_blob_of_2_36_bytes_is_refused(gpu_ctx, containers, version):
    """A small container whose header and last directory entry claim a blob of 2^36 bytes, passed with a size that
    covers it: open's rules hold (no blob CRC, so before the verdict nothing reads past the directory), but the decoders
    hold the blob's vector count in 32 bits.  The verdict refuses it for every version and gates out every decoder."""
    data, conts = containers
    buf = conts[version, 0].copy()
    n_chunks, = struct.unpack_from("<Q", buf, 24)
    blob_bytes, = struct.unpack_from("<Q", buf, 32)
    boff = buf.size - blob_bytes
    dir_last = 64 + (1024 if version == 1 else 512 * NB) + 8 * n_chunks
    struct.pack_into("<Q", buf, 32, 1 << 36)
    struct.pack_into("<Q", buf, dir_last, 1 << 36)
    rc, n, d_out = _async(gpu_ctx, version, gbc._dev(_reseal(buf)), boff + (1 << 36), data.size)
    assert rc == -4 and n == data.size, (version, rc, n)
    assert _untouched(d_out)
