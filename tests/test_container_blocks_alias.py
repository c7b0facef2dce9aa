"""The version 4 container (per-block models for the alias coder) on the host, no GPU needed:
rb200_container_blocks_alias_pack against an independent packer written from the format (struct + zlib), open of it
decoding block by block through the oracle, every version 4 rule broken on its own, the four container versions
rejecting each other, and the argument errors of pack."""
import ctypes as C
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
import test_container_blocks_coder as cc  # noqa: E402

MAGIC = 0x43324252
CRC_BLOB = api.CONTAINER_CRC_BLOB


def py_pack(sb, n_blocks, block_size, chunk, freqs, offsets, blob, flags):
    """The version 4 layout, from its description alone: version 3's with coder 2 (alias)."""
    n = n_blocks * block_size
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 4, 2, sb, 32, chunk, n, n // chunk, blob.size, flags, 0, 0, block_size, n_blocks, 0)
    model = np.asarray(freqs, "<u2").tobytes()
    directory = np.asarray(offsets, "<u8").tobytes()
    meta = zlib.crc32(hdr + model + directory)
    blob_crc = zlib.crc32(blob.tobytes()) if flags & CRC_BLOB else 0
    body = hdr[:44] + struct.pack("<II", meta, blob_crc) + hdr[52:] + model + directory
    body += b"\0" * (-len(body) % 16)
    return np.frombuffer(body + blob.tobytes(), np.uint8).copy()


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("sb", [8, 12, 14, 15])
def test_alias_pack_equals_independent_packer_and_opens(oracle_lib, sb, flags):
    assert rb.CODER_ALIAS == 2
    for i, (nb, bs, ch) in enumerate(cc.GEOMETRIES):
        data = cc.block_data(nb, bs, 70 + i)
        freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_ALIAS, sb, data, nb, bs, ch)
        assert (freqs.astype(np.uint32).sum(axis=1) == 1 << sb).all()
        buf = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        want = py_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        assert buf.size == want.size and np.array_equal(buf, want), (nb, bs, ch)
        meta, f2, o2, b2 = api.container_blocks_alias_open(buf)
        assert meta == {"coder": rb.CODER_ALIAS, "scale_bits": sb, "n_blocks": nb, "block_size": bs, "chunk_syms": ch, "flags": flags,
                        "n_symbols": nb * bs, "n_chunks": offs.size - 1, "blob_bytes": blob.size}
        assert np.array_equal(f2, freqs) and np.array_equal(o2, offs) and np.array_equal(b2, blob)
        assert np.array_equal(cc.oracle_decode_blocks(oracle_lib, orc.CODER_ALIAS, meta, f2, o2, b2), data), (nb, bs, ch)


def test_alias_pack_one_symbol_block_at_15(oracle_lib):
    """a one-symbol block at scale_bits 15: its frequency 32768 fits the u16 model section"""
    nb, bs, ch, sb = 2, 8192, 4096, 15
    data = cc.block_data(nb, bs, 3)                  # the last block is one symbol
    freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_ALIAS, sb, data, nb, bs, ch)
    assert freqs[1].max() == 32768
    meta, f2, o2, b2 = api.container_blocks_alias_open(api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob))
    assert np.array_equal(cc.oracle_decode_blocks(oracle_lib, orc.CODER_ALIAS, meta, f2, o2, b2), data)


@pytest.fixture(scope="module")
def base(oracle_lib):
    """alias coder at 14: 3 blocks of 16 KiB in chunks of 4096, 12 chunks, directory at 64 + 1536"""
    nb, bs, ch, sb = 3, 16384, 4096, 14
    data = cc.block_data(nb, bs, 9)
    freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_ALIAS, sb, data, nb, bs, ch)
    return nb, bs, ch, sb, freqs, offs, blob


def test_alias_open_rejects_each_rule(base):
    nb, bs, ch, sb, freqs, offs, blob = base
    dir_off = 64 + 512 * nb
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    assert api.container_blocks_alias_open(cc.reseal(good.copy()))[0]["n_symbols"] == nb * bs     # reseal reproduces the CRC
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
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_alias_open(cc.reseal(bad))
        assert ei.value.code == -4, name
    for flags in (0, CRC_BLOB):                                   # CRC flips in every section, truncations
        g = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        for pos in (5, 6, 7, 53, 70, 64 + 512 * 2 + 3, dir_off + 9) + ((g.size - 7,) if flags else ()):
            bad = g.copy()
            bad[pos] ^= 0x40
            cc.rejected(api.container_blocks_alias_open, bad)
        for cut in list(range(0, dir_off + 8 * offs.size + 16, 13)) + [g.size - 16, g.size - 1]:
            cc.rejected(api.container_blocks_alias_open, g[:cut].copy())
    crc = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)   # a blob CRC that does not match
    struct.pack_into("<I", crc, 48, struct.unpack_from("<I", crc, 48)[0] ^ 1)
    cc.rejected(api.container_blocks_alias_open, crc)


def test_alias_and_other_versions_reject_each_other(oracle_lib, gen, base):
    nb, bs, ch, sb, freqs, offs, blob = base
    data = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(data, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data, f, c, 4096)
    wf, woffs, wblob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_WORD, 12, cc.block_data(nb, bs, 5), nb, bs, ch)
    bf, boffs, bblob = cc.oracle_blocks_encode(oracle_lib, orc.CODER_BYTE, sb, cc.block_data(nb, bs, 6), nb, bs, ch)
    for flags in (0, CRC_BLOB):
        v1 = api.container_pack(rb.CODER_WORD, 12, 4096, data.size, f, oo, ob, flags)
        v2 = api.container_blocks_pack(nb, bs, ch, wf, woffs, wblob, flags)
        v3 = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, bf, boffs, bblob, flags)
        v4 = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
        api.container_blocks_alias_open(v4)
        for opener in (api.container_open, api.container_blocks_open, api.container_blocks_coder_open):
            cc.rejected(opener, v4)
        for buf in (v1, v2, v3):
            cc.rejected(api.container_blocks_alias_open, buf)
        # relabelled (CRC resealed): version 4 as 3 (alias is not a version 3 coder), version 3 as 4 (byte is not alias)
        as3 = v4.copy()
        struct.pack_into("<H", as3, 4, 3)
        cc.rejected(api.container_blocks_coder_open, cc.reseal(as3))
        as4 = v3.copy()
        struct.pack_into("<H", as4, 4, 4)
        cc.rejected(api.container_blocks_alias_open, cc.reseal(as4))


def test_alias_pack_argument_errors(base):
    nb, bs, ch, sb, freqs, offs, blob = base
    bad = freqs.copy()
    bad[2][int(np.flatnonzero(bad[2])[0])] -= 1                        # block 2 sums to 2^14 - 1
    with pytest.raises(rb.RansError) as ei:
        api.container_blocks_alias_pack(sb, nb, bs, ch, bad, offs, blob, 0)
    assert ei.value.code == -2
    with pytest.raises(rb.RansError) as ei:                             # the right total for another scale_bits
        api.container_blocks_alias_pack(13, nb, bs, ch, freqs, offs, blob, 0)
    assert ei.value.code == -2
    lib = rb.load().dll
    out = np.zeros(1 << 20, np.uint8)
    args = (freqs.ctypes.data, offs.ctypes.data, blob.ctypes.data, blob.size, 0, out.ctypes.data, out.size, None)
    for s in (0, 7, 16, 17, 255):
        assert lib.rb200_container_blocks_alias_pack(s, nb, bs, ch, *args) == -1, s
    for g in ((0, bs, ch), (nb, bs, 3000), (nb, 33 * 512, 512), (nb, bs, 16), (nb, 0, ch)):
        assert lib.rb200_container_blocks_alias_pack(sb, *g, *args) == -1, g
    assert lib.rb200_container_blocks_alias_pack(sb, nb, bs, ch, None, *args[1:]) == -1
    assert lib.rb200_container_blocks_alias_pack(sb, nb, bs, ch, *args[:5], None, out.size, None) == -1
    for o, b in ((offs, blob[:-16]), (offs, np.concatenate([blob, np.zeros(16, np.uint8)]))):   # directory and blob disagree
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, o, b, 0)
        assert ei.value.code == -1
    assert lib.rb200_container_blocks_alias_pack(sb, nb, bs, ch, *args[:5], out.ctypes.data, 100, None) == -3
    info = api.ContainerBlocksCoderInfo()
    assert lib.rb200_container_blocks_alias_open(None, 100, C.byref(info)) == -1
    good = api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, 0)
    assert lib.rb200_container_blocks_alias_open(good.ctypes.data, good.size, None) == -1

