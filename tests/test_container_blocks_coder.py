"""The version 3 container (per-block models for the byte and rans64 coders) on the host, no GPU needed:
rb200_container_blocks_coder_pack against an independent packer written from the format (struct + zlib), open of it
decoding block by block through the oracle, every rule open enforces broken on its own, and the three container
versions rejecting each other."""
import struct
import zlib

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

MAGIC = 0x43324252
CRC_BLOB = api.CONTAINER_CRC_BLOB
CODERS = [(rb.CODER_BYTE, orc.CODER_BYTE), (rb.CODER_RANS64, orc.CODER_RANS64)]
# (n_blocks, block_size, chunk_syms): one block; 64 KiB / 8192; chunk == block; 32 chunks per block; 17 chunks per block
GEOMETRIES = [(1, 65536, 8192), (3, 65536, 8192), (5, 4096, 4096), (3, 65536, 2048), (4, 17 * 1024, 1024)]


def block_data(n_blocks, block_size, seed):
    """per block one dominant symbol and a Zipf tail over a permuted alphabet, then a one-symbol block"""
    rng = np.random.default_rng(seed)
    blocks = []
    for b in range(n_blocks):
        p = 1.0 / np.arange(1, 257) ** (0.6 + 0.2 * (b % 5))
        p[0] = p[1:].sum() * (2 + 3 * b)
        blocks.append(rng.permutation(256).astype(np.uint8)[rng.choice(256, block_size, p=p / p.sum())])
    if n_blocks > 1:
        blocks[-1][:] = 0x41
    return np.concatenate(blocks)


def oracle_blocks_encode(oracle_lib, ocoder, sb, data, n_blocks, block_size, chunk):
    """Per-block models and encodes by the oracle, directories rebased: what rb200_blocks_coder_model_encode returns."""
    freqs, parts, offs, base = [], [], [], 0
    for b in range(n_blocks):
        blk = data[b * block_size:(b + 1) * block_size]
        f, c = oracle_lib.model(blk, sb)
        ob, oo = oracle_lib.chunked_encode(ocoder, blk, f, c, chunk, scale_bits=sb)
        freqs.append(f)
        parts.append(ob)
        offs.append(oo[:-1] + base)
        base += ob.size
    return (np.stack(freqs).astype(np.uint16), np.concatenate(offs + [[base]]).astype(np.uint64),
            np.concatenate(parts).astype(np.uint8))


def py_pack(coder, sb, n_blocks, block_size, chunk, freqs, offsets, blob, flags):
    """The version 3 layout, from its description alone."""
    n = n_blocks * block_size
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 3, coder, sb, 32, chunk, n, n // chunk, blob.size, flags, 0, 0, block_size, n_blocks, 0)
    model = np.asarray(freqs, "<u2").tobytes()
    directory = np.asarray(offsets, "<u8").tobytes()
    meta = zlib.crc32(hdr + model + directory)
    blob_crc = zlib.crc32(blob.tobytes()) if flags & CRC_BLOB else 0
    body = hdr[:44] + struct.pack("<II", meta, blob_crc) + hdr[52:] + model + directory
    body += b"\0" * (-len(body) % 16)
    return np.frombuffer(body + blob.tobytes(), np.uint8).copy()


def reseal(buf):
    """Recompute meta_crc after editing fields, so that the checks behind the checksum are what rejects the container."""
    n_chunks, = struct.unpack_from("<Q", buf, 24)
    n_blocks, = struct.unpack_from("<I", buf, 56)
    hdr = bytearray(buf[:64].tobytes())
    hdr[44:52] = b"\0" * 8
    end = 64 + 512 * n_blocks + 8 * (n_chunks + 1)
    if end > buf.size:
        return buf
    struct.pack_into("<I", buf, 44, zlib.crc32(bytes(hdr) + buf[64:end].tobytes()))
    return buf


def oracle_decode_blocks(oracle_lib, ocoder, meta, freqs, offsets, blob):
    per = meta["block_size"] // meta["chunk_syms"]
    out = []
    for b in range(meta["n_blocks"]):
        f = freqs[b].astype(np.uint32)
        c = np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)
        lo, hi = int(offsets[b * per]) & ~15, int(offsets[(b + 1) * per])
        oo = (offsets[b * per:(b + 1) * per + 1] - lo).astype(np.uint64)
        out.append(oracle_lib.chunked_decode(ocoder, blob[lo:hi], oo, meta["block_size"], f, c, meta["chunk_syms"],
                                             scale_bits=meta["scale_bits"]))
    return np.concatenate(out)


def rejected(opener, buf, code=-4):
    with pytest.raises(rb.RansError) as ei:
        opener(buf)
    assert ei.value.code == code


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("coder,ocoder", CODERS)
@pytest.mark.parametrize("sb", [8, 14, 15])
def test_coder_pack_equals_independent_packer_and_opens(oracle_lib, coder, ocoder, sb, flags):
    for i, (nb, bs, ch) in enumerate(GEOMETRIES):
        data = block_data(nb, bs, 50 + i)
        freqs, offs, blob = oracle_blocks_encode(oracle_lib, ocoder, sb, data, nb, bs, ch)
        assert (freqs.astype(np.uint32).sum(axis=1) == 1 << sb).all()
        buf = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, freqs, offs, blob, flags)
        want = py_pack(coder, sb, nb, bs, ch, freqs, offs, blob, flags)
        assert buf.size == want.size and np.array_equal(buf, want), (nb, bs, ch)
        assert buf.size == int(rb.load().dll.rb200_container_blocks_size(nb, offs.size - 1, blob.size))
        meta, f2, o2, b2 = api.container_blocks_coder_open(buf)
        assert meta == {"coder": coder, "scale_bits": sb, "n_blocks": nb, "block_size": bs, "chunk_syms": ch, "flags": flags,
                        "n_symbols": nb * bs, "n_chunks": offs.size - 1, "blob_bytes": blob.size}
        assert np.array_equal(f2, freqs) and np.array_equal(o2, offs) and np.array_equal(b2, blob)
        assert np.array_equal(oracle_decode_blocks(oracle_lib, ocoder, meta, f2, o2, b2), data), (nb, bs, ch)


@pytest.fixture(scope="module")
def base(oracle_lib):
    """byte coder at 14: 3 blocks of 16 KiB in chunks of 4096, 12 chunks, directory at 64 + 1536"""
    nb, bs, ch, sb = 3, 16384, 4096, 14
    data = block_data(nb, bs, 7)
    freqs, offs, blob = oracle_blocks_encode(oracle_lib, orc.CODER_BYTE, sb, data, nb, bs, ch)
    return nb, bs, ch, sb, freqs, offs, blob


def test_coder_open_rejects_each_rule(base):
    nb, bs, ch, sb, freqs, offs, blob = base
    dir_off = 64 + 512 * nb
    good = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, 0)
    assert api.container_blocks_coder_open(reseal(good.copy()))[0]["n_symbols"] == nb * bs     # reseal reproduces the CRC
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
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_coder_open(reseal(bad))
        assert ei.value.code == -4, name
    for flags in (0, CRC_BLOB):                                   # CRC flips in every section, truncations
        g = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, flags)
        for pos in (5, 6, 7, 53, 70, 64 + 512 * 2 + 3, dir_off + 9) + ((g.size - 7,) if flags else ()):
            bad = g.copy()
            bad[pos] ^= 0x40
            rejected(api.container_blocks_coder_open, bad)
        for cut in list(range(0, dir_off + 8 * offs.size + 16, 13)) + [g.size - 16, g.size - 1]:
            rejected(api.container_blocks_coder_open, g[:cut].copy())
    crc = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, CRC_BLOB)   # a blob CRC that does not match
    struct.pack_into("<I", crc, 48, struct.unpack_from("<I", crc, 48)[0] ^ 1)
    rejected(api.container_blocks_coder_open, crc)


def test_versions_reject_each_other(oracle_lib, gen, base):
    nb, bs, ch, sb, freqs, offs, blob = base
    data = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(data, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data, f, c, 4096)
    wdata = np.concatenate([gen("zipf", bs, 11 + b) for b in range(nb)])
    wf = np.stack([oracle_lib.model(wdata[b * bs:(b + 1) * bs], 12)[0] for b in range(nb)]).astype(np.uint16)
    wparts, woffs, wbase = [], [], 0
    for b in range(nb):
        fb = wf[b].astype(np.uint32)
        wb, wo = oracle_lib.chunked_encode(orc.CODER_WORD, wdata[b * bs:(b + 1) * bs], fb, np.concatenate([[0], np.cumsum(fb)]).astype(np.uint32),
                                           ch)
        wparts.append(wb)
        woffs.append(wo[:-1] + wbase)
        wbase += wb.size
    woffs = np.concatenate(woffs + [[wbase]]).astype(np.uint64)
    wblob = np.concatenate(wparts)
    for flags in (0, CRC_BLOB):
        v1 = api.container_pack(rb.CODER_WORD, 12, 4096, data.size, f, oo, ob, flags)
        v2 = api.container_blocks_pack(nb, bs, ch, wf, woffs, wblob, flags)
        v3 = api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, offs, blob, flags)
        api.container_open(v1)
        api.container_blocks_open(v2)
        api.container_blocks_coder_open(v3)
        for opener, others in ((api.container_open, (v2, v3)), (api.container_blocks_open, (v1, v3)),
                               (api.container_blocks_coder_open, (v1, v2))):
            for buf in others:
                rejected(opener, buf)
        # a version 3 container relabelled as version 2 (CRC resealed) is still refused: byte coder, 2^14 totals
        relabelled = v3.copy()
        struct.pack_into("<H", relabelled, 4, 2)
        rejected(api.container_blocks_open, reseal(relabelled))


def test_coder_pack_refuses_what_open_rejects(base):
    nb, bs, ch, sb, freqs, offs, blob = base
    bad = freqs.copy()
    bad[2][int(np.flatnonzero(bad[2])[0])] -= 1                        # block 2 sums to 2^14 - 1
    with pytest.raises(rb.RansError) as ei:
        api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, bad, offs, blob, 0)
    assert ei.value.code == -2
    with pytest.raises(rb.RansError) as ei:                             # the right total for another scale_bits
        api.container_blocks_coder_pack(rb.CODER_BYTE, 13, nb, bs, ch, freqs, offs, blob, 0)
    assert ei.value.code == -2
    lib = rb.load().dll
    out = np.zeros(1 << 20, np.uint8)
    args = (freqs.ctypes.data, offs.ctypes.data, blob.ctypes.data, blob.size, 0, out.ctypes.data, out.size, None)
    for coder, s in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 14), (4, 14), (-1, 14), (rb.CODER_BYTE, 7), (rb.CODER_BYTE, 16),
                     (rb.CODER_RANS64, 16)):
        assert lib.rb200_container_blocks_coder_pack(coder, s, nb, bs, ch, *args) == -1, (coder, s)
    for g in ((0, bs, ch), (nb, bs, 3000), (nb, 33 * 512, 512), (nb, bs, 16), (nb, 0, ch)):
        assert lib.rb200_container_blocks_coder_pack(rb.CODER_BYTE, sb, *g, *args) == -1, g
    for o, b in ((offs, blob[:-16]), (offs, np.concatenate([blob, np.zeros(16, np.uint8)]))):   # directory and blob disagree
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, freqs, o, b, 0)
        assert ei.value.code == -1
    assert lib.rb200_container_blocks_coder_pack(rb.CODER_BYTE, sb, nb, bs, ch, *args[:5], out.ctypes.data, 100, None) == -3
