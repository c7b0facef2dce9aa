"""The per-block container (version 2) on the host, no GPU needed: rb200_container_blocks_pack against an independent
packer written from the format (struct + zlib), rb200_container_blocks_open of it decoding block by block through the
oracle, and every rejection open makes -- bit flips, truncations and each header field edited under a valid CRC."""
import struct
import zlib

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

MAGIC = 0x43324252
CRC_BLOB = api.CONTAINER_CRC_BLOB
# (n_blocks, block_size, chunk_syms): one block; the bench's 64 KiB / 8192; 4 KiB / 4096; 32 chunks per block;
# 17 chunks per block
GEOMETRIES = [(1, 65536, 8192), (3, 65536, 8192), (5, 4096, 4096), (3, 65536, 2048), (4, 17 * 1024, 1024)]


def block_data(n_blocks, block_size, seed):
    """Zipf-like bytes with a different exponent and a permuted alphabet per block: per-block models differ."""
    rng = np.random.default_rng(seed)
    blocks = []
    for b in range(n_blocks):
        p = 1.0 / np.arange(1, 257) ** (0.6 + 0.1 * (b % 9))
        blocks.append(rng.permutation(256).astype(np.uint8)[rng.choice(256, block_size, p=p / p.sum())])
    return np.concatenate(blocks)


def oracle_blocks_encode(oracle_lib, data, n_blocks, block_size, chunk):
    """Per-block models and encodes by the oracle, directories rebased: what rb200_blocks_model_encode returns."""
    freqs, parts, offs, base = [], [], [], 0
    for b in range(n_blocks):
        f, c = oracle_lib.model(data[b * block_size:(b + 1) * block_size], 12)
        ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data[b * block_size:(b + 1) * block_size], f, c, chunk)
        freqs.append(f)
        parts.append(ob)
        offs.append(oo[:-1] + base)
        base += ob.size
    return (np.stack(freqs).astype(np.uint16), np.concatenate(offs + [[base]]).astype(np.uint64),
            np.concatenate(parts).astype(np.uint8))


def py_pack(n_blocks, block_size, chunk, freqs, offsets, blob, flags):
    """The version 2 layout, from its description alone."""
    n = n_blocks * block_size
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 2, 0, 12, 32, chunk, n, n // chunk, blob.size, flags, 0, 0, block_size, n_blocks, 0)
    model = np.asarray(freqs, "<u2").tobytes()
    directory = np.asarray(offsets, "<u8").tobytes()
    meta = zlib.crc32(hdr + model + directory)
    blob_crc = zlib.crc32(blob.tobytes()) if flags & CRC_BLOB else 0
    body = hdr[:44] + struct.pack("<II", meta, blob_crc) + hdr[52:] + model + directory
    body += b"\0" * (-len(body) % 16)
    return np.frombuffer(body + blob.tobytes(), np.uint8).copy()


def reseal(buf):
    """Recompute meta_crc after editing header / model / directory fields (layout from the edited header), so that the
    checks behind the checksum are what rejects the container."""
    n_chunks, = struct.unpack_from("<Q", buf, 24)
    n_blocks, = struct.unpack_from("<I", buf, 56)
    hdr = bytearray(buf[:64].tobytes())
    hdr[44:52] = b"\0" * 8
    end = 64 + 512 * n_blocks + 8 * (n_chunks + 1)
    if end > buf.size:
        return buf
    struct.pack_into("<I", buf, 44, zlib.crc32(bytes(hdr) + buf[64:end].tobytes()))
    return buf


def oracle_decode_blocks(oracle_lib, meta, freqs, offsets, blob):
    """Decode every block through the oracle from its row of block_freqs and its slice of directory and blob."""
    per = meta["block_size"] // meta["chunk_syms"]
    out = []
    for b in range(meta["n_blocks"]):
        f = freqs[b].astype(np.uint32)
        c = np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)
        lo, hi = int(offsets[b * per]) & ~15, int(offsets[(b + 1) * per])
        oo = (offsets[b * per:(b + 1) * per + 1] - lo).astype(np.uint64)
        out.append(oracle_lib.chunked_decode(orc.CODER_WORD, blob[lo:hi], oo, meta["block_size"], f, c, meta["chunk_syms"]))
    return np.concatenate(out)


def rejected(buf, code=-4):
    with pytest.raises(rb.RansError) as ei:
        api.container_blocks_open(buf)
    assert ei.value.code == code


def single_symbol_data():
    """two 4 KiB blocks: the first holds one symbol only (a frequency of 4096)"""
    rng = np.random.default_rng(3)
    return np.concatenate([np.full(4096, 0x41, np.uint8), rng.integers(0, 256, 4096, dtype=np.uint8)])


def cases():
    for i, (nb, bs, ch) in enumerate(GEOMETRIES):
        yield nb, bs, ch, block_data(nb, bs, 100 + i)
    yield 2, 4096, 1024, single_symbol_data()


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
def test_blocks_pack_equals_independent_packer_and_opens(oracle_lib, flags):
    for nb, bs, ch, data in cases():
        freqs, offs, blob = oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
        buf = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
        want = py_pack(nb, bs, ch, freqs, offs, blob, flags)
        assert buf.size == want.size and np.array_equal(buf, want), (nb, bs, ch, flags)
        assert buf.size == int(rb.load().dll.rb200_container_blocks_size(nb, offs.size - 1, blob.size))
        meta, f2, o2, b2 = api.container_blocks_open(buf)
        assert meta == {"n_blocks": nb, "block_size": bs, "chunk_syms": ch, "flags": flags, "n_symbols": nb * bs,
                        "n_chunks": offs.size - 1, "blob_bytes": blob.size}
        assert np.array_equal(f2, freqs) and np.array_equal(o2, offs) and np.array_equal(b2, blob)
        assert np.array_equal(oracle_decode_blocks(oracle_lib, meta, f2, o2, b2), data), (nb, bs, ch)


@pytest.fixture(scope="module")
def base(oracle_lib):
    """3 blocks of 16 KiB in chunks of 4096: 12 chunks, directory at 64 + 1536"""
    nb, bs, ch = 3, 16384, 4096
    data = block_data(nb, bs, 7)
    freqs, offs, blob = oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
    return nb, bs, ch, freqs, offs, blob


def rejected_containers(nb, bs, ch, freqs, offs, blob):
    """(name, container) pairs open must reject: bit flips in every section, truncations through the prefix, and every
    header rule broken by an edit under a valid meta CRC."""
    dir_off = 64 + 512 * nb
    out = []
    for flags in (0, CRC_BLOB):
        good = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
        for pos in (5, 53, 57, 70, 64 + 512 * 2 + 3, dir_off + 9) + ((good.size - 7,) if flags else ()):
            bad = good.copy()
            bad[pos] ^= 0x40
            out.append((f"flip at {pos}, flags {flags}", bad))
        for cut in list(range(0, dir_off + 8 * offs.size + 16, 7)) + [good.size - 16, good.size - 1]:
            out.append((f"cut at {cut}, flags {flags}", good[:cut].copy()))
    good = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, 0)
    nz = int(np.flatnonzero(freqs[1])[0])
    edits = {
        "magic": [(0, "<I", 0x12345678)], "version 1": [(4, "<H", 1)], "version 3": [(4, "<H", 3)],
        "coder byte": [(6, "<B", 1)], "scale_bits 14": [(7, "<B", 14)], "lanes 64": [(8, "<I", 64)],
        "chunk_syms 0": [(12, "<I", 0)], "chunk_syms 16 (below the kernels' minimum)": [(12, "<I", 16), (24, "<Q", nb * bs // 16)],
        "block_size % chunk_syms != 0": [(52, "<I", 6144), (56, "<I", 8)],
        "33 chunks per block": [(12, "<I", 512), (52, "<I", 33 * 512), (16, "<Q", nb * 33 * 512), (24, "<Q", nb * 33)],
        "block_size 0": [(52, "<I", 0)], "n_blocks 0": [(56, "<I", 0)], "n_blocks huge": [(56, "<I", 2 ** 32 - 1)],
        "n_symbols != n_blocks * block_size": [(16, "<Q", nb * bs + ch)], "n_symbols huge": [(16, "<Q", 2 ** 64 - 1)],
        "n_chunks + 1": [(24, "<Q", offs.size)], "n_chunks 2^31": [(24, "<Q", 2 ** 31)], "n_chunks huge": [(24, "<Q", 2 ** 40)],
        "n_chunks 2^31, consistent otherwise": [(12, "<I", 1024), (52, "<I", 32768), (56, "<I", 2 ** 26), (16, "<Q", 2 ** 41),
                                                (24, "<Q", 2 ** 31)],
        "blob_bytes odd": [(32, "<Q", blob.size + 8)], "blob_bytes beyond the buffer": [(32, "<Q", blob.size + 4096)],
        "blob_bytes short": [(32, "<Q", blob.size - 16)],
        "reserved nonzero": [(60, "<I", 1)], "unknown flag bit": [(40, "<I", 2)], "unknown flag bit with CRC_BLOB": [(40, "<I", 3)],
        "block 1 sums to 4095": [(64 + 512 + 2 * nz, "<H", int(freqs[1][nz]) - 1)],
        "block 2 sums to 4097": [(64 + 1024 + 2 * nz, "<H", int(freqs[2][nz]) + 1)],
        "first stream starts beyond the first vector": [(dir_off, "<Q", 32)],
        "directory not monotone": [(dir_off + 8, "<Q", int(offs[2]) + 16)],
        "last entry != blob size": [(dir_off + 8 * (offs.size - 1), "<Q", int(offs[-1]) - 16)],
    }
    for name, fields in edits.items():
        bad = good.copy()
        for off, fmt, val in fields:
            struct.pack_into(fmt, bad, off, val)
        out.append((name, reseal(bad)))
    crc = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, CRC_BLOB)      # a blob CRC that does not match
    struct.pack_into("<I", crc, 48, struct.unpack_from("<I", crc, 48)[0] ^ 1)
    out.append(("blob crc", crc))
    return out


def test_blocks_open_rejects_flips_truncations_and_each_rule(base):
    nb, bs, ch, freqs, offs, blob = base
    good = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, 0)
    assert api.container_blocks_open(reseal(good.copy()))[0]["n_symbols"] == nb * bs        # reseal reproduces the library's CRC
    for name, bad in rejected_containers(*base):
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_open(bad)
        assert ei.value.code == -4, name
    # random garbage with a valid magic and version never gets through either
    rng = np.random.default_rng(0)
    for _ in range(200):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        struct.pack_into("<IH", junk, 0, MAGIC, 2)
        rejected(reseal(junk))


def test_blocks_and_single_model_containers_reject_each_other(oracle_lib, gen, base):
    nb, bs, ch, freqs, offs, blob = base
    data = gen("zipf", 30000, 4)
    f, c = oracle_lib.model(data, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data, f, c, 4096)
    for flags in (0, CRC_BLOB):
        v1 = api.container_pack(rb.CODER_WORD, 12, 4096, data.size, f, oo, ob, flags)
        v2 = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
        api.container_open(v1)
        api.container_blocks_open(v2)
        rejected(v1)
        with pytest.raises(rb.RansError) as ei:
            api.container_open(v2)
        assert ei.value.code == -4


def test_blocks_pack_refuses_what_open_rejects(base):
    nb, bs, ch, freqs, offs, blob = base
    bad = freqs.copy()
    bad[2][int(np.flatnonzero(bad[2])[0])] -= 1                        # block 2 sums to 4095
    with pytest.raises(rb.RansError) as ei:
        api.container_blocks_pack(nb, bs, ch, bad, offs, blob, 0)
    assert ei.value.code == -2
    for o, b in ((offs, blob[:-16]), (offs, np.concatenate([blob, np.zeros(16, np.uint8)]))):   # directory and blob disagree
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_pack(nb, bs, ch, freqs, o, b, 0)
        assert ei.value.code == -1
    lib = rb.load().dll
    out = np.zeros(1 << 20, np.uint8)
    for g in ((0, bs, ch), (nb, bs, 3000), (nb, 33 * 512, 512), (nb, bs, 16), (nb, 0, ch)):     # geometry
        assert lib.rb200_container_blocks_pack(*g, freqs.ctypes.data, offs.ctypes.data, blob.ctypes.data, blob.size, 0, out.ctypes.data,
                                               out.size, None) == -1, g
    assert lib.rb200_container_blocks_pack(nb, bs, ch, freqs.ctypes.data, offs.ctypes.data, blob.ctypes.data, blob.size, 0,
                                           out.ctypes.data, 100, None) == -3
