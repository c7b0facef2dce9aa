"""Version 5 per-block containers (stored blocks) on the host: rb200_container_blocks_stored_pack, _open and _bound.

- pack equals a packer written from the layout's description, and open returns what went in, over the oracle's
  per-block streams of all four coders with chosen blocks replaced by stored ones (the store rule's choice, none, one,
  all), and every stored chunk holds its symbols and every coded block decodes.
- open rejects each rule broken on its own: a row neither zero nor summing, a stored chunk with a wrong step or nonzero
  padding, a bad pair, both CRCs, the version; versions 1-4 and 5 reject each other.
- pack's error codes, and the bound.  No GPU needed."""
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
import test_blocks_coder_choice as bcc  # noqa: E402
import test_container_blocks as cb2  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
OCODER = {WORD: orc.CODER_WORD, BYTE: orc.CODER_BYTE, ALIAS: orc.CODER_ALIAS, RANS64: orc.CODER_RANS64}
MAGIC = 0x43324252
CRC_BLOB = 1
PAIRS = [(WORD, 12), (BYTE, 14), (RANS64, 10), (ALIAS, 14)]
GEOMETRIES = [(3, 65536, 8192), (4, 9000, 1000), (1, 32, 32), (5, 4096, 4096)]


def r16(x):
    return (x + 15) & ~15


def mixed_data(nb, bs, seed):
    """uniform blocks (stored by the rule) between Zipf and skewed ones (coded)"""
    kinds = ["uniform", "zipf", "skewed"]
    return np.concatenate([bcc.block_data(kinds[b % 3], 1, bs, seed + b) for b in range(nb)])


def oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch):
    """(block_freqs, offsets, blob) of the per-block calls for (coder, sb), by the oracle"""
    if coder == WORD:
        return cb2.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
    return cc.oracle_blocks_encode(oracle_lib, OCODER[coder], sb, data, nb, bs, ch)


def streams(offsets, blob):
    """every chunk's stream: blob[offsets[c], offsets[c + 1] & ~15)"""
    return [blob[int(offsets[c]):int(offsets[c + 1]) & ~15] for c in range(offsets.size - 1)]


def layout(parts):
    """directory and blob of streams placed by the rule of every container: each ends on a multiple of 16 and takes its
    size rounded up to 16, zero bytes in front"""
    offs, out, end = [], [], 0
    for s in parts:
        out += [np.zeros(r16(s.size) - s.size, np.uint8), s]
        end += r16(s.size)
        offs.append(end - s.size)
    return np.array(offs + [end], np.uint64), np.concatenate(out).astype(np.uint8)


def stored_blocks(offsets, blob, nb, bs, ch):
    """the store rule: a block whose chunks take more than per_block x round16(chunk_syms) bytes of blob"""
    per = bs // ch
    size = [r16(s.size) for s in streams(offsets, blob)]
    return [b for b in range(nb) if sum(size[b * per:(b + 1) * per]) > per * r16(ch)]


def apply_store(freqs, offsets, blob, data, nb, bs, ch, which=None):
    """(block_freqs, offsets, blob, stored) of version 5 from version 2-4 streams: the blocks in `which` (default: the
    store rule's) stored, each chunk its symbols and zero padding, the row zero"""
    per = bs // ch
    which = stored_blocks(offsets, blob, nb, bs, ch) if which is None else sorted(which)
    parts = streams(offsets, blob)
    freqs = np.array(freqs, np.uint16, copy=True)
    for b in which:
        freqs[b] = 0
        for c in range(b * per, (b + 1) * per):
            parts[c] = np.concatenate([data[c * ch:(c + 1) * ch], np.zeros(r16(ch) - ch, np.uint8)])
    offs, out = layout(parts)
    return freqs, offs, out, which


def py_pack(coder, sb, nb, bs, ch, freqs, offsets, blob, flags):
    """the version 5 layout, from its description alone"""
    n = nb * bs
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 5, coder, sb, 32, ch, n, n // ch, blob.size, flags, 0, 0, bs, nb, 0)
    model = np.asarray(freqs, "<u2").tobytes()
    directory = np.asarray(offsets, "<u8").tobytes()
    meta = zlib.crc32(hdr + model + directory)
    blob_crc = zlib.crc32(blob.tobytes()) if flags & CRC_BLOB else 0
    body = hdr[:44] + struct.pack("<II", meta, blob_crc) + hdr[52:] + model + directory
    body += b"\0" * (-len(body) % 16)
    return np.frombuffer(body + blob.tobytes(), np.uint8).copy()


def decode_host(oracle_lib, coder, sb, meta, freqs, offsets, blob, nb, bs, ch):
    """every block: a stored one's chunks from the blob, a coded one by the oracle"""
    per = bs // ch
    out = []
    for b in range(nb):
        if not freqs[b].any():
            out += [blob[int(offsets[c]):int(offsets[c]) + ch] for c in range(b * per, (b + 1) * per)]
            continue
        f = freqs[b].astype(np.uint32)
        cum = np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)
        lo, hi = int(offsets[b * per]) & ~15, int(offsets[(b + 1) * per])
        oo = (offsets[b * per:(b + 1) * per + 1] - lo).astype(np.uint64)
        out.append(oracle_lib.chunked_decode(OCODER[coder], blob[lo:hi], oo, bs, f, cum, ch, scale_bits=sb))
    return np.concatenate(out)


def reseal(buf):
    return cc.reseal(buf)


def test_layout_reproduces_the_oracle_blob(oracle_lib):
    nb, bs, ch = 4, 9000, 1000
    data = mixed_data(nb, bs, 3)
    for coder, sb in PAIRS:
        _, offs, blob = oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch)
        o2, b2 = layout(streams(offs, blob))
        assert np.array_equal(o2, offs) and np.array_equal(b2, blob), coder


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("coder,sb", PAIRS)
def test_pack_equals_independent_packer_opens_and_decodes(oracle_lib, coder, sb, flags):
    for gi, (nb, bs, ch) in enumerate(GEOMETRIES):
        data = mixed_data(nb, bs, 20 + gi)
        freqs, offs, blob = oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch)
        for which in (None, [], [nb - 1], list(range(nb))):
            f5, o5, b5, st = apply_store(freqs, offs, blob, data, nb, bs, ch, which)
            case = (coder, sb, nb, bs, ch, which)
            buf = api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, flags)
            assert np.array_equal(buf, py_pack(coder, sb, nb, bs, ch, f5, o5, b5, flags)), case
            assert buf.size <= api.container_blocks_stored_bound(nb, bs, ch) or which is not None, case
            meta, f2, o2, b2 = api.container_blocks_stored_open(buf)
            assert meta == {"coder": coder, "scale_bits": sb, "n_blocks": nb, "block_size": bs, "chunk_syms": ch, "flags": flags,
                            "n_symbols": nb * bs, "n_chunks": o5.size - 1, "blob_bytes": b5.size}, case
            assert np.array_equal(f2, f5) and np.array_equal(o2, o5) and np.array_equal(b2, b5), case
            assert np.array_equal(decode_host(oracle_lib, coder, sb, meta, f2, o2, b2, nb, bs, ch), data), case
        if nb == 3:                                                  # the uniform block 0 is stored, the others are not
            assert stored_blocks(offs, blob, nb, bs, ch) == [0], coder


def test_bound():
    lib = rb.load().dll
    for nb, bs, ch in GEOMETRIES + [(8192, 65536, 8192)]:
        n_chunks = nb * (bs // ch)
        want = ((64 + 512 * nb + 8 * (n_chunks + 1) + 15) & ~15) + n_chunks * r16(ch)
        assert api.container_blocks_stored_bound(nb, bs, ch) == want
    for nb, bs, ch in ((0, 4096, 4096), (1, 4096, 31), (1, 33 * 32, 32), (1, 4000, 3000)):
        assert lib.rb200_container_blocks_stored_bound(nb, bs, ch) == 0


def test_all_stored_container_is_the_bound(oracle_lib):
    nb, bs, ch = 4, 9000, 1000
    data = mixed_data(nb, bs, 5)
    f5, o5, b5, _ = apply_store(*oracle_streams(oracle_lib, BYTE, 12, data, nb, bs, ch), data, nb, bs, ch, range(nb))
    assert api.container_blocks_stored_pack(BYTE, 12, nb, bs, ch, f5, o5, b5).size == api.container_blocks_stored_bound(nb, bs, ch)


@pytest.fixture(scope="module")
def base(oracle_lib):
    """byte coder at 14, 4 blocks of 9000 in chunks of 1000 (8 bytes of padding per stored chunk), block 0 stored"""
    nb, bs, ch, sb = 4, 9000, 1000, 14
    data = mixed_data(nb, bs, 7)
    f5, o5, b5, st = apply_store(*oracle_streams(oracle_lib, BYTE, sb, data, nb, bs, ch), data, nb, bs, ch)
    assert st == [0, 3]
    return nb, bs, ch, sb, f5, o5, b5


def test_open_rejects_each_rule(base):
    nb, bs, ch, sb, f5, o5, b5 = base
    per = bs // ch
    dir_off = 64 + 512 * nb
    boff = (dir_off + 8 * (o5.size) + 15) & ~15
    good = api.container_blocks_stored_pack(BYTE, sb, nb, bs, ch, f5, o5, b5, 0)
    assert api.container_blocks_stored_open(reseal(good.copy()))[0]["n_symbols"] == nb * bs     # reseal reproduces the CRC

    def field(edits):
        bad = good.copy()
        for pos, fmt, v in edits:
            struct.pack_into(fmt, bad, pos, v)
        return reseal(bad)

    cases = {f"version {v}": field([(4, "<H", v)]) for v in (1, 2, 3, 4, 6)}
    cases.update({"coder 4": field([(6, "<B", 4)]), "word at 14": field([(6, "<B", WORD)]), "alias at 16": field([(6, "<B", ALIAS), (7, "<B", 16)]),
                  "byte at 7": field([(7, "<B", 7)]), "rans64 at 16": field([(6, "<B", RANS64), (7, "<B", 16)])})
    nz = int(np.flatnonzero(f5[1])[0])
    cases["coded row off by one"] = field([(64 + 512 + 2 * nz, "<H", int(f5[1][nz]) - 1)])
    cases["stored row with a nonzero"] = field([(64 + 2 * 7, "<H", 1)])
    c = 3 * per + 2                                                   # a chunk of stored block 3, after a stored chunk
    cases["stored step short"] = field([(dir_off + 8 * c, "<Q", int(o5[c]) + 16)])
    c = per                                                          # block 1's first chunk: block 0's last one is stored
    cases["stored step long"] = field([(dir_off + 8 * c, "<Q", int(o5[c]) + 16)])
    bad = good.copy()
    bad[boff + int(o5[3 * per + 4]) + ch + 3] = 1                    # padding of a stored chunk (not under a CRC)
    cases["nonzero padding"] = bad
    bad = good.copy()
    bad[64 + 512 + 2 * nz] ^= 1
    cases["meta CRC"] = bad
    crc = api.container_blocks_stored_pack(BYTE, sb, nb, bs, ch, f5, o5, b5, CRC_BLOB)
    bad = crc.copy()
    bad[boff + int(o5[0]) + 5] ^= 1                                  # a stored symbol: only the blob CRC sees it
    cases["blob CRC"] = bad
    for name, bad in cases.items():
        with pytest.raises(rb.RansError) as ei:
            api.container_blocks_stored_open(bad)
        assert ei.value.code == -4, name
    # the same edit without breaking the rule is accepted: the padding check reads nothing but padding
    ok = good.copy()
    ok[boff + int(o5[3 * per + 4]) + ch - 1] ^= 1
    assert api.container_blocks_stored_open(ok)[0]["blob_bytes"] == b5.size


def test_versions_reject_each_other(oracle_lib, base):
    nb, bs, ch, sb, f5, o5, b5 = base
    v5 = api.container_blocks_stored_pack(BYTE, sb, nb, bs, ch, f5, o5, b5, 0)
    for opener in (api.container_open, api.container_blocks_open, api.container_blocks_coder_open, api.container_blocks_alias_open):
        cc.rejected(opener, v5)
    data = mixed_data(nb, bs, 9)
    others = [api.container_blocks_pack(nb, bs, ch, *oracle_streams(oracle_lib, WORD, 12, data, nb, bs, ch)),
              api.container_blocks_coder_pack(BYTE, sb, nb, bs, ch, *oracle_streams(oracle_lib, BYTE, sb, data, nb, bs, ch)),
              api.container_blocks_alias_pack(14, nb, bs, ch, *oracle_streams(oracle_lib, ALIAS, 14, data, nb, bs, ch))]
    f, cum = oracle_lib.model(data, 12)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, data, f, cum, 4096)
    others.append(api.container_pack(WORD, 12, 4096, data.size, f, oo, ob))
    for buf in others:
        cc.rejected(api.container_blocks_stored_open, buf)
        relabelled = buf.copy()
        struct.pack_into("<H", relabelled, 4, 5)
        cc.rejected(api.container_blocks_stored_open, relabelled)    # the CRC covers the version field


def test_pack_error_codes(base):
    nb, bs, ch, sb, f5, o5, b5 = base
    lib = rb.load().dll
    out = np.zeros(api.container_blocks_stored_bound(nb, bs, ch) + 64, np.uint8)
    size = C.c_size_t(0)

    def pack(coder=BYTE, s=sb, n_blocks=nb, block_size=bs, chunk=ch, freqs=f5, offs=o5, blob=b5, blob_bytes=None, cap=out.size):
        return lib.rb200_container_blocks_stored_pack(coder, s, n_blocks, block_size, chunk, freqs.ctypes.data, offs.ctypes.data,
                                                      blob.ctypes.data, blob.size if blob_bytes is None else blob_bytes, 0,
                                                      out.ctypes.data, cap, C.byref(size))
    assert pack() == 0 and size.value == boff_plus(nb, o5, b5)
    for kw in ({"coder": 4}, {"s": 16}, {"s": 7}, {"coder": WORD, "s": 14}, {"n_blocks": 0}, {"chunk": 31}, {"chunk": 1024},
               {"blob_bytes": b5.size - 16}):
        assert pack(**kw) == -1, kw
    per = bs // ch
    offs = o5.copy()
    offs[3 * per + 2] += 16                                          # a stored chunk's step
    assert pack(offs=offs) == -1
    blob = b5.copy()
    blob[int(o5[3 * per + 1]) + ch] = 9                              # a stored chunk's padding
    assert pack(blob=blob) == -1
    freqs = f5.copy()
    freqs[1][int(np.flatnonzero(freqs[1])[0])] -= 1
    assert pack(freqs=freqs) == -2
    freqs = f5.copy()
    freqs[0][3] = 1                                                  # a stored block's row, neither zero nor summing
    assert pack(freqs=freqs) == -2
    assert pack(s=13) == -2                                          # the rows sum to 2^14
    assert pack(cap=boff_plus(nb, o5, b5) - 1) == -3


def boff_plus(nb, offs, blob):
    return ((64 + 512 * nb + 8 * offs.size + 15) & ~15) + blob.size
