"""Version 7 byte-plane containers on the host: rb200_container_planes_pack, _open and _bound.

- The bound is 64 + 16 w + w * rb200_container_stored_bound(n / w, chunk_syms), and 0 for what the encode refuses.
- pack equals a packer written from the layout's description, for w = 2, 4 and 8, over planes packed with
  container_stored_pack from the oracle's streams (planes with stored chunks, coded ones, ragged last chunks); open
  returns views that container_stored_open accepts and whose decoded planes interleave back into the input.
- open rejects each rule broken on its own (the CRC resealed, so that only that rule fails), a flipped table byte, a
  truncated buffer and a corrupt plane; pack refuses planes that disagree.  Every other open rejects version 7, and
  the planes open rejects versions 1-6.  No GPU needed."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_stored as cs  # noqa: E402

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
MAGIC = 0x43324252
CRC_BLOB = 1
E_ARG, E_SPACE, E_STREAM = -1, -3, -4
PAIR_OF_PLANE = [(BYTE, 14), (WORD, 12), (RANS64, 11), (ALIAS, 12)]


def elements(kind, count, seed):
    """count elements as their little-endian bytes: bf16 / fp16 / fp32 / fp64 of N(0, 0.02), int32 small integers"""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 0.02, count)
    if kind == "bf16":
        return (x.astype(np.float32).view(np.uint32) >> 16).astype("<u2").view(np.uint8)
    if kind == "fp16":
        return x.astype("<f2").view(np.uint8)
    if kind == "fp32":
        return x.astype("<f4").view(np.uint8)
    if kind == "fp64":
        return x.astype(np.float32).astype("<f8").view(np.uint8)
    if kind == "int32":
        return rng.integers(-40, 40, count).astype("<i4").view(np.uint8)
    raise ValueError(kind)


def split(data, w):
    return [np.ascontiguousarray(data.reshape(-1, w)[:, p]) for p in range(w)]


def v6_plane(oracle_lib, plane, ch, flags, p):
    """plane p as a version 6 container: the oracle's streams for a pair, the store rule applied in Python"""
    coder, sb = PAIR_OF_PLANE[p % len(PAIR_OF_PLANE)]
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, plane, ch)
    bits, o6, b6, st = cs.apply_store(plane, ch, offs, blob)
    return api.container_stored_pack(coder, sb, ch, plane.size, freqs, bits, o6, b6, flags), (coder, sb, freqs, cum, bits, o6, b6, st)


def py_pack7(planes, w, ch, flags, n=None):
    """the version 7 layout, from its description alone"""
    m = int(planes[0][16:24].view(np.uint64)[0])
    n = m * w if n is None else n
    end, table = 64 + 16 * w, []
    for p in planes:
        table.append(struct.pack("<QQ", end, p.size))
        end += p.size
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 7, 0, 0, 32, ch, n, 0, end - 64 - 16 * w, flags, 0, 0, w, w, 0)
    return reseal(np.frombuffer(hdr + b"".join(table) + b"".join(p.tobytes() for p in planes), np.uint8).copy())


def reseal(buf, w=None):
    """recompute meta_crc over the header (crc fields zero) and the table of w entries (the header's w by default)"""
    buf = buf.copy()
    w = int(buf[52:56].view(np.uint32)[0]) if w is None else w
    buf[44:48] = 0
    buf[44:48] = np.frombuffer(struct.pack("<I", zlib.crc32(buf[:min(64 + 16 * w, buf.size)].tobytes())), np.uint8)
    return buf


def set_u32(buf, off, v):
    buf[off:off + 4] = np.frombuffer(struct.pack("<I", v), np.uint8)


def set_u64(buf, off, v):
    buf[off:off + 8] = np.frombuffer(struct.pack("<Q", v), np.uint64).view(np.uint8)


def u64(buf, off):
    return int(buf[off:off + 8].view(np.uint64)[0])


def container(oracle_lib, kind, w, ch, count, flags=0, seed=0):
    data = elements(kind, count, seed)
    planes = [v6_plane(oracle_lib, pl, ch, flags, p)[0] for p, pl in enumerate(split(data, w))]
    return data, planes, api.container_planes_pack(planes)


@pytest.mark.parametrize("w", [2, 4, 8])
@pytest.mark.parametrize("ch", [32, 8192])
def test_bound(w, ch):
    for m in (1, 31, ch, ch + 17, 10 * ch + 5):
        assert api.container_planes_bound(m * w, w, ch) == 64 + 16 * w + w * api.container_stored_bound(m, ch)
    assert api.container_planes_bound(0, w, ch) == 0
    assert api.container_planes_bound(w * 100 + 1, w, ch) == 0                     # not a multiple of w
    assert api.container_planes_bound(w << 32, w, ch) == 0                          # n / w = 2^32
    assert api.container_planes_bound(w * ((1 << 32) - 1), w, ch) == 64 + 16 * w + w * api.container_stored_bound((1 << 32) - 1, ch)
    for bad in (0, 1, 3, 16):
        assert api.container_planes_bound(bad * 64, bad, ch) == 0
    assert api.container_planes_bound(w * 64, w, 16) == 0                           # chunk_syms below 32


CASES = [("bf16", 2, 32, 5 * 32 + 17), ("fp16", 2, 64, 7 * 64), ("fp32", 4, 32, 9 * 32 + 3), ("int32", 4, 48, 200),
         ("fp64", 8, 32, 6 * 32 + 31), ("fp64", 8, 8192, 100)]


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("kind,w,ch,count", CASES)
def test_pack_and_open_round_trip(oracle_lib, kind, w, ch, count, flags):
    data = elements(kind, count, 7)
    built = [v6_plane(oracle_lib, pl, ch, flags, p) for p, pl in enumerate(split(data, w))]
    planes = [b[0] for b in built]
    buf = api.container_planes_pack(planes)
    assert np.array_equal(buf, py_pack7(planes, w, ch, flags))
    assert buf.size == 64 + 16 * w + sum(p.size for p in planes) <= api.container_planes_bound(data.size, w, ch)
    meta, views = api.container_planes_open(buf)
    assert meta == {"elem_bytes": w, "chunk_syms": ch, "flags": flags, "n": data.size}
    out = np.zeros(data.size, np.uint8)
    for p, (view, (_, (coder, sb, freqs, cum, bits, o6, b6, st))) in enumerate(zip(views, built)):
        assert np.array_equal(view, planes[p])
        info, f, b, o, blob = api.container_stored_open(view)
        assert (info["coder"], info["scale_bits"], info["n_symbols"]) == (coder, sb, count)
        out[p::w] = cs.decode_host(oracle_lib, coder, sb, f, cum, b, o, blob, count, ch)
    assert np.array_equal(out, data)
    if kind in ("bf16", "fp32"):                    # the low mantissa byte is near uniform: stored chunks, ragged last
        assert len(built[0][1][7]) > 0


def test_planes_mix_stored_and_coded(oracle_lib):
    """bf16 at chunks of 4096: the low byte's chunks are stored, the sign/exponent byte's whole chunks coded"""
    data = elements("bf16", 6 * 4096 + 9, 3)
    built = [v6_plane(oracle_lib, pl, 4096, 0, p) for p, pl in enumerate(split(data, 2))]
    n_chunks = 7
    assert len(built[0][1][7]) >= n_chunks // 2 and (n_chunks - 1) in built[0][1][7]
    assert list(built[1][1][7]) == [n_chunks - 1]                       # only the 9-symbol last chunk


@pytest.fixture(scope="module")
def good(oracle_lib):
    """(data, planes, v7 buffer) for fp32 at chunks of 32, ragged"""
    return container(oracle_lib, "fp32", 4, 32, 9 * 32 + 3, seed=11)


def rejected(buf):
    with pytest.raises(rb.RansError) as e:
        api.container_planes_open(buf)
    return e.value.code


def test_open_rejects_each_header_rule(good):
    _, _, buf = good
    assert api.container_planes_open(buf)[0]["elem_bytes"] == 4
    broken = {}
    for name, off, val in (("version 6", 4, 6), ("version 8", 4, 8), ("coder", 6, 1), ("scale_bits", 7, 12), ("lanes", 8, 16)):
        b = buf.copy()
        b[off] = val
        broken[name] = reseal(b)
    for w in (1, 3, 16):
        b = buf.copy()
        set_u32(b, 52, w)
        set_u32(b, 56, w)
        broken[f"w {w}"] = reseal(b, min(w, 8))
    b = buf.copy()
    set_u32(b, 56, 2)                                                   # n_blocks != block_size
    broken["n_blocks"] = reseal(b)
    for name, off in (("n_chunks", 24), ("reserved", 60), ("blob_crc", 48)):
        b = buf.copy()
        b[off] = 1
        broken[name] = reseal(b) if off != 48 else b
    b = buf.copy()
    set_u64(b, 16, u64(buf, 16) + 1)                                    # n not a multiple of w
    broken["n ragged"] = reseal(b)
    b = buf.copy()
    set_u64(b, 16, u64(buf, 16) + 4)                                    # n disagrees with the planes
    broken["n"] = reseal(b)
    b = buf.copy()
    set_u64(b, 32, u64(buf, 32) + 16)                                   # blob_bytes past the buffer
    broken["blob_bytes"] = reseal(b)
    b = buf.copy()
    set_u32(b, 12, 16)                                                  # chunk_syms below 32
    broken["chunk_syms"] = reseal(b)
    for name, b in broken.items():
        assert rejected(b) == E_STREAM, name


def test_open_rejects_each_table_rule(good):
    _, planes, buf = good
    w = 4
    b = buf.copy()
    set_u64(b, 64, u64(buf, 64) + 16)                                   # offset[0] off by 16
    assert rejected(reseal(b)) == E_STREAM
    b = buf.copy()
    set_u64(b, 80, u64(buf, 80) - 16)                                   # plane 1 overlaps plane 0
    assert rejected(reseal(b)) == E_STREAM
    b = buf.copy()
    set_u64(b, 72, u64(buf, 72) - 16)                                   # size[0] short: a gap before plane 1
    assert rejected(reseal(b)) == E_STREAM
    # a real gap: 16 zero bytes between planes 0 and 1, the later offsets and blob_bytes moved to match
    o1 = u64(buf, 80)
    b = np.concatenate([buf[:o1], np.zeros(16, np.uint8), buf[o1:]])
    for p in range(1, w):
        set_u64(b, 64 + 16 * p, u64(buf, 64 + 16 * p) + 16)
    set_u64(b, 32, u64(buf, 32) + 16)
    assert rejected(reseal(b)) == E_STREAM
    # size[0] that does not match plane 0's header: the 16 bytes counted in plane 0
    set_u64(b, 72, u64(buf, 72) + 16)
    for p in range(1, w):
        set_u64(b, 64 + 16 * p, u64(buf, 64 + 16 * p) + 16)
    assert rejected(reseal(b)) == E_STREAM
    b = buf.copy()
    b[64 + 16 * 2 + 3] ^= 0x40                                          # a flipped table byte: meta_crc
    assert rejected(b) == E_STREAM


def test_open_rejects_planes_that_disagree(oracle_lib, good):
    data, planes, buf = good
    w, ch, m = 4, 32, data.size // 4
    pl = split(data, w)
    odd = {
        "n": v6_plane(oracle_lib, pl[1][:m - 3], ch, 0, 1)[0],
        "chunk_syms": v6_plane(oracle_lib, pl[1], 64, 0, 1)[0],
        "flags": v6_plane(oracle_lib, pl[1], ch, CRC_BLOB, 1)[0],
    }
    for name, plane in odd.items():
        mixed = [planes[0], plane, planes[2], planes[3]]
        assert rejected(py_pack7(mixed, w, ch, 0, n=data.size)) == E_STREAM, name
        with pytest.raises(rb.RansError) as e:
            api.container_planes_pack(mixed)
        assert e.value.code == E_ARG, name


def test_open_rejects_truncated_and_corrupt(good):
    _, planes, buf = good
    for size in (0, 63, 64, 64 + 16 * 4 - 1, buf.size - 16, buf.size - 1):
        assert rejected(buf[:size].copy()) == E_STREAM, size
    o1 = u64(buf, 80)
    b = buf.copy()
    b[o1 + 64 + 4] ^= 1                                                 # plane 1's model: its own meta_crc
    assert rejected(b) == E_STREAM


def test_pack_errors(good):
    _, planes, buf = good
    lib = api.load()
    ptrs = (api.C.c_void_p * 4)(*[p.ctypes.data for p in planes])
    sizes = (api.C.c_size_t * 4)(*[p.size for p in planes])
    out = np.zeros(buf.size, np.uint8)
    size = api.C.c_size_t(0)
    assert lib.dll.rb200_container_planes_pack(4, ptrs, sizes, out.ctypes.data, out.size, api.C.byref(size)) == 0
    assert size.value == buf.size and np.array_equal(out, buf)
    assert lib.dll.rb200_container_planes_pack(4, ptrs, sizes, out.ctypes.data, out.size - 1, None) == E_SPACE
    for w in (1, 3, 16):
        assert lib.dll.rb200_container_planes_pack(w, ptrs, sizes, out.ctypes.data, out.size, None) == E_ARG
    sizes[2] = planes[2].size - 16                                      # not the plane's exact size
    assert lib.dll.rb200_container_planes_pack(4, ptrs, sizes, out.ctypes.data, out.size, None) == E_ARG
    sizes[2] = planes[2].size
    assert lib.dll.rb200_container_planes_pack(2, ptrs, sizes, out.ctypes.data, out.size, None) == 0   # 2 planes of 4 agree
    assert lib.dll.rb200_container_planes_pack(4, ptrs, sizes, None, out.size, None) == E_ARG


def test_versions_reject_each_other(oracle_lib, good):
    data, planes, buf = good
    for opener in (api.container_open, api.container_stored_open, api.container_blocks_open, api.container_blocks_stored_open,
                   api.container_blocks_alias_open, api.container_blocks_coder_open):
        with pytest.raises(rb.RansError) as e:
            opener(buf)
        assert e.value.code == E_STREAM, opener.__name__
    assert rejected(planes[0]) == E_STREAM                              # version 6
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, WORD, 12, data, 32)
    assert rejected(api.container_pack(WORD, 12, 32, data.size, freqs, offs, blob)) == E_STREAM   # version 1
    b = buf.copy()
    b[4] = 6                                                            # version 6 with a version 7 body
    assert rejected(reseal(b)) == E_STREAM
