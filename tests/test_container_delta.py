"""Version 8 delta byte-plane containers on the host: rb200_container_delta_pack and _open.

- The transform: numpy's zigzag difference and its inverse round-trip every bit pattern (wraparound, sign changes, NaN
  patterns, integer extremes) at w = 2, 4 and 8, and an unchanged tensor gives d = 0.
- pack equals a packer written from the layout's description (version 7's with version 8 and the base CRC in
  reserved), for w = 2, 4 and 8, over planes of d packed with container_stored_pack from the oracle's streams; open
  returns the base CRC and views whose decoded planes, applied to the base, give the input back.
- open rejects each header and table rule broken on its own (the CRC resealed), and meta_crc covers the base CRC.  The
  version 7 open rejects version 8 and the version 8 open rejects version 7; every other open rejects version 8.  No
  GPU needed."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_planes as cp  # noqa: E402
import test_container_stored as cs  # noqa: E402

MAGIC = 0x43324252
CRC_BLOB = 1
E_ARG, E_SPACE, E_STREAM = -1, -3, -4
UNSIGNED = {2: "<u2", 4: "<u4", 8: "<u8"}
SIGNED = {2: "<i2", 4: "<i4", 8: "<i8"}


def zigzag(x, base, w):
    """d: the bytes of zigzag((x - base) mod 2^(8w)) per w-byte element"""
    s = x.view(UNSIGNED[w]) - base.view(UNSIGNED[w])
    d = (s << 1) ^ (s.view(SIGNED[w]) >> (8 * w - 1)).view(UNSIGNED[w])
    return d.view(np.uint8)


def unzigzag(d, base, w):
    """x: base + unzigzag(d) mod 2^(8w) per element"""
    d = d.view(UNSIGNED[w])
    neg = -((d & 1).astype(SIGNED[w]))
    return (base.view(UNSIGNED[w]) + ((d >> 1) ^ neg.view(UNSIGNED[w]))).view(np.uint8)


def crafted(w, seed=0):
    """(x, base) pairs that take every edge of the transform: b = all ones and x = 0 (wraparound), x = all ones and b = 0,
    sign crossings of floats, NaN and infinity patterns, the integer extremes, equal elements, then random bits"""
    u = np.dtype(UNSIGNED[w])
    top = 1 << (8 * w - 1)
    full = (1 << (8 * w)) - 1
    vals = [0, 1, full, full - 1, top, top - 1, top + 1, 0x7F << (8 * w - 8), 0xFF << (8 * w - 8), 0x7FC << (8 * w - 12),
            (0x7FF << (8 * w - 12)) | 1, 0x80 << (8 * w - 16)]
    pairs = [(a, b) for a in vals for b in vals]
    rng = np.random.default_rng(seed)
    x = np.array([a for a, _ in pairs], dtype=u)
    b = np.array([b for _, b in pairs], dtype=u)
    rx = rng.integers(0, 256, 97 * w, dtype=np.uint8).view(u)
    rb_ = rng.integers(0, 256, 97 * w, dtype=np.uint8).view(u)
    return np.concatenate([x, rx]).view(np.uint8), np.concatenate([b, rb_]).view(np.uint8)


def step(base_bytes, kind, lr, seed):
    """a synthetic training step: the base's floats moved by lr * sign * U(0, 1) per element, rounded to the kind"""
    rng = np.random.default_rng(seed)
    if kind == "bf16":
        master = (base_bytes.view("<u2").astype(np.uint32) << 16).view(np.float32)
    else:
        master = base_bytes.view("<f4")
    moved = (master + lr * rng.choice([-1.0, 1.0], master.size) * rng.random(master.size)).astype(np.float32)
    if kind == "bf16":
        return (moved.view(np.uint32) >> 16).astype("<u2").view(np.uint8)
    return moved.astype("<f4").view(np.uint8)


@pytest.mark.parametrize("w", [2, 4, 8])
def test_transform_round_trips_every_pattern(w):
    x, b = crafted(w)
    d = zigzag(x, b, w)
    assert np.array_equal(unzigzag(d, b, w), x)
    assert np.array_equal(zigzag(b, b, w), np.zeros_like(b))                     # an unchanged tensor: d = 0
    # the definition, element by element in Python integers
    for xi, bi, di in zip(x.view(UNSIGNED[w])[:200], b.view(UNSIGNED[w])[:200], d.view(UNSIGNED[w])[:200]):
        s = (int(xi) - int(bi)) % (1 << (8 * w))
        s = s - (1 << (8 * w)) if s >> (8 * w - 1) else s
        assert int(di) == (2 * s if s >= 0 else -2 * s - 1), (xi, bi)


def py_pack8(planes, w, ch, flags, base_crc, n=None):
    """the version 8 layout, from its description alone"""
    buf = cp.py_pack7(planes, w, ch, flags, n).copy()
    buf[4] = 8
    cp.set_u32(buf, 60, base_crc)
    return cp.reseal(buf)


def delta_container(oracle_lib, kind, w, ch, count, flags=0, seed=0):
    """(x, base, planes of d, version 8 buffer): base of the kind, x one synthetic step (or int32 / fp64 redrawn)"""
    base = cp.elements(kind, count, seed)
    if kind in ("bf16", "fp32"):
        x = step(base, kind, 1e-4, seed + 1)
    else:
        x = cp.elements(kind, count, seed + 1)
    d = zigzag(x, base, w)
    planes = [cp.v6_plane(oracle_lib, pl, ch, flags, p)[0] for p, pl in enumerate(cp.split(d, w))]
    return x, base, planes, api.container_delta_pack(planes, zlib.crc32(base.tobytes()))


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("kind,w,ch,count", cp.CASES)
def test_pack_and_open_round_trip(oracle_lib, kind, w, ch, count, flags):
    base = cp.elements(kind, count, 7)
    x = step(base, kind, 1e-3, 8) if kind in ("bf16", "fp32") else cp.elements(kind, count, 8)
    d = zigzag(x, base, w)
    built = [cp.v6_plane(oracle_lib, pl, ch, flags, p) for p, pl in enumerate(cp.split(d, w))]
    planes = [b[0] for b in built]
    crc = zlib.crc32(base.tobytes())
    buf = api.container_delta_pack(planes, crc)
    assert np.array_equal(buf, py_pack8(planes, w, ch, flags, crc))
    assert buf.size <= api.container_planes_bound(x.size, w, ch)
    meta, views = api.container_delta_open(buf)
    assert meta == {"elem_bytes": w, "chunk_syms": ch, "flags": flags, "n": x.size, "base_crc": crc}
    got = np.zeros(x.size, np.uint8)
    for p, (view, (_, (coder, sb, freqs, cum, bits, o6, b6, st))) in enumerate(zip(views, built)):
        assert np.array_equal(view, planes[p])
        info, f, bb, o, blob = api.container_stored_open(view)
        got[p::w] = cs.decode_host(oracle_lib, coder, sb, f, cum, bb, o, blob, count, ch)
    assert np.array_equal(got, d)
    assert np.array_equal(unzigzag(got, base, w), x)
    # the same planes under version 7 differ only in version, reserved and meta_crc
    v7 = api.container_planes_pack(planes)
    assert np.array_equal(v7[64:], buf[64:]) and np.array_equal(v7[:4], buf[:4]) and np.array_equal(v7[5:44], buf[5:44])
    assert np.array_equal(v7[48:60], buf[48:60])


@pytest.mark.parametrize("crc", [0, 1, 0xFFFFFFFF, 0x80000000])
def test_any_base_crc_is_valid(oracle_lib, crc):
    base = cp.elements("bf16", 100, 1)
    x = step(base, "bf16", 1e-4, 2)
    planes = [cp.v6_plane(oracle_lib, pl, 32, 0, p)[0] for p, pl in enumerate(cp.split(zigzag(x, base, 2), 2))]
    buf = api.container_delta_pack(planes, crc)
    assert api.container_delta_open(buf)[0]["base_crc"] == crc


@pytest.fixture(scope="module")
def good(oracle_lib):
    """(x, base, planes, v8 buffer) for fp32 at chunks of 32, ragged"""
    return delta_container(oracle_lib, "fp32", 4, 32, 9 * 32 + 3, seed=11)


def rejected(buf):
    with pytest.raises(rb.RansError) as e:
        api.container_delta_open(buf)
    return e.value.code


def test_meta_crc_covers_the_base_crc(good):
    _, base, _, buf = good
    crc = zlib.crc32(base.tobytes())
    assert api.container_delta_open(buf)[0]["base_crc"] == crc
    for bit in (0, 13, 31):
        b = buf.copy()
        cp.set_u32(b, 60, crc ^ (1 << bit))
        assert rejected(b) == E_STREAM, bit                               # not resealed: meta_crc fails
        assert api.container_delta_open(cp.reseal(b))[0]["base_crc"] == crc ^ (1 << bit)


def test_open_rejects_each_header_rule(good):
    _, _, _, buf = good
    broken = {}
    for name, off, val in (("version 7", 4, 7), ("version 6", 4, 6), ("version 9", 4, 9), ("coder", 6, 1), ("scale_bits", 7, 12),
                           ("lanes", 8, 16)):
        b = buf.copy()
        b[off] = val
        broken[name] = cp.reseal(b)
    for w in (1, 3, 16):
        b = buf.copy()
        cp.set_u32(b, 52, w)
        cp.set_u32(b, 56, w)
        broken[f"w {w}"] = cp.reseal(b, min(w, 8))
    b = buf.copy()
    cp.set_u32(b, 56, 2)                                                # n_blocks != block_size
    broken["n_blocks"] = cp.reseal(b)
    for name, off in (("n_chunks", 24), ("blob_crc", 48)):
        b = buf.copy()
        b[off] = 1
        broken[name] = cp.reseal(b) if off != 48 else b
    b = buf.copy()
    cp.set_u64(b, 16, cp.u64(buf, 16) + 1)                              # n not a multiple of w
    broken["n ragged"] = cp.reseal(b)
    b = buf.copy()
    cp.set_u64(b, 16, cp.u64(buf, 16) + 4)                              # n disagrees with the planes
    broken["n"] = cp.reseal(b)
    b = buf.copy()
    cp.set_u64(b, 32, cp.u64(buf, 32) + 16)                             # blob_bytes past the buffer
    broken["blob_bytes"] = cp.reseal(b)
    b = buf.copy()
    cp.set_u32(b, 12, 16)                                               # chunk_syms below 32
    broken["chunk_syms"] = cp.reseal(b)
    for name, b in broken.items():
        assert rejected(b) == E_STREAM, name


def test_open_rejects_each_table_rule(good):
    _, _, planes, buf = good
    w = 4
    for off, delta in ((64, 16), (80, -16), (72, -16)):                 # offset[0], plane 1 overlapping, size[0] short
        b = buf.copy()
        cp.set_u64(b, off, cp.u64(buf, off) + delta)
        assert rejected(cp.reseal(b)) == E_STREAM, off
    o1 = cp.u64(buf, 80)
    b = np.concatenate([buf[:o1], np.zeros(16, np.uint8), buf[o1:]])    # a real gap between planes 0 and 1
    for p in range(1, w):
        cp.set_u64(b, 64 + 16 * p, cp.u64(buf, 64 + 16 * p) + 16)
    cp.set_u64(b, 32, cp.u64(buf, 32) + 16)
    assert rejected(cp.reseal(b)) == E_STREAM
    b = buf.copy()
    b[64 + 16 * 2 + 3] ^= 0x40                                          # a flipped table byte: meta_crc
    assert rejected(b) == E_STREAM
    for size in (0, 63, 64, 64 + 16 * 4 - 1, buf.size - 16, buf.size - 1):
        assert rejected(buf[:size].copy()) == E_STREAM, size
    b = buf.copy()
    b[o1 + 64 + 4] ^= 1                                                 # plane 1's model: its own meta_crc
    assert rejected(b) == E_STREAM


def test_versions_reject_each_other(oracle_lib, good):
    x, base, planes, buf = good
    with pytest.raises(rb.RansError) as e:
        api.container_planes_open(buf)                                  # the version 7 open rejects version 8
    assert e.value.code == E_STREAM
    v7 = api.container_planes_pack(planes)
    assert rejected(v7) == E_STREAM                                     # the version 8 open rejects version 7
    b = v7.copy()
    b[4] = 8                                                            # version 7 relabelled 8 (reserved 0 is a valid CRC)
    assert api.container_delta_open(cp.reseal(b))[0]["base_crc"] == 0
    b = buf.copy()
    b[4] = 7                                                            # version 8 relabelled 7: reserved must be 0 there
    assert zlib.crc32(base.tobytes()) != 0
    with pytest.raises(rb.RansError) as e:
        api.container_planes_open(cp.reseal(b))
    assert e.value.code == E_STREAM
    for opener in (api.container_open, api.container_stored_open, api.container_blocks_open, api.container_blocks_stored_open,
                   api.container_blocks_alias_open, api.container_blocks_coder_open):
        with pytest.raises(rb.RansError) as e:
            opener(buf)
        assert e.value.code == E_STREAM, opener.__name__
    assert rejected(planes[0]) == E_STREAM                              # version 6


def test_pack_errors(good):
    _, _, planes, buf = good
    lib = api.load()
    ptrs = (api.C.c_void_p * 4)(*[p.ctypes.data for p in planes])
    sizes = (api.C.c_size_t * 4)(*[p.size for p in planes])
    out = np.zeros(buf.size, np.uint8)
    size = api.C.c_size_t(0)
    crc = int(buf[60:64].view(np.uint32)[0])
    assert lib.dll.rb200_container_delta_pack(4, ptrs, sizes, crc, out.ctypes.data, out.size, api.C.byref(size)) == 0
    assert size.value == buf.size and np.array_equal(out, buf)
    assert lib.dll.rb200_container_delta_pack(4, ptrs, sizes, crc, out.ctypes.data, out.size - 1, None) == E_SPACE
    for w in (1, 3, 16):
        assert lib.dll.rb200_container_delta_pack(w, ptrs, sizes, crc, out.ctypes.data, out.size, None) == E_ARG
    sizes[2] = planes[2].size - 16
    assert lib.dll.rb200_container_delta_pack(4, ptrs, sizes, crc, out.ctypes.data, out.size, None) == E_ARG
    sizes[2] = planes[2].size
    assert lib.dll.rb200_container_delta_pack(4, ptrs, sizes, crc, None, out.size, None) == E_ARG
    info = api.ContainerPlanesInfo()
    c = api.C.c_uint32(0)
    assert lib.dll.rb200_container_delta_open(buf.ctypes.data, buf.size, api.C.byref(info), None) == E_ARG
    assert lib.dll.rb200_container_delta_open(None, buf.size, api.C.byref(info), api.C.byref(c)) == E_ARG
    assert lib.dll.rb200_container_delta_open(buf.ctypes.data, buf.size, api.C.byref(info), api.C.byref(c)) == 0
    assert c.value == crc


def test_status_code():
    assert api.E_BASE == -10
    assert api.load().dll.rb200_strerror(api.E_BASE).decode() != "unknown"
