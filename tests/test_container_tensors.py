"""Version 9 tensor-list containers on the host: rb200_container_tensors_bound, _pack and _open.

- pack equals a packer written from the layout's description (version 7 of the concatenated bytes, version 9,
  n_blocks = T, reserved = the directory's CRC, the directory zero-padded to 16 between the table and plane 0) for
  w = 2, 4 and 8, over planes packed with container_stored_pack from the oracle's streams; open returns the lengths and
  views whose decoded planes give the concatenation back; plane 0 starts at 64 + 16 w + round16(8 T).
- the bound is the version 7 bound plus the padded directory, 0 for a count outside 1..2^20.
- open rejects each header, table and directory rule broken on its own (the CRCs resealed), and meta_crc covers
  reserved.  Versions 7, 8 and 9 reject each other in both directions.  No GPU needed."""
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
MAX_T = 1 << 20


def round16(v):
    return (v + 15) & ~15


def list_bytes(kind, counts, seed):
    """the tensors of a list (element counts `counts`) and their concatenated bytes"""
    ts = [cp.elements(kind, c, seed + i) if c else np.zeros(0, np.uint8) for i, c in enumerate(counts)]
    return ts, np.concatenate(ts) if ts else np.zeros(0, np.uint8)


def planes_of(oracle_lib, data, w, ch, flags=0):
    built = [cp.v6_plane(oracle_lib, pl, ch, flags, p) for p, pl in enumerate(cp.split(data, w))]
    return [b[0] for b in built], built


def py_pack9(lengths, planes, w, ch, flags):
    """the version 9 layout, from its description alone"""
    m = int(planes[0][16:24].view(np.uint64)[0])
    t = len(lengths)
    d = struct.pack(f"<{t}Q", *lengths)
    dpad = d + bytes(round16(8 * t) - 8 * t)
    start = end = 64 + 16 * w + len(dpad)
    table = []
    for p in planes:
        table.append(struct.pack("<QQ", end, p.size))
        end += p.size
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, 9, 0, 0, 32, ch, m * w, 0, end - start, flags, 0, 0, w, t, zlib.crc32(d))
    return cp.reseal(np.frombuffer(hdr + b"".join(table) + dpad + b"".join(p.tobytes() for p in planes), np.uint8).copy())


CASES = [("bf16", 2, 32, [5 * 32 + 17]), ("bf16", 2, 64, [3, 0, 16, 17, 1, 0, 100]), ("fp32", 4, 32, [9 * 32 + 3, 7, 0, 40]),
         ("int32", 4, 48, [200, 1]), ("fp64", 8, 32, [1, 2, 3, 4, 5, 6, 7, 8, 9]), ("fp16", 2, 8192, [0, 700, 0])]


@pytest.mark.parametrize("flags", [0, CRC_BLOB])
@pytest.mark.parametrize("kind,w,ch,counts", CASES)
def test_pack_and_open_round_trip(oracle_lib, kind, w, ch, counts, flags):
    ts, data = list_bytes(kind, counts, 3)
    planes, built = planes_of(oracle_lib, data, w, ch, flags)
    lengths = [t.size for t in ts]
    buf = api.container_tensors_pack(lengths, planes)
    assert np.array_equal(buf, py_pack9(lengths, planes, w, ch, flags))
    assert buf.size <= api.container_tensors_bound(data.size, len(counts), w, ch)
    meta, got_len, views = api.container_tensors_open(buf)
    assert meta == {"elem_bytes": w, "chunk_syms": ch, "flags": flags, "n": data.size, "count": len(counts)}
    assert got_len.tolist() == lengths
    got = np.zeros(data.size, np.uint8)
    m = data.size // w
    for p, (view, (_, (coder, sb, freqs, cum, bits, o6, b6, st))) in enumerate(zip(views, built)):
        assert np.array_equal(view, planes[p])
        info, f, bb, o, blob = api.container_stored_open(view)
        got[p::w] = cs.decode_host(oracle_lib, coder, sb, f, cum, bb, o, blob, m, ch)
    assert np.array_equal(got, data)
    # the planes and the table's sizes are version 7's of the concatenation; only the offsets move past the directory
    v7 = api.container_planes_pack(planes)
    d = round16(8 * len(counts))
    assert np.array_equal(v7[64 + 16 * w:], buf[64 + 16 * w + d:])
    for p in range(w):
        assert cp.u64(buf, 64 + 16 * p) == cp.u64(v7, 64 + 16 * p) + d
        assert cp.u64(buf, 72 + 16 * p) == cp.u64(v7, 72 + 16 * p)


@pytest.mark.parametrize("t", [1, 2, 3, 4, 17, 1000])
def test_plane_offsets_after_the_padded_directory(oracle_lib, t):
    counts = [1] * (t - 1) + [40]
    ts, data = list_bytes("bf16", counts, 5)
    planes, _ = planes_of(oracle_lib, data, 2, 32)
    buf = api.container_tensors_pack([x.size for x in ts], planes)
    start = 64 + 32 + round16(8 * t)
    assert start % 16 == 0
    assert cp.u64(buf, 64) == start and cp.u64(buf, 80) == start + planes[0].size
    assert cp.u64(buf, 32) == buf.size - start                        # blob_bytes: the planes, from plane 0
    if t % 2:
        assert cp.u64(buf, 64 + 32 + 8 * t) == 0
    assert np.array_equal(buf[start:start + planes[0].size], planes[0])


@pytest.mark.parametrize("w", [2, 4, 8])
@pytest.mark.parametrize("ch", [32, 8192])
def test_bound(w, ch):
    for n in (w, 31 * w, ch * w, (10 * ch + 5) * w):
        for t in (1, 2, 3, 1000, MAX_T):
            assert api.container_tensors_bound(n, t, w, ch) == api.container_planes_bound(n, w, ch) + round16(8 * t)
        assert api.container_tensors_bound(n, 0, w, ch) == 0
        assert api.container_tensors_bound(n, MAX_T + 1, w, ch) == 0
    assert api.container_tensors_bound(w + 1, 1, w, ch) == 0
    assert api.container_tensors_bound(16, 1, 3, ch) == 0


@pytest.fixture(scope="module")
def good(oracle_lib):
    """(lengths, planes, v9 buffer): fp32 at chunks of 32, an odd count with a zero-length tensor"""
    ts, data = list_bytes("fp32", [9 * 32 + 3, 0, 17, 40, 5], 11)
    planes, _ = planes_of(oracle_lib, data, 4, 32)
    lengths = [t.size for t in ts]
    return lengths, planes, api.container_tensors_pack(lengths, planes)


def rejected(buf):
    with pytest.raises(rb.RansError) as e:
        api.container_tensors_open(buf)
    return e.value.code


DIR = 64 + 16 * 4                                                      # the directory's offset at w = 4


def with_dir(buf, lengths):
    """buf with its directory's lengths replaced (T unchanged) and both CRCs resealed"""
    b = buf.copy()
    for i, v in enumerate(lengths):
        cp.set_u64(b, DIR + 8 * i, v)
    cp.set_u32(b, 60, zlib.crc32(b[DIR:DIR + 8 * len(lengths)].tobytes()))
    return cp.reseal(b)


def test_good_opens(good):
    lengths, _, buf = good
    meta, got, _ = api.container_tensors_open(buf)
    assert got.tolist() == lengths and meta["count"] == 5


def test_meta_crc_covers_reserved(good):
    _, _, buf = good
    b = buf.copy()
    cp.set_u32(b, 60, int(b[60:64].view(np.uint32)[0]) ^ 1)
    assert rejected(b) == E_STREAM                                    # meta_crc no longer matches
    assert rejected(cp.reseal(b)) == E_STREAM                         # resealed: the directory's CRC no longer matches


def test_open_rejects_each_header_rule(good):
    _, _, buf = good
    n = cp.u64(buf, 16)
    edits = {
        "magic": (0, "<I", MAGIC ^ 1), "coder": (6, "<B", 1), "scale_bits": (7, "<B", 12), "lanes": (8, "<I", 16),
        "chunk_syms 16": (12, "<I", 16), "chunk_syms 2^24 + 1": (12, "<I", (1 << 24) + 1), "n 0": (16, "<Q", 0),
        "n not a multiple of w": (16, "<Q", n + 1), "n_chunks": (24, "<Q", 1), "blob_bytes past size": (32, "<Q", 1 << 40),
        "blob_crc": (48, "<I", 1), "w 3": (52, "<I", 3), "count 0": (56, "<I", 0), "count 2^20 + 1": (56, "<I", MAX_T + 1),
    }
    for name, (off, fmt, v) in edits.items():
        b = buf.copy()
        b[off:off + struct.calcsize(fmt)] = np.frombuffer(struct.pack(fmt, v), np.uint8)
        assert rejected(cp.reseal(b, w=4)) == E_STREAM, name
    # a count that moves the planes past the table's offsets, and one whose directory no longer fits the buffer
    for t in (4, 6, 2 * buf.size):
        b = buf.copy()
        cp.set_u32(b, 56, t)
        assert rejected(cp.reseal(b)) == E_STREAM, t
    assert rejected(buf[:DIR + 8]) == E_STREAM                        # truncated inside the directory


def test_open_rejects_each_directory_rule(good):
    lengths, _, buf = good
    assert api.container_tensors_open(with_dir(buf, lengths))[1].tolist() == lengths
    bad = {
        "sum short": [lengths[0] - 4] + lengths[1:],
        "sum long": [lengths[0] + 4] + lengths[1:],
        "not a multiple of w": [lengths[0] - 2, 2] + lengths[2:],
        "one above n, the sum wrapped": [lengths[0], (1 << 64) - 4 * 17] + lengths[2:],
    }
    for name, ls in bad.items():
        assert rejected(with_dir(buf, ls)) == E_STREAM, name
    b = buf.copy()                                                    # nonzero padding after an odd count
    cp.set_u64(b, DIR + 8 * len(lengths), 1)
    assert rejected(cp.reseal(b)) == E_STREAM
    b = buf.copy()                                                    # a wrong reserved, resealed
    cp.set_u32(b, 60, zlib.crc32(b[DIR:DIR + 8 * len(lengths)].tobytes()) ^ 0x80000000)
    assert rejected(cp.reseal(b)) == E_STREAM
    b = buf.copy()                                                    # a directory changed under its old CRC
    cp.set_u64(b, DIR, lengths[0] - 4)
    cp.set_u64(b, DIR + 8, 4)
    assert rejected(cp.reseal(b)) == E_STREAM


def test_open_rejects_each_table_rule(good):
    _, planes, buf = good
    start = DIR + round16(8 * 5)
    for name, off, v in (("plane 0 at the v7 offset", 64, DIR), ("plane 0 inside the directory", 64, start - 16),
                         ("plane 0 late", 64, start + 16), ("plane 1 size", 88, planes[1].size + 16)):
        b = buf.copy()
        cp.set_u64(b, off, v)
        assert rejected(cp.reseal(b)) == E_STREAM, name


def test_versions_reject_each_other(oracle_lib, good):
    lengths, planes, v9 = good
    v7 = api.container_planes_pack(planes)
    v8 = api.container_delta_pack(planes, 1234)
    for other in (v7, v8):
        assert rejected(other) == E_STREAM
    for opener in (api.container_planes_open, lambda b: api.container_delta_open(b)):
        with pytest.raises(rb.RansError) as e:
            opener(v9)
        assert e.value.code == E_STREAM
    # v9 with the version field rewritten is no v7 or v8 either, and v7 / v8 relabelled 9 are no v9
    for v in (7, 8):
        b = v9.copy()
        b[4] = v
        with pytest.raises(rb.RansError):
            (api.container_planes_open if v == 7 else api.container_delta_open)(cp.reseal(b))
    for b0 in (v7, v8):
        b = b0.copy()
        b[4] = 9
        assert rejected(cp.reseal(b)) == E_STREAM
    for opener in (api.container_stored_open, api.container_blocks_stored_open, api.container_open):
        with pytest.raises(rb.RansError):
            opener(v9)


def test_pack_errors(good):
    lengths, planes, _ = good
    lib = api.load()

    def pack(ls, count=None, planes_=planes, cap=1 << 20):
        ls = np.ascontiguousarray(ls, dtype=np.uint64)
        ptrs = (api.C.c_void_p * len(planes_))(*[p.ctypes.data for p in planes_])
        sizes = (api.C.c_size_t * len(planes_))(*[p.size for p in planes_])
        out = np.zeros(cap, np.uint8)
        return lib.dll.rb200_container_tensors_pack(len(planes_), ls.ctypes.data_as(api._u64p), len(ls) if count is None else count, ptrs,
                                                    sizes, out.ctypes.data, out.size, None)

    assert pack(lengths) == 0
    assert pack(lengths, count=0) == E_ARG
    assert pack(lengths[:-1] + [lengths[-1] + 4]) == E_ARG             # sum above n
    assert pack([lengths[0] - 2, 2] + lengths[2:]) == E_ARG            # not a multiple of w
    assert pack(lengths, planes_=planes[:3]) == E_ARG                  # w = 3
    assert pack(lengths, cap=100) == E_SPACE
    assert lib.dll.rb200_container_tensors_pack(4, None, 1, None, None, None, 0, None) == E_ARG
