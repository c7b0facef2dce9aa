"""Version 6 single-model containers (stored chunks) on the host: rb200_container_stored_pack, _open and _bound.

- pack equals a packer written from the layout's description, over the oracle's chunked streams of all four coders
  with the store rule applied in Python (and none, the last and every chunk stored), ragged and whole lengths, chunks
  of 32, 33 and 8192; open returns views whose coded chunks decode with the oracle and whose stored chunks are the input.
- open rejects each rule broken on its own: a bit past n_chunks, bitmap padding, a wrong step (a ragged last chunk
  given round16(chunk_syms) among them), nonzero padding, nonzero block_size / n_blocks / reserved, a bad model, both
  CRCs; versions 1-5 and 6 reject each other.
- pack's error codes, and the bound (an all-stored container is exactly the bound).  No GPU needed."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
OCODER = {WORD: orc.CODER_WORD, BYTE: orc.CODER_BYTE, ALIAS: orc.CODER_ALIAS, RANS64: orc.CODER_RANS64}
MAGIC = 0x43324252
CRC_BLOB = 1
PAIRS = [(WORD, 12), (BYTE, 14), (RANS64, 10), (ALIAS, 16)]
E_ARG, E_MODEL, E_SPACE, E_STREAM = -1, -2, -3, -4

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import _gen  # noqa: E402


def r16(x):
    return (x + 15) & ~15


def mixed_data(n, ch, seed):
    """uniform and Zipf runs whose boundaries fall inside chunks: uniform chunks are stored, Zipf ones coded (at large
    chunks)"""
    run = max(ch + ch // 3, 40)
    parts, kind, i = [], 0, 0
    while sum(p.size for p in parts) < n:
        parts.append(_gen(("uniform", "zipf")[kind], run, seed + i))
        kind ^= 1
        i += 1
    return np.concatenate(parts)[:n].copy()


def chunk_m(c, ch, n):
    return min(ch, n - c * ch)


def streams(offsets, blob):
    return [blob[int(offsets[c]):int(offsets[c + 1]) & ~15] for c in range(offsets.size - 1)]


def layout(parts):
    offs, out, end = [], [], 0
    for s in parts:
        out += [np.zeros(r16(s.size) - s.size, np.uint8), s]
        end += r16(s.size)
        offs.append(end - s.size)
    return np.array(offs + [end], np.uint64), np.concatenate(out).astype(np.uint8)


def oracle_container(oracle_lib, coder, sb, data, ch):
    freqs, cum = oracle_lib.model(data, sb)
    blob, offs = oracle_lib.chunked_encode(OCODER[coder], data, freqs, cum, ch, scale_bits=sb)
    return freqs, cum, offs, blob


def store_rule(offsets, blob, ch, n):
    """chunk c is stored when its stream rounded up to 16 is longer than round16(m_c)"""
    return [c for c, s in enumerate(streams(offsets, blob)) if r16(s.size) > r16(chunk_m(c, ch, n))]


def apply_store(data, ch, offsets, blob, which=None):
    """(bits, offsets, blob, which): the chunks in `which` (default: the store rule's) stored"""
    n = data.size
    which = store_rule(offsets, blob, ch, n) if which is None else sorted(which)
    parts = streams(offsets, blob)
    n_chunks = len(parts)
    bits = np.zeros((n_chunks + 31) // 32, np.uint32)
    for c in which:
        m = chunk_m(c, ch, n)
        parts[c] = np.concatenate([data[c * ch:c * ch + m], np.zeros(r16(m) - m, np.uint8)])
        bits[c // 32] |= np.uint32(1 << (c % 32))
    offs, out = layout(parts)
    return bits, offs, out, which


def py_pack(coder, sb, ch, n, freqs, bits, offsets, blob, flags, version=6):
    """the version 6 layout, from its description alone"""
    n_chunks = offsets.size - 1
    hdr = struct.pack("<IHBBIIQQQIIIIII", MAGIC, version, coder, sb, 32, ch, n, n_chunks, blob.size, flags, 0, 0, 0, 0, 0)
    prefix = np.asarray(freqs, "<u4").tobytes() + np.asarray(offsets, "<u8").tobytes()
    prefix += b"\0" * (-(64 + len(prefix)) % 16)
    words = np.zeros(-(-((n_chunks + 31) // 32) // 4) * 4, "<u4")
    words[:bits.size] = bits
    prefix += words.tobytes()
    meta = zlib.crc32(hdr + prefix)
    blob_crc = zlib.crc32(blob.tobytes()) if flags & CRC_BLOB else 0
    body = hdr[:44] + struct.pack("<II", meta, blob_crc) + hdr[52:] + prefix
    return np.frombuffer(body + blob.tobytes(), np.uint8).copy()


def blob_offset(n_chunks):
    return r16(1088 + 8 * (n_chunks + 1)) + 16 * ((n_chunks + 127) // 128)


def reseal(buf):
    """recompute both CRCs of a (possibly broken) version 6 buffer: meta over [0, blob offset) with the crc fields zero"""
    buf = buf.copy()
    n_chunks = int(buf[24:32].view(np.uint64)[0])
    boff = blob_offset(n_chunks)
    buf[44:52] = 0
    meta = zlib.crc32(buf[:boff].tobytes())
    flags = int(buf[40:44].view(np.uint32)[0])
    blob_crc = zlib.crc32(buf[boff:].tobytes()) if flags & CRC_BLOB else 0
    buf[44:52] = np.frombuffer(struct.pack("<II", meta, blob_crc), np.uint8)
    return buf


def decode_host(oracle_lib, coder, sb, freqs, cum, bits, offsets, blob, n, ch):
    """every chunk: a stored one from the blob, a coded one by the oracle"""
    out = []
    for c in range(offsets.size - 1):
        m = chunk_m(c, ch, n)
        if (int(bits[c // 32]) >> (c % 32)) & 1:
            out.append(blob[int(offsets[c]):int(offsets[c]) + m])
            continue
        lo, hi = int(offsets[c]) & ~15, int(offsets[c + 1])
        oo = np.array([int(offsets[c]) - lo, hi - lo], np.uint64)
        out.append(oracle_lib.chunked_decode(OCODER[coder], blob[lo:hi], oo, m, freqs, cum, ch, scale_bits=sb))
    return np.concatenate(out)


def lengths(ch):
    base = 5 * ch if ch > 64 else 40 * ch
    return [base, base + 17]                                      # whole, ragged


@pytest.mark.parametrize("ch", [32, 33, 8192])
@pytest.mark.parametrize("coder,sb", PAIRS)
def test_pack_equals_independent_packer_opens_and_decodes(oracle_lib, coder, sb, ch):
    for n in lengths(ch):
        data = mixed_data(n, ch, 11 + n)
        freqs, cum, offs, blob = oracle_container(oracle_lib, coder, sb, data, ch)
        n_chunks = offs.size - 1
        for which in (None, [], [n_chunks - 1], list(range(n_chunks))):
            bits, o6, b6, st = apply_store(data, ch, offs, blob, which)
            flags = CRC_BLOB if n % 2 else 0
            case = (coder, sb, ch, n, which)
            got = api.container_stored_pack(coder, sb, ch, n, freqs, bits, o6, b6, flags)
            assert np.array_equal(got, py_pack(coder, sb, ch, n, freqs, bits, o6, b6, flags)), case
            meta, f, b, o, bl = api.container_stored_open(got)
            assert meta == {"coder": coder, "scale_bits": sb, "chunk_syms": ch, "flags": flags, "n_symbols": n,
                            "n_chunks": n_chunks, "blob_bytes": b6.size}, case
            assert np.array_equal(f, freqs) and np.array_equal(b, bits) and np.array_equal(o, o6) and np.array_equal(bl, b6), case
            assert np.array_equal(decode_host(oracle_lib, coder, sb, freqs, cum, b, o, bl, n, ch), data), case
            if which == list(range(n_chunks)):
                assert got.size == api.container_stored_bound(n, ch), case


@pytest.fixture(scope="module")
def sample(oracle_lib):
    """a ragged container (chunks of 33, 70 chunks) with stored and coded chunks, the last stored, and the blob CRC"""
    ch, n = 33, 33 * 69 + 20
    data = mixed_data(n, 4096, 5)
    freqs, cum, offs, blob = oracle_container(oracle_lib, WORD, 12, data, ch)
    which = [c for c in range(offs.size - 1) if c % 3 == 0] + [offs.size - 2]
    bits, o6, b6, _ = apply_store(data, ch, offs, blob, sorted(set(which)))
    buf = api.container_stored_pack(WORD, 12, ch, n, freqs, bits, o6, b6, CRC_BLOB)
    return dict(buf=buf, data=data, freqs=freqs, bits=bits, offs=o6, blob=b6, n=n, ch=ch, stored=sorted(set(which)))


def _rejected(buf):
    with pytest.raises(rb.RansError) as ei:
        api.container_stored_open(buf)
    return ei.value.code


def test_sample_opens(sample):
    api.container_stored_open(sample["buf"])
    assert _rejected(sample["buf"][:-1]) == E_STREAM
    assert _rejected(sample["buf"][:63]) == E_STREAM


def _bitmap_at(n_chunks):
    return r16(1088 + 8 * (n_chunks + 1))


def test_rejects_a_bit_past_n_chunks(sample):
    buf = sample["buf"].copy()
    n_chunks = sample["offs"].size - 1                           # 70: word 2 holds chunks 64..69
    assert n_chunks % 32
    w = buf[_bitmap_at(n_chunks) + 8:_bitmap_at(n_chunks) + 12].view(np.uint32)
    w[0] |= np.uint32(1 << (n_chunks % 32))
    assert _rejected(reseal(buf)) == E_STREAM


def test_rejects_bitmap_padding(sample):
    buf = sample["buf"].copy()
    n_chunks = sample["offs"].size - 1
    assert (n_chunks + 31) // 32 < 4
    buf[_bitmap_at(n_chunks) + 12] = 1                           # the fourth word: padding
    assert _rejected(reseal(buf)) == E_STREAM


def test_rejects_a_coded_chunk_marked_stored(sample):
    buf = sample["buf"].copy()
    n_chunks = sample["offs"].size - 1
    c = next(c for c in range(n_chunks) if c not in sample["stored"])
    buf[_bitmap_at(n_chunks) + 4 * (c // 32):_bitmap_at(n_chunks) + 4 * (c // 32) + 4].view(np.uint32)[0] |= np.uint32(1 << (c % 32))
    assert _rejected(reseal(buf)) == E_STREAM


def test_rejects_a_ragged_last_chunk_stored_at_round16_chunk_syms(sample):
    s = sample
    ch, n, data = s["ch"], s["n"], s["data"]
    last = s["offs"].size - 2
    parts = streams(s["offs"], s["blob"])
    m = chunk_m(last, ch, n)
    parts[last] = np.concatenate([data[last * ch:], np.zeros(r16(ch) - m, np.uint8)])
    offs, blob = layout(parts)
    forged = py_pack(WORD, 12, ch, n, s["freqs"], s["bits"], offs, blob, CRC_BLOB)
    assert _rejected(forged) == E_STREAM
    with pytest.raises(rb.RansError) as ei:
        api.container_stored_pack(WORD, 12, ch, n, s["freqs"], s["bits"], offs, blob, CRC_BLOB)
    assert ei.value.code == E_ARG


def test_rejects_nonzero_padding(sample):
    s = sample
    buf = s["buf"].copy()
    boff = blob_offset(s["offs"].size - 1)
    c = next(c for c in s["stored"] if chunk_m(c, s["ch"], s["n"]) % 16)
    buf[boff + int(s["offs"][c]) + chunk_m(c, s["ch"], s["n"])] = 9
    assert _rejected(reseal(buf)) == E_STREAM


@pytest.mark.parametrize("at", [52, 56, 60])
def test_rejects_block_fields(sample, at):
    buf = sample["buf"].copy()
    buf[at] = 1
    assert _rejected(reseal(buf)) == E_STREAM


def test_rejects_a_bad_model(sample):
    buf = sample["buf"].copy()
    buf[64:68].view(np.uint32)[0] += 1
    assert _rejected(reseal(buf)) == E_STREAM


def test_rejects_either_crc(sample):
    buf = sample["buf"].copy()
    buf[44] ^= 1
    assert _rejected(buf) == E_STREAM
    buf = sample["buf"].copy()
    buf[-1] ^= 1
    assert _rejected(buf) == E_STREAM
    buf = sample["buf"].copy()
    buf[_bitmap_at(sample["offs"].size - 1)] ^= 2                  # the bitmap is under meta_crc
    assert _rejected(buf) == E_STREAM


@pytest.mark.parametrize("version", [1, 2, 3, 4, 5, 7])
def test_other_versions_are_rejected(sample, version):
    buf = sample["buf"].copy()
    buf[4:6].view(np.uint16)[0] = version
    assert _rejected(reseal(buf)) == E_STREAM


def test_version_6_is_rejected_by_every_other_open(sample, oracle_lib):
    buf = sample["buf"]
    for opener in (api.container_open, api.container_blocks_open, api.container_blocks_coder_open, api.container_blocks_alias_open,
                   api.container_blocks_stored_open):
        with pytest.raises(rb.RansError) as ei:
            opener(buf)
        assert ei.value.code == E_STREAM, opener
    # and a version 1 container is rejected by the version 6 open
    data = mixed_data(5000, 4096, 3)
    freqs, cum, offs, blob = oracle_container(oracle_lib, WORD, 12, data, 4096)
    v1 = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob)
    assert _rejected(v1) == E_STREAM


def test_pack_error_codes(sample):
    s = sample
    args = dict(coder=WORD, scale_bits=12, chunk_syms=s["ch"], n=s["n"], freqs=s["freqs"], stored_bits=s["bits"], offsets=s["offs"],
                blob=s["blob"])

    def code(**kw):
        a = dict(args, **kw)
        with pytest.raises(rb.RansError) as ei:
            api.container_stored_pack(**a)
        return ei.value.code

    assert code(scale_bits=14) == E_ARG                         # the word coder is at 12 only
    assert code(coder=9) == E_ARG
    assert code(chunk_syms=31) == E_ARG
    bits = s["bits"].copy()
    bits[-1] |= np.uint32(1 << 31)
    assert code(stored_bits=bits) == E_ARG                       # a bit past n_chunks
    f = s["freqs"].copy()
    f[0] += 1
    assert code(freqs=f) == E_MODEL
    blob = s["blob"].copy()
    c = next(c for c in s["stored"] if chunk_m(c, s["ch"], s["n"]) % 16)
    blob[int(s["offs"][c]) + chunk_m(c, s["ch"], s["n"])] = 1
    assert code(blob=blob) == E_ARG                              # nonzero padding
    offs = s["offs"].copy()
    offs[-1] += 16
    assert code(offsets=offs) == E_ARG                           # the directory disagrees with the blob


def test_bound():
    for n, ch in [(1, 32), (31, 32), (32, 32), (33, 32), (1_000_003, 8192), (8192 * 7, 8192), (100, 33), (1 << 20, 1 << 24)]:
        n_chunks = -(-n // ch)
        want = blob_offset(n_chunks) + (n // ch) * r16(ch) + (r16(n % ch) if n % ch else 0)
        assert api.container_stored_bound(n, ch) == want, (n, ch)
    assert api.container_stored_bound(0, 32) == 0
    assert api.container_stored_bound(100, 31) == 0
    assert api.container_stored_bound(100, (1 << 24) + 1) == 0
    assert api.container_stored_bound(1 << 32, 8192) == 0
    # uniform bytes at chunks of 8192 with every chunk stored: 1.000993 B/sym on 1 GiB
    n = 1 << 30
    assert abs(api.container_stored_bound(n, 8192) / n - 1.000993) < 5e-7
