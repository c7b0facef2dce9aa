"""CPU tests of the product's host-side code (no GPU needed): the C-ABI library loads and
exports everything include/rans_b200.h declares, and its host model construction
(rb200_count_freqs / normalize_freqs / word_tables_build / alias_tables_build) is
bit-identical to the reference algorithm (via the oracle and the golden fixtures)."""
import json
import os
import re

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = np.load(os.path.join(HERE, "golden", "golden.npz"))
INDEX = json.load(open(os.path.join(HERE, "golden", "golden.json")))
CASES = [k for k in INDEX if k != "book1"]


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "rans_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(rb200_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 20
    lib = rb.load()
    bound = {name for name, _, _ in rb.api.EXPORTS}
    assert declared == bound, f"header/binding mismatch: {declared ^ bound}"
    for name in declared:
        assert hasattr(lib.dll, name), name
    assert lib.dll.rb200_version() == 2        # RB200_VERSION: 2 added the rb200_comm_* / rb200_gather_* entry points
    assert lib.dll.rb200_strerror(-4) == b"corrupt or truncated stream"


def test_geometry_calls():
    lib = rb.load()
    assert lib.dll.rb200_chunk_count(0, 4096) == 0
    assert lib.dll.rb200_chunk_count(1, 4096) == 1
    assert lib.dll.rb200_chunk_count(8193, 4096) == 3
    # bound = per chunk round16(512 + 2 * m), valid for every coder
    assert lib.dll.rb200_encode_bound(4096, 4096) == 512 + 8192
    assert lib.dll.rb200_encode_bound(4097, 4096) == 512 + 8192 + 528
    assert lib.dll.rb200_encode_bound(0, 4096) == 0


def test_no_gpu_is_a_loud_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    with pytest.raises(rb.RansError) as ei:
        rb.Context(0)
    assert ei.value.code == -5          # RB200_E_CUDA: no silent CPU fallback exists


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("sb,cname", [(12, "word"), (14, "byte"), (16, "alias")])
def test_normalize_matches_reference_golden(case, sb, cname):
    data = GOLD[f"{case}/data"]
    st = rb.SymbolStats().count_freqs(data)
    assert np.array_equal(st.freqs, np.bincount(data, minlength=256))
    st.normalize_freqs(1 << sb)
    assert np.array_equal(st.freqs, GOLD[f"{case}/{cname}/freqs"])
    assert st.cum_freqs[256] == 1 << sb and np.array_equal(np.diff(st.cum_freqs.astype(np.int64)), st.freqs)


@pytest.mark.parametrize("seed", range(12))
def test_normalize_matches_oracle_random(oracle_lib, seed):
    rng = np.random.default_rng(seed)
    nsym = int(rng.integers(1, 257))
    raw = np.zeros(256, np.uint32)
    syms = rng.permutation(256)[:nsym]
    raw[syms] = (rng.pareto(0.7, nsym) * 50 + 1).astype(np.uint32)     # heavy tails: many squashed symbols
    for sb in (8, 12, 16):
        if nsym > (1 << sb):
            continue
        want_f, want_c = oracle_lib.normalize_freqs(raw, 1 << sb)
        st = rb.SymbolStats()
        st.freqs[:] = raw
        st.normalize_freqs(1 << sb)
        assert np.array_equal(st.freqs, want_f) and np.array_equal(st.cum_freqs, want_c)


def test_normalize_rejects_bad_input():
    st = rb.SymbolStats()
    with pytest.raises(rb.RansError):
        st.normalize_freqs(4096)             # all-zero histogram: the reference would divide by zero
    st.freqs[:] = 1
    with pytest.raises(rb.RansError):
        st.normalize_freqs(128)              # main.cpp:77 assert(target_total >= 256)


@pytest.mark.parametrize("case", CASES)
def test_word_tables_match_reference_layout(oracle_lib, case):
    data = GOLD[f"{case}/data"]
    st = rb.SymbolStats().count_freqs(data).normalize_freqs(4096)
    slots, s2s = st.word_tables()
    oslots, os2s = oracle_lib.word_tables(st.freqs, st.cum_freqs)
    assert np.array_equal(slots, oslots) and np.array_equal(s2s, os2s)


@pytest.mark.parametrize("case", CASES)
def test_alias_tables_match_reference_golden(case):
    import hashlib
    data = GOLD[f"{case}/data"]
    st = rb.SymbolStats().count_freqs(data).normalize_freqs(1 << 16).make_alias_table()
    assert np.array_equal(st.divider, GOLD[f"{case}/alias_tables/divider"])
    assert np.array_equal(st.slot_adjust, GOLD[f"{case}/alias_tables/slot_adjust"])
    assert np.array_equal(st.slot_freqs, GOLD[f"{case}/alias_tables/slot_freqs"])
    assert np.array_equal(st.sym_id, GOLD[f"{case}/alias_tables/sym_id"])
    assert hashlib.sha256(st.alias_remap.tobytes()).hexdigest() == INDEX[case]["alias_remap_sha256"]


@pytest.mark.parametrize("sb", [8, 10, 13, 16])
def test_alias_tables_match_oracle_other_scales(oracle_lib, gen, sb):
    data = gen("zipf", 40000, sb)
    st = rb.SymbolStats().count_freqs(data).normalize_freqs(1 << sb).make_alias_table()
    want = oracle_lib.alias_build(st.freqs, st.cum_freqs)
    got = (st.divider, st.slot_adjust, st.slot_freqs, st.sym_id, st.alias_remap)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_container_pack_open_roundtrip(oracle_lib, gen):
    """SURVEY 8f.3: the wire format carries coder, scale_bits, lanes, chunk size, n, model, directory, checksums."""
    from ryg_rans_b200 import api
    data = gen("zipf", 50000, 4)
    freqs, cum = oracle_lib.model(data, 12)
    blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 4096)     # the oracle stands in for the GPU here
    for flags in (0, api.CONTAINER_CRC_BLOB):
        buf = api.container_pack(rb.CODER_WORD, 12, 4096, data.size, freqs, offs, blob, flags)
        assert buf.size == 64 + 1024 + 8 * offs.size + (-(64 + 1024 + 8 * offs.size) % 16) + blob.size
        meta, f2, o2, b2 = api.container_open(buf)
        assert meta == {"coder": 0, "scale_bits": 12, "chunk_syms": 4096, "flags": flags, "n_symbols": data.size,
                        "n_chunks": offs.size - 1, "blob_bytes": blob.size}
        assert np.array_equal(f2, freqs) and np.array_equal(o2, offs) and np.array_equal(b2, blob)
        out = oracle_lib.chunked_decode(orc.CODER_WORD, b2, o2, data.size, f2, np.concatenate([[0], np.cumsum(f2)]).astype(np.uint32), 4096)
        assert np.array_equal(out, data)
        # corruption of header, model, directory (always) and payload (when its CRC is on) is detected
        for pos in (5, 70, 64 + 1024 + 9) + ((buf.size - 7,) if flags else ()):
            bad = buf.copy()
            bad[pos] ^= 0x40
            with pytest.raises(rb.RansError) as ei:
                api.container_open(bad)
            assert ei.value.code == -4
    with pytest.raises(rb.RansError):
        api.container_open(buf[:200])


def _reseal(buf):
    """Recompute the container's meta CRC (IEEE CRC-32 = zlib's) after editing header / model / directory fields, so
    that the semantic checks behind the checksum are what rejects the container."""
    import struct
    import zlib
    n_chunks = struct.unpack_from("<Q", buf, 24)[0]
    hdr = bytearray(buf[:64].tobytes())
    hdr[44:52] = b"\0" * 8                                   # meta_crc, blob_crc
    end = 64 + 1024 + 8 * (n_chunks + 1)
    if end > buf.size:
        return buf
    crc = zlib.crc32(bytes(hdr) + buf[64:end].tobytes()) & 0xffffffff
    struct.pack_into("<I", buf, 44, crc)
    return buf


def test_container_open_rejects_crafted_and_truncated_input(oracle_lib, gen):
    """The parser is the trust boundary of the wire format: every truncation and every inconsistent field must come
    back as RB200_E_STREAM (-4) -- with a VALID checksum, so the field checks themselves are exercised -- never as a
    crash or an out-of-bounds view."""
    import struct
    from ryg_rans_b200 import api
    data = gen("text", 20000, 6)
    freqs, cum = oracle_lib.model(data, 12)
    blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 4096)
    good = api.container_pack(rb.CODER_WORD, 12, 4096, data.size, freqs, offs, blob, 0)
    assert api.container_open(_reseal(good.copy()))[0]["n_symbols"] == data.size      # _reseal reproduces the library's CRC

    def rejected(buf):
        with pytest.raises(rb.RansError) as ei:
            api.container_open(buf)
        return ei.value.code

    for cut in list(range(0, 64 + 1024 + 8 * offs.size + 16, 7)) + [good.size - 16, good.size - 1]:
        assert rejected(good[:cut].copy()) == -4, cut
    edits = {
        "magic": (0, "<I", 0x12345678), "version": (4, "<H", 2), "coder": (6, "<B", 9), "scale_bits": (7, "<B", 3),
        "lanes": (8, "<I", 64), "chunk_syms zero": (12, "<I", 0), "chunk_syms other": (12, "<I", 2048),
        "n_symbols huge": (16, "<Q", 2 ** 64 - 1), "n_symbols + 1 chunk": (16, "<Q", data.size + 4096),
        "n_chunks huge": (24, "<Q", 2 ** 40), "n_chunks 2^31": (24, "<Q", 2 ** 31), "blob_bytes odd": (32, "<Q", blob.size + 8),
        "blob_bytes beyond the buffer": (32, "<Q", blob.size + 4096), "blob_bytes short": (32, "<Q", blob.size - 16),
    }
    for name, (off, fmt, val) in edits.items():
        bad = good.copy()
        struct.pack_into(fmt, bad, off, val)
        assert rejected(_reseal(bad)) == -4, name
    dir_off = 64 + 1024
    for name, idx, val in (("directory not monotone", 1, int(offs[2]) + 16), ("last entry != blob size", offs.size - 1, int(offs[-1]) - 16)):
        bad = good.copy()
        struct.pack_into("<Q", bad, dir_off + 8 * idx, val)
        assert rejected(_reseal(bad)) == -4, name
    # CRC-valid but inconsistent models / first offsets are rejected at open, not later in model_create or the kernel
    for name, off, fmt, val in (("freqs do not sum to 1 << scale_bits", 64 + 4 * 65, "<I", 7), ("word coder with scale_bits 14", 7, "<B", 14),
                                ("first stream starts beyond the first vector", dir_off, "<Q", 32)):
        bad = good.copy()
        struct.pack_into(fmt, bad, off, val)
        assert rejected(_reseal(bad)) == -4, name
    # and pack refuses to write what open would reject
    for coder, sb, f in ((256, 12, freqs), (rb.CODER_WORD, 14, freqs), (rb.CODER_ALIAS, 20, freqs), (rb.CODER_WORD, 12, freqs // 2)):
        with pytest.raises(rb.RansError) as ei:
            api.container_pack(coder, sb, 4096, data.size, f, offs, blob, 0)
        assert ei.value.code == -2, (coder, sb)
    # random garbage with a valid magic never gets through either
    rng = np.random.default_rng(0)
    for _ in range(200):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        junk[:8] = good[:8]
        assert rejected(junk) == -4


def _alias_step_plain(x, sb, divider, slot_adjust, slot_freqs, sym_id):
    """RansDecGetAlias (main_alias.cpp:252-267) on the bucket entry the decode kernels stage in shared memory
    (alias_kernels.cuh, AliasDecEntry): returns (symbol, new state before renormalisation)."""
    xm = x & np.uint32((1 << sb) - 1)
    b = (xm >> np.uint32(sb - 8)).astype(np.int64)
    own = xm < divider[b]
    fs0 = (slot_freqs[2 * b] << np.uint32(8)) | sym_id[2 * b].astype(np.uint32)
    fs1 = (slot_freqs[2 * b + 1] << np.uint32(8)) | sym_id[2 * b + 1].astype(np.uint32)
    fs = np.where(own, fs1, fs0)
    adj = np.where(own, slot_adjust[2 * b + 1], slot_adjust[2 * b]) & np.uint32(0xffff)
    rem = (xm - adj) & np.uint32(0xffff)
    return (fs & np.uint32(0xff)), (fs >> np.uint32(8)) * (x >> np.uint32(sb)) + rem


def _alias_step_lean(x, sb, divider, slot_adjust, slot_freqs, sym_id):
    """The repacked entry of alias_kernels.cuh (alias_lean_entry / AliasDecoder<SB, LEAN = 1>::step_p): the own
    count sits at the top of word 0 above the own adjust, the comparison is made on x << (40 - sb)."""
    lb, k = sb - 8, 40 - sb
    bucket = np.arange(256, dtype=np.uint32)
    own_count = divider - (bucket << np.uint32(lb))
    none = own_count == 0
    adj_other = slot_adjust[0::2] & np.uint32(0xffff)
    adj_own = np.where(none, adj_other, slot_adjust[1::2] & np.uint32(0xffff))
    fs_other = (slot_freqs[0::2] << np.uint32(8)) | sym_id[0::2].astype(np.uint32)
    fs_own = np.where(none, fs_other, (slot_freqs[1::2] << np.uint32(8)) | sym_id[1::2].astype(np.uint32))
    w0 = ((own_count - np.uint32(1)) << np.uint32(k)) | adj_own
    b = ((x >> np.uint32(lb)) & np.uint32(0xff)).astype(np.int64)
    own = (x << np.uint32(k)) <= w0[b]
    fs = np.where(own, fs_own[b], fs_other[b])
    adj = np.where(own, w0[b], adj_other[b])
    rem = (x - adj) & np.uint32((1 << sb) - 1)
    return (fs & np.uint32(0xff)), (fs >> np.uint32(8)) * (x >> np.uint32(sb)) + rem


@pytest.mark.parametrize("sb", [12, 14, 16])
@pytest.mark.parametrize("kind", ["zipf", "two_symbols", "one_symbol", "uniform"])
def test_alias_lean_entry_is_equivalent(gen, sb, kind):
    """Every slot value x & ((1 << sb) - 1), under arbitrary upper state bits, decodes to the same symbol and the same
    next state through the repacked bucket entry as through the plain one (the GPU A/B of the two is in
    tools/decode_lab.cu --coder alias; the GPU parity tests cover whichever one the library was built with)."""
    if kind == "zipf":
        data = gen("zipf", 50000, sb)
    elif kind == "two_symbols":
        data = np.concatenate([np.full(40000, 7, np.uint8), np.full(3, 250, np.uint8)])
    elif kind == "one_symbol":
        data = np.full(1000, 99, np.uint8)
    else:
        data = np.arange(1 << 16, dtype=np.uint32).astype(np.uint8)
    st = rb.SymbolStats().count_freqs(data).normalize_freqs(1 << sb).make_alias_table()
    rng = np.random.default_rng(sb)
    with np.errstate(over="ignore"):
        for _ in range(3):
            hi = rng.integers(1 << (23 - sb), 1 << (31 - sb), size=1 << sb, dtype=np.uint32)
            x = (hi << np.uint32(sb)) | np.arange(1 << sb, dtype=np.uint32)
            s0, x0 = _alias_step_plain(x, sb, st.divider, st.slot_adjust, st.slot_freqs, st.sym_id)
            s1, x1 = _alias_step_lean(x, sb, st.divider, st.slot_adjust, st.slot_freqs, st.sym_id)
            assert np.array_equal(s0, s1) and np.array_equal(x0, x1)
            # and both are the reference's arithmetic, main_alias.cpp:258-266, modulo 2^32
            xm = x & np.uint32((1 << sb) - 1)
            b2 = 2 * (xm >> np.uint32(sb - 8)).astype(np.int64)
            b2 += xm < st.divider[b2 // 2]
            assert np.array_equal(x0, st.slot_freqs[b2] * (x >> np.uint32(sb)) + xm - st.slot_adjust[b2])
            assert np.array_equal(s0, st.sym_id[b2])
