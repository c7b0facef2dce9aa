"""The stored containers, versions 5 and 6, at the geometries and sizes where their kernels could go wrong unseen.

Every container the GPU encodes is compared byte for byte with the one packed from the oracle's streams with the store
rule applied in Python (or, past 2^32, with an exactly known expected container), and every case first asserts the
edge it claims to reach.

1. Version 5 at every block geometry of test_gpu_blocks_geometry and every one of its dispatch instances: the encode
   (one forced pair, nothing written past the container); the stored decode of the GPU's container and of containers
   with none, all, the first, the last and every other block stored; a stored chunk's padding byte and a shortened
   stored step rejected with out untouched; one CUDA graph of encode and decode at TWO and RAGGED_UNALIGNED.
2. Version 6 at chunks of 8193, 65536 and 2^17 (lengths whole, +1, +15, chunk - 1) for the four coders and at 2^24 with
   a ragged chunk; each of the eleven version 6 decoders on a stored first chunk, coded chunks, a stored ragged last
   chunk, and a coded last chunk next to a stored one, at chunks of 33 and 65536.
3. The store rules' exact ties (test_stored_ties): the tie stays coded, one step over is stored.
4. Inputs 1-15 bytes past 16-byte alignment, at the end of their allocation.
5. Past 1 Mi chunks: 256 scan tiles (summed by warp 0) and 257 (tile_prefix_kernel), bitmaps past 32 768 words.
6. Blob offsets at and past 2^32: version 6 of 2^32 - 1 uniform symbols, version 5 of 520 blocks of 2^23.

Sections 5 and 6 each take a context of their own, closed after the case, so that their workspaces (up to
n_chunks x slot bytes, about 11 GB) are returned; section 6 skips when the shared GPU lacks the free memory."""
import os
import struct
import sys

import numpy as np
import pytest

import oracle as orc
import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks_coder as cc  # noqa: E402
import test_container_blocks_stored as cbs  # noqa: E402
import test_container_stored as cs  # noqa: E402
import test_gpu_blocks_geometry as gg  # noqa: E402
import test_stored_ties as ties  # noqa: E402
from conftest import _gen  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = gg.SENTINEL
THREE = [CAND(WORD, 12), CAND(ALIAS, 16), CAND(BYTE, 14)]
r16 = cs.r16


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def ctx(cuda_box):
    """this module's own context, so that its workspaces are freed when the module ends"""
    c = rb.Context(0)
    try:
        yield c
    finally:
        c.close()


def _sync(ctx):
    return ctx.lib.dll.rb200_sync(ctx.h)


def _decode(ctx, call, d_buf, size, n):
    """(sync code, *d_n_symbols, out): an async decode of d_buf into n + 64 sentinel bytes"""
    torch = _torch()
    d_out = torch.full((n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    call(d_buf.data_ptr(), size, d_out.data_ptr(), n, d_n.data_ptr())
    return _sync(ctx), int(d_n.item()), d_out


def _decodes_to(ctx, call, d_buf, size, data, what):
    rc, got_n, d_out = _decode(ctx, call, d_buf, size, data.size)
    assert rc == 0 and got_n == data.size, (what, rc, got_n)
    out = d_out.cpu().numpy()
    assert np.array_equal(out[:data.size], data), (what, int(np.flatnonzero(out[:data.size] != data)[0]))
    assert (out[data.size:] == SENTINEL).all(), (what, "written past n")


def _rejects(ctx, call, buf, n, what):
    rc, got_n, d_out = _decode(ctx, call, gg._dev_at(buf), buf.size, n)
    assert rc == -4, (what, rc)
    assert bool((d_out == SENTINEL).all().item()), (what, "out written")


# ---------------------------------------------------------------------------------------------------- 1. version 5

def v5_container(oracle_lib, inst, geo, which=None, flags=0):
    """(container, block_freqs, offsets, stored blocks): the oracle's streams at `geo`, `which` (default: the rule's)
    stored"""
    nb, bs, ch = geo
    freqs, offs, blob = gg.oracle_streams(oracle_lib, inst, geo)
    f5, o5, b5, st = cbs.apply_store(freqs, offs, blob, gg.block_data(geo), nb, bs, ch, which)
    return api.container_blocks_stored_pack(inst.coder, inst.sb, nb, bs, ch, f5, o5, b5, flags), f5, o5, st


def v5_encode(ctx, cands, in_ptr, geo, flags, tol=0):
    """(sync code, device buffer of bound + 64 bytes, sentinel-filled before the encode)"""
    torch = _torch()
    nb, bs, ch = geo
    cap = api.container_blocks_stored_bound(nb, bs, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_stored_encode_async(cands, tol, in_ptr, nb, bs, ch, flags, d_out.data_ptr(), cap)
    return _sync(ctx), d_out


def v5_blob_offset(nb, n_chunks):
    return (64 + 512 * nb + 8 * (n_chunks + 1) + 15) & ~15


@pytest.mark.parametrize("inst,geo", gg.CASES, ids=[gg._cid(c) for c in gg.CASES])
def test_v5_geometry(ctx, oracle_lib, inst, geo):
    nb, bs, ch = geo
    n, per = nb * bs, bs // ch
    data = gg.block_data(geo)
    flags = (nb + bs + inst.sb) & 1
    want, f5, o5, st = v5_container(oracle_lib, inst, geo, flags=flags)
    if ch <= 33:
        # a 32- or 33-symbol chunk stores in 32 or 48 bytes, below any stream header (128 B; 256 B for rans64)
        assert st == list(range(nb)), st
    elif nb == 1:
        assert st == [], st                                           # one Zipf block
    else:
        assert 0 < len(st) < nb, st                                   # stored and coded blocks side by side
    d_in = gg._dev_at(data)
    rc, d_out = v5_encode(ctx, [CAND(inst.coder, inst.sb)], d_in.data_ptr(), geo, flags)
    assert rc == 0
    got = d_out.cpu().numpy()
    gg.same("version 5 container", inst, geo, got[:want.size], want)
    assert (got[want.size:] == SENTINEL).all(), "written past the container"
    call = ctx.container_blocks_stored_decode_async
    _decodes_to(ctx, call, d_out, want.size, data, "the GPU's container")
    for name, which in (("none", []), ("all", range(nb)), ("first", [0]), ("last", [nb - 1]), ("alternating", range(0, nb, 2))):
        buf = v5_container(oracle_lib, inst, geo, which)[0]
        _decodes_to(ctx, call, gg._dev_at(buf), buf.size, data, name)
    # one stored chunk broken: a padding byte set (where round16(chunk_syms) > chunk_syms), its step shortened by 16
    buf, _, o5, _ = v5_container(oracle_lib, inst, geo, range(nb))
    boff = v5_blob_offset(nb, o5.size - 1)
    c = (nb // 2) * per + per // 2
    if ch % 16:
        bad = buf.copy()
        bad[boff + int(o5[c]) + ch] = 1                               # no CRC covers a stored chunk's padding (flags 0)
        _rejects(ctx, call, bad, n, "padding")
    bad = buf.copy()
    struct.pack_into("<Q", bad, 64 + 512 * nb + 8 * c, int(o5[c]) + 16)
    _rejects(ctx, call, cc.reseal(bad), n, "step")


GRAPH_CASES = [(gg.BYTE[12], gg.TWO), (gg.ALIAS[11], gg.TWO), (gg.WORD, gg.RAGGED_UNALIGNED), (gg.RANS64[14], gg.RAGGED_UNALIGNED)]


@pytest.mark.parametrize("inst,geo", GRAPH_CASES, ids=[gg._cid(c) for c in GRAPH_CASES])
def test_v5_encode_and_decode_in_one_cuda_graph(cuda_box, oracle_lib, inst, geo):
    """replayed on data whose stored blocks change (at TWO; at RAGGED_UNALIGNED every block is always stored), each
    replay's container equal to the oracle-packed one"""
    torch = _torch()
    nb, bs, ch = geo
    n = nb * bs
    stream = torch.cuda.Stream()
    c = rb.Context(0, stream=stream.cuda_stream)
    g = None
    try:
        cap = api.container_blocks_stored_bound(nb, bs, ch)
        d_in = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
        d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
        d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
        d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

        def round_trip():
            c.container_blocks_stored_encode_async([CAND(inst.coder, inst.sb)], 0, d_in.data_ptr(), nb, bs, ch, CRC_BLOB, d_buf.data_ptr(), cap)
            c.container_blocks_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

        with torch.cuda.stream(stream):
            d_in[:n].copy_(torch.from_numpy(gg.block_data(geo).copy()))
            round_trip()                                              # grows the workspace outside the capture
            assert _sync(c) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                round_trip()
            seen = set()
            for seed in (71, 72, 73):
                kinds = ["uniform", "const", "zipf", "two", "uniform", "text"]
                data = np.concatenate([_gen(kinds[(b + seed) % len(kinds)], bs, seed * 100 + b) for b in range(nb)])
                f, o, b_ = cc.oracle_blocks_encode(oracle_lib, inst.ocoder, inst.sb, data, nb, bs, ch)
                f5, o5, b5, st = cbs.apply_store(f, o, b_, data, nb, bs, ch)
                want = api.container_blocks_stored_pack(inst.coder, inst.sb, nb, bs, ch, f5, o5, b5, CRC_BLOB)
                d_in[:n].copy_(torch.from_numpy(data))
                d_out.zero_()
                d_n.zero_()
                g.replay()
                assert _sync(c) == 0
                gg.same(f"graph replay {seed}: container", inst, geo, d_buf[:want.size].cpu().numpy(), want)
                assert int(d_n.item()) == n
                gg.same(f"graph replay {seed}: decode", inst, geo, d_out[:n].cpu().numpy(), data)
                seen.add(tuple(st))
            if ch <= 33:
                assert seen == {tuple(range(nb))}
            else:
                assert len(seen) == 3, seen
    finally:
        stream.synchronize()
        del g
        c.close()


# ---------------------------------------------------------------------------------------------------- 2. version 6

def v6_container(oracle_lib, coder, sb, data, ch, which=None, flags=0):
    """(container, stored chunks, freqs): the oracle's streams of data, `which` (default: the rule's) stored"""
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, ch)
    bits, o6, b6, st = cs.apply_store(data, ch, offs, blob, which)
    return api.container_stored_pack(coder, sb, ch, data.size, freqs, bits, o6, b6, flags), st, freqs


def v6_encode(ctx, cands, in_ptr, n, ch, flags, tol=0):
    torch = _torch()
    cap = api.container_stored_bound(n, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_stored_encode_async(cands, tol, in_ptr, n, ch, flags, d_out.data_ptr(), cap)
    return _sync(ctx), d_out


def _v6_check(ctx, oracle_lib, coder, sb, data, ch, flags, what):
    want, st, _ = v6_container(oracle_lib, coder, sb, data, ch, flags=flags)
    d_in = gg._dev_at(data)
    rc, d_out = v6_encode(ctx, [CAND(coder, sb)], d_in.data_ptr(), data.size, ch, flags)
    assert rc == 0, what
    got = d_out.cpu().numpy()
    if not np.array_equal(got[:want.size], want):
        i = int(np.flatnonzero(got[:want.size] != want)[0])
        pytest.fail(f"{what}: container differs from byte {i} of {want.size} (blob at {cs.blob_offset(-(-data.size // ch))})")
    assert (got[want.size:] == SENTINEL).all(), what
    _decodes_to(ctx, ctx.container_stored_decode_async, d_out, want.size, data, what)
    return st


V6_PAIRS = [(WORD, 12), (BYTE, 14), (ALIAS, 16), (RANS64, 15)]


@pytest.mark.parametrize("ch", [8193, 65536, 1 << 17])
@pytest.mark.parametrize("coder,sb", V6_PAIRS)
def test_v6_chunks_above_8192(ctx, oracle_lib, coder, sb, ch):
    for extra in (0, 1, 15, ch - 1):
        n = 4 * ch + extra
        data = cs.mixed_data(n, ch, 40 + extra % 7)
        st = _v6_check(ctx, oracle_lib, coder, sb, data, ch, extra & 1, (coder, sb, ch, n))
        assert 0 < len(st) < -(-n // ch), (ch, n, st)                  # stored and coded chunks side by side


@pytest.mark.parametrize("coder,sb", [(WORD, 12), (BYTE, 14)])
def test_v6_largest_chunk_and_a_ragged_one(ctx, oracle_lib, coder, sb):
    ch = 1 << 24
    data = np.concatenate([_gen("zipf", ch, 3), _gen("uniform", (1 << 23) + 5, 4)])
    assert _v6_check(ctx, oracle_lib, coder, sb, data, ch, CRC_BLOB, (coder, ch)) == [1]


# the eleven version 6 decoders (rb200_container_stored_decode_async picks one by coder, scale_bits and, for the word
# coder, whether a symbol holds all 4096 slots)
DECODERS = [("word", WORD, 12), ("word-wide", WORD, 12), ("alias16", ALIAS, 16), ("alias14", ALIAS, 14), ("alias12", ALIAS, 12),
            ("alias-generic", ALIAS, 11), ("byte16", BYTE, 16), ("byte14", BYTE, 14), ("byte12", BYTE, 12), ("byte-generic", BYTE, 9),
            ("rans64", RANS64, 15)]


@pytest.mark.parametrize("ch", [33, 65536])
@pytest.mark.parametrize("name,coder,sb", DECODERS, ids=[d[0] for d in DECODERS])
def test_v6_each_decoder_on_stored_and_coded_chunks(ctx, oracle_lib, name, coder, sb, ch):
    n = 20 * ch + 7 if ch == 33 else 4 * ch + 1000                       # a ragged last chunk
    n_chunks = -(-n // ch)
    data = _gen("const", n, 0) if name == "word-wide" else cs.mixed_data(n, max(ch, 1024), 8)
    for which in ([0, n_chunks - 1], [n_chunks - 2]):                   # stored first and ragged last; coded last beside a stored one
        buf, st, freqs = v6_container(oracle_lib, coder, sb, data, ch, which, CRC_BLOB)
        meta = api.container_stored_open(buf)[0]
        assert (meta["coder"], meta["scale_bits"], meta["n_chunks"]) == (coder, sb, n_chunks)
        if coder == WORD:                                              # narrow or WIDE: a symbol at frequency 4096 or not
            assert (int(np.max(freqs)) == 4096) == (name == "word-wide"), name
        _decodes_to(ctx, ctx.container_stored_decode_async, gg._dev_at(buf), buf.size, data, (name, ch, which))


# ---------------------------------------------------------------------------------------------------- 3. ties

@pytest.mark.parametrize("edge", list(ties.EDGES))
def test_v6_store_rule_tie(ctx, oracle_lib, edge):
    data, _, _, _ = ties.v6_case(oracle_lib, edge)                       # asserts both targets on the edge
    st = _v6_check(ctx, oracle_lib, *ties.V6_PAIR, data, ties.V6_CH, 0, edge)
    for c in ties.V6_TARGETS:
        assert (c in st) == (edge == "over"), (edge, c, st)


@pytest.mark.parametrize("edge", list(ties.EDGES))
def test_v5_store_rule_tie(ctx, oracle_lib, edge):
    nb, bs, ch = ties.V5_GEO
    coder, sb = ties.V5_PAIR
    data, freqs, offs, blob = ties.v5_case(oracle_lib, edge)             # asserts the block on the edge
    f5, o5, b5, st = cbs.apply_store(freqs, offs, blob, data, nb, bs, ch)
    assert (ties.V5_TARGET in st) == (edge == "over"), (edge, st)
    want = api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, CRC_BLOB)
    d_in = gg._dev_at(data)
    rc, d_out = v5_encode(ctx, [CAND(coder, sb)], d_in.data_ptr(), ties.V5_GEO, CRC_BLOB)
    assert rc == 0
    got = d_out.cpu().numpy()
    assert np.array_equal(got[:want.size], want), (edge, int(np.flatnonzero(got[:want.size] != want)[0]))
    _decodes_to(ctx, ctx.container_blocks_stored_decode_async, d_out, want.size, data, edge)


# ---------------------------------------------------------------------------------------------------- 4. misaligned input

def _at_end(data, k):
    """data k bytes past a 16-byte boundary, ending its allocation"""
    torch = _torch()
    t = torch.empty(k + data.size, dtype=torch.uint8, device="cuda")
    t[k:] = torch.from_numpy(data)
    return t


def _poisoned(data):
    """data aligned, followed by 64 bytes that would change the model, and a stored chunk's padding, if read"""
    return gg._dev_at(data, 0, 64, fill=0xFF)


@pytest.mark.parametrize("ch", [4096, 33])
def test_v6_misaligned_input(ctx, oracle_lib, ch):
    n = 40 * ch + 17 if ch > 64 else 300 * ch + 17
    data = cs.mixed_data(n, max(ch, 4096), 12)
    torch = _torch()
    import test_gpu_container_stored as gcs
    want, st, _ = gcs.expected(oracle_lib, THREE, 0, data, ch, CRC_BLOB)
    if ch > 64:
        assert 0 < len(st) < -(-n // ch), st
    else:
        assert len(st) == -(-n // ch)                                  # 33-symbol chunks: all stored
    d_ref = _poisoned(data)
    rc, d_out = v6_encode(ctx, THREE, d_ref.data_ptr(), n, ch, CRC_BLOB)
    assert rc == 0 and np.array_equal(d_out[:want.size].cpu().numpy(), want), "aligned"
    for k in (1, 3, 8, 15):
        d_in = _at_end(data, k)
        rc, d_k = v6_encode(ctx, THREE, d_in.data_ptr() + k, n, ch, CRC_BLOB)
        assert rc == 0 and torch.equal(d_k, d_out), k


@pytest.mark.parametrize("geo", [gg.NINE, gg.SIXTEEN], ids=gg._gid)
def test_v5_misaligned_input(ctx, oracle_lib, geo):
    import test_gpu_container_blocks_stored as gcbs
    torch = _torch()
    three = gcbs.THREE                                                 # the per-block coders' list (alias at 14)
    nb, bs, ch = geo
    data = np.array(gg.block_data(geo))
    want, st = gcbs.expected(oracle_lib, three, 0, data, nb, bs, ch, CRC_BLOB)
    assert 0 < len(st) < nb, st
    d_ref = _poisoned(data)
    rc, d_out = v5_encode(ctx, three, d_ref.data_ptr(), geo, CRC_BLOB)
    assert rc == 0 and np.array_equal(d_out[:want.size].cpu().numpy(), want), "aligned"
    for k in (1, 8):
        d_in = _at_end(data, k)
        rc, d_k = v5_encode(ctx, three, d_in.data_ptr() + k, geo, CRC_BLOB)
        assert rc == 0 and torch.equal(d_k, d_out), k


# ---------------------------------------------------------------------------------------------------- 5. past 1 Mi chunks

SCAN_TILE = 4096
MI = 1 << 20


def regions(n, seed):
    """'two' and uniform runs whose boundaries fall anywhere: 'two' runs of 600-3000 symbols (three quarters of the
    input, so that a 160-symbol 'two' chunk codes to little more than its stream header), uniform ones of 200-1000"""
    rng = np.random.default_rng(seed)
    k = n // 600 + 2
    lengths = np.empty(2 * k, np.int64)
    lengths[0::2] = rng.integers(600, 3000, k)
    lengths[1::2] = rng.integers(200, 1000, k)
    uniform = np.repeat(np.tile([False, True], k), lengths)[:n]
    two = np.where(rng.random(n, dtype=np.float32) < 0.001, 7, 200).astype(np.uint8)
    return np.where(uniform, rng.integers(0, 256, n, dtype=np.uint8), two)


def v6_expected_large(data, ch, offs, blob):
    """(bits, offsets, blob, stored mask) of cs.apply_store, vectorised: runs of coded chunks are moved as one slice"""
    n = data.size
    n_chunks = offs.size - 1
    ends = offs[1:].astype(np.int64) & ~15
    sizes = ends - offs[:-1].astype(np.int64)
    m = np.full(n_chunks, ch, np.int64)
    m[-1] = n - (n_chunks - 1) * ch
    stored = ((sizes + 15) & ~15) > ((m + 15) & ~15)
    new = np.where(stored, (m + 15) & ~15, sizes)
    e6 = np.cumsum((new + 15) & ~15)
    o6 = np.concatenate([e6 - new, e6[-1:]]).astype(np.uint64)
    b6 = np.zeros(int(e6[-1]), np.uint8)
    start6 = np.concatenate([[0], e6[:-1]])
    start = np.concatenate([[0], ends[:-1]])
    flips = np.flatnonzero(np.diff(stored.astype(np.int8))) + 1
    for c0, c1 in zip(np.concatenate([[0], flips]), np.concatenate([flips, [n_chunks]])):
        if stored[c0]:
            last = c1 == n_chunks and m[-1] != ch
            c1w = c1 - 1 if last else c1                                # whole chunks of ch symbols (ch % 16 == 0)
            b6[start6[c0]:start6[c0] + (c1w - c0) * ch] = data[c0 * ch:c1w * ch]
            if last:
                b6[int(o6[-2]):int(o6[-2]) + m[-1]] = data[(n_chunks - 1) * ch:]
        else:
            b6[start6[c0]:e6[c1 - 1]] = blob[start[c0]:ends[c1 - 1]]
    words = (n_chunks + 31) // 32
    bits = np.packbits(np.concatenate([stored, np.zeros(32 * words - n_chunks, bool)]), bitorder="little").view("<u4")
    return bits, o6, b6, stored


V6_LARGE = [(WORD, MI, 160), (BYTE, MI, 160), (WORD, MI + 1, 77), (BYTE, MI + 1, 77), (WORD, MI + 33, 100), (BYTE, MI + 33, 100)]


@pytest.mark.parametrize("coder,n_chunks,last", V6_LARGE, ids=[f"{'word' if c == WORD else 'byte'}-{k}" for c, k, _ in V6_LARGE])
def test_v6_past_1mi_chunks(cuda_box, oracle_lib, coder, n_chunks, last):
    torch = _torch()
    ch, sb = 160, 12 if coder == WORD else 14
    n = (n_chunks - 1) * ch + last
    tiles = -(-n_chunks // SCAN_TILE)
    assert tiles == (256 if n_chunks == MI else 257)                  # warp 0 sums 256 tiles; tile_prefix_kernel above
    data = regions(n, n_chunks)
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, ch)
    bits, o6, b6, stored = v6_expected_large(data, ch, offs, blob)
    assert stored.sum() > 100000 and (~stored).sum() > 100000, stored.sum()
    assert stored[-1] or last >= 128                                   # a short ragged chunk is stored
    words = (n_chunks + 31) // 32
    assert words > 32768 or n_chunks == MI
    want = api.container_stored_pack(coder, sb, ch, n, freqs, bits, o6, b6, 0)
    c = rb.Context(0)
    try:
        d_in = gg._dev_at(data)
        rc, d_out = v6_encode(c, [CAND(coder, sb)], d_in.data_ptr(), n, ch, 0)
        assert rc == 0
        got = d_out.cpu().numpy()
        if not np.array_equal(got[:want.size], want):
            i = int(np.flatnonzero(got[:want.size] != want)[0])
            boff = cs.blob_offset(n_chunks)
            where = (f"directory entry {(i - 1088) // 8} (tile {(i - 1088) // 8 // SCAN_TILE})" if i < cs._bitmap_at(n_chunks) else
                     f"bitmap word {(i - cs._bitmap_at(n_chunks)) // 4}" if i < boff else
                     f"blob, chunk {int(np.searchsorted(o6, i - boff, side='right')) - 1}")
            pytest.fail(f"container differs from byte {i}: {where}")
        assert (got[want.size:] == SENTINEL).all()
        rc, got_n, d_dec = _decode(c, c.container_stored_decode_async, d_out, want.size, n)
        assert rc == 0 and got_n == n and torch.equal(d_dec[:n], d_in[:n])
        assert bool((d_dec[n:] == SENTINEL).all().item())
        del d_dec
        # one bit flipped in the last bitmap word (past word 32 768 where there is one): past n_chunks, or a coded
        # chunk whose step is not a stored chunk's
        w = words - 1
        if n_chunks % 32:
            bit = n_chunks % 32
        else:
            cands = [k for k in range(32) if not stored[32 * w + k] and int(o6[32 * w + k + 1]) - int(o6[32 * w + k]) != r16(ch)]
            bit = cands[0]
        bm = cs._bitmap_at(n_chunks)
        head = got[:cs.blob_offset(n_chunks)].copy()
        head[bm + 4 * w:bm + 4 * w + 4].view("<u4")[0] ^= np.uint32(1 << bit)
        head = cs.reseal(head)                                          # flags 0: meta_crc alone
        d_out[:head.size] = torch.from_numpy(head).cuda()
        rc, _, d_dec = _decode(c, c.container_stored_decode_async, d_out, want.size, n)
        assert rc == -4 and bool((d_dec == SENTINEL).all().item()), rc
    finally:
        c.close()
        torch.cuda.empty_cache()


def v5_large_blocks(nb, seed):
    """(contents, pattern): 12 distinct 5120-symbol blocks (4 uniform, stored; 6 'two' and 2 const, coded) and which
    one each of nb blocks holds, drawn so that runs and tile boundaries do not line up"""
    bs = 32 * 160
    contents = ([_gen("uniform", bs, seed + j) for j in range(4)] + [_gen("two", bs, seed + 10 + j) for j in range(6)]
                + [_gen("const", bs, 0), np.full(bs, 9, np.uint8)])
    return contents, np.random.default_rng(seed).integers(0, len(contents), nb)


@pytest.mark.parametrize("coder,nb", [(WORD, 32768), (BYTE, 32768), (WORD, 32769), (BYTE, 32769)],
                         ids=["word-32768", "byte-32768", "word-32769", "byte-32769"])
def test_v5_past_1mi_chunks(cuda_box, oracle_lib, coder, nb):
    torch = _torch()
    per, ch = 32, 160
    bs, sb = per * ch, 12 if coder == WORD else 14
    n_chunks = nb * per
    assert -(-n_chunks // SCAN_TILE) == (256 if nb == 32768 else 257)
    contents, pattern = v5_large_blocks(nb, nb)
    ocoder = cbs.OCODER[coder]
    enc = []
    for blk in contents:
        f, cum = oracle_lib.model(blk, sb)
        b, o = oracle_lib.chunked_encode(ocoder, blk, f, cum, ch, scale_bits=sb)
        sizes = [s.size for s in cbs.streams(o, b)]
        enc.append((f, b, sizes, sum(r16(s) for s in sizes) > per * r16(ch)))
    verdicts = [e[3] for e in enc]
    assert verdicts[:4] == [True] * 4 and verdicts[4:10] == [False] * 6, verdicts     # uniform stored, 'two' coded
    data = np.concatenate([contents[j] for j in pattern])
    st = np.array([enc[j][3] for j in pattern])
    f5 = np.stack([np.zeros(256, np.uint16) if enc[j][3] else enc[j][0].astype(np.uint16) for j in pattern])
    sizes = np.concatenate([np.full(per, ch) if enc[j][3] else enc[j][2] for j in pattern]).astype(np.int64)
    e5 = np.cumsum((sizes + 15) & ~15)
    o5 = np.concatenate([e5 - sizes, e5[-1:]]).astype(np.uint64)
    b5 = np.concatenate([contents[j] if enc[j][3] else enc[j][1] for j in pattern])
    want = api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, 0)
    c = rb.Context(0)
    try:
        d_in = gg._dev_at(data)
        rc, d_out = v5_encode(c, [CAND(coder, sb)], d_in.data_ptr(), (nb, bs, ch), 0)
        assert rc == 0
        got = d_out.cpu().numpy()
        if not np.array_equal(got[:want.size], want):
            i = int(np.flatnonzero(got[:want.size] != want)[0])
            dir_off = 64 + 512 * nb
            where = (f"model row {(i - 64) // 512}" if i < dir_off else
                     f"directory entry {(i - dir_off) // 8} (tile {(i - dir_off) // 8 // SCAN_TILE})" if i < dir_off + 8 * (n_chunks + 1) else
                     f"blob, chunk {int(np.searchsorted(o5, i - v5_blob_offset(nb, n_chunks), side='right')) - 1}")
            pytest.fail(f"container differs from byte {i}: {where}")
        assert (got[want.size:] == SENTINEL).all()
        rc, got_n, d_dec = _decode(c, c.container_blocks_stored_decode_async, d_out, want.size, data.size)
        assert rc == 0 and got_n == data.size and torch.equal(d_dec[:data.size], d_in[:data.size])
        del d_dec
        # a stored chunk past chunk 1 Mi - 32 (the last tile) with its step shortened
        b = int(np.flatnonzero(st)[-1])
        k = b * per + 5
        head = got[:v5_blob_offset(nb, n_chunks)].copy()
        struct.pack_into("<Q", head, 64 + 512 * nb + 8 * k, int(o5[k]) + 16)
        head = cc.reseal(head)
        d_out[:head.size] = torch.from_numpy(head).cuda()
        rc, _, d_dec = _decode(c, c.container_blocks_stored_decode_async, d_out, want.size, data.size)
        assert rc == -4 and bool((d_dec == SENTINEL).all().item()), rc
    finally:
        c.close()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- 6. past 2^32

def _room(need):
    """the free device memory, after skipping the test when it is less than `need`"""
    torch = _torch()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"{need / 2**30:.1f} GiB of device memory needed, {free / 2**30:.1f} GiB free on the shared GPU")
    return free


def _report(what, free0):
    """print the device memory the case holds now (input, container, workspace and output all live)"""
    torch = _torch()
    print(f"{what}: {(free0 - torch.cuda.mem_get_info()[0]) / 2**30:.2f} GiB of device memory in use")


def _equal(a, b):
    """torch.equal over the first dimension in slices of about 256 Mi elements (the size of its bool temporary)"""
    torch = _torch()
    step = max(1, (1 << 28) // max(1, a[0].numel() if a.dim() > 1 else 1))
    return all(torch.equal(a[i:i + step], b[i:i + step]) for i in range(0, a.shape[0], step))


def _untouched(t):
    step = 1 << 28
    return all(bool((t[i:i + step] == SENTINEL).all().item()) for i in range(0, t.numel(), step))


def _slot_bytes(ch):
    return r16(512 + 2 * ch)


@pytest.mark.parametrize("ch", [8192, 1000])
def test_v6_blob_past_2_32(cuda_box, ch):
    """n = 2^32 - 1 uniform symbols, every chunk stored: the blob is the input, each chunk padded to round16(ch)"""
    torch = _torch()
    n = (1 << 32) - 1
    n_chunks = -(-n // ch)
    rch, last = r16(ch), n - (n_chunks - 1) * ch
    cap = api.container_stored_bound(n, ch)
    free0 = _room(2 * n + cap + n_chunks * _slot_bytes(ch) + (3 << 30))
    boff = cs.blob_offset(n_chunks)
    total = (n_chunks - 1) * rch + r16(last)
    assert cap == boff + total and total >= 1 << 32
    c = rb.Context(0)
    try:
        g = torch.Generator(device="cuda").manual_seed(ch)
        d_in = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
        d_buf = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        c.container_stored_encode_async([CAND(BYTE, 14)], 0, d_in.data_ptr(), n, ch, 0, d_buf.data_ptr(), cap)
        assert _sync(c) == 0
        head = d_buf[:boff].cpu().numpy()
        assert struct.unpack_from("<H", head, 4)[0] == 6
        assert struct.unpack_from("<QQQ", head, 16) == (n, n_chunks, total)
        want_dir = torch.arange(n_chunks + 1, dtype=torch.int64) * rch
        want_dir[-1] = total
        got_dir = torch.from_numpy(head[1088:1088 + 8 * (n_chunks + 1)].view(np.int64).copy())
        assert torch.equal(got_dir, want_dir) and int(got_dir[-1]) >= 1 << 32
        words = head[cs._bitmap_at(n_chunks):boff].view("<u4")
        full, part = divmod(n_chunks, 32)
        assert (words[:full] == 0xFFFFFFFF).all() and (words[full + (1 if part else 0):] == 0).all()
        assert not part or words[full] == (1 << part) - 1
        blob = d_buf[boff:boff + total]
        whole = n_chunks - 1
        assert _equal(blob[:whole * rch].view(whole, rch)[:, :ch], d_in[:whole * ch].view(whole, ch))
        assert not blob[:whole * rch].view(whole, rch)[:, ch:].any().item()
        assert torch.equal(blob[whole * rch:whole * rch + last], d_in[whole * ch:]) and not blob[whole * rch + last:].any().item()
        assert _untouched(d_buf[cap:])
        d_out = torch.full((n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        c.container_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())
        assert _sync(c) == 0 and int(d_n.item()) == n
        _report(f"version 6, n = 2^32 - 1, chunks of {ch}", free0)
        assert _equal(d_out[:n], d_in) and _untouched(d_out[n:])
        # one padding byte of a stored chunk past 2^32 in the container (flags 0: no CRC covers it)
        k = n_chunks - 1 if ch == 8192 else n_chunks - 2
        pos = boff + k * rch + (last if k == n_chunks - 1 else ch)
        assert pos >= 1 << 32
        d_buf[pos] = 1
        d_out.fill_(SENTINEL)
        c.container_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())
        assert _sync(c) == -4 and _untouched(d_out)
    finally:
        c.close()
        torch.cuda.empty_cache()


def test_v5_blob_past_4_gib(cuda_box, oracle_lib):
    """520 blocks of 2^23 symbols in chunks of 2^18: uniform blocks stored, their blob the input; const blocks coded,
    three of them before the 2^32 mark of the blob and three after it"""
    torch = _torch()
    nb, bs, ch, sb = 520, 1 << 23, 1 << 18, 14
    per, n = bs // ch, nb * bs
    n_chunks = nb * per
    const = [3, 509, 510, 516, 517, 519]
    cap = api.container_blocks_stored_bound(nb, bs, ch)
    free0 = _room(2 * n + cap + n_chunks * _slot_bytes(ch) + (3 << 30))
    blk = np.full(bs, 0x41, np.uint8)
    f, cum = oracle_lib.model(blk, sb)
    ob, oo = oracle_lib.chunked_encode(orc.CODER_BYTE, blk, f, cum, ch, scale_bits=sb)
    csizes = [s.size for s in cbs.streams(oo, ob)]
    sizes = np.concatenate([np.array(csizes) if b in const else np.full(per, ch) for b in range(nb)]).astype(np.int64)
    e5 = np.cumsum((sizes + 15) & ~15)
    o5 = np.concatenate([e5 - sizes, e5[-1:]]).astype(np.uint64)
    starts = [int(o5[b * per]) & ~15 for b in const]
    assert min(starts) < 1 << 32 and sum(s >= 1 << 32 for s in starts) == 3, starts
    boff = v5_blob_offset(nb, n_chunks)
    c = rb.Context(0)
    try:
        g = torch.Generator(device="cuda").manual_seed(5)
        d_in = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
        for b in const:
            d_in[b * bs:(b + 1) * bs] = 0x41
        d_buf = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        c.container_blocks_stored_encode_async([CAND(BYTE, sb)], 0, d_in.data_ptr(), nb, bs, ch, 0, d_buf.data_ptr(), cap)
        assert _sync(c) == 0
        head = d_buf[:boff].cpu().numpy()
        assert struct.unpack_from("<QQQ", head, 16) == (n, n_chunks, int(o5[-1]))
        rows = head[64:64 + 512 * nb].view(np.uint16).reshape(nb, 256)
        for b in range(nb):
            assert np.array_equal(rows[b], f) if b in const else not rows[b].any(), b
        assert np.array_equal(head[64 + 512 * nb:64 + 512 * nb + 8 * (n_chunks + 1)].view(np.uint64), o5)
        blob = d_buf[boff:boff + int(o5[-1])]
        for b in range(nb):
            lo = int(o5[b * per]) & ~15
            if b in const:
                assert np.array_equal(blob[lo:lo + ob.size].cpu().numpy(), ob), b
            else:
                assert torch.equal(blob[lo:lo + bs], d_in[b * bs:(b + 1) * bs]), b
        assert _untouched(d_buf[boff + int(o5[-1]):])
        del blob
        d_out = torch.full((n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        c.container_blocks_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())
        assert _sync(c) == 0 and int(d_n.item()) == n
        _report("version 5, 520 blocks of 2^23", free0)
        assert _equal(d_out[:n], d_in) and _untouched(d_out[n:])
    finally:
        c.close()
        torch.cuda.empty_cache()
