"""rb200_container_stored_encode_varlen_async and rb200_container_blocks_stored_encode_varlen_async: the stored encodes
(versions 6 and 5) with the length or the block count read from device memory when the work runs, so one captured graph
writes a bounded container of any size up to the bound.

- Byte equality with the fixed stored call: version 6 over every data kind of the stored test, chunks of 32, 33, 4096
  and 8192, the three candidate lists and one candidate, flags 0 and blob CRC, lengths 1, chunk_syms - 1, chunk_syms,
  chunk_syms + 1, n_max - 1 and n_max with n_max a ragged length and about four times it (so the bitmap's padding words
  and the pad in front of the bitmap fall elsewhere for the bound than for the length); version 5 over its kinds and
  half-uniform blocks, the device-count encode's geometries and lists, counts 1, max - 1 and max with the bound at one
  and four times the base count.  Nothing past the container is written.
- A few containers of each version equal the container packed from the oracle's streams, for every coder.
- Past 256 scan tiles (the tile prefix runs from the bound's count) with the size below and at the bound.
- One graph of the varlen encode and the stored decode follows sizes 1, mid, bound, mid on data that changes which
  chunks or blocks are stored.
- out_cap = the stored bound of the bound holds every size; an out_cap the blob does not fit is -3, header unwritten.
- Bad sizes write nothing; argument errors launch nothing; launch counts are pinned."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_stored as cs  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_blocks_auto as gba  # noqa: E402
import test_gpu_container_blocks_stored as gbs  # noqa: E402
import test_gpu_container_blocks_varlen as gbv  # noqa: E402
import test_gpu_container_stored as gs  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
THREE6 = gs.THREE
LISTS6 = gs.LISTS + [[CAND(ALIAS, 14)]]
THREE5 = gbs.THREE


def _torch():
    import torch
    return torch


def _dn(value, dtype=None):
    torch = _torch()
    return torch.tensor([value], dtype=dtype or torch.int64, device="cuda")


# ---- version 6

def fixed6(ctx, cands, tol, d_in, n, ch, flags):
    """the fixed stored call's container for the first n symbols of d_in"""
    torch = _torch()
    cap = api.container_stored_bound(n, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_stored_encode_async(cands, tol, d_in.data_ptr(), n, ch, flags, d_out.data_ptr(), cap)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    buf = d_out.cpu().numpy()
    return buf[:gs.size_of(buf)]


def varlen6(ctx, cands, tol, d_in, n, n_max, ch, flags, cap=None):
    """(sync code, whole output buffer): the varlen encode of *d_n = n into a sentinel-filled buffer of cap + 64 bytes"""
    torch = _torch()
    cap = api.container_stored_bound(n_max, ch) if cap is None else cap
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = _dn(n)
    ctx.container_stored_encode_varlen_async(cands, tol, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


def _lengths(ch, n_max):
    return sorted(x for x in {1, ch - 1, ch, ch + 1, n_max - 1, n_max} if 1 <= x <= n_max)


def _pads(n_chunks):
    """(bitmap words with their padding, whether a pad sits between directory and bitmap)"""
    return ((n_chunks + 31) // 32 + 3) & ~3, (1088 + 8 * (n_chunks + 1)) % 16 != 0


@pytest.mark.parametrize("ch", [32, 33, 4096, 8192])
@pytest.mark.parametrize("kind", gs.KINDS)
def test_v6_varlen_equals_the_fixed_call(gpu_ctx, kind, ch):
    base = (6 * ch if ch > 64 else 300 * ch) + 17
    bounds = (base, 4 * base + 3)
    data = gs.data_of(kind, bounds[-1], ch, gs.KINDS.index(kind))
    d_in = gbc._dev(data)
    layouts = set()
    for li, cands in enumerate(LISTS6):
        tol = 20000 if li % 2 else 0
        for flags in (0, CRC_BLOB):
            fixed = {}
            for n_max in bounds:
                for n in _lengths(ch, n_max):
                    case = (kind, ch, li, flags, n_max, n)
                    if n not in fixed:
                        fixed[n] = fixed6(gpu_ctx, cands, tol, d_in, n, ch, flags)
                    rc, got = varlen6(gpu_ctx, cands, tol, d_in, n, n_max, ch, flags)
                    assert rc == 0, case
                    want = fixed[n]
                    assert np.array_equal(got[:want.size], want), case
                    assert (got[want.size:] == SENTINEL).all(), case
                    layouts.add((_pads(-(-n // ch)) != _pads(-(-n_max // ch))))
    assert layouts == {True, False}


@pytest.mark.parametrize("coder,sb", [(WORD, 12), (BYTE, 14), (RANS64, 10), (ALIAS, 16)])
def test_v6_varlen_equals_the_oracle_packed_container(gpu_ctx, oracle_lib, coder, sb):
    ch = 1024
    n_max = ch * 40 + 333
    data = cs.mixed_data(n_max, 4096, 5)
    d_in = gbc._dev(data)
    for n in (ch * 7 + 5, n_max):
        for flags in (0, CRC_BLOB):
            want, st, pair = gs.expected(oracle_lib, [CAND(coder, sb)], 0, data[:n], ch, flags)
            rc, got = varlen6(gpu_ctx, [CAND(coder, sb)], 0, d_in, n, n_max, ch, flags)
            assert rc == 0 and st, (coder, n, flags)
            assert np.array_equal(got[:want.size], want), (coder, n, flags)
            assert (got[want.size:] == SENTINEL).all()


# ---- version 5

def fixed5(ctx, cands, tol, d_in, nb, bs, ch, flags):
    torch = _torch()
    cap = api.container_blocks_stored_bound(nb, bs, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_stored_encode_async(cands, tol, d_in.data_ptr(), nb, bs, ch, flags, d_out.data_ptr(), cap)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    buf = d_out.cpu().numpy()
    return buf[:gba._container_size(buf)]


def varlen5(ctx, cands, tol, d_in, nb, nb_max, bs, ch, flags, cap=None):
    torch = _torch()
    cap = api.container_blocks_stored_bound(nb_max, bs, ch) if cap is None else cap
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_nb = _dn(nb, torch.int32)
    ctx.container_blocks_stored_encode_varlen_async(cands, tol, d_in.data_ptr(), d_nb.data_ptr(), nb_max, bs, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


@pytest.mark.parametrize("kind", gbs.KINDS)
def test_v5_varlen_equals_the_fixed_call(gpu_ctx, kind):
    for gi, (nb, bs, ch) in enumerate(gbv.GEOMETRIES):
        data = gbs.block_data(kind, 4 * nb, bs, 20 * gi + gbs.KINDS.index(kind))
        d_in = gbc._dev(data)
        for cands, tol in gbv.LISTS:
            for flags in (0, CRC_BLOB):
                fixed = {}
                for nb_max in (nb, 4 * nb):
                    for count in gbv._counts(nb_max):
                        case = (kind, nb, bs, ch, cands, tol, flags, nb_max, count)
                        if count not in fixed:
                            fixed[count] = fixed5(gpu_ctx, cands, tol, d_in, count, bs, ch, flags)
                        rc, got = varlen5(gpu_ctx, cands, tol, d_in, count, nb_max, bs, ch, flags)
                        assert rc == 0, case
                        want = fixed[count]
                        assert struct.unpack_from("<H", got, 4)[0] == 5 and struct.unpack_from("<I", got, 56)[0] == count, case
                        assert np.array_equal(got[:want.size], want), case
                        assert (got[want.size:] == SENTINEL).all(), case


@pytest.mark.parametrize("coder,sb", [(WORD, 12), (BYTE, 14), (RANS64, 10), (ALIAS, 13)])
def test_v5_varlen_equals_the_oracle_packed_container(gpu_ctx, oracle_lib, coder, sb):
    nb_max, bs, ch = 7, 16384, 4096
    data = gbs.block_data("halfuniform", nb_max, bs, 11)
    d_in = gbc._dev(data)
    for count in (2, 7):
        for flags in (0, CRC_BLOB):
            want, st = gbs.expected(oracle_lib, [CAND(coder, sb)], 0, data[:count * bs], count, bs, ch, flags)
            rc, got = varlen5(gpu_ctx, [CAND(coder, sb)], 0, d_in, count, nb_max, bs, ch, flags)
            assert rc == 0 and st, (coder, count, flags)
            assert np.array_equal(got[:want.size], want), (coder, count, flags)
            assert (got[want.size:] == SENTINEL).all()


# ---- past 256 scan tiles

def _decoded(ctx, call, buf_t, size, n):
    torch = _torch()
    d_out = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = _dn(-1)
    call(buf_t.data_ptr(), size, d_out.data_ptr(), n, d_n.data_ptr())
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    assert int(d_n.item()) == n
    return d_out


def test_v6_past_256_tiles(gpu_ctx):
    torch = _torch()
    ch = 32
    n_max = 40 * 2 ** 20 + 7
    assert -(-n_max // ch) > 256 * 4096 and 8 * 2 ** 20 // ch <= 256 * 4096
    data = cs.mixed_data(n_max, 4096, 9)
    d_in = gbc._dev(data)
    cap = api.container_stored_bound(n_max, ch)
    d_buf = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    d_n = _dn(0)
    for n in (8 * 2 ** 20, n_max):
        fixed = fixed6(gpu_ctx, THREE6, 20000, d_in, n, ch, CRC_BLOB)
        d_buf.fill_(SENTINEL)
        d_n.fill_(n)
        gpu_ctx.container_stored_encode_varlen_async(THREE6, 20000, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0, n
        assert torch.equal(d_buf[:fixed.size], torch.from_numpy(fixed).cuda()), n
        assert bool((d_buf[fixed.size:] == SENTINEL).all().item()), n
        out = _decoded(gpu_ctx, gpu_ctx.container_stored_decode_async, d_buf, fixed.size, n)
        assert torch.equal(out[:n], d_in[:n]) and bool((out[n:] == SENTINEL).all().item()), n
    del d_buf, d_in


def test_v5_past_256_tiles(gpu_ctx):
    torch = _torch()
    bs, ch = 1024, 32
    nb_max = 40 * 1024 + 3
    assert nb_max * (bs // ch) > 256 * 4096 and 8192 * (bs // ch) <= 256 * 4096
    data = gbs.block_data("halfuniform", nb_max, bs, 3)
    d_in = gbc._dev(data)
    cap = api.container_blocks_stored_bound(nb_max, bs, ch)
    d_buf = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    d_nb = _dn(0, torch.int32)
    for count in (8192, nb_max):
        fixed = fixed5(gpu_ctx, THREE5, 20000, d_in, count, bs, ch, CRC_BLOB)
        d_buf.fill_(SENTINEL)
        d_nb.fill_(count)
        gpu_ctx.container_blocks_stored_encode_varlen_async(THREE5, 20000, d_in.data_ptr(), d_nb.data_ptr(), nb_max, bs, ch, CRC_BLOB,
                                                            d_buf.data_ptr(), cap)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0, count
        assert torch.equal(d_buf[:fixed.size], torch.from_numpy(fixed).cuda()), count
        assert bool((d_buf[fixed.size:] == SENTINEL).all().item()), count
        n = count * bs
        out = _decoded(gpu_ctx, gpu_ctx.container_blocks_stored_decode_async, d_buf, fixed.size, n)
        assert torch.equal(out[:n], d_in[:n]) and bool((out[n:] == SENTINEL).all().item()), count


# ---- one graph

def _half(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, n // 2, dtype=np.uint8)
    return np.concatenate([a, gs.data_of("zipf", n - a.size, 4096, seed)])


def test_v6_one_graph_many_lengths():
    torch = _torch()
    ch = 4096
    n_max = ch * 48 + 77
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_stored_bound(n_max, ch)
    d_in = torch.empty(n_max, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n_max + 64, dtype=torch.uint8, device="cuda")
    d_n = _dn(n_max)
    d_nsym = _dn(0)

    def round_trip():
        ctx.container_stored_encode_varlen_async(THREE6, 20000, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n_max, d_nsym.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(gs.data_of("zipf", n_max, ch, 1)))
        round_trip()                                                 # grows the workspace outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        stored = set()
        for step, (n, kind) in enumerate(((1, "uniform"), (ch * 13 + 1000, "zipf"), (n_max, "half"), (ch * 30 + 5, "uniform"))):
            data = _half(n, 50 + step) if kind == "half" else gs.data_of(kind, n, ch, 50 + step)
            d_in[:n].copy_(torch.from_numpy(data))
            d_n.fill_(n)
            d_buf.fill_(SENTINEL)
            d_out.fill_(SENTINEL)
            d_nsym.fill_(-1)
            launches = ctx.launches
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, n
            assert ctx.launches == launches                          # a replay does not go through the library
            fixed = fixed6(ctx, THREE6, 20000, d_in, n, ch, CRC_BLOB)
            got = d_buf.cpu().numpy()
            assert np.array_equal(got[:fixed.size], fixed) and (got[fixed.size:] == SENTINEL).all(), n
            assert int(d_nsym.item()) == n
            out = d_out.cpu().numpy()
            assert np.array_equal(out[:n], data) and (out[n:] == SENTINEL).all(), n
            n_chunks = -(-n // ch)
            bits = got[cs._bitmap_at(n_chunks):cs._bitmap_at(n_chunks) + 4 * ((n_chunks + 31) // 32)].view(np.uint32)
            stored.add(sum(bin(int(w)).count("1") for w in bits) / n_chunks)
        assert 1.0 in stored and len(stored) >= 3, stored
        del g
    ctx.close()


def test_v5_one_graph_many_counts():
    torch = _torch()
    nb_max, bs, ch = 12, 65536, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_blocks_stored_bound(nb_max, bs, ch)
    d_in = torch.empty(nb_max * bs, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nb_max * bs + 64, dtype=torch.uint8, device="cuda")
    d_nsym = _dn(0)
    d_nb = _dn(nb_max, torch.int32)

    def round_trip():
        ctx.container_blocks_stored_encode_varlen_async(THREE5, 20000, d_in.data_ptr(), d_nb.data_ptr(), nb_max, bs, ch, CRC_BLOB,
                                                        d_buf.data_ptr(), cap)
        ctx.container_blocks_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb_max * bs, d_nsym.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(gbs.block_data("zipf", nb_max, bs, 1)))
        round_trip()
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        stored = set()
        for step, (count, kind) in enumerate(((1, "uniform"), (5, "zipf"), (nb_max, "halfuniform"), (7, "uniform"))):
            data = gbs.block_data(kind, count, bs, 60 + step)
            d_in[:data.size].copy_(torch.from_numpy(data))
            d_nb.fill_(count)
            d_buf.fill_(SENTINEL)
            d_out.fill_(SENTINEL)
            d_nsym.fill_(-1)
            launches = ctx.launches
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, count
            assert ctx.launches == launches
            fixed = fixed5(ctx, THREE5, 20000, d_in, count, bs, ch, CRC_BLOB)
            got = d_buf.cpu().numpy()
            assert np.array_equal(got[:fixed.size], fixed) and (got[fixed.size:] == SENTINEL).all(), count
            assert int(d_nsym.item()) == count * bs
            out = d_out.cpu().numpy()
            assert np.array_equal(out[:data.size], data) and (out[data.size:] == SENTINEL).all(), count
            rows = got[64:64 + 512 * count].view(np.uint16).reshape(count, 256)
            stored.add(int((rows.sum(axis=1) == 0).sum()) / count)
        assert 1.0 in stored and len(stored) >= 3, stored
        del g
    ctx.close()


# ---- the bound, bad sizes, errors and launches

def test_v6_bound_holds_for_every_length(gpu_ctx):
    torch = _torch()
    ch = 8192
    n_max = ch * 64 + 99
    data = gs.data_of("uniform", n_max, ch, 3)
    d_in = gbc._dev(data)
    bound = api.container_stored_bound(n_max, ch)
    for n in (1, ch - 1, ch * 5 + 3, n_max // 16, n_max - 1, n_max):
        for cands in (THREE6, [CAND(WORD, 12)]):
            rc, got = varlen6(gpu_ctx, cands, 0, d_in, n, n_max, ch, CRC_BLOB, cap=bound)
            assert rc == 0, (n, cands)
            assert gs.size_of(got) == api.container_stored_bound(n, ch) and (got[bound:] == SENTINEL).all(), (n, cands)
    boff = cs.blob_offset(-(-n_max // ch))
    rc, got = varlen6(gpu_ctx, THREE6, 0, d_in, n_max, n_max, ch, 0, cap=boff + 4096)
    assert rc == -3 and (got[:64] == SENTINEL).all()


def test_v5_bound_holds_for_every_count(gpu_ctx):
    nb_max, bs, ch = 16, 65536, 8192
    data = gbs.block_data("uniform", nb_max, bs, 3)
    d_in = gbc._dev(data)
    bound = api.container_blocks_stored_bound(nb_max, bs, ch)
    for count in (1, 2, 9, nb_max - 1, nb_max):
        for cands in (THREE5, [CAND(WORD, 12)]):
            rc, got = varlen5(gpu_ctx, cands, 0, d_in, count, nb_max, bs, ch, CRC_BLOB, cap=bound)
            assert rc == 0, (count, cands)
            size = gba._container_size(got)
            assert size == api.container_blocks_stored_bound(count, bs, ch) and (got[bound:] == SENTINEL).all(), (count, cands)
    boff = (64 + 512 * nb_max + 8 * (nb_max * bs // ch + 1) + 15) & ~15
    rc, got = varlen5(gpu_ctx, THREE5, 0, d_in, nb_max, nb_max, bs, ch, 0, cap=boff + 4096)
    assert rc == -3 and (got[:64] == SENTINEL).all()


def test_bad_sizes_write_nothing(gpu_ctx):
    ch, n_max = 4096, 4096 * 10 + 5
    data = cs.mixed_data(n_max, ch, 4)
    d_in = gbc._dev(data)
    for cands in (THREE6, [CAND(BYTE, 14)]):
        for bad, want_rc in ((0, -2), (n_max + 1, -1)):
            for flags in (0, CRC_BLOB):
                rc, got = varlen6(gpu_ctx, cands, 0, d_in, bad, n_max, ch, flags)
                assert rc == want_rc and (got == SENTINEL).all(), (cands, bad, flags)
                rc, got = varlen6(gpu_ctx, cands, 0, d_in, n_max - 3, n_max, ch, flags)
                want = fixed6(gpu_ctx, cands, 0, d_in, n_max - 3, ch, flags)
                assert rc == 0 and np.array_equal(got[:want.size], want), (cands, bad, flags)
    nb_max, bs, ch = 5, 16384, 4096
    data = gbs.block_data("halfuniform", nb_max, bs, 4)
    d_in = gbc._dev(data)
    for cands in (THREE5, [CAND(ALIAS, 14)], [CAND(WORD, 12)]):
        for bad in (0, nb_max + 1):
            for flags in (0, CRC_BLOB):
                rc, got = varlen5(gpu_ctx, cands, 0, d_in, bad, nb_max, bs, ch, flags)
                assert rc == -1 and (got == SENTINEL).all(), (cands, bad, flags)
                rc, got = varlen5(gpu_ctx, cands, 0, d_in, 3, nb_max, bs, ch, flags)
                want = fixed5(gpu_ctx, cands, 0, d_in, 3, bs, ch, flags)
                assert rc == 0 and np.array_equal(got[:want.size], want), (cands, bad, flags)


def test_v6_argument_errors_and_launch_counts(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    ch = 8192
    n_max = ch * 40 + 5
    data = cs.mixed_data(n_max, ch, 1)
    d_in = gbc._dev(data)
    bound = api.container_stored_bound(n_max, ch)
    d_buf = torch.full((bound + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n_max, n_max - 100], dtype=torch.int64, device="cuda")
    i, o, p = d_in.data_ptr(), d_buf.data_ptr(), d_n.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, np_=p, nmax=n_max, chunk=ch, flags=0, out=o, out_cap=bound):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_stored_encode_varlen_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size, tol,
                                                              inp, np_, nmax, chunk, flags, out, out_cap)
    before = gpu_ctx.launches
    for bad in ([], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 17)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
        assert call(bad) == -1, bad
    assert call(THREE6, tol=10 ** 6 + 1) == -1
    for kw in ({"ctx": None}, {"inp": None}, {"out": None}, {"out": o + 8}, {"np_": None}, {"np_": p + 4}, {"nmax": 0},
               {"chunk": 31}, {"chunk": (1 << 24) + 1}, {"nmax": 1 << 32}):
        assert call(THREE6, **kw) == -1, kw
    boff = cs.blob_offset(-(-n_max // ch))
    assert call(THREE6, out_cap=boff - 1) == -3                      # below the blob offset of n_max
    assert gpu_ctx.launches == before
    assert (d_buf.cpu().numpy() == SENTINEL).all()
    # plan + histogram + choice + model + the groups' split encoders (word: two) + store + scan + compaction + meta CRC
    # + header; with the blob CRC also the blob length kernel and the blob CRC
    for cands, flags, want in ((THREE6, 0, 13), (THREE6, CRC_BLOB, 15), ([CAND(WORD, 12)], 0, 11), ([CAND(ALIAS, 12)], CRC_BLOB, 12)):
        before = gpu_ctx.launches
        assert call(cands, flags=flags, np_=p + 8) == 0
        assert gpu_ctx.launches - before == want, (cands, flags)
        assert lib.rb200_sync(gpu_ctx.h) == 0
        fixed = fixed6(gpu_ctx, cands, 0, d_in, n_max - 100, ch, flags)
        assert np.array_equal(d_buf[:fixed.size].cpu().numpy(), fixed), (cands, flags)


def test_v5_argument_errors_and_launch_counts(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    nb_max, bs, ch = 8, 65536, 8192
    data = gbs.block_data("halfuniform", nb_max, bs, 2)
    d_in = gbc._dev(data)
    bound = api.container_blocks_stored_bound(nb_max, bs, ch)
    d_buf = torch.full((bound + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_nb = torch.tensor([nb_max, 3], dtype=torch.int32, device="cuda")
    i, o, p = d_in.data_ptr(), d_buf.data_ptr(), d_nb.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, nbp=p, nb=nb_max, block_size=bs, chunk=ch, flags=0, out=o, out_cap=bound):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_blocks_stored_encode_varlen_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None,
                                                                     c.size, tol, inp, nbp, nb, block_size, chunk, flags, out, out_cap)
    before = gpu_ctx.launches
    for bad in ([], [CAND(BYTE, 16)], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
        assert call(bad) == -1, bad
    assert call(THREE5, tol=10 ** 6 + 1) == -1
    for kw in ({"ctx": None}, {"inp": None}, {"out": None}, {"out": o + 8}, {"nbp": None}, {"nbp": p + 1}, {"nbp": p + 2}, {"nb": 0},
               {"chunk": 31}, {"chunk": 1000}, {"block_size": 33 * 32, "chunk": 32}, {"nb": 1 << 26, "block_size": 1024, "chunk": 32}):
        assert call(THREE5, **kw) == -1, kw
    boff = (64 + 512 * nb_max + 8 * (nb_max * bs // ch + 1) + 15) & ~15
    assert call(THREE5, out_cap=boff - 1) == -3
    assert gpu_ctx.launches == before
    assert (d_buf.cpu().numpy() == SENTINEL).all()
    # plan (+ memset) + choice + one split encoder per group + store + scan + compaction + meta CRC + header; with the
    # blob CRC also the blob length kernel and the blob CRC.  One candidate: the plan writes the choice record.
    for cands, flags, want in ((THREE5, 0, 10), (THREE5, CRC_BLOB, 12), ([CAND(WORD, 12)], 0, 7), ([CAND(ALIAS, 12)], CRC_BLOB, 9)):
        before = gpu_ctx.launches
        assert call(cands, flags=flags, nbp=p + 4) == 0
        assert gpu_ctx.launches - before == want, (cands, flags)
        assert lib.rb200_sync(gpu_ctx.h) == 0
        fixed = fixed5(gpu_ctx, cands, 0, d_in, 3, bs, ch, flags)
        assert np.array_equal(d_buf[:fixed.size].cpu().numpy(), fixed), (cands, flags)
