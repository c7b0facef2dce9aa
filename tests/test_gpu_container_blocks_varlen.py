"""rb200_container_blocks_model_encode_varlen_async: the per-block auto encode with the block count read from device
memory when the work runs, so one captured graph takes any count up to n_blocks_max.

- The container is byte for byte rb200_container_blocks_model_encode_auto_async's at n_blocks = *d_n_blocks, for one
  candidate of each version, {word 12, byte 14, alias 14} at tolerances 0 and 2 % and the sixteen-pair list, at four
  geometries, counts 1, max - 1 and max with n_blocks_max the count and four times it, flags 0 and blob CRC, over the
  data kinds of test_blocks_coder_choice; nothing past the container is written, and the costs of a list of two or more
  candidates are the host rule's over the first *d_n_blocks blocks.
- A few containers equal the container packed from the oracle's per-block streams (word, byte, rans64, alias).
- One captured graph of the encode and the any decode follows counts 1, mid, max, mid on skewed and Zipf blocks.
- Counts 0 and n_blocks_max + 1 are -1 from sync with out untouched, and the context is fine after them.
- Host argument errors launch nothing; a blob that does not fit out_cap is -3 with the header unwritten; launch counts
  are pinned, with no choice kernel for one candidate."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_blocks_coder_choice as bcc  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_blocks_auto as gab  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
THREE = gab.THREE
# (candidates, tolerance_ppm): each version alone, the three-pair list at 0 and 2 %, the sixteen-pair list
LISTS = [([CAND(WORD, 12)], 0), ([CAND(BYTE, 14)], 0), ([CAND(RANS64, 10)], 0), ([CAND(ALIAS, 13)], 0), (THREE, 0), (THREE, 20000),
         (bcc.LISTS[4], 20000)]
# (n_blocks, block_size, chunk_syms): one block of one chunk, ragged chunks, 4 and 8 chunks per block
GEOMETRIES = [(1, 32, 32), (4, 9000, 1000), (6, 16384, 4096), (3, 65536, 8192)]


def _torch():
    import torch
    return torch


def _counts(n_max):
    return sorted({1, max(n_max - 1, 1), n_max})


def _varlen(ctx, cands, tol, d_in, d_nb, nb_max, bs, ch, flags, d_out, cap):
    ctx.container_blocks_model_encode_varlen_async(cands, tol, d_in.data_ptr(), d_nb.data_ptr(), nb_max, bs, ch, flags, d_out.data_ptr(), cap)


def _fixed_auto(ctx, cands, tol, d_in, nb, bs, ch, flags):
    """the fixed auto call's container (whole buffer, on the host) and, for two or more candidates, its costs"""
    torch = _torch()
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_out = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_model_encode_auto_async(cands, tol, d_in.data_ptr(), nb, bs, ch, flags, d_out.data_ptr(), cap)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    return d_out.cpu().numpy()


@pytest.mark.parametrize("kind", bcc.KINDS)
def test_varlen_equals_the_fixed_auto_call(gpu_ctx, kind):
    torch = _torch()
    for gi, (nb, bs, ch) in enumerate(GEOMETRIES):
        data = bcc.block_data(kind, 4 * nb, bs, 20 * gi + bcc.KINDS.index(kind))
        d_in = gbc._dev(data)
        counts = bcc.block_counts(data, 4 * nb, bs)
        for cands, tol in LISTS:
            for flags in (0, CRC_BLOB):
                fixed = {}
                for nb_max in (nb, 4 * nb):
                    cap = gpu_ctx.container_blocks_capacity(nb_max, bs, ch)
                    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
                    for count in _counts(nb_max):
                        case = (kind, nb, bs, ch, cands, tol, flags, nb_max, count)
                        if count not in fixed:
                            fixed[count] = _fixed_auto(gpu_ctx, cands, tol, d_in, count, bs, ch, flags)
                        d_out.fill_(SENTINEL)
                        d_nb = torch.tensor([count], dtype=torch.int32, device="cuda")
                        _varlen(gpu_ctx, cands, tol, d_in, d_nb, nb_max, bs, ch, flags, d_out, cap)
                        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0, case
                        if len(cands) > 1:
                            want_i, want_costs = api.choose_blocks_coder(counts[:count], bs, ch, cands, tol)
                            assert np.array_equal(gpu_ctx.container_blocks_auto_costs(len(cands)), want_costs), case
                            assert struct.unpack_from("<BB", fixed[count], 6) == (cands[want_i] >> 8, cands[want_i] & 0xFF), case
                        got = d_out.cpu().numpy()
                        size = gab._container_size(fixed[count])
                        assert struct.unpack_from("<I", got, 56)[0] == count, case
                        assert np.array_equal(got[:size], fixed[count][:size]), case
                        assert (got[size:] == SENTINEL).all(), case


@pytest.mark.parametrize("coder,sb", [(WORD, 12), (BYTE, 14), (RANS64, 10), (ALIAS, 13)])
def test_varlen_equals_the_oracle_packed_container(gpu_ctx, oracle_lib, coder, sb):
    torch = _torch()
    nb_max, bs, ch = 7, 16384, 4096
    data = bcc.block_data("text", nb_max, bs, 11)
    d_in = gbc._dev(data)
    cap = gpu_ctx.container_blocks_capacity(nb_max, bs, ch)
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    for count in (2, 5, 7):
        for cands in ([CAND(coder, sb)], [CAND(coder, sb), CAND(BYTE, 8)]):
            for flags in (0, CRC_BLOB):
                d_out.fill_(SENTINEL)
                d_nb = torch.tensor([count], dtype=torch.int32, device="cuda")
                _varlen(gpu_ctx, cands, 0, d_in, d_nb, nb_max, bs, ch, flags, d_out, cap)
                assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
                got = d_out.cpu().numpy()
                chosen, _ = api.choose_blocks_coder(bcc.block_counts(data, count, bs), bs, ch, cands, 0)
                c_coder, c_sb = cands[chosen] >> 8, cands[chosen] & 0xFF
                want = gab._oracle_container(oracle_lib, c_coder, c_sb, data[:count * bs], count, bs, ch, flags)
                assert np.array_equal(got[:want.size], want), (coder, sb, count, len(cands), flags)
                assert (got[want.size:] == SENTINEL).all()


@pytest.mark.parametrize("kind,version", [("skewed", 3), ("zipf", 2)])
def test_one_graph_many_counts(kind, version):
    """the varlen encode and the any decode captured once, replayed with counts 1, mid, max, mid and new data each time:
    the container is the fixed call's, the decode the input, *d_n the symbol count, and nothing past either is written"""
    torch = _torch()
    nb_max, bs, ch = 12, 65536, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = ctx.container_blocks_capacity(nb_max, bs, ch)
    d_in = torch.empty(nb_max * bs, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nb_max * bs + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_nb = torch.tensor([nb_max], dtype=torch.int32, device="cuda")

    def round_trip():
        ctx.container_blocks_model_encode_varlen_async(THREE, 20000, d_in.data_ptr(), d_nb.data_ptr(), nb_max, bs, ch, CRC_BLOB,
                                                       d_buf.data_ptr(), cap)
        ctx.container_blocks_any_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb_max * bs, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(bcc.block_data("zipf", nb_max, bs, 1)))
        round_trip()                                                 # grows every group's workspace outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for step, count in enumerate((1, 5, nb_max, 7)):
            data = bcc.block_data(kind, count, bs, 60 + step)
            d_in[:data.size].copy_(torch.from_numpy(data))
            d_nb.fill_(count)
            d_buf.fill_(SENTINEL)
            d_out.fill_(SENTINEL)
            d_n.fill_(-1)
            launches = ctx.launches
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, count
            assert ctx.launches == launches                          # a replay does not go through the library
            fixed = _fixed_auto(ctx, THREE, 20000, d_in, count, bs, ch, CRC_BLOB)
            size = gab._container_size(fixed)
            assert struct.unpack_from("<H", fixed, 4)[0] == version, count
            got = d_buf.cpu().numpy()
            assert np.array_equal(got[:size], fixed[:size]) and (got[size:] == SENTINEL).all(), count
            assert int(d_n.item()) == count * bs, count
            out = d_out.cpu().numpy()
            assert np.array_equal(out[:data.size], data) and (out[data.size:] == SENTINEL).all(), count
        del g
    ctx.close()


def test_bad_counts_write_nothing(gpu_ctx):
    torch = _torch()
    nb_max, bs, ch = 5, 16384, 4096
    data = bcc.block_data("zipf", nb_max, bs, 4)
    d_in = gbc._dev(data)
    cap = gpu_ctx.container_blocks_capacity(nb_max, bs, ch)
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    for cands in (THREE, [CAND(ALIAS, 14)], [CAND(WORD, 12)]):
        for bad in (0, nb_max + 1):
            for flags in (0, CRC_BLOB):
                d_out.fill_(SENTINEL)
                d_nb = torch.tensor([bad], dtype=torch.int32, device="cuda")
                _varlen(gpu_ctx, cands, 0, d_in, d_nb, nb_max, bs, ch, flags, d_out, cap)
                assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -1, (cands, bad)
                assert bool((d_out == SENTINEL).all().item()), (cands, bad, flags)
                d_nb.fill_(3)                                        # a valid call behind it on the same context
                _varlen(gpu_ctx, cands, 0, d_in, d_nb, nb_max, bs, ch, flags, d_out, cap)
                assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
                fixed = _fixed_auto(gpu_ctx, cands, 0, d_in, 3, bs, ch, flags)
                size = gab._container_size(fixed)
                assert np.array_equal(d_out[:size].cpu().numpy(), fixed[:size]), (cands, bad, flags)


def test_argument_space_errors_and_launch_counts(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    nb_max, bs, ch = 8, 65536, 8192
    data = bcc.block_data("skewed", nb_max, bs, 2)
    d_in = gbc._dev(data)
    cap = gpu_ctx.container_blocks_capacity(nb_max, bs, ch)
    d_buf = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_nb = torch.tensor([nb_max, 3], dtype=torch.int32, device="cuda")
    i, o, p = d_in.data_ptr(), d_buf.data_ptr(), d_nb.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, nbp=p, nb=nb_max, block_size=bs, chunk=ch, flags=0, out=o, out_cap=cap):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_blocks_model_encode_varlen_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size,
                                                                    tol, inp, nbp, nb, block_size, chunk, flags, out, out_cap)
    before = gpu_ctx.launches
    for bad in ([], [CAND(BYTE, 16)], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
        assert call(bad) == -1, bad
    assert call(THREE, tol=10 ** 6 + 1) == -1
    for kw in ({"ctx": None}, {"inp": None}, {"out": None}, {"out": o + 8}, {"nbp": None}, {"nbp": p + 1}, {"nbp": p + 2}, {"nb": 0},
               {"chunk": 31}, {"chunk": 1000}, {"block_size": 33 * 32, "chunk": 32}, {"nb": 1 << 26, "block_size": 1024, "chunk": 32}):
        assert call(THREE, **kw) == -1, kw
    boff = (64 + 512 * nb_max + 8 * (nb_max * bs // ch + 1) + 15) & ~15
    assert call(THREE, out_cap=boff - 1) == -3                      # below the blob offset of n_blocks_max (not of *d_n_blocks)
    assert gpu_ctx.launches == before
    assert (d_buf.cpu().numpy() == SENTINEL).all()
    # the chosen blob does not fit: -3 from sync, the header unwritten; the count 3 at p + 4 is 4-byte aligned
    for nbp in (p, p + 4):
        d_buf.fill_(SENTINEL)
        assert call(THREE, nbp=nbp, out_cap=boff + 64) == 0
        assert lib.rb200_sync(gpu_ctx.h) == -3
        assert (d_buf[:64].cpu().numpy() == SENTINEL).all()
    # launches: plan, choice, K5f (word), K5c + scan + compaction (byte 14, alias 14), the CRCs, the header; with the
    # blob CRC also the blob length kernel.  One candidate: no choice kernel.
    for cands, flags, want in ((THREE, 0, 11), (THREE, CRC_BLOB, 13), ([CAND(WORD, 12)], 0, 4), ([CAND(BYTE, 14)], 0, 6),
                               ([CAND(ALIAS, 14)], CRC_BLOB, 8)):
        before = gpu_ctx.launches
        assert call(cands, flags=flags, nbp=p + 4) == 0
        assert gpu_ctx.launches - before == want, (cands, flags)
        assert lib.rb200_sync(gpu_ctx.h) == 0
        fixed = _fixed_auto(gpu_ctx, cands, 0, d_in, 3, bs, ch, flags)
        size = gab._container_size(fixed)
        assert np.array_equal(d_buf[:size].cpu().numpy(), fixed[:size]), (cands, flags)
