"""rb200_container_model_encode_varlen_async: rb200_container_model_encode_async with the length read from device memory
when the work runs.  Its bytes equal the oracle's container and the fixed call's for every coder and specialised
scale_bits, at n_max = n and at n_max several times n; nothing past the container is written; one captured graph encodes
every length 1 .. n_max (with *d_n = 0 and n_max + 1 refused in between, out untouched); the tile prefix of very large
directories, both word reciprocal forms, the argument and space errors, queued calls and n = 2^32 - 1 all hold."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_container as gc  # noqa: E402
import test_gpu_container_model_encode as me  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = gc.WORD, gc.BYTE, gc.ALIAS, gc.RANS64
CRC_BLOB, SENTINEL, ROWS = me.CRC_BLOB, me.SENTINEL, me.ROWS
KINDS = ["uniform", "zipf", "text", "two", "all256"]
# (n, chunk_syms): shorter than a step, the smallest chunk, a ragged last chunk, many chunks, the fused path
GEOMETRIES = [(17, 32), (5000, 32), (100003, 4096), (1 << 22, 1024), (3_000_001, 8192)]


def _torch():
    import torch
    return torch


def _boff(ctx, n, chunk):
    return (64 + 1024 + 8 * (ctx.chunk_count(n, chunk) + 1) + 15) // 16 * 16


def _varlen(ctx, coder, sb, d_in, n, n_max, chunk, flags, cap=None, fill=0xAA):
    """the varlen call with *d_n = n into a `fill`-filled buffer sized for n_max, then rb200_sync: (rc, d_out, cap)"""
    torch = _torch()
    cap = ctx.container_capacity(n_max, chunk) if cap is None else cap
    d_out = torch.full((cap + 16,), fill, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n], dtype=torch.int64, device="cuda")
    ctx.container_model_encode_varlen_async(coder, sb, d_in.data_ptr(), d_n.data_ptr(), n_max, chunk, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out, cap


def _check(ctx, oracle_lib, coder, sb, data, chunk, n_max, flags_list=(0, CRC_BLOB)):
    """the varlen container equals the oracle's and the fixed call's, both decodes round-trip it, and the bytes after it
    keep their fill"""
    torch = _torch()
    n = data.size
    wants, _ = me._oracle_container(oracle_lib, coder, sb, data, chunk, flags_list)
    d_in = gc._to_dev(data)
    for flags, want in zip(flags_list, wants):
        rc, d_out, cap = _varlen(ctx, coder, sb, d_in, n, n_max, chunk, flags, fill=SENTINEL)
        assert rc == 0, (coder, sb, n, n_max, chunk, flags, rc)
        got = d_out[:want.size].cpu().numpy()
        assert gc._container_size(got[:64], ctx.lib) == want.size
        assert np.array_equal(got, want), (coder, sb, n, n_max, chunk, flags)
        assert bool((d_out[want.size:] == SENTINEL).all().item()), (coder, sb, n, n_max, chunk, flags)
        rc, d_fixed = me._model_encode(ctx, coder, sb, d_in, n, chunk, flags)
        assert rc == 0 and torch.equal(d_fixed[:want.size], d_out[:want.size])
        d_dec = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        ctx.container_decode_async(d_out.data_ptr(), want.size, d_dec.data_ptr(), n)
        ctx.sync()
        assert torch.equal(d_dec[:n], d_in[:n]) and bool((d_dec[n:] == SENTINEL).all().item())
        assert np.array_equal(ctx.container_decode_host(got), data)


@pytest.mark.parametrize("coder,sb", ROWS)
def test_varlen_equals_oracle_and_fixed_call(gpu_ctx, oracle_lib, coder, sb):
    for kind in KINDS:
        for n, chunk in GEOMETRIES:
            data = me._data(kind, n)
            if coder == BYTE and sb == 16 and np.unique(data).size == 1:
                continue                                           # a frequency of 65536: a refused model
            for n_max in (n, 5 * n + 3):
                _check(gpu_ctx, oracle_lib, coder, sb, data, chunk, n_max)


# one graph per path: word fused, word split, alias fused, byte split, rans64
GRAPH_PATHS = [(WORD, 12, 8192), (WORD, 12, 2048), (ALIAS, 16, 4096), (BYTE, 14, 1024), (RANS64, 14, 4096)]


@pytest.mark.parametrize("coder,sb,chunk", GRAPH_PATHS)
def test_one_graph_many_lengths(cuda_box, oracle_lib, coder, sb, chunk):
    """ONE captured varlen encode + async decode, replayed over lengths 1 .. n_max and changing distributions; replays
    with *d_n = 0 and n_max + 1 in between are -2 and -1 and write nothing, and the next replay is exact again"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n_max = 2_500_003
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = ctx.container_capacity(n_max, chunk)
    d_in = torch.zeros(n_max + 16, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_dec = torch.zeros(n_max + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n_max], dtype=torch.int64, device="cuda")
    d_nsym = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_model_encode_varlen_async(coder, sb, d_in.data_ptr(), d_n.data_ptr(), n_max, chunk, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_decode_async(d_buf.data_ptr(), cap, d_dec.data_ptr(), n_max, d_nsym.data_ptr())

    kinds = ["zipf", "uniform", "text", "skew", "two"]
    lengths = [1, 31, 32, 33, chunk - 1, chunk, chunk + 1, 1_234_567, n_max]
    with torch.cuda.stream(stream):
        d_in[:n_max].copy_(torch.from_numpy(me._data("skew", n_max)))
        round_trip()                                                 # grows the workspaces for n_max outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        launches = ctx.launches
        for i, n in enumerate(lengths):
            if i in (2, 6):                                          # refused lengths between valid ones
                for bad, code in ((0, -2), (n_max + 1, -1)):
                    d_buf.fill_(SENTINEL)
                    d_n.fill_(bad)
                    g.replay()
                    assert ctx.lib.dll.rb200_sync(ctx.h) == code, (n, bad)
                    assert bool((d_buf == SENTINEL).all().item()), (n, bad)
            data = me._data(kinds[i % len(kinds)], n, 50)
            if coder == BYTE and sb == 16 and np.unique(data).size == 1:
                continue
            (want,), _ = me._oracle_container(oracle_lib, coder, sb, data, chunk, (CRC_BLOB,))
            d_in[:n].copy_(torch.from_numpy(data))
            d_buf.fill_(SENTINEL)
            d_dec.zero_()
            d_n.fill_(n)
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, n
            assert np.array_equal(d_buf[:want.size].cpu().numpy(), want), n
            assert bool((d_buf[want.size:] == SENTINEL).all().item()), n
            assert int(d_nsym.item()) == n and np.array_equal(d_dec[:n].cpu().numpy(), data), n
        assert ctx.launches == launches                              # replays do not go through the library
    del g
    ctx.close()


def test_tile_prefix_threshold(gpu_ctx):
    """rans64 at chunks of 32 with n_max past 256 scan tiles of 4096 chunks: the host launches the tile prefix; real
    lengths below and above the threshold give the fixed call's bytes and round-trip"""
    torch = _torch()
    chunk = 32
    n_max = (1 << 25) + 1                                            # 2^20 + 1 chunks: 257 tiles
    data = me._data("zipf", n_max)
    d_in = gc._to_dev(data)
    for n in (1 << 24, (1 << 25) - 5, n_max):                        # 128, 256 and 257 tiles
        for flags in (0, CRC_BLOB):
            rc, d_out, cap = _varlen(gpu_ctx, RANS64, 14, d_in, n, n_max, chunk, flags, fill=SENTINEL)
            assert rc == 0, (n, flags)
            rc, d_fixed = me._model_encode(gpu_ctx, RANS64, 14, d_in, n, chunk, flags)
            assert rc == 0
            size = gc._container_size(d_fixed[:64].cpu().numpy(), gpu_ctx.lib)
            assert torch.equal(d_out[:size], d_fixed[:size]), (n, flags)
            assert bool((d_out[size:] == SENTINEL).all().item())
            d_dec = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
            gpu_ctx.container_decode_async(d_out.data_ptr(), size, d_dec.data_ptr(), n)
            gpu_ctx.sync()
            assert torch.equal(d_dec[:n], d_in[:n])


def test_word_reciprocal_gate(gpu_ctx, oracle_lib):
    """frequencies 2963 (the 32-bit reciprocal is exact) and 2964 (it is not), on the split and fused paths"""
    for freq in (2963, 2964):
        data, freqs = me._gate_data(freq, 700)
        assert np.array_equal(oracle_lib.model(data, 12)[0], freqs)
        for chunk in (2048, 8192):
            _check(gpu_ctx, oracle_lib, WORD, 12, data, chunk, 3 * data.size + 1)


def test_space_and_argument_errors(gpu_ctx, oracle_lib):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    data = me._data("zipf", 300000)
    n, chunk = data.size, 4096
    n_max = 4 * n
    d_in = gc._to_dev(data)
    cap = gpu_ctx.container_capacity(n_max, chunk)
    boff = _boff(gpu_ctx, n_max, chunk)
    # blob larger than out_cap: -3 from rb200_sync, header unwritten
    rc, d_out, _ = _varlen(gpu_ctx, ALIAS, 14, d_in, n, n_max, chunk, 0, cap=boff + 1000, fill=SENTINEL)
    assert rc == -3 and bool((d_out[:64] == SENTINEL).all().item())
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n, 0], dtype=torch.int64, device="cuda")
    i, o, p = d_in.data_ptr(), d_out.data_ptr(), d_n.data_ptr()
    h = gpu_ctx.h
    before = gpu_ctx.launches
    # out_cap below the blob offset of n_max (but enough for n): -3 from the call
    assert lib.rb200_container_model_encode_varlen_async(h, WORD, 12, i, p, n_max, chunk, 0, o, boff - 16) == -3
    calls = [(None, WORD, 12, i, p, n_max, chunk, o), (h, WORD, 12, None, p, n_max, chunk, o), (h, WORD, 12, i, None, n_max, chunk, o),
             (h, WORD, 12, i, p + 4, n_max, chunk, o), (h, WORD, 12, i, p, n_max, chunk, None), (h, WORD, 12, i, p, n_max, chunk, o + 8),
             (h, 4, 12, i, p, n_max, chunk, o), (h, -1, 12, i, p, n_max, chunk, o), (h, WORD, 14, i, p, n_max, chunk, o),
             (h, ALIAS, 7, i, p, n_max, chunk, o), (h, BYTE, 17, i, p, n_max, chunk, o), (h, RANS64, 14, i, p, n_max, 16, o),
             (h, RANS64, 14, i, p, n_max, (1 << 24) + 1, o), (h, WORD, 12, i, p, 0, chunk, o), (h, WORD, 12, i, p, 1 << 32, chunk, o),
             (h, WORD, 12, i, p, 1 << 40, 32, o)]
    for ctx, coder, sb, ip, np_, nm, ch, op in calls:
        assert lib.rb200_container_model_encode_varlen_async(ctx, coder, sb, ip, np_, nm, ch, 0, op, cap) == -1, (coder, sb, np_, nm, ch)
    assert gpu_ctx.launches == before
    assert bool((d_out == SENTINEL).all().item())
    assert lib.rb200_sync(h) == 0
    _check(gpu_ctx, oracle_lib, ALIAS, 14, data, chunk, n_max)        # the context is fine afterwards


def test_calls_queue(gpu_ctx, oracle_lib):
    """two varlen calls with different lengths and one fixed call back to back, then one rb200_sync"""
    torch = _torch()
    zipf, text = me._data("zipf", 1_000_003), me._data("text", 2_000_000)
    d_zipf, d_text = gc._to_dev(zipf), gc._to_dev(text)
    cases = [(ALIAS, 16, zipf, d_zipf, 777_777, 4096, CRC_BLOB, True), (WORD, 12, text, d_text, 2_000_000, 8192, 0, True),
             (RANS64, 14, zipf, d_zipf, 1_000_003, 2048, CRC_BLOB, False)]
    d_ns = torch.tensor([c[4] for c in cases], dtype=torch.int64, device="cuda")
    outs = []
    for k, (coder, sb, data, d_in, n, chunk, flags, varlen) in enumerate(cases):
        n_max = 3 * data.size if varlen else n
        cap = gpu_ctx.container_capacity(n_max, chunk)
        d_out = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
        outs.append(d_out)
        if varlen:
            gpu_ctx.container_model_encode_varlen_async(coder, sb, d_in.data_ptr(), d_ns[k:].data_ptr(), n_max, chunk, flags,
                                                        d_out.data_ptr(), cap)
        else:
            gpu_ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), n, chunk, flags, d_out.data_ptr(), cap)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    for (coder, sb, data, _, n, chunk, flags, _), d_out in zip(cases, outs):
        (want,), _ = me._oracle_container(oracle_lib, coder, sb, data[:n], chunk, (flags,))
        assert np.array_equal(d_out[:want.size].cpu().numpy(), want), coder


def test_largest_length(gpu_ctx, oracle_lib):
    """n_max = 2^32 - 1 (word, chunks of 8192), replayed with *d_n = 2^32 - 1 and with a small length"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n_max, chunk = (1 << 32) - 1, 8192
    reps, rem = divmod(n_max, 251)
    d_in = torch.arange(251, dtype=torch.uint8, device="cuda").repeat(reps + 1)[:n_max]
    cap = gpu_ctx.container_capacity(n_max, chunk)
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.tensor([n_max], dtype=torch.int64, device="cuda")
    gpu_ctx.container_model_encode_varlen_async(WORD, 12, d_in.data_ptr(), d_n.data_ptr(), n_max, chunk, 0, d_out.data_ptr(), cap)
    gpu_ctx.sync()
    stats = rb.SymbolStats()
    stats.freqs[:251] = reps
    stats.freqs[:rem] += 1
    stats.normalize_freqs(4096)
    head = d_out[:64 + 1024].cpu().numpy()
    assert np.array_equal(head[64:].view(np.uint32), stats.freqs)
    size = gc._container_size(head[:64], gpu_ctx.lib)
    d_dec = torch.empty(n_max + 16, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_decode_async(d_out.data_ptr(), size, d_dec.data_ptr(), n_max)
    gpu_ctx.sync()
    assert torch.equal(d_dec[:n_max], d_in)
    del d_dec
    small = 100_003
    d_out[:size].fill_(SENTINEL)
    d_n.fill_(small)
    gpu_ctx.container_model_encode_varlen_async(WORD, 12, d_in.data_ptr(), d_n.data_ptr(), n_max, chunk, 0, d_out.data_ptr(), cap)
    gpu_ctx.sync()
    (want,), _ = me._oracle_container(oracle_lib, WORD, 12, d_in[:small].cpu().numpy(), chunk, (0,))
    assert np.array_equal(d_out[:want.size].cpu().numpy(), want)
    assert bool((d_out[want.size:size] == SENTINEL).all().item())
