"""rb200_container_model_encode_async: the single-model (version 1) container with its model built from the data on the
GPU, enqueue-only.  Its bytes equal the oracle's container and rb200_model_from_data + rb200_container_encode's for
every coder and specialised scale_bits, every data shape (one symbol, two, 256 with 255 rare) and both reciprocal forms
of the word encoder; a model rb200_model_create refuses is -2 from rb200_sync with no header written; argument errors
launch nothing; calls queue; n = 2^32 - 1 works; one captured call encodes data of a different distribution at every
replay."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_container as gc  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = gc.WORD, gc.BYTE, gc.ALIAS, gc.RANS64
CRC_BLOB = 1
SENTINEL = 0x5C

# every (coder, scale_bits) row of the async decode's variants
ROWS = [(WORD, 12), (ALIAS, 16), (ALIAS, 14), (ALIAS, 12), (ALIAS, 10), (BYTE, 16), (BYTE, 14), (BYTE, 12), (BYTE, 8),
        (RANS64, 8), (RANS64, 14), (RANS64, 16)]
# "all256": one dominant symbol and 255 rare ones; at scale_bits 8 the 255 are squashed to width 0 and each steals a
# slot from the dominant one, the only width above 1
KINDS = ["uniform", "zipf", "text", "two", "skew", "const", "all256"]
# (n, chunk_syms): shorter than a step, the smallest chunk, a ragged last chunk, a large chunk, many chunks, and a
# size that takes the fused path
GEOMETRIES = [(17, 32), (5000, 32), (100003, 4096), (200000, 65536), (1 << 24, 1024), (3_000_001, 8192)]


def _torch():
    import torch
    return torch


@functools.lru_cache(maxsize=None)
def _data(kind, n, seed=1):
    from conftest import _gen
    if kind != "all256":
        return _gen(kind, n, seed=n + seed)
    rng = np.random.default_rng(n + seed)
    data = np.full(n, 0x41, np.uint8)
    rare = np.delete(np.arange(256, dtype=np.uint8), 0x41)[:max(n - 1, 0)]
    data[rng.choice(n, rare.size, replace=False)] = rare
    return data


def _oracle_container(oracle_lib, coder, sb, data, chunk, flags):
    """(container, freqs): the oracle's model and encode, packed by rb200_container_pack"""
    from ryg_rans_b200 import api
    freqs, cum = oracle_lib.model(data, sb)
    ob, oo = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
    return [api.container_pack(coder, sb, chunk, data.size, freqs, oo, ob, f) for f in flags], freqs


def _model_encode(ctx, coder, sb, d_in, n, chunk, flags, cap=None, fill=0xAA):
    """the new call into a `fill`-filled buffer, then rb200_sync: (rc, d_out)"""
    torch = _torch()
    cap = ctx.container_capacity(n, chunk) if cap is None else cap
    d_out = torch.full((cap + 16,), fill, dtype=torch.uint8, device="cuda")
    ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), n, chunk, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out


def _check(ctx, oracle_lib, coder, sb, data, chunk, flags_list=(0, CRC_BLOB)):
    """the new call's container equals the oracle's and the existing device path's, and both decodes round-trip it"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n = data.size
    wants, freqs = _oracle_container(oracle_lib, coder, sb, data, chunk, flags_list)
    d_in = gc._to_dev(data)
    model = rb.Model.from_data(ctx, coder, sb, device_ptr=d_in.data_ptr(), n=n)
    assert np.array_equal(model.freqs, freqs)
    cap = ctx.container_capacity(n, chunk)
    for flags, want in zip(flags_list, wants):
        rc, d_out = _model_encode(ctx, coder, sb, d_in, n, chunk, flags)
        assert rc == 0, (coder, sb, n, chunk, flags, rc)
        got = d_out[:want.size].cpu().numpy()
        assert gc._container_size(got[:64], ctx.lib) == want.size
        assert np.array_equal(got, want), (coder, sb, n, chunk, flags)
        d_ref = torch.full((cap + 16,), 0x33, dtype=torch.uint8, device="cuda")
        ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, flags, d_ref.data_ptr(), cap)
        ctx.sync()
        assert torch.equal(d_ref[:want.size], d_out[:want.size])
        d_dec = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        ctx.container_decode_async(d_out.data_ptr(), want.size, d_dec.data_ptr(), n)
        ctx.sync()
        assert torch.equal(d_dec[:n], d_in[:n]) and bool((d_dec[n:] == SENTINEL).all().item())
        assert np.array_equal(ctx.container_decode_host(got), data)
    model.close()


@pytest.mark.parametrize("coder,sb", ROWS)
def test_model_encode_equals_oracle_and_existing_path(gpu_ctx, oracle_lib, coder, sb):
    for kind in KINDS:
        for n, chunk in GEOMETRIES:
            data = _data(kind, n)
            if coder == BYTE and sb == 16 and np.unique(data).size == 1:
                continue                                           # a frequency of 65536: test_refused_model
            _check(gpu_ctx, oracle_lib, coder, sb, data, chunk)


def _gate_data(freq, n_unit):
    """data whose normalised word model gives symbol 9 frequency `freq` exactly (counts are multiples of the model)"""
    freqs = np.zeros(256, np.int64)
    freqs[9] = freq
    rest = 4096 - freq
    others = np.arange(20, 120)
    freqs[others] = rest // others.size
    freqs[others[:rest % others.size]] += 1
    data = np.repeat(np.arange(256, dtype=np.uint8), freqs * n_unit)
    np.random.default_rng(freq).shuffle(data)
    return data, freqs


def run_word_gate(oracle_lib):
    """2963 (the 32-bit reciprocal is exact) and 2964 (it is not): both word encoder instances, both paths"""
    import ryg_rans_b200 as rb
    ctx = rb.Context(0)
    for freq in (2963, 2964):
        data, freqs = _gate_data(freq, 700)
        assert np.array_equal(oracle_lib.model(data, 12)[0], freqs)
        for chunk in (2048, 8192):                                 # split and fused
            _check(ctx, oracle_lib, WORD, 12, data, chunk)
    ctx.close()


def test_word_reciprocal_gate(gpu_ctx, oracle_lib):
    run_word_gate(oracle_lib)


def test_word_reciprocal_gate_forced_33bit(cuda_box):
    """RB200_WORD_RECIPROCAL=33 reaches the model kernel: every model takes the 33-bit instance, and the bytes stay"""
    here = os.path.dirname(os.path.abspath(__file__))
    code = r'''
import sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import oracle, test_gpu_container_model_encode as t
t.run_word_gate(oracle.Oracle())
print("gate ok")
''' % (os.path.dirname(here), here)
    env = dict(os.environ, RB200_WORD_RECIPROCAL="33")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "gate ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_refused_model(gpu_ctx, oracle_lib):
    """byte coder at scale_bits 16 on one symbol: a frequency of 65536, which RansDecSymbol cannot hold"""
    data = _data("const", 100003)
    d_in = gc._to_dev(data)
    lib = gpu_ctx.lib.dll
    before = gpu_ctx.launches
    rc, d_out = _model_encode(gpu_ctx, BYTE, 16, d_in, data.size, 4096, CRC_BLOB, fill=SENTINEL)
    assert gpu_ctx.launches > before                               # the call itself returned 0 and launched
    assert rc == -2
    assert bool((d_out[:64] == SENTINEL).all().item())
    assert lib.rb200_sync(gpu_ctx.h) == 0
    _check(gpu_ctx, oracle_lib, BYTE, 14, data, 4096)               # the context is fine afterwards


def test_space_and_argument_errors(gpu_ctx, oracle_lib):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    data = _data("zipf", 300000)
    n, chunk = data.size, 4096
    d_in = gc._to_dev(data)
    cap = gpu_ctx.container_capacity(n, chunk)
    boff = (64 + 1024 + 8 * (gpu_ctx.chunk_count(n, chunk) + 1) + 15) // 16 * 16
    # blob larger than out_cap: -3 from rb200_sync, header unwritten
    rc, d_out = _model_encode(gpu_ctx, ALIAS, 14, d_in, n, chunk, 0, cap=boff + 1000, fill=SENTINEL)
    assert rc == -3 and bool((d_out[:64] == SENTINEL).all().item())
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    i, o = d_in.data_ptr(), d_out.data_ptr()
    before = gpu_ctx.launches
    assert lib.rb200_container_model_encode_async(gpu_ctx.h, WORD, 12, i, n, chunk, 0, o, boff - 16) == -3
    assert lib.rb200_container_model_encode_async(gpu_ctx.h, WORD, 12, i, 0, chunk, 0, o, cap) == -2
    calls = [(None, WORD, 12, i, n, chunk, o), (gpu_ctx.h, WORD, 12, None, n, chunk, o), (gpu_ctx.h, WORD, 12, i, n, chunk, None),
             (gpu_ctx.h, WORD, 12, i, n, chunk, o + 8), (gpu_ctx.h, 4, 12, i, n, chunk, o), (gpu_ctx.h, -1, 12, i, n, chunk, o),
             (gpu_ctx.h, WORD, 14, i, n, chunk, o), (gpu_ctx.h, ALIAS, 7, i, n, chunk, o), (gpu_ctx.h, BYTE, 17, i, n, chunk, o),
             (gpu_ctx.h, RANS64, 14, i, n, 16, o), (gpu_ctx.h, RANS64, 14, i, n, (1 << 24) + 1, o),
             (gpu_ctx.h, WORD, 12, i, 1 << 32, chunk, o), (gpu_ctx.h, WORD, 12, i, 1 << 40, 32, o)]
    for ctx, coder, sb, ip, nn, ch, op in calls:
        assert lib.rb200_container_model_encode_async(ctx, coder, sb, ip, nn, ch, 0, op, cap) == -1, (coder, sb, nn, ch)
    assert gpu_ctx.launches == before
    assert bool((d_out == SENTINEL).all().item())
    assert lib.rb200_sync(gpu_ctx.h) == 0


def test_calls_queue(gpu_ctx, oracle_lib):
    """three coders back to back with an rb200_decode between two of them, then one rb200_sync"""
    torch = _torch()
    cases = [(ALIAS, 16, _data("zipf", 1_000_003), 4096, CRC_BLOB), (WORD, 12, _data("text", 2_000_000), 8192, 0),
             (RANS64, 14, _data("uniform", 400_000), 2048, CRC_BLOB)]
    plain = _data("zipf", 1_500_000, 12)
    freqs, cum = oracle_lib.model(plain, 12)
    pb, po = oracle_lib.chunked_encode(WORD, plain, freqs, cum, 4096)
    model = gpu_ctx.model(WORD, 12, freqs)
    d_pb, d_po = gc._to_dev(pb), gc._to_dev(po.view(np.uint8))
    d_pout = torch.zeros(plain.size + 16, dtype=torch.uint8, device="cuda")
    keep, outs = [], []
    for i, (coder, sb, data, chunk, flags) in enumerate(cases):
        d_in = gc._to_dev(data)
        cap = gpu_ctx.container_capacity(data.size, chunk)
        d_out = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
        keep.append(d_in)
        outs.append(d_out)
        gpu_ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), data.size, chunk, flags, d_out.data_ptr(), cap)
        if i == 0:
            gpu_ctx.decode_device(model, d_pb.data_ptr(), pb.size, d_po.data_ptr(), 4096, d_pout.data_ptr(), plain.size)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    for (coder, sb, data, chunk, flags), d_out in zip(cases, outs):
        (want,), _ = _oracle_container(oracle_lib, coder, sb, data, chunk, (flags,))
        assert np.array_equal(d_out[:want.size].cpu().numpy(), want), coder
    assert np.array_equal(d_pout[:plain.size].cpu().numpy(), plain)
    model.close()


def test_n_below_2_pow_32(gpu_ctx):
    """n = 2^32 - 1 symbols of period 251 (a ramp tiled on the device), word coder: the model section is normalize_freqs
    of the known counts, and the async decode round-trips the data"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n, chunk = (1 << 32) - 1, 8192
    reps, rem = divmod(n, 251)
    d_in = torch.arange(251, dtype=torch.uint8, device="cuda").repeat(reps + 1)[:n]
    cap = gpu_ctx.container_capacity(n, chunk)
    d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_model_encode_async(WORD, 12, d_in.data_ptr(), n, chunk, 0, d_out.data_ptr(), cap)
    gpu_ctx.sync()
    stats = rb.SymbolStats()
    stats.freqs[:251] = reps
    stats.freqs[:rem] += 1
    stats.normalize_freqs(4096)
    head = d_out[:64 + 1024].cpu().numpy()
    assert np.array_equal(head[64:].view(np.uint32), stats.freqs)
    size = gc._container_size(head[:64], gpu_ctx.lib)
    d_dec = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_decode_async(d_out.data_ptr(), size, d_dec.data_ptr(), n)
    gpu_ctx.sync()
    assert torch.equal(d_dec[:n], d_in)


def test_a_different_model_at_every_graph_replay(cuda_box, oracle_lib):
    """ONE captured model encode + async decode, replayed over data of different distributions: the model, the
    container and the round trip follow the data at every replay"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n, chunk = 2_000_003, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = ctx.container_capacity(n, chunk)
    d_in = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    for coder, sb, kinds in ((WORD, 12, ("uniform", "zipf", "text", "const")), (ALIAS, 16, ("zipf", "text"))):
        def round_trip():
            ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), n, chunk, CRC_BLOB, d_buf.data_ptr(), cap)
            ctx.container_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

        with torch.cuda.stream(stream):
            d_in.copy_(torch.from_numpy(_data("skew", n)))
            round_trip()                                             # grows the encoder's workspaces outside the capture
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                round_trip()
            launches = ctx.launches
            for kind in kinds:
                data = _data(kind, n, 40)
                (want,), freqs = _oracle_container(oracle_lib, coder, sb, data, chunk, (CRC_BLOB,))
                d_in.copy_(torch.from_numpy(data))
                d_out.zero_()
                g.replay()
                assert ctx.lib.dll.rb200_sync(ctx.h) == 0, kind
                got = d_buf[:want.size].cpu().numpy()
                assert np.array_equal(got[64:64 + 1024].view(np.uint32), freqs), kind
                assert np.array_equal(got, want), kind
                assert int(d_n.item()) == n and np.array_equal(d_out[:n].cpu().numpy(), data), kind
            assert ctx.launches == launches                          # replays do not go through the library
        del g
    ctx.close()
