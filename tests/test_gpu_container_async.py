"""rb200_container_decode_async: the single-model (version 1) container of any coder checked, its decode table built and
its decoder picked on the GPU, with nothing done on the host.  Oracle containers decode through every decoder variant
(word narrow / WIDE, alias and byte at each specialised scale_bits and the generic one, rans64) to the data and to
rb200_container_decode's output; everything rb200_container_open rejects, and what it accepts but the decoders refuse,
is -4 from rb200_sync with the output untouched; out_cap < n is -3; calls queue without synchronising; one call
captured in a CUDA graph decodes containers of different coders on replay."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks as cb  # noqa: E402
import test_gpu_container as gc  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = gc.WORD, gc.BYTE, gc.ALIAS, gc.RANS64
CRC_BLOB = 1
SENTINEL = 0x5C
MAGIC = 0x43324252

# (coder, scale_bits, data kind): one row per decoder variant; "const" has one symbol of frequency 4096 (WIDE)
VARIANTS = [(WORD, 12, "uniform"), (WORD, 12, "const"),
            (ALIAS, 16, "zipf"), (ALIAS, 14, "zipf"), (ALIAS, 12, "zipf"), (ALIAS, 10, "zipf"),
            (BYTE, 16, "zipf"), (BYTE, 14, "zipf"), (BYTE, 12, "zipf"), (BYTE, 8, "zipf"),
            (RANS64, 8, "zipf"), (RANS64, 14, "zipf"), (RANS64, 16, "zipf")]
# (n, chunk_syms): empty, shorter than a step, a ragged last chunk, the smallest and a large chunk, and more chunks than
# any decoder's grid has warps, so that every persistent warp takes several
GEOMETRIES = [(0, 4096), (17, 32), (100003, 4096), (5000, 32), (200000, 65536), (1 << 24, 1024)]


def _torch():
    import torch
    return torch


def _async(ctx, d_buf, size, n, out_cap=None):
    """the async decode of d_buf[0, size) into a sentinel-filled buffer, then one rb200_sync: (rc, *d_n_symbols or -1, out)"""
    torch = _torch()
    cap = n if out_cap is None else out_cap
    d_out = torch.full((max(n, cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    ctx.container_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())
    rc = ctx.lib.dll.rb200_sync(ctx.h)
    return rc, int(d_n.item()), d_out


def _untouched(d_out):
    return bool((d_out == SENTINEL).all().item())


def _container(oracle_lib, gen, coder, sb, kind, n, chunk, flags, seed=1):
    """(container, data): the oracle's encode of `kind` data packed by rb200_container_pack"""
    from ryg_rans_b200 import api
    data = gen(kind, n, seed=n + seed)
    freqs, cum = oracle_lib.model(data if n else gen(kind, 1000, 3), sb)
    ob, oo = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
    return api.container_pack(coder, sb, chunk, n, freqs, oo, ob, flags), data


@pytest.mark.parametrize("coder,sb,kind", VARIANTS)
def test_async_decode_of_oracle_containers(gpu_ctx, oracle_lib, gen, coder, sb, kind):
    for n, chunk in GEOMETRIES:
        for flags in (0, CRC_BLOB):
            buf, data = _container(oracle_lib, gen, coder, sb, kind, n, chunk, flags)
            rc, got_n, d_out = _async(gpu_ctx, gc._to_dev(buf), buf.size, n)
            assert rc == 0 and got_n == n, (n, chunk, flags, rc, got_n)
            out = d_out[:n].cpu().numpy()
            assert np.array_equal(out, data), (n, chunk, flags)
            assert _untouched(d_out[n:])
            rc, n2, sync_out, _ = gc._decode(gpu_ctx, buf, gc.DEVICE, out_cap=max(n, 1))
            assert rc == 0 and n2 == n and np.array_equal(sync_out[:n], out)


def test_async_round_trip_with_one_sync(gpu_ctx, oracle_lib, gen):
    torch = _torch()
    for coder, sb, kind, n, chunk in ((WORD, 12, "text", 3_000_001, 8192), (ALIAS, 16, "zipf", 1_000_000, 4096),
                                      (BYTE, 14, "zipf", 777_777, 2048), (RANS64, 14, "uniform", 500_000, 16384)):
        data = gen(kind, n, 70 + coder)
        freqs, _ = oracle_lib.model(data, sb)
        model = gpu_ctx.model(coder, sb, freqs)
        cap = gpu_ctx.container_capacity(n, chunk)
        d_in = gc._to_dev(data)
        for flags in (0, CRC_BLOB):
            d_cont = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
            d_out = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
            d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
            gpu_ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, flags, d_cont.data_ptr(), cap)
            gpu_ctx.container_decode_async(d_cont.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())
            gpu_ctx.sync()
            assert int(d_n.item()) == n
            assert torch.equal(d_out[:n], d_in[:n]), (coder, sb, flags)
            assert _untouched(d_out[n:])
        model.close()


@pytest.fixture(scope="module")
def word_case(oracle_lib, gen):
    """test_container_decode_rejects_what_open_rejects's container: text, word coder, chunks of 4096"""
    import oracle as orc
    from ryg_rans_b200 import api
    data = gen("text", 20000, 6)
    freqs, cum = oracle_lib.model(data, 12)
    blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 4096)
    good = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob, CRC_BLOB)
    plain = api.container_pack(WORD, 12, 4096, data.size, freqs, offs, blob, 0)
    return data, blob, offs, good, plain


def _rejected(data, blob, offs, good, plain):
    """every corruption of test_container_decode_rejects_what_open_rejects"""
    for base in (good, plain):
        for pos in (5, 70, 64 + 1024 + 9):                       # header, model, directory
            bad = base.copy()
            bad[pos] ^= 0x40
            yield f"flip at {pos}", bad
    bad = good.copy()
    bad[-7] ^= 0x40                                              # the blob, under its CRC
    yield "blob under its CRC", bad
    for cut in list(range(0, 64 + 1024 + 8 * offs.size + 16, 7)) + [good.size - 16, good.size - 1]:
        yield f"cut at {cut}", good[:cut].copy()
    edits = {
        "magic": (0, "<I", 0x12345678), "version": (4, "<H", 2), "coder": (6, "<B", 9), "scale_bits": (7, "<B", 3),
        "lanes": (8, "<I", 64), "chunk_syms zero": (12, "<I", 0), "chunk_syms other": (12, "<I", 2048),
        "n_symbols huge": (16, "<Q", 2 ** 64 - 1), "n_symbols + 1 chunk": (16, "<Q", data.size + 4096),
        "n_chunks huge": (24, "<Q", 2 ** 40), "n_chunks 2^31": (24, "<Q", 2 ** 31), "blob_bytes odd": (32, "<Q", blob.size + 8),
        "blob_bytes beyond the buffer": (32, "<Q", blob.size + 4096), "blob_bytes short": (32, "<Q", blob.size - 16),
        "freqs do not sum to 1 << scale_bits": (64 + 4 * 65, "<I", 7), "word coder with scale_bits 14": (7, "<B", 14),
        "first stream starts beyond the first vector": (64 + 1024, "<Q", 32),
        "directory not monotone": (64 + 1024 + 8, "<Q", int(offs[2]) + 16),
        "last entry != blob size": (64 + 1024 + 8 * (offs.size - 1), "<Q", int(offs[-1]) - 16),
    }
    for name, (off, fmt, val) in edits.items():
        bad = plain.copy()
        struct.pack_into(fmt, bad, off, val)
        yield name, gc._reseal(bad)


def _junk():
    """200 seeded buffers of random bytes with a valid magic and version 1, resealed"""
    rng = np.random.default_rng(1)
    for i in range(200):
        junk = rng.integers(0, 256, int(rng.integers(64, 4096)), dtype=np.uint8)
        struct.pack_into("<IH", junk, 0, MAGIC, 1)
        yield f"junk {i}", gc._reseal(junk)


def test_async_rejects_what_open_rejects(gpu_ctx, word_case):
    from ryg_rans_b200 import api
    data, blob, offs, good, plain = word_case
    for name, bad in list(_rejected(*word_case)) + list(_junk()):
        with pytest.raises(Exception):
            api.container_open(bad)                               # the host parser agrees
        rc, _, d_out = _async(gpu_ctx, gc._to_dev(bad), bad.size, data.size)
        assert rc == -4, (name, rc)
        assert _untouched(d_out), f"output written for a rejected container ({name})"
    rc, n, d_out = _async(gpu_ctx, gc._to_dev(good), good.size, data.size)
    assert rc == 0 and n == data.size and np.array_equal(d_out[:n].cpu().numpy(), data)


def _refused():
    """containers rb200_container_open accepts and rb200_container_decode refuses (chunk_syms 16: -1; chunk_syms
    2^24 + 32: -1; a byte model at 16 bits with one frequency of 65536: -2), packed with valid CRCs:
    (name, container, n, the synchronous call's code)"""
    from ryg_rans_b200 import api
    uniform = np.full(256, 16, np.uint32)                       # the word coder's 4096
    for name, coder, sb, freqs, n, chunk in (("chunk_syms 16", WORD, 12, uniform, 64, 16),
                                             ("chunk_syms 2^24 + 32", WORD, 12, uniform, (1 << 24) + 32, (1 << 24) + 32)):
        n_chunks = -(-n // chunk)
        offs = np.arange(n_chunks + 1, dtype=np.uint64) * 16
        yield name, api.container_pack(coder, sb, chunk, n, freqs, offs, np.zeros(16 * n_chunks, np.uint8), 0), n, -1
    one = np.zeros(256, np.uint32)
    one[0x41] = 65536
    offs = np.array([0, 144, 288], np.uint64)                    # two chunks of a 32-lane header and one vector
    yield "byte frequency 65536", api.container_pack(BYTE, 16, 32, 64, one, offs, np.zeros(288, np.uint8), CRC_BLOB), 64, -2


def test_async_rejects_what_the_decoders_refuse(gpu_ctx):
    from ryg_rans_b200 import api
    for name, buf, n, sync_rc in _refused():
        meta = api.container_open(buf)[0]                         # the container is valid
        assert meta["n_symbols"] == n, name
        rc, _, _, untouched = gc._decode(gpu_ctx, buf, gc.DEVICE, out_cap=n)
        assert rc == sync_rc and untouched, (name, rc)
        rc, got_n, d_out = _async(gpu_ctx, gc._to_dev(buf), buf.size, n)
        assert rc == -4 and _untouched(d_out), (name, rc)
        assert got_n == n, name                                   # header, model and directory passed


def test_async_rejects_version_2(gpu_ctx, oracle_lib):
    from ryg_rans_b200 import api
    nb, bs, ch = 3, 16384, 4096
    data = cb.block_data(nb, bs, 7)
    freqs, offs, blob = cb.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
    for flags in (0, CRC_BLOB):
        v2 = api.container_blocks_pack(nb, bs, ch, freqs, offs, blob, flags)
        rc, n, d_out = _async(gpu_ctx, gc._to_dev(v2), v2.size, data.size)
        assert rc == -4 and n == -1 and _untouched(d_out), flags


def test_async_space_and_the_symbol_count(gpu_ctx, word_case):
    data, _, _, good, _ = word_case
    rc, n, d_out = _async(gpu_ctx, gc._to_dev(good), good.size, data.size, out_cap=data.size - 1)
    assert rc == -3 and n == data.size and _untouched(d_out)
    # a content error comes before the space check; *d_n_symbols is written once the prefix passes, before the blob CRC
    bad = good.copy()
    bad[-7] ^= 0x40
    for cap in (data.size - 1, data.size):
        rc, n, d_out = _async(gpu_ctx, gc._to_dev(bad), bad.size, data.size, out_cap=cap)
        assert rc == -4 and n == data.size and _untouched(d_out), cap
    # a rejected prefix leaves it alone
    bad = good.copy()
    bad[70] ^= 0x40
    rc, n, d_out = _async(gpu_ctx, gc._to_dev(bad), bad.size, data.size)
    assert rc == -4 and n == -1 and _untouched(d_out)
    rc, n, d_out = _async(gpu_ctx, gc._to_dev(good), good.size, data.size)
    assert rc == 0 and np.array_equal(d_out[:n].cpu().numpy(), data)


def _corrupt_stream(buf):
    """a flags-0 container with one byte of its first stream changed: only the decoder can tell"""
    from ryg_rans_b200 import api
    meta, _, offs, _ = api.container_open(buf)
    assert meta["flags"] == 0
    bad = buf.copy()
    boff = buf.size - meta["blob_bytes"]
    bad[boff + int(offs[1]) // 2] ^= 0x5A
    return bad


def test_async_corrupt_stream_then_a_valid_container(gpu_ctx, oracle_lib, gen):
    torch = _torch()
    for coder, sb, kind in ((WORD, 12, "text"), (ALIAS, 16, "zipf"), (BYTE, 14, "zipf"), (RANS64, 12, "zipf")):
        good, data = _container(oracle_lib, gen, coder, sb, kind, 300000, 4096, 0, seed=coder)
        bad = _corrupt_stream(good)
        rc, n, _ = _async(gpu_ctx, gc._to_dev(bad), bad.size, data.size)
        assert rc == -4 and n == data.size, (coder, rc)
        # the valid one queued right behind a corrupt one, no rb200_sync in between: the sync reports the first call's
        # error, and the second call's output is complete
        d_bad, d_good = gc._to_dev(bad), gc._to_dev(good)
        d_out0 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
        d_out1 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), data.size)
        gpu_ctx.container_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), data.size)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4
        assert np.array_equal(d_out1[:data.size].cpu().numpy(), data), coder
        rc, n, d_out = _async(gpu_ctx, d_good, good.size, data.size)
        assert rc == 0 and np.array_equal(d_out[:n].cpu().numpy(), data), coder


def test_async_argument_errors_launch_nothing(gpu_ctx, word_case):
    torch = _torch()
    data, _, _, _, plain = word_case
    lib = gpu_ctx.lib.dll
    d_buf = gc._to_dev(plain, 64)
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(2, dtype=torch.int64, device="cuda")
    b, o, n = d_buf.data_ptr(), d_out.data_ptr(), d_n.data_ptr()
    before = gpu_ctx.launches
    calls = [(None, b, o, n), (gpu_ctx.h, None, o, n), (gpu_ctx.h, b, None, n), (gpu_ctx.h, b + 8, o, n), (gpu_ctx.h, b, o + 8, n),
             (gpu_ctx.h, b + 4, o, n), (gpu_ctx.h, b, o + 1, n), (gpu_ctx.h, b, o, n + 4)]
    for ctx, bp, op, np_ in calls:
        assert lib.rb200_container_decode_async(ctx, bp, plain.size, op, data.size, np_) == -1, (bp, op, np_)
    assert gpu_ctx.launches == before
    gpu_ctx.container_decode_async(b, plain.size, o, data.size, n)
    gpu_ctx.sync()
    assert torch.equal(d_out[:data.size].cpu(), torch.from_numpy(data))


def test_async_calls_queue(gpu_ctx, oracle_lib, gen):
    """three calls of different coders back to back with an rb200_decode between them, then one rb200_sync"""
    torch = _torch()
    cases = [_container(oracle_lib, gen, c, sb, k, n, ch, f, seed=9)
             for c, sb, k, n, ch, f in ((ALIAS, 14, "zipf", 1_000_003, 4096, CRC_BLOB), (WORD, 12, "text", 2_000_000, 8192, 0),
                                        (RANS64, 16, "uniform", 400_000, 2048, CRC_BLOB))]
    plain = gen("zipf", 1_500_000, 12)
    freqs, cum = oracle_lib.model(plain, 12)
    pb, po = oracle_lib.chunked_encode(WORD, plain, freqs, cum, 4096)
    model = gpu_ctx.model(WORD, 12, freqs)
    d_pb, d_po = gc._to_dev(pb), gc._to_dev(po.view(np.uint8))
    d_pout = torch.zeros(plain.size + 16, dtype=torch.uint8, device="cuda")
    keep, outs = [], []
    for i, (buf, data) in enumerate(cases):
        d_buf = gc._to_dev(buf)
        d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        keep.append(d_buf)
        outs.append(d_out)
        gpu_ctx.container_decode_async(d_buf.data_ptr(), buf.size, d_out.data_ptr(), data.size)
        if i == 0:
            gpu_ctx.decode_device(model, d_pb.data_ptr(), pb.size, d_po.data_ptr(), 4096, d_pout.data_ptr(), plain.size)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    for (_, data), d_out in zip(cases, outs):
        assert np.array_equal(d_out[:data.size].cpu().numpy(), data)
        assert _untouched(d_out[data.size:])
    assert np.array_equal(d_pout[:plain.size].cpu().numpy(), plain)
    model.close()


def test_async_decoder_picked_on_the_device_in_a_cuda_graph(oracle_lib, gen):
    """ONE captured call, replayed over containers of four coders copied into the same buffer, a corrupt stream and a
    valid container again: the decoder that runs is chosen on the GPU at every replay"""
    import ryg_rans_b200 as rb
    torch = _torch()
    conts = [_container(oracle_lib, gen, c, sb, k, n, ch, f, seed=20 + c)
             for c, sb, k, n, ch, f in ((ALIAS, 16, "zipf", 900_001, 4096, CRC_BLOB), (WORD, 12, "const", 300_000, 8192, 0),
                                        (BYTE, 10, "zipf", 500_000, 1024, CRC_BLOB), (RANS64, 14, "zipf", 600_000, 4096, 0),
                                        (WORD, 12, "uniform", 1_000_000, 8192, CRC_BLOB))]
    corrupt = _corrupt_stream(conts[3][0])
    size = max(c.size for c, _ in conts) + 256                       # fixed for the graph: the containers are shorter
    cap = max(d.size for _, d in conts)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    d_buf = torch.zeros(size, dtype=torch.uint8, device="cuda")
    d_out = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    decode = lambda: ctx.container_decode_async(d_buf.data_ptr(), size, d_out.data_ptr(), cap, d_n.data_ptr())  # noqa: E731
    with torch.cuda.stream(stream):
        def load(buf):
            d_buf.zero_()
            d_buf[:buf.size].copy_(torch.from_numpy(buf))
            d_out.fill_(SENTINEL)
            d_n.fill_(-1)
        load(conts[0][0])                                            # one call outside the graph first
        decode()
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            decode()
        launches = ctx.launches
        for buf, data, want in [(c, d, 0) for c, d in conts] + [(corrupt, None, -4), (conts[0][0], conts[0][1], 0)]:
            load(buf)
            g.replay()
            rc = ctx.lib.dll.rb200_sync(ctx.h)
            assert rc == want, (buf.size, rc)
            if data is not None:
                assert int(d_n.item()) == data.size
                assert np.array_equal(d_out[:data.size].cpu().numpy(), data), buf.size
                assert _untouched(d_out[data.size:])
        assert ctx.launches == launches                              # replays do not go through the library
    del g
    ctx.close()


def test_encode_and_async_decode_in_one_cuda_graph(oracle_lib, gen):
    """INTEGRATION.md's device-resident round trip: rb200_container_encode (alias coder) and the async decode captured
    together, replayed on new data under the same model"""
    import ryg_rans_b200 as rb
    torch = _torch()
    n, chunk, sb = 4_000_000, 8192, 16
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    freqs, _ = oracle_lib.model(gen("zipf", n, 80), sb)
    model = ctx.model(ALIAS, sb, freqs)
    cap = ctx.container_capacity(n, chunk)
    d_in = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_encode_device(model, d_in.data_ptr(), n, chunk, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(gen("zipf", n, 80)))
        round_trip()                                                 # grows the encoder's workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for seed in (81, 82):
            data = gen("zipf", n, seed)
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            assert int(d_n.item()) == n and np.array_equal(d_out[:n].cpu().numpy(), data), seed
    del g
    model.close()
    ctx.close()
