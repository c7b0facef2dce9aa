"""rb200_container_planes_encode_varlen_async: the version 7 byte-plane encode with the length read from device memory
when the work runs, so one captured graph writes a container for a tensor of any size up to the bound.

- Byte equality with the fixed call (rb200_container_planes_encode_async) at the same length: bf16, fp16, fp32 and fp64
  normal data, int32 small integers and uniform bytes of 2, 4 and 8-byte elements; chunks of 32, 8192 and 2^24; flags 0
  and blob CRC; lengths of 1 element, below one chunk, ragged, a multiple of the chunk, n_max - w and n_max.  Nothing
  past the container is written.  A few lengths also equal the composed oracle (numpy-split planes, each encoded by the
  version 6 call, packed on the host).
- Input past *d_n is not read; the bound of n_max holds every length (and is met on uniform data); a bad length writes
  nothing; argument errors launch nothing; launch counts are pinned.
- One graph of the varlen encode and the version 7 decode (captured with size = the bound) follows lengths from 1
  element to n_max, with *d_n written by a kernel inside the graph; two contexts replay their own graphs at once; a
  bf16 container whose second plane starts past 2^32 bytes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_stored as cs  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_planes as gcp  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = gcp.SENTINEL
THREE = gcp.THREE
OTHER = [CAND(RANS64, 11), CAND(BYTE, 12), CAND(ALIAS, 9)]
E_ARG, E_SPACE = -1, -3


def _torch():
    import torch
    return torch


def _dn(value):
    torch = _torch()
    return torch.tensor([value], dtype=torch.int64, device="cuda")


def fixed7(ctx, cands, tol, d_in, n, w, ch, flags):
    """the fixed call's container for the first n bytes of d_in, on the host"""
    torch = _torch()
    cap = api.container_planes_bound(n, w, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_planes_encode_async(cands, tol, w, d_in.data_ptr(), n, ch, flags, d_out.data_ptr(), cap)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    buf = d_out.cpu().numpy()
    return buf[:gcp.v7_size(buf)]


def varlen7(ctx, cands, tol, d_in, n, n_max, w, ch, flags, cap=None):
    """(sync code, whole output buffer on the host): the varlen encode of *d_n = n into a sentinel-filled buffer of
    cap + 64 bytes"""
    torch = _torch()
    cap = api.container_planes_bound(n_max, w, ch) if cap is None else cap
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = _dn(n)
    ctx.container_planes_encode_varlen_async(cands, tol, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


def data_of(kind, w, count, seed, scale=0.02):
    base = "uniform" if kind.startswith("uniform") else kind             # uniform2, uniform8: the width is w
    return gcp.elements(base, w, count, seed, scale)


def skewed(count, w, seed):
    """every byte of every element from a geometric distribution: every plane is coded"""
    rng = np.random.default_rng(seed)
    return np.minimum(rng.geometric(0.3, count * w) - 1, 255).astype(np.uint8)


def _lengths(ch, m_max):
    """element counts: 1, below one chunk, ragged, a multiple of the chunk, m_max - 1, m_max"""
    return sorted(x for x in {1, ch - 5, 3 * ch + 17, 4 * ch, m_max - 1, m_max} if 1 <= x <= m_max)


KINDS = [("bf16", 2), ("fp16", 2), ("fp32", 4), ("fp64", 8), ("int32", 4), ("uniform2", 2), ("uniform8", 8)]


@pytest.mark.parametrize("ch", [32, 8192, 1 << 24])
@pytest.mark.parametrize("kind,w", KINDS)
def test_varlen_equals_the_fixed_call(gpu_ctx, kind, w, ch):
    if ch == 1 << 24:
        # one whole 2^24 chunk per plane for the 2-byte kinds; below one chunk (ragged) for the others
        m_max = ch + 1000 if w <= 2 else 5000
        lengths = sorted({1, 1000, ch - 5, ch, m_max - 1, m_max} if w <= 2 else {1, 999, m_max - 1, m_max})
    else:
        m_max = (300 if ch == 32 else 6) * ch + 23
        lengths = _lengths(ch, m_max)
    data = data_of(kind, w, m_max, KINDS.index((kind, w)) + ch % 7)
    d_in = gbc._dev(data)
    for li, m in enumerate(lengths):
        cands, tol = (THREE, 20000) if li % 2 == 0 else (OTHER, 0)
        for flags in (0, CRC_BLOB):
            case = (kind, ch, m, flags)
            want = fixed7(gpu_ctx, cands, tol, d_in, m * w, w, ch, flags)
            rc, got = varlen7(gpu_ctx, cands, tol, d_in, m * w, m_max * w, w, ch, flags)
            assert rc == 0, case
            assert np.array_equal(got[:want.size], want), case
            assert (got[want.size:] == SENTINEL).all(), case


@pytest.mark.parametrize("kind,w", [("bf16", 2), ("fp32", 4), ("fp64", 8)])
def test_varlen_equals_the_composed_oracle(gpu_ctx, kind, w):
    ch = 8192
    m_max = 5 * ch + 77
    data = data_of(kind, w, m_max, 17)
    d_in = gbc._dev(data)
    for m in (1, 2 * ch + 3, m_max):
        for flags in (0, CRC_BLOB):
            want = gcp.expected(gpu_ctx, THREE, 20000, data[:m * w], w, ch, flags)
            rc, got = varlen7(gpu_ctx, THREE, 20000, d_in, m * w, m_max * w, w, ch, flags)
            assert rc == 0, (kind, m, flags)
            assert np.array_equal(got[:want.size], want), (kind, m, flags)
            assert (got[want.size:] == SENTINEL).all(), (kind, m, flags)


def test_input_past_the_length_is_not_read(gpu_ctx):
    ch, w = 8192, 4
    m_max = 7 * ch + 9
    data = data_of("fp32", w, m_max, 23)
    for m in (1, 3 * ch + 1, m_max - 1):
        n = m * w
        outs = []
        for pattern in (np.zeros(data.size - n, np.uint8), np.random.default_rng(m).integers(0, 256, data.size - n, dtype=np.uint8)):
            d_in = gbc._dev(np.concatenate([data[:n], pattern]))
            rc, got = varlen7(gpu_ctx, THREE, 20000, d_in, n, m_max * w, w, ch, CRC_BLOB)
            assert rc == 0, m
            outs.append(got)
        assert np.array_equal(outs[0], outs[1]), m
        want = fixed7(gpu_ctx, THREE, 20000, gbc._dev(data[:n]), n, w, ch, CRC_BLOB)
        assert np.array_equal(outs[0][:want.size], want), m


# ---- the bound, bad lengths, errors and launches

@pytest.mark.parametrize("w", [2, 4])
def test_bound_holds_for_every_length(gpu_ctx, w):
    ch = 8192
    m_max = 6 * ch + 23
    n_max = m_max * w
    d_in = gbc._dev(data_of("uniform", w, m_max, 3))
    bound = api.container_planes_bound(n_max, w, ch)
    for m in _lengths(ch, m_max):
        n = m * w
        for cands in (THREE, [CAND(WORD, 12)]):
            rc, got = varlen7(gpu_ctx, cands, 0, d_in, n, n_max, w, ch, CRC_BLOB, cap=bound)
            assert rc == 0, (m, cands)
            assert gcp.v7_size(got) == api.container_planes_bound(n, w, ch), (m, cands)   # uniform: every plane stored
            assert (got[gcp.v7_size(got):] == SENTINEL).all(), (m, cands)
    before = gpu_ctx.launches
    d_out = _torch().full((bound + 64,), SENTINEL, dtype=_torch().uint8, device="cuda")
    d_n = _dn(n_max)
    with pytest.raises(api.RansError) as e:
        gpu_ctx.container_planes_encode_varlen_async(THREE, 0, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, 0, d_out.data_ptr(), bound - 1)
    assert e.value.code == E_SPACE
    assert gpu_ctx.launches == before and (d_out.cpu().numpy() == SENTINEL).all()


def test_bound_is_met_and_not_exceeded_on_normal_data(gpu_ctx):
    ch, w = 8192, 2
    m_max = 9 * ch + 5
    d_in = gbc._dev(data_of("bf16", w, m_max, 8))
    bound = api.container_planes_bound(m_max * w, w, ch)
    for m in _lengths(ch, m_max):
        for cands in (THREE, [CAND(WORD, 12)]):
            rc, got = varlen7(gpu_ctx, cands, 0, d_in, m * w, m_max * w, w, ch, 0, cap=bound)
            assert rc == 0 and gcp.v7_size(got) <= api.container_planes_bound(m * w, w, ch), (m, cands)


@pytest.mark.parametrize("w", [2, 4])
def test_bad_lengths_write_nothing(gpu_ctx, w):
    ch = 4096
    m_max = 10 * ch + 5
    n_max = m_max * w
    data = np.concatenate([gcp.elements("uniform", w, m_max // 2, 4, 0), skewed(m_max - m_max // 2, w, 4)])
    d_in = gbc._dev(data)
    for cands in (THREE, [CAND(BYTE, 14)]):
        for bad in (0, w - 1, n_max - 1, n_max + w, -1):
            for flags in (0, CRC_BLOB):
                case = (cands, bad, flags)
                rc, got = varlen7(gpu_ctx, cands, 0, d_in, bad, n_max, w, ch, flags)
                assert rc == E_ARG and (got == SENTINEL).all(), case
                good = n_max - 3 * w
                rc, got = varlen7(gpu_ctx, cands, 0, d_in, good, n_max, w, ch, flags)
                want = fixed7(gpu_ctx, cands, 0, d_in, good, w, ch, flags)
                assert rc == 0 and np.array_equal(got[:want.size], want), case


def test_argument_errors_and_launch_counts(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    ch = 8192
    m_max = ch * 40 + 5                                                 # the version 6 varlen test's launch geometry per plane
    for w in (2, 4):
        n_max = m_max * w
        data = np.concatenate([gcp.elements("uniform", w, m_max // 2, 1, 0), skewed(m_max - m_max // 2, w, 1)])
        d_in = gbc._dev(data)
        bound = api.container_planes_bound(n_max, w, ch)
        d_buf = torch.full((bound + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        good = n_max - 100 * w
        d_n = torch.tensor([n_max, good], dtype=torch.int64, device="cuda")
        i, o, p = d_in.data_ptr(), d_buf.data_ptr(), d_n.data_ptr()

        def call(cands, tol=0, ctx=gpu_ctx.h, ew=w, inp=i, np_=p, nmax=n_max, chunk=ch, flags=0, out=o, out_cap=bound):
            c = np.ascontiguousarray(cands, dtype=np.uint32)
            return lib.rb200_container_planes_encode_varlen_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size,
                                                                  tol, ew, inp, np_, nmax, chunk, flags, out, out_cap)
        before = gpu_ctx.launches
        for bad in ([], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 17)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
            assert call(bad) == E_ARG, bad
        assert call(THREE, tol=10 ** 6 + 1) == E_ARG
        for kw in ({"ctx": None}, {"inp": None}, {"inp": i + 1}, {"out": None}, {"out": o + 8}, {"np_": None}, {"np_": p + 4},
                   {"nmax": 0}, {"nmax": n_max + 1}, {"ew": 1}, {"ew": 3}, {"ew": 16}, {"chunk": 16}, {"chunk": 31},
                   {"chunk": (1 << 24) + 1}, {"nmax": w << 32, "out_cap": 1 << 40}):
            assert call(THREE, **kw) == E_ARG, (w, kw)
        assert call(THREE, out_cap=bound - 1) == E_SPACE
        assert gpu_ctx.launches == before, w
        assert (d_buf.cpu().numpy() == SENTINEL).all(), w
        # plan + split + per plane (version 6's varlen encode + place) + finish; version 6's varlen encode at this
        # geometry: 13 for the list, 11 for the word coder alone, 2 more with the blob CRC.  The fixed call has neither
        # plan kernel nor blob-length kernels.
        for cands, flags, v6 in ((THREE, 0, 13), (THREE, CRC_BLOB, 15), ([CAND(WORD, 12)], 0, 11), ([CAND(WORD, 12)], CRC_BLOB, 13)):
            case = (w, cands, flags)
            before = gpu_ctx.launches
            assert call(cands, flags=flags, np_=p + 8) == 0, case
            got = gpu_ctx.launches - before
            assert got == 3 + w * (v6 + 1), (case, got)
            assert lib.rb200_sync(gpu_ctx.h) == 0, case
            before = gpu_ctx.launches
            want = fixed7(gpu_ctx, cands, 0, d_in, good, w, ch, flags)
            assert got - (gpu_ctx.launches - before) == 1 + w * (2 if flags else 1), case
            assert np.array_equal(d_buf[:want.size].cpu().numpy(), want), case


# ---- graphs

def _stored_fraction(buf, w, ch):
    """the share of all planes' chunks that are stored"""
    table = buf[64:64 + 16 * w].view(np.uint64).reshape(w, 2)
    stored = total = 0
    for p in range(w):
        plane = buf[int(table[p, 0]):int(table[p, 0] + table[p, 1])]
        n_chunks = int(plane[24:32].view(np.uint64)[0])
        at = cs._bitmap_at(n_chunks)
        bits = plane[at:at + 4 * ((n_chunks + 31) // 32)].view(np.uint32)
        stored += sum(bin(int(x)).count("1") for x in bits)
        total += n_chunks
    return stored / total


@pytest.mark.parametrize("kind,w", [("bf16", 2), ("fp32", 4)])
def test_one_graph_many_lengths(kind, w):
    """*d_n is written inside the graph, by a torch kernel from an element count the host sets before each replay"""
    torch = _torch()
    ch = 8192
    m_max = 40 * ch + 123
    n_max = m_max * w
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_planes_bound(n_max, w, ch)
    d_in = torch.empty(n_max + 16, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n_max + 64, dtype=torch.uint8, device="cuda")
    d_elems = _dn(m_max)
    d_n = _dn(n_max)
    d_nsym = _dn(0)

    def round_trip():
        torch.mul(d_elems, w, out=d_n)
        ctx.container_planes_encode_varlen_async(THREE, 20000, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_planes_decode_async(w, d_buf.data_ptr(), cap, d_out.data_ptr(), n_max, d_nsym.data_ptr())

    with torch.cuda.stream(stream):
        d_in[:n_max].copy_(torch.from_numpy(data_of(kind, w, m_max, 1)))
        round_trip()                                                 # grows the workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        stored = set()
        steps = ((1, "uniform"), (13 * ch + 1000, kind), (m_max, "half"), (30 * ch, "skewed"), (5 * ch + 7, kind))
        for step, (m, what) in enumerate(steps):
            n = m * w
            if what == "half":
                data = np.concatenate([gcp.elements("uniform", w, m // 2, 50 + step, 0), skewed(m - m // 2, w, 50 + step)])
            else:
                data = skewed(m, w, 50 + step) if what == "skewed" else data_of(what, w, m, 50 + step)
            d_in[:n].copy_(torch.from_numpy(data))
            d_elems.fill_(m)
            d_buf.fill_(SENTINEL)
            d_out.fill_(SENTINEL)
            d_nsym.fill_(-1)
            launches = ctx.launches
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, m
            assert ctx.launches == launches                          # a replay does not go through the library
            assert int(d_n.item()) == n
            want = fixed7(ctx, THREE, 20000, d_in, n, w, ch, CRC_BLOB)
            got = d_buf.cpu().numpy()
            assert np.array_equal(got[:want.size], want) and (got[want.size:] == SENTINEL).all(), m
            assert int(d_nsym.item()) == n, m
            out = d_out.cpu().numpy()
            assert np.array_equal(out[:n], data) and (out[n:] == SENTINEL).all(), m
            stored.add(_stored_fraction(got, w, ch))
        assert 1.0 in stored and 0.0 in stored and len(stored) >= 3, stored
        del g
    ctx.close()


def test_two_contexts_replay_their_own_graphs():
    """the length record is per context: two graphs of the same geometry replay at once at different lengths"""
    torch = _torch()
    ch, w = 8192, 2
    m_max = 24 * ch + 51
    n_max = m_max * w
    cap = api.container_planes_bound(n_max, w, ch)
    data = data_of("bf16", w, m_max, 12)
    sides = []
    for k in range(2):
        stream = torch.cuda.Stream()
        ctx = rb.Context(0, stream=stream.cuda_stream)
        d_in = gbc._dev(data if k == 0 else data[::-1].copy())
        d_buf = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        d_n = _dn(n_max)
        with torch.cuda.stream(stream):
            ctx.container_planes_encode_varlen_async(THREE, 20000, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, CRC_BLOB, d_buf.data_ptr(), cap)
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                ctx.container_planes_encode_varlen_async(THREE, 20000, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, CRC_BLOB, d_buf.data_ptr(),
                                                         cap)
        sides.append((stream, ctx, d_in, d_buf, d_n, g))
    torch.cuda.synchronize()
    for lengths in ((1, m_max), (m_max, 3 * ch + 5), (7 * ch, 7 * ch + 2), (m_max - 1, 2)):
        for (stream, ctx, d_in, d_buf, d_n, g), m in zip(sides, lengths):
            with torch.cuda.stream(stream):
                d_n.fill_(m * w)
                d_buf.fill_(SENTINEL)
                g.replay()                                           # no synchronisation between the two sides
        for (stream, ctx, d_in, d_buf, d_n, g), m in zip(sides, lengths):
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, lengths
            got = d_buf.cpu().numpy()
            with torch.cuda.stream(stream):
                want = fixed7(ctx, THREE, 20000, d_in, m * w, w, ch, CRC_BLOB)
            assert np.array_equal(got[:want.size], want) and (got[want.size:] == SENTINEL).all(), (lengths, m)
    for stream, ctx, d_in, d_buf, d_n, g in sides:
        del g
        ctx.close()


# ---- past 2^32

def test_bf16_past_4_gib():
    """n_max / 2 = 2^32 - 2^20 symbols: plane 0 (the near-uniform low byte, stored) ends past 2^32 bytes, so plane 1
    starts there.  At *d_n = n_max and at a shorter length that still crosses, the container equals the fixed call's,
    compared on the device; one context, the fixed and the varlen call sharing its workspaces."""
    torch = _torch()
    ch, w = 8192, 2
    m_max = (1 << 32) - (1 << 20)
    n_max = w * m_max
    cap = api.container_planes_bound(n_max, w, ch)
    n_chunks = -(-m_max // ch)
    scratch = n_chunks * ((512 + 2 * ch + 15) // 16 * 16)            # the stored encode's worst-case slots
    v6_cap = api.container_stored_bound(m_max, ch)
    # resident: input and two containers; the context: split planes, staging and scratch (each grows by an eighth)
    need = n_max + 2 * cap + 1.125 * (n_max + v6_cap + scratch) + (2 << 30)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} free")
    gen = torch.Generator(device="cuda").manual_seed(11)
    d_in = torch.empty(n_max, dtype=torch.uint8, device="cuda")
    step = 1 << 26
    for a in range(0, m_max, step):                                   # in slices: no full-size float32 temporary
        b = min(m_max, a + step)
        d_in.view(torch.bfloat16)[a:b] = (torch.randn(b - a, device="cuda", generator=gen) * 0.02).to(torch.bfloat16)
    torch.cuda.empty_cache()                                          # the library allocates with cudaMalloc
    d_var = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_fix = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_n = _dn(n_max)
    ctx = rb.Context(0)
    for m in (m_max, m_max - (1 << 20) - 777):
        n = w * m
        d_var.fill_(SENTINEL)
        d_n.fill_(n)
        torch.cuda.synchronize()
        ctx.container_planes_encode_varlen_async(THREE, 20000, w, d_in.data_ptr(), d_n.data_ptr(), n_max, ch, 0, d_var.data_ptr(), cap)
        ctx.sync()
        ctx.container_planes_encode_async(THREE, 20000, w, d_in.data_ptr(), n, ch, 0, d_fix.data_ptr(), api.container_planes_bound(n, w, ch))
        ctx.sync()
        head = d_fix[:64 + 16 * w].cpu().numpy()
        table = head[64:].view(np.uint64).reshape(w, 2)
        size = 64 + 16 * w + int(head[32:40].view(np.uint64)[0])
        assert int(table[1, 0]) > (1 << 32) and int(head[16:24].view(np.uint64)[0]) == n, m
        assert torch.equal(d_var[:size], d_fix[:size]), m
        assert bool((d_var[size:size + (1 << 20)] == SENTINEL).all().item()), m
    ctx.close()
