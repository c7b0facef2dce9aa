"""rb200_container_planes_encode_async and rb200_container_planes_decode_async: version 7 byte-plane containers, encoded
and decoded on the GPU.

- The container equals rb200_container_planes_pack of rb200_container_stored_encode_async run on each plane split in
  numpy, with the same candidates, tolerance, chunk_syms and flags: bf16, fp16, fp32 and fp64 of normal data at two
  scales, int32 small integers and uniform bytes; n / w a multiple of chunk_syms, ragged, below one chunk and 1; chunks
  of 32, 8192 and 2^24; flags 0 and blob CRC.  Every container fits the bound, and the decode returns the input and n.
- It is smaller than version 6 on the same bytes for bf16, fp32 and fp64 normal data.
- A plane with no feasible candidate is RB200_E_MODEL with the header unwritten; argument errors launch nothing;
  every broken decode leaves out untouched and the context decodes the intact buffer next; every other async decode
  rejects version 7.
- One CUDA graph of encode and decode replays on new data; a bf16 container past 2^32 bytes checks plane by plane."""
import ctypes as C
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
import test_gpu_blocks_coder as gbc  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
THREE = [CAND(WORD, 12), CAND(ALIAS, 16), CAND(BYTE, 14)]
E_ARG, E_MODEL, E_SPACE, E_STREAM = -1, -2, -3, -4
W_OF = {"bf16": 2, "fp16": 2, "fp32": 4, "fp64": 8, "int32": 4}


def _torch():
    import torch
    return torch


def elements(kind, w, count, seed, scale):
    """count elements of w bytes: normal floats of the given scale, small integers, or uniform bytes"""
    if kind == "uniform":
        return np.random.default_rng(seed).integers(0, 256, count * w, dtype=np.uint8)
    if kind == "int32":
        return cp.elements("int32", count, seed)
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, scale, count)
    if kind == "bf16":
        return (x.astype(np.float32).view(np.uint32) >> 16).astype("<u2").view(np.uint8)
    if kind == "fp16":
        return x.astype("<f2").view(np.uint8)
    if kind == "fp32":
        return x.astype("<f4").view(np.uint8)
    return x.astype(np.float32).astype("<f8").view(np.uint8)


def v6_size(buf):
    return cs.blob_offset(int(buf[24:32].view(np.uint64)[0])) + int(buf[32:40].view(np.uint64)[0])


def v7_size(buf):
    w = int(buf[52:56].view(np.uint32)[0])
    return 64 + 16 * w + int(buf[32:40].view(np.uint64)[0])


def encode_v6(ctx, cands, tol, data, ch, flags):
    torch = _torch()
    cap = api.container_stored_bound(data.size, ch)
    d_in = gbc._dev(data)
    d_out = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    ctx.container_stored_encode_async(cands, tol, d_in.data_ptr(), data.size, ch, flags, d_out.data_ptr(), cap)
    ctx.sync()
    out = d_out.cpu().numpy()
    return out[:v6_size(out)].copy()


def expected(ctx, cands, tol, data, w, ch, flags):
    """the composed oracle: the version 6 encode of each numpy-split plane, packed on the host"""
    return api.container_planes_pack([encode_v6(ctx, cands, tol, pl, ch, flags) for pl in cp.split(data, w)])


def encode(ctx, cands, tol, data, w, ch, flags, cap=None):
    """(sync code, whole output buffer on the host): the plane encode into a sentinel-filled buffer of cap + 64 bytes"""
    torch = _torch()
    cap = api.container_planes_bound(data.size, w, ch) if cap is None else cap
    d_in = gbc._dev(data)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_planes_encode_async(cands, tol, w, d_in.data_ptr(), data.size, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


def decode(ctx, buf, w, out_cap, size=None, decode_call=None):
    """(sync code, *d_n, whole sentinel-filled output buffer of out_cap + 64 bytes on the host)"""
    torch = _torch()
    d_buf = gbc._dev(buf)
    d_out = torch.full((out_cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    size = buf.size if size is None else size
    if decode_call is None:
        ctx.container_planes_decode_async(w, d_buf.data_ptr(), size, d_out.data_ptr(), out_cap, d_n.data_ptr())
    else:
        decode_call(d_buf.data_ptr(), size, d_out.data_ptr(), out_cap, d_n.data_ptr())
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out.cpu().numpy()


def check_case(ctx, cands, tol, data, w, ch, flags, case):
    want = expected(ctx, cands, tol, data, w, ch, flags)
    rc, got = encode(ctx, cands, tol, data, w, ch, flags)
    assert rc == 0, case
    size = v7_size(got)
    assert size == want.size <= api.container_planes_bound(data.size, w, ch), case
    assert np.array_equal(got[:size], want), case
    assert np.all(got[-64:] == SENTINEL), case                             # nothing past the bound
    rc, n, out = decode(ctx, want, w, data.size)
    assert rc == 0 and n == data.size, case
    assert np.array_equal(out[:data.size], data) and np.all(out[data.size:] == SENTINEL), case
    return want


KINDS = [("bf16", 0.02), ("bf16", 3.0), ("fp16", 0.02), ("fp16", 1.0), ("fp32", 0.02), ("fp32", 3.0), ("fp64", 0.02),
         ("int32", 0), ("uniform2", 0), ("uniform8", 0)]


@pytest.mark.parametrize("ch", [32, 8192, 1 << 24])
@pytest.mark.parametrize("kind,scale", KINDS)
def test_container_equals_the_composed_oracle(gpu_ctx, kind, scale, ch):
    base = kind[:-1] if kind.startswith("uniform") else kind
    w = int(kind[-1]) if kind.startswith("uniform") else W_OF[kind]
    if ch == 1 << 24:
        counts = [ch, 1000, 1] if w <= 2 else [1000, 1]             # one whole 2^24 chunk per plane for the 2-byte kinds
    else:
        counts = [8 * ch if ch > 64 else 300 * ch, 5 * ch + 17, ch - 5, 1]
    for i, count in enumerate(counts):
        data = elements(base, w, count, 31 * i + len(kind), scale)
        cands = THREE if i % 2 == 0 else [CAND(RANS64, 11), CAND(BYTE, 12), CAND(ALIAS, 9)]
        for tol, flags in ((20000, i & 1), (0, CRC_BLOB)) if count > 1 else ((20000, 0),):
            check_case(gpu_ctx, cands, tol, data, w, ch, flags, (kind, scale, ch, count, tol, flags))


# fp64 of fp32 values has three constant planes.  The single-model choice counts 0 bits for the word coder on one symbol,
# whose WIDE step writes 16 bits per symbol, so with the word coder first those planes are stored (a byte per symbol);
# the byte coder first codes them in 128 bytes per chunk.
BYTE_FIRST = [CAND(BYTE, 14), CAND(WORD, 12), CAND(ALIAS, 16)]


@pytest.mark.parametrize("kind,cands", [("bf16", THREE), ("fp32", THREE), ("fp64", BYTE_FIRST)])
def test_smaller_than_version_6(gpu_ctx, kind, cands):
    ch, w = 8192, W_OF[kind]
    data = elements(kind, w, 64 * ch // w * 2, 5, 0.02)
    v7 = check_case(gpu_ctx, cands, 20000, data, w, ch, 0, kind)
    v6 = encode_v6(gpu_ctx, cands, 20000, data, ch, 0)
    print(f"{kind}: {data.size} bytes, version 6 {v6.size} ({v6.size / data.size:.4f}), version 7 {v7.size} ({v7.size / data.size:.4f})")
    assert v7.size < v6.size


# ---- errors

def test_no_feasible_candidate_leaves_the_header_unwritten(gpu_ctx):
    """small non-negative int32: bytes 1..3 are zero, a plane of one symbol, which {byte 16} cannot code"""
    data = np.random.default_rng(3).integers(0, 40, 5000).astype("<i4").view(np.uint8)
    rc, got = encode(gpu_ctx, [CAND(BYTE, 16)], 0, data, 4, 8192, 0)
    assert rc == E_MODEL
    assert np.all(got[:64] == SENTINEL)
    rc, got = encode(gpu_ctx, [CAND(BYTE, 16), CAND(WORD, 12)], 0, data, 4, 8192, 0)   # the same context, a feasible list
    assert rc == 0 and np.array_equal(got[:v7_size(got)], expected(gpu_ctx, [CAND(BYTE, 16), CAND(WORD, 12)], 0, data, 4, 8192, 0))


def test_argument_errors_launch_nothing(gpu_ctx):
    torch = _torch()
    ch, w, n = 8192, 4, 4 * 10000
    d_in = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    cap = api.container_planes_bound(n, w, ch)
    d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    cands = (C.c_uint32 * 3)(*THREE)
    f = gpu_ctx.lib.dll.rb200_container_planes_encode_async
    ip, op = d_in.data_ptr(), d_out.data_ptr()
    cases = [(E_ARG, (1, ip, n, ch, op, cap)), (E_ARG, (3, ip, n, ch, op, cap)), (E_ARG, (16, ip, n, ch, op, cap)),
             (E_ARG, (w, ip, n + 2, ch, op, cap)), (E_ARG, (w, ip, 0, ch, op, cap)), (E_ARG, (w, ip + 1, n, ch, op, cap)),
             (E_ARG, (w, ip, n, ch, op + 8, cap)), (E_ARG, (w, ip, n, 16, op, cap)), (E_ARG, (w, ip, w << 32, ch, op, 1 << 40)),
             (E_SPACE, (w, ip, n, ch, op, cap - 1))]
    before = gpu_ctx.launches
    for want, (ew, i, nn, c, o, oc) in cases:
        assert f(gpu_ctx.h, cands, 3, 20000, ew, i, nn, c, 0, o, oc) == want, (ew, nn, c, oc)
    assert f(gpu_ctx.h, cands, 3, 2000000, w, ip, n, ch, 0, op, cap) == E_ARG     # tolerance above 10^6
    g = gpu_ctx.lib.dll.rb200_container_planes_decode_async
    for ew in (0, 1, 3, 16):
        assert g(gpu_ctx.h, ew, op, cap, ip, n, None) == E_ARG
    assert g(gpu_ctx.h, w, op + 8, cap, ip, n, None) == E_ARG
    assert gpu_ctx.launches == before
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0


@pytest.fixture(scope="module")
def intact(gpu_ctx):
    """(data, container) for bf16 normal data with the blob CRC, chunks of 8192, ragged"""
    data = elements("bf16", 2, 5 * 8192 + 77, 9, 0.02)
    return data, expected(gpu_ctx, THREE, 20000, data, 2, 8192, CRC_BLOB)


def broken_buffers(data, buf):
    w = 2
    out = {}
    b = buf.copy()
    cp.set_u64(b, 80, cp.u64(buf, 80) + 16)                            # plane 1's offset moved by 16
    out["offset"] = cp.reseal(b)
    b = buf.copy()
    cp.set_u64(b, 72, cp.u64(buf, 72) + 16)                            # size[0] off by 16
    out["size"] = cp.reseal(b)
    b = buf.copy()
    o1, s1 = cp.u64(buf, 64 + 16), cp.u64(buf, 64 + 24)
    b[o1 + s1 - 40] ^= 0x10                                            # a byte of plane 1's blob, under its blob CRC
    out["plane 1 blob"] = b
    b = buf.copy()
    b[o1 + 100] ^= 0x01                                                # plane 1's model
    out["plane 1 model"] = b
    b = buf.copy()
    b[64 + 3] ^= 0x01                                                  # a table byte: meta_crc
    out["table crc"] = b
    assert w == 2
    return out


def test_decode_rejects_leave_out_untouched(gpu_ctx, intact):
    data, buf = intact
    n = data.size
    cases = [(name, b, 2, n, None, E_STREAM) for name, b in broken_buffers(data, buf).items()]
    cases += [("short by 16", buf, 2, n, buf.size - 16, E_STREAM), ("elem_bytes 4", buf, 4, n, None, E_STREAM),
              ("elem_bytes 8", buf, 8, n, None, E_STREAM), ("out_cap", buf, 2, n - 1, None, E_SPACE),
              ("version 6", encode_v6(gpu_ctx, THREE, 20000, data, 8192, CRC_BLOB), 2, n, None, E_STREAM)]
    for name, b, w, cap, size, want in cases:
        rc, d_n, out = decode(gpu_ctx, b, w, cap, size)
        assert rc == want, name
        assert np.all(out == SENTINEL), name
        if want == E_SPACE:
            assert d_n == n, name
        rc, d_n, out = decode(gpu_ctx, buf, 2, n)                       # the same context decodes the intact buffer
        assert rc == 0 and d_n == n and np.array_equal(out[:n], data), name


def test_other_async_decodes_reject_version_7(gpu_ctx, intact):
    data, buf = intact
    c = gpu_ctx
    calls = {"v1": c.container_decode_async, "v6": c.container_stored_decode_async, "v5": c.container_blocks_stored_decode_async,
             "any": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_any_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v2": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v3": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_coder_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v4": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_alias_decode_async(c.h, *a[:4], a[4] or None), c.h)}
    for name, call in calls.items():
        rc, _, out = decode(c, buf, 2, data.size, decode_call=call)
        assert rc == E_STREAM and np.all(out == SENTINEL), name


# ---- graphs

def test_one_graph_encodes_and_decodes_new_data():
    torch = _torch()
    ch, w = 8192, 2
    n = 2 * (40 * ch + 123)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_planes_bound(n, w, ch)
    d_in = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_planes_encode_async(THREE, 20000, w, d_in.data_ptr(), n, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_planes_decode_async(w, d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in[:n].copy_(torch.from_numpy(elements("bf16", 2, n // 2, 1, 0.02)))
        round_trip()                                                 # grows the workspaces outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        for i, (kind, scale) in enumerate((("bf16", 3.0), ("uniform", 0), ("bf16", 0.02), ("fp16", 0.02))):
            data = elements(kind, 2, n // 2, 50 + i, scale)
            d_in[:n].copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, kind
            got = d_buf.cpu().numpy()
            want = expected(ctx, THREE, 20000, data, w, ch, CRC_BLOB)   # the eager calls, on the same context
            assert np.array_equal(got[:v7_size(got)], want), kind
            assert int(d_n.item()) == n and np.array_equal(d_out[:n].cpu().numpy(), data), kind
        del g
    ctx.close()


# ---- past 2^32

def test_bf16_past_4_gib():
    """n / 2 = 2^32 - 2^20 symbols: plane 0 (the near-uniform low byte, stored) is past 2^32 bytes, so plane 1's offset
    is too.  Encode, check each plane against its version 6 encode, decode; one context at a time."""
    torch = _torch()
    ch, w = 8192, 2
    m = (1 << 32) - (1 << 20)
    n = w * m
    cap = api.container_planes_bound(n, w, ch)
    n_chunks = -(-m // ch)
    scratch = n_chunks * ((512 + 2 * ch + 15) // 16 * 16)            # the stored encode's worst-case slots
    v6_cap = api.container_stored_bound(m, ch)
    # resident: input, container; encode: split planes, staging and scratch; oracle: a plane, its container and scratch;
    # decode: decoded planes, staging and output (each workspace grows by an eighth)
    phases = [1.125 * (n + v6_cap + scratch), m + v6_cap + 1.125 * scratch, 1.125 * (n + cap) + n]
    need = n + cap + max(phases) + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} free")
    gen = torch.Generator(device="cuda").manual_seed(7)
    d_in = torch.empty(n, dtype=torch.uint8, device="cuda")
    step = 1 << 26
    for a in range(0, m, step):                                       # in slices: no full-size float32 temporary
        b = min(m, a + step)
        d_in.view(torch.bfloat16)[a:b] = (torch.randn(b - a, device="cuda", generator=gen) * 0.02).to(torch.bfloat16)
    torch.cuda.empty_cache()                                          # the library allocates with cudaMalloc
    d_buf = torch.full((cap,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx = rb.Context(0)
    ctx.container_planes_encode_async(THREE, 20000, w, d_in.data_ptr(), n, ch, 0, d_buf.data_ptr(), cap)
    ctx.sync()
    ctx.close()
    head = d_buf[:64 + 16 * w].cpu().numpy()
    table = head[64:].view(np.uint64).reshape(w, 2)
    assert int(table[1, 0]) > (1 << 32) and int(table[0, 0]) == 64 + 16 * w
    size = 64 + 16 * w + int(head[32:40].view(np.uint64)[0])
    assert int(table[1, 0] + table[1, 1]) == size <= cap
    ctx = rb.Context(0)
    for p in range(w):
        plane = d_in.view(-1, w)[:, p].contiguous()
        d_v6 = torch.zeros(v6_cap, dtype=torch.uint8, device="cuda")
        ctx.container_stored_encode_async(THREE, 20000, plane.data_ptr(), m, ch, 0, d_v6.data_ptr(), v6_cap)
        ctx.sync()
        off, sz = int(table[p, 0]), int(table[p, 1])
        assert torch.equal(d_buf[off:off + sz], d_v6[:sz]), p
        del plane, d_v6
        torch.cuda.empty_cache()
    ctx.close()
    crc = zlib.crc32(np.concatenate([head[:44], np.zeros(8, np.uint8), head[52:]]).tobytes())
    assert crc == int(head[44:48].view(np.uint32)[0])
    ctx = rb.Context(0)
    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    ctx.container_planes_decode_async(w, d_buf.data_ptr(), size, d_out.data_ptr(), n, d_n.data_ptr())
    ctx.sync()
    assert int(d_n.item()) == n and torch.equal(d_out, d_in)
    ctx.close()
