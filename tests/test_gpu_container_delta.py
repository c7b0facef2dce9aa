"""rb200_container_delta_encode_async and rb200_container_delta_decode_async: version 8 delta byte-plane containers,
encoded and decoded on the GPU.

- Exact oracle: bytes 64 onward of the version 8 container equal bytes 64 onward of the version 7 encode of d, where d
  is the zigzag difference computed in numpy from (in, base); the headers differ only in version, reserved (=
  zlib.crc32(base)) and meta_crc (recomputed).  bf16, fp16, fp32, fp64, int32 and uniform bytes; chunks of 32, 8192
  and 2^24 at ragged counts; both candidate lists, both tolerances and the blob CRC; crafted pairs (wraparound, sign
  crossings, NaN patterns, integer extremes).
- The decode gives in back with nothing written past n, also in place (out == base); a partial overlap is RB200_E_ARG
  with nothing launched.  A base with one bit flipped is RB200_E_BASE with out untouched, in place too; corrupt
  containers are RB200_E_STREAM with out untouched; the version 7 decode and every other async decode reject version 8,
  and the version 8 decode rejects version 7.
- Sizes on synthetic training steps (printed); an unchanged tensor under each candidate list.
- One CUDA graph of encode and in-place decode replays over steps with the base advancing, on one context and on two
  at once; a bf16 tensor of 2^32 - 2^20 elements; argument errors launch nothing."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_delta as cd  # noqa: E402
import test_container_planes as cp  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_planes as gcp  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = gcp.SENTINEL
THREE = gcp.THREE                                           # word first
BYTE_FIRST = [CAND(BYTE, 14), CAND(WORD, 12), CAND(ALIAS, 16)]   # the delta list
E_ARG, E_SPACE, E_STREAM, E_BASE = -1, -3, -4, -10
W_OF = {"bf16": 2, "fp16": 2, "fp32": 4, "fp64": 8, "int32": 4, "uniform2": 2, "uniform8": 8}


def _torch():
    import torch
    return torch


def pair(kind, count, seed, lr=1e-4):
    """(in, base) of count elements: for bf16 / fp32 a synthetic training step of lr from N(0, 0.02) weights; for the
    other kinds a third of the elements redrawn; for uniform every byte independent"""
    w = W_OF[kind]
    if kind.startswith("uniform"):
        rng = np.random.default_rng(seed)
        return rng.integers(0, 256, count * w, dtype=np.uint8), rng.integers(0, 256, count * w, dtype=np.uint8)
    base = gcp.elements(kind, w, count, seed, 0.02)
    if kind in ("bf16", "fp32"):
        return cd.step(base, kind, lr, seed + 1), base
    other = gcp.elements(kind, w, count, seed + 1, 0.02).reshape(-1, w)
    x = base.reshape(-1, w).copy()
    pick = np.random.default_rng(seed + 2).random(count) < 1 / 3
    x[pick] = other[pick]
    return x.reshape(-1), base


def v8_size(buf):
    return gcp.v7_size(buf)


def expected(ctx, cands, tol, x, base, w, ch, flags):
    """the oracle: the version 7 encode of numpy's d, relabelled version 8 with the base CRC and meta_crc resealed"""
    rc, v7 = gcp.encode(ctx, cands, tol, cd.zigzag(x, base, w), w, ch, flags)
    assert rc == 0
    buf = v7[:gcp.v7_size(v7)].copy()
    buf[4] = 8
    cp.set_u32(buf, 60, zlib.crc32(base.tobytes()))
    return cp.reseal(buf)


def encode(ctx, cands, tol, x, base, w, ch, flags, cap=None):
    """(sync code, whole output buffer on the host): the delta encode into a sentinel-filled buffer of cap + 64 bytes"""
    torch = _torch()
    cap = api.container_planes_bound(x.size, w, ch) if cap is None else cap
    d_in, d_base = gbc._dev(x), gbc._dev(base)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_delta_encode_async(cands, tol, w, d_in.data_ptr(), d_base.data_ptr(), x.size, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


def decode(ctx, buf, w, base, out_cap, size=None, in_place=False):
    """(sync code, *d_n, out buffer of out_cap + 64 bytes on the host, base on the host after the call).  out is
    sentinel-filled, or in place: base followed by 64 + out_cap - n sentinel bytes"""
    torch = _torch()
    d_buf = gbc._dev(buf)
    d_out = torch.full((out_cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    size = buf.size if size is None else size
    if in_place:
        d_out[:base.size].copy_(torch.from_numpy(base))
        d_base = d_out
    else:
        d_base = gbc._dev(base)
    ctx.container_delta_decode_async(w, d_buf.data_ptr(), size, d_base.data_ptr(), d_out.data_ptr(), out_cap, d_n.data_ptr())
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out.cpu().numpy(), d_base[:base.size].cpu().numpy()


def check_case(ctx, cands, tol, x, base, w, ch, flags, case):
    want = expected(ctx, cands, tol, x, base, w, ch, flags)
    rc, got = encode(ctx, cands, tol, x, base, w, ch, flags)
    assert rc == 0, case
    size = v8_size(got)
    assert size == want.size <= api.container_planes_bound(x.size, w, ch), case
    assert np.array_equal(got[:size], want), case
    assert np.all(got[-64:] == SENTINEL), case                                  # nothing past the bound
    for in_place in (False, True):
        rc, n, out, b = decode(ctx, want, w, base, x.size, in_place=in_place)
        assert rc == 0 and n == x.size, (case, in_place)
        assert np.array_equal(out[:x.size], x) and np.all(out[x.size:] == SENTINEL), (case, in_place)
        assert np.array_equal(b, x if in_place else base), (case, in_place)
    return want


KINDS = ["bf16", "fp16", "fp32", "fp64", "int32", "uniform2", "uniform8"]


@pytest.mark.parametrize("ch", [32, 8192, 1 << 24])
@pytest.mark.parametrize("kind", KINDS)
def test_container_equals_the_version_7_encode_of_d(gpu_ctx, kind, ch):
    w = W_OF[kind]
    if ch == 1 << 24:
        counts = [ch + 5, 1000, 1] if w <= 2 else [1000, 1]
    else:
        counts = [8 * ch + 3 if ch > 64 else 300 * ch + 7, 5 * ch + 17, ch - 5, 1]
    for i, count in enumerate(counts):
        x, base = pair(kind, count, 31 * i + len(kind))
        cands = BYTE_FIRST if i % 2 == 0 else THREE
        for tol, flags in ((20000, i & 1), (0, CRC_BLOB)) if count > 1 else ((20000, 0),):
            check_case(gpu_ctx, cands, tol, x, base, w, ch, flags, (kind, ch, count, tol, flags))


@pytest.mark.parametrize("w", [2, 4, 8])
def test_crafted_pairs(gpu_ctx, w):
    """wraparound (b all ones, x 0 and the reverse), sign crossings, NaN and infinity patterns, integer extremes, equal
    elements, random bits; then in and base swapped"""
    x, base = cd.crafted(w, seed=w)
    for cands in (BYTE_FIRST, THREE):
        check_case(gpu_ctx, cands, 20000, x, base, w, 32, CRC_BLOB, (w, "crafted"))
        check_case(gpu_ctx, cands, 0, base, x, w, 32, 0, (w, "swapped"))


# ---- sizes

def _as_kind(master, kind):
    if kind == "bf16":
        return (master.view(np.uint32) >> 16).astype("<u2").view(np.uint8)        # truncated, as elements() does
    return master.astype("<f4").view(np.uint8)


def _sizes(ctx, kind, lr, steps, count, ch=8192):
    """fp32 master weights from N(0, 0.02), moved by lr * sign * U(0, 1) per step; base the first, in the last, as kind"""
    w = W_OF[kind]
    rng = np.random.default_rng(3)
    master = rng.normal(0.0, 0.02, count).astype(np.float32)
    base = _as_kind(master, kind)
    for _ in range(steps):
        master = (master + lr * rng.choice([-1.0, 1.0], count) * rng.random(count)).astype(np.float32)
    x = _as_kind(master, kind)
    rc, v7 = gcp.encode(ctx, BYTE_FIRST, 20000, x, w, ch, 0)
    assert rc == 0
    v8 = check_case(ctx, BYTE_FIRST, 20000, x, base, w, ch, 0, (kind, lr, steps))
    return gcp.v7_size(v7) / x.size, v8.size / x.size


def test_sizes_on_training_steps(gpu_ctx):
    count = 1 << 21
    got = {}
    for kind in ("bf16", "fp32"):
        for lr, steps in ((1e-5, 1), (1e-4, 1), (1e-4, 100)):
            v7, v8 = _sizes(gpu_ctx, kind, lr, steps, count)
            got[(kind, lr, steps)] = (v7, v8)
            print(f"{kind} lr {lr:g} x {steps}: version 7 {v7:.4f}, version 8 {v8:.4f} bytes per input byte")
    v7, v8 = got[("bf16", 1e-4, 1)]
    assert v8 <= v7 / 2


def test_unchanged_tensor_under_each_list(gpu_ctx):
    """A frozen layer: d is all zero.  With the byte coder first each plane is coded in about 128 bytes per chunk; with
    the word coder first the single-model choice counts 0 bits for it on one symbol and the planes are stored."""
    x = gcp.elements("bf16", 2, (1 << 20) + 4096, 8, 0.02)
    sizes = {}
    for name, cands in (("byte first", BYTE_FIRST), ("word first", THREE)):
        v8 = check_case(gpu_ctx, cands, 20000, x, x, 2, 8192, 0, name)
        sizes[name] = v8.size / x.size
        meta, planes = api.container_delta_open(v8)
        coders = [api.container_stored_open(p)[0]["coder"] for p in planes]
        print(f"unchanged bf16, {x.size} bytes, {name}: {v8.size} bytes ({sizes[name]:.4f}), plane coders {coders}")
    assert sizes["byte first"] < 0.02
    assert sizes["word first"] > 1.0


# ---- errors

@pytest.fixture(scope="module")
def intact(gpu_ctx):
    """(in, base, container) for a bf16 step with the blob CRC, chunks of 8192, ragged"""
    x, base = pair("bf16", 5 * 8192 + 77, 9, lr=1e-3)
    return x, base, expected(gpu_ctx, BYTE_FIRST, 20000, x, base, 2, 8192, CRC_BLOB)


def test_wrong_base_is_rejected_with_out_untouched(gpu_ctx, intact):
    x, base, buf = intact
    n = x.size
    for pos in (0, n // 2, n - 1):
        bad = base.copy()
        bad[pos] ^= 0x01 << (pos % 8)
        rc, _, out, b = decode(gpu_ctx, buf, 2, bad, n)
        assert rc == E_BASE and np.all(out == SENTINEL) and np.array_equal(b, bad), pos
        rc, _, out, b = decode(gpu_ctx, buf, 2, bad, n, in_place=True)
        assert rc == E_BASE and np.array_equal(out[:n], bad) and np.all(out[n:] == SENTINEL), pos
        rc, d_n, out, _ = decode(gpu_ctx, buf, 2, base, n, in_place=True)      # the same context, the right base
        assert rc == 0 and d_n == n and np.array_equal(out[:n], x), pos


def test_decode_rejects_leave_out_untouched(gpu_ctx, intact):
    x, base, buf = intact
    n = x.size
    cases = [(name, b, 2, n, None, E_STREAM) for name, b in gcp.broken_buffers(x, buf).items()]
    b = buf.copy()
    b[61] ^= 0x20                                                    # the base CRC, not resealed: meta_crc
    cases.append(("base crc", b, 2, n, None, E_STREAM))
    v7 = buf.copy()
    v7[4] = 7
    cp.set_u32(v7, 60, 0)
    cases += [("short by 16", buf, 2, n, buf.size - 16, E_STREAM), ("elem_bytes 4", buf, 4, n, None, E_STREAM),
              ("out_cap", buf, 2, n - 2, None, E_SPACE), ("version 7", cp.reseal(v7), 2, n, None, E_STREAM)]
    for name, b, w, cap, size, want in cases:
        for in_place in (False, True):
            rc, d_n, out, bb = decode(gpu_ctx, b, w, base, cap, size, in_place=in_place)
            assert rc == want, (name, in_place)
            if in_place:
                assert np.array_equal(bb, base[:bb.size]) and np.all(out[base.size:] == SENTINEL), name
            else:
                assert np.all(out == SENTINEL), name
            if want == E_SPACE:
                assert d_n == n, name
        rc, d_n, out, _ = decode(gpu_ctx, buf, 2, base, n)
        assert rc == 0 and d_n == n and np.array_equal(out[:n], x), name


def test_other_decodes_reject_version_8(gpu_ctx, intact):
    x, base, buf = intact
    c = gpu_ctx
    calls = {"v7": lambda *a: c.container_planes_decode_async(2, *a), "v1": c.container_decode_async,
             "v6": c.container_stored_decode_async, "v5": c.container_blocks_stored_decode_async,
             "any": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_any_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v2": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v3": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_coder_decode_async(c.h, *a[:4], a[4] or None), c.h),
             "v4": lambda *a: c.lib.check(c.lib.dll.rb200_container_blocks_alias_decode_async(c.h, *a[:4], a[4] or None), c.h)}
    for name, call in calls.items():
        rc, _, out = gcp.decode(c, buf, 2, x.size, decode_call=call)
        assert rc == E_STREAM and np.all(out == SENTINEL), name


def test_overlap_and_argument_errors_launch_nothing(gpu_ctx):
    torch = _torch()
    ch, w, n = 8192, 4, 4 * 10000
    d_in = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    d_base = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    cap = api.container_planes_bound(n, w, ch)
    d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    cands = (C.c_uint32 * 3)(*BYTE_FIRST)
    f = gpu_ctx.lib.dll.rb200_container_delta_encode_async
    ip, bp, op = d_in.data_ptr(), d_base.data_ptr(), d_out.data_ptr()
    cases = [(E_ARG, (1, ip, bp, n, op, cap)), (E_ARG, (3, ip, bp, n, op, cap)), (E_ARG, (16, ip, bp, n, op, cap)),
             (E_ARG, (w, ip, bp, n + 2, op, cap)), (E_ARG, (w, ip, bp, 0, op, cap)), (E_ARG, (w, ip, None, n, op, cap)),
             (E_ARG, (w, ip, bp + 8, n, op, cap)), (E_ARG, (w, ip, bp + 1, n, op, cap)), (E_ARG, (w, ip + 1, bp, n, op, cap)),
             (E_SPACE, (w, ip, bp, n, op, cap - 1))]
    before = gpu_ctx.launches
    for want, (ew, i, b, nn, o, oc) in cases:
        assert f(gpu_ctx.h, cands, 3, 20000, ew, i, b, nn, ch, 0, o, oc) == want, (ew, b, nn, oc)
    g = gpu_ctx.lib.dll.rb200_container_delta_decode_async
    d_dec = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
    dp = d_dec.data_ptr()
    for ew in (0, 1, 3, 16):
        assert g(gpu_ctx.h, ew, op, cap, bp, dp, n, None) == E_ARG
    assert g(gpu_ctx.h, w, op, cap, None, dp, n, None) == E_ARG
    assert g(gpu_ctx.h, w, op, cap, bp + 8, dp, n, None) == E_ARG
    assert g(gpu_ctx.h, w, op + 8, cap, bp, dp, n, None) == E_ARG
    for shift in (16, -16, 4096):                                      # partial overlaps of out and base
        assert g(gpu_ctx.h, w, op, cap, dp + shift, dp, n, None) == E_ARG, shift
    assert gpu_ctx.launches == before
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0


# ---- graphs

class Sync:
    """a sender and a receiver of one bf16 tensor on one context and stream: one captured graph encodes the new weights
    against the last sent version, applies the delta to the receiver's copy in place, and makes the new weights the
    last sent version"""

    def __init__(self, n, ch, seed):
        torch = _torch()
        self.n, self.ch, self.w = n, ch, 2
        self.stream = torch.cuda.Stream()
        self.ctx = rb.Context(0, stream=self.stream.cuda_stream)
        self.cap = api.container_planes_bound(n, 2, ch)
        first = gcp.elements("bf16", 2, n // 2, seed, 0.02)
        self.host = first
        self.cur = torch.from_numpy(first).cuda()
        self.prev = self.cur.clone()                                  # the last sent version
        self.recv = self.cur.clone()                                  # the receiver's copy
        self.buf = torch.zeros(self.cap + 16, dtype=torch.uint8, device="cuda")
        self.d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

    def step(self):
        self.ctx.container_delta_encode_async(BYTE_FIRST, 20000, 2, self.cur.data_ptr(), self.prev.data_ptr(), self.n, self.ch, CRC_BLOB,
                                              self.buf.data_ptr(), self.cap)
        self.ctx.container_delta_decode_async(2, self.buf.data_ptr(), self.cap, self.recv.data_ptr(), self.recv.data_ptr(), self.n,
                                              self.d_n.data_ptr())
        self.prev.copy_(self.cur)

    def capture(self):
        torch = _torch()
        with torch.cuda.stream(self.stream):
            self.step()                                               # grows the workspaces outside the capture
            assert self.ctx.lib.dll.rb200_sync(self.ctx.h) == 0
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.step()

    def advance(self, seed):
        """the next weights into cur; returns (new, last sent)"""
        torch = _torch()
        prev = self.host
        self.host = cd.step(prev, "bf16", 1e-4, seed)
        with torch.cuda.stream(self.stream):
            self.cur.copy_(torch.from_numpy(self.host).cuda(non_blocking=False))
        return self.host, prev

    def replay(self):
        torch = _torch()
        with torch.cuda.stream(self.stream):
            self.graph.replay()

    def check(self, new, prev, case):
        torch = _torch()
        assert self.ctx.lib.dll.rb200_sync(self.ctx.h) == 0, case
        got = self.buf.cpu().numpy()
        with torch.cuda.stream(self.stream):
            want = expected(self.ctx, BYTE_FIRST, 20000, new, prev, 2, self.ch, CRC_BLOB)   # the eager oracle, same context
        assert np.array_equal(got[:v8_size(got)], want), case
        assert int(self.d_n.item()) == self.n and np.array_equal(self.recv.cpu().numpy(), new), case
        assert np.array_equal(self.prev.cpu().numpy(), new), case

    def close(self):
        del self.graph
        self.ctx.close()


def test_one_graph_syncs_weights_in_place_over_steps():
    torch = _torch()
    s = Sync(2 * (40 * 8192 + 123), 8192, 1)
    s.capture()
    for i in range(4):
        new, prev = s.advance(200 + i)
        torch.cuda.synchronize()
        s.replay()
        s.check(new, prev, i)
    s.close()


def test_two_contexts_replay_their_graphs_at_once():
    torch = _torch()
    syncs = [Sync(2 * (20 * 8192 + 45 + 16 * k), 8192, 10 + k) for k in range(2)]
    for s in syncs:
        s.capture()
    for i in range(3):
        steps = [s.advance(300 + 10 * k + i) for k, s in enumerate(syncs)]
        torch.cuda.synchronize()
        for s in syncs:
            s.replay()                                                # both enqueued before either is waited for
        for k, (s, (new, prev)) in enumerate(zip(syncs, steps)):
            s.check(new, prev, (k, i))
    for s in syncs:
        s.close()


# ---- past 2^32

def _torch_zigzag16(x, b):
    torch = _torch()
    s = x.view(torch.int16) - b.view(torch.int16)                    # wraps mod 2^16
    return ((s << 1) ^ (s >> 15)).view(torch.uint8)


def _crc(t, n):
    out = (C.c_uint32 * 1)()
    ctx = rb.Context(0)
    ctx.lib.check(ctx.lib.dll.rb200_crc32(ctx.h, C.c_void_p(t.data_ptr()), n, 0, C.cast(out, api._u32p), api.MEM_DEVICE), ctx.h)
    ctx.close()
    return int(out[0])


def test_bf16_past_4_gib():
    """m = 2^32 - 2^20 bf16 elements, in uniform bytes: plane 0 ends past 2^32 bytes.  The delta encode equals the version 7 encode of d
    from byte 64 on, and its reserved word is the base's CRC; the in-place decode turns base into in (compared by
    CRC-32, so that in and the oracle's buffers are never resident at once)."""
    torch = _torch()
    ch, w = 8192, 2
    m = (1 << 32) - (1 << 20)
    n = w * m
    cap = api.container_planes_bound(n, w, ch)
    v6_cap = api.container_stored_bound(m, ch)
    scratch = -(-m // ch) * ((512 + 2 * ch + 15) // 16 * 16)
    # resident: in and base, then base, d and the oracle's container, each with a container of cap bytes; the encode's
    # split planes, staging and scratch (each workspace grows by an eighth)
    need = 2 * n + cap + 1.125 * (n + v6_cap + scratch) + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} free")
    gen = torch.Generator(device="cuda").manual_seed(7)
    d_in = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_base = torch.empty(n, dtype=torch.uint8, device="cuda")
    step = 1 << 26
    for a in range(0, m, step):
        b = min(m, a + step)
        d_base.view(torch.bfloat16)[a:b] = (torch.randn(b - a, device="cuda", generator=gen) * 0.02).to(torch.bfloat16)
    d_in.random_(0, 256, generator=gen)                                 # d near uniform: plane 0 is stored and crosses 2^32
    torch.cuda.empty_cache()
    d_buf = torch.full((cap,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx = rb.Context(0)
    ctx.container_delta_encode_async(BYTE_FIRST, 20000, w, d_in.data_ptr(), d_base.data_ptr(), n, ch, 0, d_buf.data_ptr(), cap)
    ctx.sync()
    ctx.close()
    head = d_buf[:64 + 16 * w].cpu().numpy()
    table = head[64:].view(np.uint64).reshape(w, 2)
    size = 64 + 16 * w + int(head[32:40].view(np.uint64)[0])
    assert int(table[0, 0] + table[0, 1]) > (1 << 32) and int(table[1, 0] + table[1, 1]) == size <= cap
    assert int(head[4]) == 8 and int(head[60:64].view(np.uint32)[0]) == _crc(d_base, n)
    d_v8 = d_buf[:size].clone()
    del d_buf
    crc_in = _crc(d_in, n)
    d = _torch_zigzag16(d_in, d_base)
    del d_in
    torch.cuda.empty_cache()
    d_v7 = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    ctx = rb.Context(0)
    ctx.container_planes_encode_async(BYTE_FIRST, 20000, w, d.data_ptr(), n, ch, 0, d_v7.data_ptr(), cap)
    ctx.sync()
    ctx.close()
    del d
    assert int(d_v7[32:40].cpu().numpy().view(np.uint64)[0]) == size - 64 - 16 * w
    assert torch.equal(d_v8[64:], d_v7[64:size])
    del d_v7
    torch.cuda.empty_cache()
    ctx = rb.Context(0)
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    ctx.container_delta_decode_async(w, d_v8.data_ptr(), size, d_base.data_ptr(), d_base.data_ptr(), n, d_n.data_ptr())
    ctx.sync()
    ctx.close()
    assert int(d_n.item()) == n and _crc(d_base, n) == crc_in
