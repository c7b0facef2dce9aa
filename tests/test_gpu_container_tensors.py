"""rb200_container_tensors_encode_async / _decode_async: a list of same-width tensors as one version 9 container, on the
GPU, with the list in device memory read when the work runs.

- The oracle: the version 7 GPU encode of the concatenated bytes (concatenated with torch), its planes from
  container_planes_open, packed with container_tensors_pack, equals the version 9 container byte for byte.  w = 2, 4
  and 8; chunks of 32, 8192 and 2^24; the documented candidate lists; with and without the blob CRC; lists of one
  tensor, of many, with zero-length tensors, with every length residue mod 16 elements, and element-aligned views into
  one buffer that are not 16-byte aligned.  Nothing past the container is written.
- Round trips into separate outputs, with d_lengths; nothing past each output's length is written.
- Bad lists give RB200_E_ARG from rb200_sync with out bitwise unchanged; host argument errors launch nothing.
- Decode rejects leave every output untouched: a count mismatch, a capacity one element short, a total above n_max, a
  corrupt directory, table or plane, and versions 7, 8 and 9 given to each other's decoders.
- One captured graph of encode and decode replayed with the list rewritten between replays (other addresses, other
  lengths, another total), and two contexts replaying their own graphs at once.
- A bf16 list whose concatenated bytes cross 2^32.
- Sizes of a LoRA-like list (448 bf16 tensors of 128 KiB) against the sum of per-tensor version 7 containers."""
import os
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_container_planes as gcp  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = gcp.SENTINEL
THREE = gcp.THREE                                                     # the byte-plane list
BYTE_FIRST = [CAND(BYTE, 14), CAND(WORD, 12), CAND(ALIAS, 16)]       # the delta list
OTHER = [CAND(RANS64, 11), CAND(BYTE, 12), CAND(ALIAS, 9)]
E_ARG, E_SPACE, E_STREAM = -1, -3, -4
KIND = {2: "bf16", 4: "fp32", 8: "fp64"}


def _torch():
    import torch
    return torch


def round16(v):
    return (v + 15) & ~15


def refs(pairs):
    """the rb200_tensor_ref list of (ptr, bytes) pairs, in device memory"""
    torch = _torch()
    return torch.tensor([[p, b] for p, b in pairs] or [[0, 0]], dtype=torch.int64, device="cuda")


def list_counts(shape, ch):
    """element counts of the lists the suite covers"""
    rng = np.random.default_rng(len(shape) + ch)
    if shape == "one":
        return [5 * ch + 17]
    if shape == "many":
        return rng.integers(1, 3 * min(ch, 8192), 300).tolist()
    if shape == "zeros":
        return [0, 40, 0, 0, 16, 0, ch + 3, 0]
    if shape == "residues":
        return [16 * k + r for k, r in zip(rng.integers(0, 4, 48), list(range(16)) * 3)]
    raise ValueError(shape)


class DeviceList:
    """tensors of w-byte elements on the device.  views: element-aligned views into one buffer, the first w bytes past
    its 16-byte-aligned start, each next one right after the previous; otherwise separate allocations (16-byte
    aligned)."""

    def __init__(self, counts, w, seed, views=False, scale=0.02):
        torch = _torch()
        self.w = w
        self.host = [gcp.elements(KIND[w], w, c, seed + i, scale) if c else np.zeros(0, np.uint8) for i, c in enumerate(counts)]
        self.lengths = [h.size for h in self.host]
        self.n = sum(self.lengths)
        if views:
            self.flat = torch.full((self.n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
            self.tensors, at = [], w
            for h in self.host:
                self.tensors.append(self.flat[at:at + h.size])
                if h.size:
                    self.tensors[-1].copy_(torch.from_numpy(h))
                at += h.size
        else:
            self.tensors = [torch.from_numpy(h).cuda() if h.size else torch.empty(0, dtype=torch.uint8, device="cuda") for h in self.host]
        self.d_refs = refs([(t.data_ptr() if t.numel() else 0, t.numel()) for t in self.tensors])

    def concat(self):
        torch = _torch()
        return torch.cat([t for t in self.tensors] + [torch.zeros(16, dtype=torch.uint8, device="cuda")])


def encode9(ctx, cands, tol, lst, n_max, ch, flags, cap=None):
    """(sync code, whole sentinel-filled output on the host, cap)"""
    torch = _torch()
    cap = api.container_tensors_bound(n_max, len(lst.lengths), lst.w, ch) if cap is None else cap
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_tensors_encode_async(cands, tol, lst.w, lst.d_refs.data_ptr(), len(lst.lengths), n_max, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy(), cap


def v9_size(buf):
    w, t = int(buf[52:56].view(np.uint32)[0]), int(buf[56:60].view(np.uint32)[0])
    return 64 + 16 * w + round16(8 * t) + int(buf[32:40].view(np.uint64)[0])


def oracle9(ctx, cands, tol, lst, ch, flags):
    """container_tensors_pack of the lengths and the planes of the version 7 GPU encode of the concatenated bytes"""
    v7 = gcp_fixed7(ctx, cands, tol, lst.concat(), lst.n, lst.w, ch, flags)
    _, planes = api.container_planes_open(v7)
    return api.container_tensors_pack(lst.lengths, planes)


def gcp_fixed7(ctx, cands, tol, d_in, n, w, ch, flags):
    torch = _torch()
    cap = api.container_planes_bound(n, w, ch)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_planes_encode_async(cands, tol, w, d_in.data_ptr(), n, ch, flags, d_out.data_ptr(), cap)
    assert ctx.lib.dll.rb200_sync(ctx.h) == 0
    buf = d_out.cpu().numpy()
    return buf[:gcp.v7_size(buf)]


def outputs(lengths, slack=16):
    """sentinel-filled outputs with `slack` bytes past each length, and their refs (capacity = length)"""
    torch = _torch()
    outs = [torch.full((b + slack,), SENTINEL, dtype=torch.uint8, device="cuda") for b in lengths]
    return outs, refs([(o.data_ptr(), b) for o, b in zip(outs, lengths)])


def decode9(ctx, w, buf, size, d_refs, count, n_max, d_len=None):
    ctx.container_tensors_decode_async(w, buf.data_ptr(), size, d_refs.data_ptr(), count, n_max, d_len.data_ptr() if d_len is not None else 0)
    return ctx.lib.dll.rb200_sync(ctx.h)


def check_round_trip(ctx, lst, buf_host, n_max):
    torch = _torch()
    d_buf = torch.from_numpy(buf_host).cuda()
    outs, d_refs = outputs(lst.lengths)
    d_len = torch.full((len(lst.lengths),), -1, dtype=torch.int64, device="cuda")
    assert decode9(ctx, lst.w, d_buf, buf_host.size, d_refs, len(lst.lengths), n_max, d_len) == 0
    assert d_len.cpu().numpy().astype(np.uint64).tolist() == lst.lengths
    for o, h in zip(outs, lst.host):
        got = o.cpu().numpy()
        assert np.array_equal(got[:h.size], h) and (got[h.size:] == SENTINEL).all()


CASES = ([(w, shape, 8192, THREE, CRC_BLOB, False) for w in (2, 4, 8) for shape in ("one", "many", "zeros", "residues")]
         + [(w, "residues", 8192, THREE, 0, True) for w in (2, 4, 8)]
         + [(2, "many", 32, BYTE_FIRST, 0, False), (4, "zeros", 32, OTHER, CRC_BLOB, True), (8, "residues", 32, THREE, 0, False),
            (2, "one", 1 << 24, BYTE_FIRST, CRC_BLOB, False), (4, "many", 1 << 24, THREE, 0, True)])


@pytest.mark.parametrize("w,shape,ch,cands,flags,views", CASES)
def test_equals_the_oracle_and_round_trips(gpu_ctx, w, shape, ch, cands, flags, views):
    lst = DeviceList(list_counts(shape, ch), w, 7, views=views)
    if views:
        assert any(t.data_ptr() % 16 for t in lst.tensors if t.numel())
    want = oracle9(gpu_ctx, cands, 20000, lst, ch, flags)
    n_max = lst.n + 5 * w                                             # a bound above the total
    rc, got, cap = encode9(gpu_ctx, cands, 20000, lst, n_max, ch, flags)
    assert rc == 0
    assert np.array_equal(got[:want.size], want) and (got[want.size:] == SENTINEL).all()
    assert v9_size(got) == want.size
    check_round_trip(gpu_ctx, lst, want, lst.n)


@pytest.mark.parametrize("w", [2, 4, 8])
def test_bad_lists_write_nothing(gpu_ctx, w):
    torch = _torch()
    ch = 8192
    lst = DeviceList([100, 37, 300], w, 3)
    n_max = lst.n + 16 * w
    good = [(t.data_ptr(), t.numel()) for t in lst.tensors]
    bads = {
        "length not a multiple of w": [good[0], (good[1][0], good[1][1] - 1), good[2]],
        "misaligned ptr": [good[0], (good[1][0] + 1, good[1][1] - w), good[2]],
        "total 0": [(good[0][0], 0), (0, 0), (good[2][0], 0)],
        "total above n_max": [good[0], good[1], (good[2][0], good[2][1] + 16 * w + w)],
        "null ptr": [good[0], (0, good[1][1]), good[2]],
    }
    assert encode9(gpu_ctx, THREE, 20000, lst, n_max, ch, 0)[0] == 0   # the good list
    for name, pairs in bads.items():
        lst.d_refs = refs(pairs)
        rc, got, _ = encode9(gpu_ctx, THREE, 20000, lst, n_max, ch, CRC_BLOB)
        assert rc == E_ARG, name
        assert (got == SENTINEL).all(), name
    lst.d_refs = refs(good)                                           # the context is fine afterwards
    rc, got, _ = encode9(gpu_ctx, THREE, 20000, lst, n_max, ch, 0)
    assert rc == 0 and np.array_equal(got[:v9_size(got)], oracle9(gpu_ctx, THREE, 20000, lst, ch, 0))


def test_host_argument_errors_launch_nothing(gpu_ctx):
    torch = _torch()
    ctx, lib = gpu_ctx, gpu_ctx.lib
    lst = DeviceList([64, 64], 2, 1)
    n_max, ch = lst.n, 8192
    cap = api.container_tensors_bound(n_max, 2, 2, ch)
    d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    cands = np.asarray(THREE, np.uint32)
    r = lst.d_refs.data_ptr()

    def enc(w=2, refs_=r, count=2, nm=n_max, c=ch, out=d_out.data_ptr(), oc=cap, cl=cands):
        return lib.dll.rb200_container_tensors_encode_async(ctx.h, cl.ctypes.data_as(api._u32p), cl.size, 20000, w, refs_, count, nm, c, 0,
                                                            out, oc)

    launches = ctx.launches
    for args, code in (({"w": 3}, E_ARG), ({"refs_": None}, E_ARG), ({"refs_": r + 8}, E_ARG), ({"count": 0}, E_ARG),
                       ({"count": (1 << 20) + 1}, E_ARG), ({"nm": 0}, E_ARG), ({"nm": n_max + 1}, E_ARG), ({"nm": 1 << 34}, E_ARG),
                       ({"c": 16}, E_ARG), ({"out": d_out.data_ptr() + 8}, E_ARG), ({"cl": np.asarray([CAND(WORD, 11)], np.uint32)}, E_ARG),
                       ({"oc": cap - 1}, E_SPACE), ({"count": 3, "oc": cap}, E_SPACE)):
        assert enc(**args) == code, args
    assert ctx.launches == launches
    assert enc() == 0 and lib.dll.rb200_sync(ctx.h) == 0
    buf = d_out
    d_len = torch.zeros(4, dtype=torch.int64, device="cuda")

    def dec(w=2, b=buf.data_ptr(), size=cap, refs_=r, count=2, nm=n_max, ln=None):
        return lib.dll.rb200_container_tensors_decode_async(ctx.h, w, b, size, refs_, count, nm, ln)

    launches = ctx.launches
    for args in ({"w": 3}, {"b": None}, {"b": buf.data_ptr() + 8}, {"refs_": None}, {"refs_": r + 8}, {"count": 0},
                 {"count": (1 << 20) + 1}, {"nm": 0}, {"ln": d_len.data_ptr() + 4}):
        assert dec(**args) == E_ARG, args
    assert ctx.launches == launches


@pytest.fixture(scope="module")
def made(gpu_ctx):
    """(list, its version 9 container on the host) and the same tensors' version 7 and 8 containers"""
    lst = DeviceList([3 * 32 + 5, 0, 17, 40, 200], 4, 21)
    rc, got, _ = encode9(gpu_ctx, THREE, 20000, lst, lst.n, 32, CRC_BLOB)
    assert rc == 0
    v9 = got[:v9_size(got)].copy()
    v7 = gcp_fixed7(gpu_ctx, THREE, 20000, lst.concat(), lst.n, 4, 32, 0)
    _, planes = api.container_planes_open(v7)
    v8 = api.container_delta_pack(planes, 99)
    return lst, v9, v7, v8


def test_decode_rejects_leave_outputs_untouched(gpu_ctx, made):
    torch = _torch()
    lst, v9, v7, v8 = made
    t = len(lst.lengths)
    d_dir = 64 + 16 * 4
    d_plane = d_dir + round16(8 * t)

    def attempt(buf, lengths=lst.lengths, count=t, n_max=lst.n, w=4):
        outs, d_refs = outputs(lengths)
        d_len = torch.full((max(count, 1),), -1, dtype=torch.int64, device="cuda")
        rc = decode9(gpu_ctx, w, torch.from_numpy(buf).cuda(), buf.size, d_refs, count, n_max, d_len)
        assert all((o.cpu().numpy() == SENTINEL).all() for o in outs)
        return rc, d_len.cpu().numpy()

    def flip(off, bit=1):
        b = v9.copy()
        b[off] ^= bit
        return b

    short = list(lst.lengths)
    short[4] -= 4
    for name, args, code in (
            ("count one short", dict(count=t - 1, lengths=lst.lengths[:-1]), E_STREAM),
            ("count one over", dict(count=t + 1, lengths=lst.lengths + [64]), E_STREAM),
            ("elem_bytes", dict(w=2), E_STREAM),
            ("capacity one element short", dict(lengths=short), E_SPACE),
            ("total above n_max", dict(n_max=lst.n - 4), E_SPACE)):
        rc, d_len = attempt(v9, **args)
        assert rc == code, name
        if code == E_SPACE and name.startswith("capacity"):
            assert d_len.astype(np.uint64).tolist() == lst.lengths     # the directory passed
    for name, buf in (("directory", flip(d_dir + 8 * 2)), ("directory padding", flip(d_dir + 8 * t)), ("table", flip(64 + 8)),
                      ("plane header", flip(d_plane + 16)), ("plane blob", flip(v9.size - 40, 0x10)), ("reserved", flip(60)),
                      ("truncated", v9[:-16].copy()), ("version 7", v7), ("version 8", v8)):
        assert attempt(buf)[0] == E_STREAM, name
    # and the other decoders refuse version 9
    d_v9 = torch.from_numpy(v9).cuda()
    out = torch.full((lst.n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_planes_decode_async(4, d_v9.data_ptr(), v9.size, out.data_ptr(), lst.n)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == E_STREAM
    base = torch.zeros(lst.n + 16, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_delta_decode_async(4, d_v9.data_ptr(), v9.size, base.data_ptr(), out.data_ptr(), lst.n)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == E_STREAM
    assert (out.cpu().numpy() == SENTINEL).all()


def test_intact_decode_after_rejects(gpu_ctx, made):
    lst, v9, _, _ = made
    check_round_trip(gpu_ctx, lst, v9, lst.n)


# ---- graphs

def _graph_side(torch, stream, ctx, w, ch, count, n_max):
    cap = api.container_tensors_bound(n_max, count, w, ch)
    side = {
        "cap": cap,
        "d_refs": torch.zeros((count, 2), dtype=torch.int64, device="cuda"),
        "d_orefs": torch.zeros((count, 2), dtype=torch.int64, device="cuda"),
        "d_buf": torch.zeros(cap + 64, dtype=torch.uint8, device="cuda"),
        "d_len": torch.zeros(count, dtype=torch.int64, device="cuda"),
    }

    def round_trip():
        ctx.container_tensors_encode_async(THREE, 20000, w, side["d_refs"].data_ptr(), count, n_max, ch, CRC_BLOB, side["d_buf"].data_ptr(), cap)
        ctx.container_tensors_decode_async(w, side["d_buf"].data_ptr(), cap, side["d_orefs"].data_ptr(), count, n_max, side["d_len"].data_ptr())

    side["round_trip"] = round_trip
    return side


def _load(side, lst, outs):
    side["d_refs"].copy_(lst.d_refs)
    side["d_orefs"].copy_(refs([(o.data_ptr(), b) for o, b in zip(outs, lst.lengths)]))


def test_one_graph_with_the_list_rewritten(gpu_ctx):
    torch = _torch()
    w, ch, count = 2, 8192, 24
    n_max = 3 * (1 << 20)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    side = _graph_side(torch, stream, ctx, w, ch, count, n_max)
    rng = np.random.default_rng(5)
    lists = [DeviceList(rng.integers(0, 60000, count).tolist(), w, 100 + k, views=k % 2 == 1, scale=[0.02, 3.0][k % 2]) for k in range(4)]
    lists.append(DeviceList([0] * (count - 1) + [n_max // w], w, 200))     # the whole bound in the last tensor
    with torch.cuda.stream(stream):
        outs = [torch.full((b + 16,), SENTINEL, dtype=torch.uint8, device="cuda") for b in lists[0].lengths]
        _load(side, lists[0], outs)
        side["round_trip"]()
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            side["round_trip"]()
        totals = set()
        for lst in lists:
            outs = [torch.full((b + 16,), SENTINEL, dtype=torch.uint8, device="cuda") for b in lst.lengths]
            _load(side, lst, outs)
            side["d_buf"].fill_(SENTINEL)
            launches = ctx.launches
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            assert ctx.launches == launches
            got = side["d_buf"].cpu().numpy()
            want = oracle9(ctx, THREE, 20000, lst, ch, CRC_BLOB)
            assert np.array_equal(got[:want.size], want) and (got[want.size:] == SENTINEL).all()
            assert side["d_len"].cpu().numpy().astype(np.uint64).tolist() == lst.lengths
            for o, h in zip(outs, lst.host):
                o = o.cpu().numpy()
                assert np.array_equal(o[:h.size], h) and (o[h.size:] == SENTINEL).all()
            totals.add(lst.n)
        assert len(totals) == len(lists)
        del g
    ctx.close()


def test_two_contexts_replay_their_own_graphs():
    torch = _torch()
    w, ch, count = 4, 8192, 40
    n_max = 1 << 21
    sides = []
    for k in range(2):
        stream = torch.cuda.Stream()
        ctx = rb.Context(0, stream=stream.cuda_stream)
        side = _graph_side(torch, stream, ctx, w, ch, count, n_max)
        lst = DeviceList(np.random.default_rng(k).integers(0, 10000, count).tolist(), w, 300 + k)
        outs = [torch.full((b + 16,), SENTINEL, dtype=torch.uint8, device="cuda") for b in lst.lengths]
        with torch.cuda.stream(stream):
            _load(side, lst, outs)
            side["round_trip"]()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                side["round_trip"]()
        sides.append([stream, ctx, side, g, lst, outs])
    torch.cuda.synchronize()
    for rnd in range(3):
        for k, s in enumerate(sides):
            stream, ctx, side, g, _, _ = s
            lst = DeviceList(np.random.default_rng(10 * rnd + k).integers(0, 12000, count).tolist(), w, 400 + 10 * rnd + k)
            outs = [torch.full((b + 16,), SENTINEL, dtype=torch.uint8, device="cuda") for b in lst.lengths]
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                _load(side, lst, outs)
                g.replay()                                            # no synchronisation between the two sides
            s[4], s[5] = lst, outs
        for stream, ctx, side, g, lst, outs in sides:
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            for o, h in zip(outs, lst.host):
                o = o.cpu().numpy()
                assert np.array_equal(o[:h.size], h) and (o[h.size:] == SENTINEL).all()
            got = side["d_buf"].cpu().numpy()
            with torch.cuda.stream(stream):
                want = oracle9(ctx, THREE, 20000, lst, ch, CRC_BLOB)
            assert np.array_equal(got[:want.size], want)
    for stream, ctx, side, g, lst, outs in sides:
        del g
        ctx.close()


# ---- past 2^32

def test_bf16_list_past_4_gib(gpu_ctx):
    """three bf16 tensors of 2^32 + 2^21 + 6 bytes in all: the concatenation crosses 2^32 bytes, and the second tensor
    straddles it.  The planes equal the version 7 encode's of the concatenated bytes, compared on the device, and the
    round trip gives every tensor back."""
    torch = _torch()
    ch, w = 8192, 2
    lengths = [(1 << 31) + 2, (1 << 31) + (1 << 20), (1 << 20) + 4]
    n = sum(lengths)
    gen = torch.Generator(device="cuda").manual_seed(3)
    tensors = [(torch.randn(b // 2, device="cuda", generator=gen) * 0.02).to(torch.bfloat16).view(torch.uint8) for b in lengths]
    d_refs = refs([(t.data_ptr(), t.numel()) for t in tensors])
    cap = api.container_tensors_bound(n, 3, w, ch)
    d_buf = torch.empty(cap, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_tensors_encode_async(THREE, 20000, w, d_refs.data_ptr(), 3, n, ch, 0, d_buf.data_ptr(), cap)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    head = d_buf[:4096].cpu().numpy()
    size9 = v9_size(head)
    cat = torch.cat(tensors)
    cap7 = api.container_planes_bound(n, w, ch)
    d7 = torch.empty(cap7, dtype=torch.uint8, device="cuda")
    gpu_ctx.container_planes_encode_async(THREE, 20000, w, cat.data_ptr(), n, ch, 0, d7.data_ptr(), cap7)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    del cat
    head7 = d7[:4096].cpu().numpy()
    size7 = gcp.v7_size(head7)
    start = 64 + 16 * w + 32                                          # three lengths and their padding
    assert size9 - start == size7 - 64 - 16 * w
    assert torch.equal(d_buf[start:size9], d7[64 + 16 * w:size7])
    assert head[64 + 16 * w:start].view(np.uint64).tolist() == lengths + [0]
    del d7
    outs = [torch.empty_like(t) for t in tensors]
    o_refs = refs([(o.data_ptr(), o.numel()) for o in outs])
    gpu_ctx.container_tensors_decode_async(w, d_buf.data_ptr(), size9, o_refs.data_ptr(), 3, n, 0)
    assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
    assert all(torch.equal(o, t) for o, t in zip(outs, tensors))


# ---- sizes

def test_lora_like_list_sizes(gpu_ctx):
    """448 bf16 tensors of 128 KiB: one version 9 container against 448 version 7 containers"""
    w, ch = 2, 8192
    lst = DeviceList([1 << 16] * 448, w, 9, scale=0.01)
    rc, got, _ = encode9(gpu_ctx, THREE, 20000, lst, lst.n, ch, 0)
    assert rc == 0
    size9 = v9_size(got)
    per = sum(gcp_fixed7(gpu_ctx, THREE, 20000, t, t.numel(), w, ch, 0).size for t in lst.tensors)
    print(f"\nLoRA-like 448 x 128 KiB bf16: version 9 {size9} B ({size9 / lst.n:.4f} B/B), 448 version 7 containers {per} B "
          f"({per / lst.n:.4f} B/B)")
    assert size9 < per
