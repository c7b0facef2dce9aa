"""rb200_container_blocks_stored_encode_async and rb200_container_blocks_stored_decode_async: version 5 per-block
containers, encoded and decoded on the GPU, with every block whose coded chunks take more than its stored size stored.

- The container equals the one packed from the oracle's streams for the chosen pair with the store rule applied in
  Python, over every data kind of test_blocks_coder_choice plus half-uniform mixes, the choice geometries, three
  candidate lists, tolerances 0 and 2 %, flags 0 and blob CRC.
- Where nothing is stored, everything after the header equals the auto encode's container, and the header differs only
  in its version and meta CRC.
- The decode round-trips, writes *d_n_symbols, refuses out_cap = n - 1, rejects each broken rule of a device container
  and a corrupt coded stream with out untouched, and a corrupt container ahead of a valid one does not disturb it;
  every other async decode rejects version 5.
- One CUDA graph of encode and decode follows data that changes which blocks are stored; argument errors launch
  nothing; launch counts are pinned; the output never exceeds rb200_container_blocks_stored_bound."""
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
import test_container_blocks_coder as cc  # noqa: E402
import test_container_blocks_stored as cbs  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_blocks_auto as gba  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
THREE = gba.THREE
LISTS = gba.LISTS
KINDS = bcc.KINDS + ["halfuniform"]


def _torch():
    import torch
    return torch


def block_data(kind, nb, bs, seed):
    """test_blocks_coder_choice's kinds, and uniform blocks between Zipf ones"""
    if kind != "halfuniform":
        return bcc.block_data(kind, nb, bs, seed)
    return np.concatenate([bcc.block_data("uniform" if b % 2 == 0 else "zipf", 1, bs, seed + b) for b in range(nb)])


def expected(oracle_lib, cands, tol, data, nb, bs, ch, flags):
    """(container, stored blocks): the oracle's streams for the chosen pair, the store rule applied in Python"""
    k = api.choose_blocks_coder(bcc.block_counts(data, nb, bs), bs, ch, cands, tol)[0]
    coder, sb = cands[k] >> 8, cands[k] & 0xFF
    f5, o5, b5, st = cbs.apply_store(*cbs.oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch), data, nb, bs, ch)
    return api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, flags), st


def encode(ctx, cands, tol, data, nb, bs, ch, flags, cap=None):
    """(sync code, whole output buffer on the host): the stored encode into a sentinel-filled buffer of cap + 64 bytes"""
    torch = _torch()
    cap = api.container_blocks_stored_bound(nb, bs, ch) if cap is None else cap
    d_in = gbc._dev(data)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_stored_encode_async(cands, tol, d_in.data_ptr(), nb, bs, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


@pytest.mark.parametrize("kind", KINDS)
def test_container_equals_the_oracle_packed_one(gpu_ctx, oracle_lib, kind):
    seen = set()
    for gi, (nb, bs, ch) in enumerate(gba.CHOICE_GEOMETRIES):
        data = block_data(kind, nb, bs, 10 * gi + KINDS.index(kind))
        for li, cands in enumerate(LISTS):
            for tol, flags in ((0, li & 1), (20000, CRC_BLOB)):
                want, st = expected(oracle_lib, cands, tol, data, nb, bs, ch, flags)
                rc, got = encode(gpu_ctx, cands, tol, data, nb, bs, ch, flags)
                case = (kind, nb, bs, ch, li, tol, flags, st)
                assert rc == 0, case
                assert np.array_equal(got[:want.size], want), case
                assert (got[want.size:] == SENTINEL).all(), case
                assert want.size <= api.container_blocks_stored_bound(nb, bs, ch), case
                seen.add(bool(st))
    if kind in ("uniform", "halfuniform"):
        assert True in seen


@pytest.mark.parametrize("kind", ["zipf", "skewed"])
def test_nothing_stored_is_the_auto_container(gpu_ctx, kind):
    torch = _torch()
    nb, bs, ch = 8, 65536, 8192
    data = block_data(kind, nb, bs, 4)
    for cands, tol, flags in ((THREE, 20000, 0), (THREE, 0, CRC_BLOB), ([CAND(RANS64, 11)], 0, 0), ([CAND(WORD, 12)], 0, CRC_BLOB)):
        rc, got = encode(gpu_ctx, cands, tol, data, nb, bs, ch, flags)
        assert rc == 0
        cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
        d_auto = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_blocks_model_encode_auto_async(cands, tol, gbc._dev(data).data_ptr(), nb, bs, ch, flags, d_auto.data_ptr(), cap)
        gpu_ctx.sync()
        auto = d_auto.cpu().numpy()
        size = gba._container_size(auto)
        assert struct.unpack_from("<H", got, 4)[0] == 5
        assert np.array_equal(got[6:44], auto[6:44]) and np.array_equal(got[48:size], auto[48:size]), (kind, cands)
        assert (got[:4] == auto[:4]).all()


# ---- decode

def _decode(ctx, buf, n, out_cap=None, call=None):
    """(sync code, *d_n_symbols, output buffer): an async decode into a sentinel-filled buffer"""
    torch = _torch()
    out_cap = n if out_cap is None else out_cap
    call = call or ctx.container_blocks_stored_decode_async
    d_buf = gbc._dev(buf)
    d_out = torch.full((max(n, out_cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    call(d_buf.data_ptr(), buf.size, d_out.data_ptr(), out_cap, d_n.data_ptr())
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out.cpu().numpy()


def _stored_container(oracle_lib, coder, sb, nb=4, bs=9000, ch=1000, flags=0, seed=7):
    data = cbs.mixed_data(nb, bs, seed)
    f5, o5, b5, st = cbs.apply_store(*cbs.oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch), data, nb, bs, ch)
    return api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, flags), data, f5, o5, st


PAIRS = [(WORD, 12), (BYTE, 14), (BYTE, 12), (BYTE, 9), (RANS64, 15), (ALIAS, 14), (ALIAS, 12), (ALIAS, 11)]


@pytest.mark.parametrize("coder,sb", PAIRS)
def test_round_trip_space_and_rejected_rules(gpu_ctx, oracle_lib, coder, sb):
    for geom in ((4, 9000, 1000), (3, 65536, 8192)):
        nb, bs, ch = geom
        for flags in (0, CRC_BLOB):
            buf, data, f5, o5, st = _stored_container(oracle_lib, coder, sb, nb, bs, ch, flags)
            assert st, (coder, sb)
            rc, n, out = _decode(gpu_ctx, buf, data.size)
            assert rc == 0 and n == data.size and np.array_equal(out[:data.size], data), (coder, sb, geom, flags)
            assert (out[data.size:] == SENTINEL).all()
            rc, n, out = _decode(gpu_ctx, buf, data.size, data.size - 1)
            assert rc == -3 and n == data.size and (out == SENTINEL).all()
    # each rule broken on its own (the host open agrees), then a corrupt coded stream
    nb, bs, ch = 4, 9000, 1000
    buf, data, f5, o5, st = _stored_container(oracle_lib, coder, sb, nb, bs, ch)
    per, dir_off = bs // ch, 64 + 512 * nb
    boff = (dir_off + 8 * o5.size + 15) & ~15
    coded = next(b for b in range(nb) if b not in st)
    stored = st[-1]

    def edit(pos, fmt, v):
        bad = buf.copy()
        struct.pack_into(fmt, bad, pos, v)
        return cc.reseal(bad)
    nz = int(np.flatnonzero(f5[coded])[0])
    bad_pad = buf.copy()
    bad_pad[boff + int(o5[stored * per + 1]) + ch + 2] = 7
    cases = {"coded row off by one": edit(64 + 512 * coded + 2 * nz, "<H", int(f5[coded][nz]) - 1),
             "stored row nonzero": edit(64 + 512 * stored + 10, "<H", 1),
             "stored step": edit(dir_off + 8 * (stored * per + 1), "<Q", int(o5[stored * per + 1]) + 16),
             "stored padding": bad_pad, "pair": edit(7, "<B", 16 if coder != WORD else 13), "version 4": edit(4, "<H", 4),
             "meta CRC": buf.copy()}
    cases["meta CRC"][70] ^= 1
    for name, bad in cases.items():
        with pytest.raises(rb.RansError):
            api.container_blocks_stored_open(bad)
        rc, n, out = _decode(gpu_ctx, bad, data.size)
        assert rc == -4 and (out == SENTINEL).all(), (coder, sb, name, rc)
    bad = buf.copy()
    c = coded * per + 3
    bad[boff + int(o5[c]) + 40] ^= 0x10                              # inside a coded stream: only the decoder sees it
    assert _decode(gpu_ctx, bad, data.size)[0] == -4, (coder, sb)


def test_other_decodes_reject_version_5(gpu_ctx, oracle_lib):
    for coder, sb in ((WORD, 12), (BYTE, 14), (ALIAS, 14)):
        buf, data, _, _, _ = _stored_container(oracle_lib, coder, sb)
        for call in (gpu_ctx.container_decode_async, gpu_ctx.container_blocks_decode_async, gpu_ctx.container_blocks_coder_decode_async,
                     gpu_ctx.container_blocks_alias_decode_async, gpu_ctx.container_blocks_any_decode_async):
            rc, n, out = _decode(gpu_ctx, buf, data.size, call=call)
            assert rc == -4 and n == -1 and (out == SENTINEL).all(), (coder, call.__name__)
        # and the stored decode rejects the same streams as version 2-4 containers
        for b in (gba._oracle_container(oracle_lib, coder, sb, data, 4, 9000, 1000, 0),):
            rc, n, out = _decode(gpu_ctx, b, data.size)
            assert rc == -4 and (out == SENTINEL).all()


def test_corrupt_container_then_a_valid_one(gpu_ctx, oracle_lib):
    torch = _torch()
    for coder, sb in ((WORD, 12), (BYTE, 12), (ALIAS, 14)):
        good, data, f5, o5, st = _stored_container(oracle_lib, coder, sb)
        nb, per = 4, 9
        boff = (64 + 512 * nb + 8 * o5.size + 15) & ~15
        coded = next(b for b in range(nb) if b not in st)
        bad = good.copy()
        bad[boff + int(o5[coded * per + 5]) + 40] ^= 0x10             # inside a coded stream: only the decoder sees it
        d_bad, d_good = gbc._dev(bad), gbc._dev(good)
        d_out0 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
        d_out1 = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_blocks_stored_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), data.size)
        gpu_ctx.container_blocks_stored_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), data.size)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4, coder
        assert np.array_equal(d_out1[:data.size].cpu().numpy(), data), coder
        assert (d_out1[data.size:].cpu().numpy() == SENTINEL).all()


# ---- graphs, launches, errors

def test_one_graph_follows_which_blocks_are_stored():
    torch = _torch()
    nb, bs, ch = 16, 65536, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_blocks_stored_bound(nb, bs, ch)
    d_in = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nb * bs + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_blocks_stored_encode_async(THREE, 20000, d_in.data_ptr(), nb, bs, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_blocks_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb * bs, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(block_data("zipf", nb, bs, 1)))
        round_trip()                                                 # grows the workspace outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        counts = set()
        for kind in ("halfuniform", "zipf", "uniform", "skewed", "halfuniform"):
            data = block_data(kind, nb, bs, 77 + len(counts))
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, kind
            head = d_buf[:64].cpu().numpy()
            assert struct.unpack_from("<H", head, 4)[0] == 5
            assert int(d_n.item()) == data.size and np.array_equal(d_out[:data.size].cpu().numpy(), data), kind
            rows = d_buf[64:64 + 512 * nb].cpu().numpy().view(np.uint16).reshape(nb, 256)
            counts.add(int((rows.sum(axis=1) == 0).sum()))
        assert {0, nb // 2, nb} <= counts, counts
        del g
    ctx.close()


def test_launch_counts(gpu_ctx):
    torch = _torch()
    nb, bs, ch = 8, 65536, 8192
    data = block_data("halfuniform", nb, bs, 1)
    cap = api.container_blocks_stored_bound(nb, bs, ch)
    d_in = gbc._dev(data)
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    # choice + word, byte 14 and alias 14 split encoders + store + scan + compaction + CRCs + header
    for cands, flags, want in ((THREE, 0, 9), (THREE, CRC_BLOB, 10), ([CAND(WORD, 12)], 0, 7), ([CAND(ALIAS, 12)], CRC_BLOB, 8)):
        before = gpu_ctx.launches
        gpu_ctx.container_blocks_stored_encode_async(cands, 20000, d_in.data_ptr(), nb, bs, ch, flags, d_buf.data_ptr(), cap)
        assert gpu_ctx.launches - before == want, (cands, flags)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
        before = gpu_ctx.launches
        gpu_ctx.container_blocks_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), data.size)
        assert gpu_ctx.launches - before == 13
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
        assert np.array_equal(d_out[:data.size].cpu().numpy(), data)


def test_argument_and_space_errors(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    nb, bs, ch = 4, 16384, 4096
    data = block_data("halfuniform", nb, bs, 2)
    bound = api.container_blocks_stored_bound(nb, bs, ch)
    d_in = gbc._dev(data)
    d_buf = torch.full((bound + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    i, o = d_in.data_ptr(), d_buf.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, n_blocks=nb, block_size=bs, chunk=ch, out=o, out_cap=bound):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_blocks_stored_encode_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size,
                                                              tol, inp, n_blocks, block_size, chunk, 0, out, out_cap)
    before = gpu_ctx.launches
    for bad in ([], [CAND(BYTE, 16)], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
        assert call(bad) == -1, bad
    assert call(THREE, tol=10 ** 6 + 1) == -1
    for kw in ({"ctx": None}, {"inp": None}, {"out": None}, {"out": o + 8}, {"n_blocks": 0}, {"chunk": 31}, {"chunk": 1000},
               {"block_size": 33 * 32, "chunk": 32}):
        assert call(THREE, **kw) == -1, kw
    boff = (64 + 512 * nb + 8 * (nb * bs // ch + 1) + 15) & ~15
    assert call(THREE, out_cap=boff - 1) == -3
    assert gpu_ctx.launches == before
    assert (d_buf.cpu().numpy() == SENTINEL).all()
    assert call(THREE, out_cap=boff + 64) == 0                       # the blob does not fit: -3 from sync, header unwritten
    assert lib.rb200_sync(gpu_ctx.h) == -3
    assert (d_buf[:64].cpu().numpy() == SENTINEL).all()
    d_buf.fill_(SENTINEL)
    for kind in ("uniform", "halfuniform", "const"):                 # at out_cap == bound: fits, nothing written past it
        d_in[:data.size].copy_(torch.from_numpy(block_data(kind, nb, bs, 3)))
        assert call(THREE, out_cap=bound) == 0 and lib.rb200_sync(gpu_ctx.h) == 0, kind
        got = d_buf.cpu().numpy()
        assert gba._container_size(got) <= bound and (got[bound:] == SENTINEL).all(), kind
    d_out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launches
    for args in ((None, o, bound, d_out.data_ptr(), 64, None), (gpu_ctx.h, o + 8, bound, d_out.data_ptr(), 64, None),
                 (gpu_ctx.h, o, bound, d_out.data_ptr() + 1, 64, None), (gpu_ctx.h, o, bound, d_out.data_ptr(), 64, d_out.data_ptr() + 4)):
        assert lib.rb200_container_blocks_stored_decode_async(*args) == -1
    assert gpu_ctx.launches == before


def test_uniform_container_is_within_the_aim(gpu_ctx):
    """uniform data: every block stored, so the container is its bound: models and directory on top of the input"""
    nb, bs, ch = 96, 65536, 8192
    data = block_data("uniform", nb, bs, 5)
    rc, got = encode(gpu_ctx, THREE, 20000, data, nb, bs, ch, 0)
    assert rc == 0
    size = gba._container_size(got)
    assert size == api.container_blocks_stored_bound(nb, bs, ch)
    assert size / data.size <= 1.009
