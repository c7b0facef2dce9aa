"""rb200_container_stored_encode_async and rb200_container_stored_decode_async: version 6 single-model containers, encoded
and decoded on the GPU, with every chunk whose stream is longer than its symbols stored.

- The container equals the one packed from the oracle's chunked streams for the pair choose_coder picks, with the store
  rule applied in Python: every conftest data kind and a mix of uniform and Zipf runs whose boundaries fall inside
  chunks; whole, +1, +15, +17 and chunk_syms - 1 past a multiple; chunks of 32, 33, 4096 and 8192; three candidate
  lists, tolerances 0 and 2 %, flags 0 and blob CRC.  Constant data with the word coder chosen stores every chunk and
  is exactly the bound.
- Where nothing is stored, model, directory and blob equal the auto encode's container.
- The decode round-trips and writes *d_n_symbols, refuses out_cap = n - 1, rejects each broken rule of a device
  container and a corrupt coded stream with out untouched; a corrupt container ahead of a valid one does not disturb
  it; the v1 async, any and version 5 decodes reject version 6.
- One CUDA graph of encode and decode follows data that changes which chunks are stored; argument errors launch
  nothing; launch counts are pinned; the output never exceeds rb200_container_stored_bound."""
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
from conftest import _gen  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
THREE = [CAND(WORD, 12), CAND(ALIAS, 16), CAND(BYTE, 14)]
LISTS = [THREE, [CAND(RANS64, 11), CAND(BYTE, 12), CAND(ALIAS, 9)], [CAND(BYTE, 16), CAND(WORD, 12)]]
KINDS = ["uniform", "zipf", "text", "const", "two", "skew", "mixed"]


def _torch():
    import torch
    return torch


def data_of(kind, n, ch, seed):
    if kind == "mixed":
        return cs.mixed_data(n, max(ch, 4096), seed)
    return _gen(kind, n, seed)


def expected(oracle_lib, cands, tol, data, ch, flags):
    """(container, stored chunks, pair): the oracle's streams for the chosen pair, the store rule applied in Python"""
    k = api.choose_coder(np.bincount(data, minlength=256), data.size, ch, cands, tol)[0]
    coder, sb = cands[k] >> 8, cands[k] & 0xFF
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, ch)
    bits, o6, b6, st = cs.apply_store(data, ch, offs, blob)
    return api.container_stored_pack(coder, sb, ch, data.size, freqs, bits, o6, b6, flags), st, (coder, sb)


def encode(ctx, cands, tol, data, ch, flags, cap=None):
    """(sync code, whole output buffer on the host): the stored encode into a sentinel-filled buffer of cap + 64 bytes"""
    torch = _torch()
    cap = api.container_stored_bound(data.size, ch) if cap is None else cap
    d_in = gbc._dev(data)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_stored_encode_async(cands, tol, d_in.data_ptr(), data.size, ch, flags, d_out.data_ptr(), cap)
    return ctx.lib.dll.rb200_sync(ctx.h), d_out.cpu().numpy()


def size_of(buf):
    n_chunks = int(buf[24:32].view(np.uint64)[0])
    return cs.blob_offset(n_chunks) + int(buf[32:40].view(np.uint64)[0])


@pytest.mark.parametrize("ch", [32, 33, 4096, 8192])
@pytest.mark.parametrize("kind", KINDS)
def test_container_equals_the_oracle_packed_one(gpu_ctx, oracle_lib, kind, ch):
    base = 6 * ch if ch > 64 else 300 * ch
    stored_any = False
    for li, extra in enumerate((0, 1, 15, 17, ch - 1)):
        n = base + extra
        data = data_of(kind, n, ch, 3 * li + KINDS.index(kind))
        cands = LISTS[li % len(LISTS)]
        for tol, flags in ((0, li & 1), (20000, CRC_BLOB)):
            want, st, pair = expected(oracle_lib, cands, tol, data, ch, flags)
            rc, got = encode(gpu_ctx, cands, tol, data, ch, flags)
            case = (kind, ch, n, li, tol, flags, pair, len(st))
            assert rc == 0, case
            assert np.array_equal(got[:want.size], want), case
            assert (got[want.size:] == SENTINEL).all(), case
            assert want.size <= api.container_stored_bound(n, ch), case
            stored_any |= bool(st)
    if kind in ("uniform", "mixed") or ch <= 33:
        assert stored_any


@pytest.mark.parametrize("n", [8192 * 20, 8192 * 20 + 17])
def test_constant_data_with_the_word_coder_is_all_stored(gpu_ctx, oracle_lib, n):
    data = _gen("const", n, 0)
    want, st, pair = expected(oracle_lib, THREE, 0, data, 8192, 0)
    assert pair == (WORD, 12) and len(st) == -(-n // 8192)
    rc, got = encode(gpu_ctx, THREE, 0, data, 8192, 0)
    assert rc == 0 and np.array_equal(got[:want.size], want)
    assert size_of(got) == api.container_stored_bound(n, 8192)


@pytest.mark.parametrize("kind", ["zipf", "skew", "text"])
def test_nothing_stored_is_the_auto_container(gpu_ctx, kind):
    torch = _torch()
    ch = 8192
    n = ch * 24 + 1000
    data = _gen(kind, n, 4)
    for cands, tol, flags in ((THREE, 20000, 0), (THREE, 0, CRC_BLOB), ([CAND(RANS64, 11)], 0, 0), ([CAND(ALIAS, 14)], 0, CRC_BLOB)):
        rc, got = encode(gpu_ctx, cands, tol, data, ch, flags)
        assert rc == 0
        n_chunks = -(-n // ch)
        boff = cs.blob_offset(n_chunks)
        assert not got[cs._bitmap_at(n_chunks):boff].any(), (kind, cands)
        cap = api.container_stored_bound(n, ch) * 2 + 4096
        d_auto = torch.full((cap,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_model_encode_auto_async(cands, tol, gbc._dev(data).data_ptr(), n, ch, flags, d_auto.data_ptr(), cap)
        gpu_ctx.sync()
        auto = d_auto.cpu().numpy()
        a_boff = (1088 + 8 * (n_chunks + 1) + 15) & ~15
        blob_bytes = int(auto[32:40].view(np.uint64)[0])
        assert struct.unpack_from("<H", got, 4)[0] == 6
        assert np.array_equal(got[6:44], auto[6:44]), (kind, cands)      # coder, geometry, blob size, flags
        assert np.array_equal(got[64:1088 + 8 * (n_chunks + 1)], auto[64:1088 + 8 * (n_chunks + 1)]), (kind, cands)
        assert np.array_equal(got[boff:boff + blob_bytes], auto[a_boff:a_boff + blob_bytes]), (kind, cands)


# ---- decode

def _decode(ctx, buf, n, out_cap=None, call=None):
    """(sync code, *d_n_symbols, output buffer): an async decode into a sentinel-filled buffer"""
    torch = _torch()
    out_cap = n if out_cap is None else out_cap
    call = call or ctx.container_stored_decode_async
    d_buf = gbc._dev(buf)
    d_out = torch.full((max(n, out_cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    call(d_buf.data_ptr(), buf.size, d_out.data_ptr(), out_cap, d_n.data_ptr())
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out.cpu().numpy()


def _stored_container(oracle_lib, coder, sb, n, ch, flags=0, seed=7):
    """a container of mixed data with the store rule's chunks and the last one stored"""
    data = cs.mixed_data(n, max(ch, 1024), seed)
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, ch)
    which = sorted(set(cs.store_rule(offs, blob, ch, n)) | {offs.size - 2})
    bits, o6, b6, st = cs.apply_store(data, ch, offs, blob, which)
    return api.container_stored_pack(coder, sb, ch, n, freqs, bits, o6, b6, flags), data, freqs, bits, o6, st


PAIRS = [(WORD, 12), (ALIAS, 16), (ALIAS, 14), (ALIAS, 12), (ALIAS, 11), (BYTE, 16), (BYTE, 14), (BYTE, 12), (BYTE, 9), (RANS64, 15)]


@pytest.mark.parametrize("coder,sb", PAIRS)
def test_round_trip_space_and_rejected_rules(gpu_ctx, oracle_lib, coder, sb):
    for n, ch in ((1024 * 40 + 17, 1024), (8192 * 9 + 8191, 8192), (33 * 200 + 5, 33)):
        for flags in (0, CRC_BLOB):
            buf, data, freqs, bits, o6, st = _stored_container(oracle_lib, coder, sb, n, ch, flags)
            assert st, (coder, sb, ch)
            rc, got_n, out = _decode(gpu_ctx, buf, n)
            assert rc == 0 and got_n == n and np.array_equal(out[:n], data), (coder, sb, ch, flags)
            assert (out[n:] == SENTINEL).all()
            rc, got_n, out = _decode(gpu_ctx, buf, n, n - 1)
            assert rc == -3 and got_n == n and (out == SENTINEL).all()
    # each rule broken on its own (the host open agrees), then a corrupt coded stream
    n, ch = 1024 * 40 + 17, 1024
    buf, data, freqs, bits, o6, st = _stored_container(oracle_lib, coder, sb, n, ch, CRC_BLOB)
    n_chunks = o6.size - 1
    bm, boff = cs._bitmap_at(n_chunks), cs.blob_offset(n_chunks)
    coded = next(c for c in range(n_chunks) if c not in st)
    last = n_chunks - 1

    def edit(pos, fmt, v):
        bad = buf.copy()
        struct.pack_into(fmt, bad, pos, v)
        return cs.reseal(bad)
    word = lambda c: int(bits[c // 32]) if c // 32 < bits.size else 0        # noqa: E731
    cases = {"bit past n_chunks": edit(bm + 4 * (n_chunks // 32), "<I", word(n_chunks) | 1 << (n_chunks % 32)),
             "bitmap padding": edit(bm + 12, "<I", 1),
             "coded chunk marked stored": edit(bm + 4 * (coded // 32), "<I", word(coded) | 1 << (coded % 32)),
             "stored step": edit(1088 + 8 * last, "<Q", int(o6[last]) - 16),
             "stored padding": edit(boff + int(o6[last]) + (n % ch) + 1, "<B", 3),
             "block_size": edit(52, "<I", 1), "n_blocks": edit(56, "<I", 1), "reserved": edit(60, "<I", 1),
             "model": edit(64, "<I", int(freqs[0]) + 1), "version 1": edit(4, "<H", 1), "version 5": edit(4, "<H", 5)}
    cases["meta CRC"] = buf.copy()
    cases["meta CRC"][70] ^= 1
    cases["blob CRC"] = buf.copy()
    cases["blob CRC"][-1] ^= 1
    for name, bad in cases.items():
        with pytest.raises(rb.RansError):
            api.container_stored_open(bad)
        rc, got_n, out = _decode(gpu_ctx, bad, n)
        assert rc == -4 and (out == SENTINEL).all(), (coder, sb, name, rc)
    bad = buf.copy()
    bad[boff + int(o6[coded]):boff + int(o6[coded]) + 128] ^= 0x10   # every lane's state of a coded stream: only the decoder sees it
    bad = cs.reseal(bad)
    api.container_stored_open(bad)
    assert _decode(gpu_ctx, bad, n)[0] == -4, (coder, sb)


def test_other_decodes_reject_version_6(gpu_ctx, oracle_lib):
    for coder, sb in ((WORD, 12), (BYTE, 14), (ALIAS, 14)):
        n = 4096 * 10 + 3
        buf, data, _, _, _, _ = _stored_container(oracle_lib, coder, sb, n, 4096)
        for call in (gpu_ctx.container_decode_async, gpu_ctx.container_blocks_any_decode_async, gpu_ctx.container_blocks_stored_decode_async):
            rc, got_n, out = _decode(gpu_ctx, buf, n, call=call)
            assert rc == -4 and got_n == -1 and (out == SENTINEL).all(), (coder, call.__name__)
        # and the version 6 decode rejects the version 1 container of the same streams
        freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, 4096)
        rc, got_n, out = _decode(gpu_ctx, api.container_pack(coder, sb, 4096, n, freqs, offs, blob), n)
        assert rc == -4 and got_n == -1 and (out == SENTINEL).all()


def test_corrupt_container_then_a_valid_one(gpu_ctx, oracle_lib):
    torch = _torch()
    for coder, sb in ((WORD, 12), (BYTE, 12), (ALIAS, 14), (RANS64, 12)):
        n = 2048 * 30 + 100
        good, data, _, _, o6, st = _stored_container(oracle_lib, coder, sb, n, 2048)
        coded = next(c for c in range(o6.size - 1) if c not in st)
        bad = good.copy()
        at = cs.blob_offset(o6.size - 1) + int(o6[coded])
        bad[at:at + 128] ^= 0x10                                     # every lane's state of a coded stream
        bad = cs.reseal(bad)
        d_bad, d_good = gbc._dev(bad), gbc._dev(good)
        d_out0 = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
        d_out1 = torch.full((n + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_stored_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), n)
        gpu_ctx.container_stored_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), n)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4, coder
        assert np.array_equal(d_out1[:n].cpu().numpy(), data), coder
        assert (d_out1[n:].cpu().numpy() == SENTINEL).all()


# ---- graphs, launches, errors

def test_one_graph_follows_which_chunks_are_stored():
    torch = _torch()
    ch = 8192
    n = ch * 64 + 123
    n_chunks = -(-n // ch)
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = api.container_stored_bound(n, ch)
    d_in = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")

    def round_trip():
        ctx.container_stored_encode_async(THREE, 20000, d_in.data_ptr(), n, ch, CRC_BLOB, d_buf.data_ptr(), cap)
        ctx.container_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n, d_n.data_ptr())

    with torch.cuda.stream(stream):
        d_in.copy_(torch.from_numpy(_gen("zipf", n, 1)))
        round_trip()                                                 # grows the workspace outside the capture
        assert ctx.lib.dll.rb200_sync(ctx.h) == 0
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            round_trip()
        counts = set()
        for i, kind in enumerate(("mixed", "zipf", "uniform", "const", "mixed")):
            data = data_of(kind, n, ch, 77 + i)
            d_in.copy_(torch.from_numpy(data))
            d_out.zero_()
            g.replay()
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0, kind
            head = d_buf[:64].cpu().numpy()
            assert struct.unpack_from("<H", head, 4)[0] == 6
            assert int(d_n.item()) == n and np.array_equal(d_out[:n].cpu().numpy(), data), kind
            bm = d_buf[cs._bitmap_at(n_chunks):cs._bitmap_at(n_chunks) + 4 * ((n_chunks + 31) // 32)].cpu().numpy().view(np.uint32)
            counts.add(int(sum(bin(int(w)).count("1") for w in bm)))
        # Zipf data: only the last chunk, 123 symbols under a 128-byte stream header, is stored
        assert {1, n_chunks} <= counts and len(counts) >= 3, counts
        del g
    ctx.close()


def test_launch_counts(gpu_ctx):
    torch = _torch()
    ch = 8192
    n = ch * 40 + 5
    data = cs.mixed_data(n, ch, 1)
    cap = api.container_stored_bound(n, ch)
    d_in = gbc._dev(data)
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    # histogram + choice + model + the groups' split encoders (word: two) + store + scan + compaction + CRCs + header
    for cands, flags, want in ((THREE, 0, 12), (THREE, CRC_BLOB, 13), ([CAND(WORD, 12)], 0, 10), ([CAND(ALIAS, 12)], CRC_BLOB, 10)):
        before = gpu_ctx.launches
        gpu_ctx.container_stored_encode_async(cands, 20000, d_in.data_ptr(), n, ch, flags, d_buf.data_ptr(), cap)
        assert gpu_ctx.launches - before == want, (cands, flags)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
        before = gpu_ctx.launches
        gpu_ctx.container_stored_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), n)
        assert gpu_ctx.launches - before == 17
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == 0
        assert np.array_equal(d_out[:n].cpu().numpy(), data)


def test_argument_and_space_errors(gpu_ctx):
    torch = _torch()
    lib = gpu_ctx.lib.dll
    ch = 4096
    n = ch * 16 + 77
    data = cs.mixed_data(n, ch, 2)
    bound = api.container_stored_bound(n, ch)
    d_in = gbc._dev(data)
    d_buf = torch.full((bound + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    i, o = d_in.data_ptr(), d_buf.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, length=n, chunk=ch, out=o, out_cap=bound):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_stored_encode_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size, tol, inp,
                                                       length, chunk, 0, out, out_cap)
    before = gpu_ctx.launches
    for bad in ([], [CAND(WORD, 13)], [CAND(ALIAS, 7)], [CAND(BYTE, 17)], [CAND(BYTE, 14)] * 2, [CAND(5, 12)]):
        assert call(bad) == -1, bad
    assert call(THREE, tol=10 ** 6 + 1) == -1
    for kw in ({"ctx": None}, {"inp": None}, {"out": None}, {"out": o + 8}, {"chunk": 31}, {"chunk": (1 << 24) + 1}, {"length": 1 << 32}):
        assert call(THREE, **kw) == -1, kw
    assert call(THREE, length=0) == -2
    boff = cs.blob_offset(-(-n // ch))
    assert call(THREE, out_cap=boff - 1) == -3
    assert gpu_ctx.launches == before
    assert (d_buf.cpu().numpy() == SENTINEL).all()
    assert call(THREE, out_cap=boff + 64) == 0                       # the blob does not fit: -3 from sync, header unwritten
    assert lib.rb200_sync(gpu_ctx.h) == -3
    assert (d_buf[:64].cpu().numpy() == SENTINEL).all()
    d_buf.fill_(SENTINEL)
    for kind in ("uniform", "mixed", "const", "zipf"):               # at out_cap == bound: fits, nothing written past it
        d_in[:n].copy_(torch.from_numpy(data_of(kind, n, ch, 3)))
        assert call(THREE, out_cap=bound) == 0 and lib.rb200_sync(gpu_ctx.h) == 0, kind
        got = d_buf.cpu().numpy()
        assert size_of(got) <= bound and (got[bound:] == SENTINEL).all(), kind
    d_out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launches
    for args in ((None, o, bound, d_out.data_ptr(), 64, None), (gpu_ctx.h, o + 8, bound, d_out.data_ptr(), 64, None),
                 (gpu_ctx.h, o, bound, d_out.data_ptr() + 1, 64, None), (gpu_ctx.h, o, bound, d_out.data_ptr(), 64, d_out.data_ptr() + 4)):
        assert lib.rb200_container_stored_decode_async(*args) == -1
    assert gpu_ctx.launches == before


def test_uniform_container_is_the_bound(gpu_ctx):
    """uniform data: every chunk stored, so the container is its bound (1.000993 B/sym on 1 GiB at chunks of 8192)"""
    n, ch = 8192 * 256, 8192
    data = _gen("uniform", n, 5)
    rc, got = encode(gpu_ctx, THREE, 20000, data, ch, 0)
    assert rc == 0
    assert size_of(got) == api.container_stored_bound(n, ch)
