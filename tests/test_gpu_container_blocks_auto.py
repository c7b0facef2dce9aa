"""rb200_container_blocks_model_encode_auto_async and rb200_container_blocks_any_decode_async: a per-block container
whose coder and scale_bits are chosen on the GPU from the blocks, and one async decode for versions 2, 3 and 4.

- The device choice and every cost equal rb200_choose_blocks_coder's over the corpus of test_blocks_coder_choice and
  three candidate lists (one candidate; {word 12, byte 14, alias 14}; sixteen pairs of all three versions).
- The container is byte for byte the fixed model-building call's for the chosen pair, flags 0 and blob CRC, and a few
  equal the container packed from the oracle's per-block streams.
- Every candidate's cost is within 1 % plus per-chunk state slack plus 1 B per block of the fixed call's blob.
- The any decode equals the per-version async decode (verdict, *d_n_symbols, output) on valid and corrupt containers of
  all three versions, version 1 containers, version fields 0 and 5, and out_cap one short.
- Launch counts of both calls are pinned; one CUDA graph of both follows the data across versions; argument and space
  errors launch nothing or leave the header unwritten; a corrupt container does not disturb a valid one behind it."""
import os
import struct
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_blocks_coder_choice as bcc  # noqa: E402
import test_container_blocks as cb2  # noqa: E402
import test_container_blocks_coder as cc  # noqa: E402
import test_gpu_blocks_alias as gba  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_container_blocks_coder_async as gca  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = 0x5C
LISTS = [bcc.LISTS[1], bcc.LISTS[2], bcc.LISTS[4]]
THREE = [CAND(WORD, 12), CAND(BYTE, 14), CAND(ALIAS, 14)]
STATE_SLACK = {WORD: 64, BYTE: 32, ALIAS: 32, RANS64: 128}      # per chunk, as the single-model auto encode's test
VERSION = {WORD: 2, BYTE: 3, RANS64: 3, ALIAS: 4}


def _torch():
    import torch
    return torch


def _fixed(ctx, coder, sb, d_in, nb, bs, ch, flags, d_out, cap):
    """the fixed model-building container encode of (coder, sb), DEVICE mode"""
    if coder == WORD:
        ctx.container_blocks_encode_device(d_in.data_ptr(), nb, bs, None, ch, flags, d_out.data_ptr(), cap)
    elif coder == ALIAS:
        ctx.container_blocks_alias_encode_device(sb, d_in.data_ptr(), nb, bs, None, ch, flags, d_out.data_ptr(), cap)
    else:
        ctx.container_blocks_coder_encode_device(coder, sb, d_in.data_ptr(), nb, bs, None, ch, flags, d_out.data_ptr(), cap)


def _encode_both(ctx, cands, tol, data, nb, bs, ch, flags):
    """(auto container, fixed container of the chosen pair, chosen index, device costs), whole buffers on the host"""
    torch = _torch()
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_in = gbc._dev(data)
    d_auto = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_fix = torch.full((cap + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.container_blocks_model_encode_auto_async(cands, tol, d_in.data_ptr(), nb, bs, ch, flags, d_auto.data_ptr(), cap)
    ctx.sync()
    costs = ctx.container_blocks_auto_costs(len(cands))
    auto = d_auto.cpu().numpy()
    coder, sb = int(auto[6]), int(auto[7])
    index = cands.index(CAND(coder, sb))
    _fixed(ctx, coder, sb, d_in, nb, bs, ch, flags, d_fix, cap)
    ctx.sync()
    return auto, d_fix.cpu().numpy(), index, costs


def _container_size(buf):
    nb, n_chunks, blob_bytes = struct.unpack_from("<I", buf, 56)[0], struct.unpack_from("<Q", buf, 24)[0], struct.unpack_from("<Q", buf, 32)[0]
    return ((64 + 512 * nb + 8 * (n_chunks + 1) + 15) & ~15) + blob_bytes


CHOICE_GEOMETRIES = [(1, 32, 32), (1, 32 * 1024, 1024), (6, 16384, 4096), (3, 65536, 8192), (4, 9000, 1000)]


@pytest.mark.parametrize("kind", bcc.KINDS)
def test_choice_costs_and_container_match_host_and_fixed_call(gpu_ctx, kind):
    for gi, (nb, bs, ch) in enumerate(CHOICE_GEOMETRIES):
        data = bcc.block_data(kind, nb, bs, 10 * gi + bcc.KINDS.index(kind))
        counts = bcc.block_counts(data, nb, bs)
        for li, cands in enumerate(LISTS):
            for tol, flags in ((0, 0), (20000, CRC_BLOB), (10 ** 6, li & 1)):
                want, want_costs = api.choose_blocks_coder(counts, bs, ch, cands, tol)
                auto, fixed, index, costs = _encode_both(gpu_ctx, cands, tol, data, nb, bs, ch, flags)
                case = (kind, nb, bs, ch, li, tol, flags)
                assert index == want, case
                assert np.array_equal(costs, want_costs), case
                coder = cands[want] >> 8
                assert struct.unpack_from("<H", auto, 4)[0] == VERSION[coder], case
                assert np.array_equal(auto, fixed), case              # header, models, directory, blob and the bytes after


def _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags):
    if coder == WORD:
        wf, wo, wb = cb2.oracle_blocks_encode(oracle_lib, data, nb, bs, ch)
        return api.container_blocks_pack(nb, bs, ch, wf, wo, wb, flags)
    if coder == ALIAS:
        freqs, offs, blob = gba._oracle(oracle_lib, sb, data, nb, bs, ch)
        return api.container_blocks_alias_pack(sb, nb, bs, ch, freqs, offs, blob, flags)
    return gca._oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags)


@pytest.mark.parametrize("kind,cands,tol", [("skewed", THREE, 20000), ("zipf", THREE, 20000), ("mixed", THREE, 0),
                                            ("text", [CAND(ALIAS, 13), CAND(WORD, 12)], 0), ("two", [CAND(RANS64, 10)], 0)])
def test_auto_container_equals_the_oracle_packed_one(gpu_ctx, oracle_lib, kind, cands, tol):
    torch = _torch()
    nb, bs, ch = 5, 16384, 4096
    data = bcc.block_data(kind, nb, bs, 3)
    for flags in (0, CRC_BLOB):
        auto, _, index, _ = _encode_both(gpu_ctx, cands, tol, data, nb, bs, ch, flags)
        coder, sb = cands[index] >> 8, cands[index] & 0xFF
        want = _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags)
        assert np.array_equal(auto[:want.size], want), (kind, coder, sb, flags)
        d_out = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_blocks_any_decode_async(gbc._dev(auto).data_ptr(), auto.size, d_out.data_ptr(), data.size)
        gpu_ctx.sync()
        assert np.array_equal(d_out[:data.size].cpu().numpy(), data)


@pytest.mark.parametrize("kind", bcc.KINDS)
def test_costs_estimate_the_fixed_calls_blob(gpu_ctx, kind):
    """every candidate of the sixteen-pair list: |blob - cost| <= cost / 100 + slack per chunk + 1 B per block"""
    torch = _torch()
    nb, bs, ch = 8, 65536, 8192
    cands = bcc.LISTS[4]
    data = bcc.block_data(kind, nb, bs, 40 + bcc.KINDS.index(kind))
    _, costs = api.choose_blocks_coder(bcc.block_counts(data, nb, bs), bs, ch, cands, 0)
    cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
    d_in = gbc._dev(data)
    d_out = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    n_chunks = nb * (bs // ch)
    for c, cost in zip(cands, costs):
        coder, sb = c >> 8, c & 0xFF
        _fixed(gpu_ctx, coder, sb, d_in, nb, bs, ch, 0, d_out, cap)
        gpu_ctx.sync()
        blob = struct.unpack_from("<Q", d_out[:64].cpu().numpy(), 32)[0]
        slack = int(cost) // 100 + STATE_SLACK[coder] * n_chunks + nb
        assert abs(blob - int(cost)) <= slack, (kind, coder, sb, int(cost), blob)
        if kind == "const" and coder == WORD:
            assert blob == int(cost) == 2 * nb * bs + 128 * n_chunks


# ---- the any decode against the per-version async decodes

def _per_version(ctx, version):
    return {2: ctx.container_blocks_decode_async, 3: ctx.container_blocks_coder_decode_async,
            4: ctx.container_blocks_alias_decode_async}.get(version)


def _run(call, buf, n, out_cap):
    torch = _torch()
    d_buf = gbc._dev(buf)
    d_out = torch.full((max(n, out_cap) + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    call(d_buf.data_ptr(), buf.size, d_out.data_ptr(), out_cap, d_n.data_ptr())
    ctx = call.__self__
    return ctx.lib.dll.rb200_sync(ctx.h), int(d_n.item()), d_out.cpu().numpy()


def _same_as_per_version(ctx, buf, n, out_cap=None, name=""):
    cap = n if out_cap is None else out_cap
    got = _run(ctx.container_blocks_any_decode_async, buf, n, cap)
    version = struct.unpack_from("<H", buf, 4)[0] if buf.size >= 6 else 0
    per = _per_version(ctx, version)
    if per is None:
        assert got[0] == -4 and got[1] == -1 and (got[2] == SENTINEL).all(), (name, got[:2])
        return got[0]
    want = _run(per, buf, n, cap)
    assert got[0] == want[0] and got[1] == want[1] and np.array_equal(got[2], want[2]), (name, version, got[:2], want[:2])
    return got[0]


def _valid(gpu_ctx, oracle_lib):
    """valid containers of versions 2, 3 (byte 14, byte 9, rans64 15) and 4 (alias 14, alias 11), both flag settings"""
    nb, bs, ch = 4, 16384, 4096
    data = bcc.block_data("zipf", nb, bs, 9)
    for coder, sb in ((WORD, 12), (BYTE, 14), (BYTE, 9), (RANS64, 15), (ALIAS, 14), (ALIAS, 11), (ALIAS, 12), (BYTE, 12)):
        for flags in (0, CRC_BLOB):
            yield f"{coder}/{sb}/{flags}", _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, flags), data


def _corruptions(buf):
    """field edits (resealed and not), byte flips in every section, truncations"""
    nb = struct.unpack_from("<I", buf, 56)[0]
    dir_off = 64 + 512 * nb
    for v in (0, 1, 2, 3, 4, 5, 0x102):
        bad = buf.copy()
        struct.pack_into("<H", bad, 4, v)
        yield f"version {v}", bad
        yield f"version {v} resealed", cc.reseal(bad)
    for pos in (0, 5, 6, 7, 12, 20, 53, 57, 70, 64 + 512 * (nb - 1) + 3, dir_off + 9, buf.size - 7, buf.size - 40):
        bad = buf.copy()
        bad[pos] ^= 0x40
        yield f"flip {pos}", bad
    for cut in (0, 63, 64, dir_off, dir_off + 8, buf.size - 16, buf.size - 1):
        yield f"cut {cut}", buf[:cut].copy()


def test_any_decode_equals_the_per_version_decodes(gpu_ctx, oracle_lib):
    for name, buf, data in _valid(gpu_ctx, oracle_lib):
        assert _same_as_per_version(gpu_ctx, buf, data.size, name=name) == 0
        got = _run(gpu_ctx.container_blocks_any_decode_async, buf, data.size, data.size)
        assert got[1] == data.size and np.array_equal(got[2][:data.size], data), name
        assert _same_as_per_version(gpu_ctx, buf, data.size, data.size - 1, name + " out_cap - 1") == -3
        for cname, bad in _corruptions(buf):
            _same_as_per_version(gpu_ctx, bad, data.size, name=f"{name} {cname}")


def test_any_decode_on_the_existing_corruption_cases(gpu_ctx, oracle_lib, gen):
    """version 3's rejected containers and seeded junk, version 1 and 2 containers: each the per-version verdict"""
    nb, bs, ch, sb = 3, 16384, 4096, 14
    data = cc.block_data(nb, bs, 7)
    freqs, offs, blob = cc.oracle_blocks_encode(oracle_lib, cc.orc.CODER_BYTE, sb, data, nb, bs, ch)
    for name, bad in gca._rejected_containers(nb, bs, ch, sb, freqs, offs, blob):
        _same_as_per_version(gpu_ctx, bad, data.size, name=name)
    for name, bad in list(gca._junk())[:40]:
        _same_as_per_version(gpu_ctx, bad, data.size, name=name)
    for name, buf in gca._other_versions(oracle_lib, gen):
        rc = _same_as_per_version(gpu_ctx, buf, 60000, name=name)
        assert rc == (0 if name.startswith("version 2") else -4), name


# ---- launches, errors, recovery

def test_launch_counts(gpu_ctx):
    torch = _torch()
    nb, bs, ch = 8, 65536, 8192
    data = bcc.block_data("zipf", nb, bs, 1)
    cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
    d_in = gbc._dev(data)
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    # choice + word (K5f) + byte 14 (K5, scan, compaction) + alias 14 (the same) + CRCs + header
    for flags, want in ((0, 10), (CRC_BLOB, 11)):
        before = gpu_ctx.launches
        gpu_ctx.container_blocks_model_encode_auto_async(THREE, 20000, d_in.data_ptr(), nb, bs, ch, flags, d_buf.data_ptr(), cap)
        assert gpu_ctx.launches - before == want, flags
        gpu_ctx.sync()
    before = gpu_ctx.launches
    gpu_ctx.container_blocks_model_encode_auto_async([CAND(WORD, 12)], 0, d_in.data_ptr(), nb, bs, ch, 0, d_buf.data_ptr(), cap)
    assert gpu_ctx.launches - before == 4
    gpu_ctx.sync()
    before = gpu_ctx.launches
    gpu_ctx.container_blocks_any_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), data.size)
    assert gpu_ctx.launches - before == 13
    gpu_ctx.sync()
    assert np.array_equal(d_out[:data.size].cpu().numpy(), data)


def test_argument_and_space_errors(gpu_ctx):
    import ctypes as C
    torch = _torch()
    lib = gpu_ctx.lib.dll
    nb, bs, ch = 4, 16384, 4096
    data = bcc.block_data("skewed", nb, bs, 2)
    cap = gpu_ctx.container_blocks_capacity(nb, bs, ch)
    d_in = gbc._dev(data)
    d_buf = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    i, o = d_in.data_ptr(), d_buf.data_ptr()

    def call(cands, tol=0, ctx=gpu_ctx.h, inp=i, n_blocks=nb, block_size=bs, chunk=ch, out=o, out_cap=cap):
        c = np.ascontiguousarray(cands, dtype=np.uint32)
        return lib.rb200_container_blocks_model_encode_auto_async(ctx, c.ctypes.data_as(C.POINTER(C.c_uint32)) if c.size else None, c.size,
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
    # the blob does not fit: -3 from sync, the header unwritten
    assert call(THREE, out_cap=boff + 64) == 0
    assert lib.rb200_sync(gpu_ctx.h) == -3
    assert (d_buf[:64].cpu().numpy() == SENTINEL).all()
    assert lib.rb200_container_blocks_auto_costs(gpu_ctx.h, None, 3) == -1
    # and a valid call after it
    assert call(THREE) == 0 and lib.rb200_sync(gpu_ctx.h) == 0
    want = api.choose_blocks_coder(bcc.block_counts(data, nb, bs), bs, ch, THREE)[0]
    assert struct.unpack_from("<BB", d_buf[:8].cpu().numpy(), 6) == (THREE[want] >> 8, THREE[want] & 0xFF)
    d_out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launches
    for args in ((None, o, cap, d_out.data_ptr(), 64, None), (gpu_ctx.h, o + 8, cap, d_out.data_ptr(), 64, None),
                 (gpu_ctx.h, o, cap, d_out.data_ptr() + 1, 64, None), (gpu_ctx.h, o, cap, d_out.data_ptr(), 64, d_out.data_ptr() + 4)):
        assert lib.rb200_container_blocks_any_decode_async(*args) == -1
    assert gpu_ctx.launches == before


def test_corrupt_container_then_a_valid_one(gpu_ctx, oracle_lib):
    torch = _torch()
    nb, bs, ch = 4, 16384, 4096
    data = bcc.block_data("text", nb, bs, 5)
    for coder, sb in ((WORD, 12), (BYTE, 12), (ALIAS, 14)):
        good = _oracle_container(oracle_lib, coder, sb, data, nb, bs, ch, 0)
        bad = good.copy()
        bad[good.size - 100] ^= 0x10                                 # inside the last chunk's stream: only the decoder sees it
        d_bad, d_good = gbc._dev(bad), gbc._dev(good)
        d_out0 = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
        d_out1 = torch.full((data.size + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_blocks_any_decode_async(d_bad.data_ptr(), bad.size, d_out0.data_ptr(), data.size)
        gpu_ctx.container_blocks_any_decode_async(d_good.data_ptr(), good.size, d_out1.data_ptr(), data.size)
        assert gpu_ctx.lib.dll.rb200_sync(gpu_ctx.h) == -4, coder
        assert np.array_equal(d_out1[:data.size].cpu().numpy(), data), coder
        assert (d_out1[data.size:].cpu().numpy() == SENTINEL).all()


def test_one_graph_follows_the_data_across_versions():
    """auto encode + any decode captured once, replayed on skewed (byte 14: version 3), Zipf (word: version 2) and
    constant data (byte 14 again), and with alias first (version 4 on skewed and constant data); after each replay the container is the fixed
    call's and the output the input"""
    torch = _torch()
    nb, bs, ch = 16, 65536, 8192
    stream = torch.cuda.Stream()
    ctx = rb.Context(0, stream=stream.cuda_stream)
    cap = ctx.container_blocks_capacity(nb, bs, ch)
    d_in = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_fix = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(nb * bs + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    for cands, plan in ((THREE, [("skewed", 3), ("zipf", 2), ("const", 3), ("mixed", None)]),
                        ([CAND(ALIAS, 14), CAND(WORD, 12)], [("skewed", 4), ("zipf", None), ("const", 4)])):
        def round_trip():
            ctx.container_blocks_model_encode_auto_async(cands, 20000, d_in.data_ptr(), nb, bs, ch, CRC_BLOB, d_buf.data_ptr(), cap)
            ctx.container_blocks_any_decode_async(d_buf.data_ptr(), cap, d_out.data_ptr(), nb * bs, d_n.data_ptr())

        with torch.cuda.stream(stream):
            d_in.copy_(torch.from_numpy(bcc.block_data("zipf", nb, bs, 1)))
            round_trip()                                             # grows every group's workspace outside the capture
            assert ctx.lib.dll.rb200_sync(ctx.h) == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                round_trip()
            seen = set()
            for kind, version in plan:
                data = bcc.block_data(kind, nb, bs, 77)
                d_in.copy_(torch.from_numpy(data))
                d_out.zero_()
                g.replay()
                assert ctx.lib.dll.rb200_sync(ctx.h) == 0, kind
                head = d_buf[:64].cpu().numpy()
                v = struct.unpack_from("<H", head, 4)[0]
                seen.add(v)
                if version is not None:
                    assert v == version, (kind, v)
                assert int(d_n.item()) == data.size and np.array_equal(d_out[:data.size].cpu().numpy(), data), kind
                want = api.choose_blocks_coder(bcc.block_counts(data, nb, bs), bs, ch, cands, 20000)[0]
                coder, sb = cands[want] >> 8, cands[want] & 0xFF
                assert (int(head[6]), int(head[7])) == (coder, sb), kind
                d_fix.zero_()
                _fixed(ctx, coder, sb, d_in, nb, bs, ch, CRC_BLOB, d_fix, cap)
                assert ctx.lib.dll.rb200_sync(ctx.h) == 0
                size = _container_size(head)
                assert torch.equal(d_buf[:size], d_fix[:size]), kind
            assert len(seen) >= 2 or cands != THREE
            del g
    ctx.close()
