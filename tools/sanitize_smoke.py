"""A small tour of every kernel for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py
Sizes are tiny (the tools slow kernels down ~100x) but cross every ring wrap, ragged tail, multi-slice host pipeline
(RB200_SLICE_MIB=1), persistent-grid loop and the corrupt-stream path.  Results are checked against the oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("RB200_SLICE_MIB", "1")
import oracle  # noqa: E402
import ryg_rans_b200 as rb  # noqa: E402


def main():
    rng = np.random.default_rng(5)
    p = 1.0 / np.arange(1, 257) ** 1.1
    orc = oracle.Oracle()
    ctx = rb.Context(0)
    for n in (1, 33, 40_000, 1_300_003):
        for kind in ("zipf", "uniform"):
            data = rng.choice(256, n, p=p / p.sum()).astype(np.uint8) if kind == "zipf" else rng.integers(0, 256, n, dtype=np.uint8)
            for coder, ocoder, sb in ((rb.CODER_WORD, oracle.CODER_WORD, 12), (rb.CODER_ALIAS, oracle.CODER_ALIAS, 16),
                                      (rb.CODER_ALIAS, oracle.CODER_ALIAS, 11), (rb.CODER_BYTE, oracle.CODER_BYTE, 14),
                                      (rb.CODER_RANS64, oracle.CODER_RANS64, 14)):
                f, c = orc.model(data, sb)
                m = ctx.model(coder, sb, f)
                for chunk in ((32, 4096) if n < 100_000 else (4096, 65536)):
                    blob, offs = ctx.encode_host(m, data, chunk)
                    ob, oo = orc.chunked_encode(ocoder, data, f, c, chunk, scale_bits=sb)
                    assert np.array_equal(offs, oo) and np.array_equal(blob, ob), (n, kind, coder, sb, chunk)
                    assert np.array_equal(ctx.decode_host(m, blob, offs, n, chunk), data)
                    if n == 40_000 and chunk == 4096:
                        bad = blob.copy()
                        bad[int(offs[1]) + 130:int(offs[1]) + 300] ^= 0x33
                        try:
                            ctx.decode_host(m, bad, offs, n, chunk)
                            raise SystemExit("corruption not reported")
                        except rb.RansError:
                            pass
                        assert np.array_equal(ctx.decode_host(m, blob, offs, n, chunk), data)
                m.close()
    # per-block path: fused model+encode, given-model encode, decode
    nb, bs, chunk = 23, 65536, 8192
    blocks = [rng.permutation(256).astype(np.uint8)[rng.choice(256, bs, p=(q := 1.0 / np.arange(1, 257) ** (0.7 + 0.1 * (b % 7))) / q.sum())] for b in range(nb)]
    data = np.concatenate(blocks)
    blob, offs, freqs = ctx.blocks_model_encode_host(data, nb, bs, chunk)
    assert np.array_equal(freqs, ctx.blocks_build_models(data, nb, bs))
    b2, o2 = ctx.blocks_encode_host(data, nb, bs, freqs, chunk)
    assert np.array_equal(b2, blob) and np.array_equal(o2, offs)
    assert np.array_equal(ctx.blocks_decode_host(blob, offs, freqs, nb, bs, chunk), data)
    st = rb.SymbolStats().count_freqs(data)
    assert np.array_equal(ctx.histogram(data), st.freqs.astype(np.uint64))
    # CRC-32 and the container calls: host mode over several pipeline slices, device mode, a rejected container
    import zlib
    import torch
    from ryg_rans_b200 import api
    for start in (0, 3):
        assert ctx.crc32(data[start:]) == zlib.crc32(data[start:].tobytes())
    f, c = orc.model(data, 12)
    m = ctx.model(rb.CODER_WORD, 12, f)
    cont = ctx.container_encode_host(m, data, 4096, api.CONTAINER_CRC_BLOB)
    blob, offs = ctx.encode_host(m, data, 4096)
    assert np.array_equal(cont, api.container_pack(rb.CODER_WORD, 12, 4096, data.size, f, offs, blob, api.CONTAINER_CRC_BLOB))
    assert np.array_equal(ctx.container_decode_host(cont), data)
    d_in = torch.from_numpy(data).cuda()
    d_cont = torch.zeros(cont.size + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(data.size + 16, dtype=torch.uint8, device="cuda")
    assert ctx.crc32_device(d_in.data_ptr() + 5, data.size - 5) == zlib.crc32(data[5:].tobytes())
    ctx.container_encode_device(m, d_in.data_ptr(), data.size, 4096, api.CONTAINER_CRC_BLOB, d_cont.data_ptr(), cont.size)
    ctx.sync()
    assert np.array_equal(d_cont[:cont.size].cpu().numpy(), cont)
    assert ctx.container_decode_device(d_cont.data_ptr(), cont.size, d_out.data_ptr(), data.size) == data.size
    assert torch.equal(d_out[:data.size], d_in)
    d_cont[cont.size - 20] ^= 1
    try:
        ctx.container_decode_device(d_cont.data_ptr(), cont.size, d_out.data_ptr(), data.size)
        raise SystemExit("blob corruption not reported")
    except rb.RansError:
        pass
    m.close()
    # the per-block containers decoded by kernels alone, version 2 (word) and version 4 (alias at 14, each block's alias
    # table built by its decoding CTA): valid, then a corrupt model and a corrupt blob (both rejected before any decode)
    cap = ctx.container_blocks_capacity(nb, bs, chunk)
    d_cb = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    crc = api.CONTAINER_CRC_BLOB
    for encode, decode_async, open_ in (
            (lambda: ctx.container_blocks_encode_device(d_in.data_ptr(), nb, bs, None, chunk, crc, d_cb.data_ptr(), cap),
             ctx.container_blocks_decode_async, api.container_blocks_open),
            (lambda: ctx.container_blocks_alias_encode_device(14, d_in.data_ptr(), nb, bs, None, chunk, crc, d_cb.data_ptr(), cap),
             ctx.container_blocks_alias_decode_async, api.container_blocks_alias_open)):
        encode()
        d_out.zero_()
        decode_async(d_cb.data_ptr(), cap, d_out.data_ptr(), data.size, d_n.data_ptr())
        ctx.sync()
        assert int(d_n.item()) == data.size and torch.equal(d_out[:data.size], d_in)
        h_cb = d_cb[:cap].cpu().numpy()
        boff = open_(h_cb)[3].ctypes.data - h_cb.ctypes.data
        for pos in (64 + 3, boff + 1000):
            d_cb[pos] ^= 1
            d_out.zero_()
            decode_async(d_cb.data_ptr(), cap, d_out.data_ptr(), data.size, d_n.data_ptr())
            try:
                ctx.sync()
                raise SystemExit("per-block container corruption not reported")
            except rb.RansError:
                pass
            assert not d_out.any().item()
            d_cb[pos] ^= 1
    # the single-model container decoded by kernels alone: a valid container of each coder, then (alias) a corrupt
    # model and a corrupt blob, rejected before any decode, and a corrupt stream with flags 0, which the decoder reports
    for coder, sb in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 16), (rb.CODER_BYTE, 14), (rb.CODER_RANS64, 12)):
        f, _ = orc.model(data, sb)
        m = ctx.model(coder, sb, f)
        ccap = ctx.container_capacity(data.size, 4096)
        d_c = torch.zeros(ccap + 16, dtype=torch.uint8, device="cuda")
        for flags in (api.CONTAINER_CRC_BLOB, 0):
            ctx.container_encode_device(m, d_in.data_ptr(), data.size, 4096, flags, d_c.data_ptr(), ccap)
            d_out.zero_()
            ctx.container_decode_async(d_c.data_ptr(), ccap, d_out.data_ptr(), data.size, d_n.data_ptr())
            ctx.sync()
            assert int(d_n.item()) == data.size and torch.equal(d_out[:data.size], d_in), (coder, flags)
        m.close()
        if coder != rb.CODER_ALIAS:
            continue
        h_c = d_c[:ccap].cpu().numpy()
        boff = api.container_open(h_c)[3].ctypes.data - h_c.ctypes.data
        for pos, flags in ((64 + 3, api.CONTAINER_CRC_BLOB), (boff + 1000, api.CONTAINER_CRC_BLOB), (boff + 1000, 0)):
            m = ctx.model(coder, sb, f)
            ctx.container_encode_device(m, d_in.data_ptr(), data.size, 4096, flags, d_c.data_ptr(), ccap)
            ctx.sync()
            m.close()
            d_c[pos] ^= 1
            d_out.zero_()
            ctx.container_decode_async(d_c.data_ptr(), ccap, d_out.data_ptr(), data.size, d_n.data_ptr())
            try:
                ctx.sync()
                raise SystemExit("single-model container corruption not reported")
            except rb.RansError:
                pass
            if flags:
                assert not d_out.any().item()
    # the single-model container with its model built on the GPU: every coder, valid; then a model the library
    # refuses (byte coder at scale_bits 16 on one symbol) and an argument error, which launches nothing
    ccap = ctx.container_capacity(data.size, 4096)
    d_c = torch.zeros(ccap + 16, dtype=torch.uint8, device="cuda")
    for coder, sb in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 16), (rb.CODER_BYTE, 14), (rb.CODER_RANS64, 12)):
        ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), data.size, 4096, api.CONTAINER_CRC_BLOB, d_c.data_ptr(), ccap)
        d_out.zero_()
        ctx.container_decode_async(d_c.data_ptr(), ccap, d_out.data_ptr(), data.size, d_n.data_ptr())
        ctx.sync()
        assert torch.equal(d_out[:data.size], d_in), coder
    d_one = torch.full((data.size,), 0x41, dtype=torch.uint8, device="cuda")
    ctx.container_model_encode_async(rb.CODER_BYTE, 16, d_one.data_ptr(), data.size, 4096, 0, d_c.data_ptr(), ccap)
    try:
        ctx.sync()
        raise SystemExit("refused model not reported")
    except rb.RansError as e:
        assert e.code == -2, e
    before = ctx.launches
    assert ctx.lib.dll.rb200_container_model_encode_async(ctx.h, rb.CODER_WORD, 14, d_in.data_ptr(), data.size, 4096, 0,
                                                          d_c.data_ptr(), ccap) == -1
    assert ctx.launches == before
    # the same with the length read from device memory (n_max = 3 n): valid, *d_n == n_max, then 0 and n_max + 1,
    # which the plan kernel refuses before anything reads the input or writes the output
    n_max = 3 * data.size
    vcap = ctx.container_capacity(n_max, 4096)
    d_v = torch.zeros(vcap + 16, dtype=torch.uint8, device="cuda")
    d_big = torch.cat([d_in, d_in, d_in])
    d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
    for coder, sb in ((rb.CODER_WORD, 12), (rb.CODER_ALIAS, 16), (rb.CODER_BYTE, 14), (rb.CODER_RANS64, 12)):
        for length, src in ((data.size, d_in), (n_max, d_big)):
            d_len.fill_(length)
            ctx.container_model_encode_varlen_async(coder, sb, d_big.data_ptr(), d_len.data_ptr(), n_max, 4096, api.CONTAINER_CRC_BLOB,
                                                    d_v.data_ptr(), vcap)
            d_big_out = torch.zeros(n_max + 16, dtype=torch.uint8, device="cuda")
            ctx.container_decode_async(d_v.data_ptr(), vcap, d_big_out.data_ptr(), n_max, d_n.data_ptr())
            ctx.sync()
            assert torch.equal(d_big_out[:length], src), (coder, length)
    for length, code in ((0, -2), (n_max + 1, -1)):
        d_len.fill_(length)
        d_v.fill_(0x5C)
        ctx.container_model_encode_varlen_async(rb.CODER_WORD, 12, d_in.data_ptr(), d_len.data_ptr(), n_max, 4096, 0, d_v.data_ptr(), vcap)
        try:
            ctx.sync()
            raise SystemExit("refused length not reported")
        except rb.RansError as e:
            assert e.code == code, e
        assert bool((d_v == 0x5C).all().item())
    # the coder chosen on the GPU: every gated group of a list that spans all four coders, on data that picks each side,
    # by value and from device memory; then a list with no feasible candidate
    cands = [api.CANDIDATE(rb.CODER_WORD, 12), api.CANDIDATE(rb.CODER_ALIAS, 16), api.CANDIDATE(rb.CODER_BYTE, 11),
             api.CANDIDATE(rb.CODER_RANS64, 14)]
    d_skew = torch.where(d_in < 250, torch.zeros_like(d_in), d_in)
    for src in (d_in, d_skew, d_one):
        for d_len_ptr in (0, d_len.data_ptr()):
            d_len.fill_(data.size)
            ctx.container_model_encode_auto_async(cands, 20000, src.data_ptr(), n_max if d_len_ptr else data.size, 4096,
                                                  api.CONTAINER_CRC_BLOB, d_v.data_ptr(), vcap, n_ptr=d_len_ptr)
            d_out.zero_()
            ctx.container_decode_async(d_v.data_ptr(), vcap, d_out.data_ptr(), data.size, d_n.data_ptr())
            ctx.sync()
            assert torch.equal(d_out[:data.size], src)
    ctx.container_model_encode_auto_async([api.CANDIDATE(rb.CODER_BYTE, 16)], 0, d_one.data_ptr(), data.size, 4096, 0, d_c.data_ptr(), ccap)
    try:
        ctx.sync()
        raise SystemExit("no feasible candidate not reported")
    except rb.RansError as e:
        assert e.code == -2, e
    print("sanitize smoke ok:", ctx.launches, "launches")


if __name__ == "__main__":
    main()
