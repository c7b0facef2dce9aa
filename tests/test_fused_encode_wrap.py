"""The fused encoders over many more chunks than they have resident warps.

Every worker warp of word_encode_fused_kernel (K2f), of the fused alias / byte encoder and of block_encode_fused_kernel
(K5f) cycles through a few scratch slots of its own and places a chunk a chunk late (placement.cuh: SlotQueue).  The
fused test in test_gpu_parity.py encodes 3 M symbols, fewer chunks than there are workers, so no slot is ever reused
there.  Here 64 Mi symbols at chunks of 4096 / 8192 (up to 16 384 chunks, against at most SMs x 32 worker warps) make
every worker take several chunks: the word coder with three models -- uniform, Zipf, and a two-symbol model {4095, 1}
on data that is mostly the frequency-1 symbol (about 11 bits per symbol, close to the worst case a chunk's scratch slot
is sized for) -- and the alias coder at scale_bits 16 and the byte coder at 14 with the uniform and Zipf models.  The per-block tests in
test_gpu_parity.py encode at most 200 blocks, fewer than the worker CTAs of K5f (5 per SM, less the scanner's); here
4096 blocks make every worker CTA take several blocks.
"""
import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu

N = 1 << 26


def _data(kind):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(0xF05ED)
    if kind == "uniform":
        return torch.randint(0, 256, (N,), dtype=torch.uint8, device="cuda", generator=g)
    if kind == "zipf":
        p = 1.0 / torch.arange(1, 257, dtype=torch.float64) ** 1.1
        cdf = torch.cumsum(p / p.sum(), 0).to(device="cuda", dtype=torch.float32)
        u = torch.rand(N, device="cuda", generator=g)
        return torch.searchsorted(cdf, u).clamp_(max=255).to(torch.uint8)
    # "rare": symbol 1 (frequency 1 of 4096) 90 % of the time, symbol 0 (frequency 4095) otherwise
    return (torch.rand(N, device="cuda", generator=g) < 0.9).to(torch.uint8)


# (coder, scale_bits, kind); the word coder's cases keep their ids ("rare" needs scale_bits 12)
CASES = [pytest.param("word", 12, kind, id=kind) for kind in ("uniform", "zipf", "rare")] + \
        [pytest.param(coder, sb, kind, id=f"{coder}{sb}-{kind}") for coder, sb in (("alias", 16), ("byte", 14))
         for kind in ("uniform", "zipf")]
CODERS = {"word": orc.CODER_WORD, "alias": orc.CODER_ALIAS, "byte": orc.CODER_BYTE}    # the library's numbering too


@pytest.mark.parametrize("chunk", [4096, 8192])
@pytest.mark.parametrize("coder, sb, kind", CASES)
def test_fused_encode_reuses_slots(gpu_ctx, oracle_lib, coder, sb, kind, chunk):
    import torch
    data = _data(kind)
    h_data = data.cpu().numpy()
    if kind == "rare":
        freqs = np.zeros(256, np.uint32)
        freqs[0], freqs[1] = 4095, 1
        cum = np.zeros(257, np.uint32)
        cum[1:] = np.cumsum(freqs)
    else:
        freqs, cum = oracle_lib.model(h_data, sb)
    model = gpu_ctx.model(CODERS[coder], sb, freqs)
    n_chunks = gpu_ctx.chunk_count(N, chunk)
    cap = gpu_ctx.encode_bound(N, chunk)
    blob = torch.empty(cap, dtype=torch.uint8, device="cuda")
    offsets = torch.zeros(n_chunks + 1, dtype=torch.int64, device="cuda")
    out = torch.zeros(N, dtype=torch.uint8, device="cuda")
    gpu_ctx.encode_device(model, data.data_ptr(), N, chunk, blob.data_ptr(), cap, offsets.data_ptr())
    gpu_ctx.sync()
    size = int(offsets[-1])
    oblob, ooffs = oracle_lib.chunked_encode(CODERS[coder], h_data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
    assert np.array_equal(offsets.cpu().numpy().astype(np.uint64), ooffs), "directory differs from the oracle container"
    assert size == oblob.size and np.array_equal(blob[:size].cpu().numpy(), oblob), "blob differs from the oracle container"
    if kind == "rare":
        assert size > 1.3 * N                       # the streams really are near the per-chunk worst case
    gpu_ctx.decode_device(model, blob.data_ptr(), size, offsets.data_ptr(), chunk, out.data_ptr(), N)
    gpu_ctx.sync()
    assert torch.equal(out, data)
    model.close()


def test_fused_block_encode_reuses_slots(gpu_ctx, oracle_lib):
    """K5f with and without the model build (rb200_blocks_model_encode, rb200_blocks_encode) on 4096 blocks of 64 KiB at
    chunks of 8192: models, directory and blob match the oracle block by block, and the container decodes back."""
    import torch
    n_blocks, block_size, chunk = 4096, 65536, 8192
    per = block_size // chunk
    g = torch.Generator(device="cuda")
    g.manual_seed(0xB10C)
    # block b: Zipf over 256 symbols with exponent 0.6 + 0.1 * (b % 9), as in test_gpu_parity.py's per-block cases
    expo = 0.6 + 0.1 * (torch.arange(n_blocks, dtype=torch.float64) % 9)
    p = 1.0 / torch.arange(1, 257, dtype=torch.float64)[None, :] ** expo[:, None]
    cdf = torch.cumsum(p / p.sum(1, keepdim=True), 1).to(device="cuda", dtype=torch.float32).contiguous()
    u = torch.rand(n_blocks, block_size, device="cuda", generator=g)
    data = torch.searchsorted(cdf, u).clamp_(max=255).to(torch.uint8).reshape(-1)
    n = data.numel()
    cap = gpu_ctx.encode_bound(n, chunk)

    def encode(build):
        freqs = torch.zeros((n_blocks, 256), dtype=torch.int16, device="cuda")    # u16 bit patterns
        blob = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        offs = torch.zeros(n_blocks * per + 1, dtype=torch.int64, device="cuda")
        if build:
            gpu_ctx.blocks_model_encode_device(data.data_ptr(), n_blocks, block_size, freqs.data_ptr(), chunk, blob.data_ptr(), cap,
                                               offs.data_ptr())
        else:
            gpu_ctx.blocks_build_models_device(data.data_ptr(), n_blocks, block_size, freqs.data_ptr())
            gpu_ctx.blocks_encode_device(data.data_ptr(), n_blocks, block_size, freqs.data_ptr(), chunk, blob.data_ptr(), cap,
                                         offs.data_ptr())
        gpu_ctx.sync()
        return freqs, blob, offs

    freqs, blob, offs = encode(True)
    freqs2, blob2, offs2 = encode(False)
    assert torch.equal(freqs, freqs2) and torch.equal(offs, offs2) and torch.equal(blob, blob2)

    h_data = data.cpu().numpy()
    h_freqs = freqs.cpu().numpy().view(np.uint16)
    h_offs = offs.cpu().numpy().astype(np.uint64)
    size = int(h_offs[-1])
    h_blob = blob[:size].cpu().numpy()
    base = 0
    for b in range(n_blocks):             # oracle: every block is its own container; they concatenate (16-byte aligned ends)
        blk = h_data[b * block_size:(b + 1) * block_size]
        f, c = oracle_lib.model(blk, 12)
        assert np.array_equal(h_freqs[b].astype(np.uint32), f), b
        ob, oo = oracle_lib.chunked_encode(orc.CODER_WORD, blk, f, c, chunk, nlanes=32, scale_bits=12)
        assert np.array_equal(h_offs[b * per:(b + 1) * per], oo[:-1] + np.uint64(base)), b
        assert np.array_equal(h_blob[base:base + ob.size], ob), b
        base += ob.size
    assert size == base

    out = torch.zeros_like(data)
    gpu_ctx.blocks_decode_device(blob.data_ptr(), size, offs.data_ptr(), freqs.data_ptr(), n_blocks, block_size, chunk, out.data_ptr())
    gpu_ctx.sync()
    assert torch.equal(out, data)
