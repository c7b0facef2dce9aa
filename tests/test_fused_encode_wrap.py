"""The fused word encoder (K2f) over many more chunks than it has resident warps.

Every worker warp of word_encode_fused_kernel cycles through a few scratch slots of its own and places a chunk a
chunk late.  The fused test in test_gpu_parity.py encodes 3 M symbols, fewer chunks than there are workers, so no
slot is ever reused there.  Here 64 Mi symbols at chunks of 4096 / 8192 make every worker take several chunks, with
three models: uniform, Zipf, and a two-symbol model {4095, 1} on data that is mostly the frequency-1 symbol (about
11 bits per symbol, close to the worst case a chunk's scratch slot is sized for).
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


@pytest.mark.parametrize("chunk", [4096, 8192])
@pytest.mark.parametrize("kind", ["uniform", "zipf", "rare"])
def test_fused_encode_reuses_slots(gpu_ctx, oracle_lib, kind, chunk):
    import torch
    import ryg_rans_b200 as rb
    data = _data(kind)
    h_data = data.cpu().numpy()
    if kind == "rare":
        freqs = np.zeros(256, np.uint32)
        freqs[0], freqs[1] = 4095, 1
        cum = np.zeros(257, np.uint32)
        cum[1:] = np.cumsum(freqs)
    else:
        freqs, cum = oracle_lib.model(h_data, 12)
    model = gpu_ctx.model(rb.CODER_WORD, 12, freqs)
    n_chunks = gpu_ctx.chunk_count(N, chunk)
    cap = gpu_ctx.encode_bound(N, chunk)
    blob = torch.empty(cap, dtype=torch.uint8, device="cuda")
    offsets = torch.zeros(n_chunks + 1, dtype=torch.int64, device="cuda")
    out = torch.zeros(N, dtype=torch.uint8, device="cuda")
    gpu_ctx.encode_device(model, data.data_ptr(), N, chunk, blob.data_ptr(), cap, offsets.data_ptr())
    gpu_ctx.sync()
    size = int(offsets[-1])
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, h_data, freqs, cum, chunk, nlanes=32, scale_bits=12)
    assert np.array_equal(offsets.cpu().numpy().astype(np.uint64), ooffs), "directory differs from the oracle container"
    assert size == oblob.size and np.array_equal(blob[:size].cpu().numpy(), oblob), "blob differs from the oracle container"
    if kind == "rare":
        assert size > 1.3 * N                       # the streams really are near the per-chunk worst case
    gpu_ctx.decode_device(model, blob.data_ptr(), size, offsets.data_ptr(), chunk, out.data_ptr(), N)
    gpu_ctx.sync()
    assert torch.equal(out, data)
    model.close()
