"""The spill tier of the shared-memory word encoder (K2r: encode_ring.cuh).

A warp's stream ring is smaller than a worst-case stream plus the pending one before it, so K2r frees ring space oldest
bytes first: a pending stream whose offset is not yet published goes to the warp's spill slot in global memory, then
the current stream's oldest bytes go there 1 KiB at a time; a stream is placed from the ring and from its slot.
The data here alternates in 64 KiB regions between near-worst-case symbols (about 11 bits each under a {4095, 1} model)
and the frequency-4095 symbol (almost nothing), so chunks see a pending stream placed directly and one spilled,
current streams spilled across the ring's wrap, and streams with none or all of their bytes spilled.  Every container
is compared byte for byte with the oracle and decoded back.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RING_BYTES = 9472       # K2r's stream ring (RB200_RING_BYTES): a longer stream has to go partly through its spill slot


def _alternating(n, seed):
    rng = np.random.default_rng(seed)
    data = (rng.random(n) < 0.9).astype(np.uint8)          # mostly the frequency-1 symbol: near-worst-case streams
    region = np.arange(n) // 65536
    data[region % 2 == 1] = 0                               # every other 64 KiB region: the frequency-4095 symbol
    return data


def _rare_model():
    freqs = np.zeros(256, np.uint32)
    freqs[0], freqs[1] = 4095, 1
    cum = np.zeros(257, np.uint32)
    cum[1:] = np.cumsum(freqs)
    return freqs, cum


@pytest.mark.parametrize("chunk", [4096, 8192])
@pytest.mark.parametrize("n", [8192 * 300, 8192 * 257 + 1000 + 7])
def test_spill_matches_oracle(gpu_ctx, oracle_lib, n, chunk):
    data = _alternating(n, n + chunk)
    freqs, cum = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, chunk)
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, chunk, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    assert np.array_equal(gpu_ctx.decode_host(model, blob, offs, n, chunk), data)
    sizes = np.diff(offs.astype(np.int64))
    if chunk == 8192:                   # streams that must spill, and streams that fit with room to spare
        assert (sizes > RING_BYTES).sum() > 10 and (sizes < 1024).sum() > 10
    model.close()


def test_spill_unaligned_input(gpu_ctx, oracle_lib):
    """An input pointer that is not 16-byte aligned: the stage is filled byte by byte."""
    import torch
    n, chunk = 8192 * 200 + 13, 8192
    data = _alternating(n, 3)
    freqs, cum = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    d_in = torch.zeros(n + 16, dtype=torch.uint8, device="cuda")
    d_in[1:n + 1] = torch.from_numpy(data).cuda()
    cap = gpu_ctx.encode_bound(n, chunk)
    d_blob = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_offs = torch.zeros(gpu_ctx.chunk_count(n, chunk) + 1, dtype=torch.int64, device="cuda")
    gpu_ctx.encode_device(model, d_in.data_ptr() + 1, n, chunk, d_blob.data_ptr(), cap, d_offs.data_ptr())
    torch.cuda.synchronize()
    offs = d_offs.cpu().numpy().view(np.uint64)
    blob = d_blob.cpu().numpy()[:int(offs[-1])]
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, chunk, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    model.close()


def test_spill_blob_one_byte_short(gpu_ctx, oracle_lib):
    """The final stream (near-worst-case, so partly in its spill slot) does not fit: RB200_E_SPACE, and nothing is
    written past the cap."""
    import torch
    import ryg_rans_b200 as rb
    n, chunk = 8192 * 64, 8192
    data = (np.random.default_rng(4).random(n) < 0.9).astype(np.uint8)
    freqs, _ = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, chunk)
    assert int(offs[-1]) - int(offs[-2]) > RING_BYTES       # the final stream cannot be placed from the ring alone
    cap = blob.size - 1
    d_in = torch.from_numpy(data).cuda()
    d_blob = torch.full((cap + 65536,), 0xAB, dtype=torch.uint8, device="cuda")
    d_offs = torch.zeros(gpu_ctx.chunk_count(n, chunk) + 1, dtype=torch.int64, device="cuda")
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_device(model, d_in.data_ptr(), n, chunk, d_blob.data_ptr(), cap, d_offs.data_ptr())
        gpu_ctx.sync()                  # the device call is asynchronous: its status is reported here
    assert ei.value.code == -3
    assert bool((d_blob[cap:] == 0xAB).all())
    model.close()


@pytest.mark.parametrize("where", [8192 * 3 - 5, 8192 * 5 - 3000])
def test_spill_bad_symbol(gpu_ctx, oracle_lib, where):
    """A symbol outside the model among the oldest bytes of a near-worst-case stream (a stream is encoded last symbol
    first, so the end of a chunk is what is spilled first).  The flag comes from the step; this checks that the spill
    path keeps it and fails the call cleanly."""
    import ryg_rans_b200 as rb
    data = (np.random.default_rng(6).random(8192 * 8) < 0.9).astype(np.uint8)
    freqs, _ = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    bad = data.copy()
    bad[where] = 7                     # frequency 0 in the {4095, 1} model
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_host(model, bad, 8192)
    assert ei.value.code == -7
    model.close()


def test_spill_bad_symbol_chunks(gpu_ctx, oracle_lib):
    """Whole chunks of a symbol outside the model: every step emits a word, a 16.5 KB stream, the longest a chunk of
    8192 can make.  Its spills stay inside the warp's own slots; the call fails, and the context encodes again."""
    import ryg_rans_b200 as rb
    data = _alternating(8192 * 600, 7)
    freqs, cum = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    bad = data.copy()
    bad[8192 * 100:8192 * 140] = 7
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_host(model, bad, 8192)
    assert ei.value.code == -7
    blob, offs = gpu_ctx.encode_host(model, data, 8192)
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 8192, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    model.close()


def test_spill_64mi_symbols(gpu_ctx, oracle_lib):
    """64 Mi symbols: every warp reuses its ring and both spill slots many times."""
    n, chunk = 64 << 20, 8192
    data = _alternating(n, 9)
    freqs, cum = _rare_model()
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, chunk)
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, chunk, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    assert np.array_equal(gpu_ctx.decode_host(model, blob, offs, n, chunk), data)
    model.close()


def test_spill_same_as_fused(cuda_box):
    """RB200_ENCODE_PATH=fused (K2f, no ring) builds the same container from the alternating data."""
    code = r'''
import sys, numpy as np
sys.path.insert(0, %r)
import ryg_rans_b200 as rb
rng = np.random.default_rng(12)
n = 8192 * 300 + 999
data = (rng.random(n) < 0.9).astype(np.uint8)
data[(np.arange(n) // 65536) %% 2 == 1] = 0
f = np.zeros(256, np.uint32); f[0], f[1] = 4095, 1
ctx = rb.Context(0)
m = ctx.model(rb.CODER_WORD, 12, f)
for chunk in (4096, 8192):
    blob, offs = ctx.encode_host(m, data, chunk)
    np.save(sys.argv[1] + "_%%d_blob.npy" %% chunk, blob)
    np.save(sys.argv[1] + "_%%d_offs.npy" %% chunk, offs)
m.close()
''' % ROOT
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        for tag, env in (("ring", {}), ("fused", {"RB200_ENCODE_PATH": "fused"})):
            e = dict(os.environ, **env)
            e.pop("RB200_ENCODE_PATH", None) if not env else None
            out = subprocess.run([sys.executable, "-c", code, os.path.join(tmp, tag)], env=e, capture_output=True, text=True, timeout=600)
            assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        for chunk in (4096, 8192):
            for part in ("blob", "offs"):
                a = np.load(os.path.join(tmp, "ring_%d_%s.npy" % (chunk, part)))
                b = np.load(os.path.join(tmp, "fused_%d_%s.npy" % (chunk, part)))
                assert np.array_equal(a, b), (chunk, part)
