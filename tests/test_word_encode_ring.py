"""The fused word encoder with its streams in shared memory (K2r: word_kernels.cuh, encode_ring.cuh).

It is the default word encoder for chunks of 4096..8192 symbols.  Each warp keeps finished streams in a 12 800-byte
ring and stores them with TMA bulk copies once their offsets are published.  These cases compare the container with
the oracle byte for byte and decode it back:
  - near-worst-case streams (a {4095, 1} model on data that is mostly the frequency-1 symbol, about 11 bits per symbol),
    so a finished stream and the next one do not both fit and the ring-space wait runs;
  - uniform data, whose 8.3 KB streams wrap around the ring inside a stream;
  - n not a multiple of the chunk size or of 32;
  - a one-symbol model (frequency 4096 emits a word every step, a stream larger than the ring), which the host sends to
    the other fused encoder;
  - a blob too small (RB200_E_SPACE), a symbol outside the model (RB200_E_SYMBOL);
  - the 33-bit reciprocal (RB200_WORD_RECIPROCAL=33) and RB200_ENCODE_PATH=fused|split, which run the other encoders
    and must build the same container.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _data(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "rare":
        return (rng.random(n) < 0.9).astype(np.uint8)
    if kind == "const":
        return np.full(n, 3, np.uint8)
    return rng.integers(0, 256, n, dtype=np.uint8)


def _model(oracle_lib, kind, data):
    if kind == "rare":
        freqs = np.zeros(256, np.uint32)
        freqs[0], freqs[1] = 4095, 1
        cum = np.zeros(257, np.uint32)
        cum[1:] = np.cumsum(freqs)
        return freqs, cum
    return oracle_lib.model(data, 12)


@pytest.mark.parametrize("chunk", [4096, 8192])
@pytest.mark.parametrize("n", [8192 * 600, 8192 * 200 + 1000 + 7])
@pytest.mark.parametrize("kind", ["rare", "uniform", "const"])
def test_ring_encoder_matches_oracle(gpu_ctx, oracle_lib, kind, n, chunk):
    data = _data(kind, n, n + chunk)
    freqs, cum = _model(oracle_lib, kind, data)
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, chunk)
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, chunk, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    assert np.array_equal(gpu_ctx.decode_host(model, blob, offs, n, chunk), data)
    model.close()


def test_ring_encoder_blob_too_small(gpu_ctx, oracle_lib):
    import ryg_rans_b200 as rb
    data = _data("uniform", 8192 * 64 + 77, 5)
    freqs, _ = _model(oracle_lib, "uniform", data)
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    blob, _ = gpu_ctx.encode_host(model, data, 8192)
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_host(model, data, 8192, blob_cap=blob.size - 16)
    assert ei.value.code == -3
    model.close()


@pytest.mark.parametrize("where", [100, 8192 * 3 - 5])
def test_ring_encoder_bad_symbol(gpu_ctx, oracle_lib, where):
    import ryg_rans_b200 as rb
    data = _data("rare", 8192 * 8 + 40, 6)
    freqs, cum = _model(oracle_lib, "rare", data)
    model = gpu_ctx.model(orc.CODER_WORD, 12, freqs)
    bad = data.copy()
    bad[where] = 7                     # frequency 0 in the {4095, 1} model
    with pytest.raises(rb.RansError) as ei:
        gpu_ctx.encode_host(model, bad, 8192)
    assert ei.value.code == -7
    blob, offs = gpu_ctx.encode_host(model, data, 8192)
    oblob, ooffs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 8192, nlanes=32, scale_bits=12)
    assert np.array_equal(offs, ooffs) and np.array_equal(blob, oblob)
    model.close()


@pytest.mark.parametrize("env", [{"RB200_WORD_RECIPROCAL": "33"}, {"RB200_ENCODE_PATH": "fused"}, {"RB200_ENCODE_PATH": "split"}],
                         ids=["reciprocal33", "fused", "split"])
def test_ring_encoder_environment(cuda_box, env):
    code = r'''
import sys, numpy as np
sys.path.insert(0, %r)
import oracle, ryg_rans_b200 as rb
rng = np.random.default_rng(11)
orc = oracle.Oracle()
ctx = rb.Context(0)
for data in (rng.integers(0, 256, 8192 * 300 + 999, dtype=np.uint8), (rng.random(8192 * 100 + 31) < 0.9).astype(np.uint8)):
    f, c = orc.model(data, 12)
    m = ctx.model(rb.CODER_WORD, 12, f)
    for chunk in (4096, 8192):
        blob, offs = ctx.encode_host(m, data, chunk)
        ob, oo = orc.chunked_encode(rb.CODER_WORD, data, f, c, chunk, scale_bits=12)
        assert np.array_equal(offs, oo) and np.array_equal(blob, ob), chunk
        assert np.array_equal(ctx.decode_host(m, blob, offs, data.size, chunk), data)
    m.close()
print("ring env ok")
''' % ROOT
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "ring env ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
