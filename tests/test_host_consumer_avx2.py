"""include/rans_word_avx2.h: the 32-lane AVX2 consumer for GPU chunk streams (SURVEY 8f.4).

A host without a GPU must be able to read what the GPU encoder wrote.  The header decodes the word coder's
N = 32 streams with four __m256i of states; here it is checked against the reference's own N = 32 streams (golden
fixtures made by the reference code), against oracle containers of every input shape, against corrupt streams, and
-- on the GPU box -- against containers the CUDA encoder produced.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "avx2_consumer", "consumer.cpp")


def _has_avx2():
    try:
        return " avx2 " in open("/proc/cpuinfo").read().replace("\n", " ")
    except OSError:
        return False


@pytest.fixture(scope="module")
def consumer(tmp_path_factory):
    if shutil.which("g++") is None or not _has_avx2():
        pytest.skip("needs g++ and an AVX2 host")
    so = tmp_path_factory.mktemp("avx2") / "libconsumer.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-mavx2", "-msse4.1", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                           "-o", str(so), SRC])
    lib = C.CDLL(str(so))
    lib.avx2_decode_chunk.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    lib.avx2_decode_container.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.decode_chunks.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.decode_chunks.restype = C.c_long
    return lib


def _decode_chunk(lib, stream, freqs, cum, m, via_word_tables=0):
    padded = np.zeros(stream.size + 16, np.uint8)           # the 16 readable bytes the header asks for
    padded[:stream.size] = stream
    out = np.zeros(m + 32, np.uint8)
    rc = lib.avx2_decode_chunk(padded.ctypes.data, stream.size, freqs.ctypes.data, cum.ctypes.data, out.ctypes.data, m, via_word_tables)
    return rc, out[:m]


def _decode_container(lib, blob, offs, n, chunk, freqs, cum):
    padded = np.concatenate([blob, np.zeros(16, np.uint8)])
    out = np.zeros(n, np.uint8)
    rc = lib.avx2_decode_container(padded.ctypes.data, offs.ctypes.data, offs.size - 1, chunk, n, freqs.ctypes.data, cum.ctypes.data,
                                   out.ctypes.data)
    out2 = np.zeros(n, np.uint8)                              # the header's own container loop must agree
    rc2 = lib.decode_chunks(padded.ctypes.data, offs.ctypes.data, offs.size - 1, chunk, n, freqs.ctypes.data, cum.ctypes.data,
                            out2.ctypes.data)
    assert (rc == 0) == (rc2 == 0) and (rc != 0 or np.array_equal(out, out2))
    return rc, out


def test_decodes_the_references_own_n32_streams(consumer):
    """Golden fixtures: 32-way streams written by the reference's RansWordEncPut/Flush (tests/golden/make_golden.py)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "golden.npz"))
    cases = sorted({k.split("/")[0] for k in g.files})
    assert cases
    for name in cases:
        data, freqs, stream = g[f"{name}/data"], g[f"{name}/word/freqs"].astype(np.uint32), g[f"{name}/word/N32"]
        cum = np.concatenate([[0], np.cumsum(freqs)]).astype(np.uint32)
        for via in (0, 1):
            rc, out = _decode_chunk(consumer, stream, freqs, cum, data.size, via)
            assert rc == 0 and np.array_equal(out, data), (name, via)


@pytest.mark.parametrize("kind", ["uniform", "zipf", "text", "const", "two", "skew"])
def test_decodes_oracle_containers_of_every_shape(consumer, oracle_lib, gen, kind):
    for n in (1, 31, 32, 33, 4097, 70001):
        data = gen(kind, n, 5)
        freqs, cum = oracle_lib.model(data, 12)
        for chunk in (8192, 64):
            blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, chunk)
            rc, out = _decode_container(consumer, blob, offs, n, chunk, freqs, cum)
            assert rc == 0 and np.array_equal(out, data), (kind, n, chunk)


def test_corrupt_streams_are_reported_not_followed(consumer, oracle_lib, gen):
    data = gen("zipf", 8192, 9)
    freqs, cum = oracle_lib.model(data, 12)
    blob, offs = oracle_lib.chunked_encode(orc.CODER_WORD, data, freqs, cum, 8192)
    stream = blob[int(offs[0]):int(offs[1]) & ~15]
    assert _decode_chunk(consumer, stream, freqs, cum, data.size)[0] == 0
    rng = np.random.default_rng(3)
    flagged = 0
    for _ in range(200):
        bad = stream.copy()
        pos = int(rng.integers(0, bad.size))
        bad[pos] ^= 1 << int(rng.integers(0, 8))
        rc, out = _decode_chunk(consumer, bad, freqs, cum, data.size)
        flagged += rc != 0
        assert rc != 0 or not np.array_equal(out, data) or True      # never crashes; a flipped bit may decode to other data
    assert flagged >= 190                                              # ... but the end-state check catches nearly all of them
    assert _decode_chunk(consumer, stream[:-2], freqs, cum, data.size)[0] != 0      # truncated
    assert _decode_chunk(consumer, stream[:64], freqs, cum, data.size)[0] != 0      # shorter than the header


@pytest.mark.gpu
def test_decodes_what_the_gpu_encoded(consumer, gpu_ctx, oracle_lib, gen):
    for kind, n in (("text", 1_000_003), ("uniform", 262_144), ("const", 5000)):
        data = gen(kind, n, 31)
        freqs, cum = oracle_lib.model(data, 12)
        model = gpu_ctx.model(0, 12, freqs)
        blob, offs = gpu_ctx.encode_host(model, data, 8192)
        model.close()
        rc, out = _decode_container(consumer, blob, offs, n, 8192, freqs, cum)
        assert rc == 0 and np.array_equal(out, data), kind
