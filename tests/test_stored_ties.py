"""The store rules of versions 5 and 6 at their exact boundaries, on the host.

Version 6 stores chunk c when its stream, rounded up to 16, is longer than round16(m_c); version 5 stores a block when
its chunks' rounded streams sum to more than per_block x round16(chunk_syms).  Ties stay coded.  Natural data almost
never lands on the 16-byte plateau where `>` and `>=` differ, so the inputs here are built to land on it: a target
chunk (or block) holds k copies of a cheap symbol and the rest from a pool of dear ones, shuffled by a seed.

- Version 6 (the word coder at 12, chunks of 4096 and a ragged last chunk of 1000): the symbols the targets do not take
  go to the other chunks, so the input's histogram, and with it the model, is the same for every k and seed, and the
  target's stream moves by about a byte per cheap symbol.
- Version 5 (the byte coder at 14, 3 blocks of 9 chunks of 1000): block 1 is the target; its model follows k, and the
  shuffle moves the rounding of its nine streams.

TIES_V6 and TIES_V5 pin the (k, seed) that `search_v6` and `search_v5` found for each edge: the tie, one 16-byte step
over it and one under it.  The tests re-derive every target's stream with the oracle and assert that the edge is hit,
so a change to the generators cannot lose it silently, then check the rule's verdict, pack, open and decode.
test_gpu_stored_geometry checks the GPU's containers of the same inputs against these."""
import os
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_blocks_stored as cbs  # noqa: E402
import test_container_stored as cs  # noqa: E402
from conftest import _gen  # noqa: E402

CHEAP = 0x41
EDGES = {"tie": 0, "over": 16, "under": -16}          # r16(stream) - r16(m): the rule's boundary and one step either side

# ---- version 6: chunks 0-3 of 4096, chunk 4 of 1000 (ragged); targets 0 and 4
V6_PAIR = (rb.CODER_WORD, 12)
V6_CH, V6_N = 4096, 4 * 4096 + 1000
V6_TARGETS = (0, 4)
V6_CHEAP_TOTAL = 8000

# ---- version 5: 3 blocks of 9000 in chunks of 1000 (9 chunks per block); target block 1
V5_PAIR = (rb.CODER_BYTE, 14)
V5_GEO = (3, 9000, 1000)
V5_TARGET = 1

# (k, seed) per edge; for version 6 one pair per target chunk.  Found by search_v6 / search_v5.
TIES_V6 = {"tie": ((555, 1), (196, 2)), "over": ((535, 3), (179, 4)), "under": ((568, 3), (211, 4))}
TIES_V5 = {"tie": (1756, 4), "over": (1728, 5), "under": (1772, 5)}


def r16(x):
    return (x + 15) & ~15


def _dear(n, seed):
    """n symbols uniform over every byte but CHEAP"""
    s = np.random.default_rng(seed).integers(0, 255, n, dtype=np.int64)
    return (s + (s >= CHEAP)).astype(np.uint8)


def _target(k, m, dear, seed):
    return np.random.default_rng(seed).permutation(np.concatenate([np.full(k, CHEAP, np.uint8), dear[:m - k]]))


def v6_data(picks):
    """the version 6 input for ((k0, seed0), (k4, seed4)): target chunk 0 and the ragged chunk 4 take k cheap symbols
    and the rest from their own dear pools; chunks 1-3 take every other symbol, so the histogram never changes"""
    (k0, s0), (k4, s4) = picks
    m4 = V6_N - 4 * V6_CH
    d0, d4, rest = _dear(V6_CH, 1), _dear(m4, 2), _dear(3 * V6_CH - V6_CHEAP_TOTAL, 3)
    middle = np.concatenate([np.full(V6_CHEAP_TOTAL - k0 - k4, CHEAP, np.uint8), d0[V6_CH - k0:], d4[m4 - k4:], rest])
    middle = np.random.default_rng(4).permutation(middle)
    return np.concatenate([_target(k0, V6_CH, d0, s0), middle, _target(k4, m4, d4, s4)])


def v5_data(pick):
    """the version 5 input for (k, seed): block 0 Zipf, block 1 the target, block 2 uniform"""
    nb, bs, _ = V5_GEO
    k, seed = pick
    return np.concatenate([_gen("zipf", bs, 31), _target(k, bs, _dear(bs, 5), seed), _gen("uniform", bs, 32)])


def v6_chunk_size(oracle_lib, data, c):
    """chunk c's stream size under the model of all of data, by the oracle"""
    coder, sb = V6_PAIR
    freqs, cum = oracle_lib.model(data, sb)
    chunk = data[c * V6_CH:(c + 1) * V6_CH]
    blob, offs = oracle_lib.chunked_encode(cs.OCODER[coder], chunk, freqs, cum, V6_CH, scale_bits=sb)
    return int(offs[1]) - int(offs[0])


def v5_block_sum(oracle_lib, data):
    """the target block's rounded chunk sum, by the oracle"""
    nb, bs, ch = V5_GEO
    coder, sb = V5_PAIR
    blk = data[V5_TARGET * bs:(V5_TARGET + 1) * bs]
    f, c = oracle_lib.model(blk, sb)
    blob, offs = oracle_lib.chunked_encode(cbs.OCODER[coder], blk, f, c, ch, scale_bits=sb)
    return sum(r16(s.size) for s in cbs.streams(offs, blob))


def search_v6(oracle_lib, ks=range(100, 1000), seeds=range(8)):
    """(k, seed) per edge and target, for TIES_V6: the first k (coarse) and seed (fine) whose stream lands on it"""
    found = {e: [None, None] for e in EDGES}
    for t, c in enumerate(V6_TARGETS):
        m = cs.chunk_m(c, V6_CH, V6_N)
        for e, d in EDGES.items():
            for k in ks:
                if k > m or found[e][t]:
                    break
                for seed in seeds:
                    picks = [(0, 0), (0, 0)]
                    picks[t] = (k, seed)
                    if r16(v6_chunk_size(oracle_lib, v6_data(picks), c)) == r16(m) + d:
                        found[e][t] = (k, seed)
                        break
    return {e: tuple(v) for e, v in found.items()}


def search_v5(oracle_lib, ks=range(1000, 4000, 4), seeds=range(8)):
    """(k, seed) per edge, for TIES_V5"""
    nb, bs, ch = V5_GEO
    found = {}
    for e, d in EDGES.items():
        for k in ks:
            hit = next((s for s in seeds if v5_block_sum(oracle_lib, v5_data((k, s))) == (bs // ch) * r16(ch) + d), None)
            if hit is not None:
                found[e] = (k, hit)
                break
    return found


def v6_case(oracle_lib, edge):
    """(data, freqs, offsets, blob) of the oracle for the edge's input, after asserting that both targets hit it"""
    coder, sb = V6_PAIR
    data = v6_data(TIES_V6[edge])
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, data, V6_CH)
    sizes = [s.size for s in cs.streams(offs, blob)]
    for c in V6_TARGETS:
        m = cs.chunk_m(c, V6_CH, V6_N)
        assert r16(sizes[c]) == r16(m) + EDGES[edge], (edge, c, sizes[c], m)
    return data, freqs, offs, blob


def v5_case(oracle_lib, edge):
    """(data, block_freqs, offsets, blob) of the oracle for the edge's input, after asserting that the block hits it"""
    nb, bs, ch = V5_GEO
    coder, sb = V5_PAIR
    data = v5_data(TIES_V5[edge])
    freqs, offs, blob = cbs.oracle_streams(oracle_lib, coder, sb, data, nb, bs, ch)
    per = bs // ch
    got = sum(r16(s.size) for s in cbs.streams(offs, blob)[V5_TARGET * per:(V5_TARGET + 1) * per])
    assert got == per * r16(ch) + EDGES[edge], (edge, got)
    return data, freqs, offs, blob


def test_v6_model_is_the_same_for_every_edge(oracle_lib):
    """the targets' symbols move between chunks, never in or out of the input: one model for every edge"""
    models = [oracle_lib.model(v6_data(TIES_V6[e]), V6_PAIR[1])[0] for e in EDGES]
    assert all(np.array_equal(m, models[0]) for m in models)
    assert all(v6_data(TIES_V6[e]).size == V6_N for e in EDGES)


@pytest.mark.parametrize("edge", list(EDGES))
def test_v6_edge_verdict_pack_and_decode(oracle_lib, edge):
    coder, sb = V6_PAIR
    data, freqs, offs, blob = v6_case(oracle_lib, edge)
    bits, o6, b6, stored = cs.apply_store(data, V6_CH, offs, blob)
    for c in V6_TARGETS:
        assert (c in stored) == (edge == "over"), (edge, c, stored)        # the tie and the step under it stay coded
    buf = api.container_stored_pack(coder, sb, V6_CH, V6_N, freqs, bits, o6, b6, cs.CRC_BLOB)
    assert np.array_equal(buf, cs.py_pack(coder, sb, V6_CH, V6_N, freqs, bits, o6, b6, cs.CRC_BLOB))
    meta, f, b, o, bl = api.container_stored_open(buf)
    _, cum = oracle_lib.model(data, sb)
    assert np.array_equal(cs.decode_host(oracle_lib, coder, sb, f, cum, b, o, bl, V6_N, V6_CH), data)


@pytest.mark.parametrize("edge", list(EDGES))
def test_v5_edge_verdict_pack_and_decode(oracle_lib, edge):
    nb, bs, ch = V5_GEO
    coder, sb = V5_PAIR
    data, freqs, offs, blob = v5_case(oracle_lib, edge)
    f5, o5, b5, stored = cbs.apply_store(freqs, offs, blob, data, nb, bs, ch)
    assert (V5_TARGET in stored) == (edge == "over"), (edge, stored)
    assert 2 in stored and 0 not in stored                                # the uniform block stored, the Zipf one coded
    buf = api.container_blocks_stored_pack(coder, sb, nb, bs, ch, f5, o5, b5, cbs.CRC_BLOB)
    assert np.array_equal(buf, cbs.py_pack(coder, sb, nb, bs, ch, f5, o5, b5, cbs.CRC_BLOB))
    meta, f2, o2, b2 = api.container_blocks_stored_open(buf)
    assert np.array_equal(cbs.decode_host(oracle_lib, coder, sb, meta, f2, o2, b2, nb, bs, ch), data)


if __name__ == "__main__":                                          # re-run the searches after a generator changes
    import oracle
    lib = oracle.Oracle()
    print("TIES_V6 =", search_v6(lib))
    print("TIES_V5 =", search_v5(lib))
