"""rb200_choose_blocks_coder: the per-block coder-choice rule of rb200_container_blocks_model_encode_auto_async on the
host.  Its costs and its choice equal a Python statement of the rule (each block's model from SymbolStats.normalize_freqs,
log2q by its definition, the word coder's one-symbol blocks at 2 bytes per symbol plus 128 per chunk) over blocks of
many shapes, several candidate lists and tolerances 0, 2 % and 10^6; argument errors are refused.  The one-symbol cost
is pinned against the oracle's stream.  No GPU needed."""
import numpy as np
import pytest

import oracle as orc
from ryg_rans_b200 import api

WORD, BYTE, ALIAS, RANS64 = api.CODER_WORD, api.CODER_BYTE, api.CODER_ALIAS, api.CODER_RANS64
CAND = api.CANDIDATE

LISTS = [
    [CAND(WORD, 12)],
    [CAND(BYTE, 14)],
    [CAND(WORD, 12), CAND(BYTE, 14), CAND(ALIAS, 14)],
    [CAND(ALIAS, 15), CAND(RANS64, 9), CAND(WORD, 12), CAND(BYTE, 8)],
    # sixteen distinct pairs over the three versions
    [CAND(WORD, 12)] + [CAND(BYTE, sb) for sb in (8, 10, 12, 13, 14, 15)] + [CAND(RANS64, sb) for sb in (8, 12, 15)]
    + [CAND(ALIAS, sb) for sb in (8, 9, 11, 12, 14, 15)],
]
TOLERANCES = [0, 20000, 10 ** 6]


def log2q(f):
    """log2 f in 16.16 fixed point, by the integer steps of include/rans_b200.h"""
    k = f.bit_length() - 1
    x, r = f << (31 - k), k << 16
    for i in range(15, -1, -1):
        x = (x * x) >> 31
        if x >= 1 << 32:
            x >>= 1
            r |= 1 << i
    return r


def rule(block_counts, block_size, chunk, cands, tol):
    """(index, costs): the rule as the header states it"""
    per_block = block_size // chunk
    costs = [0] * len(cands)
    for counts in block_counts:
        for i, c in enumerate(cands):
            coder, sb = c >> 8, c & 0xFF
            st = api.SymbolStats()
            st.freqs[:] = counts
            f = st.normalize_freqs(1 << sb).freqs
            if coder == WORD and int(f.max()) == 4096:
                costs[i] += 2 * block_size + 128 * per_block
                continue
            bits_q = sum(int(counts[s]) * ((sb << 16) - log2q(int(f[s]))) for s in range(256) if counts[s])
            costs[i] += -(-bits_q // (1 << 19)) + per_block * (256 if coder == RANS64 else 128)
    lo = min(costs)
    bound = lo + lo * tol // 10 ** 6
    return next(i for i, c in enumerate(costs) if c <= bound), costs


def _zipf(rng, n, s):
    p = 1.0 / np.arange(1, 257) ** s
    return rng.permutation(256)[rng.choice(256, n, p=p / p.sum())]


def _skewed(rng, n, p_top):
    tail = 1.0 / np.arange(1, 256) ** 1.1
    p = np.concatenate([[p_top], (1 - p_top) * tail / tail.sum()])
    return rng.permutation(256)[rng.choice(256, n, p=p)]


def block_data(kind, n_blocks, block_size, seed):
    """n_blocks blocks of one shape, each drawn on its own (a per-block permutation, exponent or skew)"""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(n_blocks):
        if kind == "uniform":
            d = rng.integers(0, 256, block_size)
        elif kind == "zipf":
            d = _zipf(rng, block_size, 0.6 + 0.8 * rng.random())
        elif kind == "skewed":
            d = _skewed(rng, block_size, 0.90 + 0.09 * rng.random())
        elif kind == "const":
            d = np.full(block_size, int(rng.integers(0, 256)))
        elif kind == "mixed":                        # constant and Zipf blocks in turn
            d = np.full(block_size, 0) if b % 2 == 0 else _zipf(rng, block_size, 1.1)
        elif kind == "text":
            syms = rng.permutation(256)[:82]
            d = syms[rng.choice(82, block_size, p=rng.dirichlet(np.full(82, 0.35)))]
        elif kind == "two":
            d = np.where(rng.random(block_size) < 0.01, int(rng.integers(0, 128)), int(rng.integers(128, 256)))
        else:
            raise ValueError(kind)
        out.append(np.asarray(d, dtype=np.uint8))
    return np.concatenate(out)


KINDS = ["uniform", "zipf", "skewed", "const", "mixed", "text", "two"]
# (n_blocks, block_size, chunk_syms): one block of 32 symbols, one block of 32 chunks, and ordinary shapes
GEOMETRIES = [(1, 32, 32), (1, 32 * 1024, 1024), (6, 16384, 4096), (3, 65536, 8192), (4, 9000, 1000)]


def block_counts(data, n_blocks, block_size):
    return np.stack([np.bincount(data[b * block_size:(b + 1) * block_size], minlength=256) for b in range(n_blocks)]).astype(np.uint32)


@pytest.mark.parametrize("kind", KINDS)
def test_choice_and_costs_equal_the_rule(kind):
    for gi, (nb, bs, ch) in enumerate(GEOMETRIES):
        counts = block_counts(block_data(kind, nb, bs, 10 * gi + KINDS.index(kind)), nb, bs)
        for cands in LISTS:
            for tol in TOLERANCES:
                want_i, want_costs = rule(counts, bs, ch, cands, tol)
                i, costs = api.choose_blocks_coder(counts, bs, ch, cands, tol)
                assert [int(c) for c in costs] == want_costs, (kind, nb, bs, ch, cands, tol)
                assert i == want_i, (kind, nb, bs, ch, cands, tol)


def test_word_one_symbol_cost_is_the_oracle_stream():
    """a constant block under word 12: every chunk of the oracle's stream is 2 chunk_syms + 128 bytes (before the
    16-byte pad), and that is the cost"""
    o = orc.Oracle()
    for bs, ch in ((65536, 8192), (32, 32), (9000, 1000), (99, 33)):
        data = np.full(bs, 0x41, np.uint8)
        f, c = o.model(data, 12)
        blob, offs = o.chunked_encode(orc.CODER_WORD, data, f, c, ch, nlanes=32, scale_bits=12)
        ends = np.asarray(offs[1:], dtype=np.int64)
        starts = np.asarray(offs[:-1], dtype=np.int64)
        assert np.all(ends - starts <= 2 * ch + 128 + 15) and int(ends[-1] - starts[-1]) >= 2 * ch + 128, (bs, ch)
        _, costs = api.choose_blocks_coder(block_counts(data, 1, bs), bs, ch, [CAND(WORD, 12)])
        assert int(costs[0]) == 2 * bs + 128 * (bs // ch), (bs, ch)
    # and where the chunks are 16-byte multiples the stream is exactly that long
    data = np.full(65536, 7, np.uint8)
    f, c = o.model(data, 12)
    blob, offs = o.chunked_encode(orc.CODER_WORD, data, f, c, 8192, nlanes=32, scale_bits=12)
    assert int(offs[-1]) == 2 * 65536 + 128 * 8


def test_tolerance_moves_the_choice():
    """skewed blocks: byte 14 is smaller than word 12; with 10^6 ppm the first candidate wins"""
    nb, bs, ch = 4, 65536, 8192
    counts = block_counts(block_data("skewed", nb, bs, 5), nb, bs)
    cands = [CAND(WORD, 12), CAND(BYTE, 14), CAND(ALIAS, 14)]
    i, costs = api.choose_blocks_coder(counts, bs, ch, cands, 0)
    assert i == 1 and costs[1] < costs[0] and costs[1] == costs[2]
    assert api.choose_blocks_coder(counts, bs, ch, cands, 10 ** 6)[0] == 0


def _raw(counts, nb, bs, ch, cands, tol, costs=True, chosen=True):
    import ctypes as C
    lib = api.load()
    counts = np.ascontiguousarray(counts, dtype=np.uint32)
    cands = np.ascontiguousarray(cands, dtype=np.uint32)
    out = np.zeros(16, np.uint64)
    k = C.c_uint32(99)
    rc = lib.dll.rb200_choose_blocks_coder(counts.ctypes.data_as(api._u32p) if counts.size else None, nb, bs, ch,
                                           cands.ctypes.data_as(api._u32p) if cands.size else None, cands.size, tol,
                                           out.ctypes.data_as(api._u64p) if costs else None, C.byref(k) if chosen else None)
    return rc, k.value


def test_argument_errors():
    nb, bs, ch = 2, 4096, 1024
    counts = block_counts(block_data("zipf", nb, bs, 1), nb, bs)
    good = [CAND(WORD, 12), CAND(BYTE, 14)]
    assert _raw(counts, nb, bs, ch, good, 0) == (0, _raw(counts, nb, bs, ch, good, 0)[1])
    assert _raw(counts, nb, bs, ch, good, 0, costs=False)[0] == 0
    bad_lists = [[], [CAND(WORD, 11)], [CAND(WORD, 13)], [CAND(BYTE, 16)], [CAND(ALIAS, 16)], [CAND(RANS64, 16)],
                 [CAND(BYTE, 7)], [CAND(4, 12)], [CAND(BYTE, 14), CAND(BYTE, 14)],
                 [CAND(BYTE, sb) for sb in range(8, 16)] + [CAND(RANS64, sb) for sb in range(8, 16)] + [CAND(WORD, 12)]]
    for cands in bad_lists:
        assert _raw(counts, nb, bs, ch, cands, 0)[0] == -1, cands
    assert _raw(counts, nb, bs, ch, good, 10 ** 6 + 1)[0] == -1
    assert _raw(counts, nb, bs, ch, good, 0, chosen=False)[0] == -1
    assert _raw(np.zeros(0, np.uint32), nb, bs, ch, good, 0)[0] == -1
    for g in ((0, bs, ch), (nb, 0, ch), (nb, bs, 31), (nb, bs, 1000), (nb, 33 * 32, 32), (nb, bs, 1 << 25)):
        assert _raw(counts, *g, good, 0)[0] == -1, g
    for b, d in ((0, 1), (1, -1)):                                 # a row that does not sum to block_size
        bad = counts.astype(np.int64)
        bad[b, int(np.argmax(bad[b]))] += d
        assert _raw(bad, nb, bs, ch, good, 0)[0] == -1, (b, d)
