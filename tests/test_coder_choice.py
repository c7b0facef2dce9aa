"""rb200_choose_coder: the coder-choice rule of rb200_container_model_encode_auto_async on the host.  Its costs and its
choice equal a Python statement of the rule (log2q by its definition, the models from the oracle's normalize_freqs) over
seeded histograms of many shapes, several candidate lists and tolerances from 0 to 10^6; argument errors are refused.
No GPU needed."""
import ctypes as C
import math

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

WORD, BYTE, ALIAS, RANS64 = api.CODER_WORD, api.CODER_BYTE, api.CODER_ALIAS, api.CODER_RANS64
CAND = api.CANDIDATE
INFEASIBLE = (1 << 64) - 1

LISTS = [
    [CAND(WORD, 12), CAND(ALIAS, 16)],
    [CAND(WORD, 12), CAND(BYTE, 14), CAND(RANS64, 16)],
    [CAND(BYTE, 16)],
    [CAND(BYTE, 16), CAND(ALIAS, 16), CAND(RANS64, 16)],
    [CAND(RANS64, 8), CAND(ALIAS, 10), CAND(BYTE, 15), CAND(WORD, 12), CAND(ALIAS, 13)],
    # sixteen: every byte scale_bits, three alias, three rans64, word
    [CAND(BYTE, sb) for sb in range(8, 17)] + [CAND(ALIAS, 12), CAND(ALIAS, 14), CAND(ALIAS, 16), CAND(RANS64, 8),
                                              CAND(RANS64, 14), CAND(RANS64, 16), CAND(WORD, 12)],
]
TOLERANCES = [0, 1, 20000, 300000, 10 ** 6]


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


def rule(oracle_lib, counts, n, chunk, cands, tol):
    """(index or None, costs): the rule as the header states it"""
    n_chunks = -(-n // chunk)
    costs = []
    for c in cands:
        coder, sb = c >> 8, c & 0xFF
        if n == 0:
            costs.append(INFEASIBLE)
            continue
        f, _ = oracle_lib.normalize_freqs(counts.astype(np.uint32), 1 << sb)
        if int(f.sum()) != 1 << sb or (coder == BYTE and int(f.max()) >= 65536):
            costs.append(INFEASIBLE)
            continue
        bits_q = sum(int(counts[s]) * ((sb << 16) - log2q(int(f[s]))) for s in range(256) if counts[s])
        costs.append(-(-bits_q // (1 << 19)) + n_chunks * (256 if coder == RANS64 else 128))
    lo = min(costs)
    if lo == INFEASIBLE:
        return None, costs
    bound = lo + lo * tol // 10 ** 6
    return next(i for i, c in enumerate(costs) if c <= bound), costs


def _counts(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        data = rng.integers(0, 256, n)
    elif kind == "zipf":
        p = 1.0 / np.arange(1, 257) ** 1.1
        data = rng.permutation(256)[rng.choice(256, n, p=p / p.sum())]
    elif kind.startswith("skew"):                    # one symbol at p, a Zipf tail over the other 255
        p_top = float(kind[4:])
        tail = 1.0 / np.arange(1, 256) ** 1.1
        p = np.concatenate([[p_top], (1 - p_top) * tail / tail.sum()])
        data = rng.choice(256, n, p=p)
    elif kind == "two":
        data = np.where(rng.random(n) < 0.01, 7, 200)
    elif kind == "one":
        data = np.full(n, 0x41)
    else:
        raise ValueError(kind)
    return np.bincount(data, minlength=256).astype(np.uint64)


KINDS = ["uniform", "zipf", "skew0.9", "skew0.99", "skew0.999", "two", "one"]
GEOMETRIES = [(1, 32), (1000, 32), (100_003, 4096), (1 << 20, 8192), (3_000_001, 1 << 24)]


def _check(oracle_lib, counts, n, chunk):
    for cands in LISTS:
        for tol in TOLERANCES:
            want_i, want_costs = rule(oracle_lib, counts, n, chunk, cands, tol)
            if want_i is None:
                with pytest.raises(api.RansError) as e:
                    api.choose_coder(counts, n, chunk, cands, tol)
                assert e.value.code == -2
                continue
            i, costs = api.choose_coder(counts, n, chunk, cands, tol)
            assert [int(c) for c in costs] == want_costs, (n, chunk, cands, tol)
            assert i == want_i, (n, chunk, cands, tol, costs)


@pytest.mark.parametrize("kind", KINDS)
def test_matches_the_rule(oracle_lib, kind):
    for k, (n, chunk) in enumerate(GEOMETRIES):
        _check(oracle_lib, _counts(kind, n, seed=17 * k + 3), n, chunk)


def test_matches_the_rule_on_book1(oracle_lib, book1):
    counts = np.bincount(book1, minlength=256).astype(np.uint64)
    for chunk in (32, 8192):
        _check(oracle_lib, counts, book1.size, chunk)


def test_log2q_is_log2():
    """the fixed-point log2 stays within one unit in the last place of log2 over every frequency a model can hold"""
    for f in range(1, 65537):
        assert abs(log2q(f) / 65536.0 - math.log2(f)) < 2.0 / 65536, f


def test_choice_follows_the_data(oracle_lib):
    """uniform bytes keep the word coder first in the list; at p = 0.99 alias at 16 wins by far more than 2 %; a
    tolerance of 10^6 keeps the first feasible candidate; the byte coder at 16 is infeasible on one symbol"""
    n, chunk = 1 << 20, 8192
    pair = [CAND(WORD, 12), CAND(ALIAS, 16)]
    assert api.choose_coder(_counts("uniform", n, 1), n, chunk, pair, 20000)[0] == 0
    i, costs = api.choose_coder(_counts("skew0.99", n, 2), n, chunk, pair, 20000)
    assert i == 1 and costs[1] < 0.9 * costs[0]
    assert api.choose_coder(_counts("skew0.99", n, 2), n, chunk, pair, 10 ** 6)[0] == 0
    i, costs = api.choose_coder(_counts("one", n, 3), n, chunk, [CAND(BYTE, 16), CAND(BYTE, 15)])
    assert i == 1 and int(costs[0]) == INFEASIBLE


def test_no_feasible_candidate():
    lib = rb.load()
    counts = np.zeros(256, np.uint64)
    counts[9] = 5000
    cands = np.array([CAND(BYTE, 16)], np.uint32)
    costs = np.zeros(1, np.uint64)
    chosen = C.c_uint32(77)
    rc = lib.dll.rb200_choose_coder(counts.ctypes.data_as(api._u64p), 5000, 4096, cands.ctypes.data_as(api._u32p), 1, 0,
                                    costs.ctypes.data_as(api._u64p), C.byref(chosen))
    assert rc == -2 and int(costs[0]) == INFEASIBLE and chosen.value == 77
    # n == 0: nothing to model
    zero = np.zeros(256, np.uint64)
    cands = np.array([CAND(WORD, 12), CAND(RANS64, 14)], np.uint32)
    costs = np.zeros(2, np.uint64)
    rc = lib.dll.rb200_choose_coder(zero.ctypes.data_as(api._u64p), 0, 4096, cands.ctypes.data_as(api._u32p), 2, 0,
                                    costs.ctypes.data_as(api._u64p), C.byref(chosen))
    assert rc == -2 and all(int(c) == INFEASIBLE for c in costs) and chosen.value == 77


def test_argument_errors():
    lib = rb.load()
    n = 100_000
    counts = _counts("zipf", n, 5)
    good = [CAND(WORD, 12), CAND(ALIAS, 16)]
    chosen = C.c_uint32(0)

    def call(cands, tol=0, cnt=counts, n_=n, chunk=4096, costs=True, chosen_p=True, count=None):
        c = np.array(cands, np.uint32)
        out = np.zeros(max(c.size, 1), np.uint64)
        return lib.dll.rb200_choose_coder(None if cnt is None else cnt.ctypes.data_as(api._u64p), n_, chunk,
                                          c.ctypes.data_as(api._u32p) if c.size else None, c.size if count is None else count, tol,
                                          out.ctypes.data_as(api._u64p) if costs else None, C.byref(chosen) if chosen_p else None)

    assert call(good) == 0
    assert call(good, costs=False) == 0                                  # costs may be NULL
    bad_pairs = [CAND(WORD, 14), CAND(WORD, 8), CAND(BYTE, 7), CAND(ALIAS, 17), CAND(RANS64, 17), CAND(4, 12),
                 (1 << 16) | CAND(WORD, 12), CAND(255, 12)]
    for pair in bad_pairs:
        assert call([CAND(WORD, 12), pair]) == -1, hex(pair)
    assert call([]) == -1                                                # empty list
    assert call(good, count=0) == -1
    assert call([CAND(BYTE, sb) for sb in range(8, 17)] + [CAND(ALIAS, sb) for sb in range(8, 16)]) == -1     # 17 candidates
    assert call([CAND(WORD, 12), CAND(ALIAS, 16), CAND(WORD, 12)]) == -1  # a duplicate
    assert call(good, tol=10 ** 6) == 0
    assert call(good, tol=10 ** 6 + 1) == -1
    assert call(good, chunk=16) == -1 and call(good, chunk=(1 << 24) + 1) == -1
    assert call(good, chunk=32) == 0 and call(good, chunk=1 << 24) == 0
    assert call(good, n_=n + 1) == -1                                    # counts do not sum to n
    assert call(good, cnt=None) == -1 and call(good, chosen_p=False) == -1
    big = np.zeros(256, np.uint64)
    big[0], big[1] = 1 << 31, 1 << 31
    assert call(good, cnt=big, n_=1 << 32) == -1                         # n >= 2^32
