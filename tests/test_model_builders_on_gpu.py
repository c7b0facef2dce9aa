"""Every model, table and coder-choice builder that runs on the GPU, compared table by table with its host twin over a
seeded corpus of crafted models.

The enqueue-only calls build their models and tables on the GPU with parallel restatements of sequential host loops:
block_normalize (normalize_freqs on one warp), the alias_remap slots of container_model_kernel, the slot and cum2sym
searches of container_table_kernel, block_fill_slots and block_coder_decode_table, block_build_enc_table's exactness
test, and coder_choice_kernel's rule.  A stream reads only the entries its symbols visit, so the stream tests cannot see
a wrong entry elsewhere.  Here every entry is compared, bit for bit, with model_host.cpp's tables (build_*_device_tables,
the images rb200_model_create uploads), the oracle's normalize_freqs and rb200_choose_coder.

tests/model_device/builders.cu is compiled here (NVCC_FLAGS, model_host.cpp linked in for the host twins).  It launches
the shipped __global__ kernels unchanged on workspaces it fills, and calls the shipped __device__ builders from batch
kernels, one CTA per model, with their callers' shared arrays and blockDim.  block_coder_encode_kernel packs its table
inline, so it cannot be reached without a copy of that code; its per-block streams are compared with the oracle by
test_gpu_blocks_coder.py.

The corpus is built here, seeded: raw count vectors (normalised by the builders) and normalised tables for every
scale_bits each builder takes, with the edges listed in _raw_corpus and _tables.  test_corpus_reaches_every_branch (no
GPU) states normalize_freqs and the alias pairing in Python, checks them against the oracle on the whole corpus, and
counts the branches the corpus takes, so that an edit of the corpus cannot quietly lose an edge.
"""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "model_device")
WORD, BYTE, ALIAS, RANS64 = orc.CODER_WORD, orc.CODER_BYTE, orc.CODER_ALIAS, orc.CODER_RANS64
U32MAX = (1 << 32) - 1
INFEASIBLE = (1 << 64) - 1
WORD_GATE_CLOSED = 2

SINGLE_ROWS = [(WORD, 12)] + [(c, sb) for c in (ALIAS, BYTE, RANS64) for sb in range(8, 17)]
BLOCK_SB = list(range(8, 16))


# ------------------------------------------------------------------------------------------------------------ corpus

def _fit(counts, total):
    """counts (float or int shape) scaled to sum exactly `total`, every nonzero entry kept nonzero"""
    c = np.asarray(counts, dtype=np.float64)
    nz = c > 0
    out = np.zeros(256, np.int64)
    out[nz] = np.maximum(1, np.floor(c[nz] / c.sum() * (total - nz.sum()))).astype(np.int64)
    out[np.argmax(c)] += total - int(out.sum())
    assert out.min() >= 0 and int(out.sum()) == total
    return out


@functools.lru_cache(maxsize=None)
def _raw_corpus():
    """[(name, counts)]: 256 raw counts (np.int64), each sum in [1, 2^32 - 1]"""
    rng = np.random.default_rng(0x5EED)
    out = []

    def add(name, c):
        c = np.asarray(c, dtype=np.int64)
        assert c.shape == (256,) and c.min() >= 0 and 1 <= int(c.sum()) <= U32MAX, name
        out.append((name, c))

    # Dirichlet over 1..256 symbols, from very skewed (alpha 0.01) to flat (alpha 10), totals from 1 to 2^32 - 1
    for i in range(180):
        k = int(rng.choice([1, 2, 3, 5, 8, 16, 40, 100, 200, 255, 256])) if i % 2 else int(rng.integers(1, 257))
        alpha = 10 ** rng.uniform(-2, 1)
        n = int(min(U32MAX, max(1, 10 ** rng.uniform(0, np.log10(U32MAX)))))
        p = np.zeros(256)
        p[rng.choice(256, k, replace=False)] = rng.dirichlet(np.full(k, alpha))
        c = rng.multinomial(n, p / p.sum())
        add(f"dirichlet{i}", c)
    # a single symbol, at either end and in the middle
    for s in (0, 255, 128, 77):
        for cnt in (1, 1000, U32MAX):
            c = np.zeros(256, np.int64)
            c[s] = cnt
            add(f"single{s}x{cnt}", c)
    # one dominant symbol and 255 at count 1
    for dom in (0, 0x41, 255):
        for cnt in (300, 100_000, U32MAX - 255):
            c = np.ones(256, np.int64)
            c[dom] = cnt
            add(f"dominant{dom}x{cnt}", c)
    # all counts equal, over all 256 symbols and over subsets
    for cnt in (1, 7, (1 << 24) - 1, U32MAX // 256):
        add(f"equal{cnt}", np.full(256, cnt))
    for k in (2, 17, 100):
        c = np.zeros(256, np.int64)
        c[rng.choice(256, k, replace=False)] = 1000
        add(f"equal_subset{k}", c)
    # powers of two, with zeros
    for i in range(8):
        c = (1 << rng.integers(0, 23, 256)) * (rng.random(256) < 0.7)
        c[rng.integers(256)] = 1 << 24
        add(f"pow2_{i}", c)
    # zero-count runs at both ends and between the symbols that occur
    for i, (lo, hi, step) in enumerate([(10, 246, 1), (0, 40, 3), (200, 256, 5), (64, 192, 7)]):
        c = np.zeros(256, np.int64)
        c[lo:hi:step] = rng.integers(1, 1 << 20, len(range(lo, hi, step)))
        add(f"gaps{i}", c)
    # squash-heavy: count-1 symbols among a few donors of equal count, so that the squashed symbols steal from
    # equal-width donors below and above them; totals up to 2^32 - 1
    for i, donors in enumerate([(5, 250), (0, 128, 255), (100, 101), (30, 60, 90, 120, 150, 180, 210, 240), (255,), (0,)]):
        for total in (1 << 20, 1 << 27, U32MAX):
            c = np.ones(256, np.int64)
            d = np.array(donors)
            rest = total - (256 - d.size)
            c[d] = rest // d.size
            c[d[0]] += rest - c[d].sum()
            add(f"squash{i}_{total}", c)
    # many medium donors next to many count-1 takers: donors of width 2 tie all the time
    for i in range(10):
        c = np.ones(256, np.int64)
        med = rng.choice(256, int(rng.integers(20, 120)), replace=False)
        c[med] = int(rng.integers(3, 9)) * (1 << int(rng.integers(8, 20)))
        add(f"medium{i}", c)
    # count sums of exactly 2^32 - 1 and just below it, skewed
    for i, total in enumerate([U32MAX, U32MAX, U32MAX - 1, U32MAX - 1, U32MAX - 255, U32MAX - 4096]):
        p = 1.0 / np.arange(1, 257) ** (0.8 + 0.4 * i)
        p[rng.random(256) < 0.3] *= 1e-7
        add(f"near32_{i}", _fit(rng.permutation(p), total))
    return out


def _compositions(rng, M, k):
    """k positive parts summing to M, on k random symbols"""
    f = np.zeros(256, np.int64)
    syms = rng.choice(256, k, replace=False)
    f[syms] = 1 + rng.multinomial(M - k, rng.dirichlet(np.full(k, 10 ** rng.uniform(-1.5, 1))))
    return f


@functools.lru_cache(maxsize=None)
def _constructed(sb):
    """normalised tables at 1 << sb built directly: [(name, freqs)]"""
    M, b = 1 << sb, 1 << (sb - 8)
    rng = np.random.default_rng(1000 + sb)
    out = []

    def add(name, f):
        f = np.asarray(f, dtype=np.int64)
        assert f.shape == (256,) and f.min() >= 0 and int(f.sum()) == M, (name, sb)
        out.append((name, f))

    for s in (0, 255, 128):                                  # a single symbol with f = M
        f = np.zeros(256, np.int64)
        f[s] = M
        add(f"single{s}", f)
    for dom in (0, 200, 255):                                # one dominant symbol and 255 at frequency 1
        f = np.ones(256, np.int64)
        f[dom] = M - 255
        add(f"dominant{dom}", f)
    add("equal", np.full(256, b))
    for i in range(12):                                      # powers of two: M split in halves, on random symbols
        parts = [M]
        for _ in range(int(rng.integers(1, 120))):
            j = int(rng.integers(len(parts)))
            if parts[j] > 1:
                parts[j] //= 2
                parts.append(parts[j])
        f = np.zeros(256, np.int64)
        f[rng.choice(256, len(parts), replace=False)] = parts
        add(f"pow2_{i}", f)
    for i, s in enumerate((0, 100, 254)):                    # M / 2 next to smaller symbols
        f = np.zeros(256, np.int64)
        f[s], f[s + 1] = M // 2, M // 4
        others = rng.choice(np.setdiff1d(np.arange(256), [s, s + 1]), 30, replace=False)
        f[others] = np.bincount(rng.integers(0, 30, M // 4 - 30), minlength=30) + 1
        add(f"half{i}", f)
    for i, (lo, hi, step) in enumerate([(20, 236, 1), (0, 60, 2), (190, 256, 3), (50, 200, 9)]):   # zero-width runs
        f = np.zeros(256, np.int64)
        syms = np.arange(lo, hi, step)
        f[syms] = 1 + rng.multinomial(M - syms.size, np.full(syms.size, 1.0 / syms.size))
        add(f"gaps{i}", f)
    for i in range(10):                                      # alias: exact multiples of the bucket
        parts = 1 + rng.multinomial(256 - (k := int(rng.integers(1, 200))), np.full(k, 1.0 / k))
        f = np.zeros(256, np.int64)
        f[rng.choice(256, k, replace=False)] = parts * b
        add(f"buckets{i}", f)
    for i in range(6):                                       # alias: alternately under- and over-full
        d = int(rng.integers(1, b)) if b > 1 else 1
        f = np.where(np.arange(256) % 2 == 0, b - d, b + d) if i % 2 == 0 else np.where(np.arange(256) % 2 == 0, b + d, b - d)
        if i >= 2:                                           # blocks of under-full then over-full runs
            run = 1 + i
            f = np.where((np.arange(256) // run) % 2 == 0, b - d, b + d)
            f[-1] += M - int(f.sum())
            if f[-1] < 0:
                continue
        add(f"alternate{i}", f)
    for i in range(6):                                       # descending: donors ahead of the takers they fill
        p = np.sort(rng.dirichlet(np.full(256, 0.3)))[::-1]
        add(f"descending{i}", _fit(p + 1e-9, M))
    if M >= 4096:                                            # the word coder's r32 boundary and its wide model
        for big in (2963, 2964, 4095, 4096):
            for s in (0, 9, 255):
                f = np.zeros(256, np.int64)
                f[s] = big
                rest = 4096 - big
                if rest:
                    others = np.setdiff1d(np.arange(256), [s])[: min(rest, 40)]
                    f[others] = np.bincount(np.arange(rest) % others.size, minlength=others.size)
                f[s] += M - 4096
                add(f"word{big}at{s}", f)
    for i in range(40):                                      # random tables over 1..256 symbols
        add(f"random{i}", _compositions(rng, M, int(rng.integers(1, 257))))
    return out


@functools.lru_cache(maxsize=None)
def _tables(sb):
    """the normalised corpus at 1 << sb: every raw count vector normalised by the oracle, then the constructed tables"""
    lib = orc.Oracle()
    out = [(name, lib.normalize_freqs(c.astype(np.uint32), 1 << sb)[0].astype(np.int64)) for name, c in _raw_corpus()]
    return out + _constructed(sb)


def _invalid(coder, sb):
    """[(name, freqs as u32)]: models container_table_kernel must flag (bad or refused), never read past"""
    M = 1 << sb
    out = []
    f = np.zeros(256, np.int64)
    f[3], f[40] = M // 2, M // 2 + 1
    out.append(("sum+1", f))
    f = np.zeros(256, np.int64)
    f[3], f[40] = M // 2, M // 2 - 1
    out.append(("sum-1", f))
    f = np.zeros(256, np.int64)
    f[7] = M + 1
    out.append(("above_M", f))
    f = np.zeros(256, np.int64)                              # a frequency above M whose u32 sum wraps to exactly M
    f[0], f[1] = U32MAX, M + 1
    out.append(("above_M_wrapped", f))
    f = np.zeros(256, np.int64)
    f[255] = U32MAX
    f[254] = 1
    out.append(("wrap_to_zero", f))
    if coder == BYTE and sb == 16:
        for s in (0, 255):
            f = np.zeros(256, np.int64)
            f[s] = 65536
            out.append((f"byte65536at{s}", f))
    return [(n, x.astype(np.uint64).astype(np.uint32)) for n, x in out]


# ------------------------------------------------------------------ Python statements of the builders (coverage)

def py_normalize(counts, M, tally):
    """normalize_freqs (main.cpp:68-129) on widths, counting the branches of the squashed-symbol steal"""
    raw = np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=object))])
    total = int(raw[-1])
    cum = np.array([M * int(x) // total for x in raw], dtype=np.int64)
    w = np.diff(cum)
    for s in range(256):
        if counts[s] == 0 or w[s] > 0:
            continue
        m = w[w > 1].min()
        ties = np.flatnonzero(w == m)
        victim = int(ties[0])                                # lowest index on ties
        tally["tie"] += ties.size > 1
        tally["below" if victim < s else "above"] += 1
        w[victim] -= 1
        w[s] += 1
    return w


def py_alias(freqs, bucket, tally):
    """make_alias_table's pairing and slot hand-out (main_alias.cpp:147-237): (divider, slot_adjust, slot_freqs,
    sym_id, remap), counting the branches of the pairing"""
    f = [int(x) for x in freqs]
    rest, divider, sym_id = f[:], [bucket] * 256, [s // 2 for s in range(512)]
    tally["exact"] += sum(x == bucket for x in f)
    donor = next((s for s in range(256) if rest[s] >= bucket), 256)
    taker = next((s for s in range(256) if rest[s] < bucket), 256)
    resume = taker + 1
    while donor < 256 and taker < 256:
        sym_id[2 * taker] = donor
        divider[taker] = rest[taker]
        rest[donor] -= bucket - divider[taker]
        tally["full"] += rest[donor] == bucket and resume > donor       # only >= (not >) keeps it off :199
        if rest[donor] >= bucket or resume <= donor:
            tally["resume"] += 1
            taker = resume
            while taker < 256 and rest[taker] >= bucket:
                taker += 1
            resume = taker + 1
        else:
            tally["behind"] += 1                             # :199, the donor became a taker behind us
            taker = donor
        while donor < 256 and rest[donor] < bucket:
            donor += 1
    cum = np.concatenate([[0], np.cumsum(f)])
    given = [0] * 256
    div, adj, sf = [0] * 256, [0] * 512, [0] * 512
    remap = np.zeros(int(cum[-1]), np.int64)
    for s in range(256):
        other, own = sym_id[2 * s], divider[s]
        lent, lo = bucket - own, s * bucket
        div[s] = lo + own
        sf[2 * s + 1], sf[2 * s] = f[s], f[other]
        adj[2 * s + 1] = (lo - given[s]) & U32MAX
        adj[2 * s] = (lo - (given[other] - own)) & U32MAX
        remap[cum[s] + given[s]: cum[s] + given[s] + own] = np.arange(lo, lo + own)
        given[s] += own
        remap[cum[other] + given[other]: cum[other] + given[other] + lent] = np.arange(lo + own, lo + bucket)
        given[other] += lent
    assert given == f
    return np.array(div), np.array(adj), np.array(sf), np.array(sym_id), remap


# per scale_bits, how many models of the corpus must take each branch: a steal from a donor below / above the squashed
# symbol, an arg-min tie broken by the lowest index; the pairing's :199 (the donor became a taker behind us) and its
# resume branch, a donor left exactly full while takers ahead remain, a symbol whose frequency is exactly one bucket
MIN_HITS = {"below": 40, "above": 40, "tie": 25, "behind": 100, "resume": 100, "full": 100, "exact": 15}


def test_corpus_reaches_every_branch(oracle_lib):
    """the Python statements equal the oracle on the whole corpus, and the corpus takes every branch of the squashed-
    symbol steal and of the alias pairing, at every scale_bits, at least MIN_HITS times"""
    for sb in range(8, 17):
        M = 1 << sb
        tally = dict.fromkeys(MIN_HITS, 0)
        for name, c in _raw_corpus():
            one = dict.fromkeys(MIN_HITS, 0)
            want, _ = oracle_lib.normalize_freqs(c.astype(np.uint32), M)
            assert np.array_equal(py_normalize(c, M, one), want), (name, sb)
            for k in tally:
                tally[k] += one[k] > 0
        for name, f in _tables(sb):
            one = dict.fromkeys(MIN_HITS, 0)
            f32 = f.astype(np.uint32)
            cum = np.concatenate([[0], np.cumsum(f32)]).astype(np.uint32)
            want = oracle_lib.alias_build(f32, cum)
            got = py_alias(f32, M // 256, one)
            for k, (g, w) in enumerate(zip(got, want)):
                assert np.array_equal(g, w.astype(np.int64)), (name, sb, k)
            for k in tally:
                tally[k] += one[k] > 0
        low = {k: v for k, v in tally.items() if v < MIN_HITS[k]}
        assert not low, (sb, tally)


def test_corpus_sizes():
    """several hundred models per builder and scale_bits, every one well-formed"""
    assert len(_raw_corpus()) >= 250
    for sb in range(8, 17):
        assert len(_tables(sb)) >= 300, sb


# -------------------------------------------------------------------------------------------------- the harness

SIGS = {
    "md_model": "IPPIPPi", "md_choice": "IPPPP", "md_table": "IPLP", "md_block_build": "iIIPPPIPP",
    "md_fill_slots": "IIPPP", "md_enc_table": "IIPPP", "md_enc_expand": "IPPP", "md_coder_decode_table": "IIIIPPP",
    "hw_word": "PPPPP", "hw_alias": "PIPPP", "hw_byte": "PIPP", "hw_rans64": "PIPP", "hw_model_ok": "IIP",
    "hw_model_decodable": "IP", "rb200_normalize_freqs": "PPI",
}
CT = {"I": C.c_uint32, "i": C.c_int, "L": C.c_uint64, "P": C.c_void_p}


class Harness:
    def __init__(self, path):
        import torch
        self.torch = torch
        self.dll = C.CDLL(path)
        for name, sig in SIGS.items():
            f = getattr(self.dll, name)
            f.restype = C.c_int
            f.argtypes = [CT[c] for c in sig]
        self.dll.md_layout.restype = C.c_uint64
        self.dll.md_layout.argtypes = [C.c_int]
        L = [int(self.dll.md_layout(k)) for k in range(25)]
        (self.mw_size, self.mw_counts, self.mw_freqs, self.mw_r32, self.mw_word_enc, self.mw_word_enc32, self.mw_alias_enc,
         self.mw_byte_enc, self.mw_r64_enc, self.mw_remap, self.mw_choice, self.mw_cand, self.cw_size, self.cw_ok, self.cw_bad,
         self.cw_coder, self.cw_sb, self.cw_wide, self.cw_refused, self.cw_table, self.choice_costs, self.enc_replicas,
         self.r64_replicas, self.stat_model, self.max_cands) = L

    def call(self, name, *args):
        args = [a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data if isinstance(a, np.ndarray) else a for a in args]
        rc = getattr(self.dll, name)(*args)
        if name.startswith("md_"):
            assert rc == 0, f"{name}: CUDA error {rc}"
        return rc

    def dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy()).cuda()

    def zeros(self, nbytes):
        return self.torch.zeros(nbytes, dtype=self.torch.uint8, device="cuda")

    # ---- host twins: (rc, tables)
    def host(self, coder, sb, f):
        f = np.ascontiguousarray(f, dtype=np.uint32)
        M = 1 << sb
        if coder == WORD:
            dec, enc, enc32, flags = np.zeros(4096, np.uint32), np.zeros(512, np.uint32), np.zeros(512, np.uint32), np.zeros(2, np.int32)
            rc = self.call("hw_word", f, dec, enc, enc32, flags)
            return rc, dict(dec=dec.view(np.uint8), enc=enc, enc32=enc32, wide=int(flags[0]), enc32_ok=int(flags[1]))
        if coder == ALIAS:
            dec, enc, remap = np.zeros(1024, np.uint32), np.zeros(1024, np.uint32), np.zeros(M, np.uint16)
            rc = self.call("hw_alias", f, sb, dec, enc, remap)
            return rc, dict(dec=dec.view(np.uint8), enc=enc, remap=remap)
        if coder == BYTE:
            dec, enc = np.zeros(M + 1024, np.uint8), np.zeros(1024, np.uint32)
            rc = self.call("hw_byte", f, sb, dec, enc)
            return rc, dict(dec=dec, enc=enc)
        dec, enc = np.zeros(M + 2048, np.uint8), np.zeros(2048, np.uint32)
        rc = self.call("hw_rans64", f, sb, dec, enc)
        return rc, dict(dec=dec, enc=enc)

    def normalize(self, counts, M):
        f = np.ascontiguousarray(counts, dtype=np.uint32).copy()
        cum = np.zeros(257, np.uint32)
        assert self.call("rb200_normalize_freqs", f, cum, M) == 0
        return f


@pytest.fixture(scope="module")
def hx(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from ryg_rans_b200.build import NVCC_FLAGS, _nvcc
    out = str(tmp_path_factory.mktemp("model_device") / "libbuilders.so")
    subprocess.check_call([_nvcc(), *NVCC_FLAGS, "-shared", "-o", out, os.path.join(SRC, "builders.cu"),
                           os.path.join(ROOT, "ryg_rans_b200", "csrc", "model_host.cpp")])
    return Harness(out)


def _u32(a, off, nbytes):
    """a (models x bytes) u8 array: bytes [off, off + nbytes) of every row as u32"""
    return np.ascontiguousarray(a[:, off:off + nbytes]).view(np.uint32)


def _model_work(hx, counts_list):
    """a device array of ModelAsyncWork, one per counts vector, counts filled"""
    n = len(counts_list)
    w = np.zeros((n, hx.mw_size), np.uint8)
    w[:, hx.mw_counts:hx.mw_counts + 2048] = np.asarray(counts_list, dtype=np.uint64).view(np.uint8).reshape(n, 2048)
    return hx.dev(w)


def _check_tables(hx, coder, sb, r32_allowed, got, i, host, ctx):
    """row i of a read-back ModelAsyncWork array against the host tables of its model"""
    if coder == WORD:
        assert np.array_equal(_u32(got, hx.mw_word_enc, 2048)[i], host["enc"]), ctx
        assert np.array_equal(_u32(got, hx.mw_word_enc32, 2048)[i], host["enc32"]), ctx
        assert _u32(got, hx.mw_r32, 4)[i, 0] == int(bool(host["enc32_ok"]) and bool(r32_allowed)), ctx
    elif coder == ALIAS:
        assert np.array_equal(_u32(got, hx.mw_alias_enc, 4096)[i], host["enc"]), ctx
        remap = np.ascontiguousarray(got[i, hx.mw_remap:hx.mw_remap + 2 * (1 << sb)]).view(np.uint16)
        assert np.array_equal(remap, host["remap"]), ctx
    elif coder == BYTE:
        assert np.array_equal(_u32(got, hx.mw_byte_enc, 4096)[i], host["enc"]), ctx
    else:
        assert np.array_equal(_u32(got, hx.mw_r64_enc, 8192)[i], host["enc"]), ctx


# ------------------------------------------------------------------------------- 1 + 2: container_model_kernel

@pytest.mark.gpu
@pytest.mark.parametrize("coder,sb", SINGLE_ROWS)
def test_container_model_kernel(hx, oracle_lib, coder, sb):
    """container_model_kernel<false, false> on every raw count vector: its freqs equal the oracle's normalize_freqs and
    rb200_normalize_freqs; its encode tables (word: both reciprocal forms and r32 for both r32_allowed; alias: the entries
    and the whole alias_remap[0, M); byte; rans64's 8 words) equal build_*_device_tables'; kStatModel is set exactly when
    rb200_model_create refuses the model"""
    M = 1 << sb
    corpus = _raw_corpus()
    n = len(corpus)
    for r32_allowed in ((0, 1) if coder == WORD else (1,)):
        w = _model_work(hx, [c for _, c in corpus])
        status = hx.zeros(4 * n)
        hx.call("md_model", n, np.full(n, coder, np.uint32), np.full(n, sb, np.uint32), r32_allowed, w, status, 0)
        got = w.view(n, hx.mw_size).cpu().numpy()
        st = status.cpu().numpy().view(np.uint32)
        freqs = _u32(got, hx.mw_freqs, 1024)
        for i, (name, c) in enumerate(corpus):
            ctx = (name, coder, sb, r32_allowed)
            want, _ = oracle_lib.normalize_freqs(c.astype(np.uint32), M)
            assert np.array_equal(hx.normalize(c, M), want), ctx
            assert np.array_equal(freqs[i], want), ctx
            rc, host = hx.host(coder, sb, want)
            assert st[i] == (hx.stat_model if rc else 0), (ctx, st[i], rc)
            if rc == 0:
                _check_tables(hx, coder, sb, r32_allowed, got, i, host, ctx)


# ------------------------------------------------------------------------------------ 3: container_table_kernel

TABLE_ROWS = SINGLE_ROWS + [(WORD, 8), (WORD, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("coder,sb", TABLE_ROWS)
def test_container_table_kernel(hx, coder, sb):
    """container_table_kernel on every normalised table and the invalid models: the decode table (word dec[4096], alias
    dec[256], byte M + 1024 bytes, rans64 M + 2048 bytes) and `wide` equal the host images; `bad` is set exactly when
    container_model_ok fails and `refused` exactly when the model is well-formed but rb200_model_create refuses it"""
    M = 1 << sb
    models = ([] if coder == WORD and sb != 12 else [(n, f.astype(np.uint32)) for n, f in _tables(sb)]) + _invalid(coder, sb)
    if coder == WORD and sb != 12:                           # the word coder at scale_bits != 12: every model is bad
        models += [(n, f.astype(np.uint32)) for n, f in _tables(sb)[:50]]
    n, stride = len(models), 64 + 1024
    bufs = np.zeros((n, stride), np.uint8)
    for i, (_, f) in enumerate(models):
        bufs[i, 64:] = f.view(np.uint8)
    w = np.zeros((n, hx.cw_size), np.uint8)
    w[:, hx.cw_ok:hx.cw_ok + 4] = np.array([1], np.uint32).view(np.uint8)
    w[:, hx.cw_coder:hx.cw_coder + 4] = np.array([coder], np.uint32).view(np.uint8)
    w[:, hx.cw_sb:hx.cw_sb + 4] = np.array([sb], np.uint32).view(np.uint8)
    d_w = hx.dev(w)
    hx.call("md_table", n, hx.dev(bufs), stride, d_w)
    got = d_w.view(n, hx.cw_size).cpu().numpy()
    flags = {k: _u32(got, off, 4)[:, 0] for k, off in (("bad", hx.cw_bad), ("refused", hx.cw_refused), ("wide", hx.cw_wide))}
    n_valid = 0
    for i, (name, f) in enumerate(models):
        ctx = (name, coder, sb)
        ok = hx.call("hw_model_ok", coder, sb, f) != 0
        rc, host = hx.host(coder, sb, f) if ok else (-2, None)
        assert flags["bad"][i] == (not ok), ctx
        assert flags["refused"][i] == (ok and rc != 0), ctx
        if ok and not hx.call("hw_model_decodable", coder, f):
            assert flags["refused"][i] == 1, ctx
        if not ok or rc:
            assert flags["wide"][i] == 0, ctx
            continue
        n_valid += 1
        size = {WORD: 4 * 4096, ALIAS: 16 * 256, BYTE: M + 1024, RANS64: M + 2048}[coder]
        assert np.array_equal(got[i, hx.cw_table:hx.cw_table + size], host["dec"]), ctx
        assert flags["wide"][i] == (host["wide"] if coder == WORD else 0), ctx
    assert n_valid >= (0 if coder == WORD and sb != 12 else 250), n_valid


# ------------------------------------------------------------------------------------------ 4: per-block builders

@functools.lru_cache(maxsize=None)
def _blocks():
    """(data, offsets, sizes, counts): raw blocks of many shapes, sizes not multiples of 16, starts at every offset
    0..15 from a 16-byte boundary, so that both the head and the tail loops of the histograms run"""
    rng = np.random.default_rng(0xB10C)
    blocks = []
    for i in range(360):
        kind = i % 6
        size = int([rng.integers(1, 16), rng.integers(17, 600), rng.integers(1000, 70000)][i % 3])
        if size % 16 == 0:
            size += 1
        if kind == 0:                                        # Dirichlet over 1..256 symbols
            k = int(rng.integers(1, 257))
            p = np.zeros(256)
            p[rng.choice(256, k, replace=False)] = rng.dirichlet(np.full(k, 10 ** rng.uniform(-2, 1)))
            c = rng.multinomial(size, p / p.sum())
        elif kind == 1:                                      # one symbol
            c = np.zeros(256, np.int64)
            c[int(rng.choice([0, 255, 128]))] = size
        elif kind == 2 and size > 256:                       # one dominant symbol and 255 once
            c = np.ones(256, np.int64)
            c[int(rng.integers(256))] = size - 255
        elif kind == 3 and size > 300:                       # count-1 symbols among a few equal donors
            c = np.zeros(256, np.int64)
            takers = rng.choice(256, min(200, size // 2), replace=False)
            c[takers] = 1
            donors = np.setdiff1d(np.arange(256), takers)[:: max(1, (256 - takers.size) // 3)][:3]
            c[donors] = (size - takers.size) // donors.size
            c[donors[0]] += size - int(c.sum())
        else:                                                # flat
            c = rng.multinomial(size, np.full(256, 1.0 / 256))
        blocks.append(np.asarray(c, dtype=np.int64))
    data, offs, sizes = [], [], []
    pos = 0
    for i, c in enumerate(blocks):
        pad = (16 - pos % 16) % 16 + i % 16
        data.append(np.zeros(pad, np.uint8))
        pos += pad
        d = rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), c))
        data.append(d)
        offs.append(pos)
        sizes.append(d.size)
        pos += d.size
    data.append(np.zeros(16, np.uint8))
    return np.concatenate(data), np.array(offs, np.uint64), np.array(sizes, np.uint32), blocks


@pytest.mark.gpu
@pytest.mark.parametrize("variant,threads", [("block_model_build", 256), ("block_model_build_wide", 256),
                                             ("block_model_build_wide", 1024)])
def test_block_model_build(hx, oracle_lib, variant, threads):
    """block_model_build (8 warps) and block_model_build_wide (256 and 1024 threads) on raw block bytes: the u16 row
    equals the oracle's normalize_freqs of the block's counts for every target 1 << 8 .. 1 << 15, and the status word
    stays clear (normalisation cannot fail for targets >= 256)"""
    data, offs, sizes, counts = _blocks()
    n = len(counts)
    for i, c in enumerate(counts):
        assert np.array_equal(np.bincount(data[int(offs[i]):int(offs[i]) + int(sizes[i])], minlength=256), c)
        assert int(offs[i]) % 16 == i % 16
    d_data, d_offs, d_sizes = hx.dev(data), hx.dev(offs), hx.dev(sizes)
    for sb in BLOCK_SB:
        rows, status = hx.zeros(512 * n), hx.zeros(4 * n)
        hx.call("md_block_build", int(variant.endswith("wide")), threads, n, d_data, d_offs, d_sizes, 1 << sb, rows, status)
        got = rows.cpu().numpy().view(np.uint16).reshape(n, 256)
        assert not status.cpu().numpy().any(), (variant, sb)
        for i, c in enumerate(counts):
            want, _ = oracle_lib.normalize_freqs(c.astype(np.uint32), 1 << sb)
            assert np.array_equal(got[i], want), (variant, threads, sb, i, int(sizes[i]), int(offs[i]) % 16)


def _rows(sb):
    """(u16 rows, expected block_prefix verdicts): every table of the corpus at 1 << sb, then rows that do not sum to it"""
    M = 1 << sb
    rows = [f for _, f in _tables(sb)]
    good = [True] * len(rows)
    for k, (a, b) in enumerate([(1, 0), (0, 1), (M, 1), (M - 1, 0)]):
        f = np.zeros(256, np.int64)
        f[k * 50] = a
        f[255 - k] += b + (M // 2 if a < M // 2 else 0)
        if int(f.sum()) == M:
            f[0] += 1
        rows.append(f)
        good.append(False)
    f = np.full(256, M // 256, np.int64)
    f[17] += 1
    rows.append(f)
    good.append(False)
    f = np.full(256, M // 256, np.int64)
    f[200] -= 1
    rows.append(f)
    good.append(False)
    return np.array(rows, dtype=np.uint16), np.array(good)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [128, 256, 512, 1024])
def test_block_fill_slots(hx, threads):
    """block_prefix + block_fill_slots at every blockDim it runs with (block_threads() and the planned decoder's 256):
    the slot table equals the host's word dec[4096] and `wide` the host's wide; rows that do not sum to 4096 are
    rejected"""
    rows, good = _rows(12)
    n = len(rows)
    tab, flags = hx.zeros(4 * 4096 * n), hx.zeros(8 * n)
    hx.call("md_fill_slots", threads, n, hx.dev(rows), tab, flags)
    tab = tab.cpu().numpy().view(np.uint32).reshape(n, 4096)
    flags = flags.cpu().numpy().view(np.uint32).reshape(n, 2)
    for i in range(n):
        assert flags[i, 0] == good[i], (threads, i)
        if good[i]:
            rc, host = hx.host(WORD, 12, rows[i].astype(np.uint32))
            assert rc == 0
            assert np.array_equal(tab[i], host["dec"].view(np.uint32)), (threads, i)
            assert flags[i, 1] == host["wide"], (threads, i)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [128, 256, 1024])
def test_block_build_enc_table(hx, threads):
    """block_prefix + block_build_enc_table: r32 equals the host's enc32_ok, and every replica of every symbol's entry
    equals word_enc_expand<r32> of the host's enc32 (r32) or enc entry; a rejected row gives the all-bad table"""
    rows, good = _rows(12)
    n = len(rows)
    host_e, host_r32 = np.zeros((n, 512), np.uint32), np.ones(n, np.uint32)
    host_e[:, 1::2] = 0x80000000                             # {0, kEncBadSymbol}: every symbol outside the model
    for i in np.flatnonzero(good):
        rc, host = hx.host(WORD, 12, rows[i].astype(np.uint32))
        assert rc == 0
        host_r32[i] = host["enc32_ok"]
        host_e[i] = host["enc32"] if host["enc32_ok"] else host["enc"]
    want = hx.zeros(16 * 256 * n)
    hx.call("md_enc_expand", n, hx.dev(host_e), hx.dev(host_r32), want)
    want = want.cpu().numpy().view(np.uint32).reshape(n, 256, 4)
    out, flags = hx.zeros(16 * 256 * hx.enc_replicas * n), hx.zeros(8 * n)
    hx.call("md_enc_table", threads, n, hx.dev(rows), out, flags)
    got = out.cpu().numpy().view(np.uint32).reshape(n, 256, hx.enc_replicas, 4)
    flags = flags.cpu().numpy().view(np.uint32).reshape(n, 2)
    assert host_r32.min() == 0 and host_r32[good].max() == 1             # both forms occur among the valid rows
    for i in range(n):
        assert flags[i, 0] == good[i] and flags[i, 1] == host_r32[i], (threads, i)
        for r in range(hx.enc_replicas):
            assert np.array_equal(got[i, :, r], want[i]), (threads, i, r)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [128, 256, 1024])
@pytest.mark.parametrize("coder", [BYTE, RANS64])
def test_block_coder_decode_table(hx, coder, threads):
    """block_prefix + block_coder_decode_table<BYTE | RANS64> at scale_bits 8..15: cum2sym and the symbol entries
    equal the host's decode image (rans64: every one of the kRans64DecReplicas copies); rows that do not sum to
    1 << sb are rejected and get no table"""
    for sb in BLOCK_SB:
        M = 1 << sb
        rows, good = _rows(sb)
        n = len(rows)
        sym_bytes = 1024 if coder == BYTE else 256 * hx.r64_replicas * 8
        out, ok = hx.zeros((M + sym_bytes) * n), hx.zeros(4 * n)
        hx.call("md_coder_decode_table", coder, sb, threads, n, hx.dev(rows), out, ok)
        got = out.cpu().numpy().reshape(n, M + sym_bytes)
        ok = ok.cpu().numpy().view(np.uint32)
        for i in range(n):
            ctx = (coder, sb, threads, i)
            assert ok[i] == good[i], ctx
            if not good[i]:
                continue
            rc, host = hx.host(coder, sb, rows[i].astype(np.uint32))
            assert rc == 0, ctx
            assert np.array_equal(got[i, :M], host["dec"][:M]), ctx
            if coder == BYTE:
                assert np.array_equal(got[i, M:], host["dec"][M:]), ctx
            else:
                syms = np.ascontiguousarray(got[i, M:]).view(np.uint32).reshape(256, hx.r64_replicas, 2)
                want = host["dec"][M:].view(np.uint32).reshape(256, 2)
                for r in range(hx.r64_replicas):
                    assert np.array_equal(syms[:, r], want), (ctx, r)


# ------------------------------------------------------------------------------------------ 5: coder_choice_kernel

VALID_PAIRS = [(WORD, 12)] + [(c, sb) for c in (BYTE, ALIAS, RANS64) for sb in range(8, 17)]
TOLERANCES = [0, 1, 20000, 10 ** 6]
CHUNKS = [32, 4096, 1 << 24]


def _choice_cases(oracle_lib):
    """[(counts, n, chunk, pairs, tol, want_index or None)]: corpus histograms with lists of 1..16 candidates, then
    constructed near-ties where a cost sits exactly at min + floor(min * tol / 10^6) or one above it"""
    from ryg_rans_b200 import api
    rng = np.random.default_rng(0xC401CE)
    corpus = _raw_corpus()
    cases = []
    for j, (name, c) in enumerate(corpus[::2]):
        for t, tol in enumerate(TOLERANCES):
            k = 1 + (4 * j + t) % 16
            idx = rng.choice(len(VALID_PAIRS), k, replace=False)
            pairs = [VALID_PAIRS[i] for i in idx]
            if np.count_nonzero(c) == 1 and (j + t) % 2 == 0:
                pairs[0] = (BYTE, 16)                        # infeasible on one symbol (a frequency of 65536)
                pairs = list(dict.fromkeys(pairs))
            cases.append((c, int(c.sum()), CHUNKS[(j + t) % 3], pairs, tol, None))
    for name, c in corpus:                                   # no feasible candidate at all
        if name.startswith("single"):
            cases.append((c, int(c.sum()), 4096, [(BYTE, 16)], 0, None))
    small = [c for _, c in corpus if 2000 <= c.sum() <= 900_000 and np.count_nonzero(c) > 1]
    ties = 0
    for c in small:
        n = int(c.sum())
        pairs = [VALID_PAIRS[i] for i in rng.choice(len(VALID_PAIRS), 6, replace=False)]
        _, costs = api.choose_coder(c, n, 4096, [api.CANDIDATE(*p) for p in pairs], 0)
        costs = [int(x) for x in costs]
        lo = min(costs)
        above = [i for i, x in enumerate(costs) if lo < x <= 2 * lo and x != INFEASIBLE]
        if not above or lo >= 10 ** 6:
            continue
        j = above[0]
        d = costs[j] - lo
        tol = -(-d * 10 ** 6 // lo)                          # the smallest tolerance whose bound reaches costs[j]
        assert lo + lo * tol // 10 ** 6 == costs[j] and lo + lo * (tol - 1) // 10 ** 6 == costs[j] - 1
        order = [pairs[j]] + [p for i, p in enumerate(pairs) if i != j]
        first_min = next(i for i, p in enumerate(order) if costs[pairs.index(p)] <= costs[j] - 1)
        cases.append((c, n, 4096, order, tol, 0))            # exactly at the bound: the first candidate
        cases.append((c, n, 4096, order, tol - 1, first_min))   # one above the bound: the next one within it
        ties += 1
    assert ties >= 20, ties
    return cases


@pytest.mark.gpu
def test_coder_choice_kernel(hx, oracle_lib):
    """coder_choice_kernel (list.n * 32 threads) on corpus histograms: every cand_freqs row equals normalize_freqs at its
    scale_bits; costs[0, n), index, coder, scale_bits and group equal rb200_choose_coder's (kStatModel and index 0 when
    no candidate is feasible), at tolerances 0, 1, 20000 and 10^6, small and large n_chunks, 1..16 candidates, and on
    near-ties.  Then container_model_kernel<false, true> builds the chosen row's tables from the record"""
    from ryg_rans_b200 import api
    cases = _choice_cases(oracle_lib)
    n = len(cases)
    lists = np.zeros((n, 2 * hx.max_cands + 2), np.uint32)
    n_chunks = np.zeros(n, np.uint64)
    rng = np.random.default_rng(5)
    groups = rng.integers(0, 1000, (n, hx.max_cands)).astype(np.uint32)
    for i, (c, total, chunk, pairs, tol, _) in enumerate(cases):
        lists[i, :len(pairs)] = [api.CANDIDATE(*p) for p in pairs]
        lists[i, hx.max_cands:2 * hx.max_cands] = groups[i]
        lists[i, -2:] = len(pairs), tol
        n_chunks[i] = -(-total // chunk)
    assert n_chunks.min() == 1 and n_chunks.max() > 1 << 20
    w = _model_work(hx, [c for c, *_ in cases])
    status = hx.zeros(4 * n)
    hx.call("md_choice", n, lists, n_chunks, w, status)
    got = w.view(n, hx.mw_size).cpu().numpy()
    st = status.cpu().numpy().view(np.uint32).copy()
    choice = _u32(got, hx.mw_choice, 16)
    costs = np.ascontiguousarray(got[:, hx.mw_choice + hx.choice_costs:hx.mw_choice + hx.choice_costs + 8 * hx.max_cands]).view(np.uint64)
    cand = _u32(got, hx.mw_cand, 1024 * hx.max_cands).reshape(n, hx.max_cands, 256)
    infeasible_seen = 0
    for i, (c, total, chunk, pairs, tol, want_i) in enumerate(cases):
        ctx = (i, pairs, tol, chunk)
        for k, (_, sb) in enumerate(pairs):
            assert np.array_equal(cand[i, k], oracle_lib.normalize_freqs(c.astype(np.uint32), 1 << sb)[0]), (ctx, k)
        try:
            index, want_costs = api.choose_coder(c, total, chunk, [api.CANDIDATE(*p) for p in pairs], tol)
        except api.RansError as e:
            assert e.code == -2
            index, want_costs = None, None
        if index is None:
            infeasible_seen += 1
            assert st[i] == hx.stat_model and choice[i, 2] == 0, ctx
            assert all(int(x) == INFEASIBLE for x in costs[i, :len(pairs)]), ctx
            index = 0
        else:
            assert st[i] == 0, ctx
            assert [int(x) for x in costs[i, :len(pairs)]] == [int(x) for x in want_costs], ctx
            assert choice[i, 2] == index, ctx
            if want_i is not None:
                assert index == want_i, ctx
        assert (choice[i, 0], choice[i, 1], choice[i, 3]) == (pairs[index][0], pairs[index][1], groups[i, index]), ctx
    assert infeasible_seen >= 8
    assert any(INFEASIBLE in [int(x) for x in costs[i, :len(p)]] for i, (_, _, _, p, _, _) in enumerate(cases))

    # the CHOSEN model kernel on the same workspaces
    for r32_allowed in (0, 1):
        w2 = hx.dev(got)
        hx.call("md_model", n, np.zeros(n, np.uint32), np.zeros(n, np.uint32), r32_allowed, w2, hx.dev(st), 1)
        g2 = w2.view(n, hx.mw_size).cpu().numpy()
        for i, (c, total, chunk, pairs, tol, _) in enumerate(cases):
            if st[i]:
                continue
            coder, sb = pairs[choice[i, 2]]
            f = _u32(g2, hx.mw_freqs, 1024)[i]
            assert np.array_equal(f, cand[i, choice[i, 2]]), i
            rc, host = hx.host(coder, sb, f)
            assert rc == 0, i
            _check_tables(hx, coder, sb, r32_allowed, g2, i, host, (i, coder, sb))
            if coder != WORD:
                assert _u32(g2, hx.mw_r32, 4)[i, 0] == WORD_GATE_CLOSED, i


# --------------------------------------------------------------------------------- 6: anchor to the shipped calls

ANCHOR_SB = {WORD: [12], ALIAS: list(range(8, 17)), BYTE: list(range(8, 17)), RANS64: list(range(8, 17))}


@pytest.mark.gpu
@pytest.mark.parametrize("coder", [WORD, ALIAS, BYTE, RANS64])
def test_shipped_calls_on_corpus_models(gpu_ctx, oracle_lib, coder):
    """about 20 corpus models per coder as data whose histogram is exactly the model's counts: the container of
    rb200_container_model_encode_async equals the oracle's byte for byte, and rb200_container_decode_async decodes the
    oracle's container back to the data (guards against drift between the harness build and the library)"""
    import torch
    from ryg_rans_b200 import api
    rng = np.random.default_rng(600 + coder)
    raw = [(n, c) for n, c in _raw_corpus() if c.sum() <= 3_000_000]
    picks = [raw[i] for i in rng.choice(len(raw), 12, replace=False)]
    sbs = ANCHOR_SB[coder]
    for k in range(10):
        sb = sbs[k % len(sbs)]
        tabs = _tables(sb)
        picks.append(tabs[len(_raw_corpus()) + int(rng.integers(len(tabs) - len(_raw_corpus())))])
    chunk = 4096
    for k, (name, counts) in enumerate(picks):
        sb = sbs[(k + 3) % len(sbs)] if k < 12 else sbs[(k - 12) % len(sbs)]
        if coder == BYTE and sb == 16 and np.count_nonzero(counts) == 1:
            sb = 15
        data = rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), counts))
        n = data.size
        freqs, cum = oracle_lib.model(data, sb)
        ob, oo = oracle_lib.chunked_encode(coder, data, freqs, cum, chunk, nlanes=32, scale_bits=sb)
        want = api.container_pack(coder, sb, chunk, n, freqs, oo, ob, 0)
        d_in = torch.from_numpy(data).cuda()
        cap = gpu_ctx.container_capacity(n, chunk)
        d_out = torch.full((cap,), 0xAA, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_model_encode_async(coder, sb, d_in.data_ptr(), n, chunk, 0, d_out.data_ptr(), cap)
        gpu_ctx.sync()
        assert np.array_equal(d_out[:want.size].cpu().numpy(), want), (name, coder, sb)
        d_buf = torch.from_numpy(want).cuda()
        d_dec = torch.full((n + 16,), 0x5C, dtype=torch.uint8, device="cuda")
        gpu_ctx.container_decode_async(d_buf.data_ptr(), want.size, d_dec.data_ptr(), n)
        gpu_ctx.sync()
        assert torch.equal(d_dec[:n], d_in) and bool((d_dec[n:] == 0x5C).all().item()), (name, coder, sb)
