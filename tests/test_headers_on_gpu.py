"""The source-level headers run inside CUDA kernels: every step function of rans_byte.h, rans64.h, rans_word_sse41.h
and rans_alias.h executed on the device and checked against exact arithmetic, the oracle and the host build.

A caller's kernel compiles these headers differently from a host program: RansEncPutSymbol takes `__umulhi`,
Rans64MulHi takes `__umul64hi`, the SSE4.1 section drops out, the `x / freq` / `x % freq` of the division forms become
nvcc's own division sequences, and the alias templates read `alias_remap` from device memory.  The library's own
kernels (csrc/) have their own step code, so nothing else in the suite runs this build.

tests/header_device/steps.inc holds the work items once; steps.cu runs them one thread per item and steps_host.cpp
(the host twin, g++) in a host loop.  Both are built here with -DNDEBUG (nvcc always defines `assert`, so the headers'
asserts would otherwise be live device traps); the test checks every precondition those asserts state before a call.
  A. symbol-init tables: RansEncSymbolInit / RansDecSymbolInit for every freq at scale_bits 1..16 and three starts,
     Rans64EncSymbolInit / Rans64DecSymbolInit likewise plus a sample at 17..31, RansWordTablesInitSymbol into a
     table in shared memory; field by field against the host twin and exact arithmetic, tables against the oracle;
  B. one encode step of every encoder at the edges of its range and across its renormalising branch, against numpy's
     exact uint64 arithmetic; plus a dense device sweep of the division-free steps at scale_bits 12 / 14 / 16;
  C. whole interleaved streams, one per thread, encoded with both encoder APIs and decoded with every decoder API:
     byte for byte against the host twin and the oracle, decoded symbols, bytes consumed and final states.
Every output region is fenced by sentinel bytes that are checked after each launch, regions have room for what any
32- or 64-bit state can emit, and a device decode only ever reads a stream already shown equal to the host twin's or
the oracle's, so a wrong header shows up as a failed comparison.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "header_device")
WORD, BYTE, ALIAS, RANS64 = orc.CODER_WORD, orc.CODER_BYTE, orc.CODER_ALIAS, orc.CODER_RANS64
SENT = 0xA5                    # sentinel fill of every output buffer
GUARD = 16                     # sentinel bytes around every region
BYTE_L, R64_L, WORD_L = 1 << 23, 1 << 31, 1 << 16
U64 = np.uint64

# step functions (body_step's `which`)
BYTE_PUT, BYTE_PUTSYM, R64_PUT, R64_PUTSYM, WORD_PUT, ALIAS_PUT = range(6)
STEPS = {"byte-RansEncPut": BYTE_PUT, "byte-RansEncPutSymbol": BYTE_PUTSYM, "rans64-Rans64EncPut": R64_PUT,
         "rans64-Rans64EncPutSymbol": R64_PUTSYM, "word-RansWordEncPut": WORD_PUT, "alias-RansEncPutAlias": ALIAS_PUT}
BYTE_LIKE = (BYTE_PUT, BYTE_PUTSYM, ALIAS_PUT)

# stream APIs
ENC_APIS = {"div": 0, "symbol": 1}
DEC_APIS = {"get+advance": 0, "advance_symbol": 1, "step+renorm": 2, "symbol_step+renorm": 3}
ALIAS_STATS = ("tables", "shuffled")
STREAM_CASES = ([("byte", sb) for sb in range(8, 17)] + [("alias", sb) for sb in range(8, 17)]
                + [("rans64", sb) for sb in list(range(8, 25)) + [28, 31]] + [("word", 12)])
MODELS = ("random", "ceiling", "pair", "single", "shift")
LANES = (1, 2, 8)
N_THREADS = 128

ENC32 = np.dtype([("x_max", "<u4"), ("rcp_freq", "<u4"), ("bias", "<u4"), ("cmpl_freq", "<u2"), ("rcp_shift", "<u2")])
DEC32 = np.dtype([("start", "<u2"), ("freq", "<u2")])
ENC64 = np.dtype([("rcp_freq", "<u8"), ("freq", "<u4"), ("bias", "<u4"), ("cmpl_freq", "<u4"), ("rcp_shift", "<u4")])
DEC64 = np.dtype([("start", "<u4"), ("freq", "<u4")])

# hd_<name>(uint64 n, ...): I = uint32, P = pointer
SIGS = {
    "byte_syms": "PPPPP", "rans64_syms": "PPPPP", "step": "IIPPPPPPP", "sweep": "IIIPP",
    "enc_byte": "III" + "PPP" + "PPP" + "PPP", "dec_byte": "III" + "PPP" + "PPPPPPP",
    "enc_rans64": "III" + "PPP" + "PPP" + "PPP", "dec_rans64": "III" + "PPP" + "PPPPPPP",
    "enc_word": "I" + "PPP" + "PP" + "PPP", "dec_word": "I" + "PP" + "PPPPPPP",
    "word_tables": "PPPP", "shuffle_alias": "PP",
    "enc_alias_tables": "II" + "PPP" + "P" + "PPP", "dec_alias_tables": "II" + "P" + "PPPPPPP",
    "enc_alias_shuffled": "II" + "PPP" + "P" + "PPP", "dec_alias_shuffled": "II" + "P" + "PPPPPPP",
}


# ---------------------------------------------------------------------------------------------------- the two builds

class Steps:
    def __init__(self, path):
        self.dll = C.CDLL(path)
        for name, sig in SIGS.items():
            f = getattr(self.dll, "hd_" + name)
            f.restype = C.c_int
            f.argtypes = [C.c_uint64] + [C.c_uint32 if c == "I" else C.c_void_p for c in sig]
        self.dll.hd_layout.restype = C.c_uint64
        self.dll.hd_layout.argtypes = [C.c_int]

    def layout(self):
        return [int(self.dll.hd_layout(k)) for k in range(8)]


@pytest.fixture(scope="module")
def builds(tmp_path_factory):
    """(host twin, path of the device library); both compiled from tests/header_device into the pytest tmp dir."""
    from ryg_rans_b200.build import NVCC_FLAGS, _nvcc
    out = tmp_path_factory.mktemp("header_device")
    dev = str(out / "libsteps_dev.so")
    host = str(out / "libsteps_host.so")
    subprocess.check_call([_nvcc(), *NVCC_FLAGS, "-shared", "-DNDEBUG", "-o", dev, os.path.join(SRC, "steps.cu")])
    subprocess.check_call([shutil.which("g++") or "g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DNDEBUG",
                           "-I" + os.path.join(ROOT, "include"), "-o", host, os.path.join(SRC, "steps_host.cpp")])
    return Steps(host), dev


class HostRun:
    """Runs the entries on the host twin; buffers are numpy arrays."""
    name = "host"

    def __init__(self, steps):
        self.steps = steps

    def put(self, a):
        return np.array(a, copy=True, order="C")

    def get(self, h):
        return h

    def addr(self, h):
        return h.ctypes.data

    def call(self, name, n, *args):
        rc = getattr(self.steps.dll, "hd_" + name)(n, *[a if isinstance(a, int) else self.addr(a) for a in args])
        assert rc == 0, f"hd_{name}: {rc}"


class DevRun(HostRun):
    """Runs the entries as kernels on cuda:0; buffers are (tensor, dtype, shape), moved as bytes."""
    name = "device"

    def __init__(self, steps):
        import torch
        self.torch = torch
        self.steps = steps

    def put(self, a):
        a = np.ascontiguousarray(a)
        return (self.torch.from_numpy(a.reshape(-1).view(np.uint8).copy()).cuda(), a.dtype, a.shape)

    def get(self, h):
        self.torch.cuda.synchronize()
        return h[0].cpu().numpy().view(h[1]).reshape(h[2])

    def addr(self, h):
        return h[0].data_ptr()


@pytest.fixture(scope="module")
def host(builds):
    return HostRun(builds[0])


@pytest.fixture(scope="module")
def device(builds):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return DevRun(Steps(builds[1]))


def _guarded(n):
    """a sentinel-filled buffer of n bytes with GUARD sentinel bytes on either side"""
    return np.full(n + 2 * GUARD, SENT, np.uint8)


def _check_guards(buf, what):
    assert (buf[:GUARD] == SENT).all() and (buf[-GUARD:] == SENT).all(), f"{what}: a guard byte was overwritten"


# ---------------------------------------------------------------------------------------------- preconditions

def _check_symbol_args(sb, freq, start, max_sb):
    """what RansEncSymbolInit / Rans64EncSymbolInit / the Put functions assert, checked before any call"""
    freq = np.asarray(freq, np.int64)
    start = np.asarray(start, np.int64)
    assert 1 <= sb <= max_sb
    assert (freq >= 1).all() and (start >= 0).all() and (start + freq <= (1 << sb)).all()


# ---------------------------------------------------------------------------------------------- A. symbol-init tables

def _rcp(freq, bits):
    """ceil(2^(bits + k) / freq), k = ceil(log2 freq): the reciprocal of RansEncSymbolInit (bits 31) and
    Rans64EncSymbolInit (bits 63), exact in Python integers"""
    k = (freq - 1).bit_length()
    return ((1 << (bits + k)) + freq - 1) // freq, k - 1


def _rans64_sample(sb):
    M = 1 << sb
    vals = {1, 2, 3, M, M - 1, M // 2, M // 2 + 1, M // 3 + 1}
    for k in range(sb + 1):
        vals |= {(1 << k) - 1, 1 << k, (1 << k) + 1}
    vals |= set(np.random.default_rng(sb).integers(1, M + 1, 4096).tolist())
    return np.array(sorted(v for v in vals if 1 <= v <= M), np.uint32)


def _init_items(coder):
    """(sb, freq, start) for every symbol-init item: every freq at scale_bits 1..16 with start 0, M - freq and a
    seeded random start; rans64 adds its sample at 17..31"""
    sbs, fs, cs = [], [], []
    rng = np.random.default_rng(11)
    ranges = [(sb, np.arange(1, (1 << sb) + 1, dtype=np.uint32)) for sb in range(1, 17)]
    if coder == RANS64:
        ranges += [(sb, _rans64_sample(sb)) for sb in range(17, 32)]
    for sb, f in ranges:
        M = 1 << sb
        rand = rng.integers(0, M - f.astype(np.int64) + 1).astype(np.uint32)
        for c in (np.zeros_like(f), (M - f).astype(np.uint32), rand):
            sbs.append(np.full(f.size, sb, np.uint32))
            fs.append(f)
            cs.append(c)
    return np.concatenate(sbs), np.concatenate(fs), np.concatenate(cs)


def _run_syms(run, coder):
    sb, f, c = _init_items(coder)
    enc_t, dec_t, name = (ENC32, DEC32, "byte_syms") if coder == BYTE else (ENC64, DEC64, "rans64_syms")
    for s in np.unique(sb):
        m = sb == s
        _check_symbol_args(int(s), f[m], c[m], 16 if coder == BYTE else 31)
    hs, hf, hc = run.put(sb), run.put(f), run.put(c)
    he, hd = run.put(np.zeros(f.size, enc_t)), run.put(np.zeros(f.size, dec_t))
    run.call(name, f.size, hs, hf, hc, he, hd)
    return (sb, f, c), run.get(he), run.get(hd)


def _expect_syms(coder, sb, f, c):
    sb64, f64, c64 = sb.astype(np.int64), f.astype(np.int64), c.astype(np.int64)
    M = np.int64(1) << sb64
    bits = 31 if coder == BYTE else 63
    uf = np.unique(f)
    table = {int(v): _rcp(int(v), bits) for v in uf}
    rcp = np.array([table[int(v)][0] if v >= 2 else (1 << (bits + 1)) - 1 for v in uf], dtype=object)
    shift = np.array([table[int(v)][1] if v >= 2 else 0 for v in uf], np.int64)
    pos = np.searchsorted(uf, f)
    if coder == BYTE:
        enc = np.zeros(f.size, ENC32)
        enc["x_max"] = ((BYTE_L >> sb64) << 8) * f64
        enc["rcp_freq"] = rcp.astype(np.uint64)[pos]
        enc["cmpl_freq"] = M - f64
        dec = np.zeros(f.size, DEC32)
        small = f64 < (1 << 16)
        dec["start"][small], dec["freq"][small] = c64[small], f64[small]
    else:
        enc = np.zeros(f.size, ENC64)
        enc["rcp_freq"] = np.array([int(v) for v in rcp], np.uint64)[pos]
        enc["freq"] = f64
        enc["cmpl_freq"] = M - f64
        dec = np.zeros(f.size, DEC64)
        dec["start"], dec["freq"] = c64, f64
    enc["rcp_shift"] = shift[pos]
    enc["bias"] = np.where(f64 >= 2, c64, c64 + M - 1)
    return enc, dec


def _assert_fields(got, want, items, what):
    for field in got.dtype.names:
        bad = np.nonzero(got[field] != want[field])[0]
        if bad.size:
            i = bad[0]
            pytest.fail(f"{what}.{field}: {bad.size} mismatches, first at sb={items[0][i]} freq={items[1][i]} "
                        f"start={items[2][i]}: {got[field][i]} != {want[field][i]}")


def _check_syms(runs, coder):
    results = [_run_syms(r, coder) for r in runs]
    items = results[0][0]
    want_enc, want_dec = _expect_syms(coder, *items)
    names = ("RansEncSymbol", "RansDecSymbol") if coder == BYTE else ("Rans64EncSymbol", "Rans64DecSymbol")
    for run, (_, enc, dec) in zip(runs, results):
        _assert_fields(enc, want_enc, items, f"{run.name} {names[0]}")
        _assert_fields(dec, want_dec, items, f"{run.name} {names[1]}")
    for run, (_, enc, dec) in zip(runs[1:], results[1:]):      # and byte for byte against the host twin
        assert enc.tobytes() == results[0][1].tobytes() and dec.tobytes() == results[0][2].tobytes(), run.name


def _check_word_tables(runs, oracle_lib):
    models = [_model(WORD, 12, kind, np.random.default_rng(3)) for kind in MODELS]
    freqs = np.stack([m[0] for m in models])
    cum = np.stack([m[1] for m in models])
    for run in runs:
        hs, hm = run.put(np.zeros((len(models), 4096), np.uint32)), run.put(np.zeros((len(models), 4096), np.uint8))
        run.call("word_tables", len(models), run.put(freqs), run.put(cum), hs, hm)
        slots, s2s = run.get(hs), run.get(hm)
        for b, kind in enumerate(MODELS):
            want_slots, want_s2s = oracle_lib.word_tables(freqs[b], cum[b])
            assert np.array_equal(slots[b], want_slots) and np.array_equal(s2s[b], want_s2s), f"{run.name} {kind}"


# ---------------------------------------------------------------------------------------------- B. one encode step

def _limit(which, sb, f):
    """the coder's renormalisation bound for freq f, as its step computes it (the word coder's is a u32 product)"""
    if which in BYTE_LIKE:
        return (U64(1) << U64(31 - sb)) * f
    if which in (R64_PUT, R64_PUTSYM):
        return (U64(1) << U64(63 - sb)) * f
    return (U64(1 << 20) * f) & U64(0xFFFFFFFF)


def _step_states(rng, which, sb, f):
    """(len(f), 85) states per freq: the edges of [0, x_max), 64 random ones below x_max, and states at or above x_max
    up to the largest 32- or 64-bit value, so that the renormalising branch emits"""
    f = f.astype(U64)
    wide = which in (R64_PUT, R64_PUTSYM)
    top = U64(2**64 - 1) if wide else U64(2**32 - 1)
    bound = U64(2**63 - 1) if wide else U64(2**31 - 1) if which in BYTE_LIKE else U64(2**32 - 1)
    xmax = _limit(which, sb, f)
    xmax = np.where(xmax == 0, U64(2**32), xmax)          # word, freq 4096: every state emits
    k = (xmax - U64(1)) // f
    n = f.size
    cols = [np.zeros(n, U64), np.ones(n, U64), f - U64(1), f, f + U64(1), k * f - U64(1), k * f, xmax - U64(1),
            xmax - U64(2)]
    above = np.minimum(xmax, top)
    cols += [above, np.minimum(xmax + U64(1), top), np.full(n, top), np.full(n, bound)]
    x = np.concatenate([np.stack(cols, 1), rng.integers(0, xmax[:, None], (n, 64), dtype=U64),
                        rng.integers(above[:, None], top, (n, 8), dtype=U64, endpoint=True)], 1)
    return x


def _step_expect(which, sb, f, c, x, remap):
    """the step in exact uint64 arithmetic: new state, the item's 8-byte slot and the bytes emitted"""
    n = x.size
    f, c, x = f.astype(U64), c.astype(U64), x.copy()
    slot = np.full((n, 8), SENT, np.uint8)
    cnt = np.zeros(n, np.uint8)
    lim = _limit(which, sb, f)
    if which in BYTE_LIKE:
        for _ in range(4):                                  # a byte at a time, low byte first, while x >= x_max
            e = np.nonzero(x >= lim)[0]
            if not e.size:
                break
            slot[e, 7 - cnt[e]] = (x[e] & U64(0xFF)).astype(np.uint8)
            cnt[e] += 1
            x[e] >>= U64(8)
    else:
        w = 4 if which in (R64_PUT, R64_PUTSYM) else 2     # at most one word
        e = np.nonzero(x >= lim)[0]
        words = (x[e] & U64((1 << (8 * w)) - 1)).astype("<u%d" % w)
        slot[e, 8 - w:] = words.view(np.uint8).reshape(-1, w)
        cnt[e] = w
        x[e] >>= U64(8 * w)
    q, r = x // f, x % f
    if which == ALIAS_PUT:
        new = (q << U64(sb)) + remap[(r + c).astype(np.int64)].astype(U64)
    else:
        new = (q << U64(sb)) + r + c
    if which in (BYTE_PUTSYM, R64_PUTSYM):
        # state 0 lies below every encoder's range; at freq 1 the reciprocal forms read its quotient as x - 1
        z = (x == 0) & (f == 1)
        new[z] = c[z] + U64((1 << sb) - 1)
    return new, slot, cnt


def _step_batches(which):
    """(sb, freqs, starts, seed) batches of the step sweep"""
    if which == WORD_PUT:
        sweep = [(12, np.arange(1, 4097, dtype=np.uint32))]
    else:
        sweep = [(sb, np.arange(1, (1 << sb) + 1, dtype=np.uint32)) for sb in range(1, 17)]
        if which in (R64_PUT, R64_PUTSYM):
            sweep += [(sb, _rans64_sample(sb)) for sb in range(17, 32)]
    for sb, f in sweep:
        M = 1 << sb
        rng = np.random.default_rng([which, sb])
        for kind, c in enumerate((np.zeros_like(f), (M - f).astype(np.uint32),
                                  rng.integers(0, M - f.astype(np.int64) + 1).astype(np.uint32))):
            yield sb, f, c, [which, sb, kind]


REMAP = np.random.default_rng(5).integers(0, 1 << 16, 1 << 16).astype(np.uint32)   # a stand-in alias_remap


def _check_step(runs, which):
    max_sb = 16 if which in BYTE_LIKE else 31 if which in (R64_PUT, R64_PUTSYM) else 12
    remaps = [r.put(REMAP) for r in runs]
    for sb, f, c, seed in _step_batches(which):
        _check_symbol_args(sb, f, c, max_sb)
        x = _step_states(np.random.default_rng(seed), which, sb, f)
        per = x.shape[1]
        f, c, x = np.repeat(f, per), np.repeat(c, per), x.reshape(-1)
        want, want_slot, want_cnt = _step_expect(which, sb, f, c, x, REMAP)
        outs = []
        for run, remap in zip(runs, remaps):
            hx, hcnt = run.put(np.zeros(x.size, U64)), run.put(np.zeros(x.size, np.uint8))
            hslot = run.put(_guarded(8 * x.size))
            run.call("step", x.size, which, sb, run.put(f), run.put(c), run.put(x), remap, hx,
                     run.addr(hslot) + GUARD, hcnt)
            got, slot, cnt = run.get(hx), run.get(hslot), run.get(hcnt)
            where = f"{run.name} sb={sb} start kind {seed[2]}"
            _check_guards(slot, where)
            slot = slot[GUARD:-GUARD].reshape(-1, 8)
            bad = np.nonzero((got != want) | (cnt != want_cnt) | (slot != want_slot).any(1))[0]
            if bad.size:
                i = bad[0]
                pytest.fail(f"{where}: {bad.size} wrong steps, first freq={f[i]} start={c[i]} x={x[i]}: state {got[i]} "
                            f"(exact {want[i]}), emitted {slot[i, 8 - cnt[i]:].tolist()} (exact "
                            f"{want_slot[i, 8 - want_cnt[i]:].tolist()})")
            outs.append((got, slot, cnt))
        for run, o in zip(runs[1:], outs[1:]):
            assert all(np.array_equal(a, b) for a, b in zip(o, outs[0])), f"{run.name} != host twin at sb={sb}"


def _check_sweep(run, which, sb):
    M = 1 << sb
    parts = 16 if run.name == "device" else 1
    hb, hx = run.put(np.zeros(M * parts, np.uint32)), run.put(np.zeros(M * parts, U64))
    run.call("sweep", M * parts, which, sb, parts, hb, hx)
    bad, first = run.get(hb), run.get(hx)
    if bad.any():
        i = int(np.nonzero(bad)[0][0])
        pytest.fail(f"{run.name} sb={sb}: {int(bad.sum())} states off the exact division, first freq={i // parts + 1} "
                    f"x={first[i]}")


# ---------------------------------------------------------------------------------------------- C. whole streams

DOM, ONE = 0x41, 0x07


def _cum(f):
    return np.concatenate([[0], np.cumsum(f.astype(np.uint64))]).astype(np.uint32)


def _model(coder, sb, kind, rng):
    """(freqs, cum, draw) of one stream-test model; draw(rng, n) gives n symbols"""
    M = 1 << sb
    f = np.zeros(256, np.uint64)
    if kind == "random":                                    # 1..256 symbols, random positive frequencies
        nsym = int(rng.integers(1, 257))
        syms = rng.choice(256, nsym, replace=False)
        w = rng.random(nsym) + 0.05
        f[syms] = 1 + rng.multinomial(M - nsym, w / w.sum())
        p = f / M
        draw = lambda r, n: r.choice(256, n, p=p).astype(np.uint8)        # noqa: E731
    elif kind == "ceiling":                                 # 255 x 1 + a dominant symbol; data from the rare ones
        f[:] = 1
        f[DOM] = M - 255
        ones = np.array([s for s in range(256) if s != DOM])
        draw = lambda r, n: r.choice(ones, n).astype(np.uint8)            # noqa: E731
    elif kind == "pair":                                    # {M - 1, 1}
        f[DOM], f[ONE] = M - 1, 1
        draw = lambda r, n: np.where(r.random(n) < 0.5, DOM, ONE).astype(np.uint8)   # noqa: E731
    elif kind == "single":                                  # one symbol at frequency M
        f[DOM] = M
        draw = lambda r, n: np.full(n, DOM, np.uint8)                     # noqa: E731
    else:                                                   # frequencies 2^k - 1, 2^k, 2^k + 1 and a remainder
        vals = []
        k = 1
        while len(vals) + 3 < 256 and sum(vals) + 3 * (1 << k) < M:
            vals += [(1 << k) - 1, 1 << k, (1 << k) + 1]
            k += 1
        vals.append(M - sum(vals))
        syms = (np.arange(len(vals)) * 37 + 5) % 256
        f[syms] = vals
        draw = lambda r, n: r.choice(syms, n).astype(np.uint8)            # noqa: E731
    assert int(f.sum()) == M and f.max() <= M
    f = f.astype(np.uint32)
    return f, _cum(f), draw


def _models(coder, sb):
    for kind in MODELS:
        if kind == "single" and coder == "byte" and sb == 16:
            continue                                        # RansDecSymbol's u16 freq cannot hold 65536
        yield kind, _model(coder, sb, kind, np.random.default_rng([sb, MODELS.index(kind), 17]))


def _lengths(rng, nl):
    fixed = [0, 1, max(nl - 1, 0), nl, nl + 1, 2 * nl - 1, 2 * nl + 1, 3, 7, 31, 33, 255, 1023, 2047, 2999]
    rest = rng.integers(0, 3000, N_THREADS - len(fixed) - 1)
    rest[::2] |= 1                                          # odd lengths
    return np.array(fixed + rest.tolist() + [3001], np.uint32)


def _layout(lens, nl):
    """region [begin, end) per thread: room for 4 bytes per symbol (any 32- or 64-bit state) and an 8-byte flush per
    state, 16-byte aligned, with GUARD sentinel bytes between regions"""
    region = (4 * lens.astype(np.uint64) + 8 * nl + 15) // 16 * 16
    begin = GUARD + np.concatenate([[0], np.cumsum(region + GUARD)[:-1]]).astype(np.uint64)
    end = begin + region
    return begin, end, int(end[-1]) + GUARD


def _regions_intact(buf, begin, end, stream_len, what):
    """every byte outside the streams is still the sentinel"""
    mask = np.ones(buf.size, bool)
    for e, n in zip(end.tolist(), stream_len.tolist()):
        mask[e - n:e] = False
    outside = np.nonzero(buf[mask] != SENT)[0]
    assert not outside.size, f"{what}: {outside.size} bytes written outside the streams"


class Config:
    """one (coder, scale_bits, model, lanes) of the stream test, with the model set up for a runner"""

    def __init__(self, coder, sb, kind, model, nl):
        self.coder, self.sb, self.kind, self.nl = coder, sb, kind, nl
        self.freqs, self.cum, draw = model
        rng = np.random.default_rng([sb, MODELS.index(kind), nl, len(coder)])
        self.lens = _lengths(rng, nl)
        self.seg_off = np.concatenate([[0], np.cumsum(self.lens.astype(np.uint64))[:-1]]).astype(np.uint64)
        self.data = draw(rng, int(self.lens.sum()))
        self.begin, self.end, self.size = _layout(self.lens, nl)
        self.L = {"byte": BYTE_L, "alias": BYTE_L, "rans64": R64_L, "word": WORD_L}[coder]
        self.ocoder = {"byte": BYTE, "alias": ALIAS, "rans64": RANS64, "word": WORD}[coder]

    def __str__(self):
        return f"{self.coder} sb={self.sb} {self.kind} N={self.nl}"

    def setup(self, run, host_steps):
        """the model's tables on `run`: symbols initialised by the runner itself, alias tables by RansAliasTablesInit
        on the host with alias_remap pointing at the runner's copy of the remap"""
        s = {"data": run.put(self.data), "seg_off": run.put(self.seg_off), "seg_len": run.put(self.lens),
             "freqs": run.put(self.freqs), "cum": run.put(self.cum)}
        if self.coder in ("byte", "rans64"):
            enc_t, dec_t = (ENC32, DEC32) if self.coder == "byte" else (ENC64, DEC64)
            used = self.freqs > 0
            _check_symbol_args(self.sb, self.freqs[used], self.cum[:256][used], 16 if self.coder == "byte" else 31)
            s["esyms"], s["dsyms"] = run.put(np.zeros(256, enc_t)), run.put(np.zeros(256, dec_t))
            run.call(self.coder + "_syms", 256, run.put(np.full(256, self.sb, np.uint32)), s["freqs"], s["cum"],
                     s["esyms"], s["dsyms"])
        if self.coder == "alias":
            tables, remap = _alias_tables(host_steps, self.freqs, self.cum)
            s["remap"] = run.put(remap)
            t = tables.copy()
            off = host_steps.layout()[5]
            t[off:off + 8] = np.array([run.addr(s["remap"])], "<u8").view(np.uint8)
            s["tables"] = run.put(t)
            s["shuffled"] = run.put(np.zeros(host_steps.layout()[6], np.uint8))
            run.call("shuffle_alias", 2 * 256, s["tables"], s["shuffled"])
        return s

    def encode(self, run, s, api):
        """every thread's stream on `run`: (whole buffer, stream lengths)"""
        hbuf, hlen = run.put(np.full(self.size, SENT, np.uint8)), run.put(np.zeros(N_THREADS, np.uint32))
        hend = run.put(self.end)
        head = (s["data"], s["seg_off"], s["seg_len"])
        if self.coder == "byte":
            run.call("enc_byte", N_THREADS, ENC_APIS[api], self.sb, self.nl, *head, s["freqs"], s["cum"], s["esyms"],
                     hbuf, hend, hlen)
        elif self.coder == "rans64":
            run.call("enc_rans64", N_THREADS, ENC_APIS[api], self.sb, self.nl, *head, s["freqs"], s["cum"],
                     s["esyms"], hbuf, hend, hlen)
        elif self.coder == "word":
            run.call("enc_word", N_THREADS, self.nl, *head, s["freqs"], s["cum"], hbuf, hend, hlen)
        else:
            run.call("enc_alias_" + api, N_THREADS, self.sb, self.nl, *head, s[api], hbuf, hend, hlen)
        buf, lens = run.get(hbuf), run.get(hlen)
        _check_guards(buf, f"{run.name} encode {self} {api}")
        _regions_intact(buf, self.begin, self.end, lens, f"{run.name} encode {self} {api}")
        return buf, lens

    def decode(self, run, s, api, buf, threads, stream_len):
        """decode the streams of `threads` (ending at self.end) from buf; check symbols, bytes read and final states"""
        what = f"{run.name} decode {self} {api}"
        threads = np.asarray(threads, np.int64)
        begin = (self.end[threads] - stream_len[threads].astype(np.uint64)).astype(np.uint64)
        off, lens = self.seg_off[threads], self.lens[threads]
        hdec, hcons = run.put(np.full(self.data.size + GUARD, SENT, np.uint8)), run.put(np.zeros(threads.size, np.uint32))
        hst = run.put(np.zeros((threads.size, 8), U64))
        tail = (run.put(buf), run.put(begin), run.put(off), run.put(lens), hdec, hcons, hst)
        n = threads.size
        if self.coder == "byte":
            run.call("dec_byte", n, DEC_APIS[api], self.sb, self.nl, s["freqs"], s["cum"], s["dsyms"], *tail)
        elif self.coder == "rans64":
            run.call("dec_rans64", n, DEC_APIS[api], self.sb, self.nl, s["freqs"], s["cum"], s["dsyms"], *tail)
        elif self.coder == "word":
            run.call("dec_word", n, self.nl, s["freqs"], s["cum"], *tail)
        else:
            run.call("dec_alias_" + api, n, self.sb, self.nl, s[api], *tail)
        dec, cons, st = run.get(hdec), run.get(hcons), run.get(hst)
        assert (dec[self.data.size:] == SENT).all(), f"{what}: wrote past the output"
        for j, t in enumerate(threads.tolist()):
            o, n_t = int(self.seg_off[t]), int(self.lens[t])
            assert np.array_equal(dec[o:o + n_t], self.data[o:o + n_t]), f"{what}: thread {t} decoded wrong symbols"
        bad = np.nonzero(cons != stream_len[threads])[0]
        assert not bad.size, f"{what}: thread {threads[bad[0]]} read {cons[bad[0]]} of {stream_len[threads[bad[0]]]} bytes"
        assert (st[:, :self.nl] == self.L).all(), f"{what}: a final state is not L"

    def sample(self):
        """first, last, 32 seeded random threads and every thread with fewer than 2N symbols"""
        rng = np.random.default_rng([self.sb, self.nl, 99])
        pick = {0, N_THREADS - 1} | set(rng.choice(N_THREADS, 32, replace=False).tolist())
        pick |= set(np.nonzero(self.lens < 2 * self.nl)[0].tolist())
        return sorted(pick)

    def oracle_streams(self, oracle_lib, threads):
        out = []
        for t in threads:
            o, n = int(self.seg_off[t]), int(self.lens[t])
            out.append(oracle_lib.encode(self.ocoder, self.data[o:o + n], self.freqs, self.cum, self.nl, self.sb))
        return out


def _alias_tables(host_steps, freqs, cum):
    """RansAliasTablesInit on the host: (the struct's bytes, remap)"""
    lay = host_steps.layout()
    tables = np.zeros(lay[4], np.uint8)
    remap = np.zeros(int(cum[256]), np.uint32)
    rc = host_steps.dll.hd_alias_init(C.c_void_p(freqs.ctypes.data), C.c_void_p(cum.ctypes.data),
                                      C.c_void_p(tables.ctypes.data), C.c_void_p(remap.ctypes.data))
    assert rc == 0, "RansAliasTablesInit refused the model"
    return tables, remap


def _alias_fields(tables):
    """divider, slot_adjust, slot_freqs, sym_id of a RansAliasTables (layout of rans_alias.h)"""
    u32 = tables[:(256 + 257 + 256 + 512 + 512) * 4].view("<u4")
    base = 256 + 257
    return (u32[base:base + 256], u32[base + 256:base + 768], u32[base + 768:base + 1280],
            tables[(base + 1280) * 4:(base + 1280) * 4 + 512])


def _enc_apis(coder):
    return ALIAS_STATS if coder == "alias" else ("div",) if coder == "word" else tuple(ENC_APIS)


def _dec_apis(coder):
    return ALIAS_STATS if coder == "alias" else ("sym+renorm",) if coder == "word" else tuple(DEC_APIS)


def _check_streams(coder, sb, host, oracle_lib, dev=None):
    """host twin against the oracle (and its own round trip); with `dev`, the device against the host twin, its
    decodes of its own streams, and of the oracle's"""
    for kind, model in _models(coder, sb):
        for nl in LANES:
            cfg = Config(coder, sb, kind, model, nl)
            hs = cfg.setup(host, host.steps)
            sample = cfg.sample()
            ostreams = cfg.oracle_streams(oracle_lib, sample)
            ref = None
            for api in _enc_apis(coder):
                buf, lens = cfg.encode(host, hs, api)
                for t, o in zip(sample, ostreams):
                    e = int(cfg.end[t])
                    assert np.array_equal(buf[e - int(lens[t]):e], o), f"host encode {cfg} {api}: thread {t} != oracle"
                if ref is None:
                    ref = (buf, lens)
                assert np.array_equal(buf, ref[0]) and np.array_equal(lens, ref[1]), f"host {cfg}: the two encoder APIs differ"
            if coder != "rans64" or sb <= 24:                # the oracle decodes rans64 up to scale_bits 24
                for t, o in zip(sample, ostreams):
                    o_sl = slice(int(cfg.seg_off[t]), int(cfg.seg_off[t]) + int(cfg.lens[t]))
                    got, used = oracle_lib.decode(cfg.ocoder, o, int(cfg.lens[t]), cfg.freqs, cfg.cum, nl, sb)
                    assert np.array_equal(got, cfg.data[o_sl]) and used == o.size, f"oracle decode {cfg}: thread {t}"
            if dev is None:
                for api in _dec_apis(coder):
                    cfg.decode(host, hs, api, ref[0], np.arange(N_THREADS), ref[1])
                continue
            ds = cfg.setup(dev, host.steps)
            for api in _enc_apis(coder):
                buf, lens = cfg.encode(dev, ds, api)
                bad = np.nonzero(lens != ref[1])[0]
                assert not bad.size, (f"device encode {cfg} {api}: thread {bad[0]} stream length {lens[bad[0]]} != host twin "
                                      f"{ref[1][bad[0]]}")
                diff = np.nonzero(buf != ref[0])[0]
                assert not diff.size, (f"device encode {cfg} {api}: {diff.size} bytes differ from the host twin, first in "
                                       f"thread {int(np.searchsorted(cfg.end, diff[0], side='right'))}")
            for api in _dec_apis(coder):                     # only streams shown equal to the host twin's
                cfg.decode(dev, ds, api, ref[0], np.arange(N_THREADS), ref[1])
            obuf = np.full(cfg.size, SENT, np.uint8)         # the oracle's streams, placed as the encoders place theirs
            olen = np.zeros(N_THREADS, np.uint32)
            for t, o in zip(sample, ostreams):
                obuf[int(cfg.end[t]) - o.size:int(cfg.end[t])] = o
                olen[t] = o.size
            for api in _dec_apis(coder):
                cfg.decode(dev, ds, api, obuf, sample, olen)


# ---------------------------------------------------------------------------------------------- tests without a GPU

def test_headers_compile_for_the_device_with_live_asserts(tmp_path):
    """Without NDEBUG every RansAssert / Rans64Assert of the headers is a device assert; the same kernels still
    compile for sm_90a (compile only: nothing built here is launched)."""
    from ryg_rans_b200.build import NVCC_FLAGS, _nvcc
    subprocess.check_call([_nvcc(), *NVCC_FLAGS, "-c", "-o", str(tmp_path / "steps.o"), os.path.join(SRC, "steps.cu")])


def test_both_builds_agree_on_the_struct_layouts(builds):
    """The nvcc build compiles every header function for sm_90a (the fixture built it); its host side lays the
    structs out as the host twin does, and as this test views them."""
    dev = Steps(builds[1])
    lay = builds[0].layout()
    assert dev.layout() == lay
    assert lay[:4] == [ENC32.itemsize, DEC32.itemsize, ENC64.itemsize, DEC64.itemsize]
    assert lay[7] == 4096 * 5


@pytest.mark.parametrize("coder", ["byte", "rans64"])
def test_host_twin_symbol_init(host, coder):
    _check_syms([host], BYTE if coder == "byte" else RANS64)


def test_host_twin_word_tables(host, oracle_lib):
    _check_word_tables([host], oracle_lib)


@pytest.mark.parametrize("sb", range(8, 17))
def test_host_alias_tables_match_the_oracle(host, oracle_lib, sb):
    for kind, (freqs, cum, _) in _models("alias", sb):
        tables, remap = _alias_tables(host.steps, freqs, cum)
        want = oracle_lib.alias_build(freqs, cum)
        for name, got, w in zip(("divider", "slot_adjust", "slot_freqs", "sym_id", "alias_remap"),
                                (*_alias_fields(tables), remap), want):
            assert np.array_equal(got, w), f"{kind}: {name}"


@pytest.mark.parametrize("step", list(STEPS))
def test_host_twin_one_step(host, step):
    _check_step([host], STEPS[step])


@pytest.mark.parametrize("which", ["byte", "rans64"])
def test_host_twin_dense_sweep(host, which):
    _check_sweep(host, BYTE_PUTSYM if which == "byte" else R64_PUTSYM, 10)


@pytest.mark.parametrize("coder,sb", STREAM_CASES, ids=[f"{c}-{s}" for c, s in STREAM_CASES])
def test_host_twin_streams(host, oracle_lib, coder, sb):
    _check_streams(coder, sb, host, oracle_lib)


# ---------------------------------------------------------------------------------------------- on the GPU

@pytest.mark.gpu
@pytest.mark.parametrize("coder", ["byte", "rans64"])
def test_symbol_init_on_device(host, device, coder):
    _check_syms([host, device], BYTE if coder == "byte" else RANS64)


@pytest.mark.gpu
def test_word_tables_in_shared_memory(device, oracle_lib):
    _check_word_tables([device], oracle_lib)


@pytest.mark.gpu
@pytest.mark.parametrize("step", list(STEPS))
def test_one_step_on_device(host, device, step):
    _check_step([host, device], STEPS[step])


@pytest.mark.gpu
@pytest.mark.parametrize("sb", [12, 14, 16])
@pytest.mark.parametrize("which", ["byte", "rans64"])
def test_dense_sweep_on_device(device, which, sb):
    _check_sweep(device, BYTE_PUTSYM if which == "byte" else R64_PUTSYM, sb)


@pytest.mark.gpu
@pytest.mark.parametrize("coder,sb", STREAM_CASES, ids=[f"{c}-{s}" for c, s in STREAM_CASES])
def test_streams_on_device(host, device, oracle_lib, coder, sb):
    _check_streams(coder, sb, host, oracle_lib, device)
