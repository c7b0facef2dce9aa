"""Coded streams past byte 2^32 of a blob: every coder's encode paths and decoders, compared with the oracle.

Blob offsets are 64-bit, but the decoders keep stream positions in 32 bits on purpose (StreamWindow's fill_end and
cursor, TmaWindow's ring-linear pos0 beside off % kUnit), and the encoders' placement, scan and compaction produce
offsets past 2^32 for a large enough blob.  Each case here is a blob of a little more than 4 GiB whose one stream over
the mark is placed on purpose, one of three ways (a blob has exactly one stream over 2^32, so each case realises one;
every single-model coder, the word coder's WIDE decoder included, has a case of each; the per-block coders share one
block decoder, which sees all three across them: word (a) and (c), alias (b) and (c), byte (b), rans64 (a)):
  (a) the stream's body straddles 2^32,
  (b) its 128-byte (rans64: 256-byte) header straddles 2^32,
  (c) it starts exactly at 2^32, a 512- and 1024-byte unit boundary (the directory holds the entry 2^32).

The expected container is exact without encoding gigabytes on the CPU: the data is a pattern over a few distinct
units (a chunk, or a block of chunks with its model) and a ragged last chunk, and each unit's streams depend only on
its symbols and model.  The oracle encodes each unit once; the directory is then a sum of padded stream sizes, and the
blob is each unit's padded streams (zero bytes, then the stream, as every encoder places it) at its offset.  The
pattern is drawn from a fixed seed and closed with a coin-change of units in front of the target, so that the target
chunk lands where its case needs it; every case asserts that it did (`straddle`), and that the blob passes 2^32.  The
test without a GPU builds the same layouts with the mark at 2^20 and checks them byte for byte against the oracle's
encode of the whole data and the library's container packs.

On the GPU, each case encodes through the flat (or per-block) call and the container call, compares the directory, the
header and, unit by unit, the blob with the expected one and checks nothing was written past it; then it decodes with
the host-launched and the planned (async) decoders into buffers with sentinel bytes past n.  Three corruptions must be
rejected with E_STREAM by one host-launched and one async decoder, after which the same context decodes the intact
buffer: 64 flipped body bytes of the stream over the mark, the directory entry of the first chunk past the mark moved
down by exactly 2^32 (same low 32 bits), and, in (c) cases, the entry at 2^32 moved by 16.  The entry moved down is
rejected before its chunk is decoded, so that chunk's output must stay untouched; the other two are only found at the
end of the stream, after the decoder has written its symbols.  A word and a byte case also run through the host-memory
calls, whose slice pipeline joins the slices' blobs past 2^32.

Each GPU case takes a context of its own (closed afterwards, so its workspace is returned), never holds the flat blob
and the container at once (at most about 24 GiB of device memory), and skips when the shared GPU lacks what it needs;
the host-memory cases skip when the host lacks the memory."""
import math
import os
import struct
import sys
import zlib

import numpy as np
import pytest

import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_rate_ceiling as rc  # noqa: E402

WORD, BYTE, ALIAS, RANS64 = orc.CODER_WORD, orc.CODER_BYTE, orc.CODER_ALIAS, orc.CODER_RANS64
MARK = 1 << 32
CRC_BLOB = 1
E_STREAM = -4
SENTINEL = 0x5C
MAGIC = 0x43324252
V1_DIR = 1088
BLOCK_VERSION = {WORD: 2, BYTE: 3, RANS64: 3, ALIAS: 4}


def r16(x):
    return (x + 15) & ~15


def header_bytes(coder):
    return 256 if coder == RANS64 else 128


# ---------------------------------------------------------------------------------------------------- the layout

def flat_model(coder, sb, kind):
    """the caller model of a single-model case: rate-ceiling models, or 'wide': one symbol holding all 4096 slots"""
    if kind == "wide":
        f = np.zeros(256, np.uint32)
        f[rc.DOM] = 4096
        return f
    return rc._freqs(sb, kind)


def _cum(f):
    return np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)


def _streams(oracle_lib, coder, sb, freqs, data, ch):
    blob, offs = oracle_lib.chunked_encode(coder, data, freqs, _cum(freqs), ch, nlanes=32, scale_bits=sb)
    return [blob[int(offs[c]):int(offs[c + 1]) & ~15] for c in range(offs.size - 1)]


def _padded(streams):
    return np.concatenate([np.concatenate([np.zeros(r16(s.size) - s.size, np.uint8), s]) for s in streams])


class Units:
    """K distinct units of `per` chunks each: their symbols, model rows (per-block) and oracle streams"""

    def __init__(self, oracle_lib, coder, sb, ch, per, freqs=None):
        self.oracle_lib, self.coder, self.sb, self.ch, self.per, self.freqs = oracle_lib, coder, sb, ch, per, freqs
        self.data, self.rows, self.streams, self.weights = [], [], [], []

    def add(self, data, weight, row=None):
        f = self.freqs if row is None else row.astype(np.uint32)
        self.data.append(np.ascontiguousarray(data, np.uint8))
        self.rows.append(row)
        self.streams.append(_streams(self.oracle_lib, self.coder, self.sb, f, data, self.ch))
        self.weights.append(weight)

    @property
    def K(self):
        return len(self.data)


def flat_units(oracle_lib, coder, sb, model_kind, ch, seed):
    """ceiling chunks of four seeds, floor chunks, mixtures (mostly ceiling, so that the mark needs fewer symbols)"""
    f = flat_model(coder, sb, model_kind)
    u = Units(oracle_lib, coder, sb, ch, 1, f)
    if model_kind == "wide":
        u.add(np.full(ch, rc.DOM, np.uint8), 1.0)
        return u
    for i in range(4):
        u.add(rc.rate_data(f, "ceiling", ch, seed + i), 0.7 / 4)
    u.add(rc.rate_data(f, "floor", ch, seed), 0.06)
    u.add(rc.rate_data(f, "mix97", ch, seed + 5, lo=1, hi=ch), 0.06)
    u.add(rc.rate_data(f, "mix50", ch, seed + 6), 0.06)
    u.add(rc.rate_data(f, "regions", ch, seed + 7, lo=32, hi=ch), 0.06)
    u.add(np.where(np.random.default_rng(seed + 8).random(ch) < 0.01, rc.rate_data(f, "ceiling", ch, seed + 9),
                   rc.rate_data(f, "floor", ch, 0)).astype(np.uint8), 0.06)
    return u


def flat_tail(units):
    """the ragged last chunk: ch // 2 + 5 ceiling symbols (the wide model's symbol alone)"""
    m = units.ch // 2 + 5
    if len(units.data) == 1:
        return np.full(m, rc.DOM, np.uint8)
    return rc.rate_data(units.freqs, "ceiling", m, 77)


BLOCK_MODELS = {WORD: ["dom", "2963", "2964", "pair"], BYTE: ["dom"], RANS64: ["dom"], ALIAS: ["dom"]}


def block_units(oracle_lib, coder, sb, ch, per, seed, K=8):
    """K blocks of per chunks, each with its own model (a ceiling model, symbols rotated) and chunks that are mostly at
    the ceiling, one floor chunk and one mixture"""
    u = Units(oracle_lib, coder, sb, ch, per)
    for k in range(K):
        _block(u, k, seed)
    return u


def _block(u, k, seed):
    kinds = BLOCK_MODELS[u.coder]
    row = np.roll(rc._freqs(u.sb, kinds[k % len(kinds)]), 37 * k).astype(np.uint16)
    shapes = ["ceiling"] * u.per
    shapes[k % u.per] = "floor"
    shapes[(k + 3) % u.per] = "mix97"
    data = np.concatenate([rc.rate_data(row.astype(np.uint32), s, u.ch, seed + 100 * k + j) for j, s in enumerate(shapes)])
    u.add(data, 1.0, row)


def _want_kind(kind, r, H):
    if kind == "c":
        return r % 16 == 0 and r >= 2 * H
    return r >= 2 * H + 64


def _ensure_c(units, H, seed):
    """a (c) case needs a stream whose length is a multiple of 16 (so that it starts where its region does): add
    mixtures until one unit has one"""
    for i in range(64):
        if any(_want_kind("c", s.size, H) for st in units.streams for s in st):
            return
        if units.per == 1:
            units.add(rc.rate_data(units.freqs, "mix97", units.ch, seed + 1000 + i, lo=1, hi=units.ch), 0.0)
        else:
            _block(units, units.K, seed + 1000 + i)
            units.weights[-1] = 0.0
    raise AssertionError("no unit has a stream of a multiple of 16 bytes")


def _coins(units):
    return [sum(r16(s.size) for s in st) // 16 for st in units.streams]


def _ensure_small_coins(units, seed):
    """two small units of coprime padded sizes (in 16-byte steps), so that a coin-change closes any gap of more than
    their product: floor units, and quiet ones with a 1 % mixture in one chunk"""
    f = units.freqs if units.per == 1 else None
    for i in range(64):
        small = sorted(set(_coins(units)))[:6]
        pairs = [(a * b) for a in small for b in small if a < b and math.gcd(a, b) == 1]
        if pairs:
            return min(pairs)
        row = None if units.per == 1 else np.roll(rc._freqs(units.sb, BLOCK_MODELS[units.coder][0]), 37 * i).astype(np.uint16)
        fr = f if row is None else row.astype(np.uint32)
        quiet = [rc.rate_data(fr, "floor", units.ch, 0) for _ in range(units.per)]
        if i:
            rng = np.random.default_rng(seed + 3000 + i)
            quiet[0] = np.where(rng.random(units.ch) < 0.002 * i, rc.rate_data(fr, "ceiling", units.ch, seed + 4000 + i), quiet[0]).astype(np.uint8)
        units.add(np.concatenate(quiet), 0.01, row)
    raise AssertionError("no two small units of coprime sizes")


def _coin_change(target, coins):
    """a list of coin indices whose values sum to target (all in 16-byte units), fewest coins, or None"""
    if target < 0:
        return None
    INF = 1 << 30
    best = [0] + [INF] * target
    how = [-1] * (target + 1)
    for g in range(1, target + 1):
        for i, c in enumerate(coins):
            if c <= g and best[g - c] + 1 < best[g]:
                best[g] = best[g - c] + 1
                how[g] = i
    if best[target] >= INF:
        return None
    out, g = [], target
    while g:
        out.append(how[g])
        g -= coins[how[g]]
    return out


class Layout:
    """The exact expected directory and blob of `units` laid out so that the chunk over `mark` is of `kind`"""

    def __init__(self, units, mark, kind, seed, extra, tail=None):
        H = header_bytes(units.coder)
        if kind == "c":
            _ensure_c(units, H, seed)
        frob = _ensure_small_coins(units, seed)
        self.units, self.mark, self.kind, self.tail = units, mark, kind, tail
        per = units.per
        r = np.array([[s.size for s in st] for st in units.streams], np.int64)            # [K, per]
        p = r16(r)
        P = p.sum(1)
        self.P = P
        self.W = [_padded(st) for st in units.streams]                                     # each unit's padded region
        # the target chunk (k, j): the largest stream that suits the kind, nearest the middle of its unit
        cands = [(abs(j - per // 2), -int(r[k, j]), k, j) for k in range(units.K) for j in range(per) if _want_kind(kind, int(r[k, j]), H)]
        assert cands, (kind, r)
        _, _, tk, tj = min(cands)
        rt, pt = int(r[tk, tj]), int(p[tk, tj])
        if kind == "c":
            t_chunk = mark                                                               # offset == region start
        elif kind == "b":
            t_chunk = mark - r16(H // 2 + (pt - rt))                                     # offset in (mark - H, mark)
        else:
            t_chunk = mark - r16(pt // 2)                                                # mark in the middle of the stream
        T = t_chunk - int(p[tk, :tj].sum())
        # a prefix from the seed that ends well short of T (4 units, and more than the two small units' product),
        # closed by a coin-change of units
        rng = np.random.default_rng(seed)
        w = np.array(units.weights, float)
        w /= w.sum()
        gmin = 16 * max(4 * int(P.max()) // 16, frob)
        est = int(T / float((P * w).sum()) * 1.2) + 64
        draw = rng.choice(units.K, size=est, p=w)
        ends = np.cumsum(P[draw])
        L = int(np.searchsorted(ends, T - gmin, side="right"))
        for _ in range(64):
            assert L >= 0, "the mark is too close to the start for this layout"
            e0 = int(ends[L - 1]) if L else 0
            fill = _coin_change((T - e0) // 16, [int(x) // 16 for x in P])
            if fill is not None:
                break
            L -= 1
        assert fill is not None, "no coin-change closes the prefix"
        head = np.concatenate([draw[:L], np.array(fill, np.int64), [tk]])
        # a suffix from the seed that takes the blob `extra` bytes past the mark
        sdraw = rng.choice(units.K, size=int(extra / float((P * w).sum()) * 1.2) + 64, p=w)
        sends = np.cumsum(P[sdraw])
        S = int(np.searchsorted(sends, extra)) + 1
        self.pattern = np.concatenate([head, sdraw[:S]]).astype(np.int64)
        self.target = (head.size - 1) * per + tj
        # unit starts, the directory
        uend = np.cumsum(P[self.pattern])
        self.ustart = np.concatenate([[0], uend[:-1]]).astype(np.int64)
        in_unit = np.concatenate([np.zeros((units.K, 1), np.int64), np.cumsum(p, 1)[:, :-1]], 1) + (p - r)   # [K, per]
        offs = (self.ustart[:, None] + in_unit[self.pattern]).reshape(-1)
        end = int(uend[-1])
        if tail is not None:
            self.tail_stream = _streams(units.oracle_lib, units.coder, units.sb, units.freqs, tail, units.ch)[0]
            self.tail_at = end
            offs = np.append(offs, end + r16(self.tail_stream.size) - self.tail_stream.size)
            end += r16(self.tail_stream.size)
        self.offs = np.append(offs, end).astype(np.uint64)
        self.blob_bytes = end
        self.n_chunks = self.offs.size - 1
        self.n = self.pattern.size * per * units.ch + (0 if tail is None else tail.size)
        c, got = straddle(self.offs, mark, H)
        assert (c, got) == (self.target, kind), ((c, got), (self.target, kind))
        assert self.blob_bytes > mark

    def host_data(self):
        """the whole input on the host (small layouts only)"""
        d = np.concatenate([self.units.data[k] for k in self.pattern])
        return d if self.tail is None else np.concatenate([d, self.tail])

    def host_blob(self):
        b = np.concatenate([self.W[k] for k in self.pattern])
        if self.tail is None:
            return b
        return np.concatenate([b, _padded([self.tail_stream])])

    def block_rows(self):
        return np.stack([self.units.rows[k] for k in self.pattern])

    def blob_crc(self):
        """zlib's CRC-32 of the blob, folded unit by unit: crc(A || B) = Z_|B|(crc(A)) ^ crc(B), Z_L linear"""
        tables = {}
        for L in set(int(x) for x in self.P) | ({r16(self.tail_stream.size)} if self.tail is not None else set()):
            zeros = bytes(L)
            z0 = zlib.crc32(zeros)
            tables[L] = [[zlib.crc32(zeros, b << (8 * i)) ^ z0 for b in range(256)] for i in range(4)]
        crcs = [zlib.crc32(w.tobytes()) for w in self.W]
        sizes = [int(x) for x in self.P]
        c = 0
        for k in self.pattern.tolist():
            t0, t1, t2, t3 = tables[sizes[k]]
            c = t0[c & 255] ^ t1[(c >> 8) & 255] ^ t2[(c >> 16) & 255] ^ t3[c >> 24] ^ crcs[k]
        if self.tail is not None:
            t0, t1, t2, t3 = tables[r16(self.tail_stream.size)]
            c = t0[c & 255] ^ t1[(c >> 8) & 255] ^ t2[(c >> 16) & 255] ^ t3[c >> 24] ^ zlib.crc32(_padded([self.tail_stream]).tobytes())
        return c


def straddle(offs, mark, H):
    """(chunk, kind) of the stream over `mark`: 'c' starts at it, 'b' its header straddles it, 'a' its body does;
    kind None when the mark falls in a gap or on a header's end"""
    offs = np.asarray(offs).astype(np.int64)
    c = int(np.searchsorted(offs[:-1], mark, side="right")) - 1
    lo = int(offs[c])
    hi = int(offs[c + 1]) & ~15 if c + 1 < offs.size - 1 else int(offs[-1])
    if lo == mark:
        return c, "c"
    if lo < mark < lo + H:
        return c, "b"
    if lo + H < mark < hi:
        return c, "a"
    return c, None


def _meta(h, model, dirb):
    """meta_crc: the header with its crc fields zero, the model section, the directory"""
    return zlib.crc32(dirb, zlib.crc32(model, zlib.crc32(h)))


def expected_head(lay, flags, blob_crc=0):
    """the container's bytes before the blob: version 1 (single model) or the per-block version of the coder"""
    u = lay.units
    if u.per == 1:
        version, block_size, nb = 1, 0, 0
        model = np.ascontiguousarray(u.freqs, np.uint32).tobytes()
    else:
        version, block_size, nb = BLOCK_VERSION[u.coder], u.per * u.ch, lay.pattern.size
        model = lay.block_rows().astype(np.uint16).tobytes()
    fields = [MAGIC, version, u.coder, u.sb, 32, u.ch, lay.n, lay.n_chunks, lay.blob_bytes, flags]
    h0 = struct.pack("<IHBBIIQQQIIIIII", *fields, 0, 0, block_size, nb, 0)
    dirb = lay.offs.tobytes()
    h = struct.pack("<IHBBIIQQQIIIIII", *fields, _meta(h0, model, dirb), blob_crc if flags & CRC_BLOB else 0, block_size, nb, 0)
    head = h + model + dirb
    return np.frombuffer(head + bytes(r16(len(head)) - len(head)), np.uint8)


def reseal(head, per_block):
    """recompute meta_crc of an edited head (flags 0: no blob CRC)"""
    head = head.copy()
    n_chunks, = struct.unpack_from("<Q", head, 24)
    nb, = struct.unpack_from("<I", head, 56)
    dir_at = 64 + 512 * nb if per_block else V1_DIR
    h0 = head[:64].copy()
    h0[44:52] = 0
    struct.pack_into("<I", head, 44, _meta(h0.tobytes(), head[64:dir_at].tobytes(), head[dir_at:dir_at + 8 * (n_chunks + 1)].tobytes()))
    return head


# ---------------------------------------------------------------------------------------------------- CPU: the layout

SMALL = 1 << 20                                           # the mark of the flat layouts; 2^22 for the per-block ones

CPU_FLAT = [(WORD, 12, "dom", 512), (WORD, 12, "wide", 416), (BYTE, 16, "dom", 1024), (ALIAS, 14, "dom", 512),
            (RANS64, 16, "dom", 1024)]


CPU_FLAT_KINDS = [(*c, k) for c in CPU_FLAT for k in ("a", "b", "c")]


@pytest.mark.parametrize("coder,sb,mk,ch,kind", CPU_FLAT_KINDS, ids=[f"{c}-{m}-{s}-{k}" for c, s, m, _, k in CPU_FLAT_KINDS])
def test_cpu_flat_layout_matches_oracle(oracle_lib, coder, sb, mk, ch, kind):
    from ryg_rans_b200 import api
    if mk == "wide":
        ch = wide_chunk(SMALL, kind, ch)
    units = flat_units(oracle_lib, coder, sb, mk, ch, 3)
    lay = wide_layout(units, SMALL, SMALL // 8, kind) if mk == "wide" else Layout(units, SMALL, kind, 11, SMALL // 8, flat_tail(units))
    data = lay.host_data()
    assert data.size == lay.n
    f = units.freqs
    blob, offs = oracle_lib.chunked_encode(coder, data, f, _cum(f), ch, nlanes=32, scale_bits=sb)
    assert np.array_equal(offs, lay.offs)
    assert np.array_equal(blob, lay.host_blob())
    assert lay.blob_crc() == zlib.crc32(blob.tobytes())
    for flags in (0, CRC_BLOB):
        want = api.container_pack(coder, sb, ch, data.size, f, offs, blob, flags)
        head = expected_head(lay, flags, lay.blob_crc())
        assert np.array_equal(want[:head.size], head), flags
        assert np.array_equal(want[head.size:], blob)
        # an edit resealed by reseal() is what container_pack would have written
        if flags == 0:
            o2 = offs.copy()
            o2[lay.target] += 16
            want2 = api.container_pack(coder, sb, ch, data.size, f, o2, blob, 0) if lay.target + 1 < o2.size - 1 else None
            if want2 is not None:
                edited = head.copy()
                edited[V1_DIR + 8 * lay.target:V1_DIR + 8 * lay.target + 8] = o2[lay.target:lay.target + 1].view(np.uint8)
                assert np.array_equal(reseal(edited, False), want2[:head.size])


CPU_BLOCKS = [(WORD, 12, 512, 4), (BYTE, 15, 512, 8), (RANS64, 15, 256, 8), (ALIAS, 15, 512, 8)]


@pytest.mark.parametrize("kind", ["a", "b", "c"])
@pytest.mark.parametrize("coder,sb,ch,per", CPU_BLOCKS, ids=[f"{c}-{s}" for c, s, _, _ in CPU_BLOCKS])
def test_cpu_block_layout_matches_oracle(oracle_lib, coder, sb, ch, per, kind):
    from ryg_rans_b200 import api
    units = block_units(oracle_lib, coder, sb, ch, per, 5)
    lay = Layout(units, 4 * SMALL, kind, 13, SMALL // 2)
    data = lay.host_data()
    rows = lay.block_rows()
    nb, bs = lay.pattern.size, per * ch
    offs, blob = rc._oracle_blocks(oracle_lib, coder, sb, data, rows, bs, ch)
    assert np.array_equal(offs, lay.offs)
    assert np.array_equal(blob, lay.host_blob())
    for flags in (0, CRC_BLOB):
        if coder == WORD:
            want = api.container_blocks_pack(nb, bs, ch, rows, offs, blob, flags)
        elif coder == ALIAS:
            want = api.container_blocks_alias_pack(sb, nb, bs, ch, rows, offs, blob, flags)
        else:
            want = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, rows, offs, blob, flags)
        head = expected_head(lay, flags, zlib.crc32(blob.tobytes()))
        assert np.array_equal(want[:head.size], head), flags
        assert np.array_equal(want[head.size:], blob)
        if flags == 0:
            edited = head.copy()
            at = 64 + 512 * nb + 8 * lay.target
            struct.pack_into("<Q", edited, at, int(offs[lay.target]) + 16)
            o2 = offs.copy()
            o2[lay.target] += 16
            if coder == WORD:
                want2 = api.container_blocks_pack(nb, bs, ch, rows, o2, blob, 0)
            elif coder == ALIAS:
                want2 = api.container_blocks_alias_pack(sb, nb, bs, ch, rows, o2, blob, 0)
            else:
                want2 = api.container_blocks_coder_pack(coder, sb, nb, bs, ch, rows, o2, blob, 0)
            assert np.array_equal(reseal(edited, True), want2[:head.size])


def _wide_kind(ch, mark):
    """the kind of the stream over `mark` when every stream is 2 ch + 128 bytes (the one-symbol word model), placed
    end-aligned in regions of round16(2 ch + 128)"""
    S = 2 * ch + 128
    p = r16(S)
    lo = mark // p * p + (p - S)
    if mark < lo:
        return None
    rem = mark - lo
    return "c" if rem == 0 else "b" if rem < 128 else "a" if rem > 128 else None


def wide_chunk(mark, kind, near):
    """the first chunk size from `near` up whose one-symbol streams put a stream of `kind` over `mark`"""
    for ch in range(near, near + 65536):
        if _wide_kind(ch, mark) == kind:
            return ch
    raise AssertionError((mark, kind, near))


def wide_layout(units, mark, extra, kind):
    """the one-symbol word model: every chunk's stream is S = 2 ch + 128 bytes, so chunk c's stream starts at
    c round16(S) + round16(S) - S, and the chunk size alone (wide_chunk) decides which kind of stream is over the mark"""
    S = units.streams[0][0].size
    assert S == 2 * units.ch + 128, S
    p = r16(S)
    lay = Layout.__new__(Layout)
    lay.units, lay.mark, lay.kind = units, mark, kind
    lay.tail = np.full(units.ch // 2 + 5, rc.DOM, np.uint8)
    lay.P = np.array([p], np.int64)
    lay.W = [_padded(units.streams[0])]
    full = mark // p + extra // p
    lay.pattern = np.zeros(full, np.int64)
    lay.target = mark // p
    lay.ustart = np.arange(full, dtype=np.int64) * p
    lay.tail_stream = _streams(units.oracle_lib, WORD, 12, units.freqs, lay.tail, units.ch)[0]
    lay.tail_at = full * p
    end = full * p + r16(lay.tail_stream.size)
    lay.offs = np.append(np.append(lay.ustart + (p - S), full * p + r16(lay.tail_stream.size) - lay.tail_stream.size), end).astype(np.uint64)
    lay.blob_bytes, lay.n_chunks = end, full + 1
    lay.n = full * units.ch + lay.tail.size
    assert straddle(lay.offs, mark, 128) == (lay.target, kind)
    assert lay.blob_bytes > mark
    return lay


# ---------------------------------------------------------------------------------------------------- GPU helpers

def _torch():
    import torch
    return torch


def _room(need):
    torch = _torch()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"{need / 2**30:.1f} GiB of device memory needed, {free / 2**30:.1f} GiB free on the shared GPU")
    return free


def _need(n, cap, n_chunks, ch):
    """device memory a case holds at most: input and output (n + 64 each), the blob or the container (never both),
    the encode workspace (at most a worst-case slot per chunk: the split path's), and 2 GiB for the units, the
    directory, the comparisons' temporaries and the context"""
    return 2 * (n + 64) + cap + 64 + n_chunks * r16(512 + 2 * ch) + (2 << 30)


def _equal(a, b):
    step = 1 << 28
    return all(_torch().equal(a[i:i + step], b[i:i + step]) for i in range(0, a.numel(), step))


def _untouched(t):
    step = 1 << 28
    return all(bool((t[i:i + step] == SENTINEL).all().item()) for i in range(0, t.numel(), step))


def _sync(ctx):
    return ctx.lib.dll.rb200_sync(ctx.h)


def _run(ctx, call):
    """the sync code of an enqueued call (a host-launched call may raise its error instead)"""
    import ryg_rans_b200 as rb
    try:
        call()
    except rb.RansError as e:
        _sync(ctx)
        return e.code
    return _sync(ctx)


def gpu_input(lay):
    """the input on the GPU, built by indexing the units with the pattern (never copied from the host)"""
    torch = _torch()
    u = lay.units
    U = u.per * u.ch
    d_units = torch.from_numpy(np.stack(u.data)).cuda()
    d_pat = torch.from_numpy(lay.pattern).cuda()
    d_in = torch.empty(lay.n, dtype=torch.uint8, device="cuda")
    step = max(1, (1 << 28) // U)
    nu = lay.pattern.size
    for i in range(0, nu, step):
        j = min(nu, i + step)
        d_in[i * U:j * U].view(j - i, U).copy_(d_units[d_pat[i:j]])
    if lay.tail is not None:
        d_in[nu * U:] = torch.from_numpy(lay.tail).cuda()
    return d_in


def blob_mismatch(lay, d_blob):
    """None when d_blob (the blob's first byte at index 0) holds every unit's padded streams where the layout puts
    them, else where it first does not"""
    torch = _torch()
    starts = torch.from_numpy(lay.ustart).cuda()
    pat = torch.from_numpy(lay.pattern).cuda()
    for k in range(lay.units.K):
        sel = starts[pat == k]
        if not sel.numel():
            continue
        want = torch.from_numpy(lay.W[k]).cuda()
        P = want.numel()
        ar = torch.arange(P, device="cuda", dtype=torch.int64)
        rows = max(1, (1 << 25) // P)
        for i in range(0, sel.numel(), rows):
            got = d_blob[sel[i:i + rows, None] + ar]
            bad = (got != want).any(1)
            if bool(bad.any().item()):
                r = int(torch.nonzero(bad)[0].item())
                at = int(sel[i + r].item())
                return f"unit {k} at blob byte {at} (chunk {int(np.searchsorted(lay.offs[:-1].astype(np.int64), at, side='right'))})"
    if lay.tail is not None:
        want = _padded([lay.tail_stream])
        if not np.array_equal(d_blob[lay.tail_at:lay.tail_at + want.size].cpu().numpy(), want):
            return "the ragged last chunk"
    return None


def _report(name, lay, free0):
    torch = _torch()
    H = header_bytes(lay.units.coder)
    offs = lay.offs.astype(np.int64)
    print(f"{name}: n = {lay.n}, {lay.n_chunks} chunks, blob {lay.blob_bytes} bytes ({lay.blob_bytes / 2**30:.3f} GiB); "
          f"chunk {lay.target} ({lay.kind}: {'body straddles' if lay.kind == 'a' else 'header straddles' if lay.kind == 'b' else 'starts at'} "
          f"2^32, stream [{offs[lay.target]}, {int(offs[lay.target + 1]) & ~15}), header {H}); "
          f"{(free0 - torch.cuda.mem_get_info()[0]) / 2**30:.2f} GiB of device memory in use")


def _first_past(lay):
    """the first chunk whose stream starts at or past 2^32"""
    return int(np.searchsorted(lay.offs[:-1].astype(np.int64), lay.mark, side="left"))


class Checker:
    """decode and reject checks of one encoded buffer: decode(buf) enqueues a decode of d_buf into d_out"""

    def __init__(self, ctx, d_in, lay):
        torch = _torch()
        self.ctx, self.d_in, self.lay = ctx, d_in, lay
        self.d_out = torch.full((lay.n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")

    def decodes(self, call, what, counts_n=False):
        self.d_out.fill_(SENTINEL)
        self.d_n.fill_(-1)
        rc_ = _run(self.ctx, call)
        assert rc_ == 0, (what, rc_)
        if counts_n:
            assert int(self.d_n.item()) == self.lay.n, what
        assert _equal(self.d_out[:self.lay.n], self.d_in), (what, "decoded symbols differ")
        assert _untouched(self.d_out[self.lay.n:]), (what, "written past n")

    def rejects(self, call, what, chunk=None):
        self.d_out.fill_(SENTINEL)
        rc_ = _run(self.ctx, call)
        assert rc_ == E_STREAM, (what, rc_)
        if chunk is not None:
            ch = self.lay.units.ch
            lo = chunk * ch
            assert _untouched(self.d_out[lo:min(lo + ch, self.lay.n)]), (what, "the chunk was decoded despite its entry")


def _flip_at(lay):
    """64 body bytes of the stream over the mark, past the mark.  At the ceiling one flipped byte is not enough: a byte
    that only feeds a frequency-1 symbol's slot can turn it into another frequency-1 symbol with the same next state,
    which no end-of-stream check can see (only the blob CRC, off here); one of 64 turns it into the dominant symbol."""
    return max(lay.mark, int(lay.offs[lay.target]) + header_bytes(lay.units.coder)) + 37


def _edits(lay):
    """(what, chunk, new entry) of the three corruptions: the flip (no entry), the first chunk past the mark moved down
    by 2^32 and, in (c) cases, the entry at 2^32 moved by 16.  Only the entry moved down is rejected before anything is
    decoded (its stream would be longer than 2^30 bytes), so only there is the chunk's output checked untouched; the
    other two are found at the stream's end, after its symbols were written."""
    nxt = _first_past(lay)
    edits = [("flip", None, None), ("down 2^32", nxt, int(lay.offs[nxt]) - (1 << 32))]
    if lay.kind == "c":
        edits.append(("2^32 + 16", lay.target, lay.mark + 16))
    return edits


def _flip(t, at):
    t[at:at + 64].bitwise_xor_(0x5A)


def host_rejects(chk, d_blob, d_offs, call):
    """the three corruptions of the flat (or per-block) blob and directory, through a host-launched decode, each
    followed by a good decode"""
    lay = chk.lay
    for what, c, v in _edits(lay):
        if c is None:
            _flip(d_blob, _flip_at(lay))
        else:
            d_offs[c] = v
        chk.rejects(call, ("host-launched", what), c if what == "down 2^32" else None)
        if c is None:
            _flip(d_blob, _flip_at(lay))
        else:
            d_offs[c] = int(lay.offs[c])
        chk.decodes(call, ("host-launched after", what))


def async_rejects(chk, cont, call, boff, per_block):
    """the same corruptions of the container (directory edits resealed, so that its meta CRC still holds), through an
    async decode, each followed by a good decode"""
    torch = _torch()
    lay = chk.lay
    head = cont[:boff].cpu().numpy()
    dir_at = 64 + 512 * lay.pattern.size if per_block else V1_DIR
    for what, c, v in _edits(lay):
        if c is None:
            _flip(cont, boff + _flip_at(lay))
        else:
            h = head.copy()
            struct.pack_into("<Q", h, dir_at + 8 * c, v)
            cont[:boff] = torch.from_numpy(reseal(h, per_block)).cuda()
        chk.rejects(call, ("async", what), c if what == "down 2^32" else None)
        if c is None:
            _flip(cont, boff + _flip_at(lay))
        else:
            cont[:boff] = torch.from_numpy(head).cuda()
        chk.decodes(call, ("async after", what), counts_n=True)


# ---------------------------------------------------------------------------------------------------- GPU: version 1

# id: coder, scale_bits, model, chunk, kind, flags.  Word: K2r (a ring model, chunks <= 8192), K2f (chunks above 8192;
# the one-symbol model, which K2r never takes, at chunk sizes that place each kind), split (below 4096).  Byte and alias: fused from 4096, split below;
# 16, 14 and 12 are the specialised decoder instances, 15 the generic one.  rans64: split.
FLAT = {
    "word-K2r": (WORD, 12, "dom", 8192, "a", 0),
    "word-K2f": (WORD, 12, "2964", 16384, "c", 0),
    "word-split": (WORD, 12, "2963", 2048, "b", 0),
    "word-wide-K2f-a": (WORD, 12, "wide", wide_chunk(MARK, "a", 8192), "a", 0),
    "word-wide-K2f-b": (WORD, 12, "wide", wide_chunk(MARK, "b", 8192), "b", 0),
    "word-wide-K2f-c": (WORD, 12, "wide", wide_chunk(MARK, "c", 8000), "c", 0),
    "byte16-fused": (BYTE, 16, "dom", 8192, "a", CRC_BLOB),
    "byte16-split": (BYTE, 16, "pair", 2048, "c", 0),
    "byte15-fused": (BYTE, 15, "dom", 4096, "b", 0),
    "alias16-fused": (ALIAS, 16, "dom", 8192, "b", 0),
    "alias14-split": (ALIAS, 14, "dom", 2048, "a", 0),
    "alias12-fused": (ALIAS, 12, "dom", 4096, "c", 0),
    "alias15-split": (ALIAS, 15, "dom", 1024, "b", 0),
    "rans64-split-8192": (RANS64, 16, "dom", 8192, "a", 0),
    "rans64-split-2048": (RANS64, 16, "dom", 2048, "b", 0),
    "rans64-split-4096": (RANS64, 16, "dom", 4096, "c", 0),
}
EXTRA = 1 << 28                                           # blob bytes past the mark


def flat_layout(oracle_lib, name):
    coder, sb, mk, ch, kind, _ = FLAT[name]
    units = flat_units(oracle_lib, coder, sb, mk, ch, 21)
    if mk == "wide":
        return wide_layout(units, MARK, EXTRA, kind)
    return Layout(units, MARK, kind, 31, EXTRA, flat_tail(units))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FLAT))
def test_flat_past_2_32(cuda_box, oracle_lib, name):
    torch = _torch()
    import ryg_rans_b200 as rb
    coder, sb, _, ch, kind, flags = FLAT[name]
    lay = flat_layout(oracle_lib, name)
    n, N = lay.n, lay.n_chunks
    if ch == 2048:
        assert N > 1 << 20, N                             # past 256 scan tiles: tile_prefix_kernel
    c = rb.Context(0)
    try:
        cap = c.encode_bound(n, ch)
        ccap = c.container_capacity(n, ch)
        free0 = _room(_need(n, max(cap, ccap), N, ch))
        d_in = gpu_input(lay)
        mdl = c.model(coder, sb, lay.units.freqs)
        chk = Checker(c, d_in, lay)
        # the flat call: directory, blob, nothing past it; the host-launched decoders
        d_blob = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_offs = torch.zeros(N + 1, dtype=torch.int64, device="cuda")
        assert _run(c, lambda: c.encode_device(mdl, d_in.data_ptr(), n, ch, d_blob.data_ptr(), cap, d_offs.data_ptr())) == 0
        got = d_offs.cpu().numpy().view(np.uint64)
        if not np.array_equal(got, lay.offs):
            i = int(np.flatnonzero(got != lay.offs)[0])
            pytest.fail(f"{name}: directory entry {i} is {int(got[i])}, {int(lay.offs[i])} expected")
        bad = blob_mismatch(lay, d_blob)
        assert bad is None, (name, "encode_device", bad)
        assert _untouched(d_blob[lay.blob_bytes:]), (name, "written past the blob")
        host_call = lambda: c.decode_device(mdl, d_blob.data_ptr(), lay.blob_bytes, d_offs.data_ptr(), ch, chk.d_out.data_ptr(), n)  # noqa: E731
        chk.decodes(host_call, "decode_device")
        if flags == 0:
            host_rejects(chk, d_blob, d_offs, host_call)
        del d_blob, d_offs, host_call                     # the blob and the container are never held at once
        torch.cuda.empty_cache()
        # the container call
        d_cont = torch.full((ccap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        assert _run(c, lambda: c.container_encode_device(mdl, d_in.data_ptr(), n, ch, flags, d_cont.data_ptr(), ccap)) == 0
        want = expected_head(lay, flags, lay.blob_crc() if flags & CRC_BLOB else 0)
        boff = want.size
        head = d_cont[:boff].cpu().numpy()
        if not np.array_equal(head, want):
            i = int(np.flatnonzero(head != want)[0])
            pytest.fail(f"{name}: container byte {i} differs ({'header' if i < 64 else 'model' if i < V1_DIR else 'directory'})")
        bad = blob_mismatch(lay, d_cont[boff:])
        assert bad is None, (name, "container_encode_device", bad)
        size = boff + lay.blob_bytes
        assert _untouched(d_cont[size:]), (name, "written past the container")
        dec_call = lambda: c.container_decode_device(d_cont.data_ptr(), size, chk.d_out.data_ptr(), n)  # noqa: E731
        chk.decodes(dec_call, "container_decode_device")
        async_call = lambda: c.container_decode_async(d_cont.data_ptr(), size, chk.d_out.data_ptr(), n, chk.d_n.data_ptr())  # noqa: E731
        chk.decodes(async_call, "container_decode_async", counts_n=True)
        _report(name, lay, free0)
        if flags == 0:
            async_rejects(chk, d_cont, async_call, boff, False)
        mdl.close()
    finally:
        c.close()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- GPU: versions 2-4

# id: coder, scale_bits, chunk, chunks per block, kind.  Word: K5f from 4096 symbols per chunk, split below; the byte,
# rans64 and alias per-block coders: split.
BLOCKS = {
    "word-K5f": (WORD, 12, 8192, 8, "c"),
    "word-split": (WORD, 12, 2048, 8, "a"),
    "byte15": (BYTE, 15, 4096, 8, "b"),
    "rans64-15": (RANS64, 15, 4096, 8, "a"),
    "alias15": (ALIAS, 15, 4096, 8, "c"),
    "alias12": (ALIAS, 12, 2048, 8, "b"),
}


def block_calls(c, coder, sb):
    """(flat encode, flat decode, container encode, the version's async decode) of one per-block coder"""
    if coder == WORD:
        return (c.blocks_encode_device, c.blocks_decode_device, c.container_blocks_encode_device, c.container_blocks_decode_async)
    if coder == ALIAS:
        return (lambda *a: c.blocks_alias_encode_device(sb, *a), lambda *a: c.blocks_alias_decode_device(sb, *a),
                lambda *a: c.container_blocks_alias_encode_device(sb, *a), c.container_blocks_alias_decode_async)
    return (lambda *a: c.blocks_coder_encode_device(coder, sb, *a), lambda *a: c.blocks_coder_decode_device(coder, sb, *a),
            lambda *a: c.container_blocks_coder_encode_device(coder, sb, *a), c.container_blocks_coder_decode_async)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BLOCKS))
def test_blocks_past_2_32(cuda_box, oracle_lib, name):
    torch = _torch()
    import ryg_rans_b200 as rb
    coder, sb, ch, per, kind = BLOCKS[name]
    units = block_units(oracle_lib, coder, sb, ch, per, 41)
    lay = Layout(units, MARK, kind, 43, EXTRA)
    n, N, nb, bs = lay.n, lay.n_chunks, lay.pattern.size, per * ch
    c = rb.Context(0)
    try:
        cap = c.encode_bound(n, ch)
        ccap = c.container_blocks_capacity(nb, bs, ch)
        free0 = _room(_need(n, max(cap, ccap), N, ch))
        enc, dec, cenc, cdec = block_calls(c, coder, sb)
        d_in = gpu_input(lay)
        d_rows = torch.from_numpy(np.stack(units.rows).view(np.int16)).cuda()[torch.from_numpy(lay.pattern).cuda()].contiguous()
        chk = Checker(c, d_in, lay)
        d_blob = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_offs = torch.zeros(N + 1, dtype=torch.int64, device="cuda")
        assert _run(c, lambda: enc(d_in.data_ptr(), nb, bs, d_rows.data_ptr(), ch, d_blob.data_ptr(), cap, d_offs.data_ptr())) == 0
        got = d_offs.cpu().numpy().view(np.uint64)
        if not np.array_equal(got, lay.offs):
            i = int(np.flatnonzero(got != lay.offs)[0])
            pytest.fail(f"{name}: directory entry {i} is {int(got[i])}, {int(lay.offs[i])} expected")
        bad = blob_mismatch(lay, d_blob)
        assert bad is None, (name, "block encode", bad)
        assert _untouched(d_blob[lay.blob_bytes:]), (name, "written past the blob")
        host_call = lambda: dec(d_blob.data_ptr(), lay.blob_bytes, d_offs.data_ptr(), d_rows.data_ptr(), nb, bs, ch, chk.d_out.data_ptr())  # noqa: E731
        chk.decodes(host_call, "block decode")
        host_rejects(chk, d_blob, d_offs, host_call)
        del d_blob, d_offs, host_call                     # the blob and the container are never held at once
        torch.cuda.empty_cache()
        d_cont = torch.full((ccap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        assert _run(c, lambda: cenc(d_in.data_ptr(), nb, bs, d_rows.data_ptr(), ch, 0, d_cont.data_ptr(), ccap)) == 0
        want = expected_head(lay, 0)
        boff = want.size
        head = d_cont[:boff].cpu().numpy()
        if not np.array_equal(head, want):
            i = int(np.flatnonzero(head != want)[0])
            pytest.fail(f"{name}: container byte {i} differs")
        bad = blob_mismatch(lay, d_cont[boff:])
        assert bad is None, (name, "container encode", bad)
        size = boff + lay.blob_bytes
        assert _untouched(d_cont[size:]), (name, "written past the container")
        async_call = lambda: cdec(d_cont.data_ptr(), size, chk.d_out.data_ptr(), n, chk.d_n.data_ptr())  # noqa: E731
        chk.decodes(async_call, "the version's async decode", counts_n=True)
        any_call = lambda: c.container_blocks_any_decode_async(d_cont.data_ptr(), size, chk.d_out.data_ptr(), n, chk.d_n.data_ptr())  # noqa: E731
        chk.decodes(any_call, "container_blocks_any_decode_async", counts_n=True)
        _report(name, lay, free0)
        async_rejects(chk, d_cont, async_call, boff, True)
    finally:
        c.close()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- GPU: host memory

def _host_free():
    with open("/proc/meminfo") as f:
        info = dict(line.split(":", 1) for line in f)
    return int(info["MemAvailable"].split()[0]) * 1024


def host_input(lay):
    u = lay.units
    U = u.per * u.ch
    units = np.stack(u.data)
    data = np.empty(lay.n, np.uint8)
    nu = lay.pattern.size
    step = max(1, (1 << 28) // U)
    for i in range(0, nu, step):
        j = min(nu, i + step)
        data[i * U:j * U].reshape(j - i, U)[:] = units[lay.pattern[i:j]]
    if lay.tail is not None:
        data[nu * U:] = lay.tail
    return data


def host_blob_mismatch(lay, blob):
    """blob_mismatch for a container in host memory (blob: a view of its blob)"""
    for k in range(lay.units.K):
        sel = lay.ustart[lay.pattern == k]
        want = lay.W[k]
        ar = np.arange(want.size, dtype=np.int64)
        rows = max(1, (1 << 24) // want.size)
        for i in range(0, sel.size, rows):
            bad = (blob[sel[i:i + rows, None] + ar] != want).any(1)
            if bad.any():
                return f"unit {k} at blob byte {int(sel[i + int(np.flatnonzero(bad)[0])])}"
    if lay.tail is not None and not np.array_equal(blob[lay.tail_at:], _padded([lay.tail_stream])):
        return "the ragged last chunk"
    return None


# a word and a byte case through the host-memory calls, whose slice pipeline encodes and decodes the input a slice at
# a time: the slices' running blob base crosses 2^32, and (byte, CRC_BLOB) so does the joined blob CRC
HOST = ["word-wide-K2f-b", "byte16-fused"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", HOST)
def test_host_memory_past_2_32(cuda_box, oracle_lib, name):
    import ryg_rans_b200 as rb
    coder, sb, _, ch, kind, flags = FLAT[name]
    lay = flat_layout(oracle_lib, name)
    c = rb.Context(0)
    try:
        cap = c.container_capacity(lay.n, ch)
        need = 2 * lay.n + cap + lay.blob_bytes + (2 << 30)      # input, output, the call's buffer and its result
        if _host_free() < need:
            pytest.skip(f"{need / 2**30:.1f} GiB of host memory needed, {_host_free() / 2**30:.1f} GiB available")
        data = host_input(lay)
        mdl = c.model(coder, sb, lay.units.freqs)
        cont = c.container_encode_host(mdl, data, ch, flags=flags)
        want = expected_head(lay, flags, lay.blob_crc() if flags & CRC_BLOB else 0)
        assert cont.size == want.size + lay.blob_bytes, (cont.size, want.size + lay.blob_bytes)
        if not np.array_equal(cont[:want.size], want):
            i = int(np.flatnonzero(cont[:want.size] != want)[0])
            pytest.fail(f"{name}: container byte {i} differs ({'header' if i < 64 else 'model' if i < V1_DIR else 'directory'})")
        bad = host_blob_mismatch(lay, cont[want.size:])
        assert bad is None, (name, "container_encode_host", bad)
        out = c.container_decode_host(cont)
        assert out.size == lay.n and np.array_equal(out, data), (name, "container_decode_host")
        print(f"{name} (host memory): n = {lay.n}, blob {lay.blob_bytes} bytes, chunk {lay.target} ({kind}) over 2^32")
        mdl.close()
    finally:
        c.close()
