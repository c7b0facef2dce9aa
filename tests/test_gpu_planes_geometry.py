"""The byte-plane containers, versions 7 and 8, at the geometries where their kernels could go wrong unseen.

Unless a section names another oracle, every container the GPU encodes is compared byte for byte with the host oracle:
one forced (coder, scale_bits), each plane built from the C oracle's streams with the store rule applied in Python
(cs.oracle_container, cs.apply_store, api.container_stored_pack), packed with api.container_planes_pack, or for
version 8 the planes of numpy's zigzag difference packed with api.container_delta_pack and the base's zlib CRC.  Every
case first asserts the edge it claims to reach.

1. Every tail at every width: w = 2, 4, 8 and m = 1 .. 48 elements (m % 16 every value, no whole group for m <= 15,
   m = 16, 17) and m = 16 * 4 + t for t = 0 .. 15 at chunks of 32, and m = 16 * 1100 + t at chunks of 8192.  Group
   bytes lie in [0, 128), tail bytes in [128, 256).  The version 7 fixed encode, the varlen encode at n_max = w (16 K +
   15) (its plane stride n_max's), the version 8 encode; the version 7 decode and the version 8 decode out of place and
   in place; nothing written past n or past the container.
2. Grid passes: m = P * groups_per_pass * 16 + 16 * 3 + 7 for P = 2, 3 at w = 2, 4, 8, groups_per_pass the device's
   SMs x 8 x 256 (the split, interleave, delta split and delta interleave run P + 1 passes).  The top plane is uniform
   and stored, larger than one pass of the place and fetch copies.  The version 7 encode and decode, the version 8
   encode and in-place decode, the varlen encode under a larger n_max; host oracle.  Prints the device memory in use.
3. Every lane position of the delta transform: each of cd.crafted's 144 pairs at every element position 0 .. 15 of a
   group, and at every position of a ragged tail (m % 16 = 15, 144 tensors); encode, decode out of place and in place.
4. Plane-coder order: version 7 and version 8 containers built on the host with forced per-plane pairs so that every
   ordered pair of nine plane states (word 12, alias 9 and 16, byte 9 and 14, rans64 11 and 16, every chunk stored,
   some chunks stored) is at consecutive planes somewhere, decoded back to back on one context with one sync.  A w = 8
   encode under a four-candidate list at tolerance 0 picks three coders and stores a plane (composed oracle:
   gcp.expected, the version 6 encode of each numpy-split plane).
5. Decode bounds: out_cap n, n + 1, n + w - 1, n + 16, 3 n by size exact, exact + 1 .. 15 and the bound, the version 8
   base holding other bytes in [n, out_cap) (kept in place); out_cap 0, w - 1, n - w is RB200_E_SPACE with *d_n = n;
   size 0, 63, 64 + 16 w - 1, 64 + 16 w is RB200_E_STREAM with out untouched; after each reject the intact buffer
   decodes.  The overlap rule at its boundary: out = base +- out_cap decodes, one 16-byte step inside is RB200_E_ARG
   with nothing launched.
6. Pointers 16 bytes past 32-byte alignment (+16, +48, +80): the same containers and round trips as at +0.
7. Queued calls of growing geometry with one sync: version 8 encode (w 2), version 7 decode (w 8), version 8 in-place
   decode of the first container, version 7 varlen encode (w 4), each equal to the same call made alone.

The module takes its own context, closed when it ends."""
import os
import sys
import zlib

import numpy as np
import pytest

import ryg_rans_b200 as rb
from ryg_rans_b200 import api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_container_delta as cd  # noqa: E402
import test_container_planes as cp  # noqa: E402
import test_container_stored as cs  # noqa: E402
import test_gpu_blocks_coder as gbc  # noqa: E402
import test_gpu_blocks_geometry as gg  # noqa: E402
import test_gpu_container_delta as gcd  # noqa: E402
import test_gpu_container_planes as gcp  # noqa: E402
import test_gpu_container_planes_varlen as gpv  # noqa: E402
from conftest import _gen  # noqa: E402

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = rb.CODER_WORD, rb.CODER_BYTE, rb.CODER_ALIAS, rb.CODER_RANS64
CAND = api.CANDIDATE
CRC_BLOB = 1
SENTINEL = gcp.SENTINEL
E_ARG, E_SPACE, E_STREAM = -1, -3, -4
WIDTHS = [2, 4, 8]


def _torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def ctx(cuda_box):
    """this module's own context, so that its workspaces are freed when the module ends"""
    c = rb.Context(0)
    try:
        yield c
    finally:
        c.close()


def _sync(ctx):
    return ctx.lib.dll.rb200_sync(ctx.h)


def groups_per_pass():
    """threads of one planes_grid (SMs x kPlanesCtasPerSm x kPlanesThreads): each moves one group of 16 per pass"""
    return _torch().cuda.get_device_properties(0).multi_processor_count * 8 * 256


# ---------------------------------------------------------------------------------------------------- host oracle

def host_plane(oracle_lib, plane, pair, ch, flags, which=None):
    """(version 6 container, stored chunks) of one plane from the oracle's streams, `which` (default: the rule's) stored"""
    coder, sb = pair
    freqs, cum, offs, blob = cs.oracle_container(oracle_lib, coder, sb, plane, ch)
    bits, o6, b6, st = cs.apply_store(plane, ch, offs, blob, which)
    return api.container_stored_pack(coder, sb, ch, plane.size, freqs, bits, o6, b6, flags), st


def host_planes(oracle_lib, data, w, pairs, ch, flags=0, which=None):
    """the w version 6 planes of data; pairs and which: one for every plane, or a list of one per plane"""
    pairs = pairs if isinstance(pairs, list) else [pairs] * w
    which = which if isinstance(which, list) else [which] * w
    return [host_plane(oracle_lib, pl, pairs[p], ch, flags, which[p])[0] for p, pl in enumerate(cp.split(data, w))]


def v7_of(planes):
    return api.container_planes_pack(planes)


def v8_of(planes, base):
    return api.container_delta_pack(planes, zlib.crc32(base.tobytes()))


def plane_coders(buf):
    """(coder, scale_bits, all chunks stored, some chunk stored) of every plane of a version 7 or 8 buffer"""
    opener = api.container_delta_open if buf[4] == 8 else api.container_planes_open
    out = []
    for pl in opener(buf)[1]:
        info, _, bits, _, _ = api.container_stored_open(pl)
        k = info["n_chunks"]
        stored = sum(bin(int(x)).count("1") for x in bits)
        out.append((info["coder"], info["scale_bits"], stored == k, stored > 0))
    return out


def same(rc, got, want, case):
    """an encode's whole sentinel-filled output: rc 0, the container equal to want, nothing written past it"""
    assert rc == 0, (case, rc)
    size = gcp.v7_size(got)
    if size != want.size or not np.array_equal(got[:size], want):
        diff = np.flatnonzero(got[:min(size, want.size)] != want[:min(size, want.size)])
        pytest.fail(f"{case}: container of {size} bytes, oracle {want.size}, first difference at {diff[:1]}")
    assert (got[size:] == SENTINEL).all(), (case, "written past the container")


def ragged(m, w, seed):
    """m elements of w bytes: the whole groups' bytes in [0, 128), the ragged tail's in [128, 256)"""
    rng = np.random.default_rng(seed)
    g = m // 16 * 16
    x = np.empty((m, w), np.uint8)
    x[:g] = rng.integers(0, 128, (g, w), dtype=np.uint8)
    x[g:] = rng.integers(128, 256, (m - g, w), dtype=np.uint8)
    return x.reshape(-1)


def delta_pair(d, w, seed):
    """(x, base) whose zigzag difference is d: base random, x = base + unzigzag(d)"""
    base = np.random.default_rng(seed).integers(0, 256, d.size, dtype=np.uint8)
    x = cd.unzigzag(d, base, w)
    assert np.array_equal(cd.zigzag(x, base, w), d)
    return x, base


def padded(data, size, seed):
    """data on the device followed by random bytes up to size (the varlen encode must not read them)"""
    tail = np.random.default_rng(seed).integers(0, 256, size - data.size, dtype=np.uint8)
    return gbc._dev(np.concatenate([data, tail]))


def round_trips(ctx, v7, v8, d, x, base, w, case):
    """the version 7 decode gives d, the version 8 decode x, out of place and in place, nothing written past n"""
    n = d.size
    rc, got_n, out = gcp.decode(ctx, v7, w, n)
    assert rc == 0 and got_n == n, (case, "v7", rc, got_n)
    assert np.array_equal(out[:n], d) and (out[n:] == SENTINEL).all(), (case, "v7")
    for in_place in (False, True):
        rc, got_n, out, b = gcd.decode(ctx, v8, w, base, n, in_place=in_place)
        assert rc == 0 and got_n == n, (case, "v8", in_place, rc, got_n)
        assert np.array_equal(out[:n], x) and (out[n:] == SENTINEL).all(), (case, "v8", in_place)
        assert np.array_equal(b, x if in_place else base), (case, "v8 base", in_place)


# ---------------------------------------------------------------------------------------------------- 1. every tail

TAIL_SWEEPS = [("1..48", 32, 4, list(range(1, 49))), ("16*4+t", 32, 4, [16 * 4 + t for t in range(16)]),
               ("16*1100+t", 8192, 1100, [16 * 1100 + t for t in range(16)])]


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("name,ch,k,counts", TAIL_SWEEPS, ids=[s[0] for s in TAIL_SWEEPS])
def test_every_tail(ctx, oracle_lib, w, name, ch, k, counts):
    tails = {m % 16 for m in counts}
    assert tails == set(range(16)), tails
    if name == "1..48":
        assert {1, 2, 15, 16, 17} <= set(counts)                        # no whole group; one group; one and a tail
    n_max = w * (16 * k + 15)
    assert all(w * m <= n_max for m in counts)
    pair = (WORD, 12) if ch == 32 else [(BYTE, 14), (ALIAS, 16), (RANS64, 15)][WIDTHS.index(w)]
    cands = [CAND(*pair)]
    for i, m in enumerate(counts):
        case = (w, ch, m)
        d = ragged(m, w, 1000 * w + m)
        x, base = delta_pair(d, w, 2000 * w + m)
        flags = i & 1
        planes = host_planes(oracle_lib, d, w, pair, ch, flags)
        v7, v8 = v7_of(planes), v8_of(planes, base)
        rc, got = gcp.encode(ctx, cands, 0, d, w, ch, flags)
        same(rc, got, v7, case + ("v7",))
        rc, got = gpv.varlen7(ctx, cands, 0, padded(d, n_max, m), d.size, n_max, w, ch, flags)
        same(rc, got, v7, case + ("varlen",))
        rc, got = gcd.encode(ctx, cands, 0, x, base, w, ch, flags)
        same(rc, got, v8, case + ("v8",))
        round_trips(ctx, v7, v8, d, x, base, w, case)


# ---------------------------------------------------------------------------------------------------- 2. grid passes

def pass_planes(m, w, seed):
    """w planes of m bytes: plane w - 1 uniform (stored), the others geometric at different skews (coded)"""
    rng = np.random.default_rng(seed)
    out = np.empty((m, w), np.uint8)
    for p in range(w - 1):
        out[:, p] = np.minimum(rng.geometric((0.5, 0.2, 0.05, 0.35, 0.1, 0.7, 0.03)[p], m) - 1, 255)
    out[:, w - 1] = rng.integers(0, 256, m, dtype=np.uint8)
    return out.reshape(-1)


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("passes", [2, 3])
def test_grid_passes(ctx, oracle_lib, w, passes):
    torch = _torch()
    gpp = groups_per_pass()
    ch, j, t = 8192, 3, 7
    m = passes * gpp * 16 + 16 * j + t
    groups = m // 16
    assert -(-groups // gpp) == passes + 1 and groups % gpp == j and m % 16 == t
    n = w * m
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    used = [0]

    def note():
        used[0] = max(used[0], free0 - torch.cuda.mem_get_info()[0])

    d = pass_planes(m, w, w + passes)
    x, base = delta_pair(d, w, 7 * w + passes)
    pair = (BYTE, 14)
    cands = [CAND(*pair)]
    planes = host_planes(oracle_lib, d, w, pair, ch, 0)
    top = planes[w - 1]
    n_chunks = -(-m // ch)
    assert top.size == cs.blob_offset(n_chunks) + (n_chunks - 1) * ch + cs.r16(m - (n_chunks - 1) * ch)   # every chunk stored
    assert top.size // 16 > gpp                                        # the place and fetch copies take two passes
    assert all(not pc[2] for pc in plane_coders(v7_of(planes))[:w - 1])    # the other planes code chunks
    v7, v8 = v7_of(planes), v8_of(planes, base)
    rc, got = gcp.encode(ctx, cands, 0, d, w, ch, 0)
    note()
    same(rc, got, v7, (w, passes, "v7"))
    del got
    rc, got_n, out = gcp.decode(ctx, v7, w, n)
    note()
    assert rc == 0 and got_n == n and np.array_equal(out[:n], d) and (out[n:] == SENTINEL).all(), (w, passes, "v7 decode")
    del out
    rc, got = gcd.encode(ctx, cands, 0, x, base, w, ch, 0)
    note()
    same(rc, got, v8, (w, passes, "v8"))
    del got
    rc, got_n, out, b = gcd.decode(ctx, v8, w, base, n, in_place=True)
    note()
    assert rc == 0 and got_n == n and np.array_equal(out[:n], x) and (out[n:] == SENTINEL).all(), (w, passes, "v8 decode")
    del out, b
    n_max = n + w * 16 * 40
    rc, got = gpv.varlen7(ctx, cands, 0, padded(d, n_max, 1), n, n_max, w, ch, 0)
    note()
    same(rc, got, v7, (w, passes, "varlen"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"w {w}, {passes} passes: m = {m} elements ({n / 2**20:.1f} MiB), {sms} SMs, {gpp} groups per pass; "
          f"stored plane {top.size} bytes; device memory in use at most {used[0] / 2**20:.0f} MiB")


# ---------------------------------------------------------------------------------------------------- 3. lane positions

N_PAIRS = 144                                                          # cd.crafted's 12 x 12 edge pairs, then random ones


def _crafted(w):
    x, b = cd.crafted(w, seed=w)
    return x[:N_PAIRS * w].reshape(N_PAIRS, w), b[:N_PAIRS * w].reshape(N_PAIRS, w)


def _check_v8(ctx, oracle_lib, x, base, w, case):
    d = cd.zigzag(x, base, w)
    want = v8_of(host_planes(oracle_lib, d, w, (WORD, 12), 32, CRC_BLOB), base)
    rc, got = gcd.encode(ctx, [CAND(WORD, 12)], 0, x, base, w, 32, CRC_BLOB)
    same(rc, got, want, case)
    for in_place in (False, True):
        rc, got_n, out, b = gcd.decode(ctx, want, w, base, x.size, in_place=in_place)
        assert rc == 0 and got_n == x.size, (case, in_place)
        assert np.array_equal(out[:x.size], x) and (out[x.size:] == SENTINEL).all(), (case, in_place)


@pytest.mark.parametrize("w", WIDTHS)
def test_every_lane_position(ctx, oracle_lib, w):
    px, pb = _crafted(w)
    rng = np.random.default_rng(40 + w)
    filler = lambda k: rng.integers(0, 256, (k, w), dtype=np.uint8)  # noqa: E731
    # groups: copy r is r fillers, the 144 pairs, then fillers to a whole group, so pair i sits at position (r + i) % 16
    xs, bs, idx = [], [], []
    for r in range(16):
        post = (16 - (r + N_PAIRS) % 16) % 16
        xs += [filler(r), px, filler(post)]
        bs += [filler(r), pb, filler(post)]
        idx += [-1] * r + list(range(N_PAIRS)) + [-1] * post
    x, base = np.concatenate(xs).reshape(-1), np.concatenate(bs).reshape(-1)
    idx = np.array(idx)
    assert idx.size % 16 == 0                                          # no tail: every pair goes through delta_forward
    reached = {(int(i), int(p)) for i, p in zip(idx, np.arange(idx.size) % 16) if i >= 0}
    assert len(reached) == N_PAIRS * 16
    _check_v8(ctx, oracle_lib, x, base, w, (w, "groups"))
    # tails: one group of fillers, then 15 pairs rotated by q, so pair i sits at tail position s for q = i - s
    reached = set()
    for q in range(N_PAIRS):
        sel = [(q + s) % N_PAIRS for s in range(15)]
        x = np.concatenate([filler(16), px[sel]]).reshape(-1)
        base = np.concatenate([filler(16), pb[sel]]).reshape(-1)
        assert x.size // w % 16 == 15
        reached |= {(i, s) for s, i in enumerate(sel)}
        _check_v8(ctx, oracle_lib, x, base, w, (w, "tail", q))
    assert len(reached) == N_PAIRS * 15


# ---------------------------------------------------------------------------------------------------- 4. plane-coder order

# (pair, which chunks stored): "coded" stores none, "stored" every chunk, "some" every other one
STATES = [((WORD, 12), "coded"), ((ALIAS, 9), "coded"), ((ALIAS, 16), "coded"), ((BYTE, 9), "coded"), ((BYTE, 14), "coded"),
          ((RANS64, 11), "coded"), ((RANS64, 16), "coded"), ((ALIAS, 12), "stored"), ((WORD, 12), "some")]


def de_bruijn(k):
    """a cyclic sequence over 0..k-1 in which every ordered pair (a, b) is consecutive once (order 2)"""
    a, seq = [0] * (2 * k), []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


def state_sequences():
    """windows of the linear de Bruijn sequence (82 states): eleven of w = 8, then one of w = 4 and one of w = 2, each
    overlapping the next by one state, so that their consecutive planes take every ordered pair of states"""
    s = de_bruijn(len(STATES))
    s = s + s[:1]
    out, i = [], 0
    for w in [8] * 11 + [4, 2]:
        out.append(s[i:i + w])
        i += w - 1
    assert i == len(s) - 1
    return out


def coder_order_container(oracle_lib, states, seed, ch, m):
    w = len(states)
    d = np.stack([_gen("text", m, seed + p) for p in range(w)], axis=1).reshape(-1)
    n_chunks = -(-m // ch)
    whiches = [[] if STATES[s][1] == "coded" else list(range(n_chunks)) if STATES[s][1] == "stored" else list(range(0, n_chunks, 2))
               for s in states]
    planes = host_planes(oracle_lib, d, w, [STATES[s][0] for s in states], ch, (seed // 10) & 1, whiches)
    x, base = delta_pair(d, w, seed + 99)
    v7, v8 = v7_of(planes), v8_of(planes, base)
    got = plane_coders(v7)
    assert [(c, sb) for c, sb, _, _ in got] == [STATES[s][0] for s in states]
    assert [("stored" if a else "some" if some else "coded") for _, _, a, some in got] == [STATES[s][1] for s in states]
    return d, x, base, v7, v8


def test_plane_coder_order_in_decode(ctx, oracle_lib):
    torch = _torch()
    seqs = state_sequences()
    pairs = {(a, b) for seq in seqs for a, b in zip(seq, seq[1:])}
    assert len(pairs) == len(STATES) ** 2 and [len(s) for s in seqs] == [8] * 11 + [4, 2]
    ch, m = 1024, 4 * 1024 + 100
    cases = [coder_order_container(oracle_lib, seq, 10 * i, ch, m) for i, seq in enumerate(seqs)]
    held = []
    for (d, x, base, v7, v8), seq in zip(cases, seqs):                 # every decode enqueued, one sync at the end
        w, n = len(seq), d.size
        d_v7, d_v8 = gbc._dev(v7), gbc._dev(v8)
        o7 = torch.full((n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        o8 = torch.full((n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        o8[:n] = torch.from_numpy(base.copy())                         # in place
        dn = torch.full((2,), -1, dtype=torch.int64, device="cuda")
        ctx.container_planes_decode_async(w, d_v7.data_ptr(), v7.size, o7.data_ptr(), n, dn.data_ptr())
        ctx.container_delta_decode_async(w, d_v8.data_ptr(), v8.size, o8.data_ptr(), o8.data_ptr(), n, dn.data_ptr() + 8)
        held.append((d_v7, d_v8, o7, o8, dn))
    assert _sync(ctx) == 0
    for i, ((d, x, base, v7, v8), (_, _, o7, o8, dn)) in enumerate(zip(cases, held)):
        n = d.size
        assert dn.cpu().tolist() == [n, n], i
        out7, out8 = o7.cpu().numpy(), o8.cpu().numpy()
        assert np.array_equal(out7[:n], d) and (out7[n:] == SENTINEL).all(), (i, seqs[i], "v7")
        assert np.array_equal(out8[:n], x) and (out8[n:] == SENTINEL).all(), (i, seqs[i], "v8")


# with tolerance 0 the word coder takes the ties (constant and two-symbol planes, then stored: it counts 0 bits for
# one symbol), the byte coder the plane whose rare symbol 14 bits hold as well as 16, the alias coder the skewed ones
CHOICE_LIST = [CAND(WORD, 12), CAND(BYTE, 14), CAND(ALIAS, 16), CAND(RANS64, 15)]


def test_plane_coder_choice_in_encode(ctx):
    ch, m, w = 8192, 8 * 8192 + 9, 8
    rng = np.random.default_rng(4)
    p = 1.0 / np.arange(1, 201) ** 1.1
    rare = np.zeros(m, np.uint8)
    rare[::1024] = 1
    planes = [rng.integers(0, 256, m, dtype=np.uint8), np.full(m, 7, np.uint8), rare,
              np.minimum(rng.geometric(0.5, m) - 1, 255), np.minimum(rng.geometric(0.2, m) - 1, 255),
              np.minimum(rng.geometric(0.05, m) - 1, 255), rng.choice(200, m, p=p / p.sum()),
              np.where(rng.random(m) < 0.3, 9, 200)]
    data = np.stack([np.asarray(pl).astype(np.uint8) for pl in planes], axis=1).reshape(-1)
    want = gcp.expected(ctx, CHOICE_LIST, 0, data, w, ch, CRC_BLOB)
    rc, got = gcp.encode(ctx, CHOICE_LIST, 0, data, w, ch, CRC_BLOB)
    same(rc, got, want, "eight distributions")
    coders = plane_coders(want)
    print("plane (coder, scale_bits, all stored, some stored):", coders)
    assert len({c for c, _, _, _ in coders}) >= 3, coders
    assert coders[0][2], coders                                         # uniform: every chunk stored
    rc, got_n, out = gcp.decode(ctx, want, w, data.size)
    assert rc == 0 and got_n == data.size and np.array_equal(out[:data.size], data)


# ---------------------------------------------------------------------------------------------------- 5. decode bounds

def decode8(ctx, buf, w, base, out_cap, size, in_place, junk):
    """(sync code, *d_n, out region [out_cap + 64], base region [max(n, out_cap) + 64]) on the host.  The base's
    allocation holds base, then junk over [n, out_cap), then sentinel bytes; out is that allocation in place, else a
    sentinel-filled one"""
    torch = _torch()
    n = base.size
    b = np.full(max(n, out_cap) + 64, SENTINEL, np.uint8)
    b[:n] = base
    if out_cap > n:
        b[n:out_cap] = junk[:out_cap - n]
    d_base = torch.from_numpy(b).cuda()
    d_out = d_base if in_place else torch.full((out_cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_buf = gbc._dev(buf)
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = ctx.lib.dll.rb200_container_delta_decode_async(ctx.h, w, d_buf.data_ptr(), size, d_base.data_ptr(), d_out.data_ptr(), out_cap,
                                                        d_n.data_ptr())
    if rc == 0:
        rc = _sync(ctx)
    return rc, int(d_n.item()), d_out[:out_cap + 64].cpu().numpy(), d_base.cpu().numpy()


BOUND_CH = 1024


@pytest.fixture(scope="module")
def bounded(oracle_lib):
    """per width: (d, x, base, v7, v8) of m = 16 * 200 + 9 elements at chunks of 1024, the whole groups geometric (coded
    chunks, so that the container is well below the bound)"""
    out = {}
    for w in WIDTHS:
        m = 16 * 200 + 9
        d = ragged(m, w, 70 + w)
        d[:16 * 200 * w] = np.minimum(np.random.default_rng(w).geometric(0.3, 16 * 200 * w) - 1, 127)
        x, base = delta_pair(d, w, 80 + w)
        planes = host_planes(oracle_lib, d, w, (WORD, 12), BOUND_CH, CRC_BLOB)
        out[w] = d, x, base, v7_of(planes), v8_of(planes, base)
    return out


@pytest.mark.parametrize("w", WIDTHS)
def test_decode_bounds(ctx, w, bounded):
    d, x, base, v7, v8 = bounded[w]
    n = d.size
    bound = api.container_planes_bound(n, w, BOUND_CH)
    assert bound > v7.size + 15
    junk = np.random.default_rng(w).integers(0, 256, 3 * n, dtype=np.uint8)
    assert junk[0] != SENTINEL
    for out_cap in (n, n + 1, n + w - 1, n + 16, 3 * n):
        for size in [v7.size + e for e in range(16)] + [bound]:
            case = (w, out_cap, size)
            pad = np.random.default_rng(size).integers(0, 256, size - v7.size, dtype=np.uint8)     # bytes past the container
            rc, got_n, out = gcp.decode(ctx, np.concatenate([v7, pad]), w, out_cap)
            assert rc == 0 and got_n == n, case
            assert np.array_equal(out[:n], d) and (out[n:] == SENTINEL).all(), case
            for in_place in (False, True):
                rc, got_n, out, b = decode8(ctx, np.concatenate([v8, pad]), w, base, out_cap, size, in_place, junk)
                assert rc == 0 and got_n == n, (case, in_place, rc)
                assert np.array_equal(out[:n], x), (case, in_place)
                rest = junk[:out_cap - n] if in_place else np.full(out_cap - n, SENTINEL, np.uint8)
                assert np.array_equal(out[n:out_cap], rest) and (out[out_cap:] == SENTINEL).all(), (case, in_place)
                if not in_place:
                    assert np.array_equal(b[:n], base) and np.array_equal(b[n:out_cap], junk[:out_cap - n]), case


@pytest.mark.parametrize("w", WIDTHS)
def test_decode_rejects_at_the_bounds(ctx, w, bounded):
    d, x, base, v7, v8 = bounded[w]
    n = d.size
    junk = np.random.default_rng(w).integers(0, 256, n, dtype=np.uint8)

    def intact():
        rc, got_n, out = gcp.decode(ctx, v7, w, n)
        assert rc == 0 and got_n == n and np.array_equal(out[:n], d)
        rc, got_n, out, _ = decode8(ctx, v8, w, base, n, v8.size, True, junk)
        assert rc == 0 and got_n == n and np.array_equal(out[:n], x)

    for out_cap in (0, w - 1, n - w):
        rc, got_n, out = gcp.decode(ctx, v7, w, out_cap)
        assert rc == E_SPACE and got_n == n and (out == SENTINEL).all(), (out_cap, "v7")
        for in_place in (False, True):
            rc, got_n, out, b = decode8(ctx, v8, w, base, out_cap, v8.size, in_place, junk)
            assert rc == E_SPACE and got_n == n, (out_cap, in_place, rc)
            assert np.array_equal(b[:n], base) and (b[n:] == SENTINEL).all(), (out_cap, in_place)
            if not in_place:
                assert (out == SENTINEL).all(), out_cap
        intact()
    for size in (0, 63, 64 + 16 * w - 1, 64 + 16 * w):
        rc, got_n, out = gcp.decode(ctx, v7, w, n, size=size)
        assert rc == E_STREAM and (out == SENTINEL).all(), (size, "v7")
        for in_place in (False, True):
            rc, got_n, out, b = decode8(ctx, v8, w, base, n, size, in_place, junk)
            assert rc == E_STREAM and np.array_equal(b[:n], base), (size, in_place, rc)
            if not in_place:
                assert (out == SENTINEL).all(), size
        intact()


@pytest.mark.parametrize("w", WIDTHS)
def test_overlap_rule_at_its_boundary(ctx, w, bounded):
    torch = _torch()
    d, x, base, v7, v8 = bounded[w]
    n = d.size
    out_cap = cs.r16(n) + 16                                            # pointers stay 16-byte aligned
    lib = ctx.lib.dll
    d_buf = gbc._dev(v8)
    d_n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    arena = torch.full((3 * out_cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    bp = arena.data_ptr() + out_cap
    arena[out_cap:out_cap + n] = torch.from_numpy(base.copy())
    before = ctx.launches
    for shift in (out_cap - 16, -out_cap + 16):
        assert lib.rb200_container_delta_decode_async(ctx.h, w, d_buf.data_ptr(), v8.size, bp, bp + shift, out_cap, d_n.data_ptr()) == E_ARG
    assert ctx.launches == before and _sync(ctx) == 0
    for shift in (out_cap, -out_cap):                                   # adjacent: accepted
        assert lib.rb200_container_delta_decode_async(ctx.h, w, d_buf.data_ptr(), v8.size, bp, bp + shift, out_cap, d_n.data_ptr()) == 0
        assert _sync(ctx) == 0 and int(d_n.item()) == n, shift
        a = arena.cpu().numpy()
        o = out_cap + shift
        assert np.array_equal(a[o:o + n], x), shift
        assert np.array_equal(a[out_cap:out_cap + n], base) and (a[out_cap + n:2 * out_cap] == SENTINEL).all(), shift
        arena[o:o + out_cap] = SENTINEL


# ---------------------------------------------------------------------------------------------------- 6. 16-byte alignment

@pytest.mark.parametrize("w", WIDTHS)
def test_pointers_16_past_32_byte_alignment(ctx, oracle_lib, w):
    torch = _torch()
    ch, m = 1024, 16 * 200 + 13
    d = ragged(m, w, 90 + w)
    d[: 16 * 100 * w] = np.minimum(np.random.default_rng(w).geometric(0.3, 16 * 100 * w) - 1, 127)   # coded chunks too
    x, base = delta_pair(d, w, 91 + w)
    n = d.size
    planes = host_planes(oracle_lib, d, w, (BYTE, 14), ch, CRC_BLOB)
    v7, v8 = v7_of(planes), v8_of(planes, base)
    assert any(not pc[2] for pc in plane_coders(v7))
    cands = [CAND(BYTE, 14)]
    cap = api.container_planes_bound(n, w, ch)
    n_max = n + 16 * w
    cap_max = api.container_planes_bound(n_max, w, ch)
    for k in (0, 16, 48, 80):
        assert k % 32 in (0, 16)
        at = lambda a: gg._dev_at(a, k)                                 # noqa: E731
        d_in, d_x, d_base = at(d), at(x), at(base)
        d_pad = gg._dev_at(np.concatenate([d, np.zeros(n_max - n, np.uint8)]), k)
        d_n = torch.tensor([0, n], dtype=torch.int64, device="cuda")
        outs = {}
        for name in ("v7", "varlen", "v8"):
            d_out = torch.full((k + cap_max + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
            if name == "v7":
                ctx.container_planes_encode_async(cands, 0, w, d_in.data_ptr() + k, n, ch, CRC_BLOB, d_out.data_ptr() + k, cap)
            elif name == "varlen":
                ctx.container_planes_encode_varlen_async(cands, 0, w, d_pad.data_ptr() + k, d_n.data_ptr() + 8, n_max, ch, CRC_BLOB,
                                                         d_out.data_ptr() + k, cap_max)
            else:
                ctx.container_delta_encode_async(cands, 0, w, d_x.data_ptr() + k, d_base.data_ptr() + k, n, ch, CRC_BLOB,
                                                 d_out.data_ptr() + k, cap)
            rc = _sync(ctx)
            got = d_out.cpu().numpy()
            assert (got[:k] == SENTINEL).all(), (w, k, name)
            same(rc, got[k:], v8 if name == "v8" else v7, (w, k, name))
            outs[name] = d_out
        d_o7 = torch.full((k + n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_o8 = torch.full((k + n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        ctx.container_planes_decode_async(w, outs["v7"].data_ptr() + k, v7.size, d_o7.data_ptr() + k, n, d_n.data_ptr())
        ctx.container_delta_decode_async(w, outs["v8"].data_ptr() + k, v8.size, d_base.data_ptr() + k, d_o8.data_ptr() + k, n,
                                         d_n.data_ptr() + 8)
        assert _sync(ctx) == 0 and d_n.cpu().tolist() == [n, n], (w, k)
        for name, o, want in (("v7", d_o7, d), ("v8", d_o8, x)):
            got = o.cpu().numpy()
            assert (got[:k] == SENTINEL).all() and np.array_equal(got[k:k + n], want) and (got[k + n:] == SENTINEL).all(), (w, k, name)
        ctx.container_delta_decode_async(w, outs["v8"].data_ptr() + k, v8.size, d_base.data_ptr() + k, d_base.data_ptr() + k, n)
        assert _sync(ctx) == 0
        got = d_base.cpu().numpy()
        assert (got[:k] == SENTINEL).all() and np.array_equal(got[k:k + n], x) and (got[k + n:] == SENTINEL).all(), (w, k, "in place")


# ---------------------------------------------------------------------------------------------------- 7. queued calls

def test_queued_calls_of_growing_geometry(cuda_box, oracle_lib):
    """on a fresh context, so that every call grows a workspace while the calls before it are in flight"""
    torch = _torch()
    ch = 1024
    d1 = ragged(16 * 500 + 5, 2, 1)                                    # 1: version 8 encode, w 2
    x1, b1 = delta_pair(d1, 2, 2)
    d2 = ragged(16 * 700 + 11, 8, 3)                                   # 2: version 7 decode, w 8
    v7_2 = v7_of(host_planes(oracle_lib, d2, 8, (WORD, 12), ch))
    cap3 = 3 * d2.size                                                 # 3: version 8 in place of 1's container, out_cap above 2's
    d4 = ragged(16 * 6000 + 9, 4, 4)                                   # 4: version 7 varlen encode, w 4
    n4_max = d4.size + 4 * 16 * 9
    assert d1.size < d2.size < cap3 < d4.size < n4_max
    cands = [CAND(BYTE, 14)]
    cap1 = api.container_planes_bound(d1.size, 2, ch)
    cap4 = api.container_planes_bound(n4_max, 4, ch)

    def run(c, one_at_a_time):
        t = {"x1": gbc._dev(x1), "b1": gbc._dev(b1), "v7_2": gbc._dev(v7_2), "d4": padded(d4, n4_max, 5)}
        t["o1"] = torch.full((cap1 + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        t["o2"] = torch.full((d2.size + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        t["o3"] = torch.full((cap3 + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        t["o3"][:b1.size] = torch.from_numpy(b1.copy())
        t["o4"] = torch.full((cap4 + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        t["n"] = torch.tensor([-1, -1, d4.size], dtype=torch.int64, device="cuda")
        calls = [lambda: c.container_delta_encode_async(cands, 0, 2, t["x1"].data_ptr(), t["b1"].data_ptr(), d1.size, ch, CRC_BLOB,
                                                        t["o1"].data_ptr(), cap1),
                 lambda: c.container_planes_decode_async(8, t["v7_2"].data_ptr(), v7_2.size, t["o2"].data_ptr(), d2.size, t["n"].data_ptr()),
                 lambda: c.container_delta_decode_async(2, t["o1"].data_ptr(), cap1, t["o3"].data_ptr(), t["o3"].data_ptr(), cap3,
                                                        t["n"].data_ptr() + 8),
                 lambda: c.container_planes_encode_varlen_async(cands, 0, 4, t["d4"].data_ptr(), t["n"].data_ptr() + 16, n4_max, ch, 0,
                                                                t["o4"].data_ptr(), cap4)]
        for call in calls:
            call()
            if one_at_a_time:
                assert _sync(c) == 0
        assert _sync(c) == 0
        return {k: t[k].cpu().numpy() for k in ("o1", "o2", "o3", "o4", "n")}

    c = rb.Context(0)
    try:
        queued = run(c, False)
    finally:
        c.close()
    c = rb.Context(0)
    try:
        alone = run(c, True)
    finally:
        c.close()
    for k in alone:
        assert np.array_equal(queued[k], alone[k]), k
    want1 = v8_of(host_planes(oracle_lib, cd.zigzag(x1, b1, 2), 2, (BYTE, 14), ch, CRC_BLOB), b1)
    same(0, queued["o1"], want1, "call 1")
    assert queued["n"][:2].tolist() == [d2.size, d1.size]
    assert np.array_equal(queued["o2"][:d2.size], d2) and (queued["o2"][d2.size:] == SENTINEL).all()
    assert np.array_equal(queued["o3"][:d1.size], x1) and (queued["o3"][d1.size:] == SENTINEL).all()
    same(0, queued["o4"], v7_of(host_planes(oracle_lib, d4, 4, (BYTE, 14), ch)), "call 4")
