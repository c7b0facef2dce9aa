"""Every decoder rejects a corrupt stream and a corrupt directory entry with E_STREAM (-4), and its context then decodes
the intact container correctly, twice in a row (the persistent decoders' work counter has re-armed).

Everything runs in DEVICE mode, where no host code looks at the directory before the kernel does: what rejects the
directory cases is the kernel's own check of its entry, which leaves the chunk's output untouched."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WORD, BYTE, ALIAS, RANS64 = 0, 1, 2, 3
CHUNK = 4096
N = 4 * CHUNK + 1000                     # five chunks, the last one ragged

# name, coder, scale_bits, data kind, stream unit bytes (the alignment a chunk start must have)
FLAT = [("word", WORD, 12, "zipf", 2),
        ("word-wide", WORD, 12, "const", 2),      # single-symbol model: freq 4096 (the WIDE kernel)
        ("alias16", ALIAS, 16, "zipf", 1),
        ("alias10", ALIAS, 10, "zipf", 1),        # no specialised instance for scale_bits 10
        ("byte14", BYTE, 14, "zipf", 1),
        ("byte10", BYTE, 10, "text", 1),
        ("rans64", RANS64, 14, "zipf", 4)]


def _flipped(blob, offs, c):
    """blob with bytes inside chunk c's stream flipped: past the header, or the header itself when that is all the
    stream holds (a single-symbol model never renormalises)"""
    lo, hi = int(offs[c]), int(offs[c + 1]) & ~15
    if hi - lo > 400:
        lo, hi = lo + 128, lo + 400
    bad = blob.copy()
    bad[lo:hi] ^= 0x5A
    return bad


def _bad_directories(offs, blob_size, unit):
    """(chunk, offsets): directories that are corrupt for that one chunk's entry and leave every other chunk intact"""
    last = offs.size - 2
    past = offs.copy()
    past[-1] = blob_size + 16                      # the last stream ends past the blob
    short = offs.copy()
    short[-1] = offs[-2] + 16                      # the last stream ends before its header (128 or 256 bytes) does
    cases = [(last, past), (last, short)]
    if unit > 1:
        odd = offs.copy()
        odd[1] += unit // 2                        # chunk 1 starts inside a renormalisation unit; chunk 0 keeps its end
        cases.append((1, odd))
    return cases


def _device_run(ctx, n, decode):
    """run(blob, offs) -> (output, RansError or None): decode(blob_ptr, blob_size, offsets_ptr, out_ptr) on device
    copies, into a zeroed output"""
    import torch
    import ryg_rans_b200 as rb

    def run(blob, offs):
        d_blob = torch.from_numpy(blob).cuda()
        d_offs = torch.from_numpy(offs.view(np.int64)).cuda()
        out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        err = None
        try:
            decode(d_blob.data_ptr(), blob.size, d_offs.data_ptr(), out.data_ptr())
            ctx.sync()
        except rb.RansError as e:
            err = e
        return out.cpu().numpy(), err
    return run


def _check_decoder(run, data, blob, offs, unit, flip_chunks):
    def clean_twice(what):
        for rep in range(2):
            out, err = run(blob, offs)
            assert err is None and np.array_equal(out, data), (what, rep)

    clean_twice("before")
    for c in flip_chunks:
        _, err = run(_flipped(blob, offs, c), offs)
        assert err is not None and err.code == -4, ("flip", c)
        clean_twice(("flip", c))
    # The end-of-stream check would reject most bad entries as well; the chunk's untouched output shows that the
    # kernel's directory check rejected it before anything was decoded.
    for c, o in _bad_directories(offs, blob.size, unit):
        out, err = run(blob, o)
        assert err is not None and err.code == -4, ("directory", c)
        lo, hi = c * CHUNK, min((c + 1) * CHUNK, data.size)
        assert data[lo:hi].any() and not out[lo:hi].any(), ("chunk decoded despite its directory entry", c)
        clean_twice(("directory", c))


@pytest.mark.parametrize("name,coder,sb,kind,unit", FLAT, ids=[c[0] for c in FLAT])
def test_flat_decoder_rejects(gpu_ctx, oracle_lib, gen, name, coder, sb, kind, unit):
    data = gen(kind, N, 31)
    freqs, _ = oracle_lib.model(data, sb)
    model = gpu_ctx.model(coder, sb, freqs)
    blob, offs = gpu_ctx.encode_host(model, data, CHUNK)
    run = _device_run(gpu_ctx, N, lambda b, bs, o, out: gpu_ctx.decode_device(model, b, bs, o, CHUNK, out, N))
    _check_decoder(run, data, blob, offs, unit, [1])
    model.close()


def test_block_decoder_rejects(gpu_ctx, gen):
    """Per-block decoder: block 0 has a normal model, block 1 a single-symbol one (the WIDE step)."""
    import torch
    n_blocks, block_size = 3, 4 * CHUNK
    data = np.concatenate([gen("zipf", block_size, 41), gen("const", block_size, 42), gen("uniform", block_size, 43)])
    blob, offs, freqs = gpu_ctx.blocks_model_encode_host(data, n_blocks, block_size, CHUNK)
    assert freqs[1].max() == 4096
    d_freqs = torch.from_numpy(freqs.view(np.int16)).cuda()
    run = _device_run(gpu_ctx, data.size, lambda b, bs, o, out: gpu_ctx.blocks_decode_device(
        b, bs, o, d_freqs.data_ptr(), n_blocks, block_size, CHUNK, out))
    _check_decoder(run, data, blob, offs, 2, [1, block_size // CHUNK + 1])
