#!/usr/bin/env python
"""Golden vectors: the REFERENCE's own 32-way streams of the seeded inputs the *_reference_stream_n32 GPU tests encode.

Made with the reference's primitives (oracle/_ref) where they can be built; each stream is checked to decode back to
its input with the reference's own decoder before it is stored.  The GPU tests compare the GPU's one-chunk container
against these streams byte for byte, so they need neither the reference nor oracle/_ref.  Run where oracle/_ref builds:

    python tests/golden/make_ref_streams.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import oracle  # noqa: E402
from conftest import _gen  # noqa: E402

# name: (coder, scale_bits, generator kind, n, seed) -- the inputs of tests/test_gpu_parity.py
CASES = {
    "word": (oracle.CODER_WORD, 12, "text", 50000, 5),
    "alias": (oracle.CODER_ALIAS, 16, "zipf", 60000, 6),
    "byte": (oracle.CODER_BYTE, 14, "text", 60000, 8),
    "rans64": (oracle.CODER_RANS64, 14, "text", 60000, 8),
}


def main():
    ref = oracle.Reference()
    out = {}
    for name, (coder, sb, kind, n, seed) in CASES.items():
        data = _gen(kind, n, seed)
        freqs, cum = ref.model(data, sb)
        stream = ref.encode(coder, data, freqs, cum, 32, sb)
        dec, used = ref.decode(coder, stream, data.size, freqs, cum, 32, sb)
        assert np.array_equal(dec, data) and used == stream.size, name
        out[f"{name}/freqs"] = freqs.astype(np.uint32)
        out[f"{name}/stream"] = stream
        print(name, n, "->", stream.size, "bytes")
    np.savez_compressed(os.path.join(HERE, "ref_streams_n32.npz"), **out)


if __name__ == "__main__":
    main()
