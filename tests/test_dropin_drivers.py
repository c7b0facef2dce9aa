"""BASELINE config 1 / SURVEY 8(b).1: the reference's drivers must build UNCHANGED against
this repo's source-level headers (include/rans_byte.h, rans64.h, rans_word_sse41.h,
platform.h) and print the reference's known-answer sizes and 'decode ok!'.

oracle/Makefile builds the drivers (oracle/_ref/dropin_*) where the reference sources are
present, from a temporary copy (a quoted #include looks beside the including file first, so
they cannot be compiled in place), and records the headers each one included
(oracle/_ref/dropin_*.deps) -- nothing from the reference is ever copied into the repo.  The
drivers run here on book1, recovered from tests/golden/book1_n32.npz.
"""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BUILD = os.path.join(ROOT, "oracle", "_ref")

DRIVERS = [
    ("main.cpp", [], [435113, 435117]),                    # README:48,62
    ("main64.cpp", [], [435116, 435120]),                  # README:82,96
    ("main_simd.cpp", ["-msse4.1"], [435604, 435606, 435626]),   # README:110 for the 8-way stream
    ("main_alias.cpp", [], [435059, 435063]),
]


@pytest.mark.parametrize("src,flags,sizes", DRIVERS)
def test_reference_driver_builds_unchanged_and_round_trips(tmp_path, book1, src, flags, sizes):
    stem = src[:-len(".cpp")]
    exe = os.path.join(REF_BUILD, "dropin_" + stem)
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (the reference sources were not available to build())")
    with open(exe + ".flags") as f:                      # built with the reference Makefile's flags for this driver
        assert f.read().split() == flags
    # make sure it really used OUR headers: every header it included is one of include/*.h
    with open(exe + ".deps") as f:
        deps = f.read().replace("\\\n", " ").split()
    assert deps[:2] == [stem + ".o:", src]
    headers = deps[2:]
    assert headers and all(h.startswith("../include/") and os.path.exists(os.path.join(ROOT, "include", h[11:])) for h in headers), deps
    book1.tofile(tmp_path / "book1")
    out = subprocess.run([exe], cwd=tmp_path, capture_output=True, text=True, timeout=120).stdout
    assert "ERROR" not in out and out.count("decode ok!") == len(sizes), out[-400:]
    assert [int(x) for x in re.findall(r"rANS: (\d+) bytes", out)] == sizes
