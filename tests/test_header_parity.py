"""Source-level API parity, function by function (SURVEY 8b tier 1).

tests/test_dropin_drivers.py shows that the reference's drivers build unchanged against include/*.h and print the
known-answer sizes on book1.  This goes below that: a C++ harness compiles the SAME test body twice -- against the
reference's own headers and against ours -- and requires every produced stream, every `RansEncSymbol` /
`Rans64EncSymbol` / `RansDecSymbol` field (over the whole parameter range the reference allows), every table row and
every decoder state and cursor to be identical, for the scalar, the reciprocal and the SSE4.1 code paths.
The harnesses include the reference where it lies, so oracle/Makefile builds them (oracle/_ref/header_parity_*) where
the reference sources are present; the tests run those binaries.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BUILD = os.path.join(ROOT, "oracle", "_ref")


def _harness(name):
    exe = os.path.join(REF_BUILD, name)
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref not built (the reference sources were not available to build())")
    return exe


@pytest.mark.parametrize("opt", ["-O0", "-O3"])
def test_every_api_function_matches_the_reference(tmp_path, opt):
    out = subprocess.run([_harness("header_parity" + opt.replace("-", "_"))], capture_output=True, text=True, timeout=600,
                         cwd=tmp_path)
    assert out.returncode == 0, out.stdout[-3000:]
    lines = out.stdout.strip().splitlines()
    assert len(lines) == 9 and all(" ok: " in ln for ln in lines), out.stdout


@pytest.mark.parametrize("opt", ["-O0", "-O3"])
def test_rans_alias_header_matches_the_reference_driver(tmp_path, opt):
    """include/rans_alias.h (SURVEY section 7 step 2): the alias tables, RansEncPutAlias and RansDecGetAlias against the
    reference's own code in main_alias.cpp -- tables equal field by field, encoder states, streams, decoder states and
    cursors identical at scale_bits 8 / 11 / 14 / 16, our step functions also driven on the reference's SymbolStats."""
    out = subprocess.run([_harness("header_parity_alias" + opt.replace("-", "_"))], capture_output=True, text=True,
                         timeout=600, cwd=tmp_path)
    assert out.returncode == 0, out.stdout[-3000:]
    lines = out.stdout.strip().splitlines()
    assert len(lines) == 16 and all("rans_alias.h ok" in ln for ln in lines), out.stdout
