"""Host-built device tables (csrc/model_host.cpp), checked on the CPU by emulating the kernels' arithmetic.

The word encoder trusts `enc32` (32-bit reciprocal, exact only on x < freq << 20) whenever `enc32_ok` says so;
this test links the real table builder into a small C++ harness and checks, for EVERY frequency 1..4096, that
the flag is right and that both reciprocal forms give x / freq on the states the encoder can hold.
"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ryg_rans_b200", "csrc")

HARNESS = r'''
#include "tables.h"
#include "rans_b200.h"
#include <cstdio>
#include <cstdint>
#include <random>
using namespace rb200;

// the kernels' arithmetic (word_kernels.cuh: word_enc_expand / WordEncoder::step)
static uint32_t mulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static uint32_t q33(uint32_t x, WordEncEntry e)
{
    const uint32_t shift = (e.packed >> 25) & 0xfu;
    const uint64_t lo = (uint64_t)x + mulhi(x, e.magic);          // 33 bits: the funnel shift's carry word
    return (uint32_t)(lo >> shift);
}
static uint32_t q32(uint32_t x, WordEncEntry e) { return mulhi(x, e.magic) >> ((e.packed >> 25) & 0xfu); }

int main()
{
    std::mt19937_64 rng(7);
    int n_inexact = 0, first_inexact = 0;
    static WordDeviceTables t;
    for (uint32_t f = 1; f <= 4096; f++) {
        uint32_t freqs[256] = {0};
        freqs[5] = f;                                   // symbol 5 carries the frequency under test
        uint32_t rest = 4096 - f;
        freqs[9] = rest / 2;
        freqs[200] = rest - rest / 2;
        if (build_word_device_tables(freqs, t) != RB200_OK) { printf("build failed for %u\n", f); return 1; }
        const WordEncEntry e33 = t.enc[5], e32 = t.enc32[5];
        if ((e33.packed & 0x1fffu) != f || (e32.packed & 0x1fffu) != f) { printf("freq field %u\n", f); return 1; }
        // states the encoder divides: below freq << 20 (2^32 wraps to "always renormalise", leaving x < 2^16)
        const uint64_t bound = f == 4096 ? (1ull << 16) : ((uint64_t)f << 20);
        bool exact32 = true;
        auto check = [&](uint64_t x64) {
            if (x64 >= bound) return true;
            const uint32_t x = (uint32_t)x64;
            if (q33(x, e33) != x / f) { printf("33-bit reciprocal wrong: f=%u x=%u\n", f, x); return false; }
            uint32_t q = q32(x, e32);
            if (f == 1) {                               // mulhi(x, 2^32 - 1) = x - 1; the kernel adds 4095 to start
                if (x >= 1 && q != x - 1) exact32 = false;
            } else if (q != x / f) exact32 = false;
            return true;
        };
        for (uint64_t k = 0; k < 4096; k++) {           // top of the range, multiples of f and their neighbours
            if (!check(bound - 1 - k) || !check((bound / f - 1 - k % 64) * f + (f - 1)) || !check(k * f) || !check(k * f + f - 1)) return 1;
        }
        for (int k = 0; k < 20000; k++) if (!check(rng() % bound)) return 1;
        // any 32-bit x for the 33-bit form
        for (int k = 0; k < 2000; k++) { uint32_t x = (uint32_t)rng(); if (q33(x, e33) != x / f) { printf("33-bit wrong f=%u x=%u\n", f, x); return 1; } }
        const bool flagged_ok = t.enc32_ok != 0;        // freqs[9], freqs[200] <= 2048 are always exact, so the flag is about f
        if (flagged_ok && !exact32) { printf("enc32_ok set but inexact: f=%u\n", f); return 1; }
        if (!flagged_ok) { n_inexact++; if (!first_inexact) first_inexact = f; }
    }
    printf("inexact %d first %d\n", n_inexact, first_inexact);
    return 0;
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_word_encoder_reciprocals_exhaustive(tmp_path):
    src = tmp_path / "harness.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "harness"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src),
                           os.path.join(CSRC, "model_host.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:]
    # 383 frequencies (the first is 2964) need the 33-bit form; every other model takes the 2-instruction division
    assert out.stdout.strip() == "inexact 383 first 2964", out.stdout
