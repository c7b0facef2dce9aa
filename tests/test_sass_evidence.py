"""The shipped library really contains what DESIGN.md says about the staging of the decoders (north_star: tables staged
via TMA / cp.async): checked in the SASS of the built .so with cuobjdump -- no GPU needed.  VERDICT r1 (G2) found none of
these mnemonics in round 1's library."""
import os
import re
import shutil
import subprocess
import sys

import pytest

import ryg_rans_b200 as rb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not installed")
    import sass_steps
    rb.build()
    sass = subprocess.run([CUOBJDUMP, "-sass", rb.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return sass_steps.functions(sass)


def _mnemonics(body):
    out = {}
    for _, ins in body:
        m = re.match(r"(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ins)
        if m:
            out[m.group(1)] = out.get(m.group(1), 0) + 1
    return out


def test_word_decoder_stages_with_tma_and_cp_async(kernels):
    names = [k for k in kernels if "word_decode_tma_kernel" in k]
    assert len(names) == 2                                    # <DecShip, false> and the freq-4096 WIDE variant
    for k in names:
        mn = _mnemonics(kernels[k])
        assert mn.get("UBLKCP.S.G", 0) >= 1                   # cp.async.bulk: the 16 KiB table, once per CTA
        assert any(m.startswith("SYNCS.ARRIVE.TRANS64") for m in mn) and any(m.startswith("SYNCS.PHASECHK") for m in mn)   # its mbarrier
        assert mn.get("LDGSTS.E.BYPASS.128", 0) >= 4          # cp.async.cg 16 B per lane: the stream ring
        assert mn.get("LDGDEPBAR", 0) >= 1 and mn.get("DEPBAR.LE", 0) >= 1      # commit_group / wait_group


def test_alias_decoder_ring_is_cp_async(kernels):
    names = [k for k in kernels if "alias_decode_persist_kernel" in k]
    assert len(names) == 4                                    # scale_bits 16, 14, 12 and the runtime fallback
    for k in names:
        mn = _mnemonics(kernels[k])
        assert mn.get("LDGSTS.E.BYPASS.128", 0) >= 4 and mn.get("DEPBAR.LE", 0) >= 1


def test_main_loop_step_lengths(kernels):
    """The unrolled main loops keep the instruction counts the profiles quote (a regression guard for compiler or
    source changes: 17 per 32 symbols in the word decoder, 29-30 in the alias decoder)."""
    import sass_steps
    tma = next(v for k, v in kernels.items() if "word_decode_tma_kernel" in k and "Lb0EEEv" in k)
    ali = next(v for k, v in kernels.items() if "alias_decode_persist_kernelILj16E" in k)
    assert len(sass_steps.step_between(tma, "STG.E.U8", 2)) <= 17
    assert len(sass_steps.step_between(ali, "STG.E.U8", 2)) <= 30


# The word coder's per-block decode step (vote to vote), opcodes in issue order.  block_decode_planned_kernel<word, 12>
# keeps the order of the one-CTA-per-block kernel it replaced only with its table in static shared memory and the table
# address taken per chunk (container_decode.cuh); a change to the shared per-block body that moves either step shows here.
WORD_BLOCK_STEP = {
    "block_decode_kernelILj0ELj12E": [
        "VOTE.ANY", "LOP3.LUT", "POPC", "IMAD", "LOP3.LUT", "LDS.U16", "PRMT", "LOP3.LUT", "SHF.R.U32.HI", "IMAD", "LDS",
        "SHF.R.U32.HI", "STG.E.U8", "SHF.R.U32.HI", "LOP3.LUT", "IMAD", "POPC", "ISETP.GE.U32.AND", "IMAD"],
    "block_decode_planned_kernelILj0ELj12E": [
        "VOTE.ANY", "LOP3.LUT", "POPC", "POPC", "IMAD", "IMAD", "LOP3.LUT", "LDS.U16", "PRMT", "LOP3.LUT", "SHF.R.U32.HI",
        "IMAD", "LDS", "SHF.R.U32.HI", "STG.E.U8", "SHF.R.U32.HI", "LOP3.LUT", "IMAD", "ISETP.GE.U32.AND"],
}


@pytest.mark.parametrize("name", sorted(WORD_BLOCK_STEP))
def test_word_block_decode_step(kernels, name):
    import sass_steps
    body = next(v for k, v in kernels.items() if name in k)
    step = sass_steps.step_between(body, "VOTE.ANY", 5)
    assert [re.match(r"(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ins).group(1) for _, ins in step] == WORD_BLOCK_STEP[name]
