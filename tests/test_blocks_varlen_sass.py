"""The kernels of rb200_container_blocks_model_encode_varlen_async spill no more than the shipped kernels they are built
around: every new function has no more local-memory stores and loads in its SASS than its twin of the fixed auto encode
(the 8-warp K5f instance keeps the shipped body's spill; every other one has none).  No GPU needed."""
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

# (new function, the shipped twin it is built around); a twin of None: the function has no twin and must not spill
TWINS = [
    ("blocks_varlen_plan_kernel", None),
    ("blocks_varlen_blob_len_kernel", None),
    ("blocks_choice_geom_kernel", "blocks_choice_kernel"),
    ("block_encode_fused_varlen_kernelILi8E", "block_encode_fused_gated_kernelILi8E"),
    ("block_encode_fused_varlen_kernelILi32E", "block_encode_fused_gated_kernelILi32E"),
    ("scan_tiles_blocks_kernel", "scan_tiles_kernelILb1ELb1E"),
    ("compact_blocks_kernel", "compact_kernelILb1ELb1E"),
    ("container_blocks_finish_varlen_kernel", "container_blocks_finish_chosen_kernel"),
] + [(f"block_coder_encode_varlen_kernelILj{c}ELj{sb}E", f"block_coder_encode_gated_kernelILj{c}ELj{sb}E")
     for c, sb in ((1, 0), (1, 12), (1, 14), (2, 0), (2, 12), (2, 14), (3, 0))]


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not installed")
    import sass_steps
    rb.build()
    sass = subprocess.run([CUOBJDUMP, "-sass", rb.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return sass_steps.functions(sass)


def _local(body):
    """(STL, LDL) instruction counts"""
    ops = [re.sub(r"^@!?U?P\d+\s+", "", ins) for _, ins in body]
    return sum(o.startswith("STL") for o in ops), sum(o.startswith("LDL") for o in ops)


def _one(kernels, part):
    """the function whose mangled name is part (a name, with its template arguments when it has any)"""
    base = part.split("I")[0]                                   # the kernels' names have no capital I
    needle = f"{len(base)}{part}" + ("" if base != part else "E")
    names = [k for k in kernels if k.startswith("_ZN5rb200") and needle in k]
    assert len(names) == 1, (part, names)
    return kernels[names[0]]


@pytest.mark.parametrize("new,twin", TWINS)
def test_new_kernels_spill_no_more_than_their_twins(kernels, new, twin):
    got = _local(_one(kernels, new))
    want = (0, 0) if twin is None else _local(_one(kernels, twin))
    assert got[0] <= want[0] and got[1] <= want[1], (new, got, twin, want)
