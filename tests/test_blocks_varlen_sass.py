"""The GATED and GEOM instances of the per-block container encodes (rb200_container_blocks_model_encode_auto_async and
its device-count form rb200_container_blocks_model_encode_varlen_async) spill no more than the flags-off instance of
the same stage: every such function has no more local-memory stores and loads in its SASS than the instance the fixed
calls run (the 8-warp K5f instances keep the shipped body's spill; every other one has none).  No GPU needed."""
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

# (GATED or GEOM instance, the flags-off instance of the same stage); None: the function has no flags-off instance and
# must not spill
CODER_SB = ((1, 0), (1, 12), (1, 14), (2, 0), (2, 12), (2, 14), (3, 0))
TWINS = (
    [("blocks_varlen_plan_kernel", None),
     ("varlen_blob_len_kernel", None),
     ("blocks_choice_kernelILb1E", "blocks_choice_kernelILb0E")]
    + [(f"block_encode_fused_kernelILb1ELi{w}ELb1ELb{geom}E", f"block_encode_fused_kernelILb1ELi{w}ELb0ELb0E")
       for w in (8, 32) for geom in (0, 1)]
    + [(f"{k}ILb{geom}ELb{gated}E", f"{k}ILb0ELb0E")
       for k in ("scan_tiles_kernel", "tile_prefix_kernel", "compact_kernel") for geom, gated in ((0, 1), (1, 0), (1, 1))]
    + [(f"container_blocks_finish_kernelILb{geom}E", "container_finish_kernelILb0ELb0E") for geom in (0, 1)]
    + [(f"block_coder_encode_kernelILj{c}ELj{sb}ELb1ELb1ELb{geom}E", f"block_coder_encode_kernelILj{c}ELj{sb}ELb1ELb0ELb0E")
       for c, sb in CODER_SB for geom in (0, 1)]
)


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
