"""The kernels of rb200_container_planes_encode_varlen_async (version 7 with the length in device memory) spill no more
than the kernels of the fixed call whose bodies they run: every such function has no more local-memory stores and
loads in its SASS than its twin.  The plan kernel, which has no twin, does not spill.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

TWINS = ([("planes_varlen_plan_kernel", None), ("planes_finish_varlen_kernel", "planes_finish_kernel")]
         + [(f"planes_split_varlen_kernelILi{w}E", f"planes_split_kernelILi{w}E") for w in (2, 4, 8)])

kernels = tvs.kernels


@pytest.mark.parametrize("new,twin", TWINS)
def test_planes_varlen_kernels_spill_no_more_than_their_twins(kernels, new, twin):
    got = tvs._local(tvs._one(kernels, new))
    want = (0, 0) if twin is None else tvs._local(tvs._one(kernels, twin))
    assert got[0] <= want[0] and got[1] <= want[1], (new, got, twin, want)
