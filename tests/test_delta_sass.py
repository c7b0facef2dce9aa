"""The kernels of rb200_container_delta_encode_async and rb200_container_delta_decode_async (version 8) do not spill: no
local-memory stores or loads in their SASS.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

NEW = ([f"delta_split_kernelILi{w}E" for w in (2, 4, 8)] + [f"delta_interleave_kernelILi{w}E" for w in (2, 4, 8)]
       + ["delta_finish_kernel", "delta_plan_kernel", "delta_verdict_kernel", "delta_check_kernel"])

kernels = tvs.kernels


@pytest.mark.parametrize("name", NEW)
def test_delta_kernels_do_not_spill(kernels, name):
    assert tvs._local(tvs._one(kernels, name)) == (0, 0), name
