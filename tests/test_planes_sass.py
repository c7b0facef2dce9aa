"""The kernels of rb200_container_planes_encode_async and rb200_container_planes_decode_async (version 7) do not spill:
no local-memory stores or loads in their SASS.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

NEW = ([f"planes_split_kernelILi{w}E" for w in (2, 4, 8)] + [f"planes_interleave_kernelILi{w}E" for w in (2, 4, 8)]
       + ["planes_place_kernel", "planes_finish_kernel", "planes_plan_kernel", "planes_fetch_kernel", "planes_record_kernel",
          "planes_verdict_kernel"])

kernels = tvs.kernels


@pytest.mark.parametrize("name", NEW)
def test_planes_kernels_do_not_spill(kernels, name):
    assert tvs._local(tvs._one(kernels, name)) == (0, 0), name
