"""The kernels of rb200_container_tensors_encode_async and rb200_container_tensors_decode_async (version 9) do not spill:
no local-memory stores or loads in their SASS.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

NEW = ([f"tensors_split_kernelILi{w}E" for w in (2, 4, 8)] + [f"tensors_interleave_kernelILi{w}E" for w in (2, 4, 8)]
       + ["tensors_plan_kernel", "tensors_finish_kernel", "tensors_open_kernel", "tensors_check_kernel"])

kernels = tvs.kernels


@pytest.mark.parametrize("name", NEW)
def test_tensors_kernels_do_not_spill(kernels, name):
    assert tvs._local(tvs._one(kernels, name)) == (0, 0), name
