"""The GEOM instances of rb200_container_stored_encode_varlen_async (version 6) and
rb200_container_blocks_stored_encode_varlen_async (version 5) spill no more than the flags-off instance of the same
stage: every such function has no more local-memory stores and loads in its SASS than its twin.  The plan kernel, which
has no twin, does not spill.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

TWINS = [
    ("stored_varlen_plan_kernel", None),
    ("chunks_store_varlen_kernel", "chunks_store_kernel"),
    ("chunks_stored_compaction_varlen_kernel", "chunks_stored_compaction_kernel"),
    ("container_stored_finish_varlen_kernel", "container_stored_finish_kernel"),
    ("blocks_store_varlen_kernel", "blocks_store_kernel"),
    ("compact_stored_varlen_kernel", "compact_stored_kernel"),
    ("container_blocks_stored_finish_varlen_kernel", "container_blocks_stored_finish_kernel"),
    ("block_coder_encode_kernelILj0ELj12ELb1ELb1ELb1E", "block_coder_encode_kernelILj0ELj12ELb0ELb0ELb0E"),
]

kernels = tvs.kernels


@pytest.mark.parametrize("new,twin", TWINS)
def test_stored_varlen_kernels_spill_no_more_than_their_twins(kernels, new, twin):
    got = tvs._local(tvs._one(kernels, new))
    want = (0, 0) if twin is None else tvs._local(tvs._one(kernels, twin))
    assert got[0] <= want[0] and got[1] <= want[1], (new, got, twin, want)
