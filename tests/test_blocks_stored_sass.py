"""The STORED instances of rb200_container_blocks_stored_encode_async and rb200_container_blocks_stored_decode_async
(version 5) and the gated split word encoder they run spill no more than the flags-off instance of the same stage:
every such function has no more local-memory stores and loads in its SASS than its twin.  The kernels with no twin
(the store rule and the one-pair record) do not spill.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

DECODERS = ((0, 12), (1, 14), (1, 12), (1, 0), (3, 0), (2, 14), (2, 12), (2, 0))
TWINS = (
    [("blocks_store_kernel", None), ("blocks_one_pair_kernel", None),
     ("block_coder_encode_kernelILj0ELj12ELb1ELb1ELb0E", "block_coder_encode_kernelILj0ELj12ELb0ELb0ELb0E"),
     ("compact_stored_kernel", "compact_kernelILb0ELb0E"),
     ("container_plan_kernelILb1E", "container_plan_kernelILb0E"),
     ("container_prefix_check_kernelILb1E", "container_prefix_check_kernelILb0E"),
     ("container_blocks_stored_finish_kernel", "container_blocks_finish_kernelILb0E")]
    + [(f"block_decode_planned_kernelILj{c}ELj{sb}ELb1E", f"block_decode_planned_kernelILj{c}ELj{sb}ELb0E") for c, sb in DECODERS]
)

kernels = tvs.kernels


@pytest.mark.parametrize("new,twin", TWINS)
def test_stored_kernels_spill_no_more_than_their_twins(kernels, new, twin):
    got = tvs._local(tvs._one(kernels, new))
    want = (0, 0) if twin is None else tvs._local(tvs._one(kernels, twin))
    assert got[0] <= want[0] and got[1] <= want[1], (new, got, twin, want)
