"""The STORED instances of rb200_container_stored_encode_async and rb200_container_stored_decode_async (version 6) spill
no more than the flags-off instance of the same stage: every such function has no more local-memory stores and loads in
its SASS than its twin.  The kernels with no twin (the store rule) do not spill.  No GPU needed."""
import pytest

import test_blocks_varlen_sass as tvs

V1_DECODERS = ([(f"word_decode_planned_kernelILb{w}ELb1E", f"word_decode_planned_kernelILb{w}ELb0E") for w in (0, 1)]
               + [(f"{k}_decode_planned_kernelILj{sb}ELb1E", f"{k}_decode_planned_kernelILj{sb}ELb0E")
                  for k in ("alias", "byte") for sb in (16, 14, 12, 0)]
               + [("rans64_decode_planned_stored_kernel", "rans64_decode_planned_kernel")])
TWINS = (
    [("chunks_store_kernel", None),
     ("chunks_stored_compaction_kernel", "compact_kernelILb0ELb0E"),
     ("container_stored_plan_kernel", "container_plan_kernelILb0E"),
     ("container_stored_check_kernel", "container_prefix_check_kernelILb0E"),
     ("container_stored_finish_kernel", "container_finish_kernelILb0ELb1E")]
    + V1_DECODERS
)

kernels = tvs.kernels


@pytest.mark.parametrize("new,twin", TWINS)
def test_stored_kernels_spill_no_more_than_their_twins(kernels, new, twin):
    got = tvs._local(tvs._one(kernels, new))
    want = (0, 0) if twin is None else tvs._local(tvs._one(kernels, twin))
    assert got[0] <= want[0] and got[1] <= want[1], (new, got, twin, want)
