"""CPU test of the model of the GEMM kernels' shared staged epilogue (tools/kernel_models.py: check_epilogue_staging)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.mark.parametrize("kernel,geglu", [("conv", False), ("linear", False), ("linear", True)])
def test_staging_tile_layout(kernel, geglu):
    """for the band ownership of each kernel (conv: 8 warps x 1 band, linear: 4 warps x 2 bands per staging tile), every
    (row, column pair) of the tile is written by one thread and read by one 16-byte copy-out lane of the same warp, both
    patterns free of bank conflicts per shared-memory wavefront; without the XOR swizzle the fragment stores conflict"""
    from tools import kernel_models as km
    assert km.check_epilogue_staging(kernel, geglu)
    with pytest.raises(AssertionError, match="fragment store .* bank conflict"):
        km.check_epilogue_staging(kernel, geglu, swizzle=False)


def test_residual_tile_takes_a_free_ring_slot():
    """the slot of the staging tile / residual tile 0, num_kb % stages, is the one the prefetch of a block num_kb would take:
    the ring model's rule (no slot refilled before both warpgroups retired the wgmma that read it) covers it"""
    import random
    from tools import kernel_models as km
    stages, wait_depth, dist = km.gemm_pipeline_constants()
    assert dist == 1  # the kernel issues the fetch after the loop, where a block num_kb would have been prefetched at dist 1
    rng = random.Random(5)
    for nk in (1, 2, 3, 5, 10, 45):
        for _ in range(20):
            km.simulate_gemm_ring(random.Random(rng.getrandbits(32)), nk, stages, wait_depth, dist, epilogue_tile=True)
    caught = 0
    for _ in range(20):
        try:  # a tile in the slot of the last block would be filled while its wgmma read it
            km.simulate_gemm_ring(random.Random(rng.getrandbits(32)), 10, stages, wait_depth, dist, epilogue_tile=True, tile_shift=stages - 1)
        except AssertionError:
            caught += 1
    assert caught >= 15
