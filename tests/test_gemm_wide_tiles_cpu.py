"""CPU tests of gemm_ws_kernel's 160-column tiles (tools/kernel_models.py): which GEMMs take them, the shared memory they
need, and the staged epilogue's 160-wide layout (bank-conflict-free fragment stores, copy-out and residual fetch, each
chunk in the warp that wrote it, every chunk of a ragged tile stored once), each with a negative control."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.mark.parametrize("M,N,geglu,bn", [
    (65536, 320, False, 160), (196608, 960, False, 160),  # the 64 x 64 level: 3 / 8 tiles of 128 would pad the last
    (16384, 640, False, 160), (12288, 1280, False, 160), (4096, 1280, False, 160), (16384, 1920, False, 160),
    (3072, 1280, False, 128), (1024, 1280, False, 128),   # 24 / 8 row tiles: 10 columns of 128 fill more SMs than 8 of 160
    (128, 320, False, 128), (1000, 640, False, 128),      # one wave either way: the narrower tile ends first
    (65536, 1024, False, 128), (65536, 200, False, 128),  # not a multiple of 160
    (65536, 2560, True, 128), (65536, 320, True, 128),    # GEGLU: geglu_pack's 128-wide tile
])
def test_dispatch_rule(M, N, geglu, bn):
    """on 132 SMs (H100 SXM)"""
    from tools import kernel_models as km
    assert km.ws_tile_n(M, N, geglu, sms=132) == bn


def test_shared_memory_fits():
    """4 stages of 36 KB + 2 staging tiles of 40 KB + 1 KB = 225 KB at 160 columns: within an SM's 227 KB with the ring's
    64 static bytes; the 128-wide kernel keeps its 193 KB"""
    from tools import kernel_models as km
    assert km.ws_smem_bytes(128) == 193 * 1024
    assert km.ws_smem_bytes(160) == 225 * 1024
    assert km.ws_smem_bytes(160) + 64 <= 227 * 1024


def test_staging_tile_layout():
    from tools import kernel_models as km
    assert km.check_epilogue_staging("linear", bn=160)
    with pytest.raises(AssertionError, match="fragment store of chunk 0: bank conflict"):
        km.check_epilogue_staging("linear", bn=160, swizzle=False)
    with pytest.raises(AssertionError, match="fragment store of chunk 16: bank conflict"):  # the 32-column tail's own swizzle
        km.check_epilogue_staging("linear", bn=160, tail_swizzle=False)


@pytest.mark.parametrize("M", [1, 37, 127, 128, 1000, 196608])
@pytest.mark.parametrize("N", [160, 320, 960])
def test_ragged_copy_out(M, N):
    """every tile of an M x N output, the last row tile ragged: each chunk stored once; without the tail pass a 160-wide
    tile loses its last 32 columns"""
    from tools import kernel_models as km
    m_tiles = list(range(0, M, 128))
    for m0 in m_tiles[:2] + m_tiles[-2:]:
        for n0 in range(0, N, 160):
            assert km.check_ragged_copy_out(M, N, m0, n0, bn=160)
            with pytest.raises(AssertionError, match="misses or adds"):
                km.check_ragged_copy_out(M, N, m0, n0, bn=160, passes=km.copy_out_passes(128))
