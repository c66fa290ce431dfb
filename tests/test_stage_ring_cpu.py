"""The warp-specialized kernels reach their stage ring's mbarriers only through StageRing (csrc/ring.cuh), so the one
protocol tools/kernel_models.py models (RingModel) is the one every kernel runs."""
import re

import pytest

from tools import kernel_models as km


@pytest.mark.parametrize("src,kernel", [("gemm_ws.cu", "gemm_ws_kernel"), ("attention_wgmma.cu", "attn_rows_kernel"),
                                        ("attention_wgmma.cu", "tattn_fused_kernel")])
def test_ring_barriers_only_through_stage_ring(src, kernel):
    body = km.kernel_body(src, kernel)
    assert re.search(r"__shared__ StageRing<\w+> ring;", body), f"{kernel} declares no StageRing"
    # the only other mbarrier is attn_rows_kernel's Q barrier, loaded once and outside the ring
    assert re.findall(r"__shared__[^;]*uint64_t[^;]*;", body) in ([], ["__shared__ __align__(8) uint64_t qbar;"])
    for call, args in re.findall(r"\b(mbar_\w+|tma_load_4d)\(([^;]*)\);", body):
        # mbar_*: the barrier is the first argument; tma_load_4d(dst, map, barrier, ...): the one StageRing::produce returned
        ok = args.startswith("&qbar") if call.startswith("mbar_") else re.search(r", (bar|&qbar), ", args)
        assert ok, f"{kernel}: {call}({args}) bypasses StageRing"
    assert not re.search(r"\b(full|empty)\[", body), f"{kernel} indexes a ring barrier directly"
