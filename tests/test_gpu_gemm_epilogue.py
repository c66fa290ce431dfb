"""GPU tests of the staged epilogue both GEMM kernels share (csrc/gemm_common.cuh): the output tile leaves shared memory
in 16-byte chunks, so the cases here are the ones where a chunk could be written that should not be — a row stride wider
than N (the gap must keep its poison), N of one chunk and N with a single chunk past a 64-column boundary (LINEAR, GEGLU),
and a 3-slot residual that aliases the output (conv).
Float64 contracts of tests/kernel_contracts.py within ulp16(ref) + kappa * cond, on guarded buffers (tests/guarded.py)."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_inout, guarded_input, guarded_output
from ulp_check import KAPPA_GEGLU, KAPPA_GEMM, assert_within_bound, cond_conv_abs, cond_geglu, cond_linear

pytestmark = pytest.mark.gpu
dev = "cuda"


def gin(t, **kw):
    return guarded_input(t, device=dev, **kw)


def _w(N, K, g):
    return (torch.randn(N, K, generator=g) * K ** -0.5).half()


@pytest.mark.parametrize("N,ldo", [(8, 8), (72, 72), (8, 24), (72, 136), (320, 328), (256, 512)])
def test_linear_row_stride_and_narrow_tiles(N, ldo):
    """out and residual rows ldo apart: the columns [N, ldo) of every row, and everything around the buffer, stay untouched"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(N * 1000 + ldo)
    M, K = 5 * 128 + 53, 320
    a, w = torch.randn(M, K, generator=g).half(), _w(N, K, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    rowbias = (torch.randn(M // 97 + 1, N, generator=g) * 0.5).half()
    res = torch.randn(M, N, generator=g).half()
    out = guarded_output((M, N), ld=ldo, device=dev)
    ops.linear(gin(a).view, gin(w).view, bias=gin(bias).view, rowbias=gin(rowbias).view, rows_per_rowbias=97,
               residual=gin(res, ld=ldo).view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, f"linear N={N} ldo={ldo}")
    ref = kc.linear_exact(a, w, bias=bias, rowbias=rowbias, rows_per_rowbias=97, residual=res)
    assert_within_bound(out.view.cpu(), ref, cond_linear(a, w, bias, rowbias, 97, res), KAPPA_GEMM, f"linear N={N} ldo={ldo}", shape=(M, N))


def test_geglu_row_stride():
    """GEGLU's 128 x 64 output tile with a row stride: N = 192 leaves the last column tile half empty"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(192)
    M, N, K, ldo = 3 * 128 + 19, 192, 320, 104
    a = torch.randn(M, K, generator=g).half()
    wp, bp = kc.geglu_pack(_w(N, K, g), (torch.randn(N, generator=g) * 0.5).half())
    out = guarded_output((M, N // 2), ld=ldo, device=dev)
    ops.linear(gin(a).view, gin(wp).view, bias=gin(bp).view, out=out.view, geglu=True)
    torch.cuda.synchronize()
    check_output(out, "geglu ldo")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, wp, bp, geglu=True), cond_geglu(a, wp, bp), KAPPA_GEGLU, "geglu ldo",
                        shape=(M, N // 2))


@pytest.mark.parametrize("Cout", [320, 72])
def test_conv3x3_three_slots_residual_aliases_out(Cout):
    """the conv injection with its shortcuts already in the output buffer (residual = out): every slot's tile is read whole
    before it is stored, so the in-place result is bit-identical to the out-of-place one"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(Cout)
    NF, H, W, C = 5, 27, 29, 128  # M = 3915: a ragged last row tile
    x, w = torch.randn(NF, H, W, C, generator=g).half(), _w(Cout, 9 * C, g)
    bias = (torch.randn(Cout, generator=g) * 0.1).half()
    M = NF * H * W
    res = torch.randn(3, M, Cout, generator=g).half()
    kw = dict(bias=gin(bias).view, n_slots=3, slot_stride=M * Cout)
    xg, wg = gin(x).view, gin(w).view
    apart = guarded_output((3, M, Cout), device=dev)
    ops.conv3x3(xg, wg, residual=gin(res).view, out=apart.view, **kw)
    inplace = guarded_inout(res.to(dev))
    ops.conv3x3(xg, wg, residual=inplace.view, out=inplace.view, **kw)
    torch.cuda.synchronize()
    check_output(apart, "conv3x3 3 slots")
    check_output(inplace, "conv3x3 3 slots in place")
    assert torch.equal(inplace.view, apart.view)
    acc = kc.conv3x3_exact(x, w, bias)
    cond = cond_conv_abs(kc.conv3x3_exact, x, w, bias) + res.double().abs()
    assert_within_bound(inplace.view.cpu(), acc + res.double(), cond, KAPPA_GEMM, f"conv3x3 3 slots in place Cout={Cout}",
                        shape=(3, M, Cout))
