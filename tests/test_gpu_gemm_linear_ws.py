"""GPU tests of the LINEAR-mode GEMM (csrc/gemm_ws.cu, persistent and warp-specialized) against the float64 contract
of tests/kernel_contracts.py, within ulp16(ref) + kappa * cond (tests/ulp_check.py), on guarded buffers (tests/guarded.py).

The kernel runs min(tiles, SMs) CTAs that walk a static tile schedule, two consumer warpgroups taking turns per tile, and
a stage ring that runs across tile boundaries: tile counts below, at and above the SM count (odd counts give one
warpgroup one tile more than the other), ragged M and N, K loops shorter and longer than the ring, row strides wider than
the data, two sources, rowbias, a residual that aliases out, and GEGLU."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from ulp_check import KAPPA_GEGLU, KAPPA_GEMM, assert_within_bound, cond_geglu, cond_linear

pytestmark = pytest.mark.gpu
dev = "cuda"


def gin(t, **kw):
    return guarded_input(t, device=dev, **kw)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _w(N, K, g):
    return (torch.randn(N, K, generator=g) * K ** -0.5).half()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run_linear(M, N, K, seed, lda=None, ldo=None, rowbias=True, residual=True):
    from anyv2v_b200 import ops
    g = _gen(seed)
    a = torch.randn(M, K, generator=g).half()
    w = _w(N, K, g)
    kw = dict(bias=(torch.randn(N, generator=g) * 0.1).half())
    if rowbias:
        kw.update(rowbias=(torch.randn(M // 97 + 1, N, generator=g) * 0.5).half(), rows_per_rowbias=97)
    if residual:
        kw.update(residual=torch.randn(M, N, generator=g).half())
    out = guarded_output((M, N), ld=ldo, device=dev)
    dkw = {k: gin(v).view if isinstance(v, torch.Tensor) else v for k, v in kw.items()}
    if residual and ldo is not None:
        dkw["residual"] = gin(kw["residual"], ld=ldo).view
    ops.linear(gin(a, ld=lda).view, gin(w).view, **dkw, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear")
    ref = kc.linear_exact(a, w, **kw)
    cond = cond_linear(a, w, kw["bias"], kw.get("rowbias"), kw.get("rows_per_rowbias", 0), kw.get("residual"))
    assert_within_bound(out.view.cpu(), ref, cond, KAPPA_GEMM, f"linear {M}x{N}x{K}", shape=(M, N))


@pytest.mark.parametrize("tiles", ["1", "sms-1", "sms", "sms+1", "2sms+3", "3sms+1"])
def test_tile_counts(tiles):
    """one column tile, so the row tiles are the tiles; the last one ragged"""
    sms = _sms()
    n = {"1": 1, "sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+3": 2 * sms + 3, "3sms+1": 3 * sms + 1}[tiles]
    _run_linear(n * 128 - 37, 128, 320, seed=n)


@pytest.mark.parametrize("N", [8, 72, 200])
@pytest.mark.parametrize("K", [8, 72, 320, 1024, 5120])  # K tail inside one block; 5 blocks; longer than the ring
def test_shapes(N, K):
    _run_linear(1000, N, K, seed=N * 31 + K)


def test_strided_rows():
    """lda > K and ldo > N (the residual shares out's row stride)"""
    _run_linear(2000 + 5, 200, 320, seed=7, lda=320 + 24, ldo=200 + 16)


def test_two_source():
    """A = [a | a2] along K, each with its own row stride; k_split = 128, a2 with a K tail"""
    from anyv2v_b200 import ops
    g = _gen(11)
    M, K1, K2, N = 3000 + 3, 128, 72, 200
    a, a2 = torch.randn(M, K1, generator=g).half(), torch.randn(M, K2, generator=g).half()
    w = _w(N, K1 + K2, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    out = guarded_output((M, N), device=dev)
    ops.linear(gin(a, ld=K1 + 40).view, gin(w).view, bias=gin(bias).view, a2=gin(a2, ld=K2 + 24).view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear two-source")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, w, bias, a2=a2), cond_linear(a, w, bias, a2=a2), KAPPA_GEMM,
                        "linear two-source", shape=(M, N))


def test_residual_aliases_out():
    """out += a @ w^T + bias in place: every residual read of a row lands before that row is stored"""
    from anyv2v_b200 import ops
    g = _gen(13)
    M, N, K = 3 * _sms() * 128 + 50, 320, 320
    a = torch.randn(M, K, generator=g).half()
    w = _w(N, K, g)
    bias = (torch.randn(N, generator=g) * 0.1).half()
    res = torch.randn(M, N, generator=g).half()
    out = guarded_output((M, N), device=dev)
    out.view.copy_(res)
    ops.linear(gin(a).view, gin(w).view, bias=gin(bias).view, residual=out.view, out=out.view)
    torch.cuda.synchronize()
    check_output(out, "linear residual in place")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, w, bias, residual=res), cond_linear(a, w, bias, residual=res),
                        KAPPA_GEMM, "linear residual in place", shape=(M, N))


@pytest.mark.parametrize("N", [64, 2560, 10240])
def test_geglu(N):
    from anyv2v_b200 import ops
    g = _gen(N)
    M, K = 700 + 9, 320
    a = torch.randn(M, K, generator=g).half()
    wp, bp = kc.geglu_pack(_w(N, K, g), (torch.randn(N, generator=g) * 0.5).half())
    out = guarded_output((M, N // 2), device=dev)
    ops.linear(gin(a).view, gin(wp).view, bias=gin(bp).view, out=out.view, geglu=True)
    torch.cuda.synchronize()
    check_output(out, "geglu")
    assert_within_bound(out.view.cpu(), kc.linear_exact(a, wp, bp, geglu=True), cond_geglu(a, wp, bp), KAPPA_GEGLU,
                        f"geglu {M}x{N}x{K}", shape=(M, N // 2))
