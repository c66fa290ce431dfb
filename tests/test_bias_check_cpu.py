"""Negative controls of tests/bias_check.py without a GPU.  A float64 reference over 16 binades, both signs and a per-element
condition scale, rounded to fp16 in each direction: every directed rounding passes the element-wise bound of
tests/ulp_check.py (the gap this check closes) and fails the bias check; round-to-nearest, with or without zero-mean noise
inside the bound, passes both; a half-ulp shift of one column in 320 fails on that column alone; too little evidence fails
as underpowered."""
import pytest
import torch

from bias_check import MIN_COUNT, Moments, assert_unbiased, moments, round_fp16
from ulp_check import KAPPA_GEMM, assert_within_bound, ulp16

ROWS, COLS = 1024, 320
CANCELLING = 0.05  # share of elements whose cond puts the arithmetic bound far above the store's ulp


def _reference(rows=ROWS, cols=COLS, seed=0):
    """ref [rows, cols]: random signs and mantissas over the binades 2^-12 ... 2^3; cond per element such that kappa * cond
    is 0 ... 4 ulp16(ref), and 1e3 ... 1e4 ulp16(ref) (an output that cancels) on a CANCELLING share of them"""
    g = torch.Generator().manual_seed(seed)
    ref = (torch.rand(rows, cols, generator=g, dtype=torch.float64) + 1) * 2.0 ** torch.randint(-12, 4, (rows, cols), generator=g)
    ref = ref * torch.where(torch.rand(rows, cols, generator=g) < 0.5, -1.0, 1.0).double()
    ulps = 4 * torch.rand(rows, cols, generator=g, dtype=torch.float64)
    cancels = torch.rand(rows, cols, generator=g) < CANCELLING
    ulps = torch.where(cancels, 1e3 + 9e3 * torch.rand(rows, cols, generator=g, dtype=torch.float64), ulps)
    return ref, ulps * ulp16(ref) / KAPPA_GEMM, g


def _biased(got, ref, cond, what):
    with pytest.raises(AssertionError) as e:
        assert_unbiased(got, ref, cond, KAPPA_GEMM, what)
    assert "over 0.0625" in str(e.value) and "underpowered" not in str(e.value), str(e.value)
    return str(e.value)


@pytest.mark.parametrize("mode,stat", [("zero", "mean sign(ref) e"), ("away", "mean sign(ref) e"), ("up", "mean e"),
                                       ("down", "mean e")])
def test_directed_rounding_passes_the_bound_and_fails_the_bias_check(mode, stat):
    ref, cond, _ = _reference()
    got = round_fp16(ref, mode)
    assert_within_bound(got, ref, cond, KAPPA_GEMM, f"round {mode}")
    assert_within_bound(got, ref, torch.zeros(()), 0.0, f"round {mode}, no arithmetic term")  # the store alone fits in 1 ulp
    msg = _biased(got, ref, cond, f"round {mode}")
    assert f"|{stat}| over" in msg


def test_round_to_nearest_passes():
    ref, cond, _ = _reference()
    mo = assert_unbiased(round_fp16(ref, "nearest"), ref, cond, KAPPA_GEMM, "round to nearest")
    assert abs(mo.excluded - CANCELLING) < 0.005  # the cancelling elements and only they are left out
    assert mo.n >= MIN_COUNT


def test_round_to_nearest_with_noise_inside_the_bound_passes():
    """zero-mean noise of up to half the arithmetic bound before the rounding: thousands of ulps on the cancelling elements,
    which the selection leaves out, so the case keeps its power"""
    ref, cond, g = _reference()
    noise = (2 * torch.rand(ref.shape, generator=g, dtype=torch.float64) - 1) * 0.5 * KAPPA_GEMM * cond
    got = round_fp16(ref + noise, "nearest")
    assert_within_bound(got, ref, cond, KAPPA_GEMM, "nearest + noise")
    assert float(((got.double() - ref) / ulp16(ref)).abs().max()) > 1000
    assert_unbiased(got, ref, cond, KAPPA_GEMM, "nearest + noise")


def test_half_ulp_on_one_column_fails_on_that_column():
    ref, cond, _ = _reference()
    col = 217
    shifted = ref.clone()
    shifted[:, col] += 0.5 * ulp16(ref[:, col])
    got = round_fp16(shifted, "nearest")
    assert_within_bound(got, ref, cond, KAPPA_GEMM, "one column shifted")
    pooled = moments(got, ref, cond, KAPPA_GEMM)
    assert not pooled.verdict(), pooled.line()  # the pooled mean alone does not see it
    with pytest.raises(AssertionError) as e:
        assert_unbiased(got, ref, cond, KAPPA_GEMM, "one column shifted")
    msg = str(e.value)
    assert f"worst column {col} of {COLS}" in msg and "1 column(s) over" in msg, msg


def test_too_few_elements_fail_as_underpowered():
    ref, cond, _ = _reference(rows=128)  # 40960 elements
    with pytest.raises(AssertionError, match="underpowered"):
        assert_unbiased(round_fp16(ref, "nearest"), ref, cond, KAPPA_GEMM, "too few")


def test_all_excluded_fails_as_underpowered():
    ref, cond, _ = _reference()
    with pytest.raises(AssertionError, match=r"underpowered: 0 counted"):
        assert_unbiased(round_fp16(ref, "nearest"), ref, cond + 65 * ulp16(ref) / KAPPA_GEMM, KAPPA_GEMM, "all cancelling")


def test_large_noise_fails_as_underpowered():
    """enough elements, but errors of tens of ulps inside the store-dominated selection: no power to see 1/16"""
    ref, cond, g = _reference()
    noisy = ref + (torch.rand(ref.shape, generator=g, dtype=torch.float64) - 0.5) * 100 * ulp16(ref)
    with pytest.raises(AssertionError, match="underpowered"):
        assert_unbiased(round_fp16(noisy, "nearest"), ref, cond, KAPPA_GEMM, "large noise")


def test_pooled_moments_match_one_comparison():
    """tests/call_audit.py pools the sums of many calls per op: the pooled statistics equal those of the whole"""
    ref, cond, _ = _reference()
    got = round_fp16(ref, "zero")
    whole = moments(got, ref, cond, KAPPA_GEMM)
    pooled = Moments()
    for part in range(4):
        rows = slice(part * ROWS // 4, (part + 1) * ROWS // 4)
        pooled += moments(got[rows], ref[rows], cond[rows], KAPPA_GEMM)
    assert pooled.n == whole.n and pooled.n_all == whole.n_all
    assert pooled.stats() == pytest.approx(whole.stats(), rel=1e-9)
    assert "mean sign(ref) e" in pooled.verdict()


def test_round_fp16_directions():
    x = torch.tensor([1.0 + 2.0 ** -12, -(1.0 + 2.0 ** -12), 3e-9, -3e-9, 0.5, -65000.3], dtype=torch.float64)
    up = torch.tensor([1.0 + 2.0 ** -10, -1.0, 2.0 ** -24, -0.0, 0.5, -64992.0])
    assert torch.equal(round_fp16(x, "up").double(), up.double())
    assert torch.equal(round_fp16(x, "down").double(), -round_fp16(-x, "up").double())
    assert torch.equal(round_fp16(x, "zero").abs().double(), torch.tensor([1.0, 1.0, 0, 0, 0.5, 64992.0]).double())
    assert torch.equal(round_fp16(x, "away").abs().double(), torch.tensor([1 + 2 ** -10, 1 + 2 ** -10, 2 ** -24, 2 ** -24, 0.5,
                                                                          65024.0]).double())
