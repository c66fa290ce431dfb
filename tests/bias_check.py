"""Mean error of an fp16 kernel output against its float64 contract, in fp16 ulps: the check for a systematic shift that
the element-wise bound of tests/ulp_check.py lets through.

That bound grants every element a full ulp16(ref), twice what round-to-nearest needs, so a store that rounds toward zero,
away from zero, up or down (a one-line change in the fp16 conversion every kernel stores through) passes it everywhere.
Over one 50-step inversion and the 50-step edit that starts from it, such a shift adds up step after step, where unbiased
rounding errors largely cancel.  A mean over many elements sees it:

    e = (got - ref) / ulp16(ref)        ref = the contract's float64 value before the store rounds it (as in ulp_check)

    mean(e)              round up / down, a constant offset
    mean(sign(ref) e)    round toward / away from zero, a scaling of the magnitude

Each with its standard error sigma_hat / sqrt(n).  A comparison passes when both satisfy |mean| <= BETA + Z * se, and it
must have power: Z * se <= POWER with at least MIN_COUNT counted elements, else it fails as underpowered instead of passing
on too little evidence.  The same two statistics per output column (the last dimension, a channel) over the rows, against
BETA_COL, locate a defect confined to a few channels, which the pooled mean dilutes by the column count.

Which elements count.  Those with a finite reference below the fp16 overflow edge, and where the store dominates the
arithmetic: kappa * cond <= STORE_DOMINATES * ulp16(ref).  The selection depends on ref and cond only, never on got, so it
cannot pick elements by their error.  The fraction excluded is reported.

Why these numbers:
  BETA = 1/16 ulp16.  Round-to-nearest of values spread over many fp16 spacings has mean 0 (the slope of the value density
      across one spacing leaves O(2^-11)); a directed rounding moves one of the two statistics by 1/2, so BETA is an eighth
      of the smallest store defect the check is for.  What correct arithmetic can leave in the mean: fp32 operations round to
      nearest (no bias); an approximation with a one-sided relative error r moves a result by at most r |ref| / ulp16(ref) <
      r 2^11 ulp16.  The largest such r any kernel applies to its result is the GEGLU erfc fit, 1.4e-5 (csrc/gemm_common.cuh,
      tools/erfc_poly_fit.py): 0.029 ulp16, half of BETA.  ex2.approx and rcp.approx (GroupNorm's SiLU, the erfc's t) stay
      below 2^-22: 2^-11 ulp16.  Attention needs no β of its own: P is rounded to fp16 by round-to-nearest (no bias), and the
      relative error of ex2_poly (7.5e-5, csrc/ptx.cuh) is a factor on each weight that the normalisation divides out where V
      is common to the keys, and that multiplies V_k - o, of either sign, elsewhere.
  BETA_COL = 1/8.  The rows of one column share its weights (or gamma, beta and the channel's statistics), so their
      arithmetic errors are not independent draws and average out less than the pooled ones; 1/8 still catches a 1/2-ulp
      shift of a single channel with a margin of 3/8.
  STORE_DOMINATES = 64.  The bound kappa * cond is a worst case: the fp32 accumulation error it covers is a random walk far
      below it (at cond = 64 ulp16 / kappa the typical error is a fraction of an ulp16 for the GEMM's K <= 11520).  Where
      cond is larger, the output cancels: its error in ulp16 of the small result grows into the thousands and would set
      sigma_hat, so that a few such elements make a case underpowered without adding anything a bias could be seen in.
  Z = 6, POWER = 1/8, MIN_COUNT = 2^16.  Z = 6 keeps the chance of a false failure below 1e-8 per statistic, so the several
      hundred columns of a case can be tested at once.  POWER = 1/8 means a case could not pass with a directed store: 1/2 >
      BETA + POWER.  2^16 elements keep sigma_hat itself an accurate estimate (relative error ~1 / sqrt(2 n) = 0.3 %).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from ulp_check import FP16_MAX_FINITE_EDGE, ulp16

BETA = 1.0 / 16
BETA_COL = 1.0 / 8
STORE_DOMINATES = 64.0
Z = 6.0
POWER = 1.0 / 8
MIN_COUNT = 1 << 16


@dataclass
class Moments:
    """running sums of e over the counted elements of one or more comparisons"""
    n: int = 0          # counted elements
    n_all: int = 0      # compared elements, excluded ones included
    s1: float = 0.0     # sum e
    s1s: float = 0.0    # sum sign(ref) e
    s2: float = 0.0     # sum e^2
    s2s: float = 0.0    # sum (sign(ref) e)^2

    def __iadd__(self, o: "Moments") -> "Moments":
        self.n, self.n_all = self.n + o.n, self.n_all + o.n_all
        self.s1, self.s1s, self.s2, self.s2s = self.s1 + o.s1, self.s1s + o.s1s, self.s2 + o.s2, self.s2s + o.s2s
        return self

    @property
    def excluded(self) -> float:
        return 1.0 - self.n / self.n_all if self.n_all else 1.0

    def stats(self):
        """(mean e, its standard error, mean sign(ref) e, its standard error); nan without elements"""
        if self.n < 2:
            return (math.nan,) * 4
        out = []
        for s1, s2 in ((self.s1, self.s2), (self.s1s, self.s2s)):
            m = s1 / self.n
            var = max(s2 / self.n - m * m, 0.0) * self.n / (self.n - 1)
            out += [m, math.sqrt(var / self.n)]
        return tuple(out)

    def verdict(self, beta: float = BETA):
        """'' if unbiased with power, else the reason it fails"""
        m, se, ms, ses = self.stats()
        if self.n < MIN_COUNT or not (Z * max(se, ses) <= POWER):
            return (f"underpowered: {self.n} counted elements (at least {MIN_COUNT}), {Z:g} se = {Z * max(se, ses):.3g} ulp16 "
                    f"(at most {POWER:g})")
        bad = [f"|{name}| over {beta:g} + {Z:g} se" for name, v, s in (("mean e", m, se), ("mean sign(ref) e", ms, ses))
               if not abs(v) <= beta + Z * s]
        return "; ".join(bad)

    def line(self) -> str:
        m, se, ms, ses = self.stats()
        return (f"mean e {m:+.4f} +- {se:.4f}, mean sign(ref) e {ms:+.4f} +- {ses:.4f} ulp16, n = {self.n}, "
                f"{self.excluded:.2%} excluded")


def _errors(got16, ref64, cond64, kappa):
    """flat float64 e, sign(ref), and the mask of counted elements, on ref64's device"""
    ref = torch.as_tensor(ref64).detach().to(torch.float64)
    got = torch.as_tensor(got16).detach().to(ref.device, torch.float64).reshape(-1)
    cond = torch.broadcast_to(torch.as_tensor(cond64, dtype=torch.float64).to(ref.device), ref.shape).reshape(-1)
    ref = ref.reshape(-1)
    assert got.shape == ref.shape == cond.shape, (got.shape, ref.shape, cond.shape)
    u = ulp16(ref)
    counted = torch.isfinite(ref) & (ref.abs() < FP16_MAX_FINITE_EDGE) & torch.isfinite(cond) & (kappa * cond <= STORE_DOMINATES * u)
    # a non-finite output there fails the element-wise bound; here it is left out, so that the sums stay finite
    counted &= torch.isfinite(got)
    e = torch.where(counted, (got - ref) / u, 0.0)
    return e, torch.where(counted, torch.sign(ref), 0.0), counted


def _moments(e, s, counted) -> Moments:
    es = s * e
    return Moments(int(counted.sum()), e.numel(), float(e.sum()), float(es.sum()), float((e * e).sum()), float((es * es).sum()))


def moments(got16, ref64, cond64, kappa: float) -> Moments:
    """the sums of one comparison (for pooling several, as tests/call_audit.py does per op)"""
    return _moments(*_errors(got16, ref64, cond64, kappa))


def _column_stats(e, s, counted, C):
    """per column of the last dimension: (counted [C], mean e [C], se [C], mean sign(ref) e [C], se [C])"""
    e, es, w = e.view(-1, C), (s * e).view(-1, C), counted.view(-1, C).to(torch.float64)
    n = w.sum(0)
    out = [n]
    for x in (e, es):
        m = x.sum(0) / n
        var = ((x * x).sum(0) / n - m * m).clamp_min(0) * n / (n - 1)
        out += [m, (var / n).sqrt()]
    return tuple(out)


def assert_unbiased(got16, ref64, cond64, kappa: float, what: str, beta: float = BETA, beta_col: float = BETA_COL,
                    quiet: bool = False) -> Moments:
    """fails, with the pooled statistics, their standard errors, n, the excluded fraction and the worst column, when the
    pooled mean or one column's mean is over its bias bound, or when the comparison has too little power"""
    got, ref = torch.as_tensor(got16), torch.as_tensor(ref64).to(got16.device)
    nonfinite = int((~torch.isfinite(got) & (ref.abs() < FP16_MAX_FINITE_EDGE)).sum())
    assert nonfinite == 0, f"{what}: {nonfinite} non-finite outputs where the contract is finite"
    e, sgn, counted = _errors(got16, ref64, cond64, kappa)
    mo = _moments(e, sgn, counted)
    n, m, se, ms, ses = _column_stats(e, sgn, counted, got16.shape[-1])
    # a column's excess over its bound, in ulp16, over both statistics; columns with fewer than 2 counted rows have no verdict
    excess = torch.maximum(m.abs() - beta_col - Z * se, ms.abs() - beta_col - Z * ses).nan_to_num(-math.inf)
    c = int(torch.argmax(excess))
    col = (f"worst column {c} of {got16.shape[-1]}: mean e {float(m[c]):+.4f} +- {float(se[c]):.4f}, mean sign(ref) e "
           f"{float(ms[c]):+.4f} +- {float(ses[c]):.4f} ulp16 over {int(n[c])} rows")
    line = f"{what}: {mo.line()}; {col}"
    if not quiet:
        print(line)
    verdict = mo.verdict(beta)
    assert not verdict, f"{line}: {verdict}"
    n_bad = int((excess > 0).sum())
    assert n_bad == 0, f"{line}: {n_bad} column(s) over {beta_col:g} + {Z:g} se"
    return mo


# ------------------------------------------------------------------------------------------------------------- controls
def round_fp16(x64: torch.Tensor, mode: str) -> torch.Tensor:
    """x rounded to fp16 with a directed rounding (the negative controls): "nearest", "zero" (toward zero), "away" (from
    zero), "up" or "down".  Values that fp16 represents exactly are returned as they are."""
    x = torch.as_tensor(x64).to(torch.float64)
    h = x.to(torch.float16)
    if mode == "nearest":
        return h
    hd = h.double()
    inexact = hd != x
    bits = h.view(torch.int16).to(torch.int32)
    sign, mag = bits & 0x8000, bits & 0x7FFF
    # with the magnitude bits, one step toward / away from zero is -1 / +1 (fp16 is sign-magnitude)
    if mode == "zero":
        step = torch.where(hd.abs() > x.abs(), -1, 0)
    elif mode == "away":
        step = torch.where(hd.abs() < x.abs(), 1, 0)
    elif mode == "up":
        step = torch.where(hd < x, torch.where(x > 0, 1, -1), 0)
    elif mode == "down":
        step = torch.where(hd > x, torch.where(x > 0, -1, 1), 0)
    else:
        raise ValueError(mode)
    step = torch.where(inexact, step, 0)
    # a tiny negative x that rounds to -0 must step up to -(smallest subnormal), not to +: keep the sign of x there
    sign = torch.where((mag == 0) & (x < 0), 0x8000, torch.where(mag == 0, 0, sign))
    mag = mag + step
    out = sign | mag
    return (out - ((out & 0x8000) << 1)).to(torch.int16).view(torch.float16)
