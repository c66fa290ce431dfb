"""Fit and check the erfc of the GEGLU epilogue (gelu_erf_fast in csrc/gemm_common.cuh): erfc(z) = t * exp(-z^2 + P5(t)) with
t = 1 / (1 + z/2) — the form of the erfcc routine of Numerical Recipes, with a degree-5 polynomial fitted here instead of its
degree-9 one.  The error of this form is RELATIVE, which is what gelu(g) = g/2 * erfc(-g/sqrt 2) needs on the small negative
side.  Fitted on z in [0, 5.6] (gates down to -7.9; below that |gelu| < 3e-14); emulated in float32 numpy as the device code
computes it.  Run: python tools/erfc_poly_fit.py"""
import numpy as np
from scipy.special import erfc

C = np.array([-1.2661160230636597, 1.014296054840088, 0.26681792736053467, 0.4547545611858368, -0.6940243244171143,
              0.22427836060523987], dtype=np.float32)
Z_MAX = 5.6


def fit(deg=5, iters=30):
    z = np.linspace(0, Z_MAX, 200001)
    t = 1 / (1 + 0.5 * z)
    target = np.log(erfc(z) / t) + z * z  # P(t) = log(erfc / t) + z^2: its absolute error is erfc's relative error
    w = np.ones_like(t)
    for _ in range(iters):  # iteratively re-weighted least squares -> near-minimax
        c = np.polynomial.polynomial.polyfit(t, target, deg, w=w)
        err = np.abs(np.polynomial.polynomial.polyval(t, c) - target)
        w = w * (1 + 50 * err / err.max())
        w /= w.mean()
    return c.astype(np.float32)


def erfc_fast(z):
    z = z.astype(np.float32)
    t = (np.float32(1) / (np.float32(0.5) * z + np.float32(1))).astype(np.float32)
    p = C[-1]
    for c in C[-2::-1]:
        p = (p * t + c).astype(np.float32)
    arg = ((-z * z).astype(np.float64) + p).astype(np.float32) * np.float32(1.4426950408889634)
    return (t * np.exp2(arg.astype(np.float32))).astype(np.float32)


def check():
    z = np.linspace(0, Z_MAX, 2_000_001).astype(np.float32)
    rel = np.abs(erfc_fast(z).astype(np.float64) / erfc(z.astype(np.float64)) - 1)
    return float(rel.max())


if __name__ == "__main__":
    print("refit:", [float(c) for c in fit()], "(device constants:", [float(c) for c in C], ")")
    print(f"max relative error of erfc on [0, {Z_MAX}]: {check():.3e} (fp16 half-ulp 2.4e-4 .. 4.9e-4)")
