"""Fit and check the FMA-pipe exp2 of csrc/ptx.cuh (ex2_poly, used by csrc/attention_wgmma.cu): Cody-Waite split x = n + f with the
1.5 * 2^23 rounding trick, degree-3 minimax polynomial for 2^f on [-0.5, 0.5], exponent-field add for 2^n.
Emulated in float32 / int32 numpy exactly as the device code computes it (fma -> mul+add: one extra rounding, which only
loosens this check).  Run: python tools/exp2_poly_fit.py"""
import numpy as np

C = np.array([0.9999280571937561, 0.6932609677314758, 0.2426111251115799, 0.05517164245247841], dtype=np.float32)


def fit(deg=3, iters=50):
    x = np.cos(np.pi * (np.arange(4001) + 0.5) / 4001) * 0.5
    y = 2.0 ** x
    w = np.ones_like(x)
    for _ in range(iters):  # iteratively re-weighted least squares on the relative error -> near-minimax
        A = np.vander(x, deg + 1, increasing=True) / y[:, None]
        c, *_ = np.linalg.lstsq(A * w[:, None], w, rcond=None)
        err = np.abs(A @ c - 1)
        w = w * (1 + 3 * err / err.max())
    return c.astype(np.float32)


def ex2_poly(x):
    x = np.maximum(x.astype(np.float32), np.float32(-125.0))
    magic = np.float32(12582912.0)
    t = (x + magic).astype(np.float32)
    f = (x - (t - magic).astype(np.float32)).astype(np.float32)
    p = (f * C[3] + C[2]).astype(np.float32)
    p = (p * f + C[1]).astype(np.float32)
    p = (p * f + C[0]).astype(np.float32)
    bits = p.view(np.int32) + (t.view(np.int32) << 23)  # int32 wrap-around == the device's 32-bit add / shift
    return bits.astype(np.int32).view(np.float32)


def check():
    x = np.concatenate([np.linspace(-130.0, 9.0, 2_000_001), np.array([-np.inf, -1000.0, -127.0, -126.5, 0.0, 8.0, 9.0])]).astype(np.float32)
    with np.errstate(over="ignore"):
        got = ex2_poly(x).astype(np.float64)
    assert np.isfinite(got).all() and (got > 0).all(), "exponent-field wrap-around"
    ref = np.exp2(np.maximum(x.astype(np.float64), -125.0))
    rel = np.abs(got / ref - 1.0)
    return float(rel.max()), float(got[x < -125].max())


if __name__ == "__main__":
    print("refit:", [float(c) for c in fit()], "(device constants:", [float(c) for c in C], ")")
    rel, tiny = check()
    print(f"max relative error on [-125, 9]: {rel:.3e} (fp16 half-ulp 4.9e-4); x < -125 (masked keys, -inf) -> {tiny:.3e} (packs to 0)")
