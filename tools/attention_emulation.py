"""Numerical emulation (torch, CPU) of the per-row algorithm of csrc/attention_wgmma.cu (attn_tile): 64-key tiles, running
max raised on every tile with O / l rescaled, P rounded to fp16 before the PV product, fp32 accumulation, 0 / 25 / 50 % of
the exponentials through the FMA-pipe polynomial (the kernel: 25 %, columns 24-31 of every 32), key-tail masking.  Checks the
ALGORITHM (not the hardware protocol) against exact softmax attention at the tolerance of the GPU parity tests."""
import numpy as np
import torch

from tools import exp2_poly_fit

TK = 64


def _ex2(a: torch.Tensor, poly_mask: torch.Tensor) -> torch.Tensor:
    exact = torch.exp2(a)
    if not poly_mask.any():
        return exact
    p = torch.from_numpy(exp2_poly_fit.ex2_poly(a.numpy().astype(np.float32)).astype(np.float32))
    return torch.where(poly_mask, p, exact)


def attention_rows(q, k, v, scale=0.125, poly=0, tk=TK, fused=False):
    """q [T,64], k/v [L,64] fp16 -> [T,64] fp16, one head.  tk: keys per tile (attn_tile: 64; attn_rows_kernel: 128 at
    n_v = 1, 64 at n_v = 3).  fused (attn_rows_kernel): the running max is taken over raw scores and scaled once per row,
    and the exponent is s * scale_log2 - max in one fused multiply-add (one rounding, emulated in float64)"""
    T, L = q.shape[0], k.shape[0]
    sc = np.float32(scale * 1.4426950408889634)
    qf, kf, vf = q.float(), k.float(), v.float()
    m = torch.full((T,), float("-inf"))
    l = torch.zeros(T)
    o = torch.zeros(T, 64)
    # column block j = col // 8 of a tile (accumulator registers 4j .. 4j + 3 of attn_tile) goes to the polynomial when
    # (j & 3) == 3 (25 %, the kernel) / (j & 1) == 1 (50 %)
    j8 = torch.arange(tk) // 8
    pm = ((j8 & 3) == 3) if poly == 1 else ((j8 & 1) == 1) if poly == 2 else torch.zeros(tk, dtype=torch.bool)
    for j in range((L + tk - 1) // tk):
        kt, vt = kf[j * tk:(j + 1) * tk], vf[j * tk:(j + 1) * tk]
        n = kt.shape[0]
        s = torch.full((T, tk), float("-inf"))
        s[:, :n] = qf @ kt.T                     # fp32 accumulate of fp16 products (tensor core)
        rmax = s.max(dim=1).values * sc
        m_new = torch.maximum(m, rmax)
        f = torch.exp2(m - m_new)  # 0 on the first tile (m = -inf)
        o, l = o * f[:, None], l * f
        m = m_new
        if fused:
            a = (s.double() * float(sc) - m.double()[:, None]).float()
        else:
            a = s * sc - m[:, None]
        p = _ex2(a.float(), pm[None, :].expand(T, tk))
        l = l + p.sum(dim=1)
        p16 = p.half().float()
        o = o + p16[:, :n] @ vt
    return (o / l[:, None]).half()


def check(T=192, L=880, mag=2.0, poly=2, seed=0, rising=False, tk=TK, fused=False):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(T, 64, generator=g) * mag).half()
    k = torch.randn(L, 64, generator=g) * mag
    if rising:
        k = k * torch.linspace(0.2, 6.0, L)[:, None]
    k = k.half()
    v = torch.randn(L, 64, generator=g).half()
    got = attention_rows(q, k, v, poly=poly, tk=tk, fused=fused).float()
    ref = torch.softmax(q.double() @ k.double().T * 0.125, dim=-1) @ v.double()
    err = (got.double() - ref).abs()
    tol = 2e-3 * ref.abs().max() + 1e-3 * ref.abs()
    return float((err / tol).max())


if __name__ == "__main__":
    for poly in (0, 1, 2):
        for kw in (dict(), dict(L=145, T=256), dict(mag=6.0), dict(rising=True, L=1024)):
            print(poly, kw, f"worst error / tolerance = {check(poly=poly, **kw):.3f}")
