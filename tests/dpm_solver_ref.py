"""TEST INFRASTRUCTURE — DPM-Solver++(2M) for the tests of `DPMSolverMultistepScheduler` and the fused step kernel; nothing
outside tests/ imports it.

1. Schedule, float64: the timesteps, sigmas and log-SNR lambda of diffusers 0.26's `DPMSolverMultistepScheduler` [recalled:
   diffusers is not vendored] on the I2VGen-XL config, written the way diffusers writes them (the "VE" sigma
   sqrt((1 - abar) / abar) converted back by `_sigma_to_alpha_sigma_t`), independently of anyv2v_b200/schedulers.py.
   ``coefficient_rows`` restates the update of Lu et al. 2022 (DPM-Solver++, Alg. 2, midpoint form) as the
   {alpha, sigma, a, b, c} rows the kernel takes.
2. ``DPMRef``: a stateful scheduler with the oracle's `step(model_output, t, sample) -> (prev, x0)` API (for
   oracle/loops_ref.pnp_edit_loop), diffusers' `multistep_dpm_solver_{first,second}_order_update`; in fp16 every PyTorch op
   rounds separately (oracle/schedulers_ref.py's rounding model), in fp32 it is the fp32 oracle.
3. Contract of `ops.dpmpp2m_step` (csrc/elementwise.cu dpm_step_kernel): ``dpmpp2m_step`` in fp32 tensor ops, bit for bit
   the kernel's arithmetic; ``dpmpp2m_exact`` the float64 values it rounds at its two stores, with their condition scales
   for tests/ulp_check.py.  ``patch_ops`` swaps it in next to the ``emulated_ops`` fixture.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import kernel_contracts
from oracle import schedulers_ref
from oracle.schedulers_ref import _add, _mul

N_TRAIN = 1000
STEPS_OFFSET = 1


# ------------------------------------------------------------------------------------------------------------- schedule
def alphas_cumprod64() -> np.ndarray:
    """the fp32 abar table of the I2VGen-XL config (oracle), as float64"""
    return schedulers_ref.alphas_cumprod().double().numpy()


def timesteps(n: int) -> list:
    """diffusers' "leading" spacing: step_ratio = 1000 // n, (arange(n) * ratio).round()[::-1] + steps_offset"""
    ratio = N_TRAIN // n
    return [int(t) for t in ((np.arange(0, n) * ratio).round()[::-1] + STEPS_OFFSET).astype(np.int64)]


def sigmas(n: int) -> np.ndarray:
    """the "VE" sigmas of the n timesteps, then the last one: sqrt((1 - abar_0) / abar_0) (diffusers 0.26)"""
    ac = alphas_cumprod64()
    with np.errstate(divide="ignore"):  # abar_999 = 0 (zero terminal SNR); "leading" timesteps stop before it
        ve = np.sqrt((1 - ac) / ac)
    return np.concatenate([ve[timesteps(n)], ve[[0]]])


def alpha_sigma_t(sigma_ve):
    """diffusers' `_sigma_to_alpha_sigma_t`"""
    alpha_t = 1.0 / np.sqrt(sigma_ve ** 2 + 1)
    return alpha_t, sigma_ve * alpha_t


def lambdas(n: int) -> np.ndarray:
    alpha_t, sigma_t = alpha_sigma_t(sigmas(n))
    return np.log(alpha_t) - np.log(sigma_t)


def first_order_rows(n: int, solver_order: int = 2, lower_order_final: bool = True) -> list:
    """which steps of an n-step loop over the whole schedule are first order: the first; every one with solver_order 1;
    the last when lower_order_final and n < 15"""
    return [i == 0 or solver_order == 1 or (i == n - 1 and lower_order_final and n < 15) for i in range(n)]


def coefficient_rows(n: int, t_idx: int = 0, solver_order: int = 2) -> np.ndarray:
    """[n - t_idx, 5] float64 {alpha_t, sigma_t, a, b, c} of a loop over timesteps(n)[t_idx:] (its first step first order)"""
    sig = sigmas(n)
    alpha, sigma = alpha_sigma_t(sig)
    lam = np.log(alpha) - np.log(sigma)
    first = first_order_rows(n, solver_order)
    rows = []
    for k in range(t_idx, n):
        h = lam[k + 1] - lam[k]
        a = sigma[k + 1] / sigma[k]
        b = -alpha[k + 1] * (math.exp(-h) - 1.0)
        c = 0.0
        if not (first[k] or k == t_idx):
            r0 = (lam[k] - lam[k - 1]) / h
            c = 0.5 / r0
        rows.append([alpha[k], sigma[k], a, b, c])
    return np.array(rows)


# ------------------------------------------------------------------------------------------------------------- oracle step
class DPMRef:
    """diffusers' DPMSolverMultistepScheduler.step for dpmsolver++ / midpoint / v-prediction [recalled], with the history
    of data predictions kept by the scheduler.  Computes in the dtype of its inputs (fp16: one rounding per op)."""

    def __init__(self, solver_order: int = 2):
        self.solver_order = solver_order
        self.timesteps = None

    def set_timesteps(self, n: int, device=None):
        self.n = n
        self.timesteps = torch.tensor(timesteps(n), device=device)
        sig = sigmas(n)
        self.alpha, self.sigma = alpha_sigma_t(sig)
        self.lam = np.log(self.alpha) - np.log(self.sigma)
        self.first = first_order_rows(n, self.solver_order)
        self.x0_prev = None
        self.lower_order_nums = 0

    def step(self, model_output, timestep, sample):
        k = timesteps(self.n).index(int(timestep))
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)
        x0 = _add(_mul(f32(self.alpha[k]), sample), _mul(f32(self.sigma[k]), model_output), -1.0)
        h = self.lam[k + 1] - self.lam[k]
        a = self.sigma[k + 1] / self.sigma[k]
        bm = self.alpha[k + 1] * (math.exp(-h) - 1.0)           # x_s = a x - bm D0 (- 0.5 bm D1)
        out = _add(_mul(f32(a), sample), _mul(f32(bm), x0), -1.0)
        if not (self.first[k] or self.lower_order_nums < 1):
            r0 = (self.lam[k] - self.lam[k - 1]) / h
            d1 = _mul(f32(1.0 / r0), _add(x0, self.x0_prev, -1.0))
            out = _add(out, _mul(f32(0.5 * bm), d1), -1.0)
        self.x0_prev = x0
        self.lower_order_nums = min(self.lower_order_nums + 1, self.solver_order)
        return out, x0


# ------------------------------------------------------------------------------------------------------------- contract
def _operands(x, v_neg, v_edit, x0_prev, guidance, alpha, sigma, a, b, c, coef_dev):
    for name, t in (("x", x), ("v_neg", v_neg), ("x0_prev", x0_prev)):
        kernel_contracts._f16(t, f"dpmpp2m.{name}")
        assert t.numel() == x.numel(), name
    if coef_dev is not None:
        alpha, sigma, a, b, c, guidance = (float(v) for v in coef_dev[:6].tolist())
    r16 = lambda t: t.to(torch.float16).to(torch.float32)
    f32 = lambda s: torch.tensor(s, dtype=torch.float32, device=x.device)
    xf, vn = x.float().reshape(-1), v_neg.float().reshape(-1)
    v = vn
    if v_edit is not None:  # the CFG combine of ddim_one
        d0 = r16(v_edit.float().reshape(-1) - vn)
        v = r16(vn + r16(f32(guidance) * d0))
    return xf, v, x0_prev.float().reshape(-1), [float(torch.tensor(s, dtype=torch.float32)) for s in (alpha, sigma, a, b, c)], f32


def dpmpp2m_step(x, v_neg, v_edit, x0_prev, guidance, alpha, sigma, a, b, c, out=None, coef_dev=None):
    """dpm_step_kernel in fp32 tensor ops, one IEEE rounding per op in the kernel's order: writes x0 to ``x0_prev``"""
    xf, v, p, (al, si, a, b, c), f32 = _operands(x, v_neg, v_edit, x0_prev, guidance, alpha, sigma, a, b, c, coef_dev)
    r16 = lambda t: t.to(torch.float16).to(torch.float32)
    x0 = r16((f32(al) * xf) - (f32(si) * v))
    d = x0 + f32(c) * (x0 - p) if c != 0.0 else x0
    y = (f32(a) * xf) + (f32(b) * d)
    kernel_contracts._count()
    x0_prev.copy_(x0.to(torch.float16).view(x0_prev.shape))
    return kernel_contracts._store(out, y, x.shape)


def dpmpp2m_exact(x, v_neg, v_edit, x0_prev, guidance, alpha, sigma, a, b, c, x0_got, coef_dev=None):
    """float64 values of the two stores and their condition scales: (x0, cond_x0, out, cond_out).  x0 is exact on the fp16
    (CFG-combined) operands; out is exact on the x0 the kernel stored (``x0_got``, its pinned rounding point) and x0_prev"""
    xf, v, p, (al, si, a, b, c), _ = _operands(x, v_neg, v_edit, x0_prev, guidance, alpha, sigma, a, b, c, coef_dev)
    xd, vd, pd = xf.double(), v.double(), p.double()
    x0 = al * xd - si * vd
    cond_x0 = abs(al) * xd.abs() + abs(si) * vd.abs()
    q = x0_got.double().reshape(-1)
    d = q + c * (q - pd) if c != 0.0 else q
    out = a * xd + b * d
    cond_out = abs(a) * xd.abs() + abs(b) * (q.abs() + abs(c) * (q.abs() + pd.abs()))
    return x0, cond_x0, out, cond_out


def patch_ops(monkeypatch):
    """ops.dpmpp2m_step -> the contract for one test (use together with the emulated_ops fixture)"""
    from anyv2v_b200 import ops
    monkeypatch.setattr(ops, "dpmpp2m_step", dpmpp2m_step)
