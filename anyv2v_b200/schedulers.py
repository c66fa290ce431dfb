"""DDIM / inverse-DDIM and DPM-Solver++(2M) schedulers for the I2VGen-XL scheduler config, host side + fused device step.

API of the diffusers classes the reference uses (``set_timesteps``, ``timesteps``, ``step(...).prev_sample``,
``scale_model_input``, ``init_noise_sigma``, ``order``; run_group_pnp_edit.py:69-72, pipeline_i2vgen_xl.py:1104,1173,
1359,1418).  Host side: the beta schedule, zero-terminal-SNR rescale and "leading" timestep spacing follow
consisti2v/ddim_inverse_scheduler.py:49-127, 253-289 (the reference's vendored copy of the diffusers class), config
pinned at i2vgen-xl/demo.ipynb:1209-1225.  Device side: ``step`` is ONE kernel launch (csrc/elementwise.cu) that also
folds in classifier-free guidance when given both model outputs, reproducing the reference's fp16 rounding sequence
bit for bit (each PyTorch op of scheduler.step / pipeline :1162 rounds to fp16 separately).  ``DPMSolverMultistepScheduler``
samples with about half the steps; its step is one launch of the fused DPM-Solver++(2M) kernel.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

from . import ops

DEFAULT_CONFIG = dict(num_train_timesteps=1000, beta_schedule="squaredcos_cap_v2", beta_start=1e-4, beta_end=0.02,
                      prediction_type="v_prediction", rescale_betas_zero_snr=True, clip_sample=False,
                      set_alpha_to_one=True, steps_offset=1, timestep_spacing="leading", thresholding=False)


def _alphas_cumprod(cfg) -> torch.Tensor:
    n = cfg["num_train_timesteps"]
    if cfg["beta_schedule"] != "squaredcos_cap_v2":
        raise ValueError("only the I2VGen-XL beta schedule (squaredcos_cap_v2) is supported")
    bar = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
    betas = torch.tensor([min(1 - bar((i + 1) / n) / bar(i / n), 0.999) for i in range(n)], dtype=torch.float32)
    if cfg["rescale_betas_zero_snr"]:
        s = torch.cumprod(1.0 - betas, dim=0).sqrt()
        s0, sT = s[0].clone(), s[-1].clone()
        s = (s - sT) * (s0 / (s0 - sT))
        abar = s ** 2
        betas = 1 - torch.cat([abar[0:1], abar[1:] / abar[:-1]])
    return torch.cumprod(1.0 - betas, dim=0)


def _leading(cfg, n: int) -> np.ndarray:
    """"leading" timestep spacing, ascending: 1, 1 + 1000 // n, ... (consisti2v/ddim_inverse_scheduler.py:253-289)"""
    if n > cfg.num_train_timesteps:
        raise ValueError(f"`num_inference_steps`: {n} cannot be larger than {cfg.num_train_timesteps}")
    if cfg.timestep_spacing != "leading":
        raise ValueError("only timestep_spacing='leading' is supported")
    ratio = cfg.num_train_timesteps // n
    return (np.arange(0, n) * ratio).round().astype(np.int64) + cfg.steps_offset


def _config_kwargs(config, accepted: dict, overrides: dict) -> dict:
    """the entries of a config dict / SimpleNamespace that a scheduler class takes (``accepted``), then ``overrides``"""
    cfg = dict(vars(config)) if isinstance(config, SimpleNamespace) else dict(config)
    cfg = {k: v for k, v in cfg.items() if k in accepted}
    cfg.update(overrides)
    return cfg


def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers.utils.torch_utils.randn_tensor [recalled]: a CPU generator draws on the CPU (in ``dtype``) and the result is
    moved to ``device``; a CUDA generator for a CPU tensor is an error; a list of generators draws one batch entry each (a
    list of one is a single generator)."""
    device = torch.device(device) if device is not None else torch.device("cpu")
    rand_device = device
    batch_size = shape[0]
    if generator is not None:
        gen_device_type = generator.device.type if not isinstance(generator, list) else generator[0].device.type
        if gen_device_type != device.type and gen_device_type == "cpu":
            rand_device = "cpu"
        elif gen_device_type != device.type and gen_device_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_device_type}.")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        shape = (1,) + tuple(shape[1:])
        latents = [torch.randn(shape, generator=generator[i], device=rand_device, dtype=dtype) for i in range(batch_size)]
        return torch.cat(latents, dim=0).to(device)
    return torch.randn(tuple(shape), generator=generator, device=rand_device, dtype=dtype).to(device)


class _DDIMBase:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, **config):
        cfg = dict(DEFAULT_CONFIG)
        cfg.update(config)
        if cfg["prediction_type"] != "v_prediction" or cfg["clip_sample"] or cfg["thresholding"]:
            raise ValueError("only the I2VGen-XL scheduler config (v_prediction, no clipping) is supported")
        self.config = SimpleNamespace(**cfg)
        self.alphas_cumprod = _alphas_cumprod(cfg)  # fp32, CPU
        one = torch.tensor(1.0)
        self.final_alpha_cumprod = one if cfg["set_alpha_to_one"] else self.alphas_cumprod[0]
        self.initial_alpha_cumprod = self.final_alpha_cumprod
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, cfg["num_train_timesteps"])[::-1].copy().astype(np.int64))

    @classmethod
    def from_pretrained(cls, *_args, **kwargs):
        """The reference loads the scheduler config from the hub; offline we use the pinned config."""
        kwargs.pop("subfolder", None)
        return cls(**kwargs)

    @classmethod
    def from_config(cls, config, **kwargs):
        """diffusers' ``SchedulerMixin.from_config`` [recalled]: a config dict or another scheduler's ``.config`` namespace;
        the keys this class does not take are ignored, ``kwargs`` override."""
        return cls(**_config_kwargs(config, DEFAULT_CONFIG, kwargs))

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _leading(self, n: int) -> np.ndarray:
        return _leading(self.config, n)

    def _alpha_pair(self, timestep):
        raise NotImplementedError

    def coefficients(self, timestep, eta: float = 0.0):
        """(sqrt(a_in), sqrt(1-a_in), sqrt(a_out), sqrt(1-a_out)) as Python floats holding exact fp32 values,
        computed with the same fp32 torch ops as the reference (`alpha ** 0.5`).  With ``eta > 0`` (DDIMScheduler only):
        (ca, cb, cc, cd', cs) with cs = sigma_t = eta * sqrt(variance) and cd' = sqrt(1 - a_out - sigma_t^2), the fp32 0-dim
        torch ops of diffusers' `DDIMScheduler._get_variance` / `step` [recalled: diffusers is not vendored]."""
        a_in, a_out = self._alpha_pair(int(timestep))
        if eta == 0.0:
            return tuple(float(c) for c in (a_in ** 0.5, (1 - a_in) ** 0.5, a_out ** 0.5, (1 - a_out) ** 0.5))
        std_dev_t = eta * self._variance(a_in, a_out) ** (0.5)
        return tuple(float(c) for c in (a_in ** 0.5, (1 - a_in) ** 0.5, a_out ** 0.5, (1 - a_out - std_dev_t ** 2) ** (0.5),
                                        std_dev_t))

    def _variance(self, a_in, a_out):
        raise ValueError(f"{type(self).__name__}.step has no eta (consisti2v/ddim_inverse_scheduler.py:291-297)")

    def step(self, model_output, timestep, sample, eta: float = 0.0, return_dict: bool = True, *,
             model_output_cond=None, guidance_scale: float = 1.0, out=None, coef_dev=None, generator=None,
             variance_noise=None, **_unused):
        """x_t -> x_{t-1} (DDIM) or x_t -> x_{t+1} (inverse).  With ``model_output_cond`` the CFG combine
        ``uncond + g*(cond-uncond)`` (pipeline :1162) is fused into the same launch.  ``eta > 0`` (DDIMScheduler) adds
        sigma_t * variance_noise in the same launch; the noise is drawn in ``model_output.shape`` from ``generator`` unless
        ``variance_noise`` is given (diffusers' rule [recalled]: not both)."""
        if eta < 0.0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if eta == 0.0:
            ca, cb, cc, cd = (0.0, 0.0, 0.0, 0.0) if coef_dev is not None else self.coefficients(timestep)
            prev = ops.ddim_step(sample.contiguous(), model_output.contiguous(),
                                 None if model_output_cond is None else model_output_cond.contiguous(),
                                 float(guidance_scale), ca, cb, cc, cd, out=out, inverse=self._inverse, coef_dev=coef_dev)
        else:
            if self._inverse:
                self._variance(None, None)
            if generator is not None and variance_noise is not None:
                raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or"
                                 " `variance_noise` stays `None`.")
            if variance_noise is None:
                variance_noise = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                                              dtype=model_output.dtype)
            ca, cb, cc, cd, cs = (0.0,) * 5 if coef_dev is not None else self.coefficients(timestep, eta)
            prev = ops.ddim_step_eta(sample.contiguous(), model_output.contiguous(),
                                     None if model_output_cond is None else model_output_cond.contiguous(),
                                     variance_noise.contiguous(), float(guidance_scale), ca, cb, cc, cd, cs, out=out,
                                     coef_dev=coef_dev)
        prev = prev.view(sample.shape)
        if not return_dict:
            return (prev,)
        return SimpleNamespace(prev_sample=prev)

    def coefficient_table(self, timesteps, guidance_scale: float, device, eta: float = 0.0) -> torch.Tensor:
        """[len(timesteps), 5] fp32 device table {ca, cb, cc, cd, guidance}: the per-step scalars of ``step`` as DATA,
        so a captured CUDA graph of one loop iteration can be replayed for every timestep.  ``eta > 0``: [len, 6]
        {ca, cb, cc, cd', guidance, cs}, the ``coef_dev`` layout of ``ops.ddim_step_eta``."""
        rows = []
        for t in timesteps:
            c = list(self.coefficients(t, eta))
            rows.append(c[:4] + [float(guidance_scale)] + c[4:])
        return torch.tensor(rows, dtype=torch.float32).to(device)


class DDIMScheduler(_DDIMBase):
    _inverse = False

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        # kept on the host: the loops index Python ints, never `.item()` a device tensor (pipeline :1143 does)
        self.timesteps = torch.from_numpy(self._leading(num_inference_steps)[::-1].copy())

    def _alpha_pair(self, t):
        t_prev = t - self.config.num_train_timesteps // self.num_inference_steps
        a_prev = self.alphas_cumprod[t_prev] if t_prev >= 0 else self.final_alpha_cumprod
        return self.alphas_cumprod[t], a_prev

    def _variance(self, alpha_prod_t, alpha_prod_t_prev):
        """diffusers `DDIMScheduler._get_variance` [recalled], fp32 0-dim tensors; the same sigma as
        seine/diffusion/gaussian_diffusion.py:585-589"""
        beta_prod_t = 1 - alpha_prod_t
        beta_prod_t_prev = 1 - alpha_prod_t_prev
        return (beta_prod_t_prev / beta_prod_t) * (1 - alpha_prod_t / alpha_prod_t_prev)


class DDIMInverseScheduler(_DDIMBase):
    _inverse = True

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        self.timesteps = torch.from_numpy(self._leading(num_inference_steps).copy())

    def _alpha_pair(self, t_next):
        t_cur = min(t_next - self.config.num_train_timesteps // self.num_inference_steps,
                    self.config.num_train_timesteps - 1)
        a_cur = self.alphas_cumprod[t_cur] if t_cur >= 0 else self.initial_alpha_cumprod
        return a_cur, self.alphas_cumprod[t_next]


#: DPMSolverMultistepScheduler's settings [recalled: diffusers 0.26, not vendored] on the I2VGen-XL config above
DPM_DEFAULT_CONFIG = dict(num_train_timesteps=1000, beta_schedule="squaredcos_cap_v2", beta_start=1e-4, beta_end=0.02,
                          trained_betas=None, solver_order=2, prediction_type="v_prediction", thresholding=False,
                          dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                          solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                          use_lu_lambdas=False, lambda_min_clipped=-float("inf"), variance_type=None,
                          timestep_spacing="leading", steps_offset=1, rescale_betas_zero_snr=True)


class DPMSolverMultistepScheduler:
    """DPM-Solver++(2M) (Lu et al. 2022, "DPM-Solver++", Alg. 2: multistep second order, data prediction) with the API of
    diffusers' ``DPMSolverMultistepScheduler`` [recalled], for ``algorithm_type="dpmsolver++"``, ``solver_order`` 1 or 2,
    ``solver_type="midpoint"``, on the I2VGen-XL beta schedule (zero-terminal-SNR rescale, v-prediction, "leading" spacing).

    With alpha_t = sqrt(abar_t), sigma_t = sqrt(1 - abar_t), lambda_t = log(alpha_t / sigma_t), one step t -> s is
        x0 = alpha_t x - sigma_t v                       (v-prediction -> data prediction)
        D  = x0 + c (x0 - x0_prev),   c = h / (2 h_prev) (c = 0 on a first-order step)
        x_s = a x + b D,   a = sigma_s / sigma_t,   b = -alpha_s (exp(-h) - 1),   h = lambda_s - lambda_t
    where h_prev = lambda_t - lambda_{t_prev} is the previous step's.  The first-order step is DDIM (eta = 0).  diffusers'
    rules [recalled]: the first step is first order (no x0_prev yet); the last is too when ``euler_at_final``, or when
    ``lower_order_final`` and the schedule has fewer than 15 steps; the last step's target is abar_0 (not 1).  The
    coefficients are computed in float64 from the fp32 abar table and passed to the kernel as fp32.

    The loops keep the previous step's x0 in a buffer of their own (``x0_prev``, fp16, the latents' shape), which the fused
    kernel reads and overwrites in place, so one captured graph with the per-step coefficient row as data serves every step."""
    order = 1            # diffusers' value: one model evaluation per step
    init_noise_sigma = 1.0
    multistep = True     # the sampling loops keep an x0_prev buffer for it

    def __init__(self, **config):
        unknown = sorted(set(config) - set(DPM_DEFAULT_CONFIG))
        if unknown:
            raise ValueError(f"DPMSolverMultistepScheduler: unknown setting(s) {unknown}")
        cfg = dict(DPM_DEFAULT_CONFIG)
        cfg.update(config)
        for key, ok, what in (
                ("algorithm_type", cfg["algorithm_type"] == "dpmsolver++", "only 'dpmsolver++'"),
                ("solver_order", cfg["solver_order"] in (1, 2), "1 or 2"),
                ("solver_type", cfg["solver_type"] == "midpoint", "only 'midpoint'"),
                ("prediction_type", cfg["prediction_type"] == "v_prediction", "only 'v_prediction'"),
                ("thresholding", not cfg["thresholding"], "False"),
                ("use_karras_sigmas", not cfg["use_karras_sigmas"], "False"),
                ("use_lu_lambdas", not cfg["use_lu_lambdas"], "False"),
                ("lambda_min_clipped", cfg["lambda_min_clipped"] == -float("inf"), "-inf"),
                ("variance_type", cfg["variance_type"] is None, "None"),
                ("trained_betas", cfg["trained_betas"] is None, "None"),
                ("timestep_spacing", cfg["timestep_spacing"] == "leading", "only 'leading'")):
            if not ok:
                raise ValueError(f"DPMSolverMultistepScheduler: {key}={cfg[key]!r} is not supported ({what})")
        self.config = SimpleNamespace(**cfg)
        self.alphas_cumprod = _alphas_cumprod(cfg)  # fp32, CPU
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, cfg["num_train_timesteps"])[::-1].copy().astype(np.int64))
        self.lower_order_nums = 0
        self._x0_prev = None

    @classmethod
    def from_config(cls, config, **kwargs):
        """``DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)``: the keys it does not take (DDIM's
        ``clip_sample``, ``set_alpha_to_one`` ...) are ignored, ``kwargs`` override"""
        return cls(**_config_kwargs(config, DPM_DEFAULT_CONFIG, kwargs))

    @classmethod
    def from_pretrained(cls, *_args, **kwargs):
        """offline: the pinned config (as the DDIM classes)"""
        kwargs.pop("subfolder", None)
        return cls(**kwargs)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_timesteps(self, num_inference_steps: int, device=None):
        """descending "leading" timesteps (25 steps: 961, 921, ..., 1); forgets the previous step's x0"""
        self.num_inference_steps = num_inference_steps
        self.timesteps = torch.from_numpy(_leading(self.config, num_inference_steps)[::-1].copy())
        self.lower_order_nums = 0
        self._x0_prev = None

    # -- float64 schedule --------------------------------------------------------------------------------------------
    def alpha_sigma(self, t) -> tuple:
        """(alpha_t, sigma_t) in float64; t = None: the final target, abar_0 (diffusers 0.26's last sigma [recalled])"""
        abar = float(self.alphas_cumprod[0 if t is None else int(t)])
        return math.sqrt(abar), math.sqrt(1.0 - abar)

    def lambda_(self, t) -> float:
        alpha, sigma = self.alpha_sigma(t)
        return math.log(alpha) - math.log(sigma)

    def _index(self, t) -> int:
        ts = self.timesteps.tolist()
        if int(t) not in ts:
            raise ValueError(f"timestep {int(t)} is not in the schedule {ts}")
        return ts.index(int(t))

    def _target(self, k: int):
        """the timestep step k of the schedule goes to (None: the final target)"""
        return int(self.timesteps[k + 1]) if k + 1 < len(self.timesteps) else None

    def _first_order_at(self, k: int, have_prev: bool) -> bool:
        n = len(self.timesteps)
        final = k == n - 1 and (self.config.euler_at_final or (self.config.lower_order_final and n < 15))
        return self.config.solver_order == 1 or not have_prev or final

    def coefficient_row(self, t, first_order: bool) -> tuple:
        """(alpha_t, sigma_t, a, b, c) of the step from t, float64"""
        k = self._index(t)
        s = self._target(k)
        alpha_t, sigma_t = self.alpha_sigma(t)
        alpha_s, sigma_s = self.alpha_sigma(s)
        h = self.lambda_(s) - self.lambda_(t)
        a = sigma_s / sigma_t
        b = -alpha_s * math.expm1(-h)
        c = 0.0
        if not first_order:
            if k == 0:
                raise ValueError(f"a second-order step from t={int(t)} needs the previous timestep of the schedule")
            h_prev = self.lambda_(t) - self.lambda_(int(self.timesteps[k - 1]))
            c = h / (2.0 * h_prev)  # 1 / (2 r), r = h_prev / h
        return alpha_t, sigma_t, a, b, c

    def coefficient_table(self, timesteps, guidance_scale: float, device, eta: float = 0.0) -> torch.Tensor:
        """[len(timesteps), 6] fp32 device table {alpha_t, sigma_t, a, b, c, guidance}: the ``coef_dev`` rows of
        ``ops.dpmpp2m_step`` for a loop over ``timesteps`` (consecutive timesteps of the schedule; its first step has no
        x0_prev and is first order)"""
        if eta != 0.0:
            raise ValueError(f"DPMSolverMultistepScheduler: eta={eta} is not supported (DPM-Solver++ here is deterministic)")
        rows = []
        for i, t in enumerate(timesteps):
            k = self._index(t)
            if i > 0 and (k == 0 or int(self.timesteps[k - 1]) != int(timesteps[i - 1])):
                raise ValueError(f"timesteps {list(timesteps)} are not consecutive steps of the schedule")
            rows.append(list(self.coefficient_row(t, self._first_order_at(k, i > 0))) + [float(guidance_scale)])
        return torch.tensor(rows, dtype=torch.float64).to(torch.float32).reshape(len(rows), 6).to(device)

    # -- device step -------------------------------------------------------------------------------------------------
    def step(self, model_output, timestep, sample, return_dict: bool = True, *, model_output_cond=None,
             guidance_scale: float = 1.0, out=None, coef_dev=None, x0_prev=None, eta: float = 0.0, variance_noise=None,
             generator=None, **_unused):
        """x_t -> x_s, ONE launch of the fused kernel (CFG ``uncond + g*(cond-uncond)`` with ``model_output_cond``).
        ``coef_dev`` (the loops): the step's row of ``coefficient_table`` on the device, with the loop's ``x0_prev`` buffer.
        Without it (diffusers-style use): the coefficients of ``timestep`` on the host, with the history this scheduler
        keeps itself since ``set_timesteps``."""
        if eta != 0.0 or variance_noise is not None:
            raise ValueError(f"DPMSolverMultistepScheduler: eta={eta} / variance_noise is not supported")
        mo_cond = None if model_output_cond is None else model_output_cond.contiguous()
        if x0_prev is not None and (x0_prev.shape != sample.shape or x0_prev.dtype != torch.float16):
            raise ValueError(f"DPMSolverMultistepScheduler.step: x0_prev must be an fp16 tensor of the sample's shape "
                             f"{tuple(sample.shape)}, got {x0_prev.dtype} {tuple(x0_prev.shape)}")
        if coef_dev is not None:
            if x0_prev is None:
                raise ValueError("DPMSolverMultistepScheduler.step with coef_dev needs the loop's x0_prev buffer")
            prev = ops.dpmpp2m_step(sample.contiguous(), model_output.contiguous(), mo_cond, x0_prev, 0.0, 0.0, 0.0, 0.0, 0.0,
                                    0.0, out=out, coef_dev=coef_dev)
        else:
            k = self._index(timestep)
            first = self._first_order_at(k, self.lower_order_nums >= 1)
            if x0_prev is None:
                if self._x0_prev is None or self._x0_prev.shape != sample.shape or self._x0_prev.device != sample.device:
                    self._x0_prev = torch.zeros_like(sample, dtype=torch.float16)
                    first = True
                x0_prev = self._x0_prev
            alpha_t, sigma_t, a, b, c = self.coefficient_row(timestep, first)
            prev = ops.dpmpp2m_step(sample.contiguous(), model_output.contiguous(), mo_cond, x0_prev, float(guidance_scale),
                                    alpha_t, sigma_t, a, b, c, out=out)
            self.lower_order_nums = min(self.lower_order_nums + 1, self.config.solver_order)
        prev = prev.view(sample.shape)
        if not return_dict:
            return (prev,)
        return SimpleNamespace(prev_sample=prev)
