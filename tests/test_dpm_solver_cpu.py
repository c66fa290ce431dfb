"""DPM-Solver++(2M) sampling (`DPMSolverMultistepScheduler`) in `I2VGenXLPipeline.__call__` and the PnP edit, without a GPU:
the schedule and the coefficient rows against the float64 restatement of tests/dpm_solver_ref.py, the first-order step
against DDIM, two analytic checks of the solver (a point-mass data distribution, a data prediction linear in lambda), the
product loops on the tiny UNet (kernels replaced by their contracts) against a plain loop, the inversion store a 25-step
edit reads, the refusals and the runner's ``scheduler`` key.  tests/test_gpu_dpm_solver.py runs the kernel and the full-size
loops on the GPU."""
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import dpm_solver_ref
import freeu_ref
import sampling_ref
import source_cache_ref
from test_host_model_cpu import F_, H_, W_, _models

N_STEPS = 5          # 801, 601, 401, 201, 1: every other timestep of a 10-step inversion
STORE_STEPS = 10
PNP = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.6, pnp_spatial_attn_t=0.4, pnp_temp_attn_t=0.2)


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    """the kernel contracts in place of anyv2v_b200.ops, ops.dpmpp2m_step and the source-feature kernels included"""
    sampling_ref.patch_ops(monkeypatch)
    freeu_ref.patch_ops(monkeypatch)
    source_cache_ref.patch_ops(monkeypatch)
    dpm_solver_ref.patch_ops(monkeypatch)
    return emulated_ops


def _dpm(n=None, **kw):
    from anyv2v_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(**kw)
    if n is not None:
        s.set_timesteps(n)
    return s


# ---------------------------------------------------------------------------------------------------------- schedule
@pytest.mark.parametrize("n", [10, 20, 25, 50])
def test_schedule_against_the_float64_restatement(n):
    s = _dpm(n)
    ts = s.timesteps.tolist()
    assert ts == dpm_solver_ref.timesteps(n)
    ref_alpha, ref_sigma = dpm_solver_ref.alpha_sigma_t(dpm_solver_ref.sigmas(n))
    ref_lam = dpm_solver_ref.lambdas(n)
    for k, t in enumerate(ts + [None]):
        alpha, sigma = s.alpha_sigma(t)
        assert math.isclose(alpha, ref_alpha[k], rel_tol=1e-13) and math.isclose(sigma, ref_sigma[k], rel_tol=1e-13), (k, t)
        assert math.isclose(s.lambda_(t), ref_lam[k], rel_tol=1e-12, abs_tol=1e-12), (k, t)
    rows = s.coefficient_table(ts, 9.0, "cpu")
    want = dpm_solver_ref.coefficient_rows(n)
    assert rows.dtype == torch.float32 and rows.shape == (n, 6) and bool((rows[:, 5] == 9.0).all())
    np.testing.assert_allclose(rows[:, :5].double().numpy(), want, rtol=2e-7, atol=0)
    first = [bool(c == 0) for c in rows[:, 4].tolist()]
    assert first == dpm_solver_ref.first_order_rows(n)
    assert first[-1] == (n < 15)                       # lower_order_final applies below 15 steps only
    # a loop that starts later (ddim_init_latents_t_idx = 1) starts first order, then follows the same rows
    late = s.coefficient_table(ts[1:], 9.0, "cpu")
    np.testing.assert_allclose(late[:, :5].double().numpy(), dpm_solver_ref.coefficient_rows(n, t_idx=1), rtol=2e-7, atol=0)


def test_25_steps_are_every_other_timestep_of_50():
    from anyv2v_b200.schedulers import DDIMScheduler
    d = DDIMScheduler()
    d.set_timesteps(50)
    t25 = _dpm(25).timesteps.tolist()
    assert t25[:2] == [961, 921] and t25[-1] == 1 and set(t25) <= set(d.timesteps.tolist())


@pytest.mark.parametrize("n", [10, 25, 50])
def test_first_order_step_is_ddim(n):
    """a first-order row maps (x, v) to DDIM's eta = 0 update, to float64 rounding: both are linear in x and v, so their two
    coefficients are compared; DDIM's target is the next timestep, or abar_0 at the last step (diffusers 0.26's DPM target)"""
    from anyv2v_b200.schedulers import DDIMScheduler
    s = _dpm(n)
    ddim = DDIMScheduler()
    ddim.set_timesteps(n)
    ac = s.alphas_cumprod.double()
    ts = s.timesteps.tolist()
    for k, t in enumerate(ts):
        alpha, sigma, a, b, c = s.coefficient_row(t, first_order=True)
        assert c == 0.0
        a_prev = float(ac[ts[k + 1]]) if k + 1 < n else float(ac[0])
        ca, cb, cc, cd = math.sqrt(float(ac[t])), math.sqrt(1 - float(ac[t])), math.sqrt(a_prev), math.sqrt(1 - a_prev)
        ddim_x, ddim_v = cc * ca + cd * cb, cd * ca - cc * cb       # cc * (ca x - cb v) + cd * (ca v + cb x)
        assert math.isclose(a + b * alpha, ddim_x, rel_tol=1e-12), (t, a + b * alpha, ddim_x)
        assert math.isclose(-b * sigma, ddim_v, rel_tol=1e-10, abs_tol=1e-14), (t, -b * sigma, ddim_v)
        if k + 1 < n:  # and the product's own DDIM coefficients (fp32) agree to fp32 rounding
            d = ddim.coefficients(t)
            assert math.isclose(d[0] * d[2] + d[1] * d[3], ddim_x, rel_tol=1e-6)


# ---------------------------------------------------------------------------------------------------------- analytic checks
def _solve(s, x_T, x0_fn, t_idx=0):
    """the solver in float64 with the scheduler's rows: x0_fn(x, t) is the data prediction at step t"""
    ts = s.timesteps.tolist()[t_idx:]
    rows = s.coefficient_table(ts, 1.0, "cpu")  # only to learn which rows are first order
    x, prev = x_T.clone(), None
    for i, t in enumerate(ts):
        alpha, sigma, a, b, c = s.coefficient_row(t, first_order=bool(rows[i, 4] == 0))
        x0 = x0_fn(x, t)
        d = x0 if c == 0.0 else x0 + c * (x0 - prev)
        x, prev = a * x + b * d, x0
    return x


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("n", [10, 25])
def test_exact_denoiser_of_a_point_mass_lands_on_the_point(order, n):
    """data = one point x*: the exact data prediction is x* at every t, and both orders take x_T = alpha_T x* + sigma_T eps
    exactly to alpha_0 x* + sigma_0 eps, the point at the final noise level abar_0 (sigma_0 ~ 6e-3)"""
    s = _dpm(n, solver_order=order)
    g = torch.Generator().manual_seed(1)
    xs, eps = torch.randn(64, generator=g, dtype=torch.float64), torch.randn(64, generator=g, dtype=torch.float64)
    a_T, s_T = s.alpha_sigma(s.timesteps[0])
    a_0, s_0 = s.alpha_sigma(None)
    got = _solve(s, a_T * xs + s_T * eps, lambda x, t: xs)
    torch.testing.assert_close(got, a_0 * xs + s_0 * eps, rtol=0, atol=1e-12)
    assert float((got - xs).abs().max()) < 0.05 and s_0 < 7e-3


def test_second_order_beats_first_order_on_a_prediction_linear_in_lambda():
    """x0(lambda) = A + B lambda: the probability-flow ODE in lambda, x_s / sigma_s = x_t / sigma_t + int e^lambda x0 dlambda,
    integrates in closed form; over 25 steps the 2nd-order solution is closer to it than the 1st-order one"""
    g = torch.Generator().manual_seed(2)
    A, B = torch.randn(32, generator=g, dtype=torch.float64), torch.randn(32, generator=g, dtype=torch.float64) * 0.3
    errs = {}
    for order in (1, 2):
        s = _dpm(25, solver_order=order)
        x_T = torch.randn(32, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
        got = _solve(s, x_T, lambda x, t: A + B * s.lambda_(t))
        l_T, l_0 = s.lambda_(s.timesteps[0]), s.lambda_(None)
        prim = lambda lam: math.exp(lam) * (A + B * (lam - 1.0))
        _, s_T = s.alpha_sigma(s.timesteps[0])
        _, s_0 = s.alpha_sigma(None)
        exact = s_0 * (x_T / s_T + prim(l_0) - prim(l_T))
        errs[order] = float((got - exact).abs().max() / exact.abs().max())
    assert errs[2] < 0.25 * errs[1], errs


# ---------------------------------------------------------------------------------------------------------- loops
def _call_kwargs(ns, guidance):
    return dict(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
                image_latents=ns.edit_image_latents, num_inference_steps=N_STEPS, guidance_scale=guidance, target_fps=8,
                output_type="latent")


def _plain_call(ours, ns, lat, guidance, t_idx=1):
    """the image-to-video loop in plain torch: our UNet on [uncond, cond], then the kernel contract with the restated rows"""
    cfg = guidance > 1
    prompts = torch.cat([ns.neg_prompt, ns.edit_prompt]) if cfg else ns.edit_prompt
    img_emb = torch.cat([torch.zeros_like(ns.edit_image_emb), ns.edit_image_emb]) if cfg else ns.edit_image_emb
    img_lat = torch.cat([ns.edit_image_latents] * (2 if cfg else 1))
    cond = ours.precompute_conditioning(torch.tensor([8] * img_lat.shape[0]), img_lat, img_emb, prompts)
    x, p = lat.clone(), torch.zeros_like(lat)
    ts = dpm_solver_ref.timesteps(N_STEPS)[t_idx:]
    for t, row in zip(ts, dpm_solver_ref.coefficient_rows(N_STEPS, t_idx)):
        v = ours(torch.cat([x, x]) if cfg else x, torch.tensor([t]), cond=cond)[0]
        x = dpm_solver_ref.dpmpp2m_step(x, v[0:1], v[1:2] if cfg else None, p, guidance, *row.tolist())
    return x


@torch.no_grad()
@pytest.mark.parametrize("guidance", [1.0, 9.0])
def test_call_equals_the_plain_loop(emu, guidance):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    lat = torch.randn(1, 4, F_, H_, W_, generator=torch.Generator().manual_seed(11)).half()
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    pipe.scheduler = DPMSolverMultistepScheduler.from_config(pipe.scheduler.config)
    states, real = [], pipe.prepare_call
    pipe.prepare_call = lambda *a, **k: states.append(real(*a, **k)) or states[-1]
    got = pipe(latents=lat, **_call_kwargs(ns, guidance)).frames
    st = states[0]
    assert st.timesteps == [601, 401, 201, 1] and st.x0_prev.shape == lat.shape and st.coef_table.shape == (4, 6)
    assert len(st.iterations) == 1                               # one loop iteration (graph) for every step
    want = _plain_call(ours, ns, lat, guidance)
    assert torch.isfinite(got.float()).all() and torch.equal(got, want)


@torch.no_grad()
def test_ddim_call_allocates_no_x0_prev(emu):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMScheduler
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = I2VGenXLPipeline(ours, DDIMScheduler())
    st = pipe.prepare_call(ns.video_latents, ns.edit_prompt, ns.edit_image_latents, ns.edit_image_emb, 8, N_STEPS, 9.0,
                           ns.neg_prompt)
    assert st.x0_prev is None and st.coef_table.shape == (N_STEPS - 1, 5)


def _store(steps=STORE_STEPS, seed=5, drop=()):
    """random source latents at every timestep of a ``steps``-step DDIM inversion"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(steps)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(seed)
    for t in s.timesteps.tolist():
        x = torch.randn(1, 4, F_, H_, W_, generator=g).half()
        if t not in drop:
            store.put(int(t), x)
    return store


def _edit_pipeline(ours, n_steps=N_STEPS, pnp=PNP):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    sched = _dpm(n_steps)
    pipe = I2VGenXLPipeline(ours, sched)
    init_pnp(pipe, sched, pnp)
    return pipe


def _edit(pipe, ns, store, n_steps=N_STEPS, **kw):
    return pipe.sample_with_pnp(latents=ns.video_latents.clone(), prompt_embeds=ns.edit_prompt,
                                negative_prompt_embeds=ns.neg_prompt, ddim_inv_prompt_embeds=ns.inv_prompt,
                                image_embeddings=ns.edit_image_emb, image_latents=ns.edit_image_latents,
                                ddim_inv_image_embeddings=ns.src_image_emb, ddim_inv_image_latents=ns.src_image_latents,
                                target_fps=8, num_inference_steps=n_steps, guidance_scale=9.0, ddim_init_latents_t_idx=1,
                                latent_store=store, return_dict=False, **kw)[0]


def _plain_edit(pipe, ns, store):
    """the PnP edit in plain torch: our hooked UNet on [source, uncond, cond] at every step, then the kernel contract"""
    from anyv2v_b200.pnp_utils import register_time
    ours = pipe.unet
    prompts = torch.cat([ns.inv_prompt, ns.neg_prompt, ns.edit_prompt])
    img_emb = torch.cat([ns.src_image_emb, torch.zeros_like(ns.edit_image_emb), ns.edit_image_emb])
    img_lat = torch.cat([ns.src_image_latents, ns.edit_image_latents, ns.edit_image_latents])
    cond = ours.precompute_conditioning(torch.tensor([8] * 3), img_lat, img_emb, prompts)
    x = ns.video_latents.clone()
    p = torch.zeros_like(x)
    for t, row in zip(dpm_solver_ref.timesteps(N_STEPS)[1:], dpm_solver_ref.coefficient_rows(N_STEPS, 1)):
        register_time(pipe, t)
        v = ours(torch.cat([store.get(t), x, x]), torch.tensor([t]), cond=cond)[0]
        x = dpm_solver_ref.dpmpp2m_step(x, v[1:2], v[2:3], p, 9.0, *row.tolist())
    return x


@torch.no_grad()
@pytest.mark.parametrize("skip", [True, False])
def test_edit_equals_the_plain_loop(emu, skip):
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    store = _store()
    pipe = _edit_pipeline(ours)
    got = _edit(pipe, ns, store, skip_dead_source_branch=skip)
    want = _plain_edit(pipe, ns, store)
    assert torch.isfinite(got.float()).all() and torch.equal(got, want)


@torch.no_grad()
def test_edit_with_the_source_feature_cache_equals_the_plain_loop(emu):
    """the cache keys on the timestep: a second DPM edit replays the first one's source features, bit for bit"""
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    store = _store()
    pipe = _edit_pipeline(ours)
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    first = _edit(pipe, ns, store, source_features=cache)
    assert len(cache) > 0
    g = torch.Generator().manual_seed(4)
    ns.edit_prompt = (ns.edit_prompt.float() + torch.randn(ns.edit_prompt.shape, generator=g)).half()
    states, real = [], pipe.prepare_edit
    pipe.prepare_edit = lambda *a, **k: states.append(real(*a, **k)) or states[-1]
    second = _edit(pipe, ns, store, source_features=cache)
    pipe.prepare_edit = real
    assert any(k[-1] == "replay" for k in states[0].iterations)
    want = _plain_edit(pipe, ns, store)
    assert not torch.equal(first, second) and torch.equal(second, want)


@torch.no_grad()
def test_25_step_edit_reads_a_50_step_inversion_store(emu):
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    store = _store(steps=50)
    reads, real_get = [], store.get
    store.get = lambda t, device=None: reads.append(int(t)) or real_get(t, device)
    pnp = SimpleNamespace(n_steps=25, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0)
    pipe = _edit_pipeline(ours, 25, pnp)
    out = _edit(pipe, ns, store, n_steps=25, max_steps=3)
    assert reads == [921, 881, 841] and torch.isfinite(out.float()).all()


@torch.no_grad()
def test_a_store_missing_timesteps_is_refused_before_the_first_step(emu):
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = _edit_pipeline(ours)
    n0 = emu.launch_count()
    with pytest.raises(ValueError, match=r"timestep\(s\) \[401, 1\]"):
        _edit(pipe, ns, _store(drop=(401, 1, 901)))
    assert emu.launch_count() == n0
    # the 10-step store lacks half of the timesteps of a 10-step DPM edit: listed the same way
    with pytest.raises(ValueError, match=r"\[851, 751"):
        _edit(_edit_pipeline(ours, 20, SimpleNamespace(n_steps=20, pnp_f_t=0.5, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)),
              ns, _store(), n_steps=20)


# ---------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("kw,word", [({"algorithm_type": "sde-dpmsolver++"}, "algorithm_type"), ({"solver_order": 3}, "solver_order"),
                                     ({"use_karras_sigmas": True}, "use_karras_sigmas"), ({"solver_type": "heun"}, "solver_type"),
                                     ({"prediction_type": "epsilon"}, "prediction_type"), ({"thresholding": True}, "thresholding"),
                                     ({"timestep_spacing": "trailing"}, "timestep_spacing"), ({"no_such_key": 1}, "no_such_key")])
def test_unsupported_options_are_refused(kw, word):
    with pytest.raises(ValueError, match=word):
        _dpm(**kw)


def test_from_config_takes_a_dict_or_a_config_namespace():
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler, DPMSolverMultistepScheduler
    ddim = DDIMScheduler()
    dpm = DPMSolverMultistepScheduler.from_config(ddim.config)
    assert isinstance(dpm, DPMSolverMultistepScheduler) and dpm.config.solver_order == 2
    assert torch.equal(dpm.alphas_cumprod, ddim.alphas_cumprod)
    assert DPMSolverMultistepScheduler.from_config(vars(ddim.config), solver_order=1).config.solver_order == 1
    back = DDIMScheduler.from_config(dpm.config)
    assert isinstance(back, DDIMScheduler) and vars(back.config) == vars(ddim.config)
    inv = DDIMInverseScheduler.from_config({"steps_offset": 1, "solver_order": 2})
    assert isinstance(inv, DDIMInverseScheduler)


def test_eta_is_refused():
    s = _dpm(10)
    with pytest.raises(ValueError, match="eta"):
        s.coefficient_table(s.timesteps.tolist(), 9.0, "cpu", eta=0.5)


@torch.no_grad()
def test_pipeline_refusals(emu):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from oracle import loops_ref
    _, ours = _models()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = I2VGenXLPipeline(ours, _dpm())
    with pytest.raises(ValueError, match="eta"):
        pipe(latents=ns.video_latents, eta=1.0, **_call_kwargs(ns, 9.0))
    with pytest.raises(ValueError, match="DDIMInverseScheduler"):
        pipe.invert(latents=ns.video_latents, prompt_embeds=ns.inv_prompt, image_latents=ns.src_image_latents,
                    image_embeddings=ns.src_image_emb, num_inference_steps=N_STEPS, write_files=False)


def test_step_refuses_a_wrong_x0_prev(emu):
    s = _dpm(N_STEPS)
    x, v = torch.zeros(1, 4, 2, 8, 8, dtype=torch.float16), torch.zeros(1, 4, 2, 8, 8, dtype=torch.float16)
    coef = s.coefficient_table(s.timesteps.tolist(), 1.0, "cpu")[0]
    with pytest.raises(ValueError, match="x0_prev"):
        s.step(v, None, x, coef_dev=coef)
    with pytest.raises(ValueError, match="x0_prev"):
        s.step(v, None, x, coef_dev=coef, x0_prev=torch.zeros(1, 4, 2, 8, 4, dtype=torch.float16))
    with pytest.raises(ValueError, match="x0_prev"):
        s.step(v, None, x, coef_dev=coef, x0_prev=torch.zeros(1, 4, 2, 8, 8, dtype=torch.float32))
    p = torch.zeros_like(x)
    assert torch.equal(s.step(v, None, x, coef_dev=coef, x0_prev=p).prev_sample, x)


def test_host_step_keeps_its_own_history(emu):
    """``step`` without coef_dev (diffusers-style): first order, then second order from the x0 it kept"""
    s = _dpm(N_STEPS)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 64, generator=g).half()
    ref = dpm_solver_ref.DPMRef()
    ref.set_timesteps(N_STEPS)
    want = x.clone()
    for t in s.timesteps.tolist():
        v = torch.randn(2, 64, generator=g).half()
        x = s.step(v, t, x).prev_sample
        want, _ = ref.step(v.double(), t, want.double())
        torch.testing.assert_close(x.double(), want, rtol=4e-3, atol=4e-3)
        want = x.clone()
    assert s.lower_order_nums == 2


def test_dpm_args_struct_matches_the_c_header(tmp_path):
    """ctypes mirror of av2v_dpmpp2m_args against the layout gcc gives include/anyv2v_b200.h"""
    import ctypes
    import os
    import subprocess
    from anyv2v_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cls = _lib.DpmArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "anyv2v_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(av2v_dpmpp2m_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(av2v_dpmpp2m_args, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(tmp_path / "probe.c"), "-o", str(tmp_path / "probe")], check=True)
    out = dict(l.split() for l in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    assert all(int(out[f]) == getattr(cls, f).offset for f, _ in cls._fields_)


# ---------------------------------------------------------------------------------------------------------- runner
def test_runner_scheduler_key(emu, tmp_path):
    """``scheduler: dpmsolver++`` edits a 10-step inversion in 5 DPM-Solver++ steps and saves under its own suffix; without
    the key (or with ``ddim``) the edit is the DDIM edit"""
    import yaml
    from test_gpu_runners import EDIT_TEMPLATE, INV_TEMPLATE
    from anyv2v_b200 import run_group_ddim_inversion as inv, run_group_pnp_edit as edit
    from anyv2v_b200.config import OmegaConf
    from oracle.unet_ref import TINY_CONFIG
    data = str(tmp_path)
    inv_t = dict(INV_TEMPLATE, data_dir=data, device="cpu")
    inv_t["inverse_config"] = dict(inv_t["inverse_config"], n_steps=STORE_STEPS)
    inv_t["recon_config"] = dict(inv_t["recon_config"], enable_recon=False)
    (tmp_path / "inv.yaml").write_text(yaml.safe_dump(inv_t))
    (tmp_path / "edit.yaml").write_text(yaml.safe_dump(dict(EDIT_TEMPLATE, data_dir=data, device="cpu", n_steps=STORE_STEPS)))
    base = {"active": True, "video_name": "clipA", "edited_first_frame_path": "x", "editing_prompt": "a robot",
            "edited_video_name": "robot"}
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    try:
        device = torch.device("cpu")
        inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), [base], device, unet_config=TINY_CONFIG)
        run = lambda **kw: edit.main(OmegaConf.load(str(tmp_path / "edit.yaml")), [dict(base, **kw)], device,
                                     unet_config=TINY_CONFIG)[0]
        plain = run()
        assert torch.equal(run(scheduler="ddim"), plain)
        dpm = run(scheduler="dpmsolver++", n_steps=N_STEPS)
        assert torch.isfinite(dpm.float()).all() and not torch.equal(dpm, plain)
        out = os.path.join(data, "Results", "Prompt-Based-Editing", "i2vgen-xl", "clipA", "robot")
        suffix = "ddim_init_latents_t_idx_1_nsteps_5_cfg_9.0_pnpf0.2_pnps0.2_pnpt0.5_dpmsolver++"
        assert torch.equal(torch.load(os.path.join(out, suffix, "edited_latents.pt")), dpm)
        assert os.path.exists(os.path.join(out, "ddim_init_latents_t_idx_1_nsteps_10_cfg_9.0_pnpf0.2_pnps0.2_pnpt0.5"))
        with pytest.raises(ValueError, match="scheduler"):
            run(scheduler="unipc")
    finally:
        torch.set_grad_enabled(prev)
