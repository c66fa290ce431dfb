"""DPM-Solver++(2M) on the GPU: ops.dpmpp2m_step against its contract inside guarded buffers (bit for bit against the fp32
restatement, within the ulp bound of its float64 values and unbiased), the wrapper's refusals, a 25-step `__call__` with CUDA
graphs equal to eager launches, 25-step `__call__` and PnP edit steps against the fp32 oracle at 16 x 512^2 (full-size UNet;
the edit reads a 50-step inversion), and a DDIM edit that is unchanged by a DPM edit run before it."""
from types import SimpleNamespace

import pytest
import torch

import dpm_solver_ref
import test_gpu_fullwidth as fw
from bias_check import assert_unbiased
from guarded import check_output, guarded_inout, guarded_input, guarded_output
from ulp_check import assert_within_bound

pytestmark = pytest.mark.gpu
dev = "cuda"
#: the kernel's fp32 arithmetic between its two fp16 roundings: at most a few fp32 roundings of the terms it adds
KAPPA_DPM = 2.0 ** -21
F_, H_, W_ = 16, 64, 64
N_STEPS = 25
INV_STEPS = 50
GUIDANCE = 9.0
FPS = 8
PNP = SimpleNamespace(pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)   # BASELINE config 3


def _rows():
    """a first-order row (the loop's first step) and a second-order row of the 25-step schedule"""
    from anyv2v_b200.schedulers import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(N_STEPS)
    table = s.coefficient_table(s.timesteps.tolist()[1:], GUIDANCE, "cpu")
    assert table[0, 4] == 0 and table[10, 4] != 0
    return {"first": table[0].tolist(), "second": table[10].tolist()}


@pytest.mark.parametrize("n", [4 * 16 * 64 * 64, 1001])
@pytest.mark.parametrize("order", ["first", "second"])
@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("in_place", [True, False])
def test_dpm_step_against_contract_guarded(n, order, cfg, in_place):
    from anyv2v_b200 import ops
    torch.manual_seed(n + 2 * cfg + 4 * in_place)
    x_h, vn_h, ve_h = (torch.randn(n).half() for _ in range(3))
    p_h = (torch.randn(n) * 1.5).half()
    al, si, a, b, c, g = _rows()[order]
    if not cfg:
        g = 1.0
    vn, ve = guarded_input(vn_h, device=dev), guarded_input(ve_h, device=dev)
    x = guarded_inout(x_h.to(dev)) if in_place else guarded_input(x_h, device=dev)
    out = x if in_place else guarded_output((n,), device=dev)
    p = guarded_inout(p_h.to(dev))
    coef = torch.tensor([al, si, a, b, c, g], dtype=torch.float32, device=dev)
    ops.dpmpp2m_step(x.view, vn.view, ve.view if cfg else None, p.view, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, out=out.view,
                     coef_dev=coef)
    torch.cuda.synchronize()
    check_output(out, "dpmpp2m_step out")
    check_output(p, "dpmpp2m_step x0_prev")
    # bit for bit: the fp32 restatement on the CPU
    p_cpu = p_h.clone()
    want = dpm_solver_ref.dpmpp2m_step(x_h, vn_h, ve_h if cfg else None, p_cpu, g, al, si, a, b, c)
    assert torch.equal(out.view.cpu().view(torch.int16), want.view(torch.int16))
    assert torch.equal(p.view.cpu().view(torch.int16), p_cpu.view(torch.int16))
    # float64: both stores within the ulp bound, and unbiased where there are enough elements
    x0, cx0, y, cy = dpm_solver_ref.dpmpp2m_exact(x_h, vn_h, ve_h if cfg else None, p_h, g, al, si, a, b, c, p.view.cpu())
    what = f"dpmpp2m n={n} {order} cfg={cfg} in_place={in_place}"
    assert_within_bound(p.view.cpu(), x0, cx0, KAPPA_DPM, what + " x0")
    assert_within_bound(out.view.cpu(), y, cy, KAPPA_DPM, what + " out")
    if n >= 1 << 18:  # enough elements for the bias statistics' power; 8 columns = the element's place in a 16-byte vector
        assert_unbiased(p.view.cpu().view(-1, 8), x0.view(-1, 8), cx0.view(-1, 8), KAPPA_DPM, what + " x0")
        assert_unbiased(out.view.cpu().view(-1, 8), y.view(-1, 8), cy.view(-1, 8), KAPPA_DPM, what + " out")


def test_first_order_row_does_not_read_x0_prev():
    """c = 0: x0_prev is only written (a NaN there does not reach the output)"""
    from anyv2v_b200 import ops
    n = 4096
    x, vn = torch.randn(n, device=dev).half(), torch.randn(n, device=dev).half()
    p = torch.full((n,), float("nan"), device=dev, dtype=torch.float16)
    al, si, a, b, c, _ = _rows()["first"]
    y = ops.dpmpp2m_step(x, vn, None, p, 1.0, al, si, a, b, c)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all() and torch.isfinite(p).all()


def _h(*shape, device=dev, dtype=torch.float16):
    return torch.zeros(*shape, device=device, dtype=dtype)


_BUF = {}


def _shared(n):
    """one buffer, for the aliasing refusals"""
    if n not in _BUF:
        _BUF[n] = _h(n)
    return _BUF[n]


REFUSALS = {
    "x dtype": lambda o: o.dpmpp2m_step(_h(16, dtype=torch.float32), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0),
    "x0_prev dtype": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(16, dtype=torch.float32), 1.0, 1, 0, 1, 0, 0),
    "x0_prev device": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(16, device="cpu"), 1.0, 1, 0, 1, 0, 0),
    "x0_prev strided": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(32)[::2], 1.0, 1, 0, 1, 0, 0),
    "x0_prev size": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(8), 1.0, 1, 0, 1, 0, 0),
    "v_edit size": lambda o: o.dpmpp2m_step(_h(16), _h(16), _h(24), _h(16), 1.0, 1, 0, 1, 0, 0),
    "out size": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0, out=_h(8)),
    "x0_prev is x": lambda o: o.dpmpp2m_step(_shared(16), _h(16), None, _shared(16), 1.0, 1, 0, 1, 0, 0),
    "x0_prev is v_neg": lambda o: o.dpmpp2m_step(_h(16), _shared(16), None, _shared(16), 1.0, 1, 0, 1, 0, 0),
    "x0_prev is out": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _shared(16), 1.0, 1, 0, 1, 0, 0, out=_shared(16)),
    "x0_prev overlaps v_edit": lambda o: o.dpmpp2m_step(_h(16), _h(16), _shared(32)[:16], _shared(32)[8:24], 1.0, 1, 0, 1, 0, 0),
    "out is v_edit": lambda o: o.dpmpp2m_step(_h(16), _h(16), _shared(16), _h(16), 1.0, 1, 0, 1, 0, 0, out=_shared(16)),
    "coef_dev dtype": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0, coef_dev=_h(6)),
    "coef_dev length": lambda o: o.dpmpp2m_step(_h(16), _h(16), None, _h(16), 1.0, 1, 0, 1, 0, 0,
                                                coef_dev=_h(5, dtype=torch.float32)),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_dpm_wrapper_refusals(case):
    from anyv2v_b200 import ops
    from anyv2v_b200._lib import Av2vError
    n0 = ops.launch_count()
    with pytest.raises(Av2vError):
        REFUSALS[case](ops)
    assert ops.launch_count() == n0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- full size
@pytest.fixture(scope="module")
def full():
    from oracle import unet_ref
    return fw.build_models(dev, unet_ref.I2VGEN_XL_CONFIG)


def _inputs(dtype):
    from oracle import loops_ref
    return loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=1024, seed=8888, dtype=dtype, device=dev)


def _dpm():
    from anyv2v_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler.from_config(DDIMScheduler().config)
    s.set_timesteps(N_STEPS)
    return s


@torch.no_grad()
def test_cuda_graph_call_equals_eager_25_steps(full):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    ns = _inputs(torch.float16)
    pipe = I2VGenXLPipeline(full.ours, _dpm())
    outs = {}
    for graphs in (False, True):
        pipe.use_cuda_graphs = graphs
        outs[graphs] = pipe(prompt_embeds=ns.edit_prompt, negative_prompt_embeds=ns.neg_prompt, image_embeddings=ns.edit_image_emb,
                            image_latents=ns.edit_image_latents, latents=ns.video_latents, num_frames=F_, target_fps=FPS,
                            num_inference_steps=N_STEPS, guidance_scale=GUIDANCE, output_type="latent").frames.clone()
    torch.cuda.synchronize()
    assert torch.isfinite(outs[True]).all() and torch.equal(outs[True], outs[False])


class _Rows:
    def __init__(self, title):
        self.title, self.worst = title, 0.0
        print(f"\n{title}\n{'step':>4} {'t':>4} {'ours rms_rel':>12} {'fp16 rms_rel':>12} {'ratio':>6}")

    def row(self, i, t, e_ours, e_ref):
        ratio = e_ours["rms_rel"] / max(e_ref["rms_rel"], 1e-30)
        self.worst = max(self.worst, ratio)
        print(f"{i:>4} {t:>4} {e_ours['rms_rel']:>12.3e} {e_ref['rms_rel']:>12.3e} {ratio:>6.2f}")


@torch.no_grad()
def test_teacher_forced_call_against_the_fp32_oracle(full):
    """each of the 24 steps of a 25-step `__call__` (graph path) from the oracle's x_i, against the fp32 oracle's DPM-Solver++
    step, with our error at most 3 x torch-fp16's (tests/test_gpu_schedule_parity.py's criterion); the fp16 oracle keeps its own
    x0 history along the same teacher inputs"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from oracle.schedulers_ref import cfg_combine
    fw._register(full, [], -1)
    ns32, ns16 = _inputs(torch.float32), _inputs(torch.float16)
    cond = lambda ns: (torch.cat([ns.neg_prompt, ns.edit_prompt]), torch.cat([ns.edit_image_latents] * 2),
                       torch.cat([torch.zeros_like(ns.edit_image_emb), ns.edit_image_emb]), ns.fps.repeat(2))
    p32, l32, e32, f32 = cond(ns32)
    p16, l16, e16, f16 = cond(ns16)
    r32, r16 = dpm_solver_ref.DPMRef(), dpm_solver_ref.DPMRef()
    r32.set_timesteps(N_STEPS)
    r16.set_timesteps(N_STEPS)
    ts = [int(t) for t in r32.timesteps[1:]]
    traj = [ns32.video_latents]
    for t in ts:
        x = traj[-1]
        v = full.ref32(torch.cat([x, x]), torch.tensor([t], device=dev), f32, l32, e32, p32)[0]
        traj.append(r32.step(cfg_combine(v[0:1], v[1:2], GUIDANCE), t, x)[0])
    pipe = I2VGenXLPipeline(full.ours, _dpm())
    pipe.use_cuda_graphs = True
    st = pipe.prepare_call(ns16.video_latents, ns16.edit_prompt, ns16.edit_image_latents, ns16.edit_image_emb, FPS, N_STEPS,
                           GUIDANCE, ns16.neg_prompt)
    assert st.timesteps == ts
    table = _Rows(f"teacher-forced 25-step DPM-Solver++ __call__, {F_} x {H_}x{W_}, CUDA graphs on")
    for i, t in enumerate(ts):
        x = traj[i]
        st.latents.copy_(x.half())
        got = pipe.call_step(st, i).clone()
        v16 = full.ref16(torch.cat([x.half()] * 2), torch.tensor([t], device=dev), f16, l16, e16, p16)[0]
        want16, _ = r16.step(cfg_combine(v16[0:1], v16[1:2], GUIDANCE), t, x.half())
        e_ours, e_ref = fw._check(got, traj[i + 1], want16, f"call step {i} t={t}")
        table.row(i, t, e_ours, e_ref)
    print(f"worst ratio ours / torch-fp16 = {table.worst:.2f}")
    assert len(st.iterations) == 1


@torch.no_grad()
def test_teacher_forced_pnp_edit_against_the_fp32_oracle(full):
    """a 25-step config-3 PnP edit reading the fp32 oracle's 50-step inversion, step by step against the oracle edit loop
    (oracle/loops_ref.pnp_edit_loop with the DPM-Solver++ step), criterion as above"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from oracle import loops_ref, pnp_hooks_ref
    from oracle.schedulers_ref import cfg_combine
    fw._register(full, [], -1)
    ns32, ns16 = _inputs(torch.float32), _inputs(torch.float16)
    inv = loops_ref.invert_loop(full.ref32, ns32.video_latents, ns32.inv_prompt, ns32.src_image_latents, ns32.src_image_emb,
                                ns32.fps, INV_STEPS)
    r32, r16 = dpm_solver_ref.DPMRef(), dpm_solver_ref.DPMRef()
    r32.set_timesteps(N_STEPS)
    r16.set_timesteps(N_STEPS)
    for net, sref in ((full.ref32, r32), (full.ref16, r16)):
        pnp_hooks_ref.init_pnp(SimpleNamespace(unet=net), sref, N_STEPS, PNP.pnp_f_t, PNP.pnp_spatial_attn_t, PNP.pnp_temp_attn_t)
    ts = [int(t) for t in r32.timesteps[1:]]
    traj = [inv[ts[0]].clone()]
    loops_ref.pnp_edit_loop(SimpleNamespace(unet=full.ref32), pnp_hooks_ref.register_time, inv, traj[0].clone(),
                            *loops_ref.edit_conditioning(ns32), N_STEPS, GUIDANCE, t_idx=1, scheduler=r32,
                            callback=lambda i, t, x: traj.append(x.clone()))
    assert len(traj) == len(ts) + 1
    store = LatentStore(None, write_files=False)
    for t, x in inv.items():
        store.put(t, x.half())
    sched = _dpm()
    pipe = I2VGenXLPipeline(full.ours, sched)
    init_pnp(pipe, sched, SimpleNamespace(n_steps=N_STEPS, **vars(PNP)))
    pipe.use_cuda_graphs = True
    st = pipe.prepare_edit(traj[0].half(), ns16.edit_prompt, ns16.neg_prompt, ns16.inv_prompt, ns16.edit_image_emb,
                           ns16.edit_image_latents, ns16.src_image_emb, ns16.src_image_latents, FPS, N_STEPS, GUIDANCE, 1, None,
                           store, True)
    assert st.timesteps == ts
    prompts16, img_lat16, img_emb16, fps16 = loops_ref.edit_conditioning(ns16)
    r16.set_timesteps(N_STEPS)
    table = _Rows(f"teacher-forced 25-step DPM-Solver++ PnP edit (config 3, 50-step inversion), {F_} x {H_}x{W_}")
    for i, t in enumerate(ts):
        x = traj[i].half()
        st.latents.copy_(x)
        got = pipe.edit_step(st, i).clone()
        pnp_hooks_ref.register_time(SimpleNamespace(unet=full.ref16), t)
        v16 = full.ref16(torch.cat([inv[t].half(), x, x]), torch.tensor([t], device=dev), fps16, img_lat16, img_emb16, prompts16)[0]
        want16, _ = r16.step(cfg_combine(v16[1:2], v16[2:3], GUIDANCE), t, x)
        e_ours, e_ref = fw._check(got, traj[i + 1], want16, f"edit step {i} t={t}")
        table.row(i, t, e_ours, e_ref)
    print(f"worst ratio ours / torch-fp16 = {table.worst:.2f}")
    fw._register(full, [], -1)


@torch.no_grad()
def test_ddim_edit_is_unchanged_by_a_dpm_edit_before_it():
    """on the tiny UNet with CUDA graphs: DDIM edit, DPM edit, DDIM edit again -> the two DDIM edits are bit-identical"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import loops_ref, unet_ref
    ours = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    ours.load_state_dict(unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device="cpu").state_dict())
    ours = ours.to(device=dev, dtype=torch.float16).eval()
    ns = loops_ref.synthetic_inputs(4, 16, 16, cross_dim=64, dtype=torch.float16, device=dev)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(5)
    for t in range(1, 1000, 100):   # a 10-step inversion's timesteps
        store.put(t, torch.randn(1, 4, 4, 16, 16, generator=g).half().to(dev))
    pipe = I2VGenXLPipeline(ours)
    pipe.use_cuda_graphs = True

    def edit(sched, n):
        sched.set_timesteps(n)
        pipe.scheduler = sched
        init_pnp(pipe, sched, SimpleNamespace(n_steps=n, pnp_f_t=0.6, pnp_spatial_attn_t=0.4, pnp_temp_attn_t=0.4))
        return pipe.sample_with_pnp(latents=ns.video_latents.clone(), prompt_embeds=ns.edit_prompt,
                                    negative_prompt_embeds=ns.neg_prompt, ddim_inv_prompt_embeds=ns.inv_prompt,
                                    image_embeddings=ns.edit_image_emb, image_latents=ns.edit_image_latents,
                                    ddim_inv_image_embeddings=ns.src_image_emb, ddim_inv_image_latents=ns.src_image_latents,
                                    target_fps=8, num_inference_steps=n, guidance_scale=9.0, latent_store=store,
                                    return_dict=False)[0].clone()
    alone = edit(DDIMScheduler(), 10)
    dpm = edit(DPMSolverMultistepScheduler(), 5)
    again = edit(DDIMScheduler(), 10)
    torch.cuda.synchronize()
    assert torch.isfinite(dpm).all() and not torch.equal(dpm, alone)
    assert torch.equal(alone, again)
