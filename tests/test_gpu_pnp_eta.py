"""Stochastic DDIM (eta > 0) in the PnP edit on the GPU: ``ops.ddim_step_eta`` on the UNet-output row views the edit steps
read, at 16 and 128 frames of 512 x 512 and at 704 x 1280; `sample_with_pnp(eta=...)` on the tiny UNet in every step body
against the fp32 oracle (tests/test_pnp_eta_cpu.py); and the full-size UNet at 16 x 512^2 on the BASELINE config-3 injection
schedule with eta = 1 and ``generator=torch.manual_seed(8888)`` (what the reference's runner passes): all 50 steps of the
CUDA-graph loop bit for bit against eager launches, each step against the fp32 oracle with the criterion of
tests/test_gpu_schedule_parity.py, and one edit step under tests/call_audit.py."""
from types import SimpleNamespace

import pytest
import torch

import pnp_eta_ref
import sampling_ref
import test_gpu_fullwidth as fw
from call_audit import CallAudit
from test_gpu_call import _tiny_models
from test_gpu_schedule_parity import _flag_str, _Table, expected_flags
from test_pnp_eta_cpu import run_edit_teacher_forced

pytestmark = pytest.mark.gpu
dev = "cuda"
F_, H_, W_ = 16, 64, 64
N_STEPS = 50
PNP = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)  # BASELINE config 3
GUIDANCE = 9.0
FPS = 8
SEED = 8888


@torch.no_grad()
@pytest.mark.parametrize("F,h,w", [(16, 64, 64), (128, 64, 64), (16, 88, 160)])
@pytest.mark.parametrize("lo", [0, 1])
def test_eta_step_on_unet_output_rows(F, h, w, lo):
    """branches lo / lo + 1 of a [B, 4, F, h, w] UNet output (lo = 0: pruned or dead-source batch, 1: full batch) as v_neg /
    v_edit, in place on the latents, bit for bit against the kernel's contract"""
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(50)
    g = torch.Generator().manual_seed(F + h + lo)
    v = torch.randn(lo + 2, 4, F, h, w, generator=g).half().to(dev)
    x = torch.randn(1, 4, F, h, w, generator=g).half().to(dev)
    z = torch.randn(1, 4, F, h, w, generator=g).half().to(dev)
    coef = s.coefficient_table([981], GUIDANCE, dev, eta=1.0)[0]
    want = sampling_ref.ddim_step_eta(x.cpu(), v[lo:lo + 1].cpu(), v[lo + 1:lo + 2].cpu(), z.cpu(), 0.0, 0, 0, 0, 0, 0,
                                      coef_dev=coef.cpu())
    got = s.step(v[lo:lo + 1], None, x, eta=1.0, model_output_cond=v[lo + 1:lo + 2], out=x, coef_dev=coef, variance_noise=z)
    torch.cuda.synchronize()
    assert got.prev_sample.data_ptr() == x.data_ptr()
    assert torch.equal(x.cpu().view(torch.int16), want.view(torch.int16))


@torch.no_grad()
@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("eta", [0.5, 1.0])
def test_tiny_unet_every_body_matches_the_fp32_oracle(eta, skip):
    ref32, ours = _tiny_models()
    _, st = run_edit_teacher_forced(ref32, ours, eta, skip, dev, rms=1e-2, mx=4e-2)
    assert len(st.iterations) == 4 and all(k[-1] is True for k in st.iterations)


# ------------------------------------------------------------------------------------------------- full size, config 3
def _pipeline(full):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    sch = DDIMScheduler()
    sch.set_timesteps(N_STEPS)
    pipe = I2VGenXLPipeline(full.ours, sch)
    init_pnp(pipe, sch, PNP)
    pipe.disable_freeu()
    return pipe


def _edit(full, run, graphs):
    """sample_with_pnp(eta=1, generator=torch.manual_seed(8888)) over the 50 steps -> (x_0 .. x_50, its loop state, the
    global generator's state after the loop)"""
    pipe = _pipeline(full)
    pipe.use_cuda_graphs = graphs
    states = []
    real = pipe.prepare_edit
    pipe.prepare_edit = lambda *a, **kw: states.append(real(*a, **kw)) or states[-1]
    ns16 = run.ns16
    traj = [run.x_T]
    pipe.sample_with_pnp(latents=run.x_T.clone(), prompt_embeds=ns16.edit_prompt, negative_prompt_embeds=ns16.neg_prompt,
                         ddim_inv_prompt_embeds=ns16.inv_prompt, image_embeddings=ns16.edit_image_emb,
                         image_latents=ns16.edit_image_latents, ddim_inv_image_embeddings=ns16.src_image_emb,
                         ddim_inv_image_latents=ns16.src_image_latents, target_fps=FPS, num_inference_steps=N_STEPS,
                         guidance_scale=GUIDANCE, ddim_init_latents_t_idx=0, latent_store=run.store, eta=1.0,
                         generator=torch.manual_seed(SEED), callback=lambda i, t, x: traj.append(x.clone()))
    torch.cuda.synchronize()
    return traj, states[0], torch.default_generator.get_state()


@pytest.fixture(scope="module")
def full():
    from oracle import unet_ref
    models = fw.build_models(dev, unet_ref.I2VGEN_XL_CONFIG)
    yield models
    fw._register(models, [], -1)
    del models
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def run(full):
    """the inputs (synthetic conditioning, random source latents per timestep) and the CUDA-graph edit from them"""
    from anyv2v_b200.latent_store import LatentStore
    from oracle import loops_ref
    ns16 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=1024, seed=8888, dtype=torch.float16, device=dev)
    ns32 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=1024, seed=8888, dtype=torch.float32, device=dev)
    g = torch.Generator().manual_seed(3)
    store = LatentStore(None, write_files=False)
    r = SimpleNamespace(ns16=ns16, ns32=ns32, store=store, x_T=torch.randn(1, 4, F_, H_, W_, generator=g).half().to(dev))
    sch = _pipeline(full).scheduler
    for t in sch.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, F_, H_, W_, generator=g).half().to(dev))
    with torch.no_grad():
        r.traj, r.st, r.gen_state = _edit(full, r, graphs=True)
    return r


@torch.no_grad()
def test_graph_replay_equals_eager(full, run):
    """every step of the CUDA-graph loop (three graphs: all injections on steps 0-24, conv only on 25-39, the dead-source
    body on 40-49, each captured on its second step) bit for bit against eager launches with the same draws"""
    st = run.st
    fs = full.ours.freeu_state()
    assert set(st.iterations) == {(False, (True, True, True), fs, True), (False, (True, False, False), fs, True),
                                  (True, (False,) * 3, fs, True)}
    assert all(it.graph is not None for it in st.iterations.values())
    eager, st_e, gen_state = _edit(full, run, graphs=False)
    assert all(it.graph is None for it in st_e.iterations.values())
    assert torch.equal(gen_state, run.gen_state)
    print(f"\ngraph replay vs eager, eta = 1, {F_} x {H_}x{W_}\n{'step':>4} {'flags':>5} {'max |graph - eager|':>20}")
    for i in range(N_STEPS):
        d = float((run.traj[i + 1].float() - eager[i + 1].float()).abs().max())
        print(f"{i:>4} {_flag_str(expected_flags(i)):>5} {d:>20.3e}")
    for i in range(N_STEPS):
        assert torch.equal(run.traj[i + 1], eager[i + 1]), f"edit step {i}"
    assert torch.isfinite(run.traj[-1]).all() and not torch.equal(run.traj[-1], run.traj[0])
    fw._register(full, [], -1)


@torch.no_grad()
def test_every_step_against_the_fp32_oracle(full, run):
    """each of the 50 graphed steps, from our x_i and our source latent, against the reference's stochastic step on the
    fp32 oracle; torch-fp16 is the same oracle in fp16 from the same inputs.  Both oracles draw their own noise from a
    generator seeded like ours, so a step also fails if we drew different noise"""
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    ts = run.st.timesteps
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(N_STEPS)
    for net in (full.ref32, full.ref16):
        pnp_hooks_ref.init_pnp(SimpleNamespace(unet=net), sref, N_STEPS, PNP.pnp_f_t, PNP.pnp_spatial_attn_t, PNP.pnp_temp_attn_t)
    cond32, cond16 = loops_ref.edit_conditioning(run.ns32), loops_ref.edit_conditioning(run.ns16)
    g32, g16 = torch.Generator().manual_seed(SEED), torch.Generator().manual_seed(SEED)
    table = _Table(f"teacher-forced PnP edit, eta = 1 (config 3), {F_} x {H_}x{W_}, CUDA graphs on")
    for i, t in enumerate(ts):
        x = run.traj[i]
        src = run.store.get(t, device=dev)
        want32 = pnp_eta_ref.pnp_edit_loop_eta(SimpleNamespace(unet=full.ref32), pnp_hooks_ref.register_time,
                                                {t: src.float()}, x.float(), *cond32, N_STEPS, GUIDANCE, 1.0, generator=g32,
                                                t_idx=i, max_steps=1)
        want16 = pnp_eta_ref.pnp_edit_loop_eta(SimpleNamespace(unet=full.ref16), pnp_hooks_ref.register_time, {t: src},
                                                x, *cond16, N_STEPS, GUIDANCE, 1.0, generator=g16, t_idx=i, max_steps=1)
        e_ours, e_ref = fw._check(run.traj[i + 1], want32, want16, f"eta edit step {i} t={t}")
        table.row(i, t, _flag_str(expected_flags(i)), e_ours, e_ref)
    table.done()
    assert torch.equal(g32.get_state(), run.gen_state) and torch.equal(g16.get_state(), run.gen_state)
    fw._register(full, [], -1)


@torch.no_grad()
def test_audited_eta_edit_step(full, run, monkeypatch):
    """edit step 0 (all three injections, source pruned after the temporal site) with eta = 1, every kernel call against
    its float64 contract and each op's mean error against the bias bound; the eta step kernel at n = 4 x 16 x 64 x 64,
    which tests/test_gpu_bias.py does not run"""
    from anyv2v_b200 import ops
    pipe = _pipeline(full)
    pipe.use_cuda_graphs = False
    ns16 = run.ns16
    st = pipe.prepare_edit(run.x_T.clone(), ns16.edit_prompt, ns16.neg_prompt, ns16.inv_prompt, ns16.edit_image_emb,
                           ns16.edit_image_latents, ns16.src_image_emb, ns16.src_image_latents, FPS, N_STEPS, GUIDANCE, 0, None,
                           run.store, True, 1.0, torch.Generator().manual_seed(SEED))
    audit = CallAudit(seed=11).install(monkeypatch)
    n0 = ops.launch_count()
    pipe.edit_step(st, 0)
    torch.cuda.synchronize()
    launches = ops.launch_count() - n0
    print(f"\neta edit step 0: {len(audit.records)} audited calls, {audit.launches} audited launches\n{audit.table()}")
    bias = audit.bias_by_op()
    for op, (calls, ulp, margin) in audit.families().items():
        print(f"  {op:26s} {calls:5d} calls  worst {ulp:.3g} ulp16  min margin {margin:+.3g}  {bias[op].line()}")
    audit.assert_clean()
    audit.assert_unbiased()
    assert audit.launches == launches > 0
    assert audit.seen("ddim_step_eta", n=4 * F_ * H_ * W_) and not audit.seen("ddim_step")
    # the eta step is checked bit for bit against its contract (which restates the reference's own fp16 roundings), so it
    # has no rounding of its own for the bias bound to weigh: every element is exact
    assert audit.families()["ddim_step_eta"][1] == 0
    fw._register(full, [], -1)
