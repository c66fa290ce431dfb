"""Every step of the 50-step inversion and the 50-step PnP edit at the measured geometry (16 frames x 64 x 64 latents =
512 x 512 video, the full I2VGEN_XL_CONFIG), through the product pipeline with CUDA graphs on, against the fp32 oracle.

A per-kernel contract audit (tests/test_gpu_step_audit.py) shows that each kernel computed what its arguments asked for;
only the model output against the oracle shows that the host asked the right questions at every step: the source latent
of step i, the hook flags baked into each of the three replayed edit graphs (conv + spatial + temporal on steps 0-24,
conv only on 25-39, nothing on 40-49 with the dead source branch dropped), the source branch pruned after the right
site, the timestep fed to a replayed graph.  At this geometry the UNet also runs the 48-frame GroupNorm chunking, the
fused temporal attention with F = 16 and the 4096-token spatial attention inside the whole model.

Criterion per step (test_gpu_fullwidth._check): ours-vs-fp32 <= 3 x torch-fp16-vs-fp32 in rms_rel and in rel_to_max,
where torch-fp16 is the oracle run in fp16 from the same inputs.  tests/test_schedule_parity_cpu.py re-runs these
functions on CPU with the tiny config and a shorter schedule, and shows with injected wiring faults that the criterion
fails at the first affected step."""
import time
from types import SimpleNamespace

import pytest
import torch

import test_gpu_fullwidth as fw
from parity_utils import err_stats

pytestmark = pytest.mark.gpu
dev = "cuda"
F_, H_, W_ = 16, 64, 64
N_STEPS = 50
#: None = the full-size I2VGEN_XL_CONFIG; tests/test_schedule_parity_cpu.py sets the tiny config, a smaller geometry and a
#: shorter schedule
CONFIG_OVERRIDE = None
#: BASELINE config 3: conv injection on the first 80 % of the steps, spatial and temporal attention on the first 50 %
PNP = SimpleNamespace(pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)
GUIDANCE = 9.0
FPS = 8


def _config():
    from oracle import unet_ref
    return CONFIG_OVERRIDE or unet_ref.I2VGEN_XL_CONFIG


def _n_conv():
    return int(N_STEPS * PNP.pnp_f_t)


def _n_attn():
    return int(N_STEPS * PNP.pnp_spatial_attn_t)


def expected_flags(i):
    """(conv, spatial, temporal) injection flags of edit step i under PNP"""
    return (i < _n_conv(), i < _n_attn(), i < int(N_STEPS * PNP.pnp_temp_attn_t))


def flag_change_steps():
    """first and last step of each flag set: 0, 24, 25, 39, 40, 49 for 50 steps"""
    return (0, _n_attn() - 1, _n_attn(), _n_conv() - 1, _n_conv(), N_STEPS - 1)


def _flag_str(flags):
    return "".join("T" if f else "F" for f in flags)


class _Table:
    """per-step table: step, t, flags, ours rms_rel, torch-fp16 rms_rel (both against the fp32 oracle), ratio"""

    def __init__(self, title):
        self.title, self.worst = title, 0.0
        print(f"\n{title}\n{'step':>4} {'t':>4} {'flags':>5} {'ours rms_rel':>12} {'fp16 rms_rel':>12} {'ratio':>6}")

    def row(self, step, t, flags, e_ours, e_ref):
        ratio = e_ours["rms_rel"] / max(e_ref["rms_rel"], 1e-30)
        self.worst = max(self.worst, ratio)
        print(f"{step:>4} {t:>4} {flags:>5} {e_ours['rms_rel']:>12.3e} {e_ref['rms_rel']:>12.3e} {ratio:>6.2f}")

    def done(self):
        print(f"{self.title}: worst ratio ours / torch-fp16 = {self.worst:.2f}")
        if torch.cuda.is_available() and dev == "cuda":
            print(f"peak memory allocated so far: {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


def _check_step(table, got, want32, want16, what, step, t, flags):
    e_ours, e_ref = fw._check(got, want32, want16, what)
    table.row(step, t, flags, e_ours, e_ref)


def _inputs(dtype):
    from oracle import loops_ref
    return loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=_config()["cross_attention_dim"], seed=8888, dtype=dtype, device=dev)


def _hook_oracle(net):
    """config-3 PnP hooks on an oracle model (the reference's init_pnp); -> its DDIM scheduler"""
    from oracle import pnp_hooks_ref, schedulers_ref
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(N_STEPS)
    pnp_hooks_ref.init_pnp(SimpleNamespace(unet=net), sref, N_STEPS, PNP.pnp_f_t, PNP.pnp_spatial_attn_t, PNP.pnp_temp_attn_t)
    return sref


def _edit_pipeline(full):
    """the product pipeline with the config-3 hooks registered on our UNet (run_group_pnp_edit.init_pnp)"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    sch = DDIMScheduler()
    sch.set_timesteps(N_STEPS)
    pipe = I2VGenXLPipeline(full.ours, sch)
    init_pnp(pipe, sch, SimpleNamespace(n_steps=N_STEPS, **vars(PNP)))
    return pipe


@torch.no_grad()
def build_oracle(full):
    """The fp32 oracle's trajectories, computed once: the 50-step inversion (x_0 = the video latents, x_{i+1} = the
    latent saved at the i-th inversion timestep) and the 50-step edit from its own x_T with its own inverted latents."""
    from oracle import loops_ref, pnp_hooks_ref
    ns32, ns16 = _inputs(torch.float32), _inputs(torch.float16)
    fw._register(full, [], -1)
    t0 = time.perf_counter()
    inv = loops_ref.invert_loop(full.ref32, ns32.video_latents, ns32.inv_prompt, ns32.src_image_latents, ns32.src_image_emb,
                                ns32.fps, N_STEPS)
    t1 = time.perf_counter()
    inv_ts = sorted(inv)                                        # inversion order: 1, 21, ..., 981
    sref = _hook_oracle(full.ref32)
    edit_ts = [int(t) for t in sref.timesteps]                  # 981, 961, ..., 1
    edit_traj = [inv[inv_ts[-1]].clone()]
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns32)
    loops_ref.pnp_edit_loop(SimpleNamespace(unet=full.ref32), pnp_hooks_ref.register_time, inv, edit_traj[0].clone(), prompts,
                            img_lat, img_emb, fps, N_STEPS, GUIDANCE, scheduler=sref,
                            callback=lambda i, t, x: edit_traj.append(x.clone()))
    t2 = time.perf_counter()
    fw._register(full, [], -1)
    print(f"\nfp32 oracle: {N_STEPS}-step inversion {t1 - t0:.1f} s, {N_STEPS}-step edit {t2 - t1:.1f} s")
    return SimpleNamespace(ns32=ns32, ns16=ns16, inv=inv, inv_ts=inv_ts, inv_traj=[ns32.video_latents] + [inv[t] for t in inv_ts],
                           edit_ts=edit_ts, edit_traj=edit_traj)


@pytest.fixture(scope="module")
def full():
    torch.cuda.reset_peak_memory_stats()
    return fw.build_models(dev, _config())


@pytest.fixture(scope="module")
def orc(full):
    return build_oracle(full)


@torch.no_grad()
def test_teacher_forced_inversion_every_step_graphed(full, orc):
    """(a) each of our 50 inversion steps (UNet B = 1 + fused inverse DDIM, graph path) from the oracle's x_i against the
    oracle's x_{i+1}; steps 2..49 are replays of the one graph captured at step 1"""
    from anyv2v_b200 import ops
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMInverseScheduler
    from oracle import schedulers_ref
    fw._register(full, [], -1)
    ns16 = orc.ns16
    inv_ref = schedulers_ref.DDIMInverseScheduler()
    inv_ref.set_timesteps(N_STEPS)
    pipe = I2VGenXLPipeline(full.ours, DDIMInverseScheduler())
    pipe.use_cuda_graphs = True
    st = pipe.prepare_invert(ns16.video_latents, ns16.inv_prompt, ns16.src_image_latents, ns16.src_image_emb, FPS, N_STEPS,
                             1.0, None, False, False)
    assert st.timesteps == orc.inv_ts
    table = _Table(f"teacher-forced inversion, {F_} x {H_}x{W_}, CUDA graphs on")
    launches = []
    for i, t in enumerate(st.timesteps):
        x = orc.inv_traj[i]
        st.latents.copy_(x.half())
        got = pipe.invert_step(st, i).clone()
        launches.append(ops.launch_count())
        v16 = full.ref16(x.half(), torch.tensor([t], device=dev), ns16.fps, ns16.src_image_latents, ns16.src_image_emb,
                         ns16.inv_prompt)[0]
        want16, _ = inv_ref.step(v16, t, x.half())
        _check_step(table, got, orc.inv_traj[i + 1], want16, f"inversion step {i} t={t}", i, t, "-")
    table.done()
    assert len(st.iterations) == 1
    if st.latents.is_cuda:
        it = next(iter(st.iterations.values()))
        assert it.graph is not None and it.calls == N_STEPS
        assert launches[1] > launches[0] and launches[-1] == launches[1], launches  # steps 2.. launch nothing: replays


def teacher_forced_edit(full, orc, pipe, steps, graphs):
    """our edit steps ``steps`` (in order), each from the oracle's x_i and the oracle's inverted latents (cast to fp16, as
    our inversion stores them) -> (state, {i: SimpleNamespace(x=x_{i+1}, flags, launches)})"""
    from anyv2v_b200 import ops
    from anyv2v_b200.latent_store import LatentStore
    ns16 = orc.ns16
    store = LatentStore(None, write_files=False)
    for t, x in orc.inv.items():
        store.put(t, x.half())
    pipe.use_cuda_graphs = graphs
    st = pipe.prepare_edit(orc.edit_traj[0].half(), ns16.edit_prompt, ns16.neg_prompt, ns16.inv_prompt, ns16.edit_image_emb,
                           ns16.edit_image_latents, ns16.src_image_emb, ns16.src_image_latents, FPS, N_STEPS, GUIDANCE, 0, None,
                           store, True)
    assert st.timesteps == orc.edit_ts
    out = {}
    for i in steps:
        st.latents.copy_(orc.edit_traj[i].half())
        got = pipe.edit_step(st, i).clone()
        out[i] = SimpleNamespace(x=got, flags=pipe._hook_flags(st.timesteps[i]), launches=ops.launch_count())
    return st, out


@torch.no_grad()
def test_teacher_forced_pnp_edit_every_step_graphed(full, orc):
    """(b) each of our 50 PnP edit steps (graph path: pruned-source batch on steps 0-39, two-branch dead-source batch on
    40-49) from the oracle's x_i and source latent against the oracle's three-branch step"""
    from anyv2v_b200 import ops
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    pipe = _edit_pipeline(full)
    sref = _hook_oracle(full.ref16)
    c0 = ops.launch_count()
    st, out = teacher_forced_edit(full, orc, pipe, range(N_STEPS), graphs=True)
    prompts16, img_lat16, img_emb16, fps16 = loops_ref.edit_conditioning(orc.ns16)
    table = _Table(f"teacher-forced PnP edit (config 3), {F_} x {H_}x{W_}, CUDA graphs on")
    for i, t in enumerate(orc.edit_ts):
        x = orc.edit_traj[i].half()
        pnp_hooks_ref.register_time(SimpleNamespace(unet=full.ref16), t)
        v16 = full.ref16(torch.cat([orc.inv[t].half(), x, x]), torch.tensor([t], device=dev), fps16, img_lat16, img_emb16,
                         prompts16)[0]
        want16, _ = sref.step(schedulers_ref.cfg_combine(v16[1:2], v16[2:3], GUIDANCE), t, x)
        flags = out[i].flags
        _check_step(table, out[i].x, orc.edit_traj[i + 1], want16, f"edit step {i} t={t} flags={flags}", i, t, _flag_str(flags))
        assert flags == expected_flags(i), (f"hook flags at edit step {i}", flags)
    table.done()
    fs = full.ours.freeu_state()
    assert set(st.iterations) == {(False, (True, True, True), fs), (False, (True, False, False), fs), (True, (False,) * 3, fs)}
    if st.latents.is_cuda:
        assert all(it.graph is not None for it in st.iterations.values())
        # each flag set runs eagerly on its first step and is captured on its second; every other step is a replay
        counts = [c0] + [out[i].launches for i in range(N_STEPS)]
        grew = [i for i in range(N_STEPS) if counts[i + 1] > counts[i]]
        n_attn, n_conv = _n_attn(), _n_conv()
        assert grew == [0, 1, n_attn, n_attn + 1, n_conv, n_conv + 1], grew
    fw._register(full, [], -1)


@torch.no_grad()
def test_graph_replay_equals_eager_at_flag_changes(full, orc):
    """(c) at the first and last step of each flag set, a replayed (or captured) graph gives bit for bit what a fresh
    eager state gives from the same teacher inputs"""
    pipe = _edit_pipeline(full)
    _, graphed = teacher_forced_edit(full, orc, pipe, range(N_STEPS), graphs=True)
    steps = flag_change_steps()
    _, eager = teacher_forced_edit(full, orc, pipe, steps, graphs=False)
    print(f"\ngraph replay vs eager, {F_} x {H_}x{W_}\n{'step':>4} {'t':>4} {'flags':>5} {'max |graph - eager|':>20}")
    for i in steps:
        d = float((graphed[i].x.float() - eager[i].x.float()).abs().max())
        print(f"{i:>4} {orc.edit_ts[i]:>4} {_flag_str(eager[i].flags):>5} {d:>20.3e}")
        assert eager[i].flags == graphed[i].flags == expected_flags(i)
        assert torch.equal(graphed[i].x, eager[i].x), (f"edit step {i}", d)
    fw._register(full, [], -1)


@torch.no_grad()
def test_free_running_inversion_and_edit(full, orc):
    """(d) pipe.invert + pipe.sample_with_pnp as a user calls them (50 + 50 steps, graphs on), against the fp32 oracle's
    trajectories and a free-running torch-fp16 oracle: a regression check relative to torch, since a random-init UNet
    amplifies fp16 rounding over 100 steps"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle import loops_ref, pnp_hooks_ref
    ns16 = orc.ns16
    fw._register(full, [], -1)
    inv16 = loops_ref.invert_loop(full.ref16, ns16.video_latents, ns16.inv_prompt, ns16.src_image_latents, ns16.src_image_emb,
                                  ns16.fps, N_STEPS)
    pipe = I2VGenXLPipeline(full.ours, DDIMInverseScheduler())
    pipe.use_cuda_graphs = True
    pipe.invert(latents=ns16.video_latents, prompt_embeds=ns16.inv_prompt, image_latents=ns16.src_image_latents,
                image_embeddings=ns16.src_image_emb, target_fps=FPS, num_inference_steps=N_STEPS, guidance_scale=1.0,
                write_files=False)
    store = pipe.latent_store
    table = _Table(f"free-running inversion, {F_} x {H_}x{W_}")
    for i, t in enumerate(orc.inv_ts):
        _check_step(table, store.get(t), orc.inv[t], inv16[t], f"free-running inversion t={t}", i, t, "-")
    table.done()
    # edit: the torch-fp16 oracle from its own inversion, ours from ours, both compared with the fp32 oracle's trajectory
    sref16 = _hook_oracle(full.ref16)
    traj16 = []
    loops_ref.pnp_edit_loop(SimpleNamespace(unet=full.ref16), pnp_hooks_ref.register_time, inv16, inv16[orc.inv_ts[-1]].clone(),
                            *loops_ref.edit_conditioning(ns16), N_STEPS, GUIDANCE, scheduler=sref16,
                            callback=lambda i, t, x: traj16.append(x.clone()))
    sch = DDIMScheduler()
    sch.set_timesteps(N_STEPS)
    pipe.register_modules(scheduler=sch)
    init_pnp(pipe, sch, SimpleNamespace(n_steps=N_STEPS, **vars(PNP)))
    ours = []
    final = pipe.sample_with_pnp(latents=store.get(orc.inv_ts[-1]).clone(), prompt_embeds=ns16.edit_prompt,
                                 negative_prompt_embeds=ns16.neg_prompt, ddim_inv_prompt_embeds=ns16.inv_prompt,
                                 image_embeddings=ns16.edit_image_emb, image_latents=ns16.edit_image_latents,
                                 ddim_inv_image_embeddings=ns16.src_image_emb, ddim_inv_image_latents=ns16.src_image_latents,
                                 target_fps=FPS, num_inference_steps=N_STEPS, guidance_scale=GUIDANCE, ddim_init_latents_t_idx=0,
                                 latent_store=store, callback=lambda i, t, x: ours.append(x.clone()), return_dict=False)[0]
    assert len(ours) == len(traj16) == N_STEPS
    table = _Table(f"free-running PnP edit (config 3), {F_} x {H_}x{W_} (reported per step, asserted on the final latents)")
    for i, t in enumerate(orc.edit_ts):
        table.row(i, t, _flag_str(expected_flags(i)), err_stats(ours[i], orc.edit_traj[i + 1]), err_stats(traj16[i], orc.edit_traj[i + 1]))
    table.done()
    e_ours, e16 = fw._check(final, orc.edit_traj[-1], traj16[-1], f"free-running edit, final latents after {N_STEPS} + {N_STEPS} steps")
    if e16["rms_rel"] > 0.3:
        print(f"note: torch-fp16's own final drift is {e16['rms_rel']:.3f} rms_rel: the random-init UNet amplifies fp16 rounding; "
              "the teacher-forced tests are the parity bar")
    fw._register(full, [], -1)
