"""FreeU (diffusers `enable_freeu`, pipeline_i2vgen_xl.py:623-650) without a GPU: the closed form of the kernel contract
against the oracle's torch.fft `fourier_filter` (both in tests/freeu_ref.py), and the product UNet / loops with FreeU on top of
the kernel contracts against the oracle UNet with FreeU."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import pytest
import torch

import freeu_ref
from test_host_model_cpu import F_, H_, W_, _close, _inputs, _models

FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)  # the values FreeU's authors give for Stable Diffusion 1.x
SIZES = (1, 2, 3, 5, 8, 9, 16, 18)


@pytest.fixture
def emu(emulated_ops, monkeypatch):
    """the kernel contracts in place of anyv2v_b200.ops, ops.freeu included"""
    freeu_ref.patch_ops(monkeypatch)
    return emulated_ops


@pytest.mark.parametrize("s", [0.2, 0.9, 1.0, 1.4])
def test_closed_form_equals_the_fft_fourier_filter_in_float64(s):
    torch.manual_seed(0)
    s32 = float(torch.tensor(s, dtype=torch.float32))  # the oracle's mask is float32, the kernel takes an fp32 scale
    for H in SIZES:
        for W in SIZES:
            x = torch.randn(2, H, W, 8, dtype=torch.float64)
            ref = freeu_ref.fourier_filter(x.permute(0, 3, 1, 2), threshold=1, scale=s).permute(0, 2, 3, 1)
            got = freeu_ref.fourier_filter_closed_form(x, s32)
            err = float((got - ref).abs().max())
            assert err <= 1e-12, (H, W, s, err)


def test_contract_rounds_once_and_scales_the_backbone_half_bit_exactly():
    torch.manual_seed(1)
    hidden = (torch.randn(2, 5, 7, 72) * 30).half()  # Ch / 2 = 36: the boundary splits a 16-byte vector
    skip = torch.randn(2, 5, 7, 40).half()
    h0 = hidden.clone()
    out = freeu_ref.freeu(hidden, skip, 1.37, 0.6)
    want = (h0[..., :36].float() * torch.tensor(1.37, dtype=torch.float32)).half()
    assert torch.equal(hidden[..., :36], want)
    assert torch.equal(hidden[..., 36:].view(torch.int16), h0[..., 36:].view(torch.int16))
    s32 = float(torch.tensor(0.6, dtype=torch.float32))
    assert torch.equal(out, freeu_ref.fourier_filter_closed_form(skip.double(), s32).half())


def _hooks(pipe, hooks, schedule, t):
    hooks.register_conv_injection(pipe, schedule)
    hooks.register_spatial_attention_pnp(pipe, schedule)
    hooks.register_temp_attention_pnp(pipe, schedule)
    hooks.register_time(pipe, t)


@torch.no_grad()
@pytest.mark.parametrize("t,expect_inject", [(901, True), (101, False)])
def test_product_unet_with_freeu_and_hooks_matches_the_oracle(emu, t, expect_inject):
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import pnp_hooks_ref, schedulers_ref
    ref32, ours = _models()
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    outs = {}
    for name, net, dt, hooks, freeu in (("ref_off", ref32, torch.float32, pnp_hooks_ref, False),
                                        ("ref", ref32, torch.float32, pnp_hooks_ref, True),
                                        ("ours", ours, torch.float16, ours_hooks, True)):
        _hooks(SimpleNamespace(unet=net), hooks, s.timesteps[:5], t)
        if net is ours:
            ours.enable_freeu(**FREEU)
        elif freeu:
            freeu_ref.enable_freeu(ref32, **FREEU)
        _, x3, prompts, img_lat, img_emb, fps = _inputs(dt)
        outs[name] = net(x3, torch.tensor([t]), fps, img_lat, img_emb, prompts)[0]
    _close(outs["ours"], outs["ref"], f"hooked UNet with FreeU t={t}")
    assert ours.up_blocks[2].attentions[1].transformer_blocks[0].attn1.processor.inject_now() == expect_inject
    change = (outs["ref"] - outs["ref_off"]).pow(2).mean().sqrt() / outs["ref"].pow(2).mean().sqrt()
    assert change > 0.05, f"FreeU barely changes the oracle (rms rel {float(change):.2e}): the comparison would prove nothing"


@torch.no_grad()
def test_product_unet_with_freeu_for_every_batch_size(emu):
    ref32, ours = _models()
    freeu_ref.enable_freeu(ref32, **FREEU)
    ours.enable_freeu(**FREEU)
    for b in (1, 2, 3):
        _, x3, prompts, img_lat, img_emb, fps = _inputs(torch.float32)
        ref = ref32(x3[:b], torch.tensor([501]), fps[:b], img_lat[:b], img_emb[:b], prompts[:b])[0]
        _, x3h, prompts, img_lat, img_emb, fps = _inputs(torch.float16)
        got = ours(x3h[:b], torch.tensor([501]), fps[:b], img_lat[:b], img_emb[:b], prompts[:b])[0]
        _close(got, ref, f"UNet forward with FreeU B={b}")


@torch.no_grad()
@pytest.mark.parametrize("fracs,site", [((1.0, 0.0, 0.0), (1, 1, "resnet")), ((1.0, 1.0, 1.0), (3, 2, "temporal"))])
def test_freeu_under_source_pruning_and_shared_prefix_is_bit_identical(emu, fracs, site):
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import schedulers_ref
    _, ours = _models()
    ours.enable_freeu(**FREEU)
    pipe = SimpleNamespace(unet=ours)
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    ours_hooks.register_conv_injection(pipe, s.timesteps if fracs[0] else [])
    ours_hooks.register_spatial_attention_pnp(pipe, s.timesteps if fracs[1] else [])
    ours_hooks.register_temp_attention_pnp(pipe, s.timesteps if fracs[2] else [])
    t = int(s.timesteps[2])
    ours_hooks.register_time(pipe, t)
    _, x3, prompts, img_lat, img_emb, fps = _inputs(torch.float16)
    x3 = torch.cat([x3[:2], x3[1:2]])                 # [source, x, x] as in the edit loop
    img_lat = torch.cat([img_lat[:2], img_lat[1:2]])
    args = (x3, torch.tensor([t]), fps, img_lat, img_emb, prompts)
    full = ours(*args)[0]
    assert torch.equal(ours(*args, prune_source_after=site)[0], full[1:])
    assert torch.equal(ours(*args, shared_edit_prefix=True)[0], full)
    assert torch.equal(ours(*args, shared_edit_prefix=True, prune_source_after=site)[0], full[1:])


@torch.no_grad()
def test_disable_freeu_and_zero_factors_restore_the_plain_forward_and_its_launches(emu):
    _, ours = _models()
    _, never = _models()
    _, x3, prompts, img_lat, img_emb, fps = _inputs(torch.float16)
    args = (x3, torch.tensor([501]), fps, img_lat, img_emb, prompts)

    def run(net):
        n0 = emu.launch_count()
        y = net(*args)[0]
        return y, emu.launch_count() - n0

    plain, n_plain = run(never)
    ours.enable_freeu(**FREEU)
    on, n_on = run(ours)
    assert n_on == n_plain + 6                        # 3 skip connections in each of up_blocks[0] and [1]
    assert not torch.equal(on, plain)
    ours.disable_freeu()
    off, n_off = run(ours)
    assert torch.equal(off, plain) and n_off == n_plain
    assert all(blk.freeu_factors() is None for blk in ours.up_blocks) and ours.freeu_state() == (None,) * 4
    for zero in ("s1", "s2", "b1", "b2"):             # diffusers tests the four values for truthiness
        ours.enable_freeu(**dict(FREEU, **{zero: 0.0}))
        y, n = run(ours)
        assert torch.equal(y, plain) and n == n_plain, zero


@torch.no_grad()
def test_both_loops_with_freeu_teacher_forced(emu, tmp_path):
    """pipeline.invert + sample_with_pnp with FreeU enabled through the pipeline, against oracle/loops_ref.py with the oracle's
    FreeU, teacher-forced per step"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle import loops_ref, pnp_hooks_ref, schedulers_ref
    ref32, ours = _models()
    freeu_ref.enable_freeu(ref32, **FREEU)
    n_steps = 4
    ns32 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float32, device="cpu")
    ns16 = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    pipe = I2VGenXLPipeline(ours, DDIMInverseScheduler())
    pipe.enable_freeu(**FREEU)
    assert ours.up_blocks[3].b1 == FREEU["b1"] and ours.freeu_state()[:2] == ((1.5, 0.9), (1.6, 0.2))
    seen_inv = []
    pipe.invert(latents=ns16.video_latents, prompt_embeds=ns16.inv_prompt, image_latents=ns16.src_image_latents,
                image_embeddings=ns16.src_image_emb, target_fps=8, num_inference_steps=n_steps, guidance_scale=1.0,
                output_dir=str(tmp_path / "ddim_latents"), callback=lambda i, t, x: seen_inv.append((t, x.clone())))
    inv_s = schedulers_ref.DDIMInverseScheduler()
    inv_s.set_timesteps(n_steps)
    x_prev = ns32.video_latents
    for t, x_ours in seen_inv:
        v = ref32(x_prev, torch.tensor(t), ns32.fps, ns32.src_image_latents, ns32.src_image_emb, ns32.inv_prompt)[0]
        x_ref, _ = inv_s.step(v, t, x_prev)
        _close(x_ours, x_ref, f"inversion step t={t} with FreeU", rms=3e-3, mx=1e-2)
        x_prev = x_ours.float()
    store = pipe.latent_store

    cfg = SimpleNamespace(n_steps=n_steps, pnp_f_t=0.5, pnp_spatial_attn_t=0.25, pnp_temp_attn_t=0.25)
    edit_sched = DDIMScheduler()
    edit_sched.set_timesteps(n_steps)
    pipe.scheduler = edit_sched
    init_pnp(pipe, edit_sched, cfg)
    seen = []
    pipe.sample_with_pnp(latents=ns16.video_latents.clone(), prompt_embeds=ns16.edit_prompt, negative_prompt_embeds=ns16.neg_prompt,
                         ddim_inv_prompt_embeds=ns16.inv_prompt, image_embeddings=ns16.edit_image_emb,
                         image_latents=ns16.edit_image_latents, ddim_inv_image_embeddings=ns16.src_image_emb,
                         ddim_inv_image_latents=ns16.src_image_latents, target_fps=8, num_inference_steps=n_steps,
                         guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store,
                         callback=lambda i, t, x: seen.append((t, x.clone())), return_dict=False)
    assert len(seen) == n_steps
    sref = schedulers_ref.DDIMScheduler()
    sref.set_timesteps(n_steps)
    rp = SimpleNamespace(unet=ref32)
    pnp_hooks_ref.init_pnp(rp, sref, n_steps, pnp_f_t=0.5, pnp_spatial_attn_t=0.25, pnp_temp_attn_t=0.25)
    prompts, img_lat, img_emb, fps3 = loops_ref.edit_conditioning(ns32)
    x_prev = ns16.video_latents.float()
    for t, x_ours in seen:
        pnp_hooks_ref.register_time(rp, t)
        src = store.get(t, device="cpu").float()
        v = ref32(torch.cat([src, x_prev, x_prev]), torch.tensor(t), fps3, img_lat, img_emb, prompts)[0]
        x_ref, _ = sref.step(schedulers_ref.cfg_combine(v[1:2], v[2:3], 9.0), t, x_prev)
        _close(x_ours, x_ref, f"edit step t={t} with FreeU", rms=6e-3, mx=3e-2)
        x_prev = x_ours.float()


def test_pipeline_freeu_surface():
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    with pytest.raises(ValueError, match="unet"):
        I2VGenXLPipeline(unet=None).enable_freeu(0.9, 0.2, 1.5, 1.6)


def test_freeu_args_struct_matches_the_c_header(tmp_path):
    """ctypes mirror of av2v_freeu_args against the layout gcc gives include/anyv2v_b200.h"""
    from anyv2v_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cls = _lib.FreeUArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "anyv2v_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(av2v_freeu_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(av2v_freeu_args, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


def test_freeu_abi_rejects_bad_arguments_before_any_cuda_call():
    import __graft_entry__ as g
    g.build()
    from anyv2v_b200 import _lib
    lib = _lib.lib()
    ok = dict(hidden=16, skip=32, out=48, NF=2, H=4, W=4, Ch=64, Cs=64, b=1.5, s=0.9)
    for bad, code in ((dict(Cs=12), _lib.AV2V_EINVAL), (dict(Ch=9), _lib.AV2V_EINVAL), (dict(H=0), _lib.AV2V_EINVAL),
                      (dict(skip=None), _lib.AV2V_EINVAL), (dict(out=40), _lib.AV2V_EALIGN)):
        a = _lib.FreeUArgs(**dict(ok, **bad))
        assert lib.av2v_freeu_f16(ctypes.byref(a), None) == code, bad
    empty = _lib.FreeUArgs(**dict(ok, NF=0))
    assert lib.av2v_freeu_f16(ctypes.byref(empty), None) == _lib.AV2V_OK
