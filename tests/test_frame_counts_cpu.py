"""Clips of any frame count on CPU: the slot bookkeeping of the frames-mode attention kernels (tools/kernel_models.py) for every
F up to 256, with negative controls, and the product UNet at frame counts that do not divide 128 (F = 3, 24) through the kernel
contracts, against the fp32 oracle."""
from types import SimpleNamespace

import pytest
import torch

from test_host_model_cpu import _close, _models

H_, W_ = 16, 16
HWS = (1, 6, 13, 67)  # one pixel, ragged last pixel tiles, a tile count > 1 at every F <= 10


def test_frame_slot_rules_match_the_kernel_source():
    from tools import kernel_models as km
    assert km.frame_slot_rules()


@pytest.mark.parametrize("kernel,F_max", [("attn", 256), ("fused", 128)])
def test_every_frame_row_is_stored_once_with_its_own_keys(kernel, F_max):
    """attn_kernel (frames mode: packed for F <= 128, unpacked above) and tattn_fused_kernel, every F: each (clip, pixel, frame)
    row is stored by exactly one work item, and keeps exactly the F keys of its own pixel"""
    from tools import kernel_models as km
    for F in range(1, F_max + 1):
        for HW in HWS + ((130,) if F <= 2 else ()):
            km.check_frame_slot_ownership(kernel, F, HW)


def test_fused_key_tiles_for_every_frame_count():
    from tools import kernel_models as km
    for F in range(1, 129):
        km.check_fused_key_tiles(F)


@pytest.mark.parametrize("kernel,F,HW", [("attn", 24, 13), ("attn", 72, 3), ("attn", 100, 2), ("fused", 24, 13),
                                         ("fused", 40, 7), ("fused", 120, 2)])
def test_unmasked_tail_slot_is_caught(kernel, F, HW):
    """slots past floor(128 / F) * F taken as the next pixel: that pixel's first frames are stored twice, once from an
    incomplete key set"""
    from tools import kernel_models as km
    with pytest.raises(AssertionError):
        km.check_frame_slot_ownership(kernel, F, HW, tail_masked=False)


@pytest.mark.parametrize("F", [24, 40, 48, 56])
def test_own_half_key_tile_rule_kept_at_frame_counts_not_dividing_64_is_caught(F):
    """kt = wg for every F <= 64 (right only when F divides 64): a pixel straddling slot 64 loses the keys of the other half"""
    from tools import kernel_models as km
    with pytest.raises(AssertionError):
        km.check_fused_key_tiles(F, old_rule=True)
    with pytest.raises(AssertionError):
        km.check_frame_slot_ownership("fused", F, 13, old_rule=True)


def _inputs(F, dtype):
    from oracle import loops_ref
    ns = loops_ref.synthetic_inputs(F, H_, W_, cross_dim=64, seed=8888, dtype=dtype, device="cpu")
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
    g = torch.Generator().manual_seed(8895)
    x3 = torch.randn(3, 4, F, H_, W_, generator=g).to(dtype=dtype)
    return x3, prompts, img_lat, img_emb, fps


@torch.no_grad()
@pytest.mark.parametrize("F", [3, 24])
def test_product_unet_at_frame_counts_not_dividing_128_matches_the_oracle(emulated_ops, F):
    """a hooked edit step (conv, spatial and temporal injection) and an unhooked inversion forward (B = 1)"""
    from anyv2v_b200 import pnp_utils as ours_hooks
    from oracle import pnp_hooks_ref, schedulers_ref
    ref32, ours = _models()
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    schedule = s.timesteps[:5]
    t = 901
    outs = {}
    for name, net, dt, hooks in (("ref32", ref32, torch.float32, pnp_hooks_ref), ("ours", ours, torch.float16, ours_hooks)):
        pipe = SimpleNamespace(unet=net)
        hooks.register_conv_injection(pipe, schedule)
        hooks.register_spatial_attention_pnp(pipe, schedule)
        hooks.register_temp_attention_pnp(pipe, schedule)
        hooks.register_time(pipe, t)
        x3, prompts, img_lat, img_emb, fps = _inputs(F, dt)
        outs[name] = net(x3, torch.tensor([t]), fps, img_lat, img_emb, prompts)[0]
        for reg in (hooks.register_conv_injection, hooks.register_spatial_attention_pnp, hooks.register_temp_attention_pnp):
            reg(pipe, [])
        hooks.register_time(pipe, -1)
        outs[name + " inv"] = net(x3[:1], torch.tensor([501]), fps[:1], img_lat[:1], img_emb[:1], prompts[:1])[0]
    assert outs["ours"].shape == (3, 4, F, H_, W_)
    _close(outs["ours"], outs["ref32"], f"hooked UNet F={F}")
    _close(outs["ours inv"], outs["ref32 inv"], f"unhooked UNet F={F}")


@torch.no_grad()
def test_every_temporal_self_attention_at_24_frames_goes_through_the_fused_kernel(emulated_ops, monkeypatch):
    """F = 24: every temporal self-attention is one ops.temporal_attention_fused launch (none falls back to projection +
    frames-mode ops.attention), and on an injected step the 8 hooked attn1 sites pass n_v = 3"""
    from anyv2v_b200 import ops, pnp_utils as ours_hooks
    from oracle import schedulers_ref
    F = 24
    _, ours = _models()
    pipe = SimpleNamespace(unet=ours)
    s = schedulers_ref.DDIMScheduler()
    s.set_timesteps(10)
    ours_hooks.register_temp_attention_pnp(pipe, s.timesteps[:5])
    ours_hooks.register_time(pipe, 901)
    fused, frames_attn = [], []
    real_fused, real_attn = ops.temporal_attention_fused, ops.attention

    def spy_fused(x, wqkv, heads, F_, *a, **kw):
        fused.append((F_, kw.get("n_v", 1)))
        return real_fused(x, wqkv, heads, F_, *a, **kw)

    def spy_attn(*a, **kw):
        if kw.get("frames_mode"):
            frames_attn.append(a[4])
        return real_attn(*a, **kw)

    monkeypatch.setattr(ops, "temporal_attention_fused", spy_fused)
    monkeypatch.setattr(ops, "attention", spy_attn)
    x3, prompts, img_lat, img_emb, fps = _inputs(F, torch.float16)
    out = ours(x3, torch.tensor([901]), fps, img_lat, img_emb, prompts)[0]
    assert torch.isfinite(out).all()
    n_temporal = 1 + sum(len(b.temp_attentions) for b in list(ours.down_blocks) + list(ours.up_blocks) if b.has_cross_attention) + 1
    temporal = [nv for f, nv in fused if f == F]
    assert frames_attn == []
    assert len(temporal) == 2 * n_temporal                   # attn1 + attn2 of every temporal transformer
    assert temporal.count(3) == 8                             # the 8 hooked attn1 sites (pnp_utils.py:340-346)
    ours_hooks.register_temp_attention_pnp(pipe, [])
    ours_hooks.register_time(pipe, -1)
