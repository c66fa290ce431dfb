"""GPU tests of source-feature sharing between PnP edits of one inverted clip (`I2VGenXLPipeline.source_feature_cache`).

The kernels a replayed step runs: rows- and frames-mode attention at n_v = 2 and the fused temporal attention with Q / K from
a separate source tensor (av2v_tattn_fused_qksrc_f16), each against its float64 contract inside guarded buffers (within
KAPPA_ATTN * cond element by element, and unbiased) and bit for bit equal to the edit branches of the n_v = 3 call.  Then
the full-size UNet at 16 x 512^2: a second edit of one inversion with the cache is bit-identical at every one of the 50
steps to the same edit without it, on the CUDA-graph path and eagerly, at eta 0 and 1; and the edit runner's
``share_source_features`` key leaves the output files unchanged."""
import gc
import os
from types import SimpleNamespace

import pytest
import torch
import yaml

import source_cache_ref as scr
from bias_check import assert_unbiased
from guarded import check_output, guarded_input, guarded_output
from ulp_check import KAPPA_ATTN, assert_within_bound, cond_attention

pytestmark = pytest.mark.gpu
dev = "cuda"


def _branches(rows, C, g, gap=64):
    """V of [source, uncond, cond] with `gap` NaN rows between the branches -> (values, branch stride in rows)"""
    nan = torch.full((gap, C), float("nan"), dtype=torch.float16)
    v = [torch.randn(rows, C, generator=g).half() for _ in range(3)]
    return torch.cat([v[0], nan, v[1], nan, v[2]]), rows + gap


def _attention_pair(batch, heads, seq, seq_kv, frames, HW=0, seed=0, unbiased=False):
    """ops.attention at n_v = 3 on [source, uncond, cond] and at n_v = 2 on [uncond, cond] with the same Q / K"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(seed)
    C = heads * 64
    ldq, ldk, ldv, ldo = C + 8, C + 16, C + 24, C + 40
    nk = seq_kv if seq_kv else seq
    kv_rows = batch * seq if frames else batch * nk
    q = guarded_input(torch.randn(batch * seq, C, generator=g).half(), ld=ldq, device=dev, guard=128 * ldq)
    k = guarded_input(torch.randn(kv_rows, C, generator=g).half(), ld=ldk, device=dev, guard=128 * ldk)
    vvals, vstride = _branches(kv_rows, C, g)
    v = guarded_input(vvals, ld=ldv, device=dev, guard=128 * ldv)
    rows = batch * seq
    mode = dict(frames_mode=frames, HW=HW) if frames else dict(seq_kv=seq_kv)
    out3 = guarded_output((3 * rows, C), ld=ldo, device=dev)
    ops.attention(q.view, k.view, v.view, heads, seq, batch, out3.view, n_v=3, v_branch_stride=vstride * ldv,
                  o_branch_stride=rows * ldo, **mode)
    v2 = guarded_input(vvals[vstride:], ld=ldv, device=dev, guard=128 * ldv)  # the edit branches only
    out2 = guarded_output((2 * rows, C), ld=ldo + 8, device=dev)
    kw = dict(n_v=2, v_branch_stride=vstride * ldv, o_branch_stride=rows * (ldo + 8), **mode)
    ops.attention(q.view, k.view, v2.view, heads, seq, batch, out2.view, **kw)
    torch.cuda.synchronize()
    what = f"attention n_v=2 {'frames' if frames else 'rows'} b{batch} h{heads} s{seq} kv{seq_kv} HW{HW}"
    check_output(out2, what)
    got = out2.view.cpu()
    assert torch.equal(got, out3.view.cpu()[rows:]), f"{what}: differs from the edit branches of the n_v = 3 call"
    o = torch.empty(2 * rows, ldo + 8, dtype=torch.float16)[:, :C]
    ref, cond = scr.attention_exact(q.to("cpu").view, k.to("cpu").view, v2.to("cpu").view, heads, seq, batch, o,
                                   cond=cond_attention(0.125), **kw)
    assert_within_bound(got, ref, cond, KAPPA_ATTN, what, shape=tuple(got.shape))
    if unbiased:
        assert_unbiased(got, ref, cond, KAPPA_ATTN, what)


@pytest.mark.parametrize("case", [(2, 2, 256, 0), (4, 2, 130, 145), (1, 2, 1024, 0), (2, 2, 200, 600), (1, 1, 4096, 0)],
                         ids=lambda c: "b{}h{}s{}kv{}".format(*c))
def test_attention_rows_two_branches(case):
    """below 512 keys attn_kernel<2>, from 512 on attn_rows_kernel<2> (64-key tiles, as at n_v = 3); ragged key tails"""
    batch, heads, seq, seq_kv = case
    _attention_pair(batch, heads, seq, seq_kv, frames=False, seed=seq + seq_kv, unbiased=seq == 4096)


@pytest.mark.parametrize("F,HW", [(16, 64), (24, 10), (3, 65), (256, 2)])
def test_attention_frames_two_branches(F, HW):
    _attention_pair(2 * HW, 2, F, 0, frames=True, HW=HW, seed=F)


@pytest.mark.parametrize("F,HW,src", [(16, 256, 1), (24, 40, 2), (3, 130, 1), (1, 130, 2)])
def test_tattn_qksrc(F, HW, src):
    """the fused temporal attention with Q / K from a separate source tensor (own row stride) and V from the two edit clips;
    F = 24 visits both key tiles, F = 3 leaves a tail in every x block, ragged pixel tiles; Cx = 320 (5 K blocks)"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(F + HW)
    heads, Cx = 5, 320
    C = heads * 64
    n = src * F * HW
    x3 = torch.randn(3 * n, Cx, generator=g)
    w = torch.randn(3 * C, Cx, generator=g) * Cx ** -0.5
    # as tests/test_gpu_bias.py: scores of order 1, and V with a per-channel offset, so that the outputs are far from zero
    w[:C] *= 2
    x3[:, 0] = 4.0
    w[:2 * C, 0] = 0
    w[2 * C:, 0] = (1 + torch.rand(C, generator=g)) * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0) / 4
    x3, w = x3.half(), w.half()
    gw = guarded_input(w, device=dev)
    out3 = guarded_output((3 * n, C), device=dev)
    ops.temporal_attention_fused(guarded_input(x3, ld=Cx + 8, device=dev, guard=128 * (Cx + 8)).view, gw.view, heads, F, HW,
                                 3 * src, out3.view, n_v=3)
    x2 = guarded_input(x3[n:], ld=Cx + 16, device=dev, guard=128 * (Cx + 16))
    qk = guarded_input(x3[:n], ld=Cx + 24, device=dev, guard=128 * (Cx + 24))
    out2 = guarded_output((2 * n, C), ld=C + 8, device=dev)
    ops.temporal_attention_fused_qksrc(x2.view, qk.view, gw.view, heads, F, HW, 2 * src, out2.view)
    torch.cuda.synchronize()
    what = f"temporal attention fused qksrc F={F} HW={HW} src={src}"
    check_output(out2, what)
    got = out2.view.cpu()
    assert torch.equal(got, out3.view.cpu()[n:]), f"{what}: differs from the edit clips of the n_v = 3 call"
    o = torch.empty(2 * n, C + 8, dtype=torch.float16)[:, :C]
    ref, cond = scr.temporal_attention_fused_qksrc_exact(x2.to("cpu").view, qk.to("cpu").view, w, heads, F, HW, 2 * src, o,
                                                        cond=cond_attention(0.125, rounded_operands=True))
    assert_within_bound(got, ref, cond, KAPPA_ATTN, what, shape=tuple(got.shape))
    if F == 16:
        assert_unbiased(got, ref, cond, KAPPA_ATTN, what)


def test_tattn_qksrc_refusals():
    from anyv2v_b200 import _lib, ops
    h = lambda r, c: torch.zeros(r, c, dtype=torch.float16, device=dev)
    with pytest.raises(_lib.Av2vError, match="clips"):
        ops.temporal_attention_fused_qksrc(h(48, 64), h(16, 64), h(384, 64), 2, 8, 2, 3, h(48, 128))
    with pytest.raises(_lib.Av2vError, match="qk_src"):
        ops.temporal_attention_fused_qksrc(h(32, 64), h(32, 64), h(384, 64), 2, 8, 2, 2, h(32, 128))
    with pytest.raises(_lib.Av2vError, match="n_v"):
        ops.attention(h(64, 64), h(64, 64), h(64, 64), 1, 64, 1, h(64, 64), n_v=4)


@pytest.mark.parametrize("n,rows,C", [(48, 256, 1280), (48, 64, 1280), (32, 1024, 640), (3, 16 * 4096, 320), (48, 4096, 640)])
def test_groupnorm_partition(n, rows, C):
    """GroupNorm on the last two thirds of a batch with the partition of the whole batch gives each sample the statistics the
    whole batch's call gives it, bit for bit (without it the per-frame norms of the 16 x 16 and 8 x 8 levels cut their
    reductions differently)"""
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(n + rows)
    x = (torch.randn(n, rows, C, generator=g) * 2 + 0.5).half().to(dev)
    gamma = (torch.randn(C, generator=g) * 0.2 + 1).half().to(dev)
    beta = (torch.randn(C, generator=g) * 0.2).half().to(dev)
    full = ops.groupnorm(x, gamma, beta, 32, 1e-5, True)
    part = ops.groupnorm(x[n // 3:].contiguous(), gamma, beta, 32, 1e-5, True, partition_samples=n)
    assert torch.equal(part, full[n // 3:])


# ------------------------------------------------------------------------------------------------------------- full size
N_STEPS = 50
DEMO = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0)
CONFIG3 = SimpleNamespace(n_steps=N_STEPS, pnp_f_t=0.8, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.5)


def _setup(config, F, h, w, cross_dim, n_steps):
    from anyv2v_b200 import distributed
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.run_group_pnp_edit import synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    torch.set_grad_enabled(False)
    unet = distributed.build_unet_replicated(I2VGenXLUNet, config, 8888, torch.device(dev))
    sched = DDIMScheduler()
    sched.set_timesteps(n_steps)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(3)
    for t in sched.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, F, h, w, generator=g).half().to(dev))
    edits = [{k: v.to(dev) for k, v in synthetic_conditioning(F, h, w, cross_dim, seed, "cpu").items()} for seed in (1, 2)]
    for e in edits[1:]:  # one clip and inversion: the source side of every edit is the first's
        for k in ("video_latents", "inv_prompt", "src_image_emb", "src_image_latents"):
            e[k] = edits[0][k]
    return SimpleNamespace(unet=unet, store=store, edits=edits, n_steps=n_steps)


@pytest.fixture(scope="module")
def full():
    from anyv2v_b200.unet_i2vgen_xl import I2VGEN_XL_CONFIG
    return _setup(I2VGEN_XL_CONFIG, 16, 64, 64, 1024, N_STEPS)


def _full_edit(full, pnp, c, eta, graphs, cache):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    sched = DDIMScheduler()
    sched.set_timesteps(full.n_steps)
    pipe = I2VGenXLPipeline(full.unet, sched)
    pipe.use_cuda_graphs = graphs
    init_pnp(pipe, sched, pnp)
    seen = []
    pipe.sample_with_pnp(latents=c["video_latents"].clone(), prompt_embeds=c["edit_prompt"], negative_prompt_embeds=c["neg_prompt"],
                         ddim_inv_prompt_embeds=c["inv_prompt"], image_embeddings=c["edit_image_emb"],
                         image_latents=c["edit_image_latents"], ddim_inv_image_embeddings=c["src_image_emb"],
                         ddim_inv_image_latents=c["src_image_latents"], target_fps=8, num_inference_steps=full.n_steps,
                         guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=full.store, eta=eta, num_frames=c["video_latents"].shape[2],
                         generator=torch.Generator().manual_seed(77), source_features=cache,
                         callback=lambda i, t, x: seen.append(x.clone()))
    return pipe, seen


@pytest.mark.parametrize("pnp,graphs,eta", [(DEMO, True, 0.0), (DEMO, False, 1.0), (CONFIG3, True, 1.0), (CONFIG3, False, 0.0)],
                         ids=["demo-graphs-eta0", "demo-eager-eta1", "config3-graphs-eta1", "config3-eager-eta0"])
def test_full_size_second_edit_is_bit_identical(full, pnp, graphs, eta):
    from anyv2v_b200.pipeline import SourceFeatureCache
    cache = SourceFeatureCache(full.unet, 40 << 30)
    _full_edit(full, pnp, full.edits[0], eta, graphs, cache)
    injected = int(N_STEPS * pnp.pnp_f_t)
    assert len(cache) == injected
    torch.cuda.reset_peak_memory_stats()
    _, got = _full_edit(full, pnp, full.edits[1], eta, graphs, cache)
    assert len(cache) == injected
    _, want = _full_edit(full, pnp, full.edits[1], eta, graphs, None)
    assert len(got) == len(want) == N_STEPS
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.isfinite(a.float()).all() and torch.equal(a, b), f"step {i}: the cached edit differs"
    print(f"cache {cache.nbytes / 2**30:.2f} GiB for {len(cache)} steps; peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    del cache
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("graphs", [True, False])
def test_tiny_unet_edits_are_bit_identical(graphs):
    """the tiny UNet at 4 frames of 16 x 16: its spatial attention over 16 and 4 tokens runs on the fused temporal kernel with
    the frames of every branch packed as the pixels of one clip (the protocol path of AttnProcessor), where a frame's rounding
    depends on its place in the tile; a second edit with another schedule replays the first's steps and captures its own"""
    from anyv2v_b200.pipeline import SourceFeatureCache
    from oracle.unet_ref import TINY_CONFIG
    tiny = _setup(TINY_CONFIG, 4, 16, 16, 64, 5)
    cache = SourceFeatureCache(tiny.unet, 1 << 30)
    a = SimpleNamespace(n_steps=5, pnp_f_t=1.0, pnp_spatial_attn_t=0.6, pnp_temp_attn_t=0.6)
    b = SimpleNamespace(n_steps=5, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0)
    _full_edit(tiny, a, tiny.edits[0], 0.0, graphs, cache)
    _, got = _full_edit(tiny, b, tiny.edits[1], 0.0, graphs, cache)
    _, want = _full_edit(tiny, b, tiny.edits[1], 0.0, graphs, None)
    assert len(cache) == 7   # the first edit's 3 + 2 step kinds, then the second's 2 steps with all three injections
    for i, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), f"step {i}: the cached edit differs by up to {(x.float() - y.float()).abs().max().item():.3g}"


# ------------------------------------------------------------------------------------------------------------- runner
def test_runner_shares_source_features(tmp_path):
    """three JSON edits of one clip (other prompts, first-frame file names and schedules): the same files with
    ``share_source_features`` on and off"""
    from anyv2v_b200 import run_group_ddim_inversion as inv, run_group_pnp_edit as edit
    from anyv2v_b200.config import OmegaConf
    from oracle.unet_ref import TINY_CONFIG
    from test_gpu_runners import EDIT_TEMPLATE, INV_TEMPLATE, TINY_VAE, write_demo_clip
    torch.set_grad_enabled(False)
    data = str(tmp_path)
    edited = write_demo_clip(data)
    inv_t = dict(INV_TEMPLATE, data_dir=data, device="cuda:0", synthetic=False)
    inv_t["inverse_config"] = dict(inv_t["inverse_config"], prompt="a man", negative_prompt="blurry")
    inv_t["recon_config"] = dict(inv_t["recon_config"], enable_recon=False)
    (tmp_path / "inv.yaml").write_text(yaml.safe_dump(inv_t))
    kw = dict(vae_config=TINY_VAE)
    one = [{"active": True, "video_name": "clipA", "edited_first_frame_path": edited, "editing_prompt": "x"}]
    inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), one, torch.device(dev), unet_config=TINY_CONFIG, pipeline_kwargs=kw)
    entries = [{"active": True, "video_name": "clipA", "edited_first_frame_path": edited, "editing_prompt": p,
                "edited_video_name": f"e{i}", "ddim_init_latents_t_idx": 0, "pnp_f_t": f, "pnp_spatial_attn_t": s,
                "pnp_temp_attn_t": s}
               for i, (p, f, s) in enumerate([("a robot", 1.0, 0.6), ("a cat", 0.6, 0.4), ("a dog", 1.0, 1.0)])]
    outs = {}
    for share in (False, True):
        out_dir = os.path.join(data, f"share{int(share)}")
        t = dict(EDIT_TEMPLATE, data_dir=data, device="cuda:0", synthetic=False, share_source_features=share,
                 output_dir=out_dir + "/${edited_video_name}")
        (tmp_path / "edit.yaml").write_text(yaml.safe_dump(t))
        torch.manual_seed(0)
        edit.main(OmegaConf.load(str(tmp_path / "edit.yaml")), entries, torch.device(dev), unet_config=TINY_CONFIG,
                  pipeline_kwargs=kw)
        files = {}
        for root, _, names in os.walk(out_dir):
            for n in names:
                if n.endswith((".pt", ".png")):
                    p = os.path.join(root, n)
                    files[os.path.relpath(p, out_dir)] = torch.load(p) if n.endswith(".pt") else open(p, "rb").read()
        outs[share] = files
    assert len(outs[False]) == 3 * 5 and outs[False].keys() == outs[True].keys()
    differ = sorted(n for n, a in outs[False].items()
                    if not (torch.equal(a, outs[True][n]) if torch.is_tensor(a) else a == outs[True][n]))
    assert not differ, f"differ with share_source_features: {differ}"
    shared = edit.SharedSourceFeatures()
    cfg = OmegaConf.merge(OmegaConf.load(str(tmp_path / "edit.yaml")), OmegaConf.create(entries[0]))
    assert edit.clip_key(cfg) == edit.clip_key(OmegaConf.merge(cfg, OmegaConf.create(entries[1])))
    assert shared.for_entry(SimpleNamespace(source_feature_cache=lambda max_bytes: object()), cfg) is not None
