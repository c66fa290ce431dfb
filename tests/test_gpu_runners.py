"""GPU tests of the runner / config surface: the two group runners end to end (tiny UNet), the reference's file
hand-off between the phases, and CUDA-graph replay vs eager launches."""
import json
import os
from types import SimpleNamespace

import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu
dev = "cuda"

INV_TEMPLATE = {
    "synthetic": True,  # explicit opt-in: seeded stand-ins for CLIP / VAE (SURVEY 8d); the real-input path is tested below
    "seed": 8888, "device": "cuda:0", "debug": False, "data_dir": "DATA", "model_name": "i2vgen-xl", "exp_name": "${video_name}",
    "output_dir": "${data_dir}/inversions/${model_name}/${exp_name}", "image_size": [128, 128], "video_dir": "${data_dir}/demo",
    "video_name": "ReplaceMe", "video_path": "ReplaceMe", "video_frames_path": "ReplaceMe", "n_frames": 4,
    "inverse_config": {"image_size": "${image_size}", "n_frames": "${n_frames}", "cfg": 1.0, "target_fps": 8, "prompt": "",
                       "negative_prompt": "", "n_steps": 5, "output_dir": "${output_dir}/ddim_latents",
                       "inverse_static_video": False, "null_image_inversion": False},
    "recon_config": {"enable_recon": True, "image_size": "${image_size}", "n_frames": "${n_frames}", "cfg": 9.0, "target_fps": 8,
                     "prompt": "", "negative_prompt": "x", "n_steps": 5, "ddim_init_latents_t_idx": 1,
                     "ddim_latents_path": "${inverse_config.output_dir}"},
}
EDIT_TEMPLATE = {
    "synthetic": True,
    "seed": 8888, "device": "cuda:0", "debug": False, "data_dir": "DATA", "model_name": "i2vgen-xl", "task_name": "Prompt-Based-Editing",
    "edited_video_name": "ReplaceMe", "output_dir": "${data_dir}/Results/${task_name}/${model_name}/${video_name}/${edited_video_name}/",
    "image_size": [128, 128], "video_dir": "${data_dir}/demo", "video_name": "ReplaceMe", "video_path": "ReplaceMe",
    "video_frames_path": "ReplaceMe", "edited_first_frame_path": "ReplaceMe",
    "ddim_latents_path": "${data_dir}/inversions/${model_name}/${video_name}/ddim_latents", "n_frames": 4, "cfg": 9.0, "target_fps": 8,
    "editing_prompt": "ReplaceMe", "editing_negative_prompt": "bad", "n_steps": 5, "ddim_init_latents_t_idx": 1, "ddim_inv_prompt": "",
    "random_ratio": 0.0, "pnp_f_t": 0.2, "pnp_spatial_attn_t": 0.2, "pnp_temp_attn_t": 0.5,
}


def test_group_runners_end_to_end(tmp_path):
    """run_group_ddim_inversion -> ddim_latents_{t}.pt files -> run_group_pnp_edit, same template/JSON API as the reference."""
    from anyv2v_b200 import run_group_ddim_inversion as inv, run_group_pnp_edit as edit
    from anyv2v_b200.config import OmegaConf
    from oracle.unet_ref import TINY_CONFIG
    data = str(tmp_path)
    for name, tpl in (("inv.yaml", INV_TEMPLATE), ("edit.yaml", EDIT_TEMPLATE)):
        t = dict(tpl, data_dir=data)
        (tmp_path / name).write_text(yaml.safe_dump(t))
    entries = [{"active": True, "video_name": "clipA", "edited_first_frame_path": "demo/clipA/edited.png", "editing_prompt": "a robot",
                "edited_video_name": "robot", "ddim_init_latents_t_idx": 0, "pnp_f_t": 1.0, "pnp_spatial_attn_t": 1.0, "pnp_temp_attn_t": 1.0},
               {"active": False, "video_name": "skipped", "edited_first_frame_path": "x", "editing_prompt": "x", "edited_video_name": "x"}]
    torch.set_grad_enabled(False)
    device = torch.device("cuda", 0)
    out = inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), entries, device, unet_config=TINY_CONFIG)
    assert len(out) == 1 and out[0].shape == (5, 4, 4, 16, 16)  # [steps, c, f, h, w] like the reference (:54)
    lat_dir = os.path.join(data, "inversions", "i2vgen-xl", "clipA", "ddim_latents")
    assert sorted(os.listdir(lat_dir)) == sorted(f"ddim_latents_{t}.pt" for t in (1, 201, 401, 601, 801))
    assert os.path.exists(os.path.join(data, "inversions", "i2vgen-xl", "clipA", "ddim_reconstruction", "latents.pt"))
    # second call: the reference's skip rule (existing output_dir)
    assert inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), entries, device, unet_config=TINY_CONFIG) == []
    res = edit.main(OmegaConf.load(str(tmp_path / "edit.yaml")), entries, device, unet_config=TINY_CONFIG)
    assert len(res) == 1 and res[0].shape == (1, 4, 4, 16, 16) and torch.isfinite(res[0]).all()
    suffix = "ddim_init_latents_t_idx_0_nsteps_5_cfg_9.0_pnpf1.0_pnps1.0_pnpt1.0"
    saved = os.path.join(data, "Results", "Prompt-Based-Editing", "i2vgen-xl", "clipA", "robot", suffix, "edited_latents.pt")
    assert os.path.exists(saved) and torch.equal(torch.load(saved), res[0].cpu())


def test_capture_outlives_a_loop_state_that_dies_during_it():
    """A finished loop's state is a reference cycle (its iterations' bodies close over it) holding CUDA graphs.  When it
    becomes garbage while another iteration captures, the cyclic collector must not free it there: destroying a graph
    inside a capture invalidates the capture.  It is freed at the next collection outside the capture."""
    import gc
    import weakref
    from anyv2v_b200.pipeline import _GraphedIteration

    def loop_state():
        st = SimpleNamespace(x=torch.zeros(8, device=dev))
        st.it = _GraphedIteration(lambda: st.x.add_(1))  # st -> it -> body -> st
        for _ in range(2):
            st.it.run()                                # eager, then captured: the cycle holds a CUDAGraph
        return st
    holder = [loop_state()]
    gone = weakref.ref(holder[0].it)
    x, seen = torch.zeros(1024, device=dev), []

    def body():
        seen.append(gc.isenabled())
        if torch.cuda.is_current_stream_capturing():
            holder.clear()                             # the old state becomes garbage inside the capture
            _ = [[] for _ in range(2000)]              # ... and a collection falls due
        x.add_(1)
    it = _GraphedIteration(body)
    threshold = gc.get_threshold()
    gc.set_threshold(1)
    try:
        for _ in range(3):
            it.run()                                   # eager, capture + replay, replay
    finally:
        gc.set_threshold(*threshold)
    torch.cuda.synchronize()
    assert seen == [True, False] and gc.isenabled()
    assert torch.all(x == 3)
    gc.collect()
    assert gone() is None


def test_cuda_graph_replay_equals_eager():
    """A captured loop iteration replayed with new device-resident scalars == the same kernels launched eagerly."""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import build_pipeline, init_pnp, synthetic_conditioning
    from anyv2v_b200.schedulers import DDIMInverseScheduler, DDIMScheduler
    from oracle.unet_ref import TINY_CONFIG
    torch.set_grad_enabled(False)
    device = torch.device("cuda", 0)
    pipe = build_pipeline(device, TINY_CONFIG, seed=1, broadcast=False)
    c = synthetic_conditioning(4, 16, 16, 64, 3, device)
    results = {}
    for graphs in (False, True):
        I2VGenXLPipeline.use_cuda_graphs = graphs
        pipe.scheduler = DDIMInverseScheduler()
        inv = pipe.invert(latents=c["video_latents"], prompt_embeds=c["inv_prompt"], image_latents=c["src_image_latents"],
                          image_embeddings=c["src_image_emb"], target_fps=8, num_inference_steps=6, guidance_scale=1.0, write_files=False)
        store = pipe.latent_store
        es = DDIMScheduler()
        es.set_timesteps(6)
        pipe.scheduler = es
        init_pnp(pipe, es, SimpleNamespace(n_steps=6, pnp_f_t=0.5, pnp_spatial_attn_t=0.5, pnp_temp_attn_t=0.34))
        out = pipe.sample_with_pnp(latents=store.get(es.timesteps.tolist()[0]).clone(), prompt_embeds=c["edit_prompt"],
                                   negative_prompt_embeds=c["neg_prompt"], ddim_inv_prompt_embeds=c["inv_prompt"],
                                   image_embeddings=c["edit_image_emb"], image_latents=c["edit_image_latents"],
                                   ddim_inv_image_embeddings=c["src_image_emb"], ddim_inv_image_latents=c["src_image_latents"],
                                   target_fps=8, num_inference_steps=6, guidance_scale=9.0, ddim_init_latents_t_idx=0, latent_store=store).frames
        results[graphs] = (inv.clone(), out.clone())
    I2VGenXLPipeline.use_cuda_graphs = True
    assert torch.equal(results[False][0], results[True][0]), "inversion: graph replay differs from eager launches"
    assert torch.equal(results[False][1], results[True][1]), "edit: graph replay differs from eager launches"


TINY_VAE = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(64, 64, 64, 64), layers_per_block=1,
                norm_num_groups=32, scaling_factor=0.18215)


def write_demo_clip(data_dir, name="clipA", n=4, size=(128, 128)):
    """png frames + an edited first frame in the reference's demo layout ({data_dir}/demo/{video_name}/%05d.png)"""
    import numpy as np
    from PIL import Image
    d = os.path.join(data_dir, "demo", name)
    os.makedirs(os.path.join(d, "edited_first_frame"), exist_ok=True)
    yy, xx = np.mgrid[0:size[1], 0:size[0]]
    for i in range(n):
        img = np.stack([(xx * 2 + 10 * i) % 256, (yy * 2) % 256, ((xx + yy) + 30 * i) % 256], -1).astype("uint8")
        Image.fromarray(img).save(os.path.join(d, f"{i:05d}.png"))
    Image.fromarray(np.stack([(yy * 3) % 256, (xx * 2) % 256, (xx ^ yy) % 256], -1).astype("uint8")).resize((160, 144)).save(
        os.path.join(d, "edited_first_frame", "robot.png"))
    return f"demo/{name}/edited_first_frame/robot.png"


def run_real_input_runners(tmp_path, device, cfg_inv=1.0):
    """frames on disk + prompt strings -> run_group_ddim_inversion -> run_group_pnp_edit -> png / gif / latents, with the tiny
    UNet / VAE / CLIP towers (random init): the reference's REAL input path (run_group_ddim_inversion.py:29-55,125-160;
    run_group_pnp_edit.py:95-183)"""
    from anyv2v_b200 import run_group_ddim_inversion as inv, run_group_pnp_edit as edit
    from anyv2v_b200.config import OmegaConf
    from oracle.unet_ref import TINY_CONFIG
    data = str(tmp_path)
    edited = write_demo_clip(data)
    inv_t = dict(INV_TEMPLATE, data_dir=data, device=str(device), synthetic=False)
    inv_t["inverse_config"] = dict(inv_t["inverse_config"], cfg=cfg_inv, prompt="a man", negative_prompt="blurry")
    inv_t["recon_config"] = dict(inv_t["recon_config"], enable_recon=False)
    (tmp_path / "inv.yaml").write_text(yaml.safe_dump(inv_t))
    (tmp_path / "edit.yaml").write_text(yaml.safe_dump(dict(EDIT_TEMPLATE, data_dir=data, device=str(device), synthetic=False)))
    entries = [{"active": True, "video_name": "clipA", "edited_first_frame_path": edited, "editing_prompt": "a robot doing exercises",
                "edited_video_name": "robot", "ddim_init_latents_t_idx": 0, "pnp_f_t": 1.0, "pnp_spatial_attn_t": 0.6, "pnp_temp_attn_t": 0.6,
                "random_ratio": 0.1}]
    kw = dict(vae_config=TINY_VAE)
    out = inv.main(OmegaConf.load(str(tmp_path / "inv.yaml")), entries, device, unet_config=TINY_CONFIG, pipeline_kwargs=kw)
    assert len(out) == 1 and out[0].shape == (5, 4, 4, 16, 16) and torch.isfinite(out[0]).all()
    lat_dir = os.path.join(data, "inversions", "i2vgen-xl", "clipA", "ddim_latents")
    assert sorted(os.listdir(lat_dir)) == sorted(f"ddim_latents_{t}.pt" for t in (1, 201, 401, 601, 801))
    # the files are what the reference's loader reads (i2vgen-xl/utils.py:25-39): [1, 4, F, h, w] fp16
    f = torch.load(os.path.join(lat_dir, "ddim_latents_801.pt"), map_location="cpu")
    assert f.shape == (1, 4, 4, 16, 16) and f.dtype == torch.float16 and torch.equal(f[0], out[0][0].cpu())
    res = edit.main(OmegaConf.load(str(tmp_path / "edit.yaml")), entries, device, unet_config=TINY_CONFIG, pipeline_kwargs=kw)
    assert len(res) == 1 and res[0].shape == (1, 4, 4, 16, 16) and torch.isfinite(res[0]).all()
    suffix = "ddim_init_latents_t_idx_0_nsteps_5_cfg_9.0_pnpf1.0_pnps0.6_pnpt0.6"
    od = os.path.join(data, "Results", "Prompt-Based-Editing", "i2vgen-xl", "clipA", "robot", suffix)
    names = set(os.listdir(od))
    assert {"video.gif", "edited_latents.pt"} <= names and {f"video_{i:05d}.png" for i in range(4)} <= names, names
    from PIL import Image
    assert Image.open(os.path.join(od, "video_00003.png")).size == (128, 128)
    return out, res


def test_group_runners_on_real_inputs(tmp_path):
    torch.set_grad_enabled(False)
    run_real_input_runners(tmp_path, torch.device("cuda", 0))


def test_inversion_with_guidance_matches_two_branch_oracle(tmp_path):
    """invert(guidance_scale > 1) (pipeline :1387-1388, :1407-1410): UNet on [uncond, cond], CFG folded into the fused inverse
    DDIM kernel — one teacher-forced step against the oracle"""
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.schedulers import DDIMInverseScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import loops_ref, schedulers_ref, unet_ref
    ref = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device=dev)
    net = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    net.load_state_dict(ref.state_dict())
    net = net.to(device=dev, dtype=torch.float16).eval()
    ns = loops_ref.synthetic_inputs(4, 16, 16, cross_dim=64, dtype=torch.float32, device=dev)
    h = lambda t: t.half()
    pipe = I2VGenXLPipeline(net, DDIMInverseScheduler())
    pipe.use_cuda_graphs = False
    with torch.no_grad():
        out = pipe.invert(latents=h(ns.video_latents), prompt_embeds=h(ns.inv_prompt), negative_prompt_embeds=h(ns.neg_prompt),
                          image_latents=h(ns.src_image_latents), image_embeddings=h(ns.src_image_emb), target_fps=8,
                          num_inference_steps=5, guidance_scale=3.0, max_steps=1, write_files=False)
        s = schedulers_ref.DDIMInverseScheduler()
        s.set_timesteps(5)
        t = int(s.timesteps[0])
        x = ns.video_latents
        v = ref(torch.cat([x, x]), torch.tensor([t], device=dev), ns.fps.repeat(2), torch.cat([ns.src_image_latents] * 2),
                torch.cat([torch.zeros_like(ns.src_image_emb), ns.src_image_emb]), torch.cat([ns.neg_prompt, ns.inv_prompt]))[0]
        want, _ = s.step(schedulers_ref.cfg_combine(v[0:1], v[1:2], 3.0), t, x)
    got = out[:, 0]
    err = float((got.float() - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    assert out.shape == (1, 1, 4, 4, 16, 16) and err < 5e-3, err
