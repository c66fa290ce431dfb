"""Layer-by-layer comparison of this package's UNet against the oracle (development aid)."""
import sys

import torch

sys.path.insert(0, ".")
from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet, timestep_embedding  # noqa: E402
from oracle import loops_ref, unet_ref  # noqa: E402

dev = "cuda"
B = int(sys.argv[1]) if len(sys.argv) > 1 else 1
T = int(sys.argv[2]) if len(sys.argv) > 2 else 251
F_, H_, W_ = 4, 16, 16
ref = unet_ref.seeded_unet(unet_ref.TINY_CONFIG, dtype=torch.float32, device=dev)
net = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
net.load_state_dict(ref.state_dict())
net = net.to(dev, torch.float16).eval()

acts = {}


def hook(name):
    def f(m, i, o):
        acts[name] = (o[0] if isinstance(o, tuple) else o).detach()
    return f


for name, m in ref.named_modules():
    if name and name.count(".") <= 3:
        m.register_forward_hook(hook(name))

ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float32, device=dev)
if B == 3:
    prompts, img_lat, img_emb, fps = loops_ref.edit_conditioning(ns)
    x = torch.randn(3, 4, F_, H_, W_, device=dev)
else:
    prompts, img_lat, img_emb, fps = ns.inv_prompt, ns.src_image_latents, ns.src_image_emb, ns.fps
    x = ns.video_latents
with torch.no_grad():
    out_ref = ref(x, torch.tensor([T], device=dev), fps, img_lat, img_emb, prompts)[0]


def cmp(name, got_nhwc, key=None):
    r = acts[key or name]
    g = got_nhwc.permute(0, 3, 1, 2).float() if got_nhwc.dim() == 4 else got_nhwc.float()
    e = (g - r).pow(2).mean().sqrt() / r.pow(2).mean().sqrt()
    print(f"{name:40s} rms_rel {float(e):.3e}  shape {tuple(r.shape)}", flush=True)


with torch.no_grad():
    h = lambda t: t.half()
    cond = net.precompute_conditioning(fps, h(img_lat), h(img_emb), h(prompts))
    b, c, f, hh, ww = x.shape
    t = torch.tensor([T], device=dev).expand(b)
    emb = net.time_embedding(timestep_embedding(t, 64).half()) + cond["fps_emb"]
    cmp("time_embedding", net.time_embedding(timestep_embedding(t, 64).half()))
    emb = emb.repeat_interleave(f, dim=0).contiguous()
    xx = h(x).permute(0, 2, 3, 4, 1).reshape(b * f, hh, ww, c)
    xx = torch.cat([xx, cond["image_latents_nhwc"]], dim=-1)
    xx = net.conv_in.forward_nhwc(xx)
    cmp("conv_in", xx)
    xx = net.transformer_in.forward_nhwc(xx, f)
    cmp("transformer_in", xx)
    skips = [xx]
    for bi, blk in enumerate(net.down_blocks):
        for i in range(len(blk.resnets)):
            xx = blk.resnets[i].forward_nhwc(xx, emb)
            cmp(f"down_blocks.{bi}.resnets.{i}", xx)
            xx = blk.temp_convs[i].forward_nhwc(xx, f)
            cmp(f"down_blocks.{bi}.temp_convs.{i}", xx)
            if blk.has_cross_attention:
                xx = blk.attentions[i].forward_nhwc(xx, cond["ctx"])
                cmp(f"down_blocks.{bi}.attentions.{i}", xx)
                xx = blk.temp_attentions[i].forward_nhwc(xx, f)
                cmp(f"down_blocks.{bi}.temp_attentions.{i}", xx)
            skips.append(xx)
        if blk.downsamplers is not None:
            xx = blk.downsamplers[0].forward_nhwc(xx)
            cmp(f"down_blocks.{bi}.downsamplers.0", xx)
            skips.append(xx)
    xx = net.mid_block.forward_nhwc(xx, emb, cond["ctx"], f)
    cmp("mid_block", xx)
    for bi, blk in enumerate(net.up_blocks):
        for i in range(len(blk.resnets)):
            xx = torch.cat([xx, skips.pop()], dim=-1)
            xx = blk.resnets[i].forward_nhwc(xx, emb)
            cmp(f"up_blocks.{bi}.resnets.{i}", xx)
            xx = blk.temp_convs[i].forward_nhwc(xx, f)
            cmp(f"up_blocks.{bi}.temp_convs.{i}", xx)
            if blk.has_cross_attention:
                xx = blk.attentions[i].forward_nhwc(xx, cond["ctx"])
                cmp(f"up_blocks.{bi}.attentions.{i}", xx)
                xx = blk.temp_attentions[i].forward_nhwc(xx, f)
                cmp(f"up_blocks.{bi}.temp_attentions.{i}", xx)
        if blk.upsamplers is not None:
            xx = blk.upsamplers[0].forward_nhwc(xx)
            cmp(f"up_blocks.{bi}.upsamplers.0", xx)
    out = net(h(x), torch.tensor([T], device=dev), cond=cond)[0]
    e = (out.float() - out_ref).pow(2).mean().sqrt() / out_ref.pow(2).mean().sqrt()
    print("final", float(e))
