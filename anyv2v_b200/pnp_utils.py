"""PnP hook surface — drop-in for the reference's ``i2vgen-xl/pnp_utils.py``.

Same four entry points, same call signatures and side effects (SURVEY 8b):
  register_time(model, t)                              pnp_utils.py:19-28
  register_conv_injection(model, injection_schedule)    pnp_utils.py:39-132
  register_spatial_attention_pnp(model, schedule)       pnp_utils.py:140-242
  register_temp_attention_pnp(model, schedule)          pnp_utils.py:246-346   (+ alias register_temporal_attention_pnp)
``model`` is the pipeline (anything with ``.unet``).  The hooks set ``.t`` / ``.injection_schedule``, replace
``up_blocks[1].resnets[1].forward`` and the ``attn1.processor`` of the 8 + 8 PnP sites, and re-registration is
idempotent — exactly as in the reference.  What the replaced code *does* is different: on a scheduled timestep
  * the resnet computes norm1/conv1/norm2/conv2 for the SOURCE frames only and the conv2 epilogue stores the tile to
    the three branch slots (fused conv + residual-copy, anyv2v_b200/csrc/gemm_wgmma.cu);
  * the attention projects q,k for the source third only and one wgmma kernel applies the shared probabilities
    to [V_src | V_uncond | V_cond] (anyv2v_b200/csrc/attention_wgmma.cu).
Outputs equal the reference's (which computes everything three times and then overwrites two thirds).
The membership test ``t in schedule or t == 1000`` is evaluated on the host from a Python set — no device sync.
"""
from __future__ import annotations

import logging

import torch

from .unet_i2vgen_xl import AttnProcessor, to_nchw_view, to_nhwc

logger = logging.getLogger(__name__)

_TIMED_SITES = {1: (0, 1, 2), 2: (0, 1, 2), 3: (0, 1, 2)}   # register_time touches these (pnp_utils.py:22)
_PNP_SITES = {1: (1, 2), 2: (0, 1, 2), 3: (0, 1, 2)}         # hooks are installed on these (pnp_utils.py:235, 340)


def _schedule_set(injection_schedule):
    if injection_schedule is None:
        return None
    if torch.is_tensor(injection_schedule):
        return frozenset(int(v) for v in injection_schedule.detach().cpu().reshape(-1).tolist())
    return frozenset(int(v) for v in injection_schedule)


def _fires(t, sched_set) -> bool:
    if sched_set is None or t is None:
        return False
    t = int(t)
    return t in sched_set or t == 1000


def register_time(model, t):
    conv_module = model.unet.up_blocks[1].resnets[1]
    setattr(conv_module, "t", t)
    for res, blocks in _TIMED_SITES.items():
        for block in blocks:
            up = model.unet.up_blocks[res]
            setattr(up.attentions[block].transformer_blocks[0].attn1.processor, "t", t)
            setattr(up.temp_attentions[block].transformer_blocks[0].attn1.processor, "t", t)


def register_conv_injection(model, injection_schedule):
    conv_module = model.unet.up_blocks[1].resnets[1]

    def forward(input_tensor, temb, scale: float = 1.0):
        fire = _fires(getattr(conv_module, "t", None), conv_module._injection_set)
        # a source feature in "replay" mode: the batch is [uncond, cond] and the source's conv2 input comes from the cache
        source = getattr(conv_module, "source_feature", None) if fire else None
        replay = source is not None and source.mode == "replay"
        inject = fire and not replay and input_tensor.shape[0] % 3 == 0
        if inject or replay:
            logger.debug("PnP Injecting Conv at t=%s", conv_module.t)
        return to_nchw_view(conv_module.forward_nhwc(to_nhwc(input_tensor), temb, inject=inject,
                                                     source=source if inject or replay else None))

    conv_module.forward = forward
    setattr(conv_module, "injection_schedule", injection_schedule)
    conv_module._injection_set = _schedule_set(injection_schedule)


class _PnPAttnProcessor(AttnProcessor):
    kind = "Attn"

    def __init__(self, injection_schedule):
        self.injection_schedule = injection_schedule
        self._injection_set = _schedule_set(injection_schedule)
        self.t = None

    def __setattr__(self, name, value):
        object.__setattr__(self, name, value)
        if name == "injection_schedule":
            object.__setattr__(self, "_injection_set", _schedule_set(value))

    def inject_now(self) -> bool:
        fire = _fires(self.t, self._injection_set)
        if fire:
            logger.debug("PnP Injecting %s at t=%s", self.kind, self.t)
        return fire


class ModifiedSpaAttnProcessor(_PnPAttnProcessor):
    kind = "Spa-Attn"


class ModifiedTmpAttnProcessor(_PnPAttnProcessor):
    kind = "Tmp-Attn"


def register_spatial_attention_pnp(model, injection_schedule):
    for res, blocks in _PNP_SITES.items():
        for block in blocks:
            module = model.unet.up_blocks[res].attentions[block].transformer_blocks[0].attn1
            module.processor = ModifiedSpaAttnProcessor(injection_schedule)


def register_temp_attention_pnp(model, injection_schedule):
    for res, blocks in _PNP_SITES.items():
        for block in blocks:
            module = model.unet.up_blocks[res].temp_attentions[block].transformer_blocks[0].attn1
            module.processor = ModifiedTmpAttnProcessor(injection_schedule)


#: spelling used by BASELINE.json's north_star
register_temporal_attention_pnp = register_temp_attention_pnp
