"""TEST INFRASTRUCTURE — the contracts of the kernel calls a PnP step replayed from a SourceFeatureCache makes, restated on top of
tests/kernel_contracts.py: attention with n_v = 2 (the two edit branches of the n_v = 3 call, which kernel_contracts states
directly), the fused temporal attention with Q / K from a separate source tensor, and GroupNorm with an explicit partition
(whose exact statistics do not depend on it).  ``patch_ops`` swaps them in next to the ``emulated_ops`` fixture;
tests/test_gpu_source_cache.py checks the kernels against them."""
from __future__ import annotations

import torch

import kernel_contracts as kc


attention = kc.attention
attention_exact = kc.attention_exact


def _tattn_qksrc_operands(x, qk_src, wqkv, heads, F_, HW, clips, out, scale):
    """the n_v = 2 operands of ``temporal_attention_fused_qksrc``: Q, K projected from the source clips, V from the edit clips
    [uncond | cond], each rounded to fp16 as the projection stores them"""
    assert x.dtype == qk_src.dtype == torch.float16
    assert clips % 2 == 0 and qk_src.shape[0] * 2 == x.shape[0] == clips * F_ * HW
    C = heads * 64
    qk = (qk_src.double() @ wqkv[:2 * C].double().t()).to(torch.float16)
    v = (x.double() @ wqkv[2 * C:].double().t()).to(torch.float16)
    src_rows = qk_src.shape[0]
    return ((qk[:, :C], qk[:, C:], v, heads, F_, (clips // 2) * HW, out),
            dict(scale=scale, n_v=2, v_branch_stride=src_rows * v.stride(0), o_branch_stride=src_rows * out.stride(0),
                 frames_mode=True, HW=HW))


def temporal_attention_fused_qksrc(x, qk_src, wqkv, heads, F_, HW, clips, out, scale=0.125):
    """the fused temporal attention with Q, K from a separate source tensor: ``attention`` at n_v = 2 on the fp16-rounded
    projections"""
    args, kw = _tattn_qksrc_operands(x, qk_src, wqkv, heads, F_, HW, clips, out, scale)
    return attention(*args, **kw)


def temporal_attention_fused_qksrc_exact(x, qk_src, wqkv, heads, F_, HW, clips, out, scale=0.125, cond=None):
    """the float64 values ``temporal_attention_fused_qksrc`` rounds to fp16 at the store, as ``attention_exact`` returns them"""
    args, kw = _tattn_qksrc_operands(x, qk_src, wqkv, heads, F_, HW, clips, out, scale)
    return attention_exact(*args, cond=cond, **kw)


def groupnorm(x, gamma, beta, groups, eps, silu, out=None, x2=None, partition_samples=0):
    """the exact statistics do not depend on how the kernel partitions the reduction"""
    assert partition_samples == 0 or partition_samples >= x.shape[0]
    return kc.groupnorm(x, gamma, beta, groups, eps, silu, out=out, x2=x2)


def patch_ops(monkeypatch):
    from anyv2v_b200 import ops
    for name in ("attention", "temporal_attention_fused_qksrc", "groupnorm"):
        monkeypatch.setattr(ops, name, globals()[name])
