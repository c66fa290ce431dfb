"""GPU parity tests, kernel level: each hand-written sm_90a kernel (called through the C ABI) against an fp32
PyTorch restatement of the same op on identical fp16 inputs; the DDIM step against the oracle bit for bit."""
import pytest
import torch

from parity_utils import assert_fp16_close

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def ops():
    from anyv2v_b200 import ops as o
    return o


def test_native_library_is_loaded(ops):
    from anyv2v_b200 import _lib
    import ctypes
    lib = _lib.lib()
    sm, maj, mnr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(lib.av2v_device_info(ctypes.byref(sm), ctypes.byref(maj), ctypes.byref(mnr)), "device_info")
    assert (maj.value, mnr.value) == (9, 0) and sm.value >= 100


@pytest.mark.parametrize("n", [8, 4 * 16 * 64 * 64, 1001])
def test_ddim_step_bit_exact_vs_oracle(ops, n):
    from oracle import schedulers_ref
    torch.manual_seed(n)
    n8 = n
    x, vn, ve = (torch.randn(n8, device=dev).half() for _ in range(3))
    for cls, inverse in ((schedulers_ref.DDIMScheduler, False), (schedulers_ref.DDIMInverseScheduler, True)):
        s = cls()
        s.set_timesteps(50)
        for t in (981, 501, 1):
            ca, cb, cc, cd = s.coefficients(t)
            if inverse:
                ref, _ = s.step(vn, t, x)
                got = ops.ddim_step(x, vn, None, 1.0, ca, cb, cc, cd, inverse=True)
            else:
                ref, _ = s.step(schedulers_ref.cfg_combine(vn, ve, 9.0), t, x)
                got = ops.ddim_step(x, vn, ve, 9.0, ca, cb, cc, cd)
            assert torch.equal(got, ref), f"ddim step differs at t={t} inverse={inverse}"


def test_ddim_step_empty_and_errors(ops):
    from anyv2v_b200._lib import Av2vError
    e = torch.empty(0, device=dev, dtype=torch.float16)
    assert ops.ddim_step(e, e, None, 1.0, 1, 0, 1, 0).numel() == 0
    with pytest.raises(Av2vError):
        ops.ddim_step(torch.zeros(8), torch.zeros(8), None, 1.0, 1, 0, 1, 0)  # CPU tensors: no fallback exists


@pytest.mark.parametrize("shape", [(6, 256, 2560, True, 1e-5), (4, 4096, 320, True, 1e-5), (2, 16384, 640, False, 1e-6),
                                   (3, 1024, 960, True, 1e-5), (3, 7, 64, True, 1e-5), (1, 2, 32, False, 1e-5)])
def test_groupnorm_silu(ops, shape):
    n, rows, C, silu, eps = shape
    torch.manual_seed(0)
    x = (torch.randn(n, rows, C, device=dev) * 2 + 0.5).half()
    g, b = torch.randn(C, device=dev).half(), torch.randn(C, device=dev).half()
    y = ops.groupnorm(x, g, b, 32, eps, silu)
    ref = torch.nn.functional.group_norm(x.float().permute(0, 2, 1), 32, g.float(), b.float(), eps)
    if silu:
        ref = torch.nn.functional.silu(ref.half().float())  # the reference rounds GN's output before SiLU
    assert_fp16_close(y, ref.permute(0, 2, 1), f"groupnorm {shape}")


@pytest.mark.parametrize("mnk", [(3, 1280, 320), (128, 160, 128), (1000, 320, 320), (4096, 1280, 1280), (777, 960, 320),
                                 (2048, 5120, 640), (512, 64, 4096), (256, 4096, 1024)])
def test_linear(ops, mnk):
    M, N, K = mnk
    torch.manual_seed(1)
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    bias = torch.randn(N, device=dev).half()
    res = torch.randn(M, N, device=dev).half()
    out = ops.linear(a, w, bias=bias, residual=res)
    assert_fp16_close(out, a.float() @ w.float().t() + bias.float() + res.float(), f"linear {mnk}")
    out2 = ops.linear(a, w)
    assert_fp16_close(out2, a.float() @ w.float().t(), f"linear-nobias {mnk}")


@pytest.mark.parametrize("mnk", [(100, 256, 64), (4096, 2560, 320), (1000, 5120, 640), (300, 128, 64)])
def test_linear_fused_geglu(ops, mnk):
    """FeedForward.net[0] (GEGLU): h * gelu_erf(gate) fused into the GEMM epilogue, with the reference's fp16 roundings."""
    M, N, K = mnk
    torch.manual_seed(11)
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    bias = torch.randn(N, device=dev).half()
    wp, bp = ops.geglu_pack(w, bias)
    out = ops.linear(a, wp, bias=bp, geglu=True)
    assert out.shape == (M, N // 2)
    h, gate = (a.float() @ w.float().t() + bias.float()).chunk(2, dim=-1)
    ref = h * torch.nn.functional.gelu(gate)
    assert_fp16_close(out, ref, f"geglu {mnk}", atol_frac=2e-3)


@pytest.mark.parametrize("shape", [(1000, 320), (4096, 640), (777, 1280), (50, 64), (3, 512), (9, 2048)])
def test_layernorm(ops, shape):
    rows, C = shape
    torch.manual_seed(12)
    x = (torch.randn(rows, C, device=dev) * 3 + 1).half()
    g, b = torch.randn(C, device=dev).half(), torch.randn(C, device=dev).half()
    y = ops.layernorm(x, g, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)
    assert_fp16_close(y, ref, f"layernorm {shape}")


def test_linear_strided_views(ops):
    torch.manual_seed(2)
    buf = torch.randn(300, 3 * 128, device=dev).half()
    a = buf[:, 128:256]  # row-strided view, as produced by a fused QKV projection
    w = (torch.randn(192, 128, device=dev) / 11).half()
    assert_fp16_close(ops.linear(a, w), a.float() @ w.float().t(), "linear strided A")


@pytest.mark.parametrize("geo", [(2, 16, 16, 64, 64), (3, 8, 8, 128, 160), (3, 16, 16, 2560, 1280), (2, 32, 32, 640, 640),
                                 (2, 64, 64, 320, 320), (2, 20, 24, 64, 64), (1, 40, 64, 64, 128), (5, 4, 4, 64, 64)])
def test_conv3x3(ops, geo):
    NF, H, W, Cin, Cout = geo
    torch.manual_seed(3)
    x = torch.randn(NF, H, W, Cin, device=dev).half()
    w = (torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5).half()
    bias, temb = torch.randn(Cout, device=dev).half(), torch.randn(NF, Cout, device=dev).half()
    out = ops.conv3x3(x, w.permute(0, 2, 3, 1).reshape(Cout, -1).contiguous(), bias=bias, rowbias=temb, rows_per_rowbias=H * W)
    ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float(), padding=1) + temb.float()[:, :, None, None]
    assert_fp16_close(out, ref.permute(0, 2, 3, 1), f"conv3x3 {geo}")


def test_conv3x3_inject_slots(ops):
    """fused conv + residual-copy: one accumulator tile stored to the three branch slots (pnp_utils.py:109-124)."""
    torch.manual_seed(4)
    n, H, W, C = 4, 16, 16, 128
    x = torch.randn(n, H, W, C, device=dev).half()
    w = (torch.randn(C, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    bias = torch.randn(C, device=dev).half()
    short = torch.randn(3, n, H, W, C, device=dev).half()
    out = torch.empty_like(short)
    ops.conv3x3(x, w.permute(0, 2, 3, 1).reshape(C, -1).contiguous(), bias=bias, residual=short, out=out, n_slots=3,
                slot_stride=n * H * W * C)
    h = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    assert_fp16_close(out, h[None] + short.float(), "conv3x3 3-slot")


@pytest.mark.parametrize("geo", [(1, 4, 64, 64), (2, 8, 256, 320), (3, 16, 256, 640), (1, 2, 64, 128), (2, 4, 4, 128), (1, 3, 100, 64)])
def test_temporal_conv(ops, geo):
    B, F, HW, C = geo
    torch.manual_seed(5)
    x = torch.randn(B, F * HW, C, device=dev).half()
    w = (torch.randn(C, C, 3, 1, 1, device=dev) / (3 * C) ** 0.5).half()
    bias, res = torch.randn(C, device=dev).half(), torch.randn(B, F * HW, C, device=dev).half()
    out = ops.tconv3(x, w[:, :, :, 0, 0].permute(0, 2, 1).reshape(C, -1).contiguous(), F, HW, bias=bias, residual=res)
    x5 = x.view(B, F, HW, 1, C).permute(0, 4, 1, 2, 3).float()
    ref = torch.nn.functional.conv3d(x5, w.float(), bias.float(), padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(B, F * HW, C)
    assert_fp16_close(out, ref + res.float(), f"tconv3 {geo}")


def _ref_attn(q, k, v, heads):
    B, N, C = q.shape
    sp = lambda t: t.float().view(B, -1, heads, 64).transpose(1, 2)
    p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * 0.125, dim=-1)
    return (p @ sp(v)).transpose(1, 2).reshape(B, N, C)


@pytest.mark.parametrize("case", [(1, 1, 128, 1, 1.0), (2, 2, 256, 1, 1.0), (1, 2, 256, 3, 1.0), (2, 2, 1024, 1, 3.0),
                                  (1, 1, 200, 1, 1.0), (1, 2, 880, 3, 1.0), (4, 5, 4096, 1, 1.0), (2, 5, 4096, 3, 1.0)])
def test_attention_rows(ops, case):
    batch, heads, seq, nv, mag = case
    torch.manual_seed(6)
    C = heads * 64
    nb = 3 if nv == 3 else 1
    qkv = (torch.randn(nb * batch * seq, 3 * C, device=dev) * mag).half()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    out = torch.zeros(nb * batch * seq, C, device=dev, dtype=torch.float16)
    rows = batch * seq
    if nv == 1:
        ops.attention(q, k, v, heads, seq, batch, out)
        ref = _ref_attn(q.reshape(batch, seq, C), k.reshape(batch, seq, C), v.reshape(batch, seq, C), heads)
    else:
        # injected step: q,k of the source chunk only; the reference result = every branch attends with the source q,k
        ops.attention(q[:rows], k[:rows], v, heads, seq, batch, out, n_v=3, v_branch_stride=rows * 3 * C, o_branch_stride=rows * C)
        qs, ks = q[:rows].reshape(batch, seq, C), k[:rows].reshape(batch, seq, C)
        ref = torch.cat([_ref_attn(qs, ks, v[i * rows:(i + 1) * rows].reshape(batch, seq, C), heads) for i in range(3)])
    assert_fp16_close(out.view(-1, seq, C), ref, f"attention rows {case}", atol_frac=2e-3)


@pytest.mark.parametrize("case", [(6, 2, 256, 145, 3), (4, 5, 1024, 145, 2), (2, 1, 64, 77, 1), (3, 2, 300, 64, 3),
                                  (4, 2, 200, 2100, 2)])  # long shared context: the two-threads-per-row kernel
def test_cross_attention_shared_context(ops, case):
    """attn2 of the spatial transformers: 145-token context, ONE context per clip shared by its frames (kv_batch_div)."""
    batch, heads, seq, nk, div = case
    torch.manual_seed(8)
    C = heads * 64
    q = torch.randn(batch * seq, C, device=dev).half()
    kv = torch.randn((batch // div) * nk, 2 * C, device=dev).half()
    out = torch.zeros(batch * seq, C, device=dev, dtype=torch.float16)
    ops.attention(q, kv[:, :C], kv[:, C:], heads, seq, batch, out, seq_kv=nk, kv_batch_div=div)
    k = kv[:, :C].reshape(batch // div, nk, C).repeat_interleave(div, dim=0)
    v = kv[:, C:].reshape(batch // div, nk, C).repeat_interleave(div, dim=0)
    sp = lambda t, n: t.float().view(batch, n, heads, 64).transpose(1, 2)
    p = torch.softmax(sp(q.reshape(batch, seq, C), seq) @ sp(k, nk).transpose(-1, -2) * 0.125, dim=-1)
    ref = (p @ sp(v, nk)).transpose(1, 2).reshape(batch * seq, C)
    assert_fp16_close(out, ref, f"cross attention {case}", atol_frac=2e-3)


@pytest.mark.parametrize("case", [(1, 1, 16, 64, 1), (2, 2, 16, 64, 3), (1, 2, 8, 256, 1), (1, 1, 128, 16, 1), (1, 1, 256, 8, 1),
                                  (3, 5, 16, 1024, 1), (1, 5, 16, 1024, 3), (1, 2, 4, 64, 1), (1, 1, 32, 32, 3), (2, 2, 4, 16, 1), (1, 1, 16, 4, 3)])
def test_attention_frames(ops, case):
    clips, heads, F, HW, nv = case
    torch.manual_seed(7)
    C = heads * 64
    nb = 3 if nv == 3 else 1
    x = torch.randn(nb * clips * F * HW, 3 * C, device=dev).half()
    q, k, v = x[:, :C], x[:, C:2 * C], x[:, 2 * C:]
    out = torch.zeros(nb * clips * F * HW, C, device=dev, dtype=torch.float16)
    to_seq = lambda t, n: t.reshape(n, F, HW, C).permute(0, 2, 1, 3).reshape(n * HW, F, C)
    from_seq = lambda t, n: t.reshape(n, HW, F, C).permute(0, 2, 1, 3).reshape(n * F * HW, C)
    rows = clips * F * HW
    if nv == 1:
        ops.attention(q, k, v, heads, F, clips * HW, out, frames_mode=True, HW=HW)
        ref = from_seq(_ref_attn(to_seq(q, clips), to_seq(k, clips), to_seq(v, clips), heads), clips)
    else:
        ops.attention(q[:rows], k[:rows], v, heads, F, clips * HW, out, n_v=3, v_branch_stride=rows * 3 * C,
                      o_branch_stride=rows * C, frames_mode=True, HW=HW)
        ref = torch.cat([from_seq(_ref_attn(to_seq(q[:rows], clips), to_seq(k[:rows], clips),
                                            to_seq(v[i * rows:(i + 1) * rows], clips), heads), clips) for i in range(3)])
    assert_fp16_close(out, ref, f"attention frames {case}", atol_frac=2e-3)


def test_bad_arguments_return_codes(ops):
    from anyv2v_b200._lib import Av2vError
    a = torch.randn(16, 12, device=dev).half()  # K = 12 is not a multiple of 8
    w = torch.randn(8, 12, device=dev).half()
    with pytest.raises(Av2vError, match="multiples of 8"):
        ops.linear(a, w)
    x = torch.randn(2, 8, 8, 48, device=dev).half()  # Cin not a multiple of 64
    with pytest.raises(Av2vError, match="Cin"):
        ops.conv3x3(x, torch.randn(64, 9 * 48, device=dev).half())


# ------------------------------------------------------------------------------------------------ round-2 kernels
def _ref_attn(q, k, v, heads, scale=0.125):
    B, N, C = q.shape
    sp = lambda t: t.float().view(B, -1, heads, 64).transpose(1, 2)
    p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * scale, dim=-1)
    return (p @ sp(v)).transpose(1, 2).reshape(B, N, C)


@pytest.mark.parametrize("case", [(1, 1, 128, 1.0), (2, 2, 256, 1.0), (2, 2, 1024, 3.0), (1, 1, 200, 1.0), (3, 2, 384, 1.0),
                                  (1, 2, 880, 2.0), (4, 5, 4096, 1.0), (1, 1, 64, 1.0), (2, 1, 300, 6.0),
                                  # long key loops: ragged tails, odd tile counts
                                  (2, 1, 2048, 1.0), (1, 2, 2100, 3.0), (1, 1, 2300, 6.0), (1, 3, 2176 + 64, 2.0)])
def test_attention_two_query_tiles_rows(ops, case):
    """plain (n_v = 1) rows-mode attention, 128 queries per CTA (csrc/attention_wgmma.cu): odd tile counts, ragged tails,
    large-magnitude scores (rescale path), against an fp32 restatement"""
    batch, heads, seq, mag = case
    torch.manual_seed(6)
    C = heads * 64
    qkv = (torch.randn(batch * seq, 3 * C, device=dev) * mag).half()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    out = torch.full((batch * seq, C), float("nan"), device=dev, dtype=torch.float16)
    ops.attention(q, k, v, heads, seq, batch, out)
    ref = _ref_attn(q.reshape(batch, seq, C), k.reshape(batch, seq, C), v.reshape(batch, seq, C), heads)
    assert_fp16_close(out.view(-1, seq, C), ref, f"attention2q rows {case}", atol_frac=2e-3)


@pytest.mark.parametrize("seq", [1024, 3072])
def test_attention_two_query_tiles_rescale_path(ops, seq):
    """keys whose scores grow along the sequence force the running max up again and again: O and the row sum are rescaled in
    registers on every raise"""
    torch.manual_seed(9)
    batch, heads = 1, 1
    q = torch.randn(batch * seq, 64, device=dev).half()
    ramp = torch.linspace(0.2, 6.0, seq, device=dev).view(seq, 1)
    k = (torch.randn(seq, 64, device=dev) * ramp).half()
    v = torch.randn(seq, 64, device=dev).half()
    out = torch.empty(seq, 64, device=dev, dtype=torch.float16)
    ops.attention(q, k, v, heads, seq, batch, out, scale=1.0)
    ref = _ref_attn(q.view(1, seq, 64), k.view(1, seq, 64), v.view(1, seq, 64), heads, scale=1.0)
    assert_fp16_close(out.view(1, seq, 64), ref, "attention2q rescale path", atol_frac=2e-3)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("case", [(3, 5, 16, 4096, 320), (1, 8, 16, 4096, 512), (2, 10, 16, 1024, 640), (3, 20, 16, 256, 1280), (1, 2, 8, 256, 128),
                                  (1, 1, 128, 16, 64), (2, 2, 4, 16, 128), (1, 2, 16, 100, 128), (1, 1, 32, 7, 64),
                                  # ragged pixel tiles, 2 and 5 k-blocks, 8 heads x 320
                                  (2, 5, 16, 1001, 320), (4, 2, 16, 2048, 128), (1, 8, 16, 4096, 320), (1, 5, 128, 160, 320), (2, 3, 8, 1024, 192)])
def test_temporal_attention_fused(ops, case, nv):
    """Q/K/V projection + temporal attention in ONE launch (csrc/attention_wgmma.cu, pnp_utils.py:247-334) vs the
    two-kernel path (same rounding points: Q, K, V to fp16, P to fp16) and vs an fp32 restatement.  nv = 3: PnP-injected
    (clips = [source | uncond | cond] x `clips` each; Q, K of every branch from the source clip, pnp_utils.py:295-302)."""
    clips, heads, F, HW, Cx = case
    torch.manual_seed(13)
    C = heads * 64
    nclips = clips * nv
    rows = nclips * F * HW
    x = torch.randn(rows, Cx, device=dev).half()
    w = (torch.randn(3 * C, Cx, device=dev) / Cx ** 0.5).half()
    out = torch.full((rows, C), float("nan"), device=dev, dtype=torch.float16)
    ops.temporal_attention_fused(x, w, heads, F, HW, nclips, out, n_v=nv)
    qkv = ops.linear(x, w)
    base = torch.empty_like(out)
    src = clips * F * HW
    if nv == 1:
        ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], heads, F, nclips * HW, base, frames_mode=True, HW=HW)
    else:
        ops.attention(qkv[:src, :C], qkv[:src, C:2 * C], qkv[:, 2 * C:], heads, F, clips * HW, base, n_v=3, frames_mode=True, HW=HW,
                      v_branch_stride=src * qkv.stride(0), o_branch_stride=src * C)
    to_seq = lambda t, n: t.reshape(n, F, HW, C).permute(0, 2, 1, 3).reshape(n * HW, F, C)
    from_seq = lambda t, n: t.reshape(n, HW, F, C).permute(0, 2, 1, 3).reshape(n * F * HW, C)
    q16 = (x.float() @ w.float().t()).half()
    if nv == 1:
        ref = from_seq(_ref_attn(to_seq(q16[:, :C], nclips), to_seq(q16[:, C:2 * C], nclips), to_seq(q16[:, 2 * C:], nclips), heads), nclips)
    else:
        ref = torch.cat([from_seq(_ref_attn(to_seq(q16[:src, :C], clips), to_seq(q16[:src, C:2 * C], clips),
                                            to_seq(q16[i * src:(i + 1) * src, 2 * C:], clips), heads), clips) for i in range(3)])
    assert_fp16_close(out, ref, f"fused temporal attention {case} nv={nv}", atol_frac=2e-3)
    assert_fp16_close(out, base.float(), f"fused temporal attention vs two kernels {case} nv={nv}", atol_frac=2e-3)


@pytest.mark.parametrize("shape", [(196608 // 4, 320), (1001, 320), (3, 640), (49152 // 4, 640), (12288, 1280), (7, 1280), (100, 64), (33, 2048)])
def test_layernorm_shapes(ops, shape):
    """C = 40 * LPR vectors -> the five-vectors-per-lane kernel; other widths -> the one-warp-per-row fallback"""
    rows, C = shape
    torch.manual_seed(2)
    x = (torch.randn(rows, C, device=dev) * 3 + 0.7).half()
    g, b = (1 + 0.2 * torch.randn(C, device=dev)).half(), (0.2 * torch.randn(C, device=dev)).half()
    got = ops.layernorm(x, g, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)
    assert_fp16_close(got, ref, f"layernorm {shape}")


@pytest.mark.parametrize("shape", [(6, 256, 2560, True, 1e-5), (4, 4096, 320, True, 1e-5), (2, 16384, 640, False, 1e-6), (3, 1024, 960, True, 1e-5),
                                   (3, 7, 64, True, 1e-5), (1, 2, 32, False, 1e-5), (1, 65536, 320, True, 1e-5), (3, 65536, 320, False, 1e-6),
                                   (48, 1024, 640, True, 1e-5), (1, 1000, 1280, True, 1e-5), (48, 4096, 320, True, 1e-5), (16, 4096, 960, True, 1e-5),
                                   (2, 4, 128, True, 1e-5), (5, 64, 1920, True, 1e-5), (1, 16 * 4096, 512, True, 1e-6), (50, 300, 320, False, 1e-5)])
def test_groupnorm_persistent_kernel(ops, shape):
    """the persistent L2-chunked GroupNorm(+SiLU) kernel (csrc/groupnorm.cu): one chunk, many chunks (48 frames), ragged slices,
    tiny samples, samples wider than a stage, back-to-back launches (grid-barrier state is reset by the kernel itself)"""
    n, rows, C, silu, eps = shape
    torch.manual_seed(0)
    x = (torch.randn(n, rows, C, device=dev) * 2 + 0.5).half()
    g, b = (1 + 0.2 * torch.randn(C, device=dev)).half(), (0.2 * torch.randn(C, device=dev)).half()
    got = ops.groupnorm(x, g, b, 32, eps, silu)
    again = ops.groupnorm(x, g, b, 32, eps, silu)
    ref = torch.nn.functional.group_norm(x.float().transpose(1, 2), 32, g.float(), b.float(), eps).transpose(1, 2)
    if silu:
        ref = torch.nn.functional.silu(ref.half().float())
    assert_fp16_close(got, ref, f"groupnorm {shape}", atol_frac=2e-3)
    assert torch.equal(got, again), "groupnorm is deterministic (fixed-order partial sums)"


def test_groupnorm_sample_larger_than_l2(ops):
    """a 128-frame clip at the 64 x 64 level: one sample = 336 MB > L2; phase B re-reads from HBM, results unchanged"""
    n, rows, C = 1, 128 * 4096, 320
    torch.manual_seed(1)
    x = (torch.randn(n, rows, C, device=dev) * 1.5 - 0.3).half()
    g, b = (1 + 0.2 * torch.randn(C, device=dev)).half(), (0.2 * torch.randn(C, device=dev)).half()
    got = ops.groupnorm(x, g, b, 32, 1e-5, True)
    ref = torch.nn.functional.silu(torch.nn.functional.group_norm(x.float().transpose(1, 2), 32, g.float(), b.float(), 1e-5)
                                   .transpose(1, 2).half().float())
    assert_fp16_close(got, ref, "groupnorm 128-frame clip", atol_frac=2e-3)


@pytest.mark.parametrize("geo", [(48, 64, 64, 320, 320), (6, 32, 32, 640, 640), (4, 16, 16, 1280, 1280), (3, 8, 8, 128, 64), (5, 4, 4, 64, 128), (2, 2, 2, 64, 64)])
def test_conv3x3_stride2(ops, geo):
    """Downsample2D (Conv 3x3, stride 2, pad 1; diffusers downsampling.py, twin at seine/models/resnet.py:79-110): every A row
    gathers the taps of one output pixel at twice its coordinates with cp.async; out-of-image taps are zero-filled"""
    NF, H, W, Cin, Cout = geo
    torch.manual_seed(11)
    x = torch.randn(NF, H, W, Cin, device=dev).half()
    w = (torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5).half()
    b = (0.1 * torch.randn(Cout, device=dev)).half()
    got = ops.conv3x3(x, w.permute(0, 2, 3, 1).reshape(Cout, -1).contiguous(), bias=b, stride=2)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), stride=2, padding=1).permute(0, 2, 3, 1)
    assert got.shape == (NF, H // 2, W // 2, Cout)
    assert_fp16_close(got, ref, f"conv3x3 stride 2 {geo}")


@pytest.mark.parametrize("geo", [(48, 64, 64, 8, 320), (4, 16, 16, 8, 64), (3, 32, 32, 24, 128), (16, 64, 64, 320, 4), (2, 16, 16, 64, 4)])
def test_conv3x3_padded_channels(ops, geo):
    """conv_in (8 -> 320: K blocks zero-padded to 64 channels, the cp.async channel predicate zero-fills the missing ones) and conv_out (320 -> 4:
    weight rows zero-padded to 8, result sliced) through the product module"""
    from anyv2v_b200.unet_i2vgen_xl import Conv3x3
    NF, H, W, Cin, Cout = geo
    torch.manual_seed(12)
    conv = Conv3x3(Cin, Cout).to(device=dev, dtype=torch.float16)
    x = torch.randn(NF, H, W, Cin, device=dev).half()
    got = conv.forward_nhwc(x)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), conv.weight.float(), conv.bias.float(), padding=1).permute(0, 2, 3, 1)
    assert got.shape == (NF, H, W, Cout)
    assert_fp16_close(got, ref, f"conv3x3 padded channels {geo}")


@pytest.mark.parametrize("mnk", [(196608 // 8, 320, 640, 320), (49152 // 4, 640, 1280, 640), (12288, 1280, 1280, 1280), (3072, 1280, 1280, 1280), (1000, 64, 64, 192), (130, 8, 128, 64)])
def test_linear_two_source_k_loop(ops, mnk):
    """the skip-connection concat as a two-source K loop: linear([a | a2]) without materialising torch.cat (1x1 shortcut of the
    up-block resnets, pnp_utils.py:117-122 for the patched one)"""
    M, N, K1, K2 = mnk
    torch.manual_seed(13)
    a = torch.randn(M, K1, device=dev).half()
    a2 = torch.randn(M, K2, device=dev).half()
    w = (torch.randn(N, K1 + K2, device=dev) / (K1 + K2) ** 0.5).half()
    b = (0.1 * torch.randn(N, device=dev)).half()
    got = ops.linear(a, w, bias=b, a2=a2)
    base = ops.linear(torch.cat([a, a2], dim=1), w, bias=b)
    ref = torch.cat([a, a2], dim=1).float() @ w.float().t() + b.float()
    assert_fp16_close(got, ref, f"two-source linear {mnk}")
    assert torch.equal(got, base), "same k-block order -> bit-identical to the concatenated GEMM"


@pytest.mark.parametrize("shape", [(48, 4096, 640, 320, True), (3, 1024, 1280, 640, True), (6, 256, 1280, 1280, True), (2, 64, 1280, 1280, False),
                                   (16, 4096, 320, 320, True), (3, 300, 64, 64, True), (1, 7, 128, 64, False)])
def test_groupnorm_two_sources(ops, shape):
    """norm1 of the up-block resnets normalises torch.cat([hidden, skip], dim=1) (pnp_utils.py:48 on the concatenated input): the
    kernel reads the two sources and writes the normalised concat — bit-identical to normalising the materialised cat"""
    n, rows, C1, C2, silu = shape
    torch.manual_seed(5)
    x1 = (torch.randn(n, rows, C1, device=dev) * 2 + 0.5).half()
    x2 = (torch.randn(n, rows, C2, device=dev) * 0.7 - 0.2).half()
    C = C1 + C2
    g, b = (1 + 0.2 * torch.randn(C, device=dev)).half(), (0.2 * torch.randn(C, device=dev)).half()
    got = ops.groupnorm(x1, g, b, 32, 1e-5, silu, x2=x2)
    cat = torch.cat([x1, x2], dim=2)
    base = ops.groupnorm(cat, g, b, 32, 1e-5, silu)
    ref = torch.nn.functional.group_norm(cat.float().transpose(1, 2), 32, g.float(), b.float(), 1e-5).transpose(1, 2)
    if silu:
        ref = torch.nn.functional.silu(ref.half().float())
    assert got.shape == (n, rows, C)
    assert_fp16_close(got, ref, f"two-source groupnorm {shape}", atol_frac=2e-3)
    assert torch.equal(got, base), "same partial sums in the same order -> bit-identical to the concatenated input"


@pytest.mark.parametrize("geo", [(48, 32, 32, 640), (48, 16, 16, 1280), (48, 8, 8, 1280), (6, 8, 8, 64), (3, 16, 16, 128), (5, 4, 4, 64), (2, 2, 2, 128), (4, 32, 32, 64)])
def test_upsample2x_conv3x3_fused(ops, geo):
    """Upsample2D (nearest x 2 + conv 3x3) as four 2 x 2 phase convolutions on the low-resolution input, against the literal
    F.interpolate(scale_factor=2, mode='nearest') -> conv2d of the reference stack (SURVEY A.7)"""
    NF, H, W, C = geo
    torch.manual_seed(21)
    x = torch.randn(NF, H, W, C, device=dev).half()
    w = (torch.randn(C, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    b = (0.1 * torch.randn(C, device=dev)).half()
    got = ops.upsample2x_conv3x3(x, ops.pack_upsample_weights(w), bias=b)
    up = torch.nn.functional.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    ref = torch.nn.functional.conv2d(up, w.float(), b.float(), padding=1).permute(0, 2, 3, 1)
    assert got.shape == (NF, 2 * H, 2 * W, C)
    assert_fp16_close(got, ref, f"fused upsample conv {geo}", atol_frac=2e-3)
