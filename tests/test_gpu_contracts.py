"""GPU tests of every C-ABI kernel against its float64 contract (tests/kernel_contracts.py), inside guarded buffers.

Each case runs the ``ops`` wrapper on CUDA views placed in guarded buffers (tests/guarded.py: NaN around and between the rows
of inputs, a poison pattern around outputs), and the matching ``kernel_contracts`` function on CPU copies of the same buffers,
with the same views and strides.  Outputs are compared with ``assert_fp16_close`` (the DDIM step bit for bit), and the
memory around every output is checked for stray writes and unwritten elements.  So these tests tie the kernels to the
contract the CPU model tests run on, and they target the edges of the cp.async predicates and epilogue indexing: ragged
M / N / K tails, out-of-image taps, padded channels, rows past the last key, row strides wider than the data.
"""
import pytest
import torch

import kernel_contracts as kc
from guarded import GUARD, Guarded, check_output, guarded_inout, guarded_input, guarded_output
from parity_utils import assert_fp16_close

pytestmark = pytest.mark.gpu
dev = "cuda"


def rnd(*shape, scale=1.0, shift=0.0):
    return (torch.randn(*shape) * scale + shift).half()


def gin(values, ld=None, strides=None, guard=GUARD):
    return guarded_input(values, ld=ld, strides=strides, device=dev, guard=guard)


def gout(shape, ld=None, strides=None, guard=GUARD):
    return guarded_output(shape, ld=ld, strides=strides, device=dev, guard=guard)


def _run(name, args, kwargs, outs, atol_frac=1e-3, exact=False):
    """ops.<name> on the guarded CUDA views; kernel_contracts.<name> on CPU copies of the same buffers, taken before the
    kernel runs (in-place operands); then the guards of both and the outputs against each other"""
    from anyv2v_b200 import ops
    host = {}

    def on_host(v):
        if isinstance(v, Guarded):
            if id(v) not in host:
                host[id(v)] = v.to("cpu")
            return host[id(v)].view
        return v.cpu() if isinstance(v, torch.Tensor) else v

    on_dev = lambda v: v.view if isinstance(v, Guarded) else v
    h_args, h_kwargs = [on_host(a) for a in args], {k: on_host(v) for k, v in kwargs.items()}
    getattr(ops, name)(*[on_dev(a) for a in args], **{k: on_dev(v) for k, v in kwargs.items()})
    torch.cuda.synchronize()
    getattr(kc, name)(*h_args, **h_kwargs)
    for i, g in enumerate(outs):
        what = f"{name} output {i}"
        ref = host[id(g)]
        check_output(g, what)
        check_output(ref, what + " (contract)")
        got = g.view.cpu()
        if exact:
            assert torch.equal(got, ref.view), f"{what}: differs from the contract"
        elif got.numel():
            assert_fp16_close(got, ref.view, what, atol_frac=atol_frac)


def _w(n, k):
    return rnd(n, k, scale=k ** -0.5)


# ------------------------------------------------------------------------------------------------------------- linear
@pytest.mark.parametrize("mnk", [(1, 8, 8), (77, 136, 24), (129, 200, 72), (257, 64, 200), (130, 384, 1032)])
def test_linear_k_tail(mnk):
    """K % 64 != 0 (the kval predicate of the A and B loads), K < 64, ragged M and N, lda > K with a NaN gap"""
    M, N, K = mnk
    torch.manual_seed(M)
    a = gin(rnd(M, K), ld=K + 8, guard=128 * (K + 8))
    w = gin(_w(N, K), guard=128 * K)
    out = gout((M, N), ld=N + 8)
    _run("linear", [a, w], dict(bias=gin(rnd(N)), out=out), [out])


@pytest.mark.parametrize("epi", ["bias", "rowbias1", "rowbias7", "rowbiasM", "residual", "all"])
def test_linear_epilogue(epi):
    """bias / rowbias / residual alone and together, out and residual with ldo > N"""
    M, N, K = 203, 264, 128
    torch.manual_seed(3)
    ldo = N + 24
    a, w, out = gin(rnd(M, K)), gin(_w(N, K)), gout((M, N), ld=ldo)
    kw = dict(out=out)
    if epi in ("bias", "all"):
        kw["bias"] = gin(rnd(N))
    if epi.startswith("rowbias") or epi == "all":
        rpr = {"rowbias1": 1, "rowbias7": 7, "rowbiasM": M, "all": 7}[epi]
        kw.update(rowbias=gin(rnd(-(-M // rpr), N)), rows_per_rowbias=rpr)
    if epi in ("residual", "all"):
        kw["residual"] = gin(rnd(M, N), ld=ldo)
    _run("linear", [a, w], kw, [out])


@pytest.mark.parametrize("N", [192, 320])
def test_linear_geglu_half_tile(N):
    """N % 128 == 64: the last tile holds one h / gate group; ragged M, strided A, ldo > N/2"""
    from anyv2v_b200 import ops
    M, K = 77, 128
    torch.manual_seed(N)
    wp, bp = ops.geglu_pack(_w(N, K), rnd(N))
    a, out = gin(rnd(M, K), ld=K + 16, guard=128 * (K + 16)), gout((M, N // 2), ld=N // 2 + 8)
    _run("linear", [a, gin(wp, guard=128 * K)], dict(bias=gin(bp), out=out, geglu=True), [out])


@pytest.mark.parametrize("K2", [24, 72])
def test_linear_two_source_ragged(K2):
    """two-source K loop with k_split = 64 and a second source that is not a multiple of 64 wide, NaN gaps after both"""
    M, N = 150, 136
    torch.manual_seed(K2)
    a = gin(rnd(M, 64), ld=72, guard=128 * 72)
    a2 = gin(rnd(M, K2), ld=K2 + 8, guard=128 * (K2 + 8))
    out = gout((M, N))
    _run("linear", [a, gin(_w(N, 64 + K2))], dict(bias=gin(rnd(N)), out=out, a2=a2), [out])


# ------------------------------------------------------------------------------------------------------------- conv
def _image(NF, H, W, C):
    """channels-last image with NaN guards reaching past the top-left and bottom-right taps"""
    return gin(rnd(NF, H, W, C), guard=(W + 2) * C)


@pytest.mark.parametrize("rpr", ["frame", 5])
def test_conv3x3_stride2_epilogue(rpr):
    """stride 2 with rowbias and residual, out / residual with ldo > Cout, a ragged N tile"""
    NF, H, W, C, Cout = 3, 8, 6, 64, 136
    Ho, Wo = H // 2, W // 2
    M = NF * Ho * Wo
    rpr = Ho * Wo if rpr == "frame" else rpr
    torch.manual_seed(5)
    out = gout((NF, Ho, Wo, Cout), ld=Cout + 8)
    kw = dict(bias=gin(rnd(Cout)), rowbias=gin(rnd(-(-M // rpr), Cout)), rows_per_rowbias=rpr,
              residual=gin(rnd(NF, Ho, Wo, Cout), ld=Cout + 8), out=out, stride=2)
    _run("conv3x3", [_image(NF, H, W, C), gin(_w(Cout, 9 * C))], kw, [out])


def test_conv3x3_stride2_slots():
    """stride 2 with n_slots = 3 and a guarded gap between the slots of out and residual"""
    NF, H, W, C = 2, 8, 8, 64
    M = NF * (H // 2) * (W // 2)
    ss = M * C + 64
    torch.manual_seed(6)
    out = gout((3, M, C), strides=(ss, C, 1))
    kw = dict(bias=gin(rnd(C)), residual=gin(rnd(3, M, C), strides=(ss, C, 1)), out=out, n_slots=3, slot_stride=ss, stride=2)
    _run("conv3x3", [_image(NF, H, W, C), gin(_w(C, 9 * C))], kw, [out])


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("chan", [8, 24])
def test_conv3x3_padded_channels(chan, stride):
    """chan channels present, 64 declared: the missing channels of every K block must read as zeros (the padded weights are
    random here, so a read of anything else shows)"""
    NF, H, W, Cout = 2, 6, 6, 72
    torch.manual_seed(chan + stride)
    out = gout((NF, H // stride, W // stride, Cout))
    _run("conv3x3", [_image(NF, H, W, chan), gin(_w(Cout, 9 * 64))], dict(bias=gin(rnd(Cout)), out=out, stride=stride), [out])


@pytest.mark.parametrize("hw", [(1, 1), (1, 7), (7, 1)])
def test_conv3x3_thin_images(hw):
    """images of one row or one column: every tap but the centre row / column is outside the image"""
    H, W = hw
    NF, C = 3, 64
    torch.manual_seed(H * 8 + W)
    out = gout((NF, H, W, C))
    _run("conv3x3", [_image(NF, H, W, C), gin(_w(C, 9 * C))], dict(bias=gin(rnd(C)), out=out), [out])


@pytest.mark.parametrize("hw", [(1, 1), (1, 5)])
@pytest.mark.parametrize("cio", [(64, 128), (128, 64)])
def test_upsample2x_conv3x3_edges(cio, hw):
    """Cin != Cout, 1 x 1 and 1 x 5 inputs, no bias, out with ldo > Cout"""
    from anyv2v_b200 import ops
    (Cin, Cout), (H, W) = cio, hw
    NF = 2
    torch.manual_seed(Cin + W)
    wph = ops.pack_upsample_weights(rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    out = gout((NF, 2 * H, 2 * W, Cout), ld=Cout + 8)
    _run("upsample2x_conv3x3", [_image(NF, H, W, Cin), gin(wph)], dict(out=out), [out])


@pytest.mark.parametrize("F", [1, 2, 3])
def test_tconv3_frame_edges(F):
    """F <= 3 at HW = 1: the taps for frames -1 and F land in the NaN guards (clip 0, last clip) or the neighbouring clip;
    residual without bias, out / residual with ldo > Cout"""
    B, HW, C = 2, 1, 64
    torch.manual_seed(F)
    out = gout((B, F * HW, C), ld=C + 8)
    x = gin(rnd(B, F * HW, C), guard=(HW + 1) * C)
    _run("tconv3", [x, gin(_w(C, 3 * C)), F, HW], dict(residual=gin(rnd(B, F * HW, C), ld=C + 8), out=out), [out])


# ------------------------------------------------------------------------------------------------------------- attention
def _branches(rows, C, nv, gap=64):
    """nv branches of V rows with `gap` NaN rows between them -> (values, branch stride in rows)"""
    if nv == 1:
        return rnd(rows, C), 0
    nan = torch.full((gap, C), float("nan"), dtype=torch.float16)
    parts = [rnd(rows, C), nan, rnd(rows, C), nan, rnd(rows, C)]
    return torch.cat(parts), rows + gap


@pytest.mark.parametrize("case", [
    # batch, heads, seq, seq_kv, kv_batch_div, n_v, scale
    *[(2, 2, 100, nk, 1, 1, 0.125) for nk in (1, 8, 63, 64, 65, 145)],
    (4, 2, 70, 145, 2, 3, 0.125),
    (2, 1, 130, 0, 1, 3, 0.3),
], ids=lambda c: "b{}h{}s{}kv{}div{}nv{}sc{}".format(*c))
def test_attention_rows_guarded(case):
    """ragged key tiles with NaN rows after the last key and value, ldq != ldk != ldv != ldo (all > C), n_v = 3 with a NaN gap
    between the V branches and kv_batch_div > 1, scale != 0.125"""
    batch, heads, seq, seq_kv, div, nv, scale = case
    C = heads * 64
    ldq, ldk, ldv, ldo = C + 8, C + 16, C + 24, C + 40
    kv_rows = batch // div * (seq_kv if seq_kv else seq)
    torch.manual_seed(seq + seq_kv)
    vvals, vstride = _branches(kv_rows, C, nv)
    q = gin(rnd(batch * seq, C), ld=ldq, guard=128 * ldq)
    k = gin(rnd(kv_rows, C), ld=ldk, guard=64 * ldk)
    v = gin(vvals, ld=ldv, guard=64 * ldv)
    out = gout((nv * batch * seq, C), ld=ldo)
    kw = dict(scale=scale, n_v=nv, v_branch_stride=vstride * ldv, o_branch_stride=batch * seq * ldo if nv == 3 else 0,
              seq_kv=seq_kv, kv_batch_div=div)
    _run("attention", [q, k, v, heads, seq, batch, out], kw, [out], atol_frac=2e-3)


@pytest.mark.parametrize("geo", [*[(2, 2, F, HW, nv) for F, HW in ((1, 130), (2, 65), (64, 3)) for nv in (1, 3)],
                                 (1, 1, 256, 2, 3), (2, 1, 384, 1, 3)],
                         ids=lambda g: "clips{}h{}F{}HW{}nv{}".format(*g))
def test_attention_frames_guarded(geo):
    """packed frames at F = 1, 2, 64 with a ragged pixel tile, n_v 1 and 3; unpacked F = 256, 384 at n_v = 3 (the path of an
    injected step on clips of 256 frames or more)"""
    clips, heads, F, HW, nv = geo
    C = heads * 64
    ld = C + 8
    rows = clips * F * HW
    torch.manual_seed(F * 10 + nv)
    vvals, vstride = _branches(rows, C, nv)
    q, k = gin(rnd(rows, C), ld=ld, guard=128 * ld), gin(rnd(rows, C), ld=ld, guard=128 * ld)
    v = gin(vvals, ld=ld + 8, guard=128 * (ld + 8))
    out = gout((nv * rows, C), ld=ld + 16)
    kw = dict(n_v=nv, v_branch_stride=vstride * (ld + 8), o_branch_stride=rows * (ld + 16) if nv == 3 else 0,
              frames_mode=True, HW=HW)
    _run("attention", [q, k, v, heads, F, clips * HW, out], kw, [out], atol_frac=2e-3)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("F,HW", [(1, 130), (2, 65), (64, 3)])
def test_temporal_attention_fused_guarded(F, HW, nv):
    """F <= 2 and F = 64 (the kt = wg boundary), Cx = 64 (one k-block), ldx > Cx with a NaN gap, ldo > C, scale 0.3"""
    heads, Cx, src = 2, 64, 2
    C = heads * 64
    clips = src * nv
    rows = clips * F * HW
    torch.manual_seed(F + nv)
    x = gin(rnd(rows, Cx), ld=Cx + 8, guard=128 * (Cx + 8))
    out = gout((rows, C), ld=C + 8)
    _run("temporal_attention_fused", [x, gin(_w(3 * C, Cx)), heads, F, HW, clips, out], dict(scale=0.3, n_v=nv), [out],
         atol_frac=2e-3)


# ------------------------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("shape", [(3, 37, 320, True), (2, 1, 64, False), (1, 1, 640, True)])
def test_groupnorm_guarded(shape):
    n, rows, C, silu = shape
    torch.manual_seed(rows + C)
    out = gout((n, rows, C))
    args = [gin(rnd(n, rows, C, scale=2.0, shift=0.5)), gin(rnd(C, scale=0.2, shift=1.0)), gin(rnd(C, scale=0.2)), 32, 1e-5, silu]
    _run("groupnorm", args, dict(out=out), [out])


@pytest.mark.parametrize("rows", [0, 1, 37])
@pytest.mark.parametrize("C", [160, 960])
def test_layernorm_guarded(C, rows):
    """C = 160 and 960 (24 lanes per row of 40 vectors: the one-warp kernel with 5 vectors per lane); rows = 0 launches
    nothing and leaves out untouched"""
    torch.manual_seed(C + rows)
    out = gout((rows, C))
    args = [gin(rnd(rows, C, scale=3.0, shift=1.0)), gin(rnd(C, scale=0.2, shift=1.0)), gin(rnd(C, scale=0.2)), 1e-5]
    _run("layernorm", args, dict(out=out), [out])


# ------------------------------------------------------------------------------------------------------------- DDIM
_COEF = (0.5477226, 0.8366600, 0.7071068, 0.7071068)  # sqrt(a_t), sqrt(1 - a_t), sqrt(a_prev), sqrt(1 - a_prev); a_t = 0.3


@pytest.mark.parametrize("cfg", [False, True])
def test_ddim_coef_dev(cfg):
    """coefficients read from device memory instead of the (deliberately different) by-value fields"""
    n = 1001
    torch.manual_seed(int(cfg))
    coef = torch.tensor([*_COEF, 9.0], dtype=torch.float32, device=dev)
    out = gout((n,))
    args = [gin(rnd(n)), gin(rnd(n)), gin(rnd(n)) if cfg else None, 1.0, 1.0, 0.0, 1.0, 0.0]
    _run("ddim_step", args, dict(out=out, coef_dev=coef), [out], exact=True)


@pytest.mark.parametrize("n", [7, 8, 1001])
def test_ddim_in_place(n):
    """out is x, as the pipeline calls it: bit-exact against the contract and against the out-of-place result"""
    from anyv2v_b200 import ops
    torch.manual_seed(n)
    x, vn, ve = guarded_inout(rnd(n).to(dev)), gin(rnd(n)), gin(rnd(n))
    separate = gout((n,))
    ops.ddim_step(x.view, vn.view, ve.view, 9.0, *_COEF, out=separate.view)
    _run("ddim_step", [x, vn, ve, 9.0, *_COEF], dict(out=x), [x], exact=True)
    assert torch.equal(x.view, separate.view), "in-place result differs from the out-of-place one"


# ------------------------------------------------------------------------------------------------------------- wrapper refusals
def _h(*shape):
    return torch.zeros(*shape, dtype=torch.float16, device=dev)


def _conv_args():
    return _h(2, 4, 4, 64), _h(64, 9 * 64)


REFUSALS = {
    "linear out too narrow": lambda o: o.linear(_h(16, 64), _h(32, 64), out=_h(16, 24)),
    "linear out too few rows": lambda o: o.linear(_h(16, 64), _h(32, 64), out=_h(8, 32)),
    "linear out column-strided": lambda o: o.linear(_h(16, 64), _h(32, 64), out=_h(32, 16).t()),
    "linear residual row stride": lambda o: o.linear(_h(16, 64), _h(32, 64), out=_h(16, 40)[:, :32], residual=_h(16, 32)),
    "linear residual too small": lambda o: o.linear(_h(16, 64), _h(32, 64), residual=_h(8, 32)),
    "linear bias length": lambda o: o.linear(_h(16, 64), _h(32, 64), bias=_h(24)),
    "linear rowbias rows": lambda o: o.linear(_h(16, 64), _h(32, 64), rowbias=_h(3, 32), rows_per_rowbias=8),
    "linear rowbias strided": lambda o: o.linear(_h(16, 64), _h(32, 64), rowbias=_h(2, 40)[:, :32], rows_per_rowbias=8),
    "linear rowbias without rows": lambda o: o.linear(_h(16, 64), _h(32, 64), rowbias=_h(2, 32)),
    "conv3x3 out shape": lambda o: o.conv3x3(*_conv_args(), out=_h(2, 4, 3, 64)),
    "conv3x3 out frame gap": lambda o: o.conv3x3(*_conv_args(), out=_h(2, 5, 4, 64)[:, :4]),
    "conv3x3 residual layout": lambda o: o.conv3x3(*_conv_args(), residual=_h(2, 4, 4, 72)[..., :64]),
    "conv3x3 slots in one slot": lambda o: o.conv3x3(*_conv_args(), out=_h(2, 4, 4, 64), n_slots=3, slot_stride=2048),
    "conv3x3 slot stride": lambda o: o.conv3x3(*_conv_args(), out=_h(3, 32, 64), n_slots=3, slot_stride=4096),
    "conv3x3 bias length": lambda o: o.conv3x3(*_conv_args(), bias=_h(72)),
    "conv3x3 rowbias rows": lambda o: o.conv3x3(*_conv_args(), rowbias=_h(1, 64), rows_per_rowbias=16),
    "upsample out shape": lambda o: o.upsample2x_conv3x3(_h(1, 2, 2, 64), _h(4, 64, 256), out=_h(1, 4, 2, 64)),
    "upsample bias length": lambda o: o.upsample2x_conv3x3(_h(1, 2, 2, 64), _h(4, 64, 256), bias=_h(128)),
    "tconv3 out shape": lambda o: o.tconv3(_h(1, 8, 64), _h(64, 192), 2, 4, out=_h(1, 4, 64)),
    "tconv3 residual layout": lambda o: o.tconv3(_h(1, 8, 64), _h(64, 192), 2, 4, residual=_h(1, 8, 72)[..., :64]),
    "groupnorm out strided": lambda o: o.groupnorm(_h(1, 4, 64), _h(64), _h(64), 32, 1e-5, False, out=_h(1, 4, 72)[..., :64]),
    "groupnorm out shape": lambda o: o.groupnorm(_h(1, 4, 64), _h(64), _h(64), 32, 1e-5, False, out=_h(1, 2, 64)),
    "layernorm out strided": lambda o: o.layernorm(_h(4, 64), _h(64), _h(64), out=_h(4, 72)[:, :64]),
    "layernorm out shape": lambda o: o.layernorm(_h(4, 64), _h(64), _h(64), out=_h(2, 64)),
    "layernorm gamma length": lambda o: o.layernorm(_h(4, 64), _h(32), _h(64)),
    "ddim out size": lambda o: o.ddim_step(_h(16), _h(16), None, 1.0, 1, 0, 1, 0, out=_h(8)),
    "ddim out strided": lambda o: o.ddim_step(_h(16), _h(16), None, 1.0, 1, 0, 1, 0, out=_h(32)[::2]),
    "attention out rows": lambda o: o.attention(_h(128, 64), _h(128, 64), _h(128, 64), 1, 64, 2, _h(64, 64)),
    "attention v branches": lambda o: o.attention(_h(128, 64), _h(128, 64), _h(256, 64), 1, 64, 2, _h(384, 64), n_v=3,
                                                  v_branch_stride=128 * 64, o_branch_stride=128 * 64),
    "attention k rows": lambda o: o.attention(_h(128, 64), _h(100, 64), _h(145, 64), 1, 64, 2, _h(128, 64), seq_kv=145,
                                              kv_batch_div=2),
    "fused attention out width": lambda o: o.temporal_attention_fused(_h(16, 64), _h(384, 64), 2, 8, 2, 1, _h(16, 64)),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_wrapper_refuses_misaddressed_tensors(case):
    """a tensor that does not cover what the kernel addresses, in the layout it assumes, is refused before any launch"""
    from anyv2v_b200 import ops
    from anyv2v_b200._lib import Av2vError
    before = ops.launch_count()
    with pytest.raises(Av2vError):
        REFUSALS[case](ops)
    assert ops.launch_count() == before
