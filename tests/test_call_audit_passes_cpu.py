"""tests/call_audit.py over the passes whose kernels came after it, without a GPU: the tiny UNet and VAE with the float64
contracts standing in for the kernels.  Clean passes: two DPM-Solver++(2M) edit steps (first and second order), an edit step
replayed from a SourceFeatureCache (attention at n_v = 2, the fused temporal attention with Q / K from the cached source,
GroupNorm with an explicit partition) and a tiled VAE decode.  Each negative control corrupts one call and must fail at
exactly that call.  A structural check keeps every launching entry point of anyv2v_b200.ops in the audit."""
import ast
import inspect
from types import SimpleNamespace

import pytest
import torch

import dpm_solver_ref
import freeu_ref
import kernel_contracts as kc
import sampling_ref
import source_cache_ref
import vae_tiling_ref
from call_audit import AUDITED, CallAudit
from test_call_audit_cpu import _once, _ulps
from test_host_model_cpu import F_, H_, W_, _models

ALL_FIRE = SimpleNamespace(pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0)
DPM_STEPS, STORE_STEPS = 5, 10   # the DPM timesteps 801, 601, ..., 1 are every other one of a 10-step inversion
DDIM_STEPS = 4


@pytest.fixture
def contract_ops(emulated_ops, monkeypatch):
    for ref in (sampling_ref, freeu_ref, dpm_solver_ref, source_cache_ref, vae_tiling_ref):
        ref.patch_ops(monkeypatch)
    return emulated_ops


def _store(steps, seed=5):
    """random source latents at every timestep of a ``steps``-step DDIM inversion"""
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.schedulers import DDIMScheduler
    s = DDIMScheduler()
    s.set_timesteps(steps)
    store = LatentStore(None, write_files=False)
    g = torch.Generator().manual_seed(seed)
    for t in s.timesteps.tolist():
        store.put(int(t), torch.randn(1, 4, F_, H_, W_, generator=g).half())
    return store


def _inputs(seed):
    """the synthetic clip's conditioning, with the edit prompt and edited first frame drawn from ``seed``"""
    from oracle import loops_ref
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    g = torch.Generator().manual_seed(seed)
    rn = lambda t: (t.float() + torch.randn(t.shape, generator=g)).half()
    ns.edit_prompt, ns.edit_image_emb, ns.edit_image_latents = rn(ns.edit_prompt), rn(ns.edit_image_emb), rn(ns.edit_image_latents)
    return ns


def _prepare(pipe, ns, n_steps, store, cache=None):
    return pipe.prepare_edit(ns.video_latents.clone(), ns.edit_prompt, ns.neg_prompt, ns.inv_prompt, ns.edit_image_emb,
                             ns.edit_image_latents, ns.src_image_emb, ns.src_image_latents, 8, n_steps, 9.0, 0, None, store, True,
                             source_features=cache)


def _pipeline(sched, n_steps):
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    sched.set_timesteps(n_steps)
    pipe = I2VGenXLPipeline(_models()[1], sched)
    init_pnp(pipe, sched, SimpleNamespace(n_steps=n_steps, **vars(ALL_FIRE)))
    return pipe


def _audited(monkeypatch, run, **audit_kw):
    """run() under the audit -> (audit, launches counted by ops.launch_count() over the same span)"""
    from anyv2v_b200 import ops
    audit = CallAudit(seed=1, **audit_kw).install(monkeypatch)
    n0 = ops.launch_count()
    run()
    return audit, ops.launch_count() - n0


@torch.no_grad()
def _dpm_edit_steps(monkeypatch, **audit_kw):
    """DPM-Solver++(2M) edit steps 0 (first order) and 1 (second order), every injection firing"""
    from anyv2v_b200.schedulers import DPMSolverMultistepScheduler
    pipe = _pipeline(DPMSolverMultistepScheduler(), DPM_STEPS)
    store = _store(STORE_STEPS)

    def run():
        st = _prepare(pipe, _inputs(1), DPM_STEPS, store)
        pipe.edit_step(st, 0)
        pipe.edit_step(st, 1)
    return _audited(monkeypatch, run, **audit_kw)


@torch.no_grad()
def _replayed_edit_step(monkeypatch, **audit_kw):
    """edit A's step 0 fills a SourceFeatureCache; edit B's step 0 (another prompt and first frame) replays it"""
    from anyv2v_b200.schedulers import DDIMScheduler
    pipe = _pipeline(DDIMScheduler(), DDIM_STEPS)
    store = _store(DDIM_STEPS)
    cache = pipe.source_feature_cache(max_bytes=1 << 40)
    pipe.edit_step(_prepare(pipe, _inputs(1), DDIM_STEPS, store, cache), 0)
    assert len(cache) == 1
    modes = []

    def run():
        st = _prepare(pipe, _inputs(2), DDIM_STEPS, store, cache)
        pipe.edit_step(st, 0)
        modes.extend(k[-1] for k in st.iterations)
    out = _audited(monkeypatch, run, **audit_kw)
    assert modes == ["replay"]
    return out


@torch.no_grad()
def _tiled_decode(monkeypatch, **audit_kw):
    """the tiny VAE's tiled decode of 3 latents of 16 x 20 (8-pixel latent tiles every 6: 3 x 4 tiles of 16 output pixels)"""
    from anyv2v_b200 import vae
    from oracle import vae_ref
    ours = vae.AutoencoderKL(**vae_ref.TINY_VAE_CONFIG, sample_size=16)
    ours.load_state_dict(vae_ref.seeded_vae(vae_ref.TINY_VAE_CONFIG, seed=8888, dtype=torch.float32).state_dict())
    ours = ours.half().eval()
    ours.enable_tiling()
    z = torch.randn(3, 4, 16, 20, generator=torch.Generator().manual_seed(5)).half()
    return _audited(monkeypatch, lambda: ours.decode(z), **audit_kw)


def _assert_clean(audit, launches):
    print("\n" + audit.table())
    audit.assert_clean()
    assert audit.launches == launches > 0


# ------------------------------------------------------------------------------------------------------------- clean passes
def test_dpm_edit_steps_pass(contract_ops, monkeypatch):
    audit, launches = _dpm_edit_steps(monkeypatch)
    _assert_clean(audit, launches)
    n = 4 * F_ * H_ * W_
    assert [r.sig for r in audit.seen("dpmpp2m_step")] == [f"dpmpp2m_step n={n} order=1 cfg in-place",
                                                          f"dpmpp2m_step n={n} order=2 cfg in-place"]
    assert audit.seen("attention", mode="rows", n_v=3) and audit.seen("temporal_attention_fused", n_v=3)


def test_replayed_edit_step_passes(contract_ops, monkeypatch):
    audit, launches = _replayed_edit_step(monkeypatch)
    _assert_clean(audit, launches)
    assert audit.seen("attention", mode="rows", n_v=2)
    assert audit.seen("temporal_attention_fused_qksrc", clips=2, F=F_)
    assert audit.seen("groupnorm", partition_samples=lambda v: v > 0)
    assert not audit.seen("attention", n_v=3) and not audit.seen("temporal_attention_fused", n_v=3)


def test_tiled_decode_passes(contract_ops, monkeypatch):
    audit, launches = _tiled_decode(monkeypatch)
    _assert_clean(audit, launches)
    assert [r.sig for r in audit.seen("tile_stitch")] == [
        "tile_stitch N=3 C=3 32x40 tiles=3x4 tile=16 step=12 blend=4 row_limit=12"]


# ------------------------------------------------------------------------------------------------------------- negative controls
def _attention_branch1_over(p, out):
    """the largest element of the first row of branch 1 (cond) moved far over the attention bound"""
    row = out[p["o_branch_stride"] // out.stride(0), :p["heads"] * 64]
    _ulps(row, int(row.float().abs().argmax()), 64)


def _qksrc_cond_from_uncond(p, out):
    """the cond clips written with the output of the uncond clips"""
    n = p["x"].shape[0] // 2
    out[n:] = out[:n]


def _x0_prev_1ulp(p, out):
    _ulps(p["x0_prev"], 7, 1)


def _seam_pixel_1ulp(p, out):
    """one pixel of image 0 inside the horizontal blend of tiles (0, 0) and (0, 1)"""
    out[0, 0, 1, p["row_limit"] + 1] = (out[0, 0, 1, p["row_limit"] + 1:p["row_limit"] + 2].view(torch.int16) + 1).view(torch.float16)


NEGATIVE = {
    "n_v = 2 attention, one element of branch 1 over the bound": (
        _replayed_edit_step, "attention", lambda p, o: p["n_v"] == 2 and not p["frames_mode"], _attention_branch1_over),
    "qksrc cond clips from the uncond clips": (
        _replayed_edit_step, "temporal_attention_fused_qksrc", lambda p, o: True, _qksrc_cond_from_uncond),
    "x0_prev moved 1 ulp": (_dpm_edit_steps, "dpmpp2m_step", lambda p, o: True, _x0_prev_1ulp),
    "stitch seam pixel moved 1 ulp": (_tiled_decode, "tile_stitch", lambda p, o: True, _seam_pixel_1ulp),
}


@pytest.mark.parametrize("what", list(NEGATIVE))
def test_each_corruption_fails_at_its_call(contract_ops, monkeypatch, what):
    run, op, pred, corrupt = NEGATIVE[what]
    hook, state = _once(op, pred, corrupt)
    audit, launches = run(monkeypatch, perturb=hook)
    assert state.index is not None, f"no {op} call to corrupt"
    assert audit.launches == launches
    bad = audit.failures()
    assert [r.index for r in bad] == [state.index], [r.line() for r in bad]
    with pytest.raises(AssertionError) as e:
        audit.assert_clean()
    assert f"#{state.index} {op}" in str(e.value)


def test_second_order_step_computed_as_first_order_fails(contract_ops, monkeypatch):
    """a step kernel that drops the second-order term (c = 0) fails at the second-order call only"""
    from anyv2v_b200 import ops
    real = ops.dpmpp2m_step

    def first_order_only(*args, coef_dev=None, **kw):
        if coef_dev is not None:
            coef_dev = coef_dev.clone()
            coef_dev[4] = 0.0
        return real(*args, coef_dev=coef_dev, **kw)
    monkeypatch.setattr(ops, "dpmpp2m_step", first_order_only)
    hook, state = _once("dpmpp2m_step", lambda p, o: float(p["coef_dev"][4]) != 0.0, lambda p, o: None)
    audit, _ = _dpm_edit_steps(monkeypatch, perturb=hook)
    bad = audit.failures()
    assert state.index is not None and [r.index for r in bad] == [state.index], [r.line() for r in bad]
    assert "order=2" in bad[0].sig and "dpmpp2m_step out" in bad[0].detail and "x0_prev" not in bad[0].detail


def test_dpm_snapshots_taken_after_the_call_fail(contract_ops, monkeypatch):
    """the step reads x (updated in place) and the previous x0 (overwritten): snapshots taken after it fail both steps"""
    audit, _ = _dpm_edit_steps(monkeypatch, snapshot_after=True)
    bad = [r for r in audit.failures() if r.op == "dpmpp2m_step"]
    assert [r.index for r in bad] == [r.index for r in audit.seen("dpmpp2m_step")] and len(bad) == 2
    assert "x0_prev" in bad[1].detail


# ------------------------------------------------------------------------------------------------------------- structure
def test_every_launching_entry_point_is_audited():
    """an entry point of anyv2v_b200.ops that counts a kernel launch (itself or through _gemm) is in AUDITED"""
    from anyv2v_b200 import ops
    src = inspect.getsource(ops)
    launching = {f.name for f in ast.parse(src).body if isinstance(f, ast.FunctionDef) and not f.name.startswith("_")
                 and any(s in ast.get_source_segment(src, f) for s in ("_launches +=", "_gemm("))}
    assert launching == set(AUDITED)


@pytest.mark.parametrize("frames", [False, True])
def test_attention_contract_at_two_branches_is_the_edit_branches_at_three(frames):
    """kernel_contracts.attention(_exact) at n_v = 2 on [uncond, cond]: each branch equals the same branch at n_v = 3, with
    branch strides that are not the branches' extent"""
    g = torch.Generator().manual_seed(3)
    heads, seq, batch, HW = 2, 6, (4 if frames else 3), (2 if frames else 0)
    C, rows = heads * 64, batch * seq
    gap = 5
    q, k = (torch.randn(rows, C, generator=g).half() for _ in range(2))
    v3 = torch.randn(3 * (rows + gap), C, generator=g).half()
    mode = dict(frames_mode=frames, HW=HW)
    out3 = torch.zeros(3 * rows, C, dtype=torch.float16)
    kc.attention(q, k, v3, heads, seq, batch, out3, n_v=3, v_branch_stride=(rows + gap) * C, o_branch_stride=rows * C, **mode)
    ref3, _ = kc.attention_exact(q, k, v3, heads, seq, batch, out3, n_v=3, v_branch_stride=(rows + gap) * C,
                                 o_branch_stride=rows * C, **mode)
    out2 = torch.full((2 * (rows + gap), C), float("nan"), dtype=torch.float16)
    kw = dict(n_v=2, v_branch_stride=(rows + gap) * C, o_branch_stride=(rows + gap) * C, **mode)
    kc.attention(q, k, v3[rows + gap:], heads, seq, batch, out2, **kw)
    ref2, _ = kc.attention_exact(q, k, v3[rows + gap:], heads, seq, batch, out2, **kw)
    for b in range(2):
        o2 = slice(b * (rows + gap), b * (rows + gap) + rows)
        o3 = slice((b + 1) * rows, (b + 2) * rows)
        assert torch.equal(out2[o2], out3[o3]) and torch.equal(ref2[o2], ref3[o3]), b
        assert torch.isnan(ref2[b * (rows + gap) + rows:(b + 1) * (rows + gap)]).all()
