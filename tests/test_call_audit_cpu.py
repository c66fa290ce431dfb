"""Negative controls of tests/call_audit.py without a GPU: the audit installed over the tiny-config UNet, with the float64
contracts standing in for the kernels, on one PnP edit step with every injection firing and FreeU on.  The clean step
passes; a step whose one call is corrupted by the audit's ``perturb`` hook fails at exactly that call; snapshots taken after
the call instead of before fail the in-place ops; layernorm outputs rounded toward zero pass every call's bound and fail the
mean error of the step; the unit subsets always hold the first and last unit."""
from types import SimpleNamespace

import pytest
import torch

import freeu_ref
import sampling_ref
from call_audit import ROWS_ALL, ROWS_SEEDED, ROWS_TILE, CallAudit, row_subset, unit_subset

F_, H_, W_ = 4, 16, 16
FREEU = dict(s1=0.9, s2=0.2, b1=1.5, b2=1.6)


@pytest.fixture
def contract_ops(emulated_ops, monkeypatch):
    freeu_ref.patch_ops(monkeypatch)
    sampling_ref.patch_ops(monkeypatch)
    return emulated_ops


@torch.no_grad()
def _audited_edit_step(monkeypatch, **audit_kw):
    """one injected edit step (conv, spatial and temporal injection, FreeU, in-place DDIM) of the tiny UNet under the audit
    -> (audit, launches counted by ops.launch_count())"""
    from anyv2v_b200 import ops
    from anyv2v_b200.latent_store import LatentStore
    from anyv2v_b200.pipeline import I2VGenXLPipeline
    from anyv2v_b200.run_group_pnp_edit import init_pnp
    from anyv2v_b200.schedulers import DDIMScheduler
    from anyv2v_b200.unet_i2vgen_xl import I2VGenXLUNet
    from oracle import loops_ref, unet_ref
    ours = I2VGenXLUNet(**unet_ref.TINY_CONFIG)
    ours.load_state_dict(unet_ref.seeded_unet(unet_ref.TINY_CONFIG, seed=8888, dtype=torch.float32, device="cpu").state_dict())
    ours = ours.to(dtype=torch.float16).eval()
    ns = loops_ref.synthetic_inputs(F_, H_, W_, cross_dim=64, dtype=torch.float16, device="cpu")
    sched = DDIMScheduler()
    sched.set_timesteps(4)
    pipe = I2VGenXLPipeline(ours, sched)
    init_pnp(pipe, sched, SimpleNamespace(n_steps=4, pnp_f_t=1.0, pnp_spatial_attn_t=1.0, pnp_temp_attn_t=1.0))
    pipe.enable_freeu(**FREEU)
    store = LatentStore(None, write_files=False)
    store.put(int(sched.timesteps[0]), torch.randn(1, 4, F_, H_, W_, generator=torch.Generator().manual_seed(5)).half())
    audit = CallAudit(seed=1, **audit_kw).install(monkeypatch)
    n0 = ops.launch_count()
    st = pipe.prepare_edit(ns.video_latents.clone(), ns.edit_prompt, ns.neg_prompt, ns.inv_prompt, ns.edit_image_emb,
                           ns.edit_image_latents, ns.src_image_emb, ns.src_image_latents, 8, 4, 9.0, 0, None, store, True)
    pipe.edit_step(st, 0)
    return audit, ops.launch_count() - n0


def test_clean_step_passes_and_audits_every_launch(contract_ops, monkeypatch):
    audit, launches = _audited_edit_step(monkeypatch)
    print("\n" + audit.table())
    audit.assert_clean()
    assert audit.launches == launches > 0
    assert audit.seen("attention", mode="rows", n_v=3)
    assert audit.seen("attention", mode="rows", kv_batch_div=F_)
    assert audit.seen("temporal_attention_fused", n_v=3)
    assert audit.seen("conv3x3", slots=3, residual=True)
    assert audit.seen("groupnorm", two_source=True)
    assert audit.seen("linear", geglu=True)
    assert audit.seen("layernorm") and audit.seen("tconv3") and audit.seen("upsample2x_conv3x3")
    assert len(audit.seen("freeu")) == 6  # every skip connection of up blocks 0 and 1
    assert [r.sig for r in audit.seen("ddim_step")] == [f"ddim_step n={4 * F_ * H_ * W_} cfg in-place"]


# ------------------------------------------------------------------------------------------------------------- perturbations
def _once(op, pred, corrupt):
    """perturb hook: corrupt(p, out) on the first call of `op` for which pred(p, out) holds; remembers its index"""
    state = SimpleNamespace(index=None)

    def hook(name, index, p, out):
        if state.index is None and name == op and pred(p, out):
            corrupt(p, out)
            state.index = index
    return hook, state


def _ulps(t, flat_index, n):
    """move one fp16 element of t by n ulps (away from zero for n > 0)"""
    bits = t.view(-1).view(torch.int16)
    bits[flat_index] += n


def _linear_3ulp(p, out):
    _ulps(out, int(out.float().abs().reshape(-1).argmax()), 3)


def _conv_slot_from_other(p, out):
    M = p["x"].shape[0] * p["x"].shape[1] * p["x"].shape[2]
    rows = lambda s: out.as_strided((M, out.shape[-1]), (out.stride(-2), 1), out.storage_offset() + s * p["slot_stride"])
    rows(1).copy_(rows(0))


def _attention_wrong_keys(p, out):
    """branch 2 of query sequence 0 computed with the keys of sequence 1"""
    import kernel_contracts as kc
    heads, seq, C = p["heads"], p["seq"], p["heads"] * 64
    ldv, ldo = p["v"].stride(0), out.stride(0)
    vrows, orows = p["v_branch_stride"] // ldv, p["o_branch_stride"] // ldo
    o = torch.empty(seq, C, dtype=torch.float16)
    ref, _ = kc.attention_exact(p["q"][:seq], p["k"][seq:2 * seq], p["v"][2 * vrows:2 * vrows + seq], heads, seq, 1, o, p["scale"])
    out[2 * orows:2 * orows + seq, :C] = ref.half()


def _groupnorm_neighbour_stats(p, out):
    """sample 0 normalised with the mean and variance of sample 1"""
    x = p["x"] if p["x2"] is None else torch.cat([p["x"], p["x2"]], dim=2)
    n, rows, C = x.shape
    G = p["groups"]
    xf = x.double().view(n, rows, G, C // G)
    mean, var = xf[1].mean(dim=(0, 2), keepdim=True), xf[1].var(dim=(0, 2), unbiased=False, keepdim=True)
    y = ((xf[0] - mean) * torch.rsqrt(var + p["eps"])).view(rows, C) * p["gamma"].double() + p["beta"].double()
    if p["silu"]:
        y = y.half().double()
        y = y * torch.sigmoid(y)
    out[0] = y.half()


def _layernorm_row_shift(p, out):
    row = out.view(-1, out.shape[-1])[0]
    row.copy_(row.roll(1))


def _ddim_1ulp(p, out):
    _ulps(out, 7, 1)


def _freeu_twice(p, out):
    h = p["hidden"]
    half = h.shape[-1] // 2
    h[..., :half] = (h[..., :half].float() * torch.tensor(p["b"], dtype=torch.float32)).half()


PERTURBATIONS = {
    "linear element moved 3 ulps": ("linear", lambda p, o: True, _linear_3ulp),
    "conv slot written from another slot": ("conv3x3", lambda p, o: p["n_slots"] > 1, _conv_slot_from_other),
    "attention branch from the wrong key sequence": ("attention", lambda p, o: not p["frames_mode"] and p["n_v"] == 3,
                                                     _attention_wrong_keys),
    "groupnorm sample with its neighbour's statistics": ("groupnorm", lambda p, o: p["x"].shape[0] > 1, _groupnorm_neighbour_stats),
    "layernorm row shifted": ("layernorm", lambda p, o: True, _layernorm_row_shift),
    "ddim element moved 1 ulp": ("ddim_step", lambda p, o: True, _ddim_1ulp),
    "freeu hidden half scaled twice": ("freeu", lambda p, o: True, _freeu_twice),
}


@pytest.mark.parametrize("what", list(PERTURBATIONS))
def test_each_perturbation_fails_at_its_call(contract_ops, monkeypatch, what):
    op, pred, corrupt = PERTURBATIONS[what]
    hook, state = _once(op, pred, corrupt)
    audit, launches = _audited_edit_step(monkeypatch, perturb=hook)
    assert state.index is not None, f"no {op} call to perturb"
    assert audit.launches == launches
    bad = audit.failures()
    assert [r.index for r in bad] == [state.index], [r.line() for r in bad]
    with pytest.raises(AssertionError) as e:
        audit.assert_clean()
    assert f"#{state.index} {op}" in str(e.value)


def test_snapshots_taken_after_the_call_fail_the_in_place_ops(contract_ops, monkeypatch):
    """the snapshots are what the contract reads: taken after freeu (which scales hidden in place) and after ddim_step with
    out = x, they no longer hold the kernel's inputs"""
    audit, _ = _audited_edit_step(monkeypatch, snapshot_after=True)
    bad = audit.failures()
    ops_failed = {r.op for r in bad}
    assert {"freeu", "ddim_step"} <= ops_failed, [r.line() for r in bad]
    assert len([r for r in bad if r.op == "freeu"]) == 6
    assert all("in-place" in r.sig for r in bad if r.op == "ddim_step")
    # the clean audit of the same step passes, so the snapshot timing alone makes the difference
    clean, _ = _audited_edit_step(monkeypatch)
    clean.assert_clean()


# ------------------------------------------------------------------------------------------------------------- mean error
def test_clean_step_is_unbiased(contract_ops, monkeypatch):
    audit, _ = _audited_edit_step(monkeypatch)
    for op, mo in audit.bias_by_op().items():
        print(f"{op:26s} {mo.line()}")
    audit.assert_unbiased()


def test_layernorm_rounded_toward_zero_fails_only_the_mean(contract_ops, monkeypatch):
    """every layernorm output replaced by its float64 contract rounded toward zero (the fp16 output alone can not be
    re-rounded): each call stays inside its element-wise bound, the mean error of layernorm over the step does not"""
    import kernel_contracts as kc
    from bias_check import round_fp16
    perturbed = []

    def hook(name, index, p, out):
        if name == "layernorm":
            ref = kc.layernorm_exact(p["x"], p["gamma"], p["beta"], p["eps"])
            out.copy_(round_fp16(ref, "zero").view(out.shape))
            perturbed.append(index)

    audit, _ = _audited_edit_step(monkeypatch, perturb=hook)
    assert perturbed == [r.index for r in audit.seen("layernorm")] and perturbed
    audit.assert_clean()
    with pytest.raises(AssertionError) as e:
        audit.assert_unbiased()
    failed = [line.split(":")[0] for line in str(e.value).splitlines()[1:]]
    assert failed == ["layernorm"], str(e.value)
    assert "|mean sign(ref) e| over" in str(e.value)


# ------------------------------------------------------------------------------------------------------------- subsets
@pytest.mark.parametrize("k", [0, 2, 254])
def test_unit_subsets_hold_the_first_and_last_unit(k):
    for n in list(range(1, 300)) + [4096, 14080, 225280]:
        for seed in (0, 1, 77):
            s = unit_subset(n, k, seed).tolist()
            assert s[0] == 0 and s[-1] == n - 1 and s == sorted(set(s))
            assert len(s) == min(n, k + 2)


def test_row_subsets_hold_the_first_and_last_tiles():
    for M in (1, 127, ROWS_ALL, ROWS_ALL + 1, 196608, 450560):
        for seed in (0, 5):
            s = row_subset(M, seed)
            if M <= ROWS_ALL:
                assert torch.equal(s, torch.arange(M))
                continue
            assert torch.equal(s[:ROWS_TILE], torch.arange(ROWS_TILE))
            assert torch.equal(s[-ROWS_TILE:], torch.arange(M - ROWS_TILE, M))
            assert len(s) == 2 * ROWS_TILE + ROWS_SEEDED and len(set(s.tolist())) == len(s)
