"""tests/test_gpu_schedule_parity.py (every step of the inversion and the PnP edit against the fp32 oracle) re-run on CPU
with the tiny topology-equivalent config, 4 frames x 16 x 16 and an 8-step schedule (conv + spatial + temporal injection
on steps 0-3, conv only on 4-5, nothing on 6-7), on the float64 kernel contracts: exercises the module's host wiring
before any GPU minute is spent on it.

Then negative controls: step-dependent wiring faults injected into the product side only.  Each must fail the per-step
criterion at the first step it affects, after every step before it has passed."""
from types import SimpleNamespace

import pytest
import torch

N_STEPS = 8


@pytest.fixture(scope="module")
def tiny():
    import test_gpu_schedule_parity as sp
    import test_gpu_fullwidth as fw
    from oracle import unet_ref
    with pytest.MonkeyPatch.context() as mp:
        for name, value in (("CONFIG_OVERRIDE", unet_ref.TINY_CONFIG), ("dev", "cpu"), ("F_", 4), ("H_", 16), ("W_", 16),
                            ("N_STEPS", N_STEPS)):
            mp.setattr(sp, name, value)
        with torch.no_grad():
            full = fw.build_models("cpu", unet_ref.TINY_CONFIG)
            orc = sp.build_oracle(full)
        yield SimpleNamespace(sp=sp, full=full, orc=orc)


def test_schedule_parity_gpu_module_runs_on_cpu_with_the_tiny_config(emulated_ops, tiny):
    sp = tiny.sp
    assert [sp.expected_flags(i) for i in (0, 3, 4, 5, 6, 7)] == [(True,) * 3, (True,) * 3, (True, False, False),
                                                                  (True, False, False), (False,) * 3, (False,) * 3]
    assert sp.flag_change_steps() == (0, 3, 4, 5, 6, 7)
    assert len(tiny.orc.inv_traj) == len(tiny.orc.edit_traj) == N_STEPS + 1
    sp.test_teacher_forced_inversion_every_step_graphed(tiny.full, tiny.orc)
    sp.test_teacher_forced_pnp_edit_every_step_graphed(tiny.full, tiny.orc)
    sp.test_graph_replay_equals_eager_at_flag_changes(tiny.full, tiny.orc)
    sp.test_free_running_inversion_and_edit(tiny.full, tiny.orc)


def _stale_hook_state(monkeypatch):
    """register_time keeps the first step's t and the hook flags stay the first step's: what a graph replayed with the
    flags baked in at capture would compute.  (On CPU every iteration runs eagerly, so a stale flag set alone would only
    move the prune site, and a stale t alone is hidden by the pruned batch: the hooks see two branches and cannot fire.)"""
    from anyv2v_b200 import pipeline
    first = []
    real_time, real_flags = pipeline.register_time, pipeline.I2VGenXLPipeline._hook_flags

    def stale_time(model, t):
        first.append(t)
        real_time(model, first[0])

    monkeypatch.setattr(pipeline, "register_time", stale_time)
    monkeypatch.setattr(pipeline.I2VGenXLPipeline, "_hook_flags", lambda self, t: real_flags(self, first[0] if first else t))


def _mirrored_source_latent(monkeypatch):
    """the edit reads the store in inversion order instead of edit order: step i gets the latent of the i-th inversion
    timestep (x_1 at t = 981).  A read of the NEIGHBOURING timestep is not a usable control: consecutive inverted latents
    are so close that, with random-init weights, the step moves by less than fp16 rounding does (ours / torch-fp16 rises
    from 0.94 to 1.44 at 8 steps, and to 1.03-1.13 at 16), far inside the 3x calibration of the criterion."""
    from anyv2v_b200.latent_store import LatentStore
    real = LatentStore.get

    def get(self, t, device=None):
        ts = sorted(self._mem)
        return real(self, ts[len(ts) - 1 - ts.index(int(t))], device)

    monkeypatch.setattr(LatentStore, "get", get)


def _frozen_time_embedding(monkeypatch):
    """the UNet's time embedding keeps the first step's t (its sinusoidal input is frozen; the batch may change)"""
    from anyv2v_b200.unet_i2vgen_xl import TimestepEmbedding
    real = TimestepEmbedding.forward
    kept = []

    def forward(self, x):
        if not kept:
            kept.append(x[:1].clone())
        return real(self, kept[0].expand_as(x).contiguous())

    monkeypatch.setattr(TimestepEmbedding, "forward", forward)


@torch.no_grad()
@pytest.mark.parametrize("fault,test,first_bad", [
    (_stale_hook_state, "test_teacher_forced_pnp_edit_every_step_graphed", "edit step 4"),
    (_mirrored_source_latent, "test_teacher_forced_pnp_edit_every_step_graphed", "edit step 0"),
    (_frozen_time_embedding, "test_teacher_forced_inversion_every_step_graphed", "inversion step 1"),
    (_frozen_time_embedding, "test_teacher_forced_pnp_edit_every_step_graphed", "edit step 1"),
], ids=["stale-hook-state", "mirrored-source-latent", "frozen-time-embedding-inversion", "frozen-time-embedding-edit"])
def test_per_step_criterion_catches_wiring_faults_at_the_first_affected_step(emulated_ops, tiny, monkeypatch, capsys, fault,
                                                                            test, first_bad):
    fault(monkeypatch)
    with pytest.raises(AssertionError) as e:
        getattr(tiny.sp, test)(tiny.full, tiny.orc)
    # the per-step criterion (its message starts with the step's name) failed, not another assertion
    assert str(e.value).startswith(f"('{first_bad} t="), str(e.value)
    # every earlier step was checked and passed: one table row each
    step = int(first_bad.split()[-1])
    rows = [ln.split()[0] for ln in capsys.readouterr().out.splitlines() if ln[:4].strip().isdigit()]
    assert rows == [str(i) for i in range(step)], rows
