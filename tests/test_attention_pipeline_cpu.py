"""CPU checks of attn_rows_kernel (csrc/attention_wgmma.cu), the pipelined rows-mode attention: the discrete-event model of
its producer / consumer ring and ping-pong turns (tools/kernel_models.py), with one negative control per rule, and the
numerical emulation of its per-row algorithm (tools/attention_emulation.py) against exact softmax attention."""
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_rows_ring_protocol_model():
    """stage count and empty-barrier arrivals read from the kernel source; under randomised load, MMA and softmax latencies
    no tile is read before it landed, no stage is refilled before both consumers released it, and the turns alternate —
    for key loops shorter than, equal to and many times the ring"""
    from tools import kernel_models as km
    stages, arrivals = km.rows_ring_constants()
    rng = random.Random(13)
    for n in (1, 2, stages - 1, stages, stages + 1, 2 * stages + 3, 64):
        for _ in range(20):
            km.simulate_rows_ring(random.Random(rng.getrandbits(32)), n, stages, arrivals)


@pytest.mark.parametrize("bad", [dict(release=False), dict(wrong_parity="consumer"), dict(wrong_parity="producer"),
                                 dict(pingpong=False)], ids=["no_release", "consumer_parity", "producer_parity", "no_pingpong"])
def test_rows_ring_negative_controls(bad):
    """the model catches a consumer that never releases its stage, a wait on the wrong parity (either side) and a dropped
    ping-pong barrier"""
    from tools import kernel_models as km
    stages, arrivals = km.rows_ring_constants()
    rng = random.Random(17)
    caught = 0
    for _ in range(20):
        try:
            km.simulate_rows_ring(random.Random(rng.getrandbits(32)), 3 * stages, stages, arrivals, **bad)
        except AssertionError:
            caught += 1
    assert caught >= 15, bad


@pytest.mark.parametrize("tk", [128, 64])
def test_rows_algorithm_emulation(tk):
    """128-key tiles (n_v = 1) and 64-key tiles (n_v = 3), running max over raw scores, the exponent in one FMA, the
    kernel's 25 % FMA-pipe exponentials: within the tolerance of the GPU parity tests, at ragged key tails (145, 300 keys),
    large scores, rising key norms and 4096 keys"""
    from tools import attention_emulation as em
    for kw in (dict(T=64, L=300), dict(T=128, L=145), dict(T=64, L=512, mag=6.0), dict(T=64, L=640, rising=True),
               dict(T=64, L=4096)):
        assert em.check(poly=1, tk=tk, fused=True, **kw) < 0.5, (tk, kw)
