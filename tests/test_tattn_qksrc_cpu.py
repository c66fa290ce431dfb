"""CPU model of the Q/K-source variant of the persistent fused temporal attention (tattn_fused_kernel<2, true>, behind
av2v_tattn_fused_qksrc_f16): its stage ring over three projection passes per item (Q / K of the source tensor, then the V
of each edit clip) under randomised latencies, and which clip each pass reads, with negative controls."""
import random

import pytest

from tools import kernel_models as km


def test_constants_are_the_kernels():
    stages, passes, arrivals = km.tattn_qksrc_constants()
    assert (stages, passes, arrivals) == (3, 3, 8)


@pytest.mark.parametrize("nk", [1, 5, 16, 20])
@pytest.mark.parametrize("seed", range(4))
def test_ring_three_passes(nk, seed):
    stages, passes, arrivals = km.tattn_qksrc_constants()
    assert km.simulate_tattn_ring(random.Random(seed), 4, passes, nk, stages, arrivals)


@pytest.mark.parametrize("broken", [dict(wrong_parity="producer"), dict(wrong_parity="consumer"), dict(release=False),
                                    dict(overrun=True)], ids=lambda b: "-".join(f"{k}={v}" for k, v in b.items()))
def test_ring_negative_controls(broken):
    stages, passes, arrivals = km.tattn_qksrc_constants()
    with pytest.raises(AssertionError):
        for seed in range(8):
            km.simulate_tattn_ring(random.Random(seed), 4, passes, 5, stages, arrivals, **broken)


@pytest.mark.parametrize("src_clips", [1, 2, 5])
def test_pass_sources(src_clips):
    assert km.check_tattn_qksrc_passes(src_clips)
    with pytest.raises(AssertionError):
        km.check_tattn_qksrc_passes(src_clips, off_by_one=True)
