"""CPU tests of the model of gemm_ws_kernel's schedule (tools/kernel_models.py: linear_ws_schedule, simulate_linear_ws):
the persistent tile schedule, the TMA stage ring across tile boundaries, the consumers' turn taking and the reuse of each
staging tile, each with a negative control."""
import os
import random
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.mark.parametrize("sms", [132, 114])
def test_schedule_covers_every_tile_once(sms):
    """tile counts below, equal to and above the SM count, ragged ones included; off by one computes a tile past the end"""
    from tools import kernel_models as km
    km.linear_ws_constants()
    for tiles in (1, 2, sms - 1, sms, sms + 1, 2 * sms - 1, 2 * sms + 3, 3 * sms, 12288, 12289):
        assert km.linear_ws_schedule(tiles, sms)
        with pytest.raises(AssertionError, match="past the last"):
            km.linear_ws_schedule(tiles, sms, off_by_one=True)


def _runs(rng, n_tiles, nk, **kw):
    from tools import kernel_models as km
    stages, arrivals = km.linear_ws_constants()
    return km.simulate_linear_ws(random.Random(rng.getrandbits(32)), n_tiles, nk, stages, arrivals, **kw)


def test_ring_turns_and_staging():
    """blocks of 1 .. 7 tiles per CTA (one warpgroup a tile more than the other when odd) with K loops shorter and longer
    than the ring: no block is read before it lands, no stage is refilled before it is released, the K loops alternate
    0, 1, 0, 1, ..., and a staging tile is refilled only after its copy-out"""
    rng = random.Random(3)
    for n_tiles in (1, 2, 3, 4, 7):
        for nk in (1, 2, 3, 4, 5, 20):
            for _ in range(10):
                assert _runs(rng, n_tiles, nk)


@pytest.mark.parametrize("fault,match", [
    (dict(release=False), "deadlock"),                                  # a consumer warp never arrives on empty
    (dict(wrong_parity="producer"), "refilled with block"),
    (dict(wrong_parity="consumer"), "before it landed"),
    (dict(pingpong=False), "before it landed|overlap|take turns"),      # the order barrier dropped
    (dict(early_refill=True), "staging tile .* refilled"),             # next residual fetched before the copy-out
])
def test_negative_controls(fault, match):
    rng = random.Random(7)
    caught = 0
    for _ in range(20):
        try:
            _runs(rng, 6, 5, **fault)
        except AssertionError as e:
            assert re.search(match, str(e)), str(e)
            caught += 1
    assert caught >= 15
