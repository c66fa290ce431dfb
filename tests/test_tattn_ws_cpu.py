"""CPU models of the persistent fused temporal attention (tools/kernel_models.py): its item schedule, its projection ring
and the slot map of its x box, each with a negative control."""
import random

import pytest

from tools import kernel_models as km


def test_constants_match_the_source():
    s1, s3, arrivals = km.tattn_ws_constants()
    assert s1 >= 3 and s3 >= 3 and arrivals == 8


@pytest.mark.parametrize("clips,pix_tiles,heads,sms", [(1, 512, 5, 132), (3, 128, 10, 132), (1, 3, 2, 132), (2, 8, 20, 7)])
def test_schedule_runs_every_item_once_heads_together(clips, pix_tiles, heads, sms):
    assert km.tattn_ws_schedule(clips, pix_tiles, heads, sms)


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("nk", [1, 5, 20])
def test_ring(nk, passes):
    s1, s3, arrivals = km.tattn_ws_constants()
    stages = s1 if passes == 1 else s3
    for seed in range(20):
        assert km.simulate_tattn_ring(random.Random(seed), 4, passes, nk, stages, arrivals)


@pytest.mark.parametrize("broken", [dict(release=False), dict(wrong_parity="consumer"), dict(wrong_parity="producer"),
                                    dict(overrun=True)])
def test_ring_negative_controls(broken):
    caught = 0
    for seed in range(20):
        try:
            km.simulate_tattn_ring(random.Random(seed), 4, 3, 5, 3, 8, **broken)
        except AssertionError:
            caught += 1
    assert caught > 0, f"{broken} not caught"


@pytest.mark.parametrize("F,HW", [(16, 19), (24, 11), (72, 3), (128, 2), (1, 130), (40, 7)])
def test_box_slots_equal_the_slot_map(F, HW):
    assert km.check_tattn_box_slots(F, HW)


@pytest.mark.parametrize("F,HW", [(16, 19), (24, 11)])
def test_box_slots_negative_control(F, HW):
    with pytest.raises(AssertionError):
        km.check_tattn_box_slots(F, HW, wrong_order=True)
