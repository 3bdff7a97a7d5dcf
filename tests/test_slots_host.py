"""Host-side checks of slot streams (Vid2VidModelG.stream_slots), no GPU needed: the slot bookkeeping over a scripted
schedule, the argument errors, the refusals of v2v_plan_set_image_flags, and that a slot plan (a per-sample plan reading
per-image flags) lowers every conv exactly as the per-sample plan of the same shape does -- the configuration fixes each
pixel's accumulation order, and tests/test_conv_census.py covers every per-sample configuration."""
import ctypes as C
import types

import pytest

import product_plans as PP
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200.model_g import SlotSchedule, SlotStream
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import make_opt

K, P, R, X = L.SLOT_KEEP, L.SLOT_PUSH, L.SLOT_RESTART, L.SLOT_CLEAR


def test_schedule_over_a_scripted_run():
    s = SlotSchedule(3, 3, no_first_img=True)
    # step: (starts, stops) before the step, then the expected ops / ready / join
    script = [
        ((0, 2), (), [R, K, R], [0, 0, 0], [0, 0, 0]),
        ((), (), [P, K, P], [0, 0, 0], [0, 0, 0]),
        ((1,), (), [P, R, P], [1, 0, 1], [1, 0, 1]),      # slots 0 and 2 fill their windows; slot 1 starts late
        ((2,), (), [P, P, R], [1, 0, 0], [0, 0, 0]),      # slot 2 restarts mid-clip
        ((), (), [P, P, P], [1, 1, 0], [0, 1, 0]),        # slot 1 joins while slot 0 warps
        ((), (0,), [X, P, P], [0, 1, 1], [0, 0, 1]),      # slot 0 goes idle
        ((), (), [K, P, P], [0, 1, 1], [0, 0, 0]),
        ((0,), (), [R, P, P], [0, 1, 1], [0, 0, 0]),
        ((), (), [P, P, P], [0, 1, 1], [0, 0, 0]),
        ((), (), [P, P, P], [1, 1, 1], [1, 0, 0]),
    ]
    for i, (starts, stops, ops, ready, join) in enumerate(script):
        for k in starts:
            s.start(k)
        for k in stops:
            s.stop(k)
        st = s.step()
        assert st.ops == ops, i
        assert st.ready == [bool(r) for r in ready], i
        assert st.join == [bool(j) for j in join], i
        assert st.raw_only == st.join, i                  # --no_first_img: a joining slot takes the raw composite
        assert st.flags() == [(L.IMAGE_ACTIVE if r else 0) | (L.IMAGE_RAW_ONLY if j else 0) for r, j in zip(ready, join)], i


def test_schedule_without_no_first_img_never_asks_for_raw_only():
    s = SlotSchedule(2, 2)
    s.start(1)
    for _ in range(3):
        st = s.step()
        assert st.raw_only == [False, False]
    assert st.ready == [False, True]


def test_slot_index_out_of_range():
    s = SlotSchedule(3, 3)
    for bad in (-1, 3, 1.0, True):
        with pytest.raises(IndexError, match='out of range'):
            s.start(bad)
        with pytest.raises(IndexError, match='out of range'):
            s.stop(bad)


def test_slot_count_cap():
    SlotSchedule(L.MAX_SLOTS, 3)
    for bad in (0, L.MAX_SLOTS + 1):
        with pytest.raises(ValueError, match='1 to %d slots' % L.MAX_SLOTS):
            SlotSchedule(bad, 3)
    ops = (C.c_int * (L.MAX_SLOTS + 1))()
    with pytest.raises(RuntimeError, match='at most %d' % L.MAX_SLOTS):      # refused before any launch
        L.check(L.lib().v2v_slots_window_push(C.c_void_p(16), C.c_void_p(16), 0, L.MAX_SLOTS + 1, 3, 1, 8, 8, ops, None))
    ops = (C.c_int * 2)(L.SLOT_PUSH, 7)
    with pytest.raises(RuntimeError, match='unknown op 7'):
        L.check(L.lib().v2v_slots_window_push(C.c_void_p(16), C.c_void_p(16), 0, 2, 3, 1, 8, 8, ops, None))


def _stream(B=3, use_single_G=False, **o):
    """A SlotStream over a stand-in model: the checks below run before anything touches a device."""
    return SlotStream(types.SimpleNamespace(opt=make_opt(gpu_ids=[], **o), use_single_G=use_single_G), B)


def test_frame_shape_errors():
    import torch
    street = _stream(label_nc=35, use_instance=True, use_single_G=True)
    street._check(torch.zeros(3, 8, 16, dtype=torch.uint8), None)
    for bad in (torch.zeros(2, 8, 16, dtype=torch.uint8), torch.zeros(3, 1, 8, 16, dtype=torch.uint8)):
        with pytest.raises(ValueError, match=r'\(3, H, W\) id maps'):
            street._check(bad, None)
    with pytest.raises(TypeError, match='uint8, int32 or float32'):
        street._check(torch.zeros(3, 8, 16, dtype=torch.int64), None)
    with pytest.raises(ValueError, match='does not match'):
        street._check(torch.zeros(3, 8, 16, dtype=torch.uint8), torch.zeros(3, 8, 8, dtype=torch.uint8))
    pose = _stream(label_nc=0, input_nc=6, no_first_img=True)
    pose._check(torch.zeros(3, 6, 8, 16), None)
    for bad in (torch.zeros(3, 8, 16), torch.zeros(3, 5, 8, 16), torch.zeros(3, 6, 8, 16, dtype=torch.float64)):
        with pytest.raises(ValueError, match=r'\(3, 6, H, W\) float32'):
            pose._check(bad, None)


def test_refused_configurations():
    with pytest.raises(ValueError, match='face first-frame generator'):
        _stream(label_nc=0, input_nc=15, dataset_mode='face', use_single_G=True)
    with pytest.raises(ValueError, match='no_first_img or --use_single_G'):
        _stream(label_nc=35, use_instance=True)                       # neither way to seed a joining clip's first frames
    with pytest.raises(ValueError, match='no_first_img or --use_single_G'):
        _stream(label_nc=35, use_instance=True, use_single_G=True, use_real_img=True)
    with pytest.raises(ValueError, match='1 to 64 slots'):
        _stream(B=65, label_nc=0, input_nc=6, no_first_img=True)


def test_image_flags_are_refused_on_training_and_batch_statistics_plans():
    with pytest.raises(RuntimeError, match='per-image flags are for inference plans'):
        Plan(0, precision='precise', train=True).set_image_flags(NW.S_FLAGS)
    with pytest.raises(RuntimeError, match='per-image flags need a per-sample-statistics plan'):
        Plan(0, precision='precise').set_image_flags(NW.S_FLAGS)
    p = Plan(0, precision='precise', sample_stats=True)
    p.set_image_flags(NW.S_FLAGS)
    with pytest.raises(RuntimeError, match='keeps per-sample statistics'):
        L.check(L.lib().v2v_plan_set_sample_stats(p._h, 0))


def _describe(net, B, h, w, mode, flags):
    d = PP.describe(PP.PlanSpec('slots', 'B=%d' % B, lambda p: net._describe(p, B, h, w), mode, sample_stats=True, flags=flags))
    assert d['image_flags'] == int(flags) and d['sample_stats'] == 1
    return d


@pytest.mark.parametrize('mode', ['precise', 'fast'])
@pytest.mark.parametrize('wl', list(PP.TS.WORKLOADS))
def test_slot_plans_lower_as_per_sample_plans(wl, mode):
    w = PP.TS.WORKLOADS[wl]
    for s, (net, h, w_) in enumerate(PP.scales(PP.clip_opt(w), w['H'], w['W'])):
        for B in w['bs']:
            slot, ref = _describe(net, B, h, w_, mode, True), _describe(net, B, h, w_, mode, False)
            assert slot['convs'] == ref['convs'], (wl, mode, s, B)
            assert slot['n_slots'] == NW.S_FLAGS + 1
