"""Slot streams (Vid2VidModelG.stream_slots) on the GPU: B = 3 slots whose clips start, restart and stop independently.
Every produced frame must equal, bit for bit, the same clip's batch-1 run (street: inference_stream; pose: inference on its
windows), `ready` must be exactly the expected mask, and the running statistics must end as a step-by-step replay of the
active clips' batch-1 forwards in slot order leaves them.  The composite's per-image flags are checked against the
use_raw_only plans image by image across graph replays."""
import pytest
import torch

import cases as C
import test_gpu_multiclip as TMC
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import det_fill_

pytestmark = pytest.mark.gpu

B = 3
# (step, slot, clip, frames): the clip starts in the slot at that step and feeds that many frames.  With tG = 3:
#   slot 1 starts late (step 2) and joins at step 4, while slots 0 and 2 warp (pose: a raw-only join among warping slots);
#   slot 2 is restarted mid-clip at step 3 (clip 1 has produced one frame);
#   slot 0 stays idle for steps 7-9, then takes clip 4 (clip 4 in slot 0, clip 2 in slot 1, clip 3 in slot 2).
SCHEDULE = [(0, 0, 0, 7), (0, 2, 1, 5), (2, 1, 2, 6), (3, 2, 3, 6), (10, 0, 4, 5)]
N_STEPS = 15


def _plan_steps(tG):
    """Per step: [(slot, clip, frame index) or None per slot], the expected ready mask, and the starts / stops to issue."""
    running = [None] * B
    steps = []
    for t in range(N_STEPS):
        starts, stops = [], []
        for st, k, c, n in SCHEDULE:
            if st == t:
                starts.append(k)
                running[k] = (c, st, n)
        for k in range(B):
            if running[k] is not None and t - running[k][1] >= running[k][2]:
                running[k] = None
                stops.append(k)
        feed = [None if r is None else (k, r[0], t - r[1]) for k, r in enumerate(running)]
        steps.append((feed, [f is not None and f[2] >= tG - 1 for f in feed], starts, stops))
    return steps


def _running(nets):
    return {(i, k): v.clone() for i, net in enumerate(nets) for k, v in net.state_dict().items()
            if 'running' in k or 'num_batches' in k}


def _restore(nets, state):
    with torch.no_grad():
        for i, net in enumerate(nets):
            sd = net.state_dict()
            for (j, k), v in state.items():
                if j == i:
                    sd[k].copy_(v)


def _run_slots(m, frames_of, steps, garbage):
    slots = m.stream_slots(B)
    got = {}
    for t, (feed, want_ready, starts, stops) in enumerate(steps):
        for k in stops:
            slots.stop(k)
        for k in starts:
            slots.start(k)
        rows = [frames_of(f[1], f[2]) if f is not None else garbage(t, k) for k, f in enumerate(feed)]
        out, ready = slots.step(torch.stack(rows).cuda())
        assert ready == want_ready, 'step %d: ready %s, expected %s' % (t, ready, want_ready)
        for k, f in enumerate(feed):
            if ready[k]:
                got.setdefault(f[1], []).append(out[k:k + 1].clone())
    return got


class _Clips:
    """Batch-1 per-clip state of the model (the stream windows and previous frames), so that the replay can interleave
    the clips step by step on the same modules."""
    KEYS = ('fake_B_prev', '_win_A', '_win_I', '_win_n')

    def __init__(self, m):
        self.m, self.state = m, {}

    def enter(self, c, fresh):
        if fresh:
            self.m.reset_stream()
        else:
            for k, v in self.state[c].items():
                setattr(self.m, k, v)

    def leave(self, c):
        self.state[c] = {k: getattr(self.m, k, None) for k in self.KEYS}


def _replay(m, steps, one_step):
    """Batch-1 run of every clip, interleaved step by step in slot order: each clip's frames, and the running statistics
    that order leaves."""
    clips, ref = _Clips(m), {}
    for feed, _, _, _ in steps:
        for f in feed:
            if f is None:
                continue
            _, c, j = f
            clips.enter(c, j == 0)
            r = one_step(c, j)
            if r is not None:
                ref.setdefault(c, []).append(r.clone())
            clips.leave(c)
    return ref


def _check(got, ref):
    assert sorted(got) == sorted(ref)
    for c in ref:
        assert len(got[c]) == len(ref[c]), c
        for j, (a, b) in enumerate(zip(got[c], ref[c])):
            assert torch.equal(a, b), 'clip %d frame %d: max |d| %.3g' % (c, j, (a - b).abs().max().item())


def _check_schedule(m, frames_of, garbage, one_step):
    tG = m.opt.n_frames_G
    steps = _plan_steps(tG)
    nets = [getattr(m, 'netG%d' % s) for s in range(m.n_scales)] + ([m.netG_i] if m.netG_i is not None else [])
    start = _running(nets)
    got = _run_slots(m, frames_of, steps, garbage)
    after_slots = _running(nets)
    _restore(nets, start)
    ref = _replay(m, steps, one_step)
    _check(got, ref)
    replayed = _running(nets)
    assert after_slots.keys() == replayed.keys() and after_slots
    for k in after_slots:
        assert torch.equal(after_slots[k], replayed[k]), k
    assert any(not torch.equal(start[k], replayed[k]) for k in start)
    # every clip produced a frame for each frame it fed from its tG-th on (clip 1 was restarted after three)
    fed = {}
    for feed, _, _, _ in steps:
        for f in feed:
            if f is not None:
                fed[f[1]] = f[2] + 1
    assert fed[1] == 3
    assert {c: len(v) for c, v in got.items()} == {c: n - tG + 1 for c, n in fed.items()}


@pytest.mark.parametrize('mode', TMC.MODES)
def test_street_slots_equal_each_clip_stream(mode):
    NW.set_default_precision(mode)
    try:
        m, clip = TMC._street()
        labels = [clip(c)[0][0, :, 0].to(torch.uint8) for c in range(len(SCHEDULE))]    # (frames, H, W) uint8 id maps
        g = torch.Generator().manual_seed(9)
        garbage = lambda t, k: torch.randint(0, 35, labels[0].shape[1:], generator=g, dtype=torch.uint8)
        _check_schedule(m, lambda c, j: labels[c][j], garbage,
                        lambda c, j: m.inference_stream(labels[c][j].cuda(), labels[c][j].cuda()))
    finally:
        NW.set_default_precision('precise')


@pytest.mark.parametrize('mode', TMC.MODES)
def test_pose_slots_equal_each_clip_inference(mode):
    NW.set_default_precision(mode)
    try:
        m, clip = TMC._pose()
        tG = m.opt.n_frames_G
        A = [clip(c)[0] for c in range(len(SCHEDULE))]                                    # (1, frames, 6, H, W)
        g = torch.Generator().manual_seed(9)
        garbage = lambda t, k: torch.rand(A[0].shape[2:], generator=g) * 2 - 1

        def one_step(c, j):
            if j < tG - 1:
                return None
            return m.inference(A[c][:, j - tG + 1:j + 1].cuda(), None, None)[0]
        _check_schedule(m, lambda c, j: A[c][0, j], garbage, one_step)
    finally:
        NW.set_default_precision('precise')


def test_slot_stream_u8_output_and_model_state():
    """out_u8 gives util.tensor2im of the float frames; the model's own stream state is untouched by a slot stream."""
    m, clip = TMC._street()
    lab = clip(0)[0][0, :, 0].to(torch.uint8).cuda()
    H, W = lab.shape[-2:]
    m.inference_stream(lab[0], lab[0])
    win = m._win_A.clone()
    slots, slots_f = m.stream_slots(B), m.stream_slots(B)
    out = torch.empty(B, H, W, 3, dtype=torch.uint8)
    for k in range(B):
        slots.start(k)
        slots_f.start(k)
    for t in range(4):
        fr = torch.stack([lab[t + k] for k in range(B)])
        o, ready = slots.step(fr, out_u8=out)
        f, ready_f = slots_f.step(fr)
        assert ready == ready_f == [t >= 2] * B
        torch.cuda.synchronize()
        ref = ((f.permute(0, 2, 3, 1) + 1) / 2 * 255).clamp(0, 255).to(torch.uint8).cpu()
        assert o is out and torch.equal(out, ref)
    assert torch.equal(m._win_A, win) and m._win_n == 1
    with pytest.raises(ValueError, match='runs 128x256 frames'):
        slots.step(torch.zeros(B, 64, 64, dtype=torch.uint8))


@pytest.mark.parametrize('mode', TMC.MODES)
def test_composite_flags_across_graph_replays_equal_the_raw_only_plans(mode):
    c = C.CASES['g0_small']
    net = det_fill_(C.build_module(c), seed=c['seed']).cuda()
    net.precision = mode
    net.sample_stats = True
    x = [torch.cat([t[i] for t in [TMC._clip_inputs(net, c, k) for k in range(B)]]) if i < 3 else None for i in range(6)]
    with torch.no_grad():
        warp = [o.clone() for o in net(*x, False)[:4] if o is not None]
        raw = [o.clone() for o in net(*x, True)[:4] if o is not None]
        flags = torch.zeros(B, dtype=torch.int32, device='cuda')
        A, R = L.IMAGE_ACTIVE, L.IMAGE_RAW_ONLY
        for fl in ([A, A | R, 0], [A | R, A, A | R], [0, 0, A], [A | R, A | R, A | R], [A, A, A]):   # eager, then graph replays
            flags.copy_(torch.tensor(fl, dtype=torch.int32))
            outs = [o for o in net(*x, False, image_flags=flags)[:4] if o is not None]
            for k in range(B):
                want = raw if fl[k] & R else warp
                for name, o, w in zip(('fake_B', 'flow', 'weight', 'fake_B_raw'), outs, want):
                    assert torch.equal(o[k], w[k]), '%s of image %d with flags %s' % (name, k, fl)
    assert not torch.equal(warp[0], raw[0])
    with pytest.raises(RuntimeError, match='no gradient'):
        net(*[t.requires_grad_() if i == 0 else t for i, t in enumerate(x)], False, image_flags=flags)
