"""Times a slot stream (Vid2VidModelG.stream_slots: B slots whose clips start and stop independently, every clip
bit-identical to its own run) under a traffic mix of clips of seeded random lengths, and prints one JSON line per
(workload, mode, B):

  fps_total       frames produced per second over all slots
  occupancy       frames produced / slot-steps
  step_ms_p50 / step_ms_p99   step times (a join step includes its first-frame generation)
  speedup         fps_total over the same clips run one after another at B = 1 (a one-slot stream)
  gpu, power_limit   the card and its power limit, read in the same run

Workloads (random-init weights, synthetic inputs):
  street_512   label2city 512x256, n_scales_spatial 1, --fg --use_instance --use_single_G (netG_i: the 512 'global'
               first-frame generator, run at batch 1 for every joining clip)
  pose_512     pose2body H512 x W256, input_nc 6, n_scales_spatial 2, --fg --fg_labels 2 --no_first_img

A new clip takes a slot as soon as the slot's clip ends.  Each B > 1 run is preceded by the B = 1 run of the same clips in
the same process.  Each step ends in a device synchronise, so the step times are device-bound step latencies.

    python tools/time_slots.py [--clips 24] [--min-len 30] [--max-len 120] [--only pose_512] [--modes precise,fast]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import time_multiclip as TM                                # noqa: E402
from vid2vid_b200 import networks as NW                    # noqa: E402
from vid2vid_b200.model_g import Vid2VidModelG             # noqa: E402
from vid2vid_b200.utils import make_opt, synth_label_sequence   # noqa: E402

WORKLOADS = {
    'street_512': dict(H=256, W=512, bs=(2, 4, 8), opt=dict(TM.WORKLOADS['street_512']['opt'], use_single_G=True,
                                                           dataroot='datasets/Cityscapes/', loadSize=512)),
    'pose_512': dict(H=512, W=256, bs=(2, 4, 8), opt=dict(TM.WORKLOADS['pose_512']['opt'])),
}


def make_model(wl):
    opt = make_opt(gpu_ids=[0], synthetic_weights=True, **WORKLOADS[wl]['opt'])
    m = Vid2VidModelG().initialize(opt)
    for s in range(m.n_scales):
        with torch.no_grad():                          # small flow heads: random ones give multi-pixel noise flows
            getattr(m, 'netG%d' % s).model_final_flow[1].weight.mul_(0.05)
            getattr(m, 'netG%d' % s).model_final_flow[1].bias.mul_(0.05)
    return m


def frame_bank(wl, n=16, seed=0):
    """n distinct device frames a clip cycles through (the generators' cost does not depend on the content)."""
    w = WORKLOADS[wl]
    H, W, o = w['H'], w['W'], w['opt']
    if o['label_nc']:
        return synth_label_sequence(n, H, W, label_nc=o['label_nc'], block=16, seed=seed)[0, :, 0].to(torch.uint8).cuda()
    g = torch.Generator().manual_seed(seed)
    A = torch.rand(n, o['input_nc'], H, W, generator=g) * 2 - 1
    A[..., :H // 4, :] = 0
    return A.cuda()


def run(m, bank, lengths, B):
    """Feeds the clips (lengths in frames) through a B-slot stream, a new clip taking the first free slot.  Returns
    (frames produced, slot-steps, wall seconds, per-step seconds)."""
    slots = m.stream_slots(B)
    queue = list(enumerate(lengths))
    left = [0] * B                                     # frames the slot's clip still has to feed
    offset = [0] * B
    produced = slot_steps = 0
    times = []
    frames = torch.empty((B,) + tuple(bank.shape[1:]), dtype=bank.dtype, device='cuda')
    torch.cuda.synchronize()
    t_all = time.perf_counter()
    while queue or any(left):
        for k in range(B):
            if left[k] == 0 and queue:
                c, n = queue.pop(0)
                slots.start(k)
                left[k], offset[k] = n, c
            elif left[k] == 0:
                slots.stop(k)
        for k in range(B):
            frames[k] = bank[(offset[k] + left[k]) % bank.shape[0]]
        t0 = time.perf_counter()
        _, ready = slots.step(frames)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        produced += sum(ready)
        slot_steps += B
        left = [max(n - 1, 0) for n in left]
    return produced, slot_steps, time.perf_counter() - t_all, times


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(q / 100 * (len(xs) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=24)
    ap.add_argument('--min-len', dest='min_len', type=int, default=30)
    ap.add_argument('--max-len', dest='max_len', type=int, default=120)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--modes', default='precise,fast')
    ap.add_argument('--only', default='')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_slots.py needs a CUDA device'
    name, power = TM.card()
    rng = random.Random(a.seed)
    lengths = [rng.randint(a.min_len, a.max_len) for _ in range(a.clips)]
    for wl in (a.only.split(',') if a.only else WORKLOADS):
        m = make_model(wl)
        bank = frame_bank(wl)
        for mode in a.modes.split(','):
            NW.set_default_precision(mode)
            for B in WORKLOADS[wl]['bs']:
                run(m, bank, [m.opt.n_frames_G + 2] * B, B)            # warm-up: builds and captures this B's plans
                run(m, bank, [m.opt.n_frames_G + 2], 1)
                p1, _, s1, _ = run(m, bank, lengths, 1)
                pb, steps, sb, times = run(m, bank, lengths, B)
                assert p1 == pb == sum(n - m.opt.n_frames_G + 1 for n in lengths)
                print(json.dumps({'workload': wl, 'mode': mode, 'B': B, 'clips': len(lengths), 'fps_total': round(pb / sb, 2),
                                  'occupancy': round(pb / steps, 3), 'step_ms_p50': round(1e3 * statistics.median(times), 2),
                                  'step_ms_p99': round(1e3 * pct(times, 99), 2), 'speedup': round((pb / sb) / (p1 / s1), 3),
                                  'gpu': name, 'power_limit': power}), flush=True)
        del m
        torch.cuda.empty_cache()
    NW.set_default_precision('precise')


if __name__ == '__main__':
    main()
