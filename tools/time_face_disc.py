"""Times the pose demo's face discriminator (--add_face_disc) on one GPU and prints one JSON line:

  train_step_ms     a pose-512p-shaped training step (512x512, label_nc 0, input_nc 6, no_first_img, two spatial scales,
                    num_D 3, fineSize 512 so the face crop is 128x128, ngf 128 / ndf 64, random-init weights) with
                    add_face_disc off and on, the two alternated over `--rounds` windows of `--steps` steps each; CUDA
                    events around whole steps after 12 warm-up steps each, so the host wait for the face box is included
  face_region_us    ops.face_region alone on the step's merged batch (1 x 6 x 512 x 512) and on 8 x 6 x 1024 x 1024: CUDA
                    events over back-to-back calls (reset + search kernels, the 20-byte copy and the host work of each call;
                    no host wait), so small inputs measure the per-call overhead rather than the kernel
  gpu, power_limit  the card the numbers were measured on

    python tools/time_face_disc.py [--steps 10] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from vid2vid_b200 import ops                                  # noqa: E402
from oracle import face_disc_oracle as FD                      # noqa: E402

# The measured step's options (tests/product_plans.py lowers the same networks at the same size for the conv census).
SIZE = 512
OPT = dict(label_nc=0, input_nc=6, use_instance=False, fg=False, n_scales_spatial=2, ngf=128, ndf=64, num_D=3, n_scales_temporal=2,
           isTrain=True, no_vgg=True, n_frames_total=12, no_first_img=True, dataroot='datasets/pose', dataset_mode='pose')


def _trainer(add_face_disc, H, W):
    from vid2vid_b200 import flownet as FN
    from vid2vid_b200.model_d import Vid2VidModelD
    from vid2vid_b200.model_g import Vid2VidModelG
    from vid2vid_b200.trainer import Trainer
    from vid2vid_b200.utils import make_opt
    opt = make_opt(gpu_ids=[0], add_face_disc=add_face_disc, fineSize=H, loadSize=H, **OPT)
    torch.manual_seed(1234)
    G, D, F = Vid2VidModelG().initialize(opt), Vid2VidModelD().initialize(opt), FN.FlowNet().initialize(opt)
    return Trainer(opt, G, D, F, world=1), opt


def train_steps(H, W, steps, rounds):
    T = 40
    A, B = FD.pose_clip(T, H, W, 5, blob_rows=(100, 160), blob_cols=(200, 260))
    A, B = A.cuda(), B.cuda()
    runs = {flag: _trainer(flag, H, W) for flag in (False, True)}
    pos = {False: 0, True: 0}

    def run(flag, n):
        tr, opt = runs[flag]
        tG = opt.n_frames_G
        for _ in range(n):
            t = pos[flag] % (T - tG)
            if t == 0:
                tr.reset_clip()
            tr.step(A[:, t:t + tG], B[:, t:t + tG], A[:, t:t + tG])
            pos[flag] += 1

    for flag in (False, True):
        run(flag, 12)                         # every shape, both temporal scales and the allocator warmed up
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(rounds):
        for flag in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(flag, steps)
            e1.record()
            torch.cuda.synchronize()
            times[flag].append(e0.elapsed_time(e1) / steps)
    return {'face_disc_off': times[False], 'face_disc_on': times[True],
            'median_off': sorted(times[False])[rounds // 2], 'median_on': sorted(times[True])[rounds // 2]}


def region_us(N, H, W, reps=200):
    x = FD.pose_maps(N, H, W, 9, (N - 1, H // 4, H // 4 + 40, W // 3, W // 3 + 30)).cuda()
    for _ in range(10):
        ops.face_region(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        h = ops.face_region(x)
    e1.record()
    torch.cuda.synchronize()
    assert h.get() == FD.face_box(x.cpu(), False)
    return 1e3 * e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True).stdout.strip()
    out = {'gpu': torch.cuda.get_device_name(0), 'power_limit': limit,
           'face_region_us': {'1x6x512x512': region_us(1, 512, 512), '8x6x1024x1024': region_us(8, 1024, 1024)},
           'train_step_ms': train_steps(SIZE, SIZE, args.steps, args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
