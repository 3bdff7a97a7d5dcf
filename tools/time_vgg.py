"""Times the VGG19 perceptual loss (networks.VGGLoss, precise mode) on one GPU and prints one JSON line:

  loss_ms          forward and forward + backward ms per VGGLoss call at 1024x512 and 2048x1024 (the latter includes the
                   2x2 downsample), CUDA events over repeated calls after warm-up
  conv_rate        algorithmic conv TFLOP/s of the loss plan at 1024x512: 2 * MACs over the summed conv-kernel time of
                   plan.profile() (eager launches with an event after each kernel)
  train_step_ms    the cfg3 training step (bench.py's configuration: 1024x512, two spatial scales, ngf 128) with no_vgg on
                   and off, random-init weights

    python tools/time_vgg.py [--steps 10] [--no-train]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from vid2vid_b200 import networks as NW                     # noqa: E402

LOSS_SIZES = ((512, 1024), (1024, 2048))      # (H, W) of the timed loss calls; tests/product_plans.py lowers their plans


def _ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def loss_times(crit, H, W, reps):
    g = torch.Generator().manual_seed(H + W)
    x = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda()
    y = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda()
    xr = x.clone().requires_grad_(True)

    def fwd():
        with torch.no_grad():
            crit(x, y)

    def fwd_bwd():
        crit(xr, y).backward()
        xr.grad = None
    return {'forward_ms': _ms(fwd, reps), 'forward_backward_ms': _ms(fwd_bwd, reps)}


def conv_rate(crit, H, W):
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda()
    y = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda()
    with torch.no_grad():
        crit.vgg.feature_l1(x, y)
    ent = [e for k, e in crit.vgg._plans().items() if k[0] == 'VGGL' and k[2:4] == (H, W) and 'train' not in k][0]
    plan = ent['plan']
    plan.profile()                                            # (first eager pass: module loading)
    prof = plan.profile()
    conv = [(ms, macs) for kind, ms, macs in prof if kind == 1]
    ms = sum(m for m, _ in conv)
    macs = sum(a for _, a in conv)
    return {'conv_ms': ms, 'all_kernels_ms': sum(m for _, m, _ in prof), 'gmac': macs / 1e9,
            'tflops': 2 * macs / (ms * 1e-3) / 1e12, 'n_convs': len(conv)}


def train_step_ms(no_vgg, steps):
    from vid2vid_b200 import flownet as FN
    from vid2vid_b200.model_d import Vid2VidModelD
    from vid2vid_b200.model_g import Vid2VidModelG
    from vid2vid_b200.trainer import Trainer
    from vid2vid_b200.utils import make_opt, synth_label_sequence
    H, W = 512, 1024
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=2, ngf=128, num_D=3, n_scales_temporal=2,
                   n_frames_D=3, isTrain=True, no_vgg=no_vgg, gpu_ids=[0], n_frames_total=30, dataroot='datasets/Cityscapes/', loadSize=W)
    torch.manual_seed(1234)
    G, D, F = Vid2VidModelG().initialize(opt), Vid2VidModelD().initialize(opt), FN.FlowNet().initialize(opt)
    tr = Trainer(opt, G, D, F, world=1)
    tG, warm = opt.n_frames_G, opt.n_frames_D ** (opt.n_scales_temporal - 1) * (opt.n_frames_D - 1) + 3
    T = steps + warm + tG + 2
    A = synth_label_sequence(T, H, W, label_nc=35, block=64, seed=0)
    g = torch.Generator().manual_seed(77)
    B = torch.nn.functional.interpolate(torch.rand(T, 3, H // 16, W // 16, generator=g) * 2 - 1, size=(H, W), mode='bilinear',
                                        align_corners=False).view(1, T, 3, H, W)
    t = 0
    for _ in range(warm):
        tr.step(A[:, t:t + tG].cuda(), B[:, t:t + tG].cuda(), A[:, t:t + tG].cuda())
        t += 1
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.step(A[:, t:t + tG].cuda(), B[:, t:t + tG].cuda(), A[:, t:t + tG].cuda())
        t += 1
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del tr, G, D, F
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--no-train', action='store_true')
    args = ap.parse_args()
    crit = NW.VGGLoss(0, synthetic=True)
    crit.vgg.precision = 'precise'
    out = {'gpu': torch.cuda.get_device_name(0), 'precision': 'precise',
           'loss_ms': {'%dx%d' % (W, H): loss_times(crit, H, W, args.reps) for H, W in LOSS_SIZES},
           'conv_rate_1024x512': conv_rate(crit, 512, 1024)}
    if not args.no_train:
        del crit
        torch.cuda.empty_cache()
        out['train_step_ms'] = {'cfg3_no_vgg': train_step_ms(True, args.steps), 'cfg3_vgg': train_step_ms(False, args.steps)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
