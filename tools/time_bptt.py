"""Times back-propagation into previously generated frames and the fixed-global-scale mode on one GPU; prints one JSON line:

  composite_bwd_us  composite_bwd_kernel alone (torch.profiler, CUDA activity) at 1 x 2048 x 1024 with img_prev of 6 channels,
                    fg on, for moderate flows (uniform within +-8 px) and border-saturating ones (+-1000 px: every pixel samples
                    a frame corner, as randomly initialised x20 flow heads do), without and with the img_prev gradient (d_prev)
  train_step_ms     the cfg3-geometry training step (1024x512, two spatial scales, ngf 128, num_D 3, two temporal scales, two
                    generated frames per step, random-init weights) in three settings of ONE trainer, alternated over `--rounds`
                    windows of `--steps` steps: n_frames_bp 1, n_frames_bp 2, and niter_fix_global 1 (only the finest scale
                    trains; the coarse scale runs its inference plan); CUDA events around whole steps after warm-up
  gpu, power_limit  the card the numbers were measured on

    python tools/time_bptt.py [--steps 6] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from vid2vid_b200.networks import S_FG, S_FINAL, S_FLOW, S_MASK, S_PREV, S_RAW, S_RAWC, S_W      # noqa: E402
from vid2vid_b200.plan import Plan                                                              # noqa: E402


def _kernel_us(prof, name):
    for k in prof.key_averages():
        if name in k.key:
            t = getattr(k, 'device_time_total', None)
            if t is None:
                t = k.cuda_time_total
            return t / k.count
    raise RuntimeError('no %s kernel in the trace' % name)


def composite_bwd_us(flow_kind, with_prev, N=1, H=1024, W=2048, pc=6, reps=50):
    from torch.profiler import ProfilerActivity, profile
    g = torch.Generator().manual_seed(3)
    if flow_kind == 'moderate':
        flow = (torch.rand(N, 2, H, W, generator=g) * 2 - 1) * 8
    else:
        flow = torch.sign(torch.randn(N, 2, H, W, generator=g)) * 1e3
    plan = Plan(0, precision='precise', train=True)
    plan.input(S_PREV, N, pc, 0, pc, H, W)
    plan.composite(S_RAW, S_FLOW, S_W, S_PREV, pc, S_FG, S_MASK, S_FINAL, N, H, W, True, False, s_raw_out=S_RAWC)
    plan.finalize()
    r = lambda c: (torch.rand(N, c, H, W, generator=g) * 2 - 1).cuda()
    io = [None] * 15
    io[S_RAW], io[S_FLOW], io[S_W], io[S_PREV], io[S_FG] = r(3), flow.cuda(), r(1).abs(), r(pc), r(3)
    io[S_MASK] = (torch.rand(N, 1, H, W, generator=g) > 0.8).float().cuda()
    io[S_FINAL], io[S_RAWC] = torch.empty(N, 3, H, W, device='cuda'), torch.empty(N, 3, H, W, device='cuda')
    plan.run(io, False)
    gio = [None] * 15
    gio[S_FINAL] = r(3)
    if with_prev:
        gio[S_PREV] = torch.zeros(N, pc, H, W, device='cuda')
    for _ in range(5):
        plan.backward(io, gio, [], [])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            plan.backward(io, gio, [], [])
        torch.cuda.synchronize()
    return _kernel_us(prof, 'composite_bwd_kernel')


def train_steps(steps, rounds, H=512, W=1024):
    from vid2vid_b200 import flownet as FN
    from vid2vid_b200.model_d import Vid2VidModelD
    from vid2vid_b200.model_g import Vid2VidModelG, _adam
    from vid2vid_b200.trainer import Trainer
    from vid2vid_b200.utils import make_opt, synth_label_sequence
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=2, ngf=128, num_D=3, n_scales_temporal=2,
                   n_frames_D=3, isTrain=True, no_vgg=True, gpu_ids=[0], n_frames_total=30, dataroot='datasets/Cityscapes/',
                   loadSize=W, max_frames_per_gpu=2, max_frames_backpropagate=2)
    torch.manual_seed(1234)
    G, D, F = Vid2VidModelG().initialize(opt), Vid2VidModelD().initialize(opt), FN.FlowNet().initialize(opt)
    tr = Trainer(opt, G, D, F, world=1)
    tG, nf = opt.n_frames_G, G.n_frames_load
    T = 40
    A = synth_label_sequence(T, H, W, label_nc=35, block=64, seed=0).cuda()
    g = torch.Generator().manual_seed(77)
    coarse = torch.rand(T, 3, H // 16, W // 16, generator=g) * 2 - 1
    B = torch.nn.functional.interpolate(coarse, size=(H, W), mode='bilinear', align_corners=False).view(1, T, 3, H, W).cuda()
    optimizers = {True: G.optimizer_G, False: _adam(G.netG1.parameters(), lr=opt.lr, betas=(opt.beta1, 0.999))}
    settings = {'n_frames_bp_1': (1, True), 'n_frames_bp_2': (2, True), 'niter_fix_global_1': (1, False)}
    pos = [0]

    def run(name, n):
        G.n_frames_bp, G.finetune_all = settings[name]
        G.optimizer_G = optimizers[G.finetune_all]
        for _ in range(n):
            t = pos[0] % (T - tG - nf)
            if t == 0:
                tr.reset_clip()
            tr.step(A[:, t:t + tG + nf - 1], B[:, t:t + tG + nf - 1], A[:, t:t + tG + nf - 1])
            pos[0] += nf

    for name in settings:
        run(name, 8)                              # every plan, both temporal scales and the allocator warmed up
    torch.cuda.synchronize()
    times = {name: [] for name in settings}
    for _ in range(rounds):
        for name in settings:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(name, steps)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    return {name: {'ms': [round(x, 2) for x in v], 'median': sorted(v)[rounds // 2]} for name, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=6)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True).stdout.strip()
    comp = {'%s_%s' % (k, 'with_d_prev' if p else 'without'): composite_bwd_us(k, p) for k in ('moderate', 'saturating') for p in (False, True)}
    out = {'gpu': torch.cuda.get_device_name(0), 'power_limit': limit, 'composite_bwd_us': comp,
           'train_step_ms': train_steps(args.steps, args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
