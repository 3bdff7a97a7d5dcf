"""Times Vid2VidModelG.inference on B clips at once (per-sample-statistics plans, every clip bit-identical to its own run)
against one clip, on one GPU, and prints one JSON line per (workload, mode, B):

  fps_total     generated frames per second summed over the B clips (steady-state frames: the first frames are warm-up)
  fps_per_clip  frames per second each clip advances
  speedup       fps_total over the B = 1 run of the same workload and mode
  arena_bytes   plan arena bytes of the generator plans the B-clip run uses
  gpu, power_limit   the card and its power limit, read in the same run

Workloads (random-init weights, synthetic inputs; the first frames come from the real-frame input, --use_real_img, so no
first-frame generator weights are needed; steady-state frames run the same generators as with --use_single_G):
  street_512   label2city 512x256, n_scales_spatial 1, --fg (bench.py cfg2)
  pose_512     pose2body H512 x W256, input_nc 6, n_scales_spatial 2, --fg --fg_labels 2 --no_first_img (cfg5 geometry)
  face_512     edge2face 512x512, input_nc 15 (scripts/face/test_512.sh)
  street_2048  label2city 2048x1024, n_scales_spatial 3, --fg (bench.py cfg4), B in {1, 2} only

Each B > 1 run is preceded by a B = 1 run of the same workload and mode in the same process (alternated, --rounds times);
the reported numbers are the medians over the rounds.  CUDA events around --frames frames after --warmup frames.

    python tools/time_multiclip.py [--frames 40] [--warmup 5] [--rounds 2] [--only street_512,pose_512]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from vid2vid_b200 import networks as NW                    # noqa: E402
from vid2vid_b200.model_g import Vid2VidModelG             # noqa: E402
from vid2vid_b200.utils import make_opt, synth_label_sequence   # noqa: E402

WORKLOADS = {
    'street_512': dict(H=256, W=512, bs=(1, 2, 4, 8), opt=dict(label_nc=35, use_instance=True, fg=True, fg_labels=[26],
                                                                n_scales_spatial=1, ngf=128)),
    'pose_512': dict(H=512, W=256, bs=(1, 2, 4, 8), opt=dict(label_nc=0, input_nc=6, fg=True, fg_labels=[2], n_scales_spatial=2,
                                                              ngf=128, no_first_img=True)),
    'face_512': dict(H=512, W=512, bs=(1, 2, 4, 8), opt=dict(label_nc=0, input_nc=15, dataset_mode='face', n_scales_spatial=1,
                                                              ngf=128)),
    'street_2048': dict(H=1024, W=2048, bs=(1, 2), opt=dict(label_nc=35, use_instance=True, fg=True, fg_labels=[26],
                                                            n_scales_spatial=3, ngf=128)),
}


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def clip_inputs(wl, b, n, seed):
    """(A, B, inst) of b clips over n frames: (b, n, C, H, W) id maps / pose maps / edge maps, and real frames."""
    w = WORKLOADS[wl]
    H, W, o = w['H'], w['W'], w['opt']
    g = torch.Generator().manual_seed(seed)
    if o['label_nc']:
        A = torch.cat([synth_label_sequence(n, H, W, label_nc=o['label_nc'], block=16, seed=seed + k) for k in range(b)])
        inst = A
    elif o.get('dataset_mode') == 'face':
        A = (torch.rand(b, n, o['input_nc'], H, W, generator=g) < 0.1).float()
        inst = torch.cat([synth_label_sequence(n, H, W, label_nc=7, block=16, seed=seed + k) for k in range(b)])   # part map
    else:
        A = torch.rand(b, n, o['input_nc'], H, W, generator=g) * 2 - 1
        A[..., :H // 4, :] = 0
        inst = None
    real = torch.rand(b, n, 3, H, W, generator=g) * 2 - 1
    return A.cuda(), real.cuda(), inst.cuda() if inst is not None else None


def make_model(wl):
    o = dict(WORKLOADS[wl]['opt'])
    opt = make_opt(use_single_G=False, use_real_img=not o.get('no_first_img', False), gpu_ids=[0], synthetic_weights=True, **o)
    m = Vid2VidModelG().initialize(opt)
    for s in range(m.n_scales):
        net = getattr(m, 'netG%d' % s)
        torch.manual_seed(s)
        with torch.no_grad():                          # small flow heads: random ones give multi-pixel noise flows
            for head in ('model_final_flow',):
                if hasattr(net, head):
                    getattr(net, head)[1].weight.mul_(0.05)
                    getattr(net, head)[1].bias.mul_(0.05)
    return m


def run(m, wl, b, frames, warmup):
    """(frames/s over all clips, frames/s per clip, arena bytes of the plans the run built)"""
    tG = m.opt.n_frames_G
    A, real, inst = clip_inputs(wl, b, frames + warmup + tG, seed=b)
    win = lambda x, t: x[:, t:t + tG] if x is not None else None
    nets = [getattr(m, 'netG%d' % s) for s in range(m.n_scales)]
    for net in nets:                                   # only this run's plans hold device memory
        net._plans().clear()
    torch.cuda.empty_cache()
    m.reset_stream()
    for t in range(warmup):
        m.inference(win(A, t), win(real, t), win(inst, t))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(warmup, warmup + frames):
        m.inference(win(A, t), win(real, t), win(inst, t))
    e1.record()
    torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3
    return b * frames / s, frames / s, sum(e['plan'].workspace_bytes for net in nets for e in net._plans().values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--modes', default='precise,fast')
    ap.add_argument('--only', default='')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_multiclip.py needs a CUDA device'
    name, power = card()
    for wl in (a.only.split(',') if a.only else WORKLOADS):
        m = make_model(wl)
        for mode in a.modes.split(','):
            NW.set_default_precision(mode)
            bs = WORKLOADS[wl]['bs']
            res = {b: [] for b in bs}
            for _ in range(a.rounds):
                for b in bs[1:]:                       # B = 1, then B, alternated
                    res[1].append(run(m, wl, 1, a.frames, a.warmup))
                    res[b].append(run(m, wl, b, a.frames, a.warmup))
            base = statistics.median(r[0] for r in res[1])
            for b in bs:
                tot = statistics.median(r[0] for r in res[b])
                print(json.dumps({'workload': wl, 'mode': mode, 'B': b, 'fps_total': round(tot, 2),
                                  'fps_per_clip': round(statistics.median(r[1] for r in res[b]), 2),
                                  'speedup': round(tot / base, 3), 'arena_bytes': res[b][-1][2],
                                  'gpu': name, 'power_limit': power}), flush=True)
        del m
        torch.cuda.empty_cache()
    NW.set_default_precision('precise')


if __name__ == '__main__':
    main()
