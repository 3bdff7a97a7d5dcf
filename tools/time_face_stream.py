"""Times Vid2VidModelG.inference_stream on the edge2face and pose2body demos on one GPU and prints one JSON line per
(workload, B):

  fps_total      generated frames per second summed over the B clips, each step uploading the newest frame and writing
                 uint8 RGB on the device (out_u8), after the window filled and the first frames were generated
  fps_per_clip   frames per second each clip advances
  first_ms       the step that generates the first frames (face: Encoder, per-clip features and Global_with_z on the B clips)
  gpu, power_limit   the card and its power limit, read in the same run

Workloads (random-init weights, synthetic inputs and features table, precise mode):
  face_512   scripts/face/test_512.sh: 512x512, --input_nc 15 --use_single_G (ngf 128, one scale), B in {1, 4}
  pose_1024  scripts/pose/test_1024p.sh: H 1024 x W 512, --input_nc 6 --n_scales_spatial 3 --no_first_img, B = 1

CUDA events around --frames steps after --warmup steps.

    python tools/time_face_stream.py [--frames 30] [--warmup 5] [--only face_512]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from vid2vid_b200 import networks as NW                    # noqa: E402
from vid2vid_b200.model_g import Vid2VidModelG             # noqa: E402
from vid2vid_b200.utils import make_opt, synth_label_sequence   # noqa: E402
from time_multiclip import card                            # noqa: E402

WORKLOADS = {
    'face_512': dict(H=512, W=512, bs=(1, 4), opt=dict(dataset_mode='face', dataroot='datasets/face/', label_nc=0, input_nc=15,
                                                        use_single_G=True, n_scales_spatial=1)),
    'pose_1024': dict(H=1024, W=512, bs=(1,), opt=dict(dataset_mode='pose', dataroot='datasets/pose/', label_nc=0, input_nc=6,
                                                       n_scales_spatial=3, no_first_img=True)),
}


def make_opt_for(wl):
    return make_opt(gpu_ids=[0], synthetic_weights=True, **WORKLOADS[wl]['opt'])


def frames(wl, b, n, seed):
    """(A, real, part) of b clips over n frames, on the host in pinned memory: (n, b, C, H, W) dense frames, and for face
    (n, b, 3, H, W) real frames and (n, b, H, W) uint8 part maps."""
    w = WORKLOADS[wl]
    H, W, o = w['H'], w['W'], w['opt']
    g = torch.Generator().manual_seed(seed)
    if o['dataset_mode'] == 'face':
        A = (torch.rand(n, b, o['input_nc'], H, W, generator=g) < 0.1).float()
        part = torch.cat([synth_label_sequence(n, H, W, label_nc=7, block=16, seed=seed + k) for k in range(b)])
        part = part[:, :, 0].transpose(0, 1).to(torch.uint8)
        real = torch.rand(n, b, 3, H, W, generator=g) * 2 - 1
        return A.pin_memory(), real.pin_memory(), part.pin_memory()
    A = torch.rand(n, b, o['input_nc'], H, W, generator=g) * 2 - 1
    A[..., :H // 4, :] = 0
    return A.pin_memory(), None, None


def run(m, wl, b, n_frames, warmup):
    tG = m.opt.n_frames_G
    A, real, part = frames(wl, b, tG + warmup + n_frames, seed=b)
    sq = (lambda x: x[0]) if b == 1 else (lambda x: x)
    out = torch.empty(((b,) if b > 1 else ()) + (WORKLOADS[wl]['H'], WORKLOADS[wl]['W'], 3), dtype=torch.uint8).pin_memory()
    m.reset_stream()
    for t in range(tG - 1):                                # the window fills (face: with the real frames and part maps)
        m.inference_stream(sq(A[t]), out_u8=out, **({} if real is None else dict(real_frame=sq(real[t]), inst_frame=sq(part[t]))))
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    e[0].record()                                          # first frames, then the first generated frame
    m.inference_stream(sq(A[tG - 1]), out_u8=out)
    e[1].record()
    for t in range(tG, tG + warmup):
        m.inference_stream(sq(A[t]), out_u8=out)
    torch.cuda.synchronize()
    e[2].record()
    for t in range(tG + warmup, A.shape[0]):
        m.inference_stream(sq(A[t]), out_u8=out)
    e[3].record()
    torch.cuda.synchronize()
    s = e[2].elapsed_time(e[3]) / 1e3
    return b * n_frames / s, n_frames / s, e[0].elapsed_time(e[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--only', default='')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_face_stream.py needs a CUDA device'
    NW.set_default_precision('precise')
    name, power = card()
    for wl in (a.only.split(',') if a.only else WORKLOADS):
        torch.manual_seed(0)
        m = Vid2VidModelG().initialize(make_opt_for(wl))
        for b in WORKLOADS[wl]['bs']:
            run(m, wl, b, 2, 1)                            # plans, graphs and first-launch module loads of this B
            tot, per, first = run(m, wl, b, a.frames, a.warmup)
            print(json.dumps({'workload': wl, 'B': b, 'fps_total': round(tot, 2), 'fps_per_clip': round(per, 2),
                              'first_ms': round(first, 2), 'size': '%dx%d' % (WORKLOADS[wl]['W'], WORKLOADS[wl]['H']),
                              'precision': 'precise', 'gpu': name, 'power_limit': power}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
