"""Times the edge2face generator on one GPU at the demo size (512x512, precise mode) and prints one JSON line:

  first_frame_ms   one first frame: Encoder + nearest-neighbour features + Global_with_z (ngf 64, 9 residual blocks), as
                   Vid2VidModelG.get_face_features / generate_first_frame run it
  encoder_ms, features_ms, global_with_z_ms   its three parts
  frame_ms         one steady-state frame: the CompositeGenerator of scripts/face/test_512.sh (input_nc 15, 3 frames, ngf 128)
  gpu, power_limit the card and its power limit, read in the same run

CUDA events over repeated calls after warm-up; random-init weights and a synthetic features table.

    python tools/time_face.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from vid2vid_b200 import networks as NW, ops               # noqa: E402
from vid2vid_b200.utils import make_opt                    # noqa: E402

SIZE = 512          # the demo's square frames (tests/product_plans.py lowers the first-frame networks at this size)


def _ms(fn, reps, warm=3):
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


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--size', type=int, default=SIZE)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_face.py needs a CUDA device'
    NW.set_default_precision('precise')
    torch.manual_seed(0)
    H = W = a.size
    opt = make_opt(dataset_mode='face', label_nc=0, input_nc=15, feat_num=16, gpu_ids=[0])
    enc = NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []).cuda()
    gz = NW.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt).cuda()
    g0 = NW.build_netG(opt, 0).cuda()
    table, rows, num = NW.pack_face_features(NW.synthetic_face_features(64, 16, 0), 16)
    table = table.cuda()
    g = torch.Generator().manual_seed(1)
    B = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).cuda()
    inst = torch.randint(0, 7, (1, 1, H // 16, W // 16), generator=g).float()
    inst = inst.repeat_interleave(16, 2).repeat_interleave(16, 3).contiguous().cuda()
    x = (torch.rand(1, 15, H, W, generator=g) < 0.1).float().cuda()
    A = (torch.rand(1, 45, H, W, generator=g) < 0.1).float().cuda()
    prev = (torch.rand(1, 6, H, W, generator=g) * 2 - 1).cuda()
    with torch.no_grad():
        pooled = enc(B, inst)
        fmap, _ = ops.face_features(pooled, inst, table, rows, num)

        def first():
            p = enc(B, inst)
            f, _ = ops.face_features(p, inst, table, rows, num)
            return gz(x, f)
        res = {
            'first_frame_ms': _ms(first, a.reps),
            'encoder_ms': _ms(lambda: enc(B, inst), a.reps),
            'features_ms': _ms(lambda: ops.face_features(pooled, inst, table, rows, num), a.reps),
            'global_with_z_ms': _ms(lambda: gz(x, fmap), a.reps),
            'frame_ms': _ms(lambda: g0(A, prev, None, None, None, None, False), a.reps),
        }
    name, power = card()
    res.update(size='%dx%d' % (W, H), precision='precise', gpu=name, power_limit=power)
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == '__main__':
    main()
