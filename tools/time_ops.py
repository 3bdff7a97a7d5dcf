"""Times every HBM-bound stand-alone kernel of the hot path at its BASELINE-config size with CUDA events and reports achieved
GB/s against its ALGORITHMIC bytes (SURVEY 8d) and the H100 SXM data-sheet HBM3 bandwidth:  python tools/time_ops.py [op ...]"""
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import torch                                  # noqa: E402
from vid2vid_b200 import ops                  # noqa: E402
from vid2vid_b200 import networks as NW       # noqa: E402
from vid2vid_b200 import flownet as FN        # noqa: E402
from vid2vid_b200.plan import Plan            # noqa: E402

import bench                                  # noqa: E402
PEAK = bench.peaks()[1]
dev = torch.device('cuda', 0)
g = torch.Generator(device='cuda').manual_seed(0)
rnd = lambda *s: torch.rand(*s, device=dev, generator=g)


def timeit(fn, reps=int(os.environ.get("V2V_TIMEOPS_REPS", "20"))):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    big = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # > L2: flushed between repetitions
    best = 1e9
    for _ in range(reps):
        big.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def composite_case(H, W):
    plan = Plan(0)
    plan.composite(0, 1, 2, 3, 6, 4, 5, 6, 1, H, W, True, False)
    plan.finalize()
    io = [rnd(1, 3, H, W) * 2 - 1, (rnd(1, 2, H, W) - 0.5) * 8, rnd(1, 1, H, W), rnd(1, 6, H, W) * 2 - 1, rnd(1, 3, H, W) * 2 - 1,
          (rnd(1, 1, H, W) > 0.8).float(), torch.empty(1, 3, H, W, device=dev)]
    return (lambda: plan.run(io, False)), 76.0 * H * W


def cases():
    H, W = 1024, 2048
    lab = torch.randint(0, 35, (1, 3, 1, H, W), device=dev).float()
    oh = ops.onehot_edges(lab, lab, 35, True)
    c = {}
    c['onehot_edges 3x36x1024x2048'] = (lambda: ops.onehot_edges(lab, lab, 35, True), 3 * H * W * (36 * 4 + 8))
    c['avgpool3s2 108x1024x2048'] = (lambda: ops.avgpool3s2(oh), 108 * H * W * 5)
    c['fg_mask 1024x2048'] = (lambda: ops.fg_mask(oh, 2, [26]), H * W * 8)
    c['composite 1024x2048'] = composite_case(H, W)
    c['composite 256x512'] = composite_case(256, 512)
    img, flow = rnd(1, 3, H, W), (rnd(1, 2, H, W) - 0.5) * 8
    c['resample 3x1024x2048'] = (lambda: ops.resample(img, flow), H * W * 32)
    h, w = 512, 1024                      # FlowNet2 on a 1024x512 pair (BASELINE config 3)
    im, fl = rnd(1, 3, h, w), (rnd(1, 2, h, w) - 0.5) * 8
    c['resample2d 3x512x1024'] = (lambda: ops.resample2d(im, fl), h * w * 32)
    c['channelnorm 3x512x1024'] = (lambda: ops.channelnorm(im), h * w * 16)
    f1, f2 = rnd(1, 256, 64, 128), rnd(1, 256, 64, 128)
    c['correlation 256ch 64x128 -> 441'] = (lambda: ops.correlation(f1, f2, 20, 1, 20, 1, 2), 64 * 128 * 3812)
    fl4 = rnd(1, 2, h // 4, w // 4)
    c['upsample4 bilinear 2x128x256'] = (lambda: FN.resize(fl4, h, w, 'bilinear', True, mul=20.0, div=20.0), h * w * 2 * 4 * 2 + h * w // 16 * 8)
    a, b, m = rnd(1, 3, h, w), rnd(1, 3, h, w), (rnd(1, 1, h, w) > 0.5).float()
    c['masked l1 loss fwd 3x512x1024'] = (lambda: ops.l1_loss(a, b, m), h * w * 28)
    return c


def main():
    sel = sys.argv[1:]
    print('%-38s %10s %12s %10s %8s' % ('kernel @ size', 'us', 'alg MB', 'GB/s', 'of peak'))
    with torch.no_grad():
        for name, (fn, nbytes) in cases().items():
            if sel and not any(s in name for s in sel):
                continue
            ms = timeit(fn)
            gbs = nbytes / (ms * 1e-3) / 1e9
            extra = ''
            if name.startswith('correlation'):
                extra = '  (%.1f GFLOP/s fp32 FMA: 441 x 256 MAC per output pixel)' % (2 * 441 * 256 * 64 * 128 / (ms * 1e-3) / 1e9)
            print('%-38s %10.1f %12.1f %10.0f %7.1f%%%s' % (name, ms * 1e3, nbytes / 1e6, gbs, 100 * gbs / PEAK, extra), flush=True)


if __name__ == '__main__':
    main()
