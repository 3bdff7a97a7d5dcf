"""Times single conv units through the plan runtime (CUDA events around the conv kernel only)."""
import os, sys
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import torch, torch.nn as nn
from vid2vid_b200 import networks as NW

BN = NW.get_norm_layer('batch')
SHAPES = {
    'c1024': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(1024, 1024, 3), BN(1024), nn.ReLU(True)], (1, 1024, 32, 64)),
    'c512': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(512, 512, 3), BN(512), nn.ReLU(True)], (1, 512, 32, 64)),
    'c128_256x512': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 256, 512)),
    'c64_512x1024': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)], (1, 64, 512, 1024)),
    'stem108_32': (lambda: NW._stem(108, 32, BN), (1, 108, 1024, 2048)),
    'stem108_48': (lambda: NW._stem(108, 48, BN), (1, 108, 1024, 2048)),
    'stem108_96': (lambda: NW._stem(108, 96, BN), (1, 108, 512, 1024)),
    'stem108_192': (lambda: NW._stem(108, 192, BN), (1, 108, 256, 512)),
    'head32_2048': (lambda: [nn.ReflectionPad2d(3), nn.Conv2d(32, 3, 7), nn.Tanh()], (1, 32, 1024, 2048)),
    'up64_32': (lambda: [nn.ConvTranspose2d(64, 32, 3, stride=2, padding=1, output_padding=1), BN(32), nn.ReLU(True)], (1, 64, 512, 1024)),
    'c32_512x1024': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(32, 32, 3), BN(32), nn.ReLU(True)], (1, 32, 512, 1024)),
}
names = sys.argv[1:] or list(SHAPES)
for n in names:
    build, shape = SHAPES[n]
    net = NW.SequentialRunner(build()).cuda()
    x = torch.randn(*shape, device='cuda')
    with torch.no_grad():
        net(x); net(x)
        plan = list(net._plans().values())[0]['plan']
        best = None
        for _ in range(5):
            prof = plan.profile()
            ms = [p[1] for p in prof if p[0] == 1]
            macs = [p[2] for p in prof if p[0] == 1]
            best = ms if best is None else [min(a, b) for a, b in zip(best, ms)]
    print('%-14s conv_ms=%s TF=%s' % (n, ['%.4f' % m for m in best], ['%.1f' % (2 * a / (m * 1e-3) / 1e12) for a, m in zip(macs, best)]), flush=True)
