"""Tensor-core backward vs the fp32 SIMT backward on single conv units: per-tap / per-channel-block error of dW and the
error of dX.  Usage: python tools/debug/wgrad_check.py [unit ...]"""
import os, sys
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..', '..'))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch, torch.nn as nn
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import det_fill_
BN = NW.get_norm_layer('batch')
UNITS = {
    'c128': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 12, 72)),
    'c64': (lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)], (1, 64, 8, 16)),
    'down': (lambda: NW._down(64, 128, BN), (1, 64, 16, 80)),
    'up': (lambda: NW._up(128, 64, BN), (1, 128, 8, 40)),
}


def grads(build, x, mode):
    if mode == 'simt': os.environ['V2V_BWD'] = 'simt'
    else: os.environ.pop('V2V_BWD', None)
    r = det_fill_(NW.SequentialRunner(build()), seed=5).cuda(); r.precision = 'precise'
    xr = x.clone().requires_grad_(True)
    out = r(xr)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).cuda()
    (out * g).sum().backward()
    return xr.grad.clone(), [p for p in r.parameters() if p.dim() == 4][0].grad.clone()


for name in (sys.argv[1:] or list(UNITS)):
    build, shape = UNITS[name]
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1)).cuda()
    dx_t, dw_t = grads(build, x, 'tensor')
    dx_s, dw_s = grads(build, x, 'simt')
    rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-20)).item()
    print('%s: dX rel %.3e  dW rel %.3e  |dW simt| %.3e |dW tensor| %.3e' % (name, rel(dx_t, dx_s), rel(dw_t, dw_s), dw_s.norm().item(), dw_t.norm().item()))
    kh, kw = dw_s.shape[2:]
    print('  per tap:', ' '.join('%.1e' % rel(dw_t[:, :, i, j], dw_s[:, :, i, j]) for i in range(kh) for j in range(kw)))
    M, N = dw_s.shape[:2]
    print('  per 32-row block (dim 0):', ' '.join('%.1e' % rel(dw_t[i:i + 32], dw_s[i:i + 32]) for i in range(0, M, 32)))
    print('  per 32-col block (dim 1):', ' '.join('%.1e' % rel(dw_t[:, i:i + 32], dw_s[:, i:i + 32]) for i in range(0, N, 32)))
    ratio = (dw_t.flatten()[:8] / dw_s.flatten()[:8]).tolist()
    print('  first ratios:', ['%.3f' % v for v in ratio])
