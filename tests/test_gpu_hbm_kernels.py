"""The fp32 HBM-bound kernels of the hot path against fp64, at the shapes bench.py runs and on every launch branch:
  * the fused composite forward (composite_vec4_kernel / composite_kernel) and its backward (composite_bwd_kernel<PREV>),
    every gradient: d_raw, d_flow, d_weight and d_fg seen through an identity 7x7 head, d_prev directly;
  * the stand-alone resample and its backward;
  * avgpool3s2 and avgpool2, forward and backward, vector and scalar kernels and the alignment fallbacks;
  * l1_loss and mse_to_const at the element counts the training step reduces;
  * the FlowNet2 glue: resize, flow_conf, flownet_prep, sub_channels, and the correlation at FlowNetC's size.

Every bound is derived in a comment from the arithmetic (term counts, EPS = fp32 machine epsilon 2^-23, the float spacing of a
sample coordinate) and every case prints its observed error next to it."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import bench
from oracle import flowops
from vid2vid_b200 import _lib as L
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import ops
from vid2vid_b200.networks import S_FG, S_FINAL, S_FLOW, S_IN, S_MASK, S_PREV, S_RAW, S_RAWC, S_W
from vid2vid_b200.plan import Plan, conv_desc

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23


@pytest.fixture(autouse=True, scope='module')
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    yield
    torch.set_num_threads(n)


def _wl(name, div=1):
    w = bench.WORKLOADS[name]
    return w['H'] // div, w['W'] // div


# bench.py's shapes: cfg3 generator scales (and discriminator pyramid levels), cfg4 inference scales
G3 = [_wl('cfg3'), _wl('cfg3', 2)]
D3 = [_wl('cfg3'), _wl('cfg3', 2), _wl('cfg3', 4)]
G4 = [_wl('cfg4'), _wl('cfg4', 2), _wl('cfg4', 4)]
FN2 = _wl('flownet2')


def _report(what, err, bound):
    print('%-58s max err/bound %.3g  (max err %.3g)' % (what, err, bound))


def _check(what, got, ref, tol):
    """|got - ref| <= tol elementwise; prints the worst ratio."""
    d = (got.double().cpu() - ref).abs()
    ratio = (d / tol.clamp_min(1e-300)).max().item() if d.numel() else 0.0
    _report(what, ratio, d.max().item() if d.numel() else 0.0)
    assert torch.isfinite(got).all(), what
    assert ratio <= 1.0, (what, ratio)


def _smooth(shape, g, freq=3.0):
    """Low-frequency image in [-1, 1]: a few sinusoids over the frame, so the coordinate-spacing term of the bounds stays small."""
    *lead, H, W = shape
    y = torch.linspace(0, 1, H, dtype=torch.float64).view(H, 1)
    x = torch.linspace(0, 1, W, dtype=torch.float64).view(1, W)
    n = int(np.prod(lead)) if lead else 1
    ph = torch.rand(n, 4, generator=g, dtype=torch.float64) * 6.28
    out = torch.empty(n, H, W, dtype=torch.float64)
    for i in range(n):
        out[i] = 0.5 * torch.sin(freq * 6.28 * x + ph[i, 0]) * torch.cos(freq * 3.1 * y + ph[i, 1]) + \
            0.4 * torch.sin(2.1 * x * 6.28 - 1.3 * y * 6.28 + ph[i, 2])
    return out.view(shape).float()


def _noise(shape, g):
    return torch.rand(shape, generator=g) * 2 - 1


def _flow(kind, N, H, W, g):
    """The flow kinds of test_gpu_bptt: fractional, integer, zero, leaving the frame, saturated (every pixel on a corner)."""
    if kind == 'frac':
        return torch.randn(N, 2, H, W, generator=g) * 2.5
    if kind == 'int':
        return torch.randint(-3, 4, (N, 2, H, W), generator=g).float()
    if kind == 'zero':
        return torch.zeros(N, 2, H, W)
    if kind == 'out':
        return (torch.rand(N, 2, H, W, generator=g) * 2 - 1) * torch.tensor([1.5 * W, 1.5 * H]).view(1, 2, 1, 1)
    return torch.sign(torch.randn(N, 2, H, W, generator=g)) * 1e3


# ------------------------------------------------------------------------------------------------ warp reference
def _axis(f, n, ac, along_x):
    """fp32 sample coordinate along one axis, with torch ops in the kernels' order (tensor operands throughout, so nothing is
    computed at another precision): torch.linspace grid, + flow / ((n - 1) / 2), unnormalise.  Not clamped."""
    lin = torch.linspace(-1, 1, n)
    lin = lin.view(1, 1, n) if along_x else lin.view(1, n, 1)
    full = lambda v: torch.full_like(f, v)
    gx = lin + f / full((n - 1.0) / 2.0)
    if ac:
        return ((gx + full(1.0)) / full(2.0)) * full(float(n - 1))
    return ((gx + full(1.0)) * full(float(n)) - full(1.0)) / full(2.0)


class Warp:
    """The bilinear border-padded warp of `flow` (N,2,H,W) as the kernels evaluate it: the cell is the one the fp32 coordinate
    selects, weights and everything after them in fp64."""

    def __init__(self, flow, ac):
        N, _, H, W = flow.shape
        self.N, self.H, self.W = N, H, W
        self.ix, self.iy = _axis(flow[:, 0], W, ac, True), _axis(flow[:, 1], H, ac, False)
        # one float spacing of a coordinate: the grid value (|.| <= 1, spacing <= EPS) scaled by n/2, plus the spacing of the
        # coordinate itself; x2 for the one rounding FMA contraction of the unnormalise may save.  Differences between the
        # kernel's coordinate and this one stay below it.
        self.spx = 2 * EPS * (self.ix.abs().double() + W / 2 + 1)
        self.spy = 2 * EPS * (self.iy.abs().double() + H / 2 + 1)
        self.cx, self.cy = self._cell(self.ix, W), self._cell(self.iy, H)
        # d(sample coordinate)/d(flow), zero where the pre-clamp coordinate is clipped (ATen clip_coordinates_set_grad)
        dsx, dsy = (1.0, 1.0) if ac else (W / (W - 1.0), H / (H - 1.0))
        self.dsx = torch.where((self.ix <= 0) | (self.ix >= W - 1), 0.0, dsx).double()
        self.dsy = torch.where((self.iy <= 0) | (self.iy >= H - 1), 0.0, dsy).double()
        self.dsx_nom, self.dsy_nom = dsx, dsy

    @staticmethod
    def _cell(i, n):
        c = i.clamp(0, n - 1)
        i0 = c.floor()
        w = (c - i0).double()               # exact in fp32
        i0 = i0.long()
        return i0, (i0 + 1).clamp(max=n - 1), w

    def gather(self, img, y, x):
        """img (N,C,H,W) at per-pixel integer positions y, x (N,H,W)."""
        N, Cc, H, W = img.shape
        idx = (y * W + x).reshape(N, 1, -1).expand(N, Cc, H * W)
        return img.reshape(N, Cc, -1).gather(2, idx).view(N, Cc, H, W)

    def corners(self, img, x0=None, x1=None, y0=None, y1=None):
        x0 = self.cx[0] if x0 is None else x0
        x1 = self.cx[1] if x1 is None else x1
        y0 = self.cy[0] if y0 is None else y0
        y1 = self.cy[1] if y1 is None else y1
        return self.gather(img, y0, x0), self.gather(img, y0, x1), self.gather(img, y1, x0), self.gather(img, y1, x1)

    def sample(self, img):
        """-> (value, sum of |corner * weight|, slope term: coordinate spacing x the largest neighbouring first difference)."""
        v00, v01, v10, v11 = self.corners(img)
        wx, wy = self.cx[2].unsqueeze(1), self.cy[2].unsqueeze(1)
        a = [(1 - wx) * (1 - wy), wx * (1 - wy), (1 - wx) * wy, wx * wy]
        val = v00 * a[0] + v01 * a[1] + v10 * a[2] + v11 * a[3]
        mag = v00.abs() * a[0] + v01.abs() * a[1] + v10.abs() * a[2] + v11.abs() * a[3]
        return val, mag, self.slope(img)

    def slope(self, img):
        """Coordinate spacing x the largest first difference in the 3x3 cells around the sample: bounds what a one-spacing
        move of the coordinate changes, including a move into the neighbouring cell."""
        dx = F.pad((img[..., 1:] - img[..., :-1]).abs(), (0, 1))
        dy = F.pad((img[..., 1:, :] - img[..., :-1, :]).abs(), (0, 0, 0, 1))
        dx, dy = F.max_pool2d(dx, 3, 1, 1), F.max_pool2d(dy, 3, 1, 1)
        gx = self.gather(dx, self.cy[0], self.cx[0])
        gy = self.gather(dy, self.cy[0], self.cx[0])
        return gx * self.spx.unsqueeze(1) + gy * self.spy.unsqueeze(1)

    def ddx(self, img, x0=None, x1=None):
        """d(sample)/d(x coordinate) in a given x cell: (v01 - v00)(1 - wy) + (v11 - v10) wy, and its magnitude."""
        v00, v01, v10, v11 = self.corners(img, x0=x0, x1=x1)
        wy = self.cy[2].unsqueeze(1)
        return (v01 - v00) * (1 - wy) + (v11 - v10) * wy, (v01.abs() + v00.abs()) * (1 - wy) + (v11.abs() + v10.abs()) * wy

    def ddy(self, img, y0=None, y1=None):
        v00, v01, v10, v11 = self.corners(img, y0=y0, y1=y1)
        wx = self.cx[2].unsqueeze(1)
        return (v10 - v00) * (1 - wx) + (v11 - v01) * wx, (v10.abs() + v00.abs()) * (1 - wx) + (v11.abs() + v01.abs()) * wx

    def edge(self, axis):
        """Pixels whose pre-clamp coordinate lies within one spacing of an integer of [0, n - 1] (the clamp limits included):
        there the kernel's d/d(flow) is one of the two one-sided derivatives.  -> (mask, k = that integer)."""
        i, sp, n = (self.ix, self.spx, self.W) if axis == 0 else (self.iy, self.spy, self.H)
        k = i.double().round().clamp(0, n - 1)
        return ((i.double() - k).abs() <= sp), k.long()

    def one_sided(self, axis, img, coef, ds_nom):
        """Candidate values of sum_c coef_c * d(sample_c)/d(coordinate) * ds at edge pixels: the cell left and right of the
        integer k (where they exist) and 0 (past a clamp limit).  -> (candidates (3,N,H,W), valid (3,N,H,W), magnitude)."""
        m, k = self.edge(axis)
        n = self.W if axis == 0 else self.H
        f = self.ddx if axis == 0 else self.ddy
        lo0, lo1 = (k - 1).clamp(min=0), k
        hi0, hi1 = k, (k + 1).clamp(max=n - 1)
        kw = (lambda a, b: dict(x0=a, x1=b)) if axis == 0 else (lambda a, b: dict(y0=a, y1=b))
        dl, ml = f(img, **kw(lo0, lo1))
        dr, mr = f(img, **kw(hi0, hi1))
        cl, cr = (coef * dl).sum(1) * ds_nom, (coef * dr).sum(1) * ds_nom
        mag = (coef.abs() * (ml + mr)).sum(1) * ds_nom
        zero = torch.zeros_like(cl)
        cand = torch.stack([cl, cr, zero])
        valid = torch.stack([k >= 1, k <= n - 2, (k == 0) | (k == n - 1)])
        return m, cand, valid, mag


def _check_flow_grad(what, got, ref, tol, w, axis, img, coef, bound_eps):
    """d/d(flow) component `axis`: ordinary pixels against `ref` within `tol`; edge pixels against the nearest one-sided
    candidate within bound_eps * magnitude (+ tol).  Returns the number of pixels that took the one-sided path."""
    m, cand, valid, mag = w.one_sided(axis, img, coef, w.dsx_nom if axis == 0 else w.dsy_nom)
    got = got.double().cpu()
    d = (got - ref).abs()
    ratio_plain = (d / tol.clamp_min(1e-300))[~m]
    etol = tol + bound_eps * mag
    dc = (got.unsqueeze(0) - cand).abs()
    dc = torch.where(valid, dc, torch.full_like(dc, float('inf'))).min(0).values
    ratio_edge = (dc / etol.clamp_min(1e-300))[m]
    worst = max(ratio_plain.max().item() if ratio_plain.numel() else 0.0, ratio_edge.max().item() if ratio_edge.numel() else 0.0)
    _report('%s (%d one-sided px)' % (what, int(m.sum())), worst, d[~m].max().item() if (~m).any() else 0.0)
    assert torch.isfinite(got).all(), what
    assert worst <= 1.0, (what, worst)
    return int(m.sum())


# ------------------------------------------------------------------------------------------------ composite forward
def _composite_plan(N, H, W, pc, fg, warp, ac, train=False, head=None):
    p = Plan(0, impl=L.IMPL_SIMT if head is not None else None, precision='precise', train=train)
    if head is not None:
        v = p.input(S_IN, N, 9, 0, 9, H, W, exact_bf16=True)
        p.head(v, conv_desc(head, L.PAD_REFLECT, 3), HEAD_CHANNELS)
    if warp:
        p.input(S_PREV, N, pc, 0, pc, H, W)
    p.composite(S_RAW, S_FLOW if warp else -1, S_W if warp else -1, S_PREV if warp else -1, pc, S_FG if fg else -1,
                S_MASK if fg else -1, S_FINAL, N, H, W, warp, ac, s_raw_out=S_RAWC if fg else -1)
    p.finalize()
    return p


def _composite_ref(raw, flow, w, prev, fgi, mask, ac, warp):
    """fp64 composite from fp32 inputs -> (final, raw composited, tolerance of final, tolerance of raw composited)."""
    r = raw.double()
    if warp:
        wp = Warp(flow, ac)
        val, mag, slope = wp.sample(prev[:, -3:].double())
        w64 = w.double()
        fin = r * w64 + val * (1 - w64)
        # bilinear: 4 weight products (1 rounding each, (1 - w) another), 4 products, 3 adds -> <= 6 EPS of mag; the blend
        # r*w + v*(1-w): 1 - w, two products, one add -> 4 EPS of its terms: 10 EPS of |r| w + mag (1 - w)
        tmag = r.abs() * w64 + mag * (1 - w64)
        tol = 10 * EPS * tmag + slope * (1 - w64)
    else:
        fin, tmag, tol = r, r.abs(), torch.zeros_like(r)
    rc, rtol = r, torch.zeros_like(r)
    if fgi is not None:
        m = mask.double()
        g = fgi.double()
        # g*m + f*(1-m): 1 - m, two products, one add -> 4 EPS of |g| m + |f| (1 - m), after the incoming error x (1 - m)
        tol = 4 * EPS * (g.abs() * m + tmag * (1 - m)) + tol * (1 - m)
        fin = g * m + fin * (1 - m)
        rtol = 4 * EPS * (g.abs() * m + r.abs() * (1 - m))
        rc = g * m + r * (1 - m)
    return fin, rc, tol + 1e-30, rtol + 1e-30


def _composite_fwd(N, H, W, pc, fg, warp, ac, kind, smooth, seed=1):
    g = torch.Generator().manual_seed(seed)
    img = _smooth if smooth else _noise
    raw, prev = img((N, 3, H, W), g), img((N, pc, H, W), g)
    w = torch.rand(N, 1, H, W, generator=g)
    flow = _flow(kind, N, H, W, g)
    fgi = img((N, 3, H, W), g) if fg else None
    mask = torch.rand(N, 1, H, W, generator=g) if fg else None
    p = _composite_plan(N, H, W, pc, fg, warp, ac)
    io = [None] * 16
    io[S_RAW], io[S_FINAL] = raw.cuda(), torch.empty(N, 3, H, W, device='cuda')
    if warp:
        io[S_FLOW], io[S_W], io[S_PREV] = flow.cuda(), w.cuda(), prev.cuda()
    if fg:
        io[S_FG], io[S_MASK], io[S_RAWC] = fgi.cuda(), mask.cuda(), torch.empty(N, 3, H, W, device='cuda')
    p.run(io, False)
    torch.cuda.synchronize()
    fin, rc, tol, rtol = _composite_ref(raw, flow, w, prev, fgi, mask, ac, warp)
    tag = 'composite %s %dx%d pc%d fg%d warp%d ac%d %s' % ('vec4' if W % 4 == 0 else 'scalar', H, W, pc, fg, warp, ac, kind)
    _check(tag + ' final', io[S_FINAL], fin, tol)
    if fg:
        _check(tag + ' rawc', io[S_RAWC], rc, rtol)
    assert torch.equal(io[S_RAW].cpu(), raw)            # with fg the head output slot keeps its value


@pytest.mark.parametrize('W', [24, 22, 37], ids=['vec4', 'scalar22', 'scalar37'])
@pytest.mark.parametrize('kind', ['frac', 'int', 'zero', 'out', 'saturated'])
@pytest.mark.parametrize('fg', [False, True], ids=['nofg', 'fg'])
@pytest.mark.parametrize('ac', [0, 1], ids=['ac0', 'ac1'])
def test_composite_forward_small(W, kind, fg, ac):
    _composite_fwd(2, 13, W, 6 if fg else 3, fg, True, ac, kind, smooth=False)


@pytest.mark.parametrize('W', [24, 22], ids=['vec4', 'scalar'])
@pytest.mark.parametrize('fg', [False, True], ids=['nofg', 'fg'])
def test_composite_forward_nowarp(W, fg):
    _composite_fwd(2, 9, W, 3, fg, False, 0, 'zero', smooth=False)


@pytest.mark.parametrize('HW', G3 + G4, ids=lambda s: '%dx%d' % s)
@pytest.mark.parametrize('kind', ['frac', 'saturated'])
def test_composite_forward_bench_shapes(HW, kind):
    """cfg3 generator scales and cfg4 inference scales (fg, warp, 6-channel prev as the generators run), vec4 kernel."""
    H, W = HW
    _composite_fwd(1, H, W, 6, True, True, 0, kind, smooth=True)


# ------------------------------------------------------------------------------------------------ composite backward
# identity 7x7 head: input channel j -> output channel j through the centre tap; channels mapped as networks.emit_head /
# emit_head_pair map the generator heads (3 raw tanh, 2 flow, 1 weight sigmoid, 3 fg tanh).  The plan is a SIMT plan so the
# head's data gradient is fp32 SIMT (asserted below): with one nonzero tap of 1.0 and bf16-exact inputs the forward is exact
# and the input gradient is exactly the composite's slot gradient times the activation's derivative.
HEAD_CHANNELS = [(S_RAW, j, 3, L.ACT_TANH, 1.0) for j in range(3)] + [(S_FLOW, j, 2, L.ACT_NONE, 1.0) for j in range(2)] + \
    [(S_W, 0, 1, L.ACT_SIGMOID, 1.0)] + [(S_FG, j, 3, L.ACT_TANH, 1.0) for j in range(3)]


def _identity_head():
    conv = nn.Conv2d(9, 9, 7).cuda()
    with torch.no_grad():
        conv.weight.zero_()
        conv.bias.zero_()
        for j in range(9):
            conv.weight[j, j, 3, 3] = 1.0
    return conv


def _bf16(t):
    return t.bfloat16().float()


def _composite_bwd(N, H, W, pc, fg, warp, ac, kind, prev_grad, smooth, seed=3):
    g = torch.Generator().manual_seed(seed)
    img = _smooth if smooth else _noise
    x = torch.cat([_bf16(img((N, 3, H, W), g) * 1.5), _bf16(_flow(kind, N, H, W, g)), _bf16(torch.rand(N, 1, H, W, generator=g) * 6 - 3),
                   _bf16(img((N, 3, H, W), g) * 1.5)], 1)
    prev = img((N, pc, H, W), g)
    mask = torch.rand(N, 1, H, W, generator=g)
    g_final, g_rawout = img((N, 3, H, W), g), img((N, 3, H, W), g)
    head = _identity_head()
    p = _composite_plan(N, H, W, pc, fg, warp, ac, train=True, head=head)
    (rec,) = p.describe()['backward']
    assert rec['mode'] == 0, rec                          # the head's data gradient runs on the fp32 SIMT path
    io = [None] * 16
    io[S_IN], io[S_FINAL] = x.cuda(), torch.empty(N, 3, H, W, device='cuda')
    io[S_RAW], io[S_FLOW], io[S_W], io[S_FG] = (torch.empty(N, c, H, W, device='cuda') for c in (3, 2, 1, 3))
    if warp:
        io[S_PREV] = prev.cuda()
    if fg:
        io[S_MASK], io[S_RAWC] = mask.cuda(), torch.empty(N, 3, H, W, device='cuda')
    p.run(io, False)
    gio = [None] * 16
    gio[S_FINAL], gio[S_IN] = g_final.cuda(), torch.zeros(N, 9, H, W, device='cuda')
    if fg:
        gio[S_RAWC] = g_rawout.cuda()
    if prev_grad and warp:
        gio[S_PREV] = torch.zeros(N, pc, H, W, device='cuda')
    p.backward(io, gio, [], [])
    torch.cuda.synchronize()
    raw, flow, w, fgo = (io[s].cpu() for s in (S_RAW, S_FLOW, S_W, S_FG))
    assert torch.equal(flow, x[:, 3:5])                   # the identity head is exact
    tag = 'composite bwd<%s> %dx%d pc%d fg%d warp%d ac%d %s' % ('PREV' if prev_grad and warp else 'noPREV', H, W, pc, fg, warp, ac, kind)

    gf, gr = g_final.double(), (g_rawout.double() if fg else torch.zeros(N, 3, H, W, dtype=torch.float64))
    m = mask.double() if fg else torch.zeros(N, 1, H, W, dtype=torch.float64)
    om = 1 - m
    w64, r64 = w.double(), raw.double()
    gin = gio[S_IN].cpu()
    # head backward: dz = g_slot * act'(out) with act' = 1 - t^2 (tanh) or t (1 - t) (sigmoid) in fp32: 3 more roundings
    dtanh = lambda t: 1 - t.double() ** 2
    d_fg = (gf + gr) * m                                  # (gf + gr) * m: 2 roundings
    _check(tag + ' d_fg', gin[:, 6:9], d_fg * dtanh(fgo) if fg else torch.zeros_like(d_fg),
           5 * EPS * ((gf.abs() + gr.abs()) * m * dtanh(fgo)) + 1e-30)
    if not warp:
        d_raw = (gf + gr) * om                            # 2 roundings (+ 1 in 1 - m)
        _check(tag + ' d_raw', gin[:, 0:3], d_raw * dtanh(raw), 6 * EPS * ((gf.abs() + gr.abs()) * om * dtanh(raw)) + 1e-30)
        assert not gin[:, 3:6].any()
        return
    wp = Warp(flow, ac)
    pv = prev[:, -3:].double()
    val, mag, slope = wp.sample(pv)
    gg = gf * om                                          # gradient reaching img_raw * w + warp * (1 - w)
    # d_raw = g*w + gr*om: 1 - m, g, two products, one add: 5 roundings of its terms
    d_raw = gg * w64 + gr * om
    _check(tag + ' d_raw', gin[:, 0:3], d_raw * dtanh(raw), 8 * EPS * ((gg.abs() * w64 + gr.abs() * om) * dtanh(raw)) + 1e-30)
    # d_weight = sum_c g_c (raw_c - warp_c): warp to 10 EPS of mag (+ the slope term), one subtraction, one product, 3 adds
    dsig = (w64 * (1 - w64)).squeeze(1)
    d_w = (gg * (r64 - val)).sum(1)
    tol_w = ((gg.abs() * (8 * EPS * (r64.abs() + val.abs()) + 10 * EPS * mag + slope)).sum(1) + 3 * EPS * (gg * (r64 - val)).abs().sum(1)) * dsig
    _check(tag + ' d_weight', gin[:, 5], d_w * dsig, tol_w + 1e-30)
    # d_flow = sum_c g_c (1 - w) ddx_c * ds: ddx 2 products 3 subtractions/adds (5 EPS of its magnitude), ds one division
    # (1 EPS), 4 more products and 2 adds (6 EPS): 16 EPS of |g| (1 - w) |ddx| ds, plus wy moved by one spacing (2 x slope)
    coef = gg * (1 - w64)
    ddx, mx = wp.ddx(pv)
    ddy, my = wp.ddy(pv)
    sl = slope * 2
    ref_x = (coef * ddx).sum(1) * wp.dsx
    ref_y = (coef * ddy).sum(1) * wp.dsy
    tol_x = (coef.abs() * (16 * EPS * mx + sl)).sum(1) * wp.dsx_nom + 1e-30
    tol_y = (coef.abs() * (16 * EPS * my + sl)).sum(1) * wp.dsy_nom + 1e-30
    n1 = _check_flow_grad(tag + ' d_flow x', gin[:, 3], ref_x, tol_x, wp, 0, pv, coef, 16 * EPS)
    n2 = _check_flow_grad(tag + ' d_flow y', gin[:, 4], ref_y, tol_y, wp, 1, pv, coef, 16 * EPS)
    if kind == 'int' and ac:
        assert n1 + n2 > N * H * W, (n1, n2)               # integer flows with align_corners land on integers
    if not (prev_grad and warp):
        return
    # d_prev: the four corner contributions gp * weight, accumulated with fp32 atomics in any order.  A source pixel with k
    # contributions is within (k + 1) EPS of their |sum| (k - 1 adds, 1 rounding of each product chain; +1 for the weight
    # product), plus what a one-spacing move of the sample coordinate shifts between neighbouring corners.
    gp = gg * (1 - w64)
    wx, wy = wp.cx[2].unsqueeze(1), wp.cy[2].unsqueeze(1)
    ref = torch.zeros(N, 3, H * W, dtype=torch.float64)
    cnt, absum = torch.zeros_like(ref), torch.zeros_like(ref)
    for (yy, xx, a) in ((wp.cy[0], wp.cx[0], (1 - wx) * (1 - wy)), (wp.cy[0], wp.cx[1], wx * (1 - wy)),
                        (wp.cy[1], wp.cx[0], (1 - wx) * wy), (wp.cy[1], wp.cx[1], wx * wy)):
        c = (gp * a).reshape(N, 3, -1)
        idx = (yy * W + xx).reshape(N, -1)
        for n in range(N):
            for ch in range(3):
                ref[n, ch].index_add_(0, idx[n], c[n, ch])
                absum[n, ch].index_add_(0, idx[n], c[n, ch].abs())
                cnt[n, ch].index_add_(0, idx[n], (c[n, ch] != 0).double())
    move = (gp.abs() * (wp.spx + wp.spy).unsqueeze(1)).reshape(N, 3, -1)
    mv = torch.zeros_like(ref)
    for n in range(N):
        for ch in range(3):
            mv[n, ch].index_add_(0, (wp.cy[0] * W + wp.cx[0]).reshape(N, -1)[n], move[n, ch])
    mv = F.conv2d(mv.view(N * 3, 1, H, W), torch.ones(1, 1, 5, 5, dtype=torch.float64), padding=2).view(N, 3, -1)
    tol = (cnt + 2) * EPS * absum + 2 * mv + 1e-30
    ours = gio[S_PREV].cpu()
    assert not ours[:, :pc - 3].any()                    # channels below prev_C - 3 get nothing from the composite
    _check(tag + ' d_prev (max %d contributions)' % int(cnt.max()), ours[:, pc - 3:].reshape(N, 3, -1), ref, tol)


@pytest.mark.parametrize('W', [24, 22], ids=['vec4', 'scalar'])
@pytest.mark.parametrize('kind', ['frac', 'int', 'zero', 'out', 'saturated'])
@pytest.mark.parametrize('fg', [False, True], ids=['nofg', 'fg'])
@pytest.mark.parametrize('ac', [0, 1], ids=['ac0', 'ac1'])
@pytest.mark.parametrize('prev_grad', [True, False], ids=['PREV', 'noPREV'])
def test_composite_backward_small(W, kind, fg, ac, prev_grad):
    _composite_bwd(2, 13, W, 6 if fg else 3, fg, True, ac, kind, prev_grad, smooth=False)


@pytest.mark.parametrize('fg', [False, True], ids=['nofg', 'fg'])
def test_composite_backward_nowarp(fg):
    _composite_bwd(2, 9, 24, 3, fg, False, 0, 'zero', False, smooth=False)


@pytest.mark.parametrize('HW,kind', [(G3[0], 'saturated'), (G3[0], 'frac'), (G3[1], 'frac'), (G3[1], 'int')],
                         ids=lambda v: '%dx%d' % v if isinstance(v, tuple) else v)
def test_composite_backward_bench_shapes(HW, kind):
    """cfg3 generator scales, as the training step runs them: fg, 6-channel prev, img_prev gradient (--n_frames_bp)."""
    H, W = HW
    _composite_bwd(1, H, W, 6, True, True, 0, kind, True, smooth=True)


def test_composite_refuses_misaligned_slots():
    """A composite that runs the vec4 kernel refuses caller tensors that are not 16-byte aligned; the scalar one takes them."""
    g = torch.Generator().manual_seed(5)
    for W in (24, 22):
        N, H = 1, 7
        p = _composite_plan(N, H, W, 3, False, True, 0)
        raw, flow, w, prev = _noise((N, 3, H, W), g), _flow('frac', N, H, W, g), torch.rand(N, 1, H, W, generator=g), _noise((N, 3, H, W), g)
        io = [None] * 16
        io[S_FLOW], io[S_W], io[S_PREV] = flow.cuda(), w.cuda(), prev.cuda()
        io[S_RAW], io[S_FINAL] = raw.cuda(), torch.empty(N, 3, H, W, device='cuda')
        p.run(io, False)
        aligned = io[S_FINAL].clone()
        store = torch.empty(raw.numel() + 1, device='cuda')
        io[S_RAW] = store[1:].view(N, 3, H, W)            # contiguous, at a one-float storage offset
        io[S_RAW].copy_(raw)
        if W % 4 == 0:
            with pytest.raises(RuntimeError, match='aligned'):
                p.run(io, False)
            io[S_RAW] = raw.cuda()
        p.run(io, False)
        torch.cuda.synchronize()
        assert torch.equal(io[S_FINAL], aligned), W


# ------------------------------------------------------------------------------------------------ resample
def _resample_case(N, Cc, H, W, ac, kind, need_img, need_flow, smooth, seed=11):
    g = torch.Generator().manual_seed(seed)
    img = (_smooth if smooth else _noise)((N, Cc, H, W), g)
    flow = _flow(kind, N, H, W, g)
    go = (_smooth if smooth else _noise)((N, Cc, H, W), g)
    ic, fc = img.cuda().requires_grad_(need_img), flow.cuda().requires_grad_(need_flow)
    out = ops.resample(ic, fc, bool(ac))
    wp = Warp(flow, ac)
    val, mag, slope = wp.sample(img.double())
    tag = 'resample %dx%dx%d ac%d %s img%d flow%d' % (Cc, H, W, ac, kind, need_img, need_flow)
    # the bilinear expression: 6 EPS of mag (see _composite_ref) + the coordinate-spacing term
    _check(tag + ' fwd', out.detach(), val, 6 * EPS * mag + slope + 1e-30)
    if not (need_img or need_flow):
        return
    out.backward(go.cuda())
    torch.cuda.synchronize()
    gd = go.double()
    if need_flow:
        ddx, mx = wp.ddx(img.double())
        ddy, my = wp.ddy(img.double())
        # fp32: ddx 5 EPS, * g * ds 3 more, C-term sum: 16 EPS of the magnitudes, + wy moved by one spacing
        tol_x = (gd.abs() * (16 * EPS * mx + 2 * slope)).sum(1) * wp.dsx_nom + 1e-30
        tol_y = (gd.abs() * (16 * EPS * my + 2 * slope)).sum(1) * wp.dsy_nom + 1e-30
        _check_flow_grad(tag + ' gflow x', fc.grad[:, 0], (gd * ddx).sum(1) * wp.dsx, tol_x, wp, 0, img.double(), gd, 16 * EPS)
        _check_flow_grad(tag + ' gflow y', fc.grad[:, 1], (gd * ddy).sum(1) * wp.dsy, tol_y, wp, 1, img.double(), gd, 16 * EPS)
    else:
        assert fc.grad is None
    if need_img:
        ref = torch.zeros(N, Cc, H * W, dtype=torch.float64)
        absum, cnt = torch.zeros_like(ref), torch.zeros_like(ref)
        wx, wy = wp.cx[2].unsqueeze(1), wp.cy[2].unsqueeze(1)
        for (yy, xx, a) in ((wp.cy[0], wp.cx[0], (1 - wx) * (1 - wy)), (wp.cy[0], wp.cx[1], wx * (1 - wy)),
                            (wp.cy[1], wp.cx[0], (1 - wx) * wy), (wp.cy[1], wp.cx[1], wx * wy)):
            c = (gd * a).reshape(N, Cc, -1)
            idx = (yy * W + xx).reshape(N, -1)
            for n in range(N):
                for ch in range(Cc):
                    ref[n, ch].index_add_(0, idx[n], c[n, ch])
                    absum[n, ch].index_add_(0, idx[n], c[n, ch].abs())
                    cnt[n, ch].index_add_(0, idx[n], torch.ones_like(c[n, ch]))
        move = (gd.abs() * (wp.spx + wp.spy).unsqueeze(1)).reshape(N, Cc, -1)
        mv = torch.zeros_like(ref)
        for n in range(N):
            for ch in range(Cc):
                mv[n, ch].index_add_(0, (wp.cy[0] * W + wp.cx[0]).reshape(N, -1)[n], move[n, ch])
        mv = F.conv2d(mv.view(N * Cc, 1, H, W), torch.ones(1, 1, 5, 5, dtype=torch.float64), padding=2).view(N, Cc, -1)
        # atomics: (k + 2) EPS of the sum of |contributions| (k - 1 adds, weight product and g * weight), + coordinate moves
        _check(tag + ' gimg (max %d contributions)' % int(cnt.max()), ic.grad.reshape(N, Cc, -1), ref, (cnt + 2) * EPS * absum + 2 * mv + 1e-30)
    else:
        assert ic.grad is None


@pytest.mark.parametrize('shape', [(2, 3, 13, 22), (1, 2, 9, 37)], ids=['13x22', '9x37'])
@pytest.mark.parametrize('kind', ['frac', 'int', 'zero', 'out', 'saturated'])
@pytest.mark.parametrize('ac', [0, 1], ids=['ac0', 'ac1'])
@pytest.mark.parametrize('need', [(True, True), (True, False), (False, True), (False, False)], ids=['gimg_gflow', 'gimg', 'gflow', 'nograd'])
def test_resample_small(shape, kind, ac, need):
    _resample_case(*shape, ac, kind, need[0], need[1], smooth=False)


@pytest.mark.parametrize('HW', G3, ids=lambda s: '%dx%d' % s)
@pytest.mark.parametrize('kind', ['frac', 'out'])
def test_resample_bench_shapes(HW, kind):
    """The warp losses of the cfg3 step: real_B_prev (3 channels) warped by the generated flow at each generator scale."""
    _resample_case(1, 3, *HW, 0, kind, True, True, smooth=True)


# ------------------------------------------------------------------------------------------------ pooling
def _pool3_fwd_check(x, tag):
    out = ops.avgpool3s2(x)
    torch.cuda.synchronize()
    xd = x.double().cpu()
    ref = F.avg_pool2d(xd.flatten(0, -3).unsqueeze(1), 3, 2, 1, count_include_pad=False)
    mag = F.avg_pool2d(xd.abs().flatten(0, -3).unsqueeze(1), 3, 2, 1, count_include_pad=False)
    # <= 9 sequential adds and one division: 10 EPS of the window's mean |x| (x count for the mean: the sum's error / count)
    _check(tag, out.flatten(0, -3).unsqueeze(1), ref, 10 * EPS * mag * 9 / 4 + 1e-30)
    return out


@pytest.mark.parametrize('shape', [(3, 13, 24), (3, 14, 24), (3, 13, 22), (3, 14, 23), (5, 14, 4), (5, 7, 5), (70, 9, 16), (70, 10, 18)],
                         ids=['vec_oddH', 'vec_evenH', 'scalar_evenW', 'scalar_oddW', 'vec_W4', 'scalar_W5', 'vec_P70', 'scalar_P70'])
def test_avgpool3s2_forward(shape):
    g = torch.Generator().manual_seed(21)
    x = _noise(shape, g).cuda()
    out = _pool3_fwd_check(x, 'avgpool3s2 fwd %s' % (shape,))
    if shape[-1] % 4 == 0:
        # the same data at a one-float storage offset takes the scalar kernel; both claim the same summation order
        store = torch.empty(x.numel() + 1, device='cuda')
        xm = store[1:].view(shape)
        xm.copy_(x)
        assert xm.is_contiguous() and xm.data_ptr() % 16 != 0
        assert torch.equal(ops.avgpool3s2(xm), out)
        # and through the C ABI with an output pointer that is not 8-byte aligned
        ostore = torch.empty(out.numel() + 1, device='cuda')
        h, w = shape[-2:]
        L.check(L.lib().v2v_avgpool3s2(C.c_void_p(x.data_ptr()), C.c_void_p(ostore.data_ptr() + 4), x.numel() // (h * w), h, w,
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        assert torch.equal(ostore[1:].view(out.shape), out)


@pytest.mark.parametrize('HW', D3 + G4, ids=lambda s: '%dx%d' % s)
def test_avgpool3s2_bench_shapes(HW):
    """The D pyramid of cfg3 (label + image channels, 39 planes) and the cfg4 label pyramid, forward and backward."""
    g = torch.Generator().manual_seed(22)
    H, W = HW
    planes = 39 if HW in D3 else 36
    x = _smooth((1, planes, H, W), g).cuda()
    _pool3_fwd_check(x, 'avgpool3s2 fwd %dx%dx%d' % (planes, H, W))
    if HW in D3:
        _pool3_bwd_check(x.shape, g, 'avgpool3s2 bwd %dx%dx%d' % (planes, H, W))


def _pool3_bwd_check(shape, g, tag):
    x = torch.zeros(shape, device='cuda', requires_grad=True)
    out = ops.avgpool3s2(x)
    go = _noise(out.shape, g)
    out.backward(go.cuda())
    torch.cuda.synchronize()
    xd = torch.zeros(shape, dtype=torch.float64, requires_grad=True)
    F.avg_pool2d(xd.flatten(0, -3).unsqueeze(1), 3, 2, 1, count_include_pad=False).backward(go.double().flatten(0, -3).unsqueeze(1))
    xa = torch.zeros(shape, dtype=torch.float64, requires_grad=True)
    F.avg_pool2d(xa.flatten(0, -3).unsqueeze(1), 3, 2, 1, count_include_pad=False).backward(go.double().abs().flatten(0, -3).unsqueeze(1))
    # <= 4 windows: one division each, 3 adds -> 5 EPS of sum |g| / count
    _check(tag, x.grad, xd.grad, 5 * EPS * xa.grad + 1e-30)


@pytest.mark.parametrize('shape', [(3, 13, 24), (3, 14, 24), (3, 13, 22), (3, 14, 23), (5, 14, 4), (5, 7, 5), (70, 9, 16), (2, 2, 2)],
                         ids=['oddH', 'evenH', 'evenW', 'oddW', 'W4', 'W5', 'P70', '2x2'])
def test_avgpool3s2_backward(shape):
    _pool3_bwd_check(shape, torch.Generator().manual_seed(23), 'avgpool3s2 bwd %s' % (shape,))


def _offset_copy(t):
    store = torch.empty(t.numel() + 1, device='cuda')
    v = store[1:].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize('shape', [(2, 3, 12, 16), (2, 3, 13, 16), (2, 3, 12, 18), (2, 3, 13, 17)] + [(1, 3) + s for s in G4[:1]],
                         ids=['vec', 'vec_oddH', 'scalar_W18', 'scalar_oddHW', 'cfg4_%dx%d' % G4[0]])
def test_avgpool2_forward_backward(shape):
    """nn.AvgPool2d(2) (VGGLoss's downsample of a frame wider than 1024, as at cfg4's size), forward and backward, with the
    unaligned fallback on the same data."""
    g = torch.Generator().manual_seed(24)
    x = _smooth(shape, g).cuda() if shape[-1] > 1000 else _noise(shape, g).cuda()
    xr = x.clone().requires_grad_(True)
    out = ops.avgpool2(xr)
    xd = x.double().cpu()
    # (((a + b) + c) + d) / 4: 3 adds, the division by 4 is exact: 3 EPS of the window's mean |x| x 4 / 4
    _check('avgpool2 fwd %s' % (shape,), out.detach(), F.avg_pool2d(xd, 2), 3 * EPS * F.avg_pool2d(xd.abs(), 2) + 1e-30)
    assert torch.equal(ops.avgpool2(_offset_copy(x)), out.detach())          # scalar fallback, same summation order
    go = _noise(out.shape, g)
    out.backward(go.cuda())
    ref = torch.zeros(shape, dtype=torch.float64)
    Ho, Wo = shape[-2] // 2, shape[-1] // 2
    for dy in (0, 1):
        for dx in (0, 1):
            ref[..., dy:2 * Ho:2, dx:2 * Wo:2] = go.double() / 4
    assert torch.equal(xr.grad.cpu().double(), ref)                            # g / 4 is exact, dropped rows / columns 0
    xm = x.clone().requires_grad_(True)
    ops.avgpool2(xm).backward(_offset_copy(go.cuda()))
    assert torch.equal(xm.grad, xr.grad)


# ------------------------------------------------------------------------------------------------ losses
def _partial_len(total):
    """Terms per thread under grid1d's 132 * 8-block cap of 256 threads (csrc/losses.cu)."""
    blocks = min((total + 255) // 256, 132 * 8)
    return -(-total // (blocks * 256))


def _sum_bound(total):
    """Relative error of the mean of non-negative fp32 terms: per-thread sequential sum (L - 1 adds), the block's 8-level
    shuffle tree, the fp32 rounding of the fp64 mean and of 1 / numel: (L + 10) / 2 EPS; EPS per unit of rounding for safety."""
    return (_partial_len(total) + 10) * EPS


def _l1_case(shape, mask_shape, with_b, tag, seed=31):
    g = torch.Generator().manual_seed(seed)
    a = _noise(shape, g)
    b = _noise(shape, g) if with_b else None
    m = torch.rand(mask_shape, generator=g) if mask_shape else None
    ac_, bc = a.cuda().requires_grad_(True), (b.cuda().requires_grad_(True) if with_b else None)
    mc = m.cuda() if m is not None else None
    loss = ops.l1_loss(ac_, bc, mc)
    again = [ops.l1_loss(ac_.detach(), bc.detach() if bc is not None else None, mc) for _ in range(3)]
    a64 = a.double()
    if m is not None:
        m64 = m.double()
        if a.dim() == 5:
            m64 = m64.view(-1, 1, *shape[-2:]).view(shape[0], shape[1], 1, *shape[-2:]) if m.dim() == 5 else m64
        am, bm = a64 * m64, (b.double() * m64 if with_b else torch.zeros_like(a64))
    else:
        am, bm = a64, (b.double() if with_b else torch.zeros_like(a64))
    terms = (am - bm).abs()
    total = a.numel()
    ref = terms.sum().item() / total
    # each term: two products and a subtraction in fp32: 2 EPS of |a m| + |b m|; then the reduction
    bound = _sum_bound(total) * ref + 2 * EPS * (am.abs() + bm.abs()).sum().item() / total
    err = abs(loss.item() - ref)
    _report('l1 %s fwd (n=%d, %d terms/thread)' % (tag, total, _partial_len(total)), err / bound, err)
    assert err <= bound
    for t in again:
        assert torch.equal(t, loss.detach())             # the mean does not depend on the block order
    gs = torch.tensor(0.75)
    loss.backward(gs.cuda())
    torch.cuda.synchronize()
    d32 = (am - bm).float()
    sgn = torch.sign(am - bm)
    mm = m64.expand_as(a64) if m is not None else torch.ones_like(a64)
    ref_g = sgn * mm * (0.75 * np.float32(1.0 / total))
    # r = sign * m * (g * inv_numel): 2 roundings; where |d| is within the term's rounding of 0 the sign is free
    free = (am - bm).abs() <= 2 * EPS * (am.abs() + bm.abs())
    ga = ac_.grad.double().cpu()
    bad = ((ga - ref_g).abs() > 3 * EPS * ref_g.abs()) & ~free
    _report('l1 %s bwd ga (%d sign-free terms)' % (tag, int(free.sum())), float(bad.sum()), (ga - ref_g)[~free].abs().max().item())
    assert not bad.any()
    if with_b:
        assert torch.equal(bc.grad, -ac_.grad)
    del d32


@pytest.mark.parametrize('shape,mask,with_b', [
    ((2, 3, 13, 22), (2, 1, 13, 22), True),
    ((2, 3, 13, 22), None, True),
    ((2, 1, 13, 22), (2, 1, 13, 22), False),
    ((1, 3, 2, 11, 20), None, True),
    ((1, 3) + G3[0], (1, 1) + G3[0], True),
    ((1, 2) + G3[0], (1, 1) + G3[0], True),
    ((1, 1) + G3[0], (1, 1) + G3[0], False),
    ((1, 64) + G3[0], None, True),
], ids=['masked', 'plain', 'b_none', '5d', 'cfg3_warp_%dx%d' % G3[0], 'cfg3_flow_%dx%d' % G3[0], 'cfg3_weight_%dx%d' % G3[0],
        'cfg3_feat_2^25'])
def test_l1_loss(shape, mask, with_b):
    _l1_case(shape, mask, with_b, '%s mask=%s b=%d' % (shape, mask is not None, with_b))


@pytest.mark.parametrize('shape', [(2, 1, 13, 22), (1, 1, 64, 128), (1, 1) + G3[0], (1, 32) + G3[0]],
                         ids=['small', 'D_logit', 'cfg3_%dx%d' % G3[0], '2^24'])
@pytest.mark.parametrize('target', [0.0, 1.0])
def test_mse_to_const(shape, target):
    g = torch.Generator().manual_seed(32)
    x = torch.randn(shape, generator=g)
    xc = x.cuda().requires_grad_(True)
    loss = ops.mse_to_const(xc, target)
    again = [ops.mse_to_const(xc.detach(), target) for _ in range(3)]
    t64 = (x.double() - np.float64(np.float32(target)))
    total = x.numel()
    ref = (t64 ** 2).sum().item() / total
    # each term: a subtraction and a square: 3 EPS; then the reduction
    bound = (_sum_bound(total) + 3 * EPS) * ref
    err = abs(loss.item() - ref)
    _report('mse_to_const %s t=%g fwd (%d terms/thread)' % (shape, target, _partial_len(total)), err / bound, err)
    assert err <= bound
    for t in again:
        assert torch.equal(t, loss.detach())
    loss.backward(torch.tensor(1.5).cuda())
    gs = np.float64(np.float32(np.float32(2.0) * np.float32(1.5) * np.float32(1.0 / total)))
    ref_g = t64 * gs
    # (x - t) * gs: 2 roundings (gs itself is taken as the kernel forms it: 2 * g * inv_numel in fp32)
    _check('mse_to_const %s t=%g bwd' % (shape, target), xc.grad, ref_g, 2 * EPS * ref_g.abs() + 1e-30)


# ------------------------------------------------------------------------------------------------ FlowNet glue
def _resize_scales(h, w, H, W, use_sf):
    f = np.float32
    if use_sf:
        return f(f(1.0) / f(f(H) / f(h))), f(f(1.0) / f(f(W) / f(w)))
    return f(f(h) / f(H)), f(f(w) / f(W))


def _resize_ref(x, H, W, mode, use_sf, mul, pre_div):
    """ATen upsample_{bilinear,nearest}2d index rule (align_corners=False) with the fp32 scale; bilinear weights and blend in
    fp64, the index arithmetic in fp32 as the kernel forms it."""
    h, w = x.shape[-2:]
    sh, sw = _resize_scales(h, w, H, W, use_sf)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)
    Y, X = torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32)
    v = x.float()
    v = v / f32(pre_div) if pre_div != 1.0 else v * f32(mul)            # fp32, as the kernel rounds each read value
    if mode == 'nearest':
        ys = torch.floor(Y * f32(sh)).long().clamp(max=h - 1)
        xs = torch.floor(X * f32(sw)).long().clamp(max=w - 1)
        return v[..., ys, :][..., xs].double(), None
    fy = (f32(sh) * (Y + f32(0.5)) - f32(0.5)).clamp(min=0)
    fx = (f32(sw) * (X + f32(0.5)) - f32(0.5)).clamp(min=0)
    y0, x0 = fy.long().clamp(max=h - 1), fx.long().clamp(max=w - 1)
    y1, x1 = (y0 + 1).clamp(max=h - 1), (x0 + 1).clamp(max=w - 1)
    ly, lx = (fy - y0.float()).double().view(H, 1), (fx - x0.float()).double().view(1, W)
    vd = v.double()
    g = lambda yy, xx: vd[..., yy, :][..., xx]
    top = (1 - lx) * g(y0, x0) + lx * g(y0, x1)
    bot = (1 - lx) * g(y1, x0) + lx * g(y1, x1)
    ref = (1 - ly) * top + ly * bot
    mag = (1 - ly) * ((1 - lx) * g(y0, x0).abs() + lx * g(y0, x1).abs()) + ly * ((1 - lx) * g(y1, x0).abs() + lx * g(y1, x1).abs())
    return ref, mag


@pytest.mark.parametrize('case', [
    ((1, 2) + (FN2[0] // 4, FN2[1] // 4), FN2, 'bilinear', True, 20.0, 1.0, 20.0),     # flownetc / flownets_1 x4 upsampling
    ((1, 2) + (FN2[0] // 4, FN2[1] // 4), FN2, 'nearest', True, 20.0, 1.0, 20.0),      # flownets_2
    ((1, 2) + (FN2[0] // 4, FN2[1] // 4), FN2, 'nearest', True, 1.0, 20.0, None),      # flownets_d, divided by div_flow
    ((2, 3, 540, 960), (512, 960), 'bilinear', False, 1.0, 1.0, None),                  # to a multiple of 64
    ((2, 2, 512, 960), (540, 960), 'bilinear', False, 540 / 512, 1.0, None),            # the flow back, scaled
    ((2, 1, 512, 960), (540, 960), 'bilinear', False, 1.0, 1.0, None),                  # the confidence back
    ((1, 3, 7, 9), (20, 13), 'bilinear', False, 1.0, 1.0, 3.0),
    ((1, 3, 20, 13), (7, 9), 'nearest', False, 2.5, 1.0, None),
], ids=['x4_bilinear', 'x4_nearest', 'x4_nearest_prediv', 'to64', 'flow_back', 'conf_back', 'up_odd', 'down_nearest'])
def test_resize(case):
    shape, (H, W), mode, use_sf, mul, pre_div, div = case
    g = torch.Generator().manual_seed(41)
    x = _noise(shape, g) * 4
    out = FN.resize(x.cuda(), H, W, mode, use_sf, mul=mul, pre_div=pre_div, div=div)
    out, out_div = out if div is not None else (out, None)
    torch.cuda.synchronize()
    ref, mag = _resize_ref(x, H, W, mode, use_sf, mul, pre_div)
    tag = 'resize %s %s -> %dx%d mul %g pre_div %g' % (mode, shape, H, W, mul, pre_div)
    if mode == 'nearest':
        assert torch.equal(out.cpu().double(), ref), tag          # an index and one fp32 product / quotient: exact
        _report(tag, 0.0, 0.0)
    else:
        # 2 + 2 products, 2 adds, 2 (1 - l) and the fp32 rounding of the result: 8 EPS of the weighted |values|
        _check(tag, out, ref, 8 * EPS * mag + 1e-30)
    if div is not None:
        assert torch.equal(out_div, out / torch.tensor(div, dtype=torch.float32, device='cuda')), tag


def _below(v):
    return np.nextafter(np.float32(v), np.float32(0))


def _conf_pixels():
    """(im1 - warp) triples whose fp32 sequential sum of squares is exactly 0.02f and the float just below it."""
    t = np.float32(0.02)
    found = {}
    base = np.float32(math.sqrt(0.02))
    d0s = base + (np.arange(-400, 400, dtype=np.float32) * np.spacing(base))
    for d1 in np.float32([0.0, 1e-4, 2e-4, 3e-4, 1e-3, 2e-3]):
        for d0 in d0s:
            s = np.float32(np.float32(d0 * d0) + np.float32(d1 * d1))
            for want in (t, _below(t)):
                if s == want and want not in found:
                    found[want] = (d0, d1)
    assert set(found) == {t, _below(t)}, found
    return found[t], found[_below(t)]


@pytest.mark.parametrize('shape', [(2, 3, 13, 22), (1, 3) + FN2], ids=['small', 'flownet2_%dx%d' % FN2])
def test_flow_conf(shape):
    g = torch.Generator().manual_seed(42)
    N, Cc, H, W = shape
    im1 = _noise(shape, g) * 0.1
    warp = im1 + torch.randn(shape, generator=g) * 0.06
    (e0, e1), (b0, b1) = _conf_pixels()
    for (n, y, x), (d0, d1) in (((0, 1, 2), (e0, e1)), ((N - 1, H - 1, W - 1), (b0, b1))):
        im1[n, :, y, x] = torch.tensor([d0, d1, 0.0])
        warp[n, :, y, x] = 0.0
    conf = torch.empty(N, 1, H, W, device='cuda')
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    ic, wc = im1.cuda(), warp.cuda()
    L.check(L.lib().v2v_flow_conf(p(ic), p(wc), p(conf), N, Cc, H, W, 0.02, st))
    torch.cuda.synchronize()
    d = im1 - warp                                        # fp32, then a sequential fp32 sum of the unfused squares
    s = torch.zeros(N, 1, H, W)
    for c in range(Cc):
        s = s + d[:, c:c + 1] * d[:, c:c + 1]
    ref = (s < torch.tensor(0.02, dtype=torch.float32)).float()
    assert ref[0, 0, 1, 2] == 0 and ref[N - 1, 0, H - 1, W - 1] == 1
    mism = int((conf.cpu() != ref).sum())
    _report('flow_conf %s (%.1f%% confident)' % (shape, 100 * ref.mean().item()), float(mism), float(mism))
    assert mism == 0


@pytest.mark.parametrize('B,HW', [(2, (13, 22)), (1, FN2)], ids=['small', 'flownet2_%dx%d' % FN2])
@pytest.mark.parametrize('layout', ['stacked', 'separate'])
def test_flownet_prep_and_sub_channels(B, HW, layout):
    H, W = HW
    hw = H * W
    g = torch.Generator().manual_seed(43)
    pair = torch.randint(0, 256, (B, 3, 2, H, W), generator=g).float() / 255.0
    rgb_max = 1.0 if layout == 'stacked' else 255.0
    if layout == 'stacked':                               # FlowNet2.forward: (B,3,2,H,W)
        src = pair.cuda()
        f0, f1, bs, cs = src, src.view(-1)[hw:], 6 * hw, 2 * hw
    else:                                                 # FlowNet.compute_flow_and_conf: two (B,3,H,W) images
        a, b = pair[:, :, 0].contiguous().cuda(), pair[:, :, 1].contiguous().cuda()
        f0, f1, bs, cs = a, b, 3 * hw, hw
    x, x1 = torch.empty(B, 6, H, W, device='cuda'), torch.empty(B, 3, H, W, device='cuda')
    ws = torch.empty(B * 3, device='cuda')
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    L.check(L.lib().v2v_flownet_prep(p(f0), p(f1), bs, cs, p(x), p(x1), p(ws), B, H, W, rgb_max, st))
    torch.cuda.synchronize()
    # the mean over both frames in fp64 rounded to fp32; then the fp32 subtraction and division
    mean = pair.double().mean(dim=(2, 3, 4)).float().view(B, 3, 1, 1, 1)
    ref = ((pair - mean) / torch.tensor(rgb_max)).permute(0, 2, 1, 3, 4).reshape(B, 6, H, W)
    assert torch.equal(ws.cpu().view(B, 3), mean.view(B, 3))
    assert torch.equal(x.cpu(), ref)
    assert torch.equal(x1.cpu(), ref[:, 3:])
    # sub_channels: x[:, 0:3] - warped, exact
    warped = torch.randn(B, 3, H, W, generator=g).cuda()
    diff = torch.empty_like(warped)
    L.check(L.lib().v2v_sub_channels(p(x), p(warped), p(diff), B, 6, 0, 3, H, W, st))
    torch.cuda.synchronize()
    assert torch.equal(diff, x[:, 0:3] - warped)
    _report('flownet_prep / sub_channels %s %dx%d B%d' % (layout, H, W, B), 0.0, 0.0)


def test_correlation_flownetc_size():
    """FlowNetC correlates its two conv3 features (256 channels) at 1/8 of the flownet2 workload's frame."""
    g = torch.Generator().manual_seed(44)
    H, W = FN2[0] // 8, FN2[1] // 8
    a, b = torch.randn(1, 256, H, W, generator=g) * 0.5, torch.randn(1, 256, H, W, generator=g) * 0.5
    out = ops.correlation(a.cuda(), b.cuda())
    torch.cuda.synchronize()
    ref = torch.from_numpy(np.asarray(flowops.correlation(a.double().numpy(), b.double().numpy()), dtype=np.float64))
    mag = torch.from_numpy(np.asarray(flowops.correlation(a.abs().double().numpy(), b.abs().double().numpy()), dtype=np.float64))
    # a 256-term fp32 dot product (any order) and the division by 256 (exact): (256 + 1) EPS of sum |a b| / 256
    _check('correlation 256x%dx%d' % (H, W), out, ref, 257 * EPS * mag + 1e-30)
