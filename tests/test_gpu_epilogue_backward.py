"""The CUDA-core epilogue backward (csrc/backward.cu) against fp64 at the shapes cfg3's training step runs, on every launch path:
norm_bwd_reduce_vec_kernel / norm_bwd_reduce_kernel, norm_bwd_apply_kernel, norm_param_grad_kernel, convact_bwd_kernel,
head_bwd_kernel, bias_grad_kernel and the gradient import / export (tiled and scalar).

Each case is a training plan (fp32 SIMT backward, V2V_BWD=simt) whose every input is known exactly to the test:
  * inputs on the grid k / 256, |k| <= 255: bf16-exact, and their sums and squares fall on the 2^-20 / 2^-16 grids of the
    fixed-point statistics rows, so the batch statistics are exact up to the fp32 rounding of mean, rstd, scale and shift
    (checked through the exported normalised output against a forward bound that assumes exact statistics);
  * an identity 1x1 conv (stacked [I 0] / [0 I] for channel slices): the raw conv output is the input, and the conv's SIMT data
    gradient is an exact copy of draw (one nonzero product of 1.0 per output);
  * beta is placed so that every pre-activation z lies at least DELTA from zero in fp64: the fp32 ReLU / LeakyReLU gates equal
    the fp64 gates, also where addends hide the gate from the output.
The input and every addend come from their own caller slot through a channel window, and the caller gradient tensors are
pre-filled with a pattern, since the export adds (+=) into them.  Addend gradients must equal the incoming gradient bit for bit,
and every element outside the windows must keep the pattern bit for bit.

Bounds (EPS = 2^-23, fp32 machine epsilon; a rounding costs at most EPS / 2, so k roundings stay within k EPS / 2):
  * a per-channel sum of M terms: each term passes D additions, D = T sequential terms in its thread + the block's combine (ppb
    shared atomics for the vectorised reduce, 8 tree levels for the scalar and bias kernels) + the global atomics of the blocks
    that share its row + the rows norm_param_grad_kernel adds; error <= D EPS sum|term|;
  * dgamma's terms dz (raw - mean) rstd carry the rounding of the fp32 mean (EPS |mean| rstd |dz|) and ~5 EPS of their size
    (rstd after its Newton step, the subtraction and two products);
  * dX = sc (dz - s1 inv_m - xhat s2 inv_m): the errors of s1 and s2 over M, plus 12 EPS of sc (|dz| + |s1| / M + |xhat s2| / M)
    for the six roundings of the expression, inv_m, xhat and sc = gamma rstd;
  * the export adds onto the pattern: one more rounding, EPS |pattern + dX|.
Every tensor prints observed error / bound."""
import collections
import math

import pytest
import torch
import torch.nn as nn

from vid2vid_b200 import _lib as L
from vid2vid_b200.plan import Plan, conv_desc, norm_desc

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
DELTA = 1e-3
SLOPE = 0.2
SLOPE32 = float(torch.tensor(SLOPE, dtype=torch.float32))     # the fp32 slope the kernels multiply by
C_PAD = 3            # extra channels of every caller tensor around its window

# Norm: a 1x1 identity conv, then one normalise pass per (c_off, Cn) slice of its raw output (`pair` stacks two identity convs
# as emit_unit_pair does), each with `adds` addends; `twice` normalises the raw a second time with its own addends, as
# CompositeLocalGenerator's defer_last does.
Norm = collections.namedtuple('Norm', 'N C H W norm act adds pair twice fast')
# Head: a 1x1 identity head over `C` input channels, channel j -> (act, scale); `split` stacks a second conv from channel split on
# (emit_head_pair).  ConvAct: a biased 1x1 identity conv with an activation (the discriminator's first layer).
Head = collections.namedtuple('Head', 'N H W chans split')
ConvAct = collections.namedtuple('ConvAct', 'N C H W act')


def _n(N, C, H, W, act, adds=0, norm='batch', pair=None, twice=False, fast=False):
    return Norm(N, C, H, W, norm, act, adds, pair, twice, fast)


RELU, LRELU, NONE, TANH, SIGM = L.ACT_RELU, L.ACT_LRELU, L.ACT_NONE, L.ACT_TANH, L.ACT_SIGMOID

CASES = [
    # cfg3's generator scales (G1 = 512x1024, G0 = 256x512), N = 1, BatchNorm
    ('g1_stem_pair_64_32', _n(1, 96, 512, 1024, RELU, pair=(64, 32))),                 # 528 blocks, ragged chunk 993; 32 ch at c_off 64
    ('g1_128_256x512_relu_add2_twice', _n(1, 128, 256, 512, RELU, 2, twice=True)),     # gate hidden by the addends; 2 passes
    ('g1_128_256x512_add1', _n(1, 128, 256, 512, NONE, 1)),                            # resblock
    ('g1_64_256x512_relu_add1', _n(1, 64, 256, 512, RELU, 1)),
    ('g0_512_64x128_relu', _n(1, 512, 64, 128, RELU)),                                 # chunk 16, not ragged
    ('g0_512_32x64_add1', _n(1, 512, 32, 64, NONE, 1)),
    ('g0_1024_32x64_relu', _n(1, 1024, 32, 64, RELU)),                                 # ppb 1, chunk 8
    ('g0_1024_32x64_add1', _n(1, 1024, 32, 64, NONE, 1)),
    ('g0_1024_32x64_add2', _n(1, 1024, 32, 64, NONE, 2)),
    # the discriminator towers: LeakyReLU norm units on the avg-pool pyramid
    ('d_512_66x130_lrelu', _n(1, 512, 66, 130, LRELU)),                                # 505 blocks, ragged chunk 17
    # per-image rows and inv_m, at HW % 32 != 0 and C % 32 != 0 (tiled import / export edges)
    ('bn_n2_40_37x45_relu_add1', _n(2, 40, 37, 45, RELU, 1)),
    ('in_n2_40_37x45_lrelu', _n(2, 40, 37, 45, LRELU, norm='instance')),
    # the scalar reduce (C % 4 != 0; C > 1024); C = 6 also takes the scalar import / export kernels (C < 8)
    ('scalar_c6_33x47_relu', _n(1, 6, 33, 47, RELU)),
    ('scalar_c1032_96x176_relu', _n(1, 1032, 96, 176, RELU)),
    # a bf16-raw (fast-mode) plan
    ('fast_128_64x96_relu_add1', _n(1, 128, 64, 96, RELU, 1, fast=True)),
    # heads: the image head (tanh) and the stacked flow (x 20 * 2^1 at cfg3's finest scale) + weight (sigmoid) pair, the
    # discriminator logits with several and with one bias-gradient block per channel; conv_act LeakyReLU + bias at the first
    # discriminator layer, likewise; the 3-channel heads also take the scalar export of the input gradient (C < 8)
    ('head_tanh_512x1024', Head(1, 512, 1024, [(TANH, 1.0)] * 3, None)),
    ('head_flow_w_512x1024', Head(1, 512, 1024, [(NONE, 40.0), (NONE, 40.0), (SIGM, 1.0)], 2)),
    ('head_logit_67x131', Head(1, 67, 131, [(NONE, 1.0)], None)),
    ('head_logit_35x67', Head(1, 35, 67, [(NONE, 1.0)], None)),
    ('convact_lrelu_64_257x513', ConvAct(1, 64, 257, 513, LRELU)),
    ('convact_lrelu_64_65x65', ConvAct(1, 64, 65, 65, LRELU)),
]

S_X = 0          # input slot; addends, outputs and head planes follow


def precision(spec):
    return 'fast' if isinstance(spec, Norm) and spec.fast else 'precise'


def _identity(cin, cout, first, bias, device):
    """1x1 conv cin -> cout whose output channel j reads input channel first + j with weight 1."""
    conv = nn.Conv2d(cin, cout, 1, bias=bias).to(device)
    with torch.no_grad():
        conv.weight.zero_()
        for j in range(cout):
            conv.weight[j, first + j, 0, 0] = 1.0
        if bias:
            conv.bias.copy_((torch.arange(cout, dtype=torch.float32) % 7 - 3) / 256.0)
    return conv


def _slices(spec):
    return [(0, spec.pair[0]), (spec.pair[0], spec.pair[1])] if spec.pair else [(0, spec.C)]


def build(plan, spec, device):
    """Describe the case on `plan` with its modules on `device` -> context for the test (modules, slots, ...)."""
    ctx = {}
    if isinstance(spec, Norm):
        x = plan.input(S_X, spec.N, spec.C + C_PAD, 2, spec.C, spec.H, spec.W, exact_bf16=True)
        if spec.pair:
            ca, cb = (_identity(spec.C, c, f, False, device) for c, f in ((spec.pair[0], 0), (spec.pair[1], spec.pair[0])))
            raw = plan.conv(x, conv_desc(ca, m2=cb))
            ctx['convs'] = [ca, cb]
        else:
            conv = _identity(spec.C, spec.C, 0, False, device)
            raw = plan.conv(x, conv_desc(conv))
            ctx['convs'] = [conv]
        slot = S_X + 1
        units = []
        for c_off, cn in _slices(spec):
            nm = (nn.BatchNorm2d(cn) if spec.norm == 'batch' else nn.InstanceNorm2d(cn, affine=True)).to(device)
            for p_ in range(2 if spec.twice else 1):
                adds, add_slots = [], []
                for a in range(spec.adds):
                    adds.append(plan.input(slot, spec.N, cn + C_PAD, 1, cn, spec.H, spec.W, exact_bf16=True))
                    add_slots.append(slot)
                    slot += 1
                v = plan.norm_act(raw, norm_desc(nm), spec.act, SLOPE if spec.act == LRELU else 0.0, adds,
                                  **({'c_off': c_off, 'Cn': cn} if spec.pair else {}))
                plan.export(v, slot)
                units.append(dict(c_off=c_off, Cn=cn, norm=nm, add_slots=add_slots, out_slot=slot))
                slot += 1
        ctx['units'] = units
    elif isinstance(spec, Head):
        C = len(spec.chans)
        x = plan.input(S_X, spec.N, C + C_PAD, 2, C, spec.H, spec.W, exact_bf16=True)
        groups = [(0, spec.split), (spec.split, C - spec.split)] if spec.split else [(0, C)]
        convs = [_identity(C, n, f, True, device) for f, n in groups]
        slots = [S_X + 1 + i for i in range(len(groups))]
        chans = []
        for (f, n), s in zip(groups, slots):
            chans += [(s, j, n, spec.chans[f + j][0], spec.chans[f + j][1]) for j in range(n)]
        plan.head(x, conv_desc(convs[0], m2=convs[1] if spec.split else None), chans)
        ctx.update(convs=convs, groups=groups, slots=slots)
    else:
        x = plan.input(S_X, spec.N, spec.C + C_PAD, 2, spec.C, spec.H, spec.W, exact_bf16=True)
        conv = _identity(spec.C, spec.C, 0, True, device)
        v = plan.conv_act(x, conv_desc(conv), spec.act, SLOPE)
        plan.export(v, S_X + 1)
        ctx.update(convs=[conv], out_slot=S_X + 1)
    return ctx


# ------------------------------------------------------------------------------------------------ helpers
def _report(what, ratio, err):
    print('%-64s observed/bound %.3g  (max err %.3g)' % (what, ratio, err))


def _check(what, got, ref, bound):
    d = (got.double() - ref).abs()
    ratio = (d / bound.clamp_min(1e-300)).max().item()
    _report(what, ratio, d.max().item())
    assert torch.isfinite(got).all(), what
    assert ratio <= 1.0, (what, ratio)


def _grid(shape, g, lim=255):
    """Values k / 256, |k| <= lim, drawn on the CPU (seeded) and moved to the GPU."""
    return (torch.randint(-lim, lim + 1, shape, generator=g).float() / 256.0).cuda()


def _pattern(shape, g):
    return _grid(shape, g) * 3.0


def _incoming(shape, g):
    """Incoming gradient with a mean of its own: its per-channel sums grow with the pixel count, so a dropped or rescaled
    term, or a wrong 1 / M, shows well above the rounding bounds."""
    return (torch.randn(shape, generator=g) * 0.5 + 0.75).cuda()


def _window(t, c_off, C):
    return t[:, c_off:c_off + C]


def _outside_equal(what, got, pattern, c_off, C):
    m = torch.ones(got.shape[1], dtype=torch.bool, device=got.device)
    m[c_off:c_off + C] = False
    assert torch.equal(got[:, m], pattern[:, m]), what + ': elements outside the window changed'


def _sum_depth(rec, group_images):
    """Additions a term of a per-channel sum passes in the norm backward (module docstring), plus one for LeakyReLU's dz."""
    HW = rec['H'] * rec['W']
    rows = 1 if rec['batch_stats'] else rec['N']
    blocks = rec['grid'][0] if rec['reduce'] == 'vec' else rec['grid'][2]
    if rec['reduce'] == 'vec':
        inner = math.ceil(rec['chunk'] / rec['ppb']) + rec['ppb']
    else:
        inner = math.ceil(HW / (256 * rec['grid'][2])) + 8
    return inner + blocks * group_images + rows + 1


# ------------------------------------------------------------------------------------------------ norm units
def _beta_off_grid(x, gamma, norm, eps):
    """beta per channel so that z = gamma (x - mean) rstd + beta sits halfway between two of the values the grid k / 256
    gives it, for every image (the instance case draws its images as shifts of one another, which keeps them on one lattice)."""
    dims = (0, 2, 3) if norm == 'batch' else (2, 3)
    mean = x.mean(dims, keepdim=True)
    var = x.var(dims, unbiased=False, keepdim=True)
    a = gamma.view(1, -1, 1, 1) * (var + eps).rsqrt() / 256.0            # spacing of z along the grid
    b0 = -gamma.view(1, -1, 1, 1) * (var + eps).rsqrt() * mean             # z at x = 0
    frac = torch.remainder(b0[:1] / a[:1], 1.0)
    return (a[:1] * (0.5 - frac) + a[:1] * 3.0).flatten()                   # b0 + beta == (j + 0.5) a, plus three steps


def _norm_case(spec, plan, ctx, g):
    N, C, H, W = spec.N, spec.C, spec.H, spec.W
    if spec.norm == 'instance':
        base = torch.randint(-200, 201, (1, C, H, W), generator=g)
        x = torch.cat([base, base.flatten(2)[..., torch.randperm(H * W, generator=g)].view(1, C, H, W) + 37], 0).float() / 256.0
        x = x.cuda()
    else:
        x = _grid((N, C, H, W), g)
    units = ctx['units']
    io = [None] * plan.n_slots
    gio = [None] * plan.n_slots
    io[S_X] = torch.zeros(N, C + C_PAD, H, W, device='cuda')
    io[S_X][:, 2:2 + C] = x
    gio[S_X] = _pattern((N, C + C_PAD, H, W), g)
    pat_x = gio[S_X].clone()
    params, grads = [], []
    x64 = x.double()
    norms = list(dict.fromkeys(u['norm'] for u in units))       # one per slice; the passes of a twice-normalised slice share it
    for nm in norms:
        u = next(u for u in units if u['norm'] is nm)
        with torch.no_grad():
            gam = torch.randint(192, 385, (u['Cn'],), generator=g).float() / 256.0 * (torch.randint(0, 2, (u['Cn'],), generator=g) * 2 - 1)
            nm.weight.copy_(gam.cuda())
            xs = _window(x64, u['c_off'], u['Cn'])
            nm.bias.copy_(_beta_off_grid(xs, nm.weight.double(), spec.norm, nm.eps).float())
        params += [nm.weight, nm.bias]
        grads += [torch.zeros_like(nm.weight), torch.zeros_like(nm.bias)]
    for u in units:
        for s in u['add_slots']:
            io[s] = torch.zeros(N, u['Cn'] + C_PAD, H, W, device='cuda')
            io[s][:, 1:1 + u['Cn']] = _grid((N, u['Cn'], H, W), g)
            gio[s] = _pattern((N, u['Cn'] + C_PAD, H, W), g)
        io[u['out_slot']] = torch.empty(N, u['Cn'], H, W, device='cuda')
        gio[u['out_slot']] = _incoming((N, u['Cn'], H, W), g)
    pats = {s: gio[s].clone() for u in units for s in u['add_slots']}
    d = plan.describe()
    assert all(b['mode'] == 0 for b in d['backward']), d['backward']      # SIMT: the identity conv's data gradient copies draw
    recs = [r for r in d['epilogue_backward'] if r['kind'] == 'norm_act']
    assert len(recs) == len(units)
    plan.run(io, use_graph=False)
    plan.backward(io, gio, params, grads)
    torch.cuda.synchronize()

    fwd_rel = 2.0 ** -8 if spec.fast else 2.0 ** -16        # bf16 output / split (hi + lo) bf16 output
    dims = (0, 2, 3) if spec.norm == 'batch' else (2, 3)
    dX = torch.zeros_like(x64)
    dX_bound = torch.zeros_like(x64)
    pgrad = {nm: [0.0, 0.0, 0.0, 0.0] for nm in norms}                    # norm -> [dgamma, dbeta, bound g, bound b]
    for u, rec in zip(units, recs):
        tag = '%s pass @%d' % (spec_tag(spec), u['out_slot'])
        assert (rec['c_off'], rec['C']) == (u['c_off'], u['Cn'])
        nm = u['norm']
        xs = _window(x64, u['c_off'], u['Cn'])
        gam, bet = nm.weight.detach().double().view(1, -1, 1, 1), nm.bias.detach().double().view(1, -1, 1, 1)
        mean = xs.mean(dims, keepdim=True)
        rstd = (xs.var(dims, unbiased=False, keepdim=True) + nm.eps).rsqrt()
        xhat = (xs - mean) * rstd
        z = gam * xhat + bet
        adds = [_window(io[s], 1, u['Cn']).double() for s in u['add_slots']]
        if spec.act != NONE:
            zmin = z.abs().min().item()
            assert zmin >= DELTA, (tag, zmin)
        gate = torch.ones_like(z) if spec.act == NONE else torch.where(z > 0, 1.0, 0.0 if spec.act == RELU else SLOPE32)
        out = z * gate + sum(adds) if adds else z * gate
        sc = gam * rstd
        # forward: exact statistics leave the fp32 mean / rstd / scale / shift (~4 EPS of their terms) and the fma; then the addends
        # and the output's bf16 (split) rounding
        fb = fwd_rel * out.abs() + 8 * EPS * ((xs * sc).abs() + (mean * sc).abs() + bet.abs() + sum(a.abs() for a in adds))
        got_out = io[u['out_slot']]
        _check(tag + ' forward (exact statistics)', got_out, out, fb + 1e-30)
        if spec.act != NONE and not adds:
            assert torch.equal(got_out > 0, z > 0), tag + ': fp32 gates differ from fp64'
        dy = gio[u['out_slot']].double()
        dz = dy * gate
        M = xs.numel() // u['Cn'] if spec.norm == 'batch' else spec.H * spec.W
        D = _sum_depth(rec, N if spec.norm == 'batch' else 1)
        s1, s2 = dz.sum(dims, keepdim=True), (dz * xhat).sum(dims, keepdim=True)
        a1, a2 = dz.abs().sum(dims, keepdim=True), (dz * xhat).abs().sum(dims, keepdim=True)
        e1 = D * EPS * a1
        e2 = (D + 5) * EPS * a2 + EPS * a1 * (mean * rstd).abs()
        dx = sc * (dz - s1 / M - xhat * s2 / M)
        bx = sc.abs() * (e1 / M + xhat.abs() * e2 / M + 12 * EPS * (dz.abs() + s1.abs() / M + (xhat * s2).abs() / M))
        sl = slice(u['c_off'], u['c_off'] + u['Cn'])
        dX_bound[:, sl] += bx + EPS * (dX[:, sl] + dx).abs()            # a second pass adds onto draw: one rounding
        dX[:, sl] += dx
        pg = pgrad[nm]
        pg[0] = pg[0] + s2.sum((0, 2, 3)) if spec.norm == 'instance' else pg[0] + s2.flatten()
        pg[1] = pg[1] + s1.sum((0, 2, 3)) if spec.norm == 'instance' else pg[1] + s1.flatten()
        pg[2] = pg[2] + (e2.sum((0, 2, 3)) if spec.norm == 'instance' else e2.flatten()) + EPS * pg[0].abs()
        pg[3] = pg[3] + (e1.sum((0, 2, 3)) if spec.norm == 'instance' else e1.flatten()) + EPS * pg[1].abs()
        # addends: the incoming gradient, bit for bit, added onto the pattern inside the window only
        for s in u['add_slots']:
            want = pats[s].clone()
            want[:, 1:1 + u['Cn']] += gio[u['out_slot']]
            assert torch.equal(gio[s], want), tag + ': addend gradient differs from the incoming gradient'
    for k, nm in enumerate(norms):            # params / grads hold (weight, bias) per norm, in this order
        pg = pgrad[nm]
        _check('%s dgamma' % spec_tag(spec), grads[2 * k], pg[0], pg[2] + 1e-30)
        _check('%s dbeta' % spec_tag(spec), grads[2 * k + 1], pg[1], pg[3] + 1e-30)
    ref = pat_x.double()
    ref[:, 2:2 + C] += dX
    bound = torch.zeros_like(ref)
    bound[:, 2:2 + C] = dX_bound + EPS * ref[:, 2:2 + C].abs()
    _check('%s dX' % spec_tag(spec), gio[S_X], ref, bound + 1e-30)
    _outside_equal(spec_tag(spec) + ' dX', gio[S_X], pat_x, 2, C)


# ------------------------------------------------------------------------------------------------ heads and conv_act
def _bias_bound(dz, dz_err, rec):
    """Per channel: sum dz (fp64 reference, elementwise error bound dz_err) as bias_grad_kernel sums the kernel's own dz:
    T strided terms per thread, 8 tree levels, grid.y blocks per channel meeting in global atomics, over terms of size up to
    |dz| + dz_err; plus the sum of the terms' own errors."""
    npix = dz.shape[0] * dz.shape[2] * dz.shape[3]
    G = rec['bias_grid'][1]
    D = math.ceil(npix / (256 * G)) + 8 + G
    return D * EPS * (dz.abs() + dz_err).sum((0, 2, 3)) + dz_err.sum((0, 2, 3))


def _check_input_grad(tag, got, pat, dz, dz_err, C):
    """Input gradient of an identity head / conv_act: dz added (+=) onto the pattern inside the window, one more rounding;
    the pattern untouched outside it."""
    ref = pat.double()
    ref[:, 2:2 + C] += dz
    bound = torch.zeros_like(ref)
    bound[:, 2:2 + C] = dz_err + EPS * ref[:, 2:2 + C].abs()
    _check(tag + ' dz (exported onto the pattern)', got, ref, bound + 1e-30)
    _outside_equal(tag + ' dX', got, pat, 2, C)


def _head_case(spec, plan, ctx, g):
    N, H, W = spec.N, spec.H, spec.W
    C = len(spec.chans)
    io, gio = [None] * plan.n_slots, [None] * plan.n_slots
    io[S_X] = torch.zeros(N, C + C_PAD, H, W, device='cuda')
    io[S_X][:, 2:2 + C] = _grid((N, C, H, W), g, 200) * 2
    gio[S_X] = _pattern((N, C + C_PAD, H, W), g)
    pat = gio[S_X].clone()
    for (f, n), s in zip(ctx['groups'], ctx['slots']):
        io[s] = torch.empty(N, n, H, W, device='cuda')
        gio[s] = _incoming((N, n, H, W), g)
    params = [p_ for c in ctx['convs'] for p_ in (c.bias,)]
    grads = [torch.zeros_like(p_) for p_ in params]
    d = plan.describe()
    assert all(b['mode'] == 0 for b in d['backward']), d['backward']
    (rec,) = d['epilogue_backward']
    plan.run(io, use_graph=False)
    plan.backward(io, gio, params, grads)
    torch.cuda.synchronize()
    tag = spec_tag(spec)
    refs, bounds = [], []
    for (f, n), s in zip(ctx['groups'], ctx['slots']):
        for j in range(n):
            act, scale = spec.chans[f + j]
            gs = gio[s][:, j].double() * scale
            t = io[s][:, j].double() / scale
            # g * scale, out / scale, then tanh: t*t, 1 - ., * (sigmoid: 1 - t, t * ., *): <= 5 roundings of their terms
            if act == TANH:
                refs.append(gs * (1 - t * t)); bounds.append(3 * EPS * gs.abs() * ((1 - t * t).abs() + t * t))
            elif act == SIGM:
                refs.append(gs * t * (1 - t)); bounds.append(3 * EPS * gs.abs() * ((t * (1 - t)).abs() + t.abs()))
            else:
                refs.append(gs); bounds.append(EPS * gs.abs())
    dz, dz_err = torch.stack(refs, 1), torch.stack(bounds, 1)
    _check_input_grad(tag, gio[S_X], pat, dz, dz_err, C)
    sums = dz.sum((0, 2, 3))
    bb = _bias_bound(dz, dz_err, rec)
    for (f, n), gr in zip(ctx['groups'], grads):
        _check('%s dbias[%d:%d] (C1 %d)' % (tag, f, f + n, rec['C1']), gr, sums[f:f + n], bb[f:f + n] + 1e-30)


def _convact_case(spec, plan, ctx, g):
    N, C, H, W = spec.N, spec.C, spec.H, spec.W
    io, gio = [None] * plan.n_slots, [None] * plan.n_slots
    io[S_X] = torch.zeros(N, C + C_PAD, H, W, device='cuda')
    io[S_X][:, 2:2 + C] = _grid((N, C, H, W), g)
    gio[S_X] = _pattern((N, C + C_PAD, H, W), g)
    pat = gio[S_X].clone()
    s = ctx['out_slot']
    io[s] = torch.empty(N, C, H, W, device='cuda')
    gio[s] = _incoming((N, C, H, W), g)
    conv = ctx['convs'][0]
    grads = [torch.zeros_like(conv.bias)]
    d = plan.describe()
    assert all(b['mode'] == 0 for b in d['backward']), d['backward']
    (rec,) = d['epilogue_backward']
    plan.run(io, use_graph=False)
    plan.backward(io, gio, [conv.bias], grads)
    torch.cuda.synchronize()
    tag = spec_tag(spec)
    out = io[s]
    z = _window(io[S_X], 2, C).double() + conv.bias.detach().double().view(1, -1, 1, 1)
    _check(tag + ' forward', out, torch.where(z > 0, z, z * SLOPE32), 2.0 ** -16 * z.abs() * (1 + SLOPE32) + 1e-30)
    dy = gio[s].double()
    dz = dy * torch.where(out > 0, 1.0, SLOPE32).double()           # the gate of the plan's own output, as convact_bwd reads it
    dz_err = 0.5 * EPS * dz.abs()                                       # dy * slope: one rounding
    _check_input_grad(tag, gio[S_X], pat, dz, dz_err, C)
    _check('%s dbias (%d blocks per channel)' % (tag, rec['bias_grid'][1]), grads[0], dz.sum((0, 2, 3)), _bias_bound(dz, dz_err, rec) + 1e-30)


def spec_tag(spec):
    return next(n for n, s in CASES if s is spec)


@pytest.mark.parametrize('name,spec', CASES, ids=[c[0] for c in CASES])
def test_epilogue_backward(name, spec, monkeypatch):
    monkeypatch.setenv('V2V_BWD', 'simt')
    plan = Plan(0, precision=precision(spec), train=True)
    ctx = build(plan, spec, 'cuda')
    plan.finalize()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if isinstance(spec, Norm):
        _norm_case(spec, plan, ctx, g)
    elif isinstance(spec, Head):
        _head_case(spec, plan, ctx, g)
    else:
        _convact_case(spec, plan, ctx, g)
