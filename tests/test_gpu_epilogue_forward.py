"""The forward epilogue of the norm layers against fp64 at the products' conv configurations: the statistics conv_umma_kernel
accumulates in its epilogue (fp32 column sums per 32 rows, a shared per-(quarter, column) accumulator over the units a CTA runs,
64-bit fixed-point rows), their finalisation in the conv's tail (channel_side_effects: scale / shift, running statistics,
num_batches_tracked, per-sample flag-gated updates) and the normalise pass (norm_apply_rows_kernel), halos included.

Each case is one conv unit at a product's shape -- Cin, Cout, k, stride, H, W, N -- so that it lowers the product's
accumulation key (tests/test_epilogue_forward_census.py), with exact operands:
  * inputs on the grid k / 16 and weights on j / 16: every product is a multiple of 2^-8, and the fp32 (and tensor-core) sums of
    such terms are exact while sum |x| |w| < 2^16, asserted per case from conv(|x|, |w|).  The raw conv output is then exactly
    the fp64 conv; in fast mode the normalise pass reads bf16(raw), which the reference emulates, while the statistics are
    those of the fp32 values.  The conv biases are nonzero: they cancel in the output and appear in the running mean.
  * momentum 1.0 makes the running buffers the batch mean (plus the conv bias) and the unbiased variance themselves; a second
    run at momentum 0.1 on pre-filled buffers checks the update expression.
  * addends are fp32 values off the bf16 grid, imported as bf16 (fast) or [hi | lo] (precise), which the reference emulates.
    Every output tensor is prefilled with a pattern, so an element the plan leaves unwritten fails the comparison.
  * the value's halo layout is read back through a head (a stride-2 layout: a conv and a norm-less pass) whose output channel j
    copies input channel c_j at one tap: that product is exact (a bf16 pair times 1.0), so the read-back equals the padded
    layout bit for bit.

Bounds (EPS = 2^-23; a rounding costs at most EPS / 2 of its result):
  * sum and sumsq of a channel: a term passes 31 fp32 additions down its 32 rows, then up to u additions into the shared
    accumulator (u = MG x the units a CTA runs), then 3 quarter additions: (34 + u) EPS sum |v| (sum v^2), plus 2^-21 (2^-17)
    per flush onto the fixed-point row (F flushes: at most one per key and image a CTA visits, <= its units).
  * mean = S / cnt, var = Q / cnt - mean^2 (double): dm = dS / cnt, dvar = dQ / cnt + 2 |mean| dm -- on channels whose mean
    dwarfs their spread this cancellation is the bound, not a failure -- plus 2^-50 Q / cnt for the double roundings of the
    kernel's scaling, divisions, product and subtraction (and of the fp64 reference), each 2^-53 of a term <= Q / cnt.
  * rstd = rsqrtf(float(var) + eps) with one Newton step: relative 0.5 dvar / (var + eps) + 3 EPS; scale = gamma rstd: + EPS;
    shift = beta - float(mean) scale: |scale| dm + EPS (|mean scale| + |shift|) + |mean scale| rel(scale).
  * out = fmaf(raw, scale, shift): |raw| |scale| rel(scale) + d(shift) + EPS |z|; LeakyReLU's product one rounding more; each
    fp32 addend addition (two per addend in precise plans) EPS of the running sum; then the output rounding: bf16 (2^-8 relative)
    or the [hi | lo] pair (2^-16 relative), read back through the export's one fp32 addition (EPS).
  * running mean (momentum m): (1 - m) old + m (float(mean) + bias), four roundings; running var: float(var * cnt / (cnt - 1)).
Every tensor prints observed error / bound."""
import collections

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from vid2vid_b200 import _lib as L
from vid2vid_b200.plan import Plan, conv_desc, norm_desc

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
SLOPE = 0.2
SLOPE32 = float(torch.tensor(SLOPE, dtype=torch.float32))
C_PAD = 3
RELU, LRELU, NONE = L.ACT_RELU, L.ACT_LRELU, L.ACT_NONE
ZERO, REFLECT = L.PAD_ZERO, L.PAD_REFLECT

# One conv unit: conv Cin -> Cout (k x k, stride, pad, zero / reflect), then normalise passes.  norm: 'batch' | 'instance' |
# 'bias' (norm-less biased conv, FlowNet2) | 'none'.  pair: (C1, C2) stacks two weight sets along Cout, each slice its own
# BatchNorm (two tail slots).  twice: the slice is normalised a second time (defer_last).  adds: addends per pass.  readback:
# (k, stride, pad, mode) of the consumer that sets the value's layout, read back through a head; None: export only.  N images;
# sample: per-sample statistics; flags: per-image flags (active, inactive, active, ...).  pos: positive inputs and weights
# (mean-dominated channels).  modes: arithmetic modes the case runs in; train: a training plan (saves mean / rstd).  exact: the
# input is declared bf16-exact (the finest scale's label maps), which changes the conv's configuration.  transposed: a stride-2
# ConvTranspose2d (k 3, pad 1, output_padding 1: the generators' upsampling units, four phases).  ident: an identity 1x1 conv
# on fp32 inputs off the bf16 grid (precise plans: raw = hi + lo exactly), whose sums leave the fixed-point grids.
Unit = collections.namedtuple('Unit', 'N Cin Cout k stride pad pmode H W norm act adds pair twice readback sample flags pos modes '
                                   'train exact transposed ident')


def _u(N, Cin, Cout, k, H, W, stride=1, pad=None, pmode=ZERO, norm='batch', act=RELU, adds=0, pair=None, twice=False,
       readback=None, sample=False, flags=False, pos=False, modes=('precise', 'fast'), train=False, exact=True, transposed=False, ident=False):
    return Unit(N, Cin, Cout, k, stride, (k - 1) // 2 if pad is None else pad, pmode, H, W, norm, act, adds, pair, twice,
                readback, sample, flags, pos, ('precise',) if train else modes, train, exact, transposed, ident)


R1, R3, P2 = (3, 1, 1, REFLECT), (7, 1, 3, REFLECT), (3, 2, 1, ZERO)

CASES = [
    # cfg4 / cfg3 G0 (256x512): the stacked stem pair into two tail slots (inference and training); 128 -> 256 -> 512 -> 1024
    # downsampling; resblocks
    ('g0_stem_pair_192', _u(1, 108, 192, 7, 256, 512, pmode=REFLECT, pad=3, pair=(128, 64), readback=P2, exact=False)),
    ('g0_stem_pair_192_train', _u(1, 108, 192, 7, 256, 512, pmode=REFLECT, pad=3, pair=(128, 64), readback=P2, exact=False,
                                  train=True)),
    ('g0_res_1024_add1_zero', _u(1, 1024, 1024, 3, 32, 64, pmode=REFLECT, act=NONE, adds=1, readback=(3, 1, 1, ZERO))),
    ('g0_res_1024_add1_export', _u(1, 1024, 1024, 3, 32, 64, pmode=REFLECT, act=NONE, adds=1)),
    # the upsampling units: ConvTranspose2d + BatchNorm, four phases (G0 1024 -> 512 -> 256 -> 128, G1 128 -> 64)
    ('g0_up_1024_512', _u(1, 1024, 512, 3, 32, 64, stride=2, pad=1, transposed=True, readback=(3, 1, 1, ZERO))),
    ('g1_up_128_64', _u(1, 128, 64, 3, 256, 512, stride=2, pad=1, transposed=True, readback=R3)),
    ('g0_up_512_256_32x64', _u(1, 512, 256, 3, 32, 64, stride=2, pad=1, transposed=True, readback=(3, 1, 1, ZERO))),
    # cfg4 / cfg3 G1 (512x1024): the 64-channel 7x7 stem (MG 2, many units per CTA), the 128-channel 3x3 units; defer_last
    ('g1_stem_64_512x1024', _u(1, 6, 64, 7, 512, 1024, pmode=REFLECT, pad=3, readback=P2)),
    ('g1_128_256x512_twice_add2', _u(1, 128, 128, 3, 256, 512, pmode=REFLECT, act=NONE, adds=2, twice=True, readback=R1)),
    ('g1_128_256x512_export', _u(1, 64, 128, 3, 256, 512)),
    ('g1_64_256x512_add1', _u(1, 64, 64, 3, 256, 512, pmode=REFLECT, act=NONE, adds=1, readback=R1)),
    # cfg3's discriminator: LeakyReLU units with zero pad 2 (4x4 convs), ragged widths
    ('d_128_129x257_lrelu', _u(1, 64, 128, 4, 257, 513, stride=2, pad=2, act=LRELU, readback=(4, 2, 2, ZERO), modes=('precise',))),
    ('d_256_65x129_lrelu', _u(1, 128, 256, 4, 129, 257, stride=2, pad=2, act=LRELU, readback=(4, 1, 2, ZERO), modes=('precise',))),
    # the face first-frame generator's 528-channel units: idle threads (256 % 66 != 0)
    ('face_528_64x64', _u(1, 528, 528, 3, 64, 64, pmode=REFLECT, readback=R1)),
    ('face_528_64x64_add1', _u(1, 528, 528, 3, 64, 64, pmode=REFLECT, act=NONE, adds=1, readback=R1)),
    ('face_528_64x64_add1_export', _u(1, 528, 528, 3, 64, 64, pmode=REFLECT, act=NONE, adds=1)),
    # InstanceNorm (the City first-frame generator)
    ('in_64_256x512', _u(1, 32, 64, 3, 256, 512, norm='instance', readback=R1, modes=('fast',))),
    # FlowNet2's norm-less biased units (LeakyReLU(0.1) convs into 5x5 / 3x3 / 1x1 consumers and the correlation), a
    # predict_flow head padded to 8 channels
    ('flow_conv1_64', _u(1, 3, 64, 7, 512, 1024, stride=2, pad=3, norm='bias', act=LRELU, readback=(5, 2, 2, ZERO), modes=('precise',))),
    ('flow_conv3_256_redir', _u(1, 128, 256, 5, 128, 256, stride=2, pad=2, norm='bias', act=LRELU, readback=(1, 1, 0, ZERO), modes=('precise',))),
    ('flow_conv3_256_corr', _u(1, 128, 256, 5, 128, 256, stride=2, pad=2, norm='bias', act=LRELU, modes=('precise',))),
    ('flow_redir_32', _u(1, 256, 32, 1, 64, 128, norm='bias', act=LRELU, modes=('precise',))),
    ('flow_conv3_1_256', _u(1, 473, 256, 3, 64, 128, norm='bias', act=LRELU, readback=P2, modes=('precise',))),
    ('flow_predict_2', _u(1, 64, 2, 3, 16, 32, norm='bias', act=NONE, readback=(3, 1, 1, ZERO), modes=('precise',))),
    # several clips: per-sample statistics, N = 2, with flags
    ('multiclip_pose_192_pair_n2', _u(2, 108, 192, 7, 256, 128, pmode=REFLECT, pad=3, pair=(128, 64), sample=True, readback=P2,
                                      exact=False)),
    ('multiclip_stem_64_n2', _u(2, 6, 64, 7, 512, 256, pmode=REFLECT, pad=3, sample=True, readback=P2)),
    ('multiclip_up_1024_512_n2', _u(2, 1024, 512, 3, 32, 64, stride=2, pad=1, transposed=True, sample=True, modes=('precise',))),
    ('multiclip_up_512_256_n2', _u(2, 512, 256, 3, 32, 64, stride=2, pad=1, transposed=True, sample=True, modes=('precise',))),
    ('multiclip_pose_up_1024_512_n2', _u(2, 1024, 512, 3, 32, 16, stride=2, pad=1, transposed=True, sample=True,
                                         modes=('precise',))),
    ('multiclip_512_n2', _u(2, 256, 512, 3, 64, 128, stride=2, sample=True, readback=R1)),
    ('slots_192_pair_n2_flags', _u(2, 108, 192, 7, 256, 512, pmode=REFLECT, pad=3, pair=(128, 64), sample=True, flags=True,
                                   readback=P2, modes=('precise',))),
]

# Arithmetic edges at launch paths CASES already reach (tests/test_epilogue_forward_census.py counts CASES only): per-image
# flags over N = 3 (active, inactive, active), channels whose mean dwarfs their spread, and raw values off the bf16 grid, so that
# the column sums leave the 2^-20 / 2^-16 grids and the fixed-point conversion of every flush rounds.
EDGE_CASES = [
    ('fixed_point_identity_64', _u(1, 64, 64, 1, 256, 512, ident=True, exact=False, adds=2, readback=R1, modes=('precise',))),
    ('fixed_point_identity_n2_sample', _u(2, 128, 128, 1, 128, 256, ident=True, exact=False, sample=True, modes=('precise',))),
    ('slots_128_n3_flags', _u(3, 64, 128, 3, 128, 256, sample=True, flags=True, readback=R1)),
    ('mean_dominated_64', _u(1, 64, 64, 3, 128, 256, pos=True, modes=('precise',))),
]

S_X, S_FLAGS = 0, 1


def plan_options(spec, mode=None):
    return dict(precision=mode or spec.modes[0], sample_stats=spec.sample, flags=spec.flags, train=spec.train)


def _slices(spec):
    return [(0, spec.pair[0]), (spec.pair[0], spec.pair[1])] if spec.pair else [(0, spec.Cout)]


def build(plan, spec, device, momentum=1.0):
    """Describe the case on `plan` with its modules on `device` -> context (modules, slots)."""
    if spec.flags:
        plan.set_image_flags(S_FLAGS)
    slot = S_FLAGS + 1
    x = plan.input(S_X, spec.N, spec.Cin + C_PAD, 2, spec.Cin, spec.H, spec.W, exact_bf16=spec.exact)
    bias = spec.norm != 'none'
    if spec.transposed:
        mk = lambda c: nn.ConvTranspose2d(spec.Cin, c, spec.k, spec.stride, spec.pad, output_padding=1, bias=bias).to(device)
        Ho, Wo = spec.H * spec.stride, spec.W * spec.stride
    else:
        mk = lambda c: nn.Conv2d(spec.Cin, c, spec.k, spec.stride, spec.pad, bias=bias).to(device)
        Ho = (spec.H + 2 * spec.pad - spec.k) // spec.stride + 1
        Wo = (spec.W + 2 * spec.pad - spec.k) // spec.stride + 1
    convs = [mk(c) for _, c in _slices(spec)]
    raw = plan.conv(x, conv_desc(convs[0], spec.pmode, spec.pad, m2=convs[1] if spec.pair else None))
    units = []
    for c_off, cn in _slices(spec):
        nm = None
        if spec.norm == 'batch':
            nm = nn.BatchNorm2d(cn, momentum=momentum).to(device)
        elif spec.norm == 'instance':
            nm = nn.InstanceNorm2d(cn, affine=True, track_running_stats=True, momentum=momentum).to(device)
        for _ in range(2 if spec.twice else 1):
            add_slots = []
            adds = []
            for a in range(spec.adds):
                adds.append(plan.input(slot, spec.N, cn + C_PAD, 1, cn, Ho, Wo))
                add_slots.append(slot)
                slot += 1
            v = plan.norm_act(raw, norm_desc(nm), spec.act, SLOPE if spec.act == LRELU else 0.0, adds,
                              **({'c_off': c_off, 'Cn': cn} if spec.pair else {}))
            u = dict(c_off=c_off, Cn=cn, norm=nm, add_slots=add_slots, out_slot=slot)
            slot += 1
            if spec.readback:
                k, s, p, m = spec.readback
                nh = min(cn, 16)
                head = nn.Conv2d(cn, nh, k, s, p, bias=False).to(device)
                if s == 1:
                    plan.head(v, conv_desc(head, m, p), [(slot, j, nh, NONE, 1.0) for j in range(nh)])
                else:       # heads are stride-1: a stride-2 (parity) layout is read through a conv, a norm-less pass and an export
                    plan.export(plan.norm_act(plan.conv(v, conv_desc(head, m, p)), norm_desc(None)), slot)
                u.update(head=head, head_slot=slot)
                slot += 1
            plan.export(v, u['out_slot'])
            units.append(u)
    return dict(convs=convs, units=units, Ho=Ho, Wo=Wo)


# ------------------------------------------------------------------------------------------------ helpers
def _check(what, got, ref, bound):
    d = (got.double() - ref).abs()
    ratio = (d / bound.clamp_min(1e-300)).max().item()
    print('%-72s observed/bound %.3g  (max err %.3g)' % (what, ratio, d.max().item()))
    assert torch.isfinite(got).all(), what
    assert ratio <= 1.0, (what, ratio)


def _grid(shape, g, lo, hi, den=16.0):
    return (torch.randint(lo, hi + 1, shape, generator=g).double() / den).cuda()


def _bf16(t):
    return t.float().bfloat16().double()


def _stored(t, prec):
    """An fp32 tensor as an import leaves it in the plan: bf16(t) (fast), or the [hi | lo] pair hi + lo (precise)."""
    t = t.float()
    hi = t.bfloat16().float()
    return (hi.double() + (t - hi).bfloat16().double()) if prec else hi.double()


def _pattern(shape, g):
    """Prefill of every output tensor: an element the plan leaves unwritten keeps it and fails the comparison."""
    return _grid(shape, g, -255, 255, 64.0).float() + 1000.0


def _pad(t, p, mode):
    return F.pad(t, (p, p, p, p), mode='reflect' if mode == REFLECT else 'constant')


def _readback_taps(nh, k, s):
    """Output channel j of the readback head reads input channel c_j at tap (dy, dx): the corners (stride 1), every parity plane
    (stride 2); channels spread over the slice, the last one included."""
    taps = [(0, 0), (0, k - 1), (k - 1, 0), (k - 1, k - 1)] if s == 1 else [(0, 0), (1, 1), (0, 1), (1, 0), (k - 1, k - 1)]
    return [taps[j % len(taps)] for j in range(nh)]


def _tiles_per_cta(rec):
    return rec['MG'] * -(-rec['units'] // rec['ctas'])


# ------------------------------------------------------------------------------------------------ the test
def _run_case(name, spec, mode):
    g = torch.Generator().manual_seed(sum(map(ord, name + mode)))
    plan = Plan(0, precision=mode, sample_stats=spec.sample, train=spec.train)
    ctx = build(plan, spec, 'cuda')
    N, H, W, Ho, Wo = spec.N, spec.H, spec.W, ctx['Ho'], ctx['Wo']
    prec = mode == 'precise'
    # exact operands: inputs k / 16, weights j / 16, biases nonzero
    if spec.ident:       # fp32 inputs with a mean per channel; raw = the input as stored (hi + lo)
        x = ((torch.randn(N, spec.Cin, H, W, generator=g) + torch.randn(1, spec.Cin, 1, 1, generator=g) * 3) * 0.7).cuda()
    else:
        x = _grid((N, spec.Cin, H, W), g, 0 if spec.pos else -24, 24)
    with torch.no_grad():
        for c in ctx['convs']:
            if spec.ident:
                c.weight.zero_()
                for j in range(spec.Cout):
                    c.weight[j, j, 0, 0] = 1.0
            else:
                c.weight.copy_(_grid(c.weight.shape, g, 0 if spec.pos else -3, 3).float())
            if c.bias is not None:
                c.bias.copy_(_grid(c.bias.shape, g, -64, 64, 64.0).float())
    w = torch.cat([c.weight.detach().double() for c in ctx['convs']])
    xs = _stored(x, True) if spec.ident else x
    if spec.transposed:
        conv = lambda a, b: F.conv_transpose2d(a, b, stride=spec.stride, padding=spec.pad, output_padding=1)
        raw, mag = conv(xs, w), conv(xs.abs(), w.abs()).max().item()
    else:
        xp = _pad(xs, spec.pad, spec.pmode)
        raw, mag = F.conv2d(xp, w, stride=spec.stride), F.conv2d(xp.abs(), w.abs(), stride=spec.stride).max().item()
    assert mag < 2.0 ** 16, (name, mag)                       # fp32 sums of these products are exact
    io = [None] * plan.n_slots
    io[S_X] = torch.zeros(N, spec.Cin + C_PAD, H, W, device='cuda')
    io[S_X][:, 2:2 + spec.Cin] = x.float()
    flags = None
    if spec.flags:
        flags = torch.tensor([L.IMAGE_ACTIVE if n % 2 == 0 else 0 for n in range(N)], dtype=torch.int32, device='cuda')
        io[S_FLAGS] = flags
    active = [n for n in range(N) if flags is None or n % 2 == 0]
    for u in ctx['units']:
        for s in u['add_slots']:
            io[s] = torch.zeros(N, u['Cn'] + C_PAD, Ho, Wo, device='cuda')
            io[s][:, 1:1 + u['Cn']] = (torch.randn(N, u['Cn'], Ho, Wo, generator=g) * 0.6).cuda()   # off the bf16 grid
        io[u['out_slot']] = _pattern((N, u['Cn'], Ho, Wo), g)
        if 'head' in u:
            k, s_, p, m = spec.readback
            nh = u['head'].out_channels
            chans = torch.linspace(0, u['Cn'] - 1, nh).round().long().tolist()
            taps = _readback_taps(nh, k, s_)
            with torch.no_grad():
                u['head'].weight.zero_()
                for j, (c, (dy, dx)) in enumerate(zip(chans, taps)):
                    u['head'].weight[j, c, dy, dx] = 1.0
            u['rb'] = (chans, taps)
            hh = (Ho + 2 * p - k) // s_ + 1
            hw = (Wo + 2 * p - k) // s_ + 1
            io[u['head_slot']] = _pattern((N, nh, hh, hw), g)
    norms = list(dict.fromkeys(u['norm'] for u in ctx['units'] if u['norm'] is not None))
    for nm in norms:
        u = next(u for u in ctx['units'] if u['norm'] is nm)
        with torch.no_grad():
            nm.weight.copy_(_grid((u['Cn'],), g, 128, 384, 256.0).float() * (torch.randint(0, 2, (u['Cn'],), generator=g) * 2 - 1).cuda())
            nm.bias.copy_(_grid((u['Cn'],), g, -128, 128, 256.0).float())
            nm.running_mean.fill_(7.0)
            nm.running_var.fill_(5.0)
            nm.num_batches_tracked.zero_()
    plan.finalize()                                    # packs the weights, writes the bias-affine shifts
    d = plan.describe()
    (srec,) = [r for r in d['epilogue_forward'] if r['kind'] == 'stats'] or [None]

    def snapshot():
        return [t.clone() for t in io if t is not None] + [b.clone() for nm in norms for b in (nm.running_mean, nm.running_var)]

    plan.run(io, use_graph=False)
    torch.cuda.synchronize()
    first = snapshot()
    _verify(name, mode, spec, ctx, srec, d, io, raw, prec, active, momentum=1.0)
    # the fixed-point statistics are order independent: a second run (graph) leaves every output and buffer bit for bit
    for nm in norms:
        nm.running_mean.fill_(7.0); nm.running_var.fill_(5.0)
    plan.run(io, use_graph=False)
    plan.run(io, use_graph=True)          # captures
    for nm in norms:
        nm.running_mean.fill_(7.0); nm.running_var.fill_(5.0)
    plan.run(io, use_graph=True)
    torch.cuda.synchronize()
    again = snapshot()
    for a, b in zip(first, again):
        assert torch.equal(a, b), '%s %s: a repeated run differs' % (name, mode)
    for nm in norms:        # four runs; per-sample plans count the active images of each
        want = 4 * (len(active) if spec.sample else 1)
        assert nm.num_batches_tracked.item() == want, (name, nm.num_batches_tracked.item(), want)
    # momentum 0.1 on pre-filled buffers: the update expression
    plan2 = Plan(0, precision=mode, sample_stats=spec.sample, train=spec.train)
    build_ctx2 = build(plan2, spec, 'cuda', momentum=0.1)
    for c2, c in zip(build_ctx2['convs'], ctx['convs']):
        with torch.no_grad():
            c2.weight.copy_(c.weight)
            if c.bias is not None:
                c2.bias.copy_(c.bias)
    for u2, u in zip(build_ctx2['units'], ctx['units']):
        if 'head' in u:
            with torch.no_grad():
                u2['head'].weight.copy_(u['head'].weight)
        if u['norm'] is not None:
            with torch.no_grad():
                u2['norm'].weight.copy_(u['norm'].weight); u2['norm'].bias.copy_(u['norm'].bias)
                u2['norm'].running_mean.copy_(_grid((u['Cn'],), g, -512, 512, 64.0).float())
                u2['norm'].running_var.copy_(_grid((u['Cn'],), g, 1, 512, 64.0).float())
    olds = {id(u2['norm']): (u2['norm'].running_mean.clone(), u2['norm'].running_var.clone())
            for u2 in build_ctx2['units'] if u2['norm'] is not None}
    plan2.finalize()
    plan2.run(io, use_graph=False)
    torch.cuda.synchronize()
    _verify_running(name + ' momentum 0.1', spec, build_ctx2, srec, raw, active, olds, 0.1)


def _stats_ref(spec, srec, raw, c_off, cn, n=None):
    """fp64 mean, biased var, count and their derived error bounds for slice [c_off, c_off + cn) (image n, or the batch)."""
    v = raw[:, c_off:c_off + cn] if n is None else raw[n:n + 1, c_off:c_off + cn]
    cnt = v.shape[0] * v.shape[2] * v.shape[3]
    S, Q = v.sum((0, 2, 3)), (v * v).sum((0, 2, 3))
    A, B = v.abs().sum((0, 2, 3)), Q
    u = _tiles_per_cta(srec)
    flushes = srec['units']                 # each flush onto a row publishes at least one unit
    dS = (34 + u) * EPS * A + flushes * 2.0 ** -21
    dQ = (34 + u) * EPS * B + flushes * 2.0 ** -17
    mean = S / cnt
    var = Q / cnt - mean * mean
    dm = dS / cnt
    dvar = dQ / cnt + 2 * mean.abs() * dm + 2.0 ** -50 * (Q / cnt)
    return mean, var.clamp_min(0), cnt, dm, dvar


def _affine_ref(nm, mean, var, dm, dvar):
    gam, bet = nm.weight.detach().double(), nm.bias.detach().double()
    rstd = (var + nm.eps).rsqrt()
    scale = gam * rstd
    rel = 0.5 * dvar / (var + nm.eps) + 4 * EPS
    shift = bet - mean * scale
    dshift = scale.abs() * dm + (mean * scale).abs() * rel + EPS * ((mean * scale).abs() + shift.abs())
    return scale, shift, rel, dshift


def _verify(name, mode, spec, ctx, srec, d, io, raw, prec, active, momentum):
    tag = '%s [%s]' % (name, mode)
    rin = raw if prec else _bf16(raw)                  # what the normalise pass reads
    v4 = lambda t: t.view(1, -1, 1, 1)
    for u in ctx['units']:
        c_off, cn = u['c_off'], u['Cn']
        r = rin[:, c_off:c_off + cn]
        if u['norm'] is not None:
            per_image = spec.sample or spec.norm == 'instance'
            outs, bounds = [], []
            for n in range(spec.N) if per_image else [None]:
                mean, var, cnt, dm, dvar = _stats_ref(spec, srec, raw, c_off, cn, n)
                scale, shift, rel, dshift = _affine_ref(u['norm'], mean, var, dm, dvar)
                rr = r if n is None else r[n:n + 1]
                z = rr * v4(scale) + v4(shift)
                dz = rr.abs() * v4(scale.abs() * rel) + v4(dshift) + EPS * z.abs()
                outs.append(z); bounds.append(dz)
            z, dz = torch.cat(outs), torch.cat(bounds)
        elif spec.norm == 'bias':
            b = ctx['convs'][0].bias.detach().double()
            z = r + v4(b)
            dz = EPS * z.abs()
        else:
            z, dz = r.clone(), torch.zeros_like(r)
        if spec.act == RELU:
            z = z.clamp_min(0)
        elif spec.act == LRELU:
            neg = z < 0
            z = torch.where(neg, z * SLOPE32, z)
            dz = dz + EPS * z.abs()
        adds = [_stored(io[s][:, 1:1 + cn], prec) for s in u['add_slots']]
        out = z + sum(adds) if adds else z
        n_sum = len(adds) * (2 if prec else 1)
        dz = dz + n_sum * EPS * (z.abs() + sum(a.abs() for a in adds)) if adds else dz
        fb = dz * (1 + 2.0 ** -7) + (2.0 ** -16 + EPS if prec else 2.0 ** -8) * out.abs() + 1e-30
        _check('%s slice %d:%d out @%d' % (tag, c_off, c_off + cn, u['out_slot']), io[u['out_slot']], out, fb)
        if 'head' in u:
            # the padded layout, read back through the head: exactly the exported interior at the mapped position
            k, s_, p, m = spec.readback
            got = io[u['head_slot']]
            ref = _pad(io[u['out_slot']].double(), p, m)
            chans, taps = u['rb']
            hh, hw = got.shape[2], got.shape[3]
            want = torch.stack([ref[:, c, dy:dy + s_ * (hh - 1) + 1:s_, dx:dx + s_ * (hw - 1) + 1:s_]
                                for c, (dy, dx) in zip(chans, taps)], 1)
            assert torch.equal(got.double(), want), '%s: the %s halo layout (pad %d, stride %d) differs from the interior' % (
                tag, 'reflect' if m == REFLECT else 'zero', p, s_)
            print('%-72s halo layout bit-exact' % (tag + ' readback'))
    _verify_running(tag, spec, ctx, srec, raw, active, None, momentum)


def _verify_running(tag, spec, ctx, srec, raw, active, olds, momentum):
    m32 = float(torch.tensor(momentum, dtype=torch.float32))
    seen = set()
    for i, u in enumerate(ctx['units']):
        nm = u['norm']
        if nm is None or id(nm) in seen:
            continue
        seen.add(id(nm))
        c_off, cn = u['c_off'], u['Cn']
        bias = ctx['convs'][0 if c_off == 0 else 1].bias.detach().double()
        if olds is None:
            rm, rv = torch.full((cn,), 7.0, device='cuda').double(), torch.full((cn,), 5.0, device='cuda').double()
        else:
            rm, rv = (t.double() for t in olds[id(nm)])
        drm, drv = torch.zeros_like(rm), torch.zeros_like(rv)
        steps = [[n] for n in active] if spec.sample else [None]
        for st in steps:
            n = None if st is None else st[0]
            mean, var, cnt, dm, dvar = _stats_ref(spec, srec, raw, c_off, cn, n)
            if spec.norm == 'instance' and n is None:
                per = [_stats_ref(spec, srec, raw, c_off, cn, k) for k in range(spec.N)]
                mean = sum(p_[0] for p_ in per) / spec.N; dm = sum(p_[3] for p_ in per) / spec.N
                vu = sum(p_[1] * p_[2] / (p_[2] - 1) for p_ in per) / spec.N
                dvu = sum(p_[4] * p_[2] / (p_[2] - 1) for p_ in per) / spec.N
            else:
                vu, dvu = var * cnt / (cnt - 1), dvar * cnt / (cnt - 1)
            xm = mean + bias
            new_m = (1 - m32) * rm + m32 * xm
            new_v = (1 - m32) * rv + m32 * vu
            drm = (1 - m32) * drm + m32 * (dm + EPS * (mean.abs() + xm.abs())) + 2 * EPS * ((1 - m32) * rm.abs() + m32 * xm.abs() + new_m.abs())
            drv = (1 - m32) * drv + m32 * (dvu + EPS * vu) + 2 * EPS * ((1 - m32) * rv.abs() + m32 * vu + new_v.abs())
            rm, rv = new_m, new_v
        _check('%s running_mean %d:%d' % (tag, c_off, c_off + cn), nm.running_mean, rm, drm + 1e-30)
        _check('%s running_var %d:%d' % (tag, c_off, c_off + cn), nm.running_var, rv, drv + 1e-30)


@pytest.mark.parametrize('name,spec', CASES + EDGE_CASES, ids=[c[0] for c in CASES + EDGE_CASES])
def test_epilogue_forward(name, spec):
    for mode in spec.modes:
        _run_case(name, spec, mode)
