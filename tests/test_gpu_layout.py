"""The layout kernels bit for bit: every one of them copies, rounds to bf16 (RNE) or adds exact values, so each is held to
torch.equal against a CPU reference of the same operation, never to a tolerance.

  * import_nchw_kernel<16|64> (csrc/layout.cu): the plan is finalized into a caller-owned workspace and every activation
    buffer is decoded from the byte offsets v2v_plan_describe reports ("buffers").  At every padded position (halo, parity-plane
    slack and padded channels included) the buffer must hold hi = bf16(x) and lo = bf16(x - hi) of the reflect- or zero-padded
    caller window, and lo == 0 where the input is declared exact (skip_lo).  The inputs mix bf16 ties, +-0, subnormal-free
    small and large magnitudes.  The correlation's import must equal the split of LeakyReLU of the fp32 scratch it reads.
  * export_nchw_kernel: each input is also exported straight from its (halo-padded, possibly parity-split) buffer: the output
    must equal hi.float() + lo.float().
  * act_copy_kernel: a concat's output buffer must equal the padded concatenation of its sources' buffers, hi and lo alike.
  * pack_weights_kernel / pack_weights_tiled_kernel: the packed matrix at the conv's w_off must equal a numpy packing of the
    torch weights, before and after an in-place weight update and repack().
  * grad_import / grad_export / grad_layout_tiled_kernel: in a training plan input -> export, d(input) is d(output) added onto
    the caller's prefilled gradient tensor, inside the channel window only.
  * fold_add_kernel, the dgrad packing and unstage_wgrad_kernel (csrc/wgrad_umma.cu): single norm-less, bias-less conv units on
    small integers (inputs in [-4, 4], weights in [-2, 2], dY in [-3, 3]): every product and sum is an integer far below 2^24,
    so the forward output, dX and dW are exactly torch's fp64 autograd result.  A second backward must double them exactly
    (the += of fold, export and unstage).  Fast plans run the same units through the fp32 SIMT backward.

Each case is named once in CASES; tests/test_layout_census.py checks that the cases reach every layout launch path the product
plans take."""
import collections

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from vid2vid_b200 import _lib as L
from vid2vid_b200.plan import Plan, conv_desc, norm_desc

pytestmark = pytest.mark.gpu

CORR_SLOPE = 0.1
REFLECT, ZERO = L.PAD_REFLECT, L.PAD_ZERO

# One caller input: channels [c_off, c_off + C) of a C_src-channel tensor, read by a conv (k, stride, pad, pad mode) that sets
# its buffer's halo, or by nothing (no halo); exact: the caller declares the values bf16-exact (skip_lo).
In = collections.namedtuple('In', 'N C_src c_off C H W exact conv', defaults=(None,))
Imports = collections.namedtuple('Imports', 'prec inputs')
Corr = collections.namedtuple('Corr', 'prec N C H W')
# A concat of inputs with `chans` channels, read by each conv of `convs` (k, stride, pad, pad mode).
Cat = collections.namedtuple('Cat', 'prec N H W chans convs')
# Convs whose packed weights are compared: (kind, Cin, Cout, k, stride, pad, Cout2); kind 'conv', 'deconv' or 'head'.
Pack = collections.namedtuple('Pack', 'prec H W convs')
# Training plan: caller inputs (N, C_src, c_off, C, H, W), each exported straight back.
Grad = collections.namedtuple('Grad', 'pairs')
# Integer-valued conv unit: ReflectionPad2d / zero padding `pad` then conv (or transposed conv) Cin -> Cout (+ Cout2 fused).
Int = collections.namedtuple('Int', 'prec N Cin Cout H W k stride pad mode transposed Cout2', defaults=(False, 0))

CASES = [
    # CT 16 and 64 imports in both modes: no halo (export only), zero halo, parity planes, reflect halo, channel windows
    # (face's 16 of 31 at 15, FlowNet's 3 of 6 at 3), Wpad above 128 and ragged, N = 2, exact (skip_lo) inputs
    ('imports_fast', Imports('fast', [In(1, 16, 0, 16, 20, 40, False), In(1, 31, 15, 16, 12, 200, False),
                                      In(2, 6, 0, 6, 14, 150, False, (7, 1, 3, REFLECT)),
                                      In(1, 128, 0, 128, 6, 100, False), In(1, 128, 0, 128, 5, 300, False),
                                      In(1, 108, 0, 108, 9, 150, False, (7, 1, 3, REFLECT)),
                                      In(1, 108, 0, 108, 9, 150, True, (7, 1, 3, REFLECT))])),
    ('imports_precise', Imports('precise', [In(1, 16, 0, 16, 20, 40, False), In(2, 6, 0, 6, 7, 300, False),
                                            In(1, 6, 3, 3, 10, 200, False), In(1, 6, 0, 6, 10, 200, False, (3, 1, 1, ZERO)),
                                            In(1, 13, 0, 13, 10, 201, False, (4, 2, 2, ZERO)),
                                            In(1, 6, 3, 3, 11, 203, False, (7, 2, 3, ZERO)),
                                            In(2, 6, 0, 6, 9, 150, False, (7, 1, 3, REFLECT)),
                                            In(1, 128, 0, 128, 6, 100, False), In(1, 128, 0, 128, 5, 300, False),
                                            In(1, 24, 0, 24, 6, 129, False), In(1, 72, 0, 72, 5, 64, False),
                                            In(1, 64, 0, 64, 5, 130, False, (3, 1, 1, REFLECT)),
                                            In(1, 39, 0, 39, 9, 261, False, (4, 2, 2, ZERO)),
                                            In(1, 108, 0, 108, 9, 150, False, (7, 1, 3, REFLECT))])),
    ('stem108_exact_256x512', Imports('precise', [In(1, 108, 0, 108, 256, 512, True, (7, 1, 3, REFLECT))])),
    ('corr_lrelu', Corr('precise', 1, 32, 12, 40)),
    # concat: zero and reflect output halos, parity planes, odd channel offsets (FlowNet fusion's 6 + 3 + 2 + 1 + 1), Global_with_z's
    # [down, z]
    ('concat_fast', Cat('fast', 1, 10, 140, [16, 8], [(3, 1, 1, ZERO), (7, 1, 3, REFLECT)])),
    ('concat_precise', Cat('precise', 1, 10, 140, [6, 3, 2, 1, 1], [(3, 1, 1, ZERO), (3, 2, 1, ZERO)])),
    ('concat_z_precise', Cat('precise', 1, 8, 16, [512, 8], [(3, 1, 1, REFLECT)])),
    # packing: 1x1, 3x3, 5x5, 4x4 stride 2, 7x7 (TC 32 / 8 / 16 / 4), fused Cout2, transposed, kx-GEMM 7x7 heads (single and fused)
    ('pack_fast', Pack('fast', 16, 40, [('conv', 64, 96, 1, 1, 0, 0), ('conv', 64, 96, 3, 1, 1, 0), ('conv', 6, 64, 7, 1, 3, 0),
                                        ('conv', 24, 48, 7, 1, 3, 16), ('deconv', 64, 32, 3, 2, 1, 0), ('head', 32, 3, 7, 1, 3, 0),
                                        ('head', 32, 3, 7, 1, 3, 1)])),
    ('pack_precise', Pack('precise', 16, 40, [('conv', 64, 96, 1, 1, 0, 0), ('conv', 64, 96, 3, 1, 1, 0), ('conv', 40, 72, 5, 1, 2, 0),
                                              ('conv', 39, 64, 4, 2, 2, 0), ('conv', 6, 64, 7, 1, 3, 0), ('conv', 24, 48, 7, 1, 3, 16),
                                              ('deconv', 64, 32, 3, 2, 1, 0), ('head', 32, 3, 7, 1, 3, 0), ('head', 32, 3, 7, 1, 3, 1)])),
    # gradient layout: scalar (C = 3) and tiled paths, ragged channel tiles (16, 40), HW % 32 != 0, channel windows
    ('grad_layout', Grad([(1, 3, 0, 3, 32, 48), (2, 5, 1, 3, 37, 45), (1, 64, 0, 64, 32, 64), (2, 20, 3, 16, 37, 45),
                          (1, 40, 0, 40, 24, 40), (1, 64, 0, 64, 20, 30)])),
    # integer-valued conv units: fold (modes 1 / 2 / 3, reflect, crop, overlapping mirrors), dgrad packing (TC 4 / 16 / 32, w2),
    # unstage (swap, dw2 rows)
    ('int_c7_reflect', Int('precise', 1, 16, 64, 20, 24, 7, 1, 3, REFLECT)),
    ('int_c3_reflect_overlap', Int('precise', 1, 64, 64, 3, 24, 3, 1, 1, REFLECT)),       # H = 3: both row mirrors hit row 1
    ('int_c3_zero_swap', Int('precise', 2, 64, 16, 12, 40, 3, 1, 1, ZERO)),
    ('int_c4_s1', Int('precise', 1, 64, 64, 12, 24, 4, 1, 2, ZERO)),
    ('int_c3_s2', Int('precise', 1, 64, 64, 20, 40, 3, 2, 1, ZERO)),
    ('int_c4_s2_crop', Int('precise', 1, 64, 64, 20, 40, 4, 2, 2, ZERO)),
    ('int_deconv', Int('precise', 1, 64, 32, 10, 20, 3, 2, 1, ZERO, True)),
    ('int_c7_fused', Int('precise', 1, 16, 48, 20, 24, 7, 1, 3, REFLECT, False, 16)),
    ('int_c7_fused_swap', Int('precise', 1, 64, 16, 20, 24, 7, 1, 3, REFLECT, False, 16)),
    # a stride-2 conv behind ReflectionPad2d: its data gradient must mirror the halo rows and columns back
    ('int_s2_reflect', Int('precise', 1, 64, 64, 20, 40, 3, 2, 1, REFLECT)),
    # the same integers through the fp32 SIMT backward of fast plans
    ('int_fast_c7_reflect', Int('fast', 1, 16, 64, 20, 24, 7, 1, 3, REFLECT)),
    ('int_fast_s2_reflect', Int('fast', 1, 64, 64, 20, 40, 3, 2, 1, REFLECT)),
    ('int_fast_c4_s2', Int('fast', 1, 64, 64, 20, 40, 4, 2, 2, ZERO)),
    ('int_fast_deconv', Int('fast', 1, 64, 32, 10, 20, 3, 2, 1, ZERO, True)),
]


def precision(spec):
    return spec.prec if hasattr(spec, 'prec') else 'precise'


def is_train(spec):
    return isinstance(spec, (Grad, Int))


# ------------------------------------------------------------------------------------------------ plan builders
def _gen(seed=0):
    return torch.Generator().manual_seed(seed)


def _conv_mod(Cin, Cout, k, stride, pad, device, transposed=False):
    if transposed:
        return nn.ConvTranspose2d(Cin, Cout, k, stride, pad, output_padding=1, bias=False).to(device)
    return nn.Conv2d(Cin, Cout, k, stride, pad, bias=False).to(device)


def _consume(plan, v, C, conv, device, ctx, slot):
    """conv (k, stride, pad, mode) of value v, normalise-less pass, export into `slot`."""
    k, stride, pad, mode = conv
    m = _conv_mod(C, 16, k, stride, pad, device)
    ctx.setdefault('mods', []).append(m)
    raw = plan.conv(v, conv_desc(m, pad_mode=mode, pad=pad))
    plan.export(plan.norm_act(raw, norm_desc(None)), slot)


def build(plan, spec, device):
    """Describe the case on `plan` with its modules on `device` -> context for the test."""
    ctx = {'values': [], 'slots': []}
    if isinstance(spec, Imports):
        slot = 0
        for inp in spec.inputs:
            v = plan.input(slot, inp.N, inp.C_src, inp.c_off, inp.C, inp.H, inp.W, exact_bf16=inp.exact)
            plan.export(v, slot + 1)
            ctx['values'].append(v)
            ctx['slots'].append((slot, slot + 1))
            if inp.conv:
                _consume(plan, v, inp.C, inp.conv, device, ctx, slot + 2)
            slot += 3
    elif isinstance(spec, Corr):
        va = plan.input(0, spec.N, spec.C, 0, spec.C, spec.H, spec.W)
        vb = plan.input(1, spec.N, spec.C, 0, spec.C, spec.H, spec.W)
        vc = plan.correlation(va, vb, 20, 1, 20, 1, 2, L.ACT_LRELU, CORR_SLOPE)
        plan.export(vc, 2)
        ctx['values'] = [vc]
    elif isinstance(spec, Cat):
        vs = [plan.input(i, spec.N, c, 0, c, spec.H, spec.W) for i, c in enumerate(spec.chans)]
        vc = plan.concat(vs)
        n = len(vs)
        plan.export(vc, n)
        for j, conv in enumerate(spec.convs):
            _consume(plan, vc, sum(spec.chans), conv, device, ctx, n + 1 + j)
        ctx['values'] = vs + [vc]
    elif isinstance(spec, Pack):
        slot = 1
        ctx['convs'] = []
        for kind, Cin, Cout, k, stride, pad, Cout2 in spec.convs:
            v = plan.input(0, 1, 64, 0, Cin, spec.H, spec.W)
            if kind == 'deconv':
                m = _conv_mod(Cin, Cout, k, stride, pad, device, transposed=True)
                m2 = None
            else:
                m = nn.Conv2d(Cin, Cout, k, stride, pad, bias=kind == 'head').to(device)
                m2 = nn.Conv2d(Cin, Cout2, k, stride, pad, bias=kind == 'head').to(device) if Cout2 else None
            d = conv_desc(m, m2=m2)
            if kind == 'head':
                chans = [(slot, j, Cout + Cout2, L.ACT_NONE, 1.0) for j in range(Cout + Cout2)]
                plan.head(v, d, chans)
                slot += 1
            else:
                raw = plan.conv(v, d)
                plan.export(plan.norm_act(raw, norm_desc(None)), slot)
                slot += 1
            ctx['convs'].append((kind, m, m2))
    elif isinstance(spec, Grad):
        for i, (N, C_src, c_off, C, H, W) in enumerate(spec.pairs):
            v = plan.input(2 * i, N, C_src, c_off, C, H, W)
            plan.export(v, 2 * i + 1)
    else:
        mode_pad = spec.pad
        m = _conv_mod(spec.Cin, spec.Cout, spec.k, spec.stride, spec.pad, device, spec.transposed)
        m2 = _conv_mod(spec.Cin, spec.Cout2, spec.k, spec.stride, spec.pad, device) if spec.Cout2 else None
        v = plan.input(0, spec.N, spec.Cin + 2, 1, spec.Cin, spec.H, spec.W, exact_bf16=True)
        raw = plan.conv(v, conv_desc(m, pad_mode=spec.mode, pad=mode_pad, m2=m2))
        plan.export(plan.norm_act(raw, norm_desc(None)), 1)
        ctx.update(m=m, m2=m2)
    return ctx


def _make(spec):
    plan = Plan(0, precision=precision(spec), train=is_train(spec))
    ctx = build(plan, spec, 'cuda')
    ws = torch.zeros(plan.workspace_bytes + 1024, dtype=torch.uint8, device='cuda')
    plan.finalize(workspace=ws)
    ctx['ws0'] = (ws.data_ptr() + 1023) // 1024 * 1024 - ws.data_ptr()
    ctx['ws'] = ws
    return plan, ctx


# ------------------------------------------------------------------------------------------------ decoding and references
def _bytes(ctx, off, n):
    b = ctx['ws0'] + off
    return ctx['ws'][b:b + n]


def decode(ctx, rec):
    """Activation buffer -> (hi, lo) float tensors [N, C, Hp_total, Wp_total] over the padded extent of its planes (parity
    planes interleaved back: 2 Hp x 2 Wp, the slack row / column past the padding included)."""
    sp = 2 if rec['split'] else 1
    n = rec['N'] * rec['P'] * rec['Hp'] * rec['Wp'] * rec['C'] * sp
    t = _bytes(ctx, rec['off'], 2 * n).view(torch.bfloat16).float().cpu()
    t = t.view(rec['N'], rec['P'], rec['Hp'], rec['Wp'], sp, rec['C'])
    if rec['parity']:
        full = torch.zeros(rec['N'], 2 * rec['Hp'], 2 * rec['Wp'], sp, rec['C'])
        for pl in range(4):
            full[:, pl >> 1::2, pl & 1::2] = t[:, pl]
        t = full
    else:
        t = t[:, 0]
    t = t.permute(0, 3, 4, 1, 2)           # N, sp, C, H, W
    return t[:, 0], (t[:, 1] if sp == 2 else torch.zeros_like(t[:, 0]))


def split(x):
    hi = x.bfloat16()
    return hi.float(), (x - hi.float()).bfloat16().float()


def padded(x, rec):
    """The caller window x [N, Cvalid, H, W] as the buffer holds it: halo per the buffer's mode, channels padded to C, the
    plane slack zero -> [N, C, Htot, Wtot]."""
    pt, pl, pb, pr = rec['pads']
    if rec['mode'] == REFLECT:
        y = F.pad(x, (pl, pr, pt, pb), mode='reflect')
    else:
        y = F.pad(x, (pl, pr, pt, pb))
    Ht = 2 * rec['Hp'] if rec['parity'] else rec['Hp']
    Wt = 2 * rec['Wp'] if rec['parity'] else rec['Wp']
    return F.pad(y, (0, Wt - y.shape[3], 0, Ht - y.shape[2], 0, rec['C'] - y.shape[1]))


def buffers_of(d, value):
    return [b for b in d['buffers'] if b['value'] == value]


def _assert_equal(what, got, ref):
    if not torch.equal(got, ref):
        bad = (got != ref).nonzero()
        raise AssertionError('%s: %d of %d elements differ, first at %s: got %r, expected %r' % (
            what, bad.shape[0], got.numel(), tuple(bad[0].tolist()), got[tuple(bad[0])].item(), ref[tuple(bad[0])].item()))


def awkward(shape, g):
    """fp32 values that probe the hi / lo split: exact bf16 ties (RNE to even), +-0, ordinary values over many binades and
    magnitudes up to 1e30."""
    n = int(np.prod(shape))
    base = torch.randn(n, generator=g) * torch.pow(10.0, torch.randint(-6, 7, (n,), generator=g).float())
    hi = base.bfloat16().float()
    ulp = torch.pow(2.0, torch.floor(torch.log2(hi.abs().clamp_min(1e-30))) - 7)
    tie = hi + 0.5 * ulp
    kind = torch.randint(0, 6, (n,), generator=g)
    x = torch.where(kind == 0, tie, base)
    x = torch.where(kind == 1, torch.where(torch.rand(n, generator=g) < 0.5, 0.0, -0.0), x)
    x = torch.where(kind == 2, torch.randn(n, generator=g) * 1e30, x)
    x = torch.where(kind == 3, hi, x)
    return x.view(shape)


# ------------------------------------------------------------------------------------------------ tests
def _cases(kind):
    return [pytest.param(spec, id=name) for name, spec in CASES if isinstance(spec, kind)]


@pytest.mark.parametrize('spec', _cases(Imports))
def test_import_export(spec):
    plan, ctx = _make(spec)
    g = _gen(1)
    io = [None] * plan.n_slots
    xs = []
    for inp, (s_in, s_out) in zip(spec.inputs, ctx['slots']):
        x = awkward((inp.N, inp.C_src, inp.H, inp.W), g)
        if inp.exact:
            x = x.bfloat16().float()
        io[s_in] = x.cuda()
        io[s_out] = torch.full((inp.N, inp.C, inp.H, inp.W), float('nan'), device='cuda')
        if inp.conv:
            k, s, p, _ = inp.conv
            io[s_in + 2] = torch.empty(inp.N, 16, (inp.H + 2 * p - k) // s + 1, (inp.W + 2 * p - k) // s + 1, device='cuda')
        xs.append(x)
    d = plan.describe()
    plan.run(io, use_graph=False)
    torch.cuda.synchronize()
    imports = {r['buf']: r for r in d['layout'] if r['kind'] == 'import'}
    for i, (inp, v, x) in enumerate(zip(spec.inputs, ctx['values'], xs)):
        win = x[:, inp.c_off:inp.c_off + inp.C]
        recs = buffers_of(d, v)
        for rec in recs:
            imp = imports[rec['buf']]
            tag = 'input %d (CT %d, mode %d, parity %d, skip_lo %d)' % (i, imp['CT'], rec['mode'], rec['parity'], imp['skip_lo'])
            hi, lo = decode(ctx, rec)
            rhi, rlo = split(padded(win, rec))
            if not rec['split']:
                rlo = torch.zeros_like(rlo)
            if imp['skip_lo']:
                assert torch.equal(lo, torch.zeros_like(lo)), tag + ': lo half written for an exact input'
            _assert_equal(tag + ' hi', hi, rhi)
            _assert_equal(tag + ' lo', lo, rlo)
        # export of the first buffer: hi + lo of the interior
        rhi, rlo = split(win)
        ref = rhi + (rlo if recs[0]['split'] else 0.0)
        _assert_equal('input %d export' % i, io[ctx['slots'][i][1]].cpu(), ref)


@pytest.mark.parametrize('spec', _cases(Corr))
def test_correlation_import(spec):
    plan, ctx = _make(spec)
    g = _gen(2)
    io = [torch.randn(spec.N, spec.C, spec.H, spec.W, generator=g).cuda() for _ in range(2)]
    d = plan.describe()
    sc = d['scratch'][0]
    io.append(torch.full((spec.N, sc['C_out'], sc['H_out'], sc['W_out']), float('nan'), device='cuda'))
    plan.run(io, use_graph=False)
    torch.cuda.synchronize()
    n_in = sc['N'] * sc['C'] * sc['H'] * sc['W']
    n_out = sc['N'] * sc['C_out'] * sc['H_out'] * sc['W_out']
    out = _bytes(ctx, sc['off'] + 8 * n_in, 4 * n_out).view(torch.float32).cpu().view(sc['N'], sc['C_out'], sc['H_out'], sc['W_out'])
    assert torch.isfinite(out).all() and out.abs().max() > 0
    slope = torch.tensor(CORR_SLOPE, dtype=torch.float32)
    act = torch.where(out > 0, out, out * slope)
    (rec,) = buffers_of(d, ctx['values'][0])
    imp = next(r for r in d['layout'] if r['kind'] == 'import' and r['buf'] == rec['buf'])
    assert imp['act'] == L.ACT_LRELU and imp['direct'] == 1
    hi, lo = decode(ctx, rec)
    rhi, rlo = split(padded(act, rec))
    _assert_equal('correlation import hi', hi, rhi)
    _assert_equal('correlation import lo', lo, rlo)
    _assert_equal('correlation export', io[2].cpu(), split(act)[0] + split(act)[1])


@pytest.mark.parametrize('spec', _cases(Cat))
def test_concat(spec):
    plan, ctx = _make(spec)
    g = _gen(3)
    n = len(spec.chans)
    io = [awkward((spec.N, c, spec.H, spec.W), g).cuda() for c in spec.chans]
    io.append(torch.empty(spec.N, sum(spec.chans), spec.H, spec.W, device='cuda'))
    for k, s, p, _ in spec.convs:
        io.append(torch.empty(spec.N, 16, (spec.H + 2 * p - k) // s + 1, (spec.W + 2 * p - k) // s + 1, device='cuda'))
    d = plan.describe()
    plan.run(io, use_graph=False)
    torch.cuda.synchronize()
    srcs = []
    for i, v in enumerate(ctx['values'][:n]):
        (rec,) = buffers_of(d, v)
        hi, lo = decode(ctx, rec)
        srcs.append((hi[:, :spec.chans[i], :spec.H, :spec.W], lo[:, :spec.chans[i], :spec.H, :spec.W]))
    cat_hi = torch.cat([h for h, _ in srcs], 1)
    cat_lo = torch.cat([l_ for _, l_ in srcs], 1)
    recs = buffers_of(d, ctx['values'][n])
    assert len(recs) == len({(c[1] > 1, c[3]) for c in spec.convs})
    for rec in recs:
        tag = 'concat buffer (mode %d, parity %d)' % (rec['mode'], rec['parity'])
        hi, lo = decode(ctx, rec)
        _assert_equal(tag + ' hi', hi, padded(cat_hi, rec))
        _assert_equal(tag + ' lo', lo, padded(cat_lo, rec))
    ref = cat_hi + cat_lo
    _assert_equal('concat export', io[n].cpu(), ref)


def pack_reference(kind, m, m2, rec):
    """numpy packing of torch weights: row co (kx * Cout + co for kx-GEMM heads), column t * Cp + c over the filter taps t =
    ky * kw + kx (the filter rows ky for kx-GEMM heads); transposed weights [Cin][Cout] read as [c][co]; the fused second set
    from row Cout1 on; channels past Cin zero; precise plans append the lo half to each row."""
    w = m.weight.detach().float().cpu().numpy()
    if kind == 'deconv':
        w = w.transpose(1, 0, 2, 3)
    if m2 is not None:
        w = np.concatenate([w, m2.weight.detach().float().cpu().numpy()], 0)
    Cout, Cin, kh, kw = w.shape
    Cp = rec['Cp']
    wp = np.zeros((Cout, Cp, kh, kw), np.float32)
    wp[:, :Cin] = w
    if rec['headkx']:
        mat = wp.transpose(3, 0, 2, 1).reshape(kw * Cout, kh * Cp)         # [kx][co] x [ky][c]
    else:
        mat = wp.transpose(0, 2, 3, 1).reshape(Cout, kh * kw * Cp)         # [co] x [ky][kx][c]
    t = torch.from_numpy(np.ascontiguousarray(mat))
    hi, lo = split(t)
    return torch.cat([hi, lo], 1) if rec['split'] else hi


@pytest.mark.parametrize('spec', _cases(Pack))
def test_pack_weights(spec):
    plan, ctx = _make(spec)
    d = plan.describe()
    packs = [r for r in d['layout'] if r['kind'] == 'pack']
    assert len(packs) == len(ctx['convs'])
    g = _gen(4)
    for rnd in range(2):
        if rnd:                                     # an in-place optimiser step, then repack()
            with torch.no_grad():
                for _, m, m2 in ctx['convs']:
                    for mm in (m, m2):
                        if mm is not None:
                            mm.weight.add_(awkward(tuple(mm.weight.shape), g).clamp(-1e3, 1e3).cuda())
            plan.repack()
            torch.cuda.synchronize()
        for (kind, m, m2), rec in zip(ctx['convs'], packs):
            sp = 2 if rec['split'] else 1
            got = _bytes(ctx, rec['w_off'], 2 * rec['rows'] * sp * rec['Ktotal']).view(torch.bfloat16).float().cpu()
            got = got.view(rec['rows'], sp * rec['Ktotal'])
            tag = '%s %d->%d %dx%d (TC %d, headkx %d, w2 %d)%s' % (kind, rec['Cin'], rec['Cout'], rec['k'][0], rec['k'][1],
                                                                rec['TC'], rec['headkx'], rec['w2'], ' after repack' if rnd else '')
            _assert_equal(tag, got, pack_reference(kind, m, m2, rec))


@pytest.mark.parametrize('spec', _cases(Grad))
def test_gradient_layout(spec):
    """d(input) = d(output) exactly, added onto the caller's prefilled gradient inside the window only."""
    plan, ctx = _make(spec)
    g = _gen(5)
    io, gio, pats = [], [], []
    for N, C_src, c_off, C, H, W in spec.pairs:
        io += [torch.randn(N, C_src, H, W, generator=g).cuda(), torch.empty(N, C, H, W, device='cuda')]
        pat = torch.randn(N, C_src, H, W, generator=g)
        pats.append(pat)
        gio += [pat.clone().cuda(), torch.randn(N, C, H, W, generator=g).cuda()]
    d = plan.describe()
    kinds = collections.Counter((r['kind'], r['tiled']) for r in d['layout'] if r['kind'].startswith('grad_'))
    assert kinds[('grad_export', 0)] and kinds[('grad_export', 1)], kinds
    plan.run(io, use_graph=False)
    plan.backward(io, gio, [], [])
    torch.cuda.synchronize()
    for i, ((N, C_src, c_off, C, H, W), pat) in enumerate(zip(spec.pairs, pats)):
        ref = pat.clone()
        ref[:, c_off:c_off + C] += gio[2 * i + 1].cpu()
        _assert_equal('pair %d (C %d of %d at %d, %dx%d)' % (i, C, C_src, c_off, H, W), gio[2 * i].cpu(), ref)


def _int(shape, lim, g):
    return torch.randint(-lim, lim + 1, shape, generator=g).float()


@pytest.mark.parametrize('spec', _cases(Int))
def test_integer_conv_backward(spec):
    """Forward, dX and dW of one conv unit on small integers equal torch's fp64 results exactly, and a second backward
    doubles dX (added onto the caller's prefilled tensor) and dW exactly."""
    plan, ctx = _make(spec)
    g = _gen(6)
    m, m2 = ctx['m'], ctx['m2']
    with torch.no_grad():
        for mm in (m, m2):
            if mm is not None:
                mm.weight.copy_(_int(tuple(mm.weight.shape), 2, g))
    plan.repack()
    N, Cin, H, W = spec.N, spec.Cin, spec.H, spec.W
    x = _int((N, Cin, H, W), 4, g)
    x_io = torch.zeros(N, Cin + 2, H, W)
    x_io[:, 1:1 + Cin] = x
    # fp64 reference: ReflectionPad2d + unpadded conv, or the conv's own zero padding
    xd = x.double().requires_grad_(True)
    ws = [mm.weight.detach().cpu().double().requires_grad_(True) for mm in (m, m2) if mm is not None]
    if spec.transposed:
        ref = F.conv_transpose2d(xd, ws[0], stride=spec.stride, padding=spec.pad, output_padding=1)
    else:
        wcat = torch.cat(ws, 0)
        if spec.mode == REFLECT:
            ref = F.conv2d(F.pad(xd, (spec.pad,) * 4, mode='reflect'), wcat, stride=spec.stride)
        else:
            ref = F.conv2d(xd, wcat, stride=spec.stride, padding=spec.pad)
    dy = _int(tuple(ref.shape), 3, g)
    ref.backward(dy.double())
    ref_dx, ref_dw = xd.grad.float(), [w.grad.float() for w in ws]
    ref_out = ref.detach().float()
    if spec.prec == 'fast':
        ref_out = ref_out.bfloat16().float()            # the fast plan's bf16 raw and output: one RNE of the exact sum

    pat = _int((N, Cin + 2, H, W), 5, g)
    io = [x_io.cuda(), torch.empty(tuple(ref.shape), device='cuda')]
    gio = [pat.clone().cuda(), dy.cuda()]
    params = [mm.weight for mm in (m, m2) if mm is not None]
    grads = [torch.zeros_like(p_) for p_ in params]
    d = plan.describe()
    (unit,) = d['backward']
    print('%s: data-gradient mode %d%s' % (spec, unit['mode'], (' (SIMT: %s)' % unit['simt']) if unit['simt'] else ''))
    if spec.prec == 'precise' and not (spec.stride == 2 and spec.mode == REFLECT):
        assert unit['mode'] > 0 and unit['wgrad'] is not None, unit
    plan.run(io, use_graph=False)
    _assert_equal('forward', io[1].cpu(), ref_out)
    for rnd in (1, 2):
        plan.backward(io, gio, params, grads)
        torch.cuda.synchronize()
        got = gio[0].cpu()
        _assert_equal('dX outside the window (backward %d)' % rnd, got[:, [0, Cin + 1]], pat[:, [0, Cin + 1]])
        _assert_equal('dX (backward %d)' % rnd, got[:, 1:1 + Cin] - pat[:, 1:1 + Cin], rnd * ref_dx)
        for j, (gw, rw) in enumerate(zip(grads, ref_dw)):
            _assert_equal('dW%s (backward %d)' % ('2' if j else '', rnd), gw.cpu(), rnd * rw)
