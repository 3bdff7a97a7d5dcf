"""GPU parity of the hand-written backward kernels (SURVEY 8 row T): gradients through the C-ABI plan backward
(v2v_plan_backward behind torch.autograd.Function) against PyTorch autograd of the same layers evaluated in fp64, unit by
unit, then the whole CompositeGenerator / MultiscaleDiscriminator against the oracle's autograd (pinned against the reference
module's gradients in tests/test_oracle_vs_reference.py), and the loss / resample / avg-pool backward kernels.
Stated tolerance (precise forward, fp32 SIMT backward): shallow units |d| <= 2e-3 * max|ref| per tensor, relative L2 error <= 1e-3.

ReLU-gate flips.  The forward activations carry the precise mode's ~6e-5 absolute error, so roughly one pre-activation per
layer output (|z| < 6e-5 among ~3e4 elements) lands on the other side of zero than in the fp64 reference.  That single gate
changes a bias gradient (a sum of ~2e3 O(1) terms) by one O(1) term, i.e. by ~2 %, and every gradient upstream of it by a
similar fraction -- measured: tools/debug/dduu.py shows our d(beta) equal to sum(g * (our_output > 0)) to 1e-6 and
differing from the reference by exactly the gradient of the one flipped element.  The fp32 reference itself flips ~60x more
rarely (its forward error is ~1e-6).  Chains deeper than ~4 layers and the whole networks are therefore checked with a
flip-tolerant criterion: relative L2 <= 8e-2 per tensor, the MEDIAN tensor <= 1.5e-2, and the last layer's bias gradient must
equal the gate sum of OUR forward output exactly (test_backward_is_consistent_with_our_forward_gates)."""
import pytest
import torch
import torch.nn as nn

import bf16_emul as E
import cases as C
from vid2vid_b200 import networks as NW
from vid2vid_b200 import ops
from vid2vid_b200.utils import det_fill_

pytestmark = pytest.mark.gpu
BN = NW.get_norm_layer('batch')


def _cmp(name, ours, ref, tol=2e-3, l2=1e-3):
    ours, ref = ours.double().cpu(), ref.double().cpu()
    assert ours.shape == ref.shape, (name, ours.shape, ref.shape)
    assert torch.isfinite(ours).all(), name
    scale = max(ref.abs().max().item(), 1e-12)
    mx = (ours - ref).abs().max().item() / scale
    rel = ((ours - ref).norm() / max(ref.norm().item(), 1e-12)).item()
    print('%-44s max|d|/max|ref|=%.2e  rel L2=%.2e  (max|ref|=%.3e)' % (name, mx, rel, scale))
    assert (tol is None or mx <= tol) and rel <= l2, (name, mx, rel)
    return rel


DEEP = {'enc_dec', 'dduu', 'ddu', 'duu', 'down_res_up', 'd_layers', 'up_up', 'up_up_wide', 'stem_down', 'down_down', 'down_res64', 'res64_up'}


UNITS = [
    ('c3s1_reflect_bn_relu', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(16, 32, 3), BN(32), nn.ReLU(True)], (2, 16, 12, 20)),
    ('c7_stem_reflect', lambda: NW._stem(6, 16, BN), (1, 6, 16, 24)),
    ('c3s2_zero', lambda: NW._down(16, 32, BN), (2, 16, 12, 20)),
    ('c3s2_odd', lambda: NW._down(8, 16, BN), (1, 8, 13, 19)),
    ('deconv', lambda: NW._up(32, 16, BN), (1, 32, 8, 12)),
    ('resblock', lambda: [NW.ResnetBlock(32, 'reflect', BN)], (2, 32, 8, 12)),
    ('down_res_up', lambda: NW._down(16, 32, BN) + [NW.ResnetBlock(32, 'reflect', BN)] + NW._up(32, 16, BN), (1, 16, 16, 16)),
    ('up_up', lambda: NW._up(64, 32, BN) + NW._up(32, 16, BN), (1, 64, 8, 16)),
    ('up_up_wide', lambda: NW._up(64, 32, BN) + NW._up(32, 16, BN), (1, 64, 8, 32)),
    ('stem_down', lambda: NW._stem(6, 16, BN) + NW._down(16, 32, BN), (1, 6, 32, 64)),
    ('down_down', lambda: NW._down(16, 32, BN) + NW._down(32, 64, BN), (1, 16, 32, 64)),
    ('down_res64', lambda: NW._down(32, 64, BN) + [NW.ResnetBlock(64, 'reflect', BN)], (1, 32, 16, 32)),
    ('res64_up', lambda: [NW.ResnetBlock(64, 'reflect', BN)] + NW._up(64, 32, BN), (1, 64, 8, 16)),
    ('ddu', lambda: NW._down(16, 32, BN) + NW._down(32, 64, BN) + NW._up(64, 32, BN), (1, 16, 32, 64)),
    ('dduu', lambda: NW._down(16, 32, BN) + NW._down(32, 64, BN) + NW._up(64, 32, BN) + NW._up(32, 16, BN), (1, 16, 32, 64)),
    ('duu', lambda: NW._down(32, 64, BN) + NW._up(64, 32, BN) + NW._up(32, 16, BN), (1, 32, 16, 32)),
    ('enc_dec', lambda: NW._stem(6, 16, BN) + NW._down(16, 32, BN) + NW._down(32, 64, BN) + [NW.ResnetBlock(64, 'reflect', BN)] +
     NW._up(64, 32, BN) + NW._up(32, 16, BN), (1, 6, 32, 64)),
    ('d_first_layer_lrelu', lambda: [nn.Conv2d(9, 16, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True)], (2, 9, 16, 24)),
    ('d_layers', lambda: [nn.Conv2d(9, 16, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True), nn.Conv2d(16, 32, 4, stride=2, padding=2),
                          BN(32), nn.LeakyReLU(0.2, True), nn.Conv2d(32, 32, 4, stride=1, padding=2), BN(32), nn.LeakyReLU(0.2, True)],
     (2, 9, 20, 28)),
]
# shapes that reach the tensor-core backward (csrc/wgrad_umma.cu needs >= 64 padded channels on both operands and buffer rows of
# >= 16 pixels; the data gradient runs as a forward conv on conv_umma_kernel for every stride-1 / stride-2 / transposed conv)
TENSOR_UNITS = [
    ('t_c3_128', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 12, 72)),      # KP 64, ragged row
    ('t_c3_64_192', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 192, 3), BN(192), nn.ReLU(True)], (2, 64, 10, 40)),    # partial M tile, KP 32
    ('t_c3_192_64', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(192, 64, 3), BN(64), nn.ReLU(True)], (1, 192, 10, 40)),    # 64-channel OUT
    ('t_stem108', lambda: NW._stem(108, 64, BN), (1, 108, 10, 70)),                                                       # 7x7, 49 taps
    ('t_down128', lambda: NW._down(64, 128, BN), (1, 64, 16, 80)),                                                        # stride 2
    ('t_up128', lambda: NW._up(128, 64, BN), (1, 128, 8, 40)),                                                            # transposed
    ('t_d_k4s1', lambda: [nn.Conv2d(64, 128, 4, stride=1, padding=2), BN(128), nn.LeakyReLU(0.2, True)], (1, 64, 12, 40)),
    ('t_d_k4s2', lambda: [nn.Conv2d(64, 128, 4, stride=2, padding=2), BN(128), nn.LeakyReLU(0.2, True)], (1, 64, 16, 80)),      # cropped transposed conv
    ('t_resblock128', lambda: [NW.ResnetBlock(128, 'reflect', BN)], (1, 128, 16, 32)),
    ('t_c3_256_128', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(256, 128, 3), BN(128), nn.ReLU(True)], (1, 256, 8, 40)),   # 256-wide N tile
    ('t_c3_320_64', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(320, 64, 3), BN(64), nn.ReLU(True)], (1, 320, 8, 40)),     # partial 256-wide tile
    # one narrow operand (16 / 32 padded channels) on the N side of the weight-gradient GEMM
    ('t_stem6', lambda: NW._stem(6, 64, BN), (1, 6, 12, 40)),                                                            # narrow activation
    ('t_c3_24_128', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(24, 128, 3), BN(128), nn.ReLU(True)], (1, 24, 10, 40)),    # 32-channel rows
    ('t_d_last', lambda: [nn.Conv2d(64, 1, 4, stride=1, padding=2)], (2, 64, 12, 40)),                                   # narrow gradient (swap)
    ('t_down_24', lambda: NW._down(64, 24, BN), (1, 64, 16, 80)),                                                        # stride 2, narrow gradient
    ('t_head_tanh', lambda: NW._stem(8, 64, BN), (1, 8, 12, 40), lambda: NW._head(64, 3, nn.Tanh()), 1.0),
    ('t_head_flow', lambda: NW._stem(8, 128, BN), (1, 8, 12, 40), lambda: NW._head(128, 2), 20.0),
    ('t_head_both_narrow', lambda: NW._stem(8, 32, BN), (1, 8, 12, 40), lambda: NW._head(32, 3, nn.Tanh()), 1.0),       # dY padded to 64 channels
]


@pytest.mark.parametrize('unit', TENSOR_UNITS, ids=[u[0] for u in TENSOR_UNITS])
def test_tensor_core_backward_units(unit, monkeypatch):
    """Gradients of the tensor-core backward (data gradient as a forward conv + fold, weight gradient with pixels as the K
    dimension) against fp64 autograd, and against the fp32 SIMT backward kernels of the same plan description."""
    name, build, shape = unit[:3]
    head, scale = (unit[3], unit[4]) if len(unit) > 3 else (None, 1.0)
    make = lambda: NW.SequentialRunner(build(), head(), scale) if head else NW.SequentialRunner(build())
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1)).cuda()
    runner = det_fill_(make(), seed=5).cuda()
    runner.precision = 'precise'
    names, ours, refs, out, ref = _grads(runner, x)
    monkeypatch.setenv('V2V_BWD', 'simt')
    simt = det_fill_(make(), seed=5).cuda()
    simt.precision = 'precise'
    _, ours_simt, _, _, _ = _grads(simt, x)
    bad = []
    for n, o, r, so in zip(names, ours, refs, ours_simt):
        if n.endswith('.bias') and r.abs().max().item() < 1e-6:
            continue
        try:
            _cmp('%s tensor vs simt d/d %s' % (name, n), o, so, tol=2e-4, l2=5e-5)
            _cmp('%s d/d %s' % (name, n), o, r, tol=None, l2=8e-2)       # flip-tolerant (module docstring); the strict check is the line above
        except AssertionError as e:
            bad.append(str(e)[:160])
    assert not bad, bad


HEADS = [
    ('head_tanh', lambda: NW._stem(8, 16, BN), lambda: NW._head(16, 3, nn.Tanh()), 1.0, (1, 8, 12, 20)),
    ('head_flow_x20', lambda: NW._stem(8, 16, BN), lambda: NW._head(16, 2), 20.0, (1, 8, 12, 20)),
    ('head_sigmoid', lambda: NW._stem(8, 16, BN), lambda: NW._head(16, 1, nn.Sigmoid()), 1.0, (2, 8, 12, 20)),
]


def _grads(runner, x, gout_seed=3):
    params = list(runner.parameters())
    for p in params:
        p.grad = None
    xr = x.clone().requires_grad_(True)
    out = runner(xr)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(gout_seed)).cuda()
    (out * g).sum().backward()
    ours = [xr.grad.clone()] + [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in params]
    # reference: the same layers by PyTorch in fp64 with autograd
    for p in params:
        p.grad = None
    E.ROUND[0], E.GRAD[0] = False, True
    try:
        xd = x.clone().double().requires_grad_(True)
        ref = E.run_units(list(runner.seq), xd)
        if runner.head is not None:
            ref = E.run_head(list(runner.head), ref, runner.head_scale)
        (ref * g.double()).sum().backward()
    finally:
        E.ROUND[0], E.GRAD[0] = True, False
    refs = [xd.grad.clone()] + [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in params]
    names = ['input'] + [n for n, _ in runner.named_parameters()]
    return names, ours, refs, out, ref


@pytest.mark.parametrize('name,build,shape', UNITS, ids=[u[0] for u in UNITS])
def test_unit_gradients(name, build, shape):
    runner = det_fill_(NW.SequentialRunner(build()), seed=5).cuda()
    runner.precision = 'precise'
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1)).cuda()
    names, ours, refs, out, ref = _grads(runner, x)
    _cmp(name + ' forward', out.detach(), ref.detach(), tol=3e-4, l2=1e-4)
    bad = []
    for n, o, r in zip(names, ours, refs):
        if n.endswith('.bias') and r.abs().max().item() < 1e-6:
            assert o.abs().max().item() < 1e-4, n        # bias in front of a norm: zero gradient (rounding noise in the reference)
            continue
        try:
            if name in DEEP:
                _cmp('%s d/d %s' % (name, n), o, r, tol=None, l2=8e-2)       # flip-tolerant (see the module docstring)
            else:
                _cmp('%s d/d %s' % (name, n), o, r)
        except AssertionError as e:
            bad.append(str(e)[:120])
    assert not bad, bad


def test_backward_is_consistent_with_our_forward_gates():
    """The last BatchNorm's bias gradient is sum(g * relu'(z)); with OUR forward output as the gate it must match to fp32
    rounding, whatever the fp64 reference's gates are."""
    mods = NW._down(16, 32, BN) + NW._down(32, 64, BN) + NW._up(64, 32, BN) + NW._up(32, 16, BN)
    runner = det_fill_(NW.SequentialRunner(mods), seed=5).cuda()
    runner.precision = 'precise'
    x = torch.randn(1, 16, 32, 64, generator=torch.Generator().manual_seed(1)).cuda().requires_grad_(True)
    out = runner(x)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).cuda()
    (out * g).sum().backward()
    manual = (g * (out > 0)).sum(dim=(0, 2, 3))
    assert torch.allclose(runner.seq[10].bias.grad, manual, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize('name,build,head,scale,shape', HEADS, ids=[h[0] for h in HEADS])
def test_head_gradients(name, build, head, scale, shape):
    runner = det_fill_(NW.SequentialRunner(build(), head(), scale), seed=6).cuda()
    runner.precision = 'precise'
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(2)).cuda()
    names, ours, refs, out, ref = _grads(runner, x)
    for n, o, r in zip(names, ours, refs):
        if n.endswith('.bias') and r.abs().max().item() < 1e-6 * max(1.0, scale):
            continue
        _cmp('%s d/d %s' % (name, n), o, r)


def test_second_forward_in_between_triggers_recomputation():
    runner = det_fill_(NW.SequentialRunner(NW._down(16, 32, BN) + [NW.ResnetBlock(32, 'reflect', BN)]), seed=7).cuda()
    x1 = torch.randn(1, 16, 12, 12, generator=torch.Generator().manual_seed(1)).cuda().requires_grad_(True)
    x2 = torch.randn(1, 16, 12, 12, generator=torch.Generator().manual_seed(2)).cuda().requires_grad_(True)
    o1 = runner(x1)
    nb = int(runner.seq[1].num_batches_tracked.item())
    o1.sum().backward()
    g_direct = x1.grad.clone()
    x1.grad = None
    o1 = runner(x1)
    runner(x2)                      # overwrites the plan's buffers
    o1.sum().backward()             # -> re-executes the first forward, without touching the running statistics again
    # (not bit for bit: the per-channel sums of the norm backward meet through float atomics, whose order varies run to run)
    assert torch.allclose(x1.grad, g_direct, rtol=1e-4, atol=1e-6)
    assert int(runner.seq[1].num_batches_tracked.item()) == nb + 2


@pytest.mark.parametrize('name', ['g0_small', 'gl_small_s1'])
def test_generator_gradients_vs_oracle(name):
    from oracle import generator_oracle as GO
    from oracle.make_golden import coarse_feats
    c = C.CASES[name]
    net = det_fill_(C.build_module(c), seed=c['seed'])
    sd = {k: v.clone().double().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
          for k, v in net.state_dict().items()}
    inp, img_prev, mask = C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed'], block=c.get('block', 4))
    local = c['kind'] == 'compositeLocal'
    coarse = tuple(coarse_feats(c)) if local else (None, None, None)
    gs = [torch.randn(1, ch, c['h'], c['w'], generator=torch.Generator().manual_seed(20 + i)) for i, ch in
          enumerate((3, 2, 1, 3, c['ngf'], c['ngf'], c['ngf'] // 2 if c['nd'] > 2 else c['ngf']))]
    torch.set_default_dtype(torch.float64)
    try:
        cd = [t.detach().clone().double().requires_grad_(True) if t is not None else None for t in coarse]
        if local:
            ref = GO.composite_local_generator(sd, inp.double(), img_prev.double(), mask.double(), *cd, False,
                                               n_blocks_local=c['n_blocks_local'], use_fg_model=c['fg'], scale=c['scale'])
        else:
            ref = GO.composite_generator(sd, inp.double(), img_prev.double(), mask.double(), False, n_downsampling=c['nd'],
                                         n_blocks=c['n_blocks'], use_fg_model=c['fg'], no_flow=c['no_flow'])
        sum(((r * g.double()).sum() for r, g in zip(ref, gs) if r is not None)).backward()
    finally:
        torch.set_default_dtype(torch.float32)
    # the fp32 noise floor of these gradients: the same oracle evaluated in fp32 against its fp64 evaluation
    sd32 = {k: v.detach().float().requires_grad_(v.requires_grad) for k, v in sd.items()}
    c32 = [t.detach().clone().float().requires_grad_(True) if t is not None else None for t in coarse]
    if local:
        r32 = GO.composite_local_generator(sd32, inp, img_prev, mask, *c32, False, n_blocks_local=c['n_blocks_local'],
                                           use_fg_model=c['fg'], scale=c['scale'])
    else:
        r32 = GO.composite_generator(sd32, inp, img_prev, mask, False, n_downsampling=c['nd'], n_blocks=c['n_blocks'],
                                     use_fg_model=c['fg'], no_flow=c['no_flow'])
    sum(((r * g).sum() for r, g in zip(r32, gs) if r is not None)).backward()
    floor = {k: ((sd32[k].grad.double() - sd[k].grad).norm() / max(sd[k].grad.norm().item(), 1e-12)).item()
             for k in sd if sd[k].grad is not None and sd32[k].grad is not None}
    print('fp32-oracle vs fp64-oracle gradient rel L2: max %.2e median %.2e' % (max(floor.values()), sorted(floor.values())[len(floor) // 2]))
    net = net.cuda()
    net.precision = 'precise'
    cg = [t.detach().clone().cuda().requires_grad_(True) if t is not None else None for t in coarse]
    out = net(inp.cuda(), img_prev.cuda(), mask.cuda(), *cg, False)
    sum(((o * g.cuda()).sum() for o, g in zip(out, gs) if o is not None)).backward()
    for key, o, r in zip(C.GEN_OUT_NAMES, out, ref):
        if o is not None:
            _cmp('%s forward %s' % (name, key), o.detach(), r.detach(), tol=2e-3, l2=1e-3)
    bad, rels = [], []
    for k, p in net.named_parameters():
        r = sd[k].grad if sd[k].grad is not None else torch.zeros_like(sd[k])
        if k.endswith('.bias') and r.abs().max().item() < 1e-7:
            continue
        try:
            rels.append(_cmp('%s d/d %s' % (name, k), p.grad, r, tol=None, l2=8e-2))     # flip-tolerant (module docstring)
        except AssertionError as e:
            bad.append(str(e))
    for i, (t, tr) in enumerate(zip(cg, cd)):
        if t is not None:
            _cmp('%s d/d coarse feature %d' % (name, i), t.grad, tr.grad, tol=None, l2=8e-2)
    assert not bad, bad[:5]
    rels.sort()
    print('%s: median relative L2 over %d parameter tensors %.2e, max %.2e' % (name, len(rels), rels[len(rels) // 2], rels[-1]))
    assert rels[len(rels) // 2] <= 1.5e-2


def test_discriminator_gradients_vs_oracle():
    from oracle import generator_oracle as GO
    c = C.CASES['D_small']
    net = det_fill_(C.build_module(c), seed=c['seed'])
    sd = {k: v.clone().double().requires_grad_(k.split('.')[-1] in ('weight', 'bias')) for k, v in net.state_dict().items()}
    x = torch.randn(c['batch'], c['input_nc'], c['h'], c['w'], generator=torch.Generator().manual_seed(c['seed'] + 1))
    torch.set_default_dtype(torch.float64)
    try:
        xd = x.double().requires_grad_(True)
        ref = GO.multiscale_discriminator(sd, xd, num_D=c['num_D'], n_layers=c['n_layers'], norm='batch', getIntermFeat=True)
        gs = [[torch.randn(t.shape, generator=torch.Generator().manual_seed(100 + 10 * i + j)) for j, t in enumerate(tw)] for i, tw in enumerate(ref)]
        sum((t * g).sum() for tw, gw in zip(ref, gs) for t, g in zip(tw, gw)).backward()
    finally:
        torch.set_default_dtype(torch.float32)
    net = net.cuda()
    net.precision = 'precise'
    xg = x.cuda().requires_grad_(True)
    out = net(xg)
    sum((t * g.float().cuda()).sum() for tw, gw in zip(out, gs) for t, g in zip(tw, gw)).backward()
    _cmp('D d/d input', xg.grad, xd.grad, tol=None, l2=3e-2)
    for k, p in net.named_parameters():
        r = sd[k].grad if sd[k].grad is not None else torch.zeros_like(sd[k])
        if k.endswith('.bias') and r.abs().max().item() < 1e-7:
            continue
        _cmp('D d/d %s' % k, p.grad, r, tol=None, l2=3e-2)


def test_loss_and_helper_backward_kernels():
    g = torch.Generator().manual_seed(4)
    a = torch.randn(2, 3, 20, 28, generator=g)
    b = torch.randn(2, 3, 20, 28, generator=g)
    m = (torch.rand(2, 1, 20, 28, generator=g) > 0.4).float()
    for mask in (None, m):
        ad, bd = a.double().requires_grad_(True), b.double().requires_grad_(True)
        md = mask.double().expand(-1, 3, -1, -1) if mask is not None else 1.0
        ref = torch.mean(torch.abs(ad * md - bd * md)) * 3.0
        ref.backward()
        ag, bg = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
        out = ops.l1_loss(ag, bg, mask.cuda() if mask is not None else None) * 3.0
        out.backward()
        assert abs(out.item() - ref.item()) < 1e-6 * max(1.0, abs(ref.item()))
        _cmp('l1 d/da', ag.grad, ad.grad, tol=1e-5, l2=1e-5)
        _cmp('l1 d/db', bg.grad, bd.grad, tol=1e-5, l2=1e-5)
    xd = a.double().requires_grad_(True)
    ref = torch.mean((xd - 1.0) ** 2)
    ref.backward()
    xg = a.cuda().requires_grad_(True)
    out = ops.mse_to_const(xg, 1.0)
    out.backward()
    assert abs(out.item() - ref.item()) < 1e-6
    _cmp('mse d/dx', xg.grad, xd.grad, tol=1e-5, l2=1e-5)
    # resample: gradients wrt image and flow against grid_sample autograd (oracle.generator_oracle.resample)
    from oracle import generator_oracle as GO
    img = torch.rand(2, 3, 20, 28, generator=g)
    flow = torch.randn(2, 2, 20, 28, generator=g) * 2.5
    go = torch.randn(2, 3, 20, 28, generator=g)
    for ac in (False, True):
        i_d, f_d = img.clone().requires_grad_(True), flow.clone().requires_grad_(True)
        (GO.resample(i_d, f_d, ac) * go).sum().backward()
        i_g, f_g = img.cuda().requires_grad_(True), flow.cuda().requires_grad_(True)
        (ops.resample(i_g, f_g, ac) * go.cuda()).sum().backward()
        _cmp('resample d/d image (ac=%d)' % ac, i_g.grad, i_d.grad, tol=1e-4, l2=1e-4)
        _cmp('resample d/d flow (ac=%d)' % ac, f_g.grad, f_d.grad, tol=1e-3, l2=1e-3)
    x = torch.randn(3, 5, 17, 22, generator=g)
    xd = x.clone().requires_grad_(True)
    gp = torch.randn(3, 5, 9, 11, generator=g)
    (torch.nn.functional.avg_pool2d(xd, 3, stride=2, padding=1, count_include_pad=False) * gp).sum().backward()
    xg = x.cuda().requires_grad_(True)
    (ops.avgpool3s2(xg) * gp.cuda()).sum().backward()
    _cmp('avgpool3s2 backward', xg.grad, xd.grad, tol=1e-6, l2=1e-6)
