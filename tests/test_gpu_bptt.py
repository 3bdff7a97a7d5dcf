"""Gradient into previously generated frames and fixed coarse scales on the GPU (vid2vid_model_G.py:167-168, :181-186).
  * the composite backward's img_prev gradient (grid_sample's input gradient, border padding) against fp64 autograd;
  * the generators' img_prev gradient (warp + image-branch stem) against the reference fixture and the fp64 oracle;
  * a two-frame training step with n_frames_bp 2 against the detach-aware oracle, and --niter_fix_global 1."""
import pytest
import torch
import torch.nn as nn

import cases as C
import reference_inputs as RI
from oracle.bptt_oracle import BPTTModelGOracle
from oracle import flownet2_oracle as FO
from oracle import generator_oracle as GO
from oracle import losses_oracle as LO
from test_gpu_train_step import _setup
from vid2vid_b200 import networks as NW
from vid2vid_b200.networks import S_FG, S_FINAL, S_FLOW, S_MASK, S_PREV, S_RAW, S_RAWC, S_W
from vid2vid_b200.plan import Plan
from vid2vid_b200.trainer import Trainer
from vid2vid_b200.utils import det_fill_, make_opt

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


# ------------------------------------------------------------------------------------------------ composite kernel
def _flow(kind, N, H, W, g):
    if kind == 'frac':
        return torch.randn(N, 2, H, W, generator=g) * 2.5
    if kind == 'int':
        return torch.randint(-3, 4, (N, 2, H, W), generator=g).float()
    if kind == 'zero':
        return torch.zeros(N, 2, H, W)
    if kind == 'out':        # leaves the frame on every side: border clamping, many pixels onto one
        return (torch.rand(N, 2, H, W, generator=g) * 2 - 1) * torch.tensor([1.5 * W, 1.5 * H]).view(1, 2, 1, 1)
    return torch.sign(torch.randn(N, 2, H, W, generator=g)) * 1e3      # 'saturated': every pixel samples a corner


@pytest.mark.parametrize('shape', [(2, 6, 13, 22), (2, 12, 10, 37)])
@pytest.mark.parametrize('fg', [False, True])
@pytest.mark.parametrize('flow_kind', ['frac', 'int', 'zero', 'out', 'saturated'])
@pytest.mark.parametrize('ac', [False, True])
def test_composite_prev_gradient_vs_fp64(shape, fg, flow_kind, ac):
    N, pc, H, W = shape
    g = torch.Generator().manual_seed(7)
    raw, w = torch.rand(N, 3, H, W, generator=g) * 2 - 1, torch.rand(N, 1, H, W, generator=g)
    prev, flow = torch.rand(N, pc, H, W, generator=g) * 2 - 1, _flow(flow_kind, N, H, W, g)
    fgi, mask = torch.rand(N, 3, H, W, generator=g) * 2 - 1, (torch.rand(N, 1, H, W, generator=g) > 0.5).float()
    g_final = torch.randn(N, 3, H, W, generator=g)
    plan = Plan(0, precision='precise', train=True)
    plan.input(S_PREV, N, pc, 0, pc, H, W)
    plan.composite(S_RAW, S_FLOW, S_W, S_PREV, pc, S_FG if fg else -1, S_MASK if fg else -1, S_FINAL, N, H, W, True, ac,
                   s_raw_out=S_RAWC if fg else -1)
    plan.finalize()
    io = [None] * 15
    io[S_RAW], io[S_FLOW], io[S_W], io[S_PREV] = raw.cuda(), flow.cuda(), w.cuda(), prev.cuda()
    io[S_FINAL] = torch.empty(N, 3, H, W, device='cuda')
    if fg:
        io[S_FG], io[S_MASK], io[S_RAWC] = fgi.cuda(), mask.cuda(), torch.empty(N, 3, H, W, device='cuda')
    plan.run(io, False)
    gio = [None] * 15
    gio[S_FINAL], gio[S_PREV] = g_final.cuda(), torch.zeros(N, pc, H, W, device='cuda')
    plan.backward(io, gio, [], [])
    torch.cuda.synchronize()
    p64 = prev.double().requires_grad_(True)
    w64 = w.double()
    final = raw.double() * w64 + GO.resample(p64[:, -3:], flow.double(), ac) * (1 - w64)
    if fg:
        final = fgi.double() * mask.double() + final * (1 - mask.double())
    (final * g_final.double()).sum().backward()
    ours = gio[S_PREV].cpu()
    assert torch.isfinite(ours).all()
    assert not ours[:, :pc - 3].any()                  # channels before the last three get nothing from the composite
    rel = _rel(ours, p64.grad)
    print('composite d/d img_prev %s fg=%d %-9s ac=%d: rel L2 %.2e' % (shape, fg, flow_kind, ac, rel))
    assert rel <= 1e-5


# ------------------------------------------------------------------------------------------------ generators
def _stem_only(monkeypatch):
    """Make the oracle's warp read a detached img_prev: its img_prev gradient is then the stem's alone."""
    resample = GO.resample
    monkeypatch.setattr(GO, 'resample', lambda image, flow, align_corners=False: resample(image.detach(), flow, align_corners))


def test_composite_generator_img_prev_gradient_vs_reference(monkeypatch):
    """The seed-31 coarse generator whose gradients the reference fixture stores (grad/img_prev)."""
    gold = RI.golden()
    opt = make_opt(ngf=8, n_blocks=2, fg=True, n_downsample_G=2, gpu_ids=[])
    net = det_fill_(NW.define_G(18, 3, 6, 8, 'composite', 2, 'batch', 0, [], opt), seed=31)
    C.condition_flow_heads(net, 0.05)
    net = net.cuda()
    net.precision = 'precise'
    inp, img_prev, mask = RI.gen_inputs(6, 16, 32, seed=2)
    p = img_prev.cuda().requires_grad_(True)
    outs = net(inp.cuda(), p, mask.cuda(), None, None, None, False)
    cot = RI.cotangents([o.cpu() if o is not None else None for o in outs])
    RI.objective(outs, [c.cuda() if c is not None else None for c in cot]).backward()
    ref = torch.from_numpy(gold['grad/img_prev'])
    rel = _rel(p.grad, ref)
    # the stem's part alone (the parent's gradient) misses the reference by the warp term
    _stem_only(monkeypatch)
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    p_stem = img_prev.clone().requires_grad_(True)
    out = GO.composite_generator(sd, inp, p_stem, mask, False, n_downsampling=2, n_blocks=2, use_fg_model=True)
    RI.objective(out, RI.cotangents(out)).backward()
    rel_stem = _rel(p_stem.grad, ref)
    print('CompositeGenerator d/d img_prev vs reference: rel L2 %.2e (stem path alone %.2e)' % (rel, rel_stem))
    assert rel <= 0.1 * rel_stem


def _oracle_prev_grad(c, net, inp, img_prev, mask, coarse, gs, use_raw_only):
    sd = {k: v.detach().clone().double() for k, v in net.state_dict().items()}
    p = img_prev.double().requires_grad_(True)
    cd = [t.double() if t is not None else None for t in coarse]
    torch.set_default_dtype(torch.float64)
    try:
        if c['kind'] == 'compositeLocal':
            ref = GO.composite_local_generator(sd, inp.double(), p, mask.double(), *cd, use_raw_only, n_blocks_local=c['n_blocks_local'],
                                               use_fg_model=c['fg'], scale=c['scale'])
        else:
            ref = GO.composite_generator(sd, inp.double(), p, mask.double(), use_raw_only, n_downsampling=c['nd'], n_blocks=c['n_blocks'],
                                         use_fg_model=c['fg'], no_flow=c['no_flow'])
        sum(((r * g.double()).sum() for r, g in zip(ref, gs) if r is not None)).backward()
    finally:
        torch.set_default_dtype(torch.float32)
    return p.grad


@pytest.mark.parametrize('name,use_raw_only', [('gl_small_s1', False), ('g0_small', False), ('g0_small', True), ('g0_noflow', False)])
def test_generator_img_prev_gradient_vs_oracle(name, use_raw_only, monkeypatch):
    """Warp + stem (CompositeLocalGenerator / CompositeGenerator); use_raw_only and no_flow reach img_prev through the stem only.
    The warp term is pinned where it exceeds the error of the stem path: in gl_small_s1 it is 6 % of the gradient, against our
    4e-4.  In g0_small (nine residual blocks) it is 1 %, below the ReLU-flip noise of the deep stem path (1.7 %), so that case
    is checked with the flip-tolerant bound only."""
    from oracle.make_golden import coarse_feats
    c = C.CASES[name]
    net = det_fill_(C.build_module(c), seed=c['seed'])
    C.condition_flow_heads(net, 0.05)
    inp, img_prev, mask = C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed'], block=c.get('block', 4))
    coarse = tuple(coarse_feats(c)) if c['kind'] == 'compositeLocal' else (None, None, None)
    gs = [torch.randn(1, ch, c['h'], c['w'], generator=torch.Generator().manual_seed(20 + i)) for i, ch in
          enumerate((3, 2, 1, 3, c['ngf'], c['ngf'], c['ngf'] // 2 if c['nd'] > 2 else c['ngf']))]
    ref = _oracle_prev_grad(c, net, inp, img_prev, mask, coarse, gs, use_raw_only)
    net = net.cuda()
    net.precision = 'precise'
    p = img_prev.cuda().requires_grad_(True)
    out = net(inp.cuda(), p, mask.cuda(), *[t.cuda() if t is not None else None for t in coarse], use_raw_only)
    sum(((o * g.cuda()).sum() for o, g in zip(out, gs) if o is not None)).backward()
    rel = _rel(p.grad, ref)
    print('%s use_raw_only=%d d/d img_prev vs fp64 oracle: rel L2 %.2e' % (name, use_raw_only, rel))
    assert rel <= 8e-2
    if name == 'gl_small_s1':
        _stem_only(monkeypatch)
        rel_stem = _rel(_oracle_prev_grad(c, net.cpu(), inp, img_prev, mask, coarse, gs, use_raw_only), ref)
        print('  stem path alone vs fp64 oracle: rel L2 %.2e' % rel_stem)
        assert rel <= 0.1 * rel_stem


# ------------------------------------------------------------------------------------------------ training step
def _step_grads(opt, G, D, flow, A, B, T):
    tr = Trainer(opt, G, D, flow, world=1)
    a, b = A[:, :T].cuda(), B[:, :T].cuda()
    loss_G, loss_D, _, ld, _ = tr.losses(a, b, a)
    tr.grads.zero()
    loss_G.backward()
    gG = {'%d.%s' % (s, n): q.grad.detach().cpu().double().clone() for s in range(2) for n, q in getattr(G, 'netG%d' % s).named_parameters()}
    tr.grads.zero(1)
    loss_D.backward()
    gD = {n: q.grad.detach().cpu().double().clone() for n, q in D.netD.named_parameters()}
    return tr, ld, gG, gD


def _oracle_step(opt, G, D, flow, A, B, T, **kw):
    """Losses and first-step G / D gradients of the oracle (as tests/test_gpu_train_step.py) over T - tG + 1 frames."""
    sds = [{k: v.detach().cpu().clone().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
            for k, v in getattr(G, 'netG%d' % s).state_dict().items()} for s in range(2)]
    sdD = {k: v.detach().cpu().clone().requires_grad_(k.split('.')[-1] in ('weight', 'bias')) for k, v in D.netD.state_dict().items()}
    sdF = {k: v.detach().cpu() for k, v in flow.flowNet.state_dict().items()}
    fake_B, raws, flows, weights, real_A, real_Bp, _ = BPTTModelGOracle(opt, sds).train_forward(
        A[:, :T], B[:, :T], A[:, :T], None, n_frames_load=T - opt.n_frames_G + 1, **kw)
    real_B_prev, real_B = real_Bp[:, :-1], real_Bp[:, 1:]
    m = lambda t: t.reshape(-1, *t.shape[2:])
    with torch.no_grad():
        flow_ref, conf_ref = FO.flow_and_conf(sdF, m(real_B), m(real_B_prev))
    fake_B_prev = torch.cat([real_B_prev[:, 0:1], fake_B[:, :-1].detach()], dim=1)           # compute_fake_B_prev
    lo = LO.spatial_losses(sdD, m(real_B), m(fake_B), m(raws), m(real_A), m(real_B_prev), m(fake_B_prev), m(flows), m(weights),
                           flow_ref, conf_ref, lambda_F=opt.lambda_F, lambda_T=opt.lambda_T, lambda_feat=opt.lambda_feat,
                           n_scales_spatial=2, no_first_img=False, num_D=opt.num_D, n_layers_D=opt.n_layers_D, norm=opt.norm)
    od = dict(zip(D.loss_names, [torch.mean(x) for x in lo]))
    (od['G_GAN'] + od['G_GAN_Feat'] + od['G_VGG'] + od['G_Warp'] + od['F_Flow'] + od['F_Warp'] + od['W']).backward(retain_graph=True)
    gG = {'%d.%s' % (s, k): v.grad.double().clone() for s in range(2) for k, v in sds[s].items() if v.grad is not None}
    for v in sdD.values():
        v.grad = None
    ((od['D_fake'] + od['D_real']) * 0.5).backward()
    gD = {k: v.grad.double().clone() for k, v in sdD.items() if v.grad is not None}
    return od, gG, gD


def _compare(name, ours, ref, lim_max, lim_med, prefix=''):
    gmax = max(r.abs().max().item() for r in ref.values())
    rels = []
    for k, r in ref.items():
        if not k.startswith(prefix) or r.abs().max().item() < 1e-9 or \
                (k.endswith('.bias') and ours[k].abs().max().item() == 0 and r.abs().max().item() < 1e-5 * gmax):
            continue          # conv bias in front of a norm layer: exactly zero here, rounding noise in the reference
        rels.append((_rel(ours[k], r), k))
    rels.sort()
    print('%s: %d tensors, median rel L2 %.2e, max %.2e; largest %s' % (name, len(rels), rels[len(rels) // 2][0], rels[-1][0],
                                                                      ['%s %.3f' % (k, v) for v, k in rels[-4:]]))
    assert lim_max is None or rels[-1][0] <= lim_max, (name, rels[-1])
    return rels[len(rels) // 2][0]


def test_two_frame_step_backpropagates_into_the_previous_frame():
    opt, G, D, flow, A, B = _setup()
    # Random x20 flow heads give noise-like multi-pixel flows.  Each warp then turns tiny forward differences into different
    # bilinear cells, and the gradient that crosses frames passes two of them.  Shrink the heads, as the reference fixtures do.
    # Unscaled, this step measured G median 4.8e-2 / max 0.18 on the precise path and 4.3e-2 / 0.12 on V2V_CONV_IMPL=simt
    # (whose forward matches fp32 to 1e-5), against 3.3e-2 (coarse scale) and 6e-3 (finest) at n_frames_bp 1.
    for s in range(2):
        C.condition_flow_heads(getattr(G, 'netG%d' % s), 0.05)
    opt.max_frames_per_gpu, opt.max_frames_backpropagate = 2, 2
    G.init_train()
    G.n_frames_bp = 2
    T = opt.n_frames_G + 1
    _, ld, gG, gD = _step_grads(opt, G, D, flow, A, B, T)
    od, rG, rD = _oracle_step(opt, G, D, flow, A, B, T, n_frames_bp=2)
    for n in D.loss_names:
        assert abs(float(ld[n]) - float(od[n])) <= 2e-3 * max(1.0, abs(float(od[n]))), n
    assert _compare('G gradients, n_frames_bp 2', gG, rG, 0.15, 3e-2) <= 3e-2
    assert _compare('D gradients', gD, rD, 0.1, 2e-2) <= 2e-2
    _, rG1, _ = _oracle_step(opt, G, D, flow, A, B, T, n_frames_bp=1)
    for s in range(2):        # the gradient that crosses the cut is far above the tolerance, at both scales
        assert _compare('G%d gradients vs the n_frames_bp 1 oracle' % s, gG, rG1, None, None, prefix='%d.' % s) > 0.1


def _bn_state(net):
    return [(m.running_mean.clone(), int(m.num_batches_tracked)) for m in net.modules() if isinstance(m, nn.BatchNorm2d)]


def test_fixed_global_scale_runs_the_inference_plan_with_the_training_plan_outputs():
    opt, G, D, flow, A, B = _setup(seed=4)
    tG = opt.n_frames_G
    real_A, real_B, _ = G.encode_input(A[:, :tG].cuda(), B[:, :tG].cuda(), A[:, :tG].cuda())
    rA, rB = G.build_pyr(real_A)[1], G.build_pyr(real_B)[1]
    h, w = rA.shape[-2:]
    args = (rA[:, :tG].reshape(1, -1, h, w), rB[:, :tG - 1].reshape(1, -1, h, w), G.compute_mask(rA, tG - 1), None, None, None, False)
    with torch.no_grad():
        inf = G.netG0(*args)
    train = G.netG0(*args)
    assert train[0].requires_grad
    for n, a, b in zip(C.GEN_OUT_NAMES, inf, train):
        if b is not None:
            assert torch.equal(a, b.detach()), n


def test_niter_fix_global_trains_only_the_finest_scale():
    opt, G, D, flow, A, B = _setup(seed=5)
    opt.niter_fix_global = 1
    G.init_train()
    assert [id(p) for g in G.optimizer_G.param_groups for p in g['params']] == [id(p) for p in G.netG1.parameters()]
    T = opt.n_frames_G
    p0 = {n: q.detach().clone() for n, q in G.netG0.named_parameters()}
    bn0 = _bn_state(G.netG0)
    tr, _, gG, _ = _step_grads(opt, G, D, flow, A, B, T)
    assert not any(v.any() for k, v in gG.items() if k.startswith('0.'))
    _, rG, _ = _oracle_step(opt, G, D, flow, A, B, T, finetune_all=False)
    assert not any(k.startswith('0.') for k in rG)
    assert _compare('G1 gradients, finetune_all False', gG, rG, 0.15, 3e-2, prefix='1.') <= 3e-2
    tr.reset_clip()
    tr.step(A[:, :T].cuda(), B[:, :T].cuda(), A[:, :T].cuda())
    for n, q in G.netG0.named_parameters():
        assert torch.equal(q.detach(), p0[n]), n
        assert not q.grad.any(), n
    for (rm, nb), (rm0, nb0) in zip(_bn_state(G.netG0), bn0):         # one netG0 forward in each of the two steps
        assert nb == nb0 + 2 and not torch.equal(rm, rm0)
    G.update_fixed_params()
    p1 = {n: q.detach().clone() for n, q in G.named_parameters()}
    tr.reset_clip()
    tr.step(A[:, 1:T + 1].cuda(), B[:, 1:T + 1].cuda(), A[:, 1:T + 1].cuda())
    for prefix in ('netG0', 'netG1'):
        assert max((q.detach() - p1[n]).abs().max().item() for n, q in G.named_parameters() if n.startswith(prefix)) > 0, prefix
