"""VGG19 perceptual loss on the GPU: the max-pool and feature-L1 plan nodes, the 2x2 average pool, VGGLoss's value and input
gradient against the fp64 CPU oracle (oracle/vgg_oracle.py, pinned against the reference in tests/test_vgg_oracle.py), the
forward-only target branch, and the training step with the VGG term.

Tolerances.  Precise plans carry every conv operand as hi + lo bf16 (16 significand bits, relative representation error
<= 2^-17) and drop the lo*lo product (<= 2^-18); accumulation is fp32.  A layer therefore adds at most ~2 * 2^-17 + 2^-18
~= 1.9e-5 relative error to its output on top of what its input carried, and the 13 conv layers of VGG19 up to relu5_1
accumulate at most ~13 * 1.9e-5 ~= 2.5e-4 relative error per feature element (bound, linear accumulation; the 2x2 max-pool
and ReLU do not amplify it).  The per-level loss mean |x_k - y_k| inherits at most that relative error of the feature
magnitudes, which for random inputs are of the order of |x_k - y_k| itself.  The value tolerance is 4x that bound:
1e-3 relative.  Fast plans (bf16 operands, 2^-9) scale the same bound by 2^8: ~6e-2, the fast mode's image-class tolerance
order; the fast test uses 1e-1."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import vgg_oracle as VO
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200 import ops
from vid2vid_b200.plan import Plan, conv_desc

pytestmark = pytest.mark.gpu

TOL_PRECISE = 1e-3
TOL_FAST = 1e-1


def _cmp(name, ours, ref, tol=2e-3, l2=1e-3):
    """tests/test_gpu_backward.py's criterion: max error relative to the largest reference element, and relative L2 error
    (a ReLU gate or max-pool argmax that flips between two nearly equal values moves a few elements, not the norm)."""
    ours, ref = ours.double().cpu(), ref.double().cpu()
    assert ours.shape == ref.shape, (name, ours.shape, ref.shape)
    assert torch.isfinite(ours).all(), name
    scale = max(ref.abs().max().item(), 1e-12)
    mx = (ours - ref).abs().max().item() / scale
    rel = ((ours - ref).norm() / max(ref.norm().item(), 1e-12)).item()
    print('%-36s max|d|/max|ref|=%.2e  rel L2=%.2e' % (name, mx, rel))
    assert (tol is None or mx <= tol) and rel <= l2, (name, mx, rel)


def _tied(shape, seed, levels=9):
    """Values on a coarse grid (many ties inside pool windows), exact in bf16 and therefore in either precision."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-levels, levels + 1, shape, generator=g).float() / 8).cuda()


@pytest.mark.parametrize('precision', ['precise', 'fast'])
@pytest.mark.parametrize('N,C,H,W', [(2, 64, 16, 24), (1, 128, 13, 19), (1, 16, 7, 9)])
def test_maxpool_node(precision, N, C, H, W):
    x = _tied((N, C, H, W), seed=H * W)
    p = Plan(precision=precision, train=True)
    v = p.maxpool2(p.input(0, N, C, 0, C, H, W))
    p.export(v, 1)
    p.finalize()
    out = torch.empty(N, C, H // 2, W // 2, device='cuda')
    p.run([x, out], use_graph=False)
    xr = x.clone().requires_grad_(True)
    ref = F.max_pool2d(xr, 2, 2)
    assert torch.equal(out, ref.detach())
    g = _tied(out.shape, seed=7)
    ref.backward(g)
    gx = torch.zeros_like(x)
    p.backward([x, out], [gx, g], [], [])
    torch.cuda.synchronize()
    assert torch.equal(gx, xr.grad)


def test_maxpool_node_precise_lo_halves():
    """Precise plans: values of 9-16 significant bits, whose bf16 hi halves tie inside most windows and differ only in the
    lo half.  The pooled value must be the exact fp32 maximum (hi + lo compared, the winner's lo copied) and the gradient must
    go to that element."""
    N, C, H, W = 2, 64, 14, 18
    g = torch.Generator().manual_seed(11)
    hi = (torch.randint(8, 10, (N, C, H, W), generator=g).float() / 8) * (torch.randint(0, 2, (N, C, H, W), generator=g).float() * 2 - 1)
    lo = torch.randint(-3, 4, (N, C, H, W), generator=g).float() * 2.0 ** -10      # |lo| < half a bf16 ulp of hi (2^-8)
    x = (hi + lo).cuda()
    assert (x.cpu() != x.cpu().bfloat16().float()).float().mean() > 0.5              # most values need the lo half
    p = Plan(precision='precise', train=True)
    p.export(p.maxpool2(p.input(0, N, C, 0, C, H, W)), 1)
    p.finalize()
    out = torch.empty(N, C, H // 2, W // 2, device='cuda')
    p.run([x, out], use_graph=False)
    xr = x.clone().requires_grad_(True)
    ref = F.max_pool2d(xr, 2, 2)
    assert torch.equal(out, ref.detach())
    # the case exercises what it is for: windows whose largest hi is shared by elements that differ in lo
    win = lambda t: t[..., :H // 2 * 2, :W // 2 * 2].unfold(2, 2, 2).unfold(3, 2, 2).reshape(N, C, H // 2, W // 2, 4)
    hw, xw = win((hi + lo).bfloat16().float()), win(hi + lo)          # the hi half the import stores, and the value
    top = hw == hw.amax(-1, keepdim=True)
    split = (xw.masked_fill(~top, float('inf')).amin(-1) != xw.masked_fill(~top, -float('inf')).amax(-1))
    assert split.float().mean() > 0.2
    gout = torch.randn(out.shape, generator=g).cuda()
    ref.backward(gout)
    gx = torch.zeros_like(x)
    p.backward([x, out], [gx, gout], [], [])
    torch.cuda.synchronize()
    assert torch.equal(gx, xr.grad)


@pytest.mark.parametrize('precision', ['precise', 'fast'])
def test_feature_l1_node(precision):
    N, C, H, W = 2, 64, 24, 40
    g_ = torch.Generator().manual_seed(1)
    x = (torch.randint(-128, 129, (N, C, H, W), generator=g_).float() / 64).cuda()       # <= 8 significant bits: exact in bf16
    y = (torch.randint(-128, 129, (N, C, H, W), generator=g_).float() / 64).cuda()
    y[:, :, :4] = x[:, :, :4]                                                             # sign(0) = 0 region
    p = Plan(precision=precision, train=True)
    p.feature_l1(p.input(0, N, C, 0, C, H, W), p.input(1, N, C, 0, C, H, W), 2, 1)
    p.finalize()
    out = torch.full((2,), -1.0, device='cuda')
    p.run([x, y, out], use_graph=False)
    first = out.clone()
    p.run([x, y, out], use_graph=True)
    p.run([x, y, out], use_graph=True)
    assert torch.equal(out, first)                                    # deterministic (ordered partial sums)
    assert out[0].item() == -1.0                                      # only its own element is written
    ref = (x.double() - y.double()).abs().mean()
    assert abs(out[1].item() - ref.item()) <= 1e-6 * ref.item()
    gout = torch.tensor([0.0, 3.0], device='cuda')
    gx, gy = torch.zeros_like(x), torch.zeros_like(y)
    p.backward([x, y, out], [gx, gy, gout], [], [])          # y's gradient is asked for: the plan must leave it untouched
    xr = x.clone().requires_grad_(True)
    ((xr - y).abs().mean() * 3.0).backward()
    torch.cuda.synchronize()
    assert torch.allclose(gx, xr.grad, rtol=1e-6, atol=0)
    assert gy.abs().max().item() == 0


@pytest.mark.parametrize('shape', [(2, 3, 64, 2080), (1, 3, 33, 50), (3, 7, 9)])
def test_avgpool2(shape):
    g = torch.Generator().manual_seed(len(shape))
    x = (torch.rand(shape, generator=g) * 2 - 1).cuda().requires_grad_(True)
    out = ops.avgpool2(x)
    ref = F.avg_pool2d(x.detach().reshape(-1, 1, *shape[-2:]), 2, 2, count_include_pad=False).reshape(out.shape)
    assert torch.allclose(out, ref, rtol=1e-6, atol=1e-7)
    go = torch.randn(out.shape, generator=g).cuda()
    out.backward(go)
    xr = x.detach().clone().requires_grad_(True)
    F.avg_pool2d(xr.reshape(-1, 1, *shape[-2:]), 2, 2, count_include_pad=False).reshape(out.shape).backward(go)
    assert torch.allclose(x.grad, xr.grad, rtol=1e-6, atol=0)


def _our_activations(vgg, x):
    """Every intermediate of our VGG branch on x, from a plan of the same units as the loss plan with each value exported:
    (layers, activations, slice ends); layers[i] = (kind, module), activations[i] = its output as fp64 CPU tensor."""
    N, _, H, W = x.shape
    p = Plan(precision=vgg._precision())
    v = p.input(0, N, 3, 0, 3, H, W)
    layers, ids, ends = [], [], []
    for k in range(5):
        for m in getattr(vgg, 'slice%d' % (k + 1)):
            if isinstance(m, nn.Conv2d):
                v = p.conv_act(v, conv_desc(m), L.ACT_RELU, 0.0)
            elif isinstance(m, nn.MaxPool2d):
                v = p.maxpool2(v)
            else:
                continue
            layers.append(('conv' if isinstance(m, nn.Conv2d) else 'pool', m))
            ids.append(v)
        ends.append(len(layers) - 1)
    for i, v in enumerate(ids):
        p.export(v, 1 + i)
    p.finalize()
    vals = {d['id']: d for d in p.describe()['values']}
    outs = [torch.empty(N, vals[v]['C'], vals[v]['H'], vals[v]['W'], device=x.device) for v in ids]
    p.run([x] + outs, use_graph=False)
    return layers, [o.cpu().double() for o in outs], ends


def _masked_backward(vgg, x_in, y_in):
    """fp64 gradient of sum_k w_k mean |x_k - y_k| wrt the VGG input x_in, taken with OUR forward's decisions: the L1 signs of
    our features, the ReLU gates of our conv outputs and the argmax of our max-pool inputs.  Linear given those masks, so it
    is what our backward must compute up to its own rounding."""
    layers, ax, ends = _our_activations(vgg, x_in)
    _, ay, _ = _our_activations(vgg, y_in)
    g = [torch.zeros_like(a) for a in ax]
    for k, i in enumerate(ends):
        g[i] += VO.WEIGHTS[k] * torch.sign(ax[i] - ay[i]) / ax[i].numel()
    for i in reversed(range(len(layers))):
        kind, m = layers[i]
        if kind == 'conv':
            gin = F.conv_transpose2d(g[i] * (ax[i] > 0), m.weight.detach().cpu().double(), padding=1)
        else:
            src = ax[i - 1]
            _, idx = F.max_pool2d(src, 2, 2, return_indices=True)
            gin = torch.zeros_like(src).flatten(2).scatter_add_(2, idx.flatten(2), g[i].flatten(2)).view_as(src)
        if i == 0:
            return gin
        g[i - 1] += gin


def _vgg_loss(precision='precise', seed=VO.SEED):
    crit = NW.VGGLoss(0, synthetic=True)
    NW.vgg19_synthetic_(crit.vgg, seed)
    crit.vgg.precision = precision
    return crit


def _inputs(N, H, W):
    x, y = VO.case_inputs(N, H, W, seed=H + W)
    return x.cuda(), y.cuda()


@pytest.mark.parametrize('N,H,W', [(1, 128, 256), (1, 512, 1024), (1, 64, 2048)])
def test_vgg_loss_value_and_grad(N, H, W):
    """Width >= 256 keeps every level on the tensor-core gradient path; W = 2048 runs the downsample once."""
    crit = _vgg_loss()
    sd = {k: v.detach().cpu().double() for k, v in crit.vgg.state_dict().items()}
    x, y = _inputs(N, H, W)
    xr = x.clone().requires_grad_(True)
    loss = crit(xr, y)
    loss.backward()
    xo = x.cpu().double().requires_grad_(True)
    ref, per = VO.vgg_loss(sd, xo, y.cpu().double(), levels=True)
    ref.backward()
    with torch.no_grad():
        xs, ys = x, y
        while xs.shape[3] > 1024:
            xs, ys = ops.avgpool2(xs), ops.avgpool2(ys)
        levels = crit.vgg.feature_l1(xs, ys)
    for k in range(5):
        print('level %d ours %.8f oracle %.8f rel %.2e' % (k, levels[k].item(), per[k].item(), abs(levels[k].item() / per[k].item() - 1)))
        assert abs(levels[k].item() - per[k].item()) <= TOL_PRECISE * per[k].item(), k
    print('loss ours %.8f oracle %.8f' % (loss.item(), ref.item()))
    assert abs(loss.item() - ref.item()) <= TOL_PRECISE * ref.item()
    # (1) Against the fp64 backward taken with OUR forward's L1 signs, ReLU gates and max-pool argmaxes: the backward is
    # then a fixed linear map, and ours must match it to fp32-class rounding (the suite's shallow-unit criterion).  This
    # fails if any one level's term is lost (dropping relu1_1's alone moves the gradient by ~2 % in relative L2).
    xd = x.cpu().double().requires_grad_(True)
    xd_s = xd
    while xd_s.shape[3] > 1024:
        xd_s = F.avg_pool2d(xd_s, 2, 2)
    xd_s.backward(_masked_backward(crit.vgg, xs, ys))
    _cmp('vgg input grad %dx%d (our masks)' % (H, W), xr.grad, xd.grad)
    # (2) Against fp64 autograd of the oracle, with the suite's flip-tolerant criterion for chains deeper than ~4 layers: an
    # L1 sign, ReLU gate or argmax that falls on the other side in the oracle moves the gradient upstream of it.
    _cmp('vgg input grad %dx%d (oracle)' % (H, W), xr.grad, xo.grad, tol=None, l2=8e-2)
    assert all(p.grad is None for p in crit.vgg.parameters())


def test_vgg_loss_deterministic_and_recompute():
    """Two calls on one plan give the same bits; the backward of the first call, whose plan ran again in between on OTHER
    inputs, re-executes its forward and yields the gradient a lone call yields."""
    crit = _vgg_loss()
    x, y = _inputs(1, 128, 256)
    x2, _ = _inputs(1, 128, 257)
    x2 = x2[..., :256].contiguous()
    xr = x.clone().requires_grad_(True)
    a = crit(xr, y)
    a.backward()
    alone = xr.grad.clone()
    xr.grad = None
    a2 = crit(xr, y)
    b = crit(x2.clone().requires_grad_(True), y)                      # same plan, other input, run after a2
    assert torch.equal(a, a2)
    a2.backward()
    assert (xr.grad - alone).abs().max().item() <= 1e-6 * alone.abs().max().item()
    assert all(p.grad is None for p in crit.vgg.parameters())


def test_vgg_loss_fast():
    crit = _vgg_loss('fast')
    sd = {k: v.detach().cpu().double() for k, v in crit.vgg.state_dict().items()}
    x, y = _inputs(1, 128, 256)
    loss = crit(x, y)
    ref = VO.vgg_loss(sd, x.cpu().double(), y.cpu().double())
    print('fast loss %.6f oracle %.6f' % (loss.item(), ref.item()))
    assert abs(loss.item() - ref.item()) <= TOL_FAST * ref.item()


def test_vgg_features_forward():
    crit = _vgg_loss()
    sd = {k: v.detach().cpu().double() for k, v in crit.vgg.state_dict().items()}
    x, _ = _inputs(1, 64, 256)
    with torch.no_grad():
        ours = crit.vgg(x)
    ref = VO.features(sd, x.cpu().double())
    for k, (a, b) in enumerate(zip(ours, ref)):
        assert a.shape == b.shape
        _cmp('relu%d_1' % (k + 1), a, b, tol=TOL_PRECISE, l2=TOL_PRECISE)


def _setup(no_vgg, H=64, W=128, seed=3):
    """tests/test_gpu_train_step.py's small two-scale configuration, with the VGG term on or off (built by
    Vid2VidModelD.initialize itself)."""
    from vid2vid_b200 import flownet as FN
    from vid2vid_b200.model_d import Vid2VidModelD
    from vid2vid_b200.model_g import Vid2VidModelG
    from vid2vid_b200.utils import det_fill_, make_opt, synth_label_sequence
    torch.manual_seed(0)                       # (FlowNet2's weights are random-initialised)
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=2, ngf=16, n_downsample_G=2, n_blocks=4,
                   n_blocks_local=2, num_D=2, ndf=16, n_scales_temporal=2, isTrain=True, no_vgg=no_vgg, gpu_ids=[0], n_frames_total=12,
                   dataroot='datasets/Cityscapes/')
    G = Vid2VidModelG().initialize(opt)
    D = Vid2VidModelD().initialize(opt)
    for s in range(2):
        det_fill_(getattr(G, 'netG%d' % s), seed=seed + s)
    det_fill_(D.netD, seed=seed + 10)
    for s in range(2):
        det_fill_(getattr(D, 'netD_T%d' % s), seed=seed + 20 + s)
    flow = FN.FlowNet().initialize(opt)
    g = torch.Generator().manual_seed(seed)
    T = 8
    A = synth_label_sequence(T, H, W, label_nc=35, block=8, seed=seed)
    coarse = torch.rand(1, T, 3, H // 8, W // 8, generator=g) * 2 - 1
    B = F.interpolate(coarse.view(T, 3, H // 8, W // 8), size=(H, W), mode='bilinear', align_corners=False).view(1, T, 3, H, W)
    return opt, G, D, flow, A, B


def test_train_step_with_vgg():
    """Trainer step with the VGG term (fg on, so fake_B_raw adds the second term, and its call shares the fake_B call's plan:
    the fake_B backward re-executes that plan's forward).  The other eight losses are bit-identical to a no_vgg run, G_VGG
    and the generator gradients match the oracle (Vid2VidModelG / Vid2VidModelD.forward restated, plus oracle/vgg_oracle.py)
    with tests/test_gpu_train_step.py's criteria, and the VGG weights get no gradient."""
    from oracle import flownet2_oracle as FO
    from oracle import generator_oracle as GO
    from oracle import losses_oracle as LO
    from vid2vid_b200.trainer import Trainer
    res = {}
    for no_vgg in (True, False):
        opt, G, D, flow, A, B = _setup(no_vgg)
        assert hasattr(D, 'criterionVGG') == (not no_vgg)
        tr = Trainer(opt, G, D, flow, world=1)
        tG = opt.n_frames_G
        a, b = A[:, :tG].cuda(), B[:, :tG].cuda()
        loss_G, loss_D, _, ld, _ = tr.losses(a, b, a)
        tr.grads.zero()
        loss_G.backward()
        res[no_vgg] = ({k: float(v.detach()) for k, v in ld.items()}, opt, G, D, flow, A, B)
    ld0, ld1 = res[True][0], res[False][0]
    for n in ld0:
        if n != 'G_VGG':
            assert ld0[n] == ld1[n], n
    assert ld0['G_VGG'] == 0 and ld1['G_VGG'] > 0
    _, opt, G, D, flow, A, B = res[False]
    assert all(p.grad is None for p in D.criterionVGG.vgg.parameters())
    gG = {'%d.%s' % (s, n): q.grad.detach().cpu().double().clone() for s in range(2) for n, q in getattr(G, 'netG%d' % s).named_parameters()}

    # ---- oracle (as tests/test_gpu_train_step.py, plus the VGG term of vid2vid_model_D.py:136,143-144)
    tG = opt.n_frames_G
    sds = [{k: v.detach().cpu().clone().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
            for k, v in getattr(G, 'netG%d' % s).state_dict().items()} for s in range(2)]
    sdD = {k: v.detach().cpu().clone() for k, v in D.netD.state_dict().items()}
    sdF = {k: v.detach().cpu() for k, v in flow.flowNet.state_dict().items()}
    sdV = {k: v.detach().cpu().clone() for k, v in D.criterionVGG.vgg.state_dict().items()}
    fake_B, raws, flows, weights, real_A, real_Bp, _ = GO.ModelGOracle(opt, sds).train_forward(A[:, :tG], B[:, :tG], A[:, :tG], None,
                                                                                               n_frames_load=1)
    real_B_prev, real_B = real_Bp[:, :-1], real_Bp[:, 1:]
    with torch.no_grad():
        flow_ref, conf_ref = FO.flow_and_conf(sdF, real_B[:, 0], real_B_prev[:, 0])
    m = lambda t: t.reshape(-1, *t.shape[2:])
    lo = LO.spatial_losses(sdD, m(real_B), m(fake_B), m(raws), m(real_A), m(real_B_prev), m(real_B_prev[:, 0:1]), m(flows), m(weights),
                           flow_ref, conf_ref, lambda_F=opt.lambda_F, lambda_T=opt.lambda_T, lambda_feat=opt.lambda_feat,
                           n_scales_spatial=2, no_first_img=False, num_D=opt.num_D, n_layers_D=opt.n_layers_D, norm=opt.norm)
    od = dict(zip(D.loss_names, [torch.mean(x) for x in lo]))
    od['G_VGG'] = opt.lambda_feat * (VO.vgg_loss(sdV, m(fake_B), m(real_B)) + VO.vgg_loss(sdV, m(raws), m(real_B)))
    print('G_VGG ours %.6f oracle %.6f' % (ld1['G_VGG'], od['G_VGG'].item()))
    assert abs(ld1['G_VGG'] - od['G_VGG'].item()) <= 2e-3 * max(1.0, abs(od['G_VGG'].item()))
    oG = od['G_GAN'] + od['G_GAN_Feat'] + od['G_VGG'] + od['G_Warp'] + od['F_Flow'] + od['F_Warp'] + od['W']
    oG.backward()
    ref_gG = {'%d.%s' % (s, k): v.grad.double().clone() for s in range(2) for k, v in sds[s].items() if v.grad is not None}
    rels = []
    gmax = max(r.abs().max().item() for r in ref_gG.values())
    for k, r in ref_gG.items():
        if r.abs().max().item() < 1e-9 or (k.endswith('.bias') and gG[k].abs().max().item() == 0 and r.abs().max().item() < 1e-5 * gmax):
            continue          # conv bias in front of a norm layer: exactly zero here, rounding noise in the reference
        rel = ((gG[k] - r).norm() / r.norm()).item()
        rels.append(rel)
        assert rel <= 0.15, (k, rel)
    rels.sort()
    print('G gradients with VGG: %d tensors, median rel L2 %.2e, max %.2e' % (len(rels), rels[len(rels) // 2], rels[-1]))
    assert rels[len(rels) // 2] <= 3e-2
