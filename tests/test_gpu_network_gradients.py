"""Whole-network and training-step gradients against fp64 autograd of the oracle, with the gate flips taken out, so that the
composition of the backward kernels -- the plan backward's wiring (addend gradients, stacked stems and head pairs, the
composite, coarse-feature and img_prev exports), the loss wiring of Vid2VidModelD / Trainer (weights, detach points, which
tensor feeds which term) and the accumulation over discriminator scales, temporal scales and frames -- is held to fp32-class
bounds instead of tests/test_gpu_backward.py's flip-tolerant ones.

Flips.  The precise forward differs from fp64 by ~6e-5, so roughly one ReLU gate per layer output, and one kink of |a - b| per
L1 term, sits on the other side of zero; each moves the gradients upstream of it by 1-2 %.  Two things remove them:
  * gate-free networks: every ReLU and LeakyReLU of the generators and discriminators becomes LeakyReLU(1.0), the identity with
    gradient 1 on both sides of zero -- in the engine through a proxy of the Plan their descriptions are lowered onto (ResNet
    blocks pass ACT_RELU by hand), in the oracle through its `F`.  Tanh and sigmoid heads stay: they are smooth.  FlowNet2 keeps
    its LeakyReLU(0.1): it runs without a gradient and its flows are an input of the losses.
  * L1 signs pinned to the engine's: every ops.l1_loss call of the engine is recorded, and each L1 site of the oracle
    (losses_oracle.l1_mean) takes the sign pattern of the engine call whose operands it matches, read from the engine's own
    backward kernel (d/da of mean |a m - b m| is sign * m / numel).
The oracle reads the engine's reference flow and confidence (FlowNet2 is tested on its own; a confidence pixel on the other
side of its threshold would be a flip of another kind).  What remains non-smooth is the bilinear warp's cell boundaries,
which the low-pass images of these cases make nearly smooth.

Bounds.  A precise-mode conv carries its operands as hi + lo bf16 (relative representation error <= 2^-17 each) and drops
lo * lo (<= 2^-18): eps = 2 * 2^-17 + 2^-18 ~= 1.9e-5 relative per layer (tests/test_gpu_vgg.py).  A parameter gradient is the
product of a forward activation and a back-propagated gradient; the forward reaches it through at most L conv layers and the
backward through at most L more, where L is the longest conv chain from the network's input to the loss.  Linear
accumulation gives 2 L eps; that is the bound.  Independent errors add as sqrt(2 L) eps, and the factor sqrt(2 L) >= 4
between the two is what the norm backward's cancellation may use: it subtracts each channel's mean and its x-hat component
from dy, so its result carries the error of dy relative to |dy| while it can be several times smaller.  L per case:
  generators   stem + downsampling + residual convs + upsampling + head along the longest branch (CompositeGenerator:
               1 + nd + 2 * (n_blocks - n_blocks // 2) + 2 * (n_blocks // 2) + nd + 1; local: 2 + 2 * n_blocks_local + 2)
  D            n_layers + 2 convs per tower
  steps        G0 + G1 + D (the generated frame feeds the discriminator); the two-frame step adds one more G0 + G1 through
               the previous frame; the temporal step is netD_T's alone.
A discriminator's gradient from loss_D is the sum of a real and a fake pass, whose gradients point against each other; each
carries its own error, so N passes get N times the bound: 4 for netD (it judges fake_B and fake_B_raw), 2 for netD_f and netD_T.
Every case prints its worst ratio of error to bound.  Conv biases that feed a norm layer have an exact gradient of zero: ours
must be exactly zero, the oracle's rounding noise is not compared."""
import contextlib

import pytest
import torch
import torch.nn.functional as TF

import cases as C
import test_gpu_face_disc as FDT
import test_gpu_train_step as TS
from oracle import face_disc_oracle as FD
from oracle import generator_oracle as GO
from oracle import losses_oracle as LO
from oracle.bptt_oracle import BPTTModelGOracle
from oracle.make_golden import coarse_feats
from vid2vid_b200 import _lib as L
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import networks as NW
from vid2vid_b200 import ops
from vid2vid_b200.plan import Plan
from vid2vid_b200.trainer import Trainer
from vid2vid_b200.utils import det_fill_

EPS_LAYER = 2 * 2 ** -17 + 2 ** -18
GATED = (NW.CompositeGenerator, NW.MultiscaleDiscriminator)      # CompositeLocalGenerator is a CompositeGenerator
G_TERMS = ('G_GAN', 'G_GAN_Feat', 'G_VGG', 'G_Warp', 'F_Flow', 'F_Warp', 'W')


def bound(L_convs, passes=1):
    return 2 * passes * L_convs * EPS_LAYER


def _g_depth(c):
    if c['kind'] == 'compositeLocal':
        return 2 + 2 * c['n_blocks_local'] + 2
    return 1 + c['nd'] + 2 * c['n_blocks'] + c['nd'] + 1


def _step_depth(opt):
    g0 = 1 + opt.n_downsample_G + 2 * opt.n_blocks + opt.n_downsample_G + 1
    g1 = 2 + 2 * opt.n_blocks_local + 2
    return g0 + (opt.n_scales_spatial - 1) * g1, opt.n_layers_D + 2


# ------------------------------------------------------------------------------------------------ gate-free harness
class _GateFreePlan:
    """A Plan whose ReLU / LeakyReLU epilogues are LeakyReLU(1.0); counts the remaps."""

    def __init__(self, plan, remaps):
        self._plan, self._remaps = plan, remaps

    def __getattr__(self, name):
        return getattr(self._plan, name)

    def _act(self, act, slope):
        if act in (L.ACT_RELU, L.ACT_LRELU):
            self._remaps[0] += 1
            return L.ACT_LRELU, 1.0
        return act, slope

    def norm_act(self, raw, ndesc, act=L.ACT_NONE, slope=0.0, *rest, **kw):
        return self._plan.norm_act(raw, ndesc, *self._act(act, slope), *rest, **kw)

    def conv_act(self, vin, desc, act=L.ACT_NONE, slope=0.0):
        return self._plan.conv_act(vin, desc, *self._act(act, slope))


class _GateFreeF:
    """torch.nn.functional with relu and leaky_relu replaced by the identity."""

    @staticmethod
    def relu(x, inplace=False):
        return x

    @staticmethod
    def leaky_relu(x, negative_slope=0.01, inplace=False):
        return x

    def __getattr__(self, name):
        return getattr(TF, name)


@pytest.fixture
def gate_free(monkeypatch):
    """Gate-free generators and discriminators on both sides; yields the engine's remap count."""
    remaps = [0]
    get_plan = NW._Planned._get_plan

    def _get_plan(self, key, device, build, train=False):
        # gate-free plans are cached under a key of their own, so a plan built with real gates is never reused
        if isinstance(self, GATED):
            return get_plan(self, ('gate_free',) + key, device, lambda p: build(_GateFreePlan(p, remaps)), train)
        return get_plan(self, key, device, build, train)

    monkeypatch.setattr(NW._Planned, '_get_plan', _get_plan)
    monkeypatch.setattr(GO, 'F', _GateFreeF())
    monkeypatch.setattr(FD, 'F', _GateFreeF())
    return remaps


class _L1Pins:
    """Records the engine's ops.l1_loss calls and hands each L1 site of the oracle the sign pattern of its engine call."""

    def __init__(self, l1):
        self.l1, self.calls, self.used = l1, [], set()

    def __call__(self, a, b=None, mask=None):
        keep = lambda t: t.detach().clone() if t is not None else None
        self.calls.append((keep(a), keep(b), keep(mask)))
        return self.l1(a, b, mask)

    def clear(self):
        self.calls, self.used = [], set()

    def sign(self, a, b):
        """a, b: the oracle's operands, mask applied.  Pairs them with the engine call whose masked operands agree to forward
        precision and far better than any other call's; each engine call serves one oracle site."""
        dist = []
        scale = (a.norm() + b.norm()).item()
        for i, (ea, eb, em) in enumerate(self.calls):
            if ea.shape != a.shape:
                continue
            m = em.double().cpu() if em is not None else 1.0
            ea64 = ea.double().cpu() * m
            eb64 = eb.double().cpu() * m if eb is not None else torch.zeros_like(ea64)
            dist.append((((ea64 - a).norm() + (eb64 - b).norm()).item() / max(scale, 1e-30), i))
        dist.sort()
        assert dist and dist[0][0] <= 2e-3, ('no engine L1 call matches an oracle site', tuple(a.shape), dist[:3])
        assert len(dist) == 1 or dist[1][0] >= 10 * dist[0][0], ('ambiguous L1 pairing', tuple(a.shape), dist[:3])
        i = dist[0][1]
        assert i not in self.used, ('two oracle L1 sites pair with one engine call', i)
        self.used.add(i)
        ea, eb, em = self.calls[i]
        x = ea.clone().requires_grad_(True)
        g, = torch.autograd.grad(self.l1(x, eb, em), x)
        return torch.sign(g).double().cpu()


@pytest.fixture
def l1_pins(monkeypatch):
    pins = _L1Pins(ops.l1_loss)
    monkeypatch.setattr(ops, 'l1_loss', pins)
    monkeypatch.setattr(LO, 'L1_SIGN', pins.sign)
    return pins


# ------------------------------------------------------------------------------------------------ helpers
@contextlib.contextmanager
def _fp64():
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(torch.float32)


def _leaf(net, dtype=torch.float64):
    """The oracle's state dict of `net`: floating tensors in `dtype`, weights and biases asking for a gradient."""
    return {k: v.detach().cpu().to(dtype).requires_grad_(k.rsplit('.', 1)[-1] in ('weight', 'bias')) if v.dtype.is_floating_point
            else v.detach().cpu() for k, v in net.state_dict().items()}


def _grads(sd, prefix=''):
    return {prefix + k: (v.grad if v.grad is not None else torch.zeros_like(v)).to(torch.float64, copy=True) for k, v in sd.items()
            if v.requires_grad}


def _ours(net, prefix=''):
    return {prefix + n: (p.grad if p.grad is not None else torch.zeros_like(p)).detach().cpu().double().clone()
            for n, p in net.named_parameters()}


def _vanishing(net, prefix=''):
    """The first norm layer's bias of every ResNet block: in a gate-free network its output reaches the rest only through a
    reflect-padded conv (a per-channel constant stays constant) and the block's second norm (which subtracts it), so its
    exact gradient is zero."""
    return {'%s%s.conv_block.2.bias' % (prefix, n) for n, m in net.named_modules() if isinstance(m, NW.ResnetBlock)}


def _check(what, ours, ref, lim, zero=(), vanishing=()):
    """Every tensor within `lim` relative L2 of the fp64 oracle; the biases in `zero` exactly zero; those in `vanishing`
    (exact gradient zero, ours the rounding residue of a per-channel sum that cancels) within `lim` of the norm of the same
    layer's weight gradient."""
    worst, bad, n = (0.0, ''), [], 0
    for k, r in ref.items():
        o = ours[k]
        assert o.shape == r.shape and torch.isfinite(o).all(), (what, k)
        if k in zero:
            assert o.abs().max().item() == 0, (what, k, 'bias in front of a norm layer')
            continue
        rn = r.norm().item()
        if k in vanishing:
            rn = ref[k[:-len('bias')] + 'weight'].norm().item()
            r = torch.zeros_like(r)
        rel = (o - r).norm().item() / rn if rn > 0 else (0.0 if o.abs().max().item() == 0 else float('inf'))
        n += 1
        worst = max(worst, (rel / lim, k))
        if rel > lim:
            bad.append('%s %.2e' % (k, rel))
    print('%s: %d tensors, bound %.2e, worst error/bound %.3f (%s)' % (what, n, lim, worst[0], worst[1]))
    assert n and not bad, (what, bad[:6])
    return worst[0]


def _capture(D):
    """Records the tensor lists Vid2VidModelD.forward receives, by temporal scale."""
    caps, fwd = {}, D.forward

    def forward(scale_T, tensors_list, *a, **kw):
        caps[scale_T] = [t.detach().clone() if t is not None else None for t in tensors_list]
        return fwd(scale_T, tensors_list, *a, **kw)
    D.forward = forward
    return caps


# ------------------------------------------------------------------------------------------------ generators and D
GEN_CASES = ['g0_small', 'g0_small_ac', 'g0_nofg_nd2', 'g0_noflow', 'gl_small_s1', 'gl_small_s2']


def _run_oracle_g(c, sd, inp, img_prev, mask, coarse, ac):
    if c['kind'] == 'compositeLocal':
        return GO.composite_local_generator(sd, inp, img_prev, mask, *coarse, False, n_blocks_local=c['n_blocks_local'],
                                            use_fg_model=c['fg'], scale=c['scale'], align_corners=ac)
    return GO.composite_generator(sd, inp, img_prev, mask, False, n_downsampling=c['nd'], n_blocks=c['n_blocks'],
                                  use_fg_model=c['fg'], no_flow=c['no_flow'], align_corners=ac)


def _oracle_g(c, net, inp, img_prev, mask, coarse, gs, ac, dtype):
    sd = _leaf(net, dtype)
    p = img_prev.detach().to(dtype, copy=True).requires_grad_(True)
    cf = [t.detach().to(dtype, copy=True).requires_grad_(True) if t is not None else None for t in coarse]
    with (_fp64() if dtype == torch.float64 else contextlib.nullcontext()):
        out = _run_oracle_g(c, sd, inp.to(dtype), p, mask.to(dtype), cf, ac)
        sum((o * g.to(dtype)).sum() for o, g in zip(out, gs) if o is not None).backward()
    ref = _grads(sd)
    ref['input img_prev'] = p.grad.double()
    for i, t in enumerate(cf):
        if t is not None:
            ref['input coarse feature %d' % i] = t.grad.double()
    return ref


def _floor(what, r32, r64):
    top = max(r.norm().item() for r in r64.values())
    rels = sorted(((r32[k] - r).norm() / r.norm()).item() for k, r in r64.items() if r.norm() > 1e-9 * top)
    print('%s fp32-oracle vs fp64-oracle gradient rel L2: max %.2e median %.2e' % (what, rels[-1], rels[len(rels) // 2]))


@pytest.mark.gpu
@pytest.mark.parametrize('name', GEN_CASES)
def test_generator_gradients_gate_free(name, gate_free):
    """Every parameter, img_prev and coarse-feature gradient of one generator under random cotangents on all seven outputs."""
    c = C.CASES[name]
    ac = c.get('align_corners', False)
    net = det_fill_(C.build_module(c), seed=c['seed'])
    inp, img_prev, mask = C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed'], block=c.get('block', 4))
    coarse = tuple(coarse_feats(c)) if c['kind'] == 'compositeLocal' else (None, None, None)
    gs = [torch.randn(1, ch, c['h'], c['w'], generator=torch.Generator().manual_seed(20 + i)) for i, ch in
          enumerate((3, 2, 1, 3, c['ngf'], c['ngf'], c['ngf'] // 2 if c['nd'] > 2 else c['ngf']))]
    ref = _oracle_g(c, net, inp, img_prev, mask, coarse, gs, ac, torch.float64)
    _floor(name, _oracle_g(c, net, inp, img_prev, mask, coarse, gs, ac, torch.float32), ref)
    zero, vanishing = FDT._biases_before_norm(net), _vanishing(net)
    net = net.cuda()
    net.precision, net.align_corners = 'precise', ac
    pg = img_prev.cuda().requires_grad_(True)
    cg = [t.cuda().requires_grad_(True) if t is not None else None for t in coarse]
    out = net(inp.cuda(), pg, mask.cuda(), *cg, False)
    sum((o * g.cuda()).sum() for o, g in zip(out, gs) if o is not None).backward()
    assert gate_free[0] > 0
    ours = _ours(net)
    ours['input img_prev'] = pg.grad.cpu().double()
    for i, t in enumerate(cg):
        if t is not None:
            ours['input coarse feature %d' % i] = t.grad.cpu().double()
    _check(name, ours, ref, bound(_g_depth(c)), zero, vanishing)


@pytest.mark.gpu
def test_multiscale_discriminator_gradients_gate_free(gate_free):
    """D_small (three towers, every intermediate feature an output): parameter and input gradients."""
    c = C.CASES['D_small']
    net = det_fill_(C.build_module(c), seed=c['seed'])
    x = torch.randn(c['batch'], c['input_nc'], c['h'], c['w'], generator=torch.Generator().manual_seed(c['seed'] + 1))
    refs, gs = {}, None
    for dtype in (torch.float64, torch.float32):
        sd = _leaf(net, dtype)
        xd = x.detach().to(dtype, copy=True).requires_grad_(True)
        with (_fp64() if dtype == torch.float64 else contextlib.nullcontext()):
            out = GO.multiscale_discriminator(sd, xd, num_D=c['num_D'], n_layers=c['n_layers'], norm='batch', getIntermFeat=True)
            if gs is None:
                gs = [[torch.randn(t.shape, generator=torch.Generator().manual_seed(100 + 10 * i + j)) for j, t in enumerate(tw)]
                      for i, tw in enumerate(out)]
            sum((t * g.to(dtype)).sum() for tw, gw in zip(out, gs) for t, g in zip(tw, gw)).backward()
        refs[dtype] = dict(_grads(sd), **{'input': xd.grad.double()})
    _floor('D_small', refs[torch.float32], refs[torch.float64])
    zero = FDT._biases_before_norm(net)
    net = net.cuda()
    net.precision = 'precise'
    xg = x.cuda().requires_grad_(True)
    out = net(xg)
    sum((t * g.float().cuda()).sum() for tw, gw in zip(out, gs) for t, g in zip(tw, gw)).backward()
    ours = dict(_ours(net), input=xg.grad.cpu().double())
    _check('D_small', ours, refs[torch.float64], bound(c['n_layers'] + 2), zero)


# ------------------------------------------------------------------------------------------------ training steps
def _engine_step(opt, G, D, flow, A, B, T, face):
    """Trainer.losses over T input frames, then loss_G and loss_D backward as Trainer.step does."""
    caps = _capture(D)
    tr = Trainer(opt, G, D, flow, world=1)
    a, b = A[:, :T].cuda(), B[:, :T].cuda()
    loss_G, loss_D, loss_D_T, ld, _ = tr.losses(a, b, a)
    assert not loss_D_T
    tr.grads.zero()
    loss_G.backward()
    ours = {'G': {k: v for s in range(opt.n_scales_spatial) for k, v in _ours(getattr(G, 'netG%d' % s), '%d.' % s).items()}}
    tr.grads.zero(1)
    loss_D.backward()
    ours['D'] = _ours(D.netD)
    if face:
        ours['D_f'] = _ours(D.netD_f)
    return ours, ld, caps[0]


def _oracle_step(opt, G, D, A, B, T, cap, face, n_frames_bp=None, dtype=torch.float64):
    """The same step by the oracle chain of tests/test_gpu_train_step.py (with tests/test_gpu_bptt.py's detach points and
    tests/test_gpu_face_disc.py's face terms), on the engine's reference flow and confidence."""
    S, tG = opt.n_scales_spatial, opt.n_frames_G
    sds = [_leaf(getattr(G, 'netG%d' % s), dtype) for s in range(S)]
    sdD = _leaf(D.netD, dtype)
    sdDf = _leaf(D.netD_f, dtype) if face else None
    m = lambda t: t.reshape(-1, *t.shape[2:]) if t is not None else None
    with (_fp64() if dtype == torch.float64 else contextlib.nullcontext()):
        a, b = A[:, :T].to(dtype), B[:, :T].to(dtype)
        fake_B, raws, flows, weights, real_A, real_Bp, _ = BPTTModelGOracle(opt, sds).train_forward(
            a, b, a, None, n_frames_load=T - tG + 1, n_frames_bp=n_frames_bp)
        real_B_prev, real_B = real_Bp[:, :-1], real_Bp[:, 1:]
        fake_B_prev = torch.cat([real_B_prev[:, 0:1], fake_B[:, :-1].detach()], dim=1)            # compute_fake_B_prev
        flow_ref, conf_ref = cap[8].cpu().to(dtype), cap[9].cpu().to(dtype)
        inputs = [m(real_B), m(fake_B), m(raws), m(real_A), m(real_B_prev), m(fake_B_prev), m(flows), m(weights), flow_ref, conf_ref]
        if face:
            lo = FD.face_disc_losses(sdD, sdDf, FD.running_stats({k: v.detach() for k, v in sdDf.items()}), inputs, opt)
        else:
            lo = LO.spatial_losses(sdD, *inputs, lambda_F=opt.lambda_F, lambda_T=opt.lambda_T, lambda_feat=opt.lambda_feat,
                                   n_scales_spatial=S, no_first_img=opt.no_first_img, num_D=opt.num_D, n_layers_D=opt.n_layers_D,
                                   norm=opt.norm)
        od = dict(zip(D.loss_names, [torch.mean(x) for x in lo]))
        terms = G_TERMS + (('G_f_GAN', 'G_f_GAN_Feat') if face else ())
        sum(od[n] for n in terms).backward(retain_graph=True)
        ref = {'G': {k: v for s in range(S) for k, v in _grads(sds[s], '%d.' % s).items()}}
        for v in list(sdD.values()) + (list(sdDf.values()) if face else []):
            v.grad = None
        oD = (od['D_fake'] + od['D_real']) * 0.5
        if face:
            oD = oD + (od['D_f_fake'] + od['D_f_real']) * 0.5
        oD.backward()
    ref['D'] = _grads(sdD)
    if face:
        ref['D_f'] = _grads(sdDf)
    return ref, od


def _compare_step(what, opt, G, D, ours, ref, ld, od, extra_G=0, ref32=None):
    if ref32 is not None:
        for k in ref:
            _floor('%s %s' % (what, k), ref32[k], ref[k])
    for n in D.loss_names:
        print('%-13s ours %.6f oracle %.6f' % (n, float(ld[n]), float(od[n])))
    g_depth, d_depth = _step_depth(opt)
    zero = {'G': set().union(*(FDT._biases_before_norm(getattr(G, 'netG%d' % s), '%d.' % s) for s in range(opt.n_scales_spatial))),
            'D': FDT._biases_before_norm(D.netD)}
    if 'D_f' in ours:
        zero['D_f'] = FDT._biases_before_norm(D.netD_f)
    vanishing = set().union(*(_vanishing(getattr(G, 'netG%d' % s), '%d.' % s) for s in range(opt.n_scales_spatial)))
    worst = [_check('%s G' % what, ours['G'], ref['G'], bound((1 + extra_G) * g_depth + d_depth), zero['G'], vanishing)]
    for k in ('D', 'D_f'):
        if k in ours:
            # loss_D sums a real and a fake pass per discriminator call: two calls of netD (fake_B and fake_B_raw), one of netD_f
            worst.append(_check('%s %s' % (what, k), ours[k], ref[k], bound(d_depth, passes=4 if k == 'D' else 2), zero[k]))
    print('%s: worst error/bound %.3f' % (what, max(worst)))


@pytest.mark.gpu
def test_first_training_step_gradients_gate_free(gate_free, l1_pins):
    """The cfg3-geometry first step of tests/test_gpu_train_step.py: every G parameter of both scales from loss_G and every
    netD parameter from loss_D."""
    opt, G, D, flow, A, B = TS._setup()
    T = opt.n_frames_G
    ours, ld, cap = _engine_step(opt, G, D, flow, A, B, T, face=False)
    ref, od = _oracle_step(opt, G, D, A, B, T, cap, face=False)
    assert l1_pins.used
    l1_pins.used = set()
    ref32, _ = _oracle_step(opt, G, D, A, B, T, cap, face=False, dtype=torch.float32)
    _compare_step('first step', opt, G, D, ours, ref, ld, od, ref32=ref32)


@pytest.mark.gpu
def test_two_frame_bptt_step_gradients_gate_free(gate_free, l1_pins):
    """tests/test_gpu_bptt.py's two-frame step with n_frames_bp 2: the second frame's gradient reaches both generators again
    through the first generated frame."""
    opt, G, D, flow, A, B = TS._setup()
    for s in range(2):
        C.condition_flow_heads(getattr(G, 'netG%d' % s), 0.05)
    opt.max_frames_per_gpu, opt.max_frames_backpropagate = 2, 2
    G.init_train()
    G.n_frames_bp = 2
    T = opt.n_frames_G + 1
    ours, ld, cap = _engine_step(opt, G, D, flow, A, B, T, face=False)
    ref, od = _oracle_step(opt, G, D, A, B, T, cap, face=False, n_frames_bp=2)
    _compare_step('two-frame step', opt, G, D, ours, ref, ld, od, extra_G=1)


@pytest.mark.gpu
def test_pose_face_disc_step_gradients_gate_free(gate_free, l1_pins):
    """One pose step with --add_face_disc (tests/test_gpu_face_disc.py's setup, real first frames): G, netD and netD_f."""
    opt, G, D, flow, A, B = FDT._setup(False, no_first_img=False)
    T = opt.n_frames_G
    ours, ld, cap = _engine_step(opt, G, D, flow, A, B, T, face=True)
    assert FD.face_box(cap[3].cpu(), opt.openpose_only) is not None
    ref, od = _oracle_step(opt, G, D, A, B, T, cap, face=True)
    l1_pins.used = set()
    ref32, _ = _oracle_step(opt, G, D, A, B, T, cap, face=True, dtype=torch.float32)
    _compare_step('pose step', opt, G, D, ours, ref, ld, od, ref32=ref32)


@pytest.mark.gpu
def test_temporal_discriminator_gradients_gate_free(gate_free, l1_pins):
    """Trainer.step until the temporal discriminator runs; then the oracle's temporal losses on the engine's own frame groups
    and flows (detached) and netD_T0's gradient from loss_D_T, against the parameters it had before that step's update."""
    opt, G, D, flow, A, B = TS._setup(seed=5)
    tr = Trainer(opt, G, D, flow, world=1)
    caps = _capture(D)
    tG = opt.n_frames_G
    for i in range(A.shape[1] - tG + 1):
        sdT = _leaf(D.netD_T0)
        caps.clear()
        l1_pins.clear()
        ld, ldT = tr.step(A[:, i:i + tG].cuda(), B[:, i:i + tG].cuda(), A[:, i:i + tG].cuda())
        if ldT:
            break
    assert 1 in caps and 2 not in caps, 'the temporal discriminator never ran'
    ours = _ours(D.netD_T0)
    real, fake, flow_ref, conf_ref = [t.cpu().double() for t in caps[1]]
    with _fp64():
        lt = LO.temporal_losses(sdT, real, fake, flow_ref, conf_ref, n_frames_D=opt.n_frames_D, output_nc=opt.output_nc,
                                lambda_feat=opt.lambda_feat, num_D=opt.num_D, n_layers_D=opt.n_layers_D, norm=opt.norm)
        ((torch.mean(lt[3]) + torch.mean(lt[2])) * 0.5).backward()
    for n, v in zip(D.loss_names_T, lt):
        print('%-13s ours %.6f oracle %.6f' % (n, ldT[0][n], float(torch.mean(v))))
    _check('temporal step netD_T0', ours, _grads(sdT), bound(opt.n_layers_D + 2, passes=2), FDT._biases_before_norm(D.netD_T0))


# ------------------------------------------------------------------------------------------------ harness self-check (CPU)
def _acts(desc):
    out = []
    for group in ('epilogue_forward', 'epilogue_backward', 'layout'):
        for r in desc.get(group, ()):
            out += [r['act']] if 'act' in r else r.get('acts', [])
    return out


def test_gate_free_harness_takes_effect(gate_free, monkeypatch):
    """Lower every G / D plan of the cases above host-side through the fixture: no record applies ACT_RELU and the proxy
    counts a remap per ReLU / LeakyReLU, while FlowNet2's plans keep their LeakyReLU."""
    monkeypatch.setattr(Plan, 'finalize', lambda self, workspace=None: None)
    dev = torch.device('cuda', 0)
    describe = lambda net, key, build: net._get_plan(key, dev, build, train=True).describe()
    nets = []
    for name in GEN_CASES:
        c = C.CASES[name]
        nets.append((name, C.build_module(c), (1, c['h'], c['w'])))
    c = C.CASES['D_small']
    d = C.build_module(c)
    nets += [('D_small tower %d' % t, d, (t, c['batch'], c['h'] >> (d.num_D - 1 - t), c['w'] >> (d.num_D - 1 - t))) for t in range(d.num_D)]
    for tag, opt_, H, W, face in (('cfg3 step', _train_opt(), 64, 128, False), ('pose step', _pose_opt(), 128, 128, True)):
        for s, net in enumerate(NW.build_netGs(opt_)):
            nets.append(('%s G%d' % (tag, s), net, (1, H >> (1 - s), W >> (1 - s))))
        nc = (opt_.label_nc or opt_.input_nc) + int(opt_.use_instance)
        ds = [('D', NW.define_D(nc + 3, opt_.ndf, opt_.n_layers_D, opt_.norm, opt_.num_D, True, []), H, W),
              ('D_T', NW.define_D(3 * opt_.n_frames_D + 2 * (opt_.n_frames_D - 1), opt_.ndf, opt_.n_layers_D, opt_.norm, opt_.num_D,
                                  True, []), H, W)]
        if face:
            crop = opt_.fineSize // 32 * 8
            ds.append(('D_f', NW.define_D(nc + 3, opt_.ndf, opt_.n_layers_D, opt_.norm, max(1, opt_.num_D - 2), True, []), crop, crop))
        for dn, d, h, w in ds:
            for t in range(d.num_D):
                nets.append(('%s %s tower %d' % (tag, dn, t), d, (t, 1, h >> (d.num_D - 1 - t), w >> (d.num_D - 1 - t))))
    for tag, net, shape in nets:
        before = gate_free[0]
        acts = _acts(describe(net, ('selfcheck',) + shape, lambda p: net._describe(p, *shape)))
        assert gate_free[0] > before, tag
        assert L.ACT_RELU not in acts and L.ACT_LRELU in acts, (tag, acts)
    f = FN.FlowNet2()
    before = gate_free[0]
    for sub in ('flownetc', 'flownets_1', 'flownetfusion'):
        acts = _acts(f._sub_plan(sub, 1, 64, 64, dev).describe())
        assert L.ACT_LRELU in acts, sub
    assert gate_free[0] == before


def _train_opt():
    from vid2vid_b200.utils import make_opt
    return make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=2, ngf=16, n_downsample_G=2, n_blocks=4,
                    n_blocks_local=2, num_D=2, ndf=16, n_scales_temporal=2, isTrain=True, no_vgg=True, gpu_ids=[], n_frames_total=12,
                    dataroot='datasets/Cityscapes/')


def _pose_opt():
    from vid2vid_b200.utils import make_opt
    return make_opt(label_nc=0, input_nc=6, use_instance=False, fg=False, n_scales_spatial=2, ngf=16, n_downsample_G=2, n_blocks=4,
                    n_blocks_local=2, num_D=3, ndf=16, n_scales_temporal=2, isTrain=True, no_vgg=True, gpu_ids=[], n_frames_total=12,
                    no_first_img=False, add_face_disc=True, fineSize=256, dataroot='datasets/pose', dataset_mode='pose')
