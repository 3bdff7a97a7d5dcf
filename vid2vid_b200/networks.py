"""H100 drop-ins for the generator / discriminator modules of models/networks.py.

Each class keeps the reference's constructor signature, attribute names and state_dict keys
(index-based Sequential keys included, e.g. `model_down_img.4.weight`), so reference checkpoints load
unchanged (models/base_model.py:63-107) -- the torch.nn layers below are *parameter containers*
only.  forward() never calls them: it describes the network once per input shape to the plan
runtime (vid2vid_b200/plan.py -> libv2v_b200.so), which runs hand-written sm_90a kernels.
There is no PyTorch/cuDNN fallback.

Norm semantics (SURVEY App. B #1): Batch/InstanceNorm always use the statistics of the current
tensor, as the reference does at inference because it never calls .eval() on G/D.
"""
import copy
import functools
import os
import sys

import torch
import torch.nn as nn

from . import _lib as L
from .plan import Plan, conv_desc, norm_desc


# ------------------------------------------------------------------------------------ init / factories
def weights_init(m):
    """models/networks.py:15-21."""
    name = m.__class__.__name__
    if name.find('Conv') != -1 and hasattr(m, 'weight'):
        m.weight.data.normal_(0.0, 0.02)
    elif name.find('BatchNorm2d') != -1:
        m.weight.data.normal_(1.0, 0.02)
        m.bias.data.fill_(0)


def get_norm_layer(norm_type='instance'):
    """models/networks.py:23-30."""
    if norm_type == 'batch':
        return functools.partial(nn.BatchNorm2d, affine=True)
    if norm_type == 'instance':
        return functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=True)
    raise NotImplementedError('normalization layer [%s] is not found' % norm_type)


def define_G(input_nc, output_nc, prev_output_nc, ngf, which_model_netG, n_downsampling, norm, scale, gpu_ids=[],
             opt=[]):
    """models/networks.py:32-59 (`local_with_features` is not built: no vid2vid code path uses it)."""
    norm_layer = get_norm_layer(norm_type=norm)
    if which_model_netG == 'global':
        netG = GlobalGenerator(input_nc, output_nc, ngf, n_downsampling, opt.n_blocks, norm_layer)
    elif which_model_netG == 'local':
        netG = LocalEnhancer(input_nc, output_nc, ngf, n_downsampling, opt.n_blocks, opt.n_local_enhancers,
                             opt.n_blocks_local, norm_layer)
    elif which_model_netG == 'global_with_features':
        netG = Global_with_z(input_nc, output_nc, opt.feat_num, ngf, n_downsampling, opt.n_blocks, norm_layer)
    elif which_model_netG == 'encoder':
        netG = Encoder(input_nc, output_nc, ngf, n_downsampling, norm_layer)
    elif which_model_netG == 'local_with_features':
        raise NotImplementedError('Generator model name [local_with_features] (Local_with_z) is not implemented')
    elif which_model_netG == 'composite':
        netG = CompositeGenerator(opt, input_nc, output_nc, prev_output_nc, ngf, n_downsampling, opt.n_blocks,
                                  opt.fg, opt.no_flow, norm_layer)
    elif which_model_netG == 'compositeLocal':
        netG = CompositeLocalGenerator(opt, input_nc, output_nc, prev_output_nc, ngf, n_downsampling,
                                       opt.n_blocks_local, opt.fg, opt.no_flow, norm_layer, scale=scale)
    else:
        raise NotImplementedError('Generator model name [%s] is not recognized' % which_model_netG)
    if len(gpu_ids) > 0:
        netG.cuda(gpu_ids[0])
    netG.apply(weights_init)
    return netG


def define_D(input_nc, ndf, n_layers_D, norm='instance', num_D=1, getIntermFeat=False, gpu_ids=[]):
    """models/networks.py:61-68."""
    netD = MultiscaleDiscriminator(input_nc, ndf, n_layers_D, get_norm_layer(norm), num_D, getIntermFeat)
    if len(gpu_ids) > 0:
        netD.cuda(gpu_ids[0])
    netD.apply(weights_init)
    return netD


# ------------------------------------------------------------------------------------ layer containers
def _stem(cin, cout, norm_layer):
    return [nn.ReflectionPad2d(3), nn.Conv2d(cin, cout, kernel_size=7, padding=0), norm_layer(cout), nn.ReLU(True)]


def _down(cin, cout, norm_layer):
    return [nn.Conv2d(cin, cout, kernel_size=3, stride=2, padding=1), norm_layer(cout), nn.ReLU(True)]


def _up(cin, cout, norm_layer):
    return [nn.ConvTranspose2d(cin, cout, kernel_size=3, stride=2, padding=1, output_padding=1), norm_layer(cout),
            nn.ReLU(True)]


def _head(cin, cout, act=None):
    return [nn.ReflectionPad2d(3), nn.Conv2d(cin, cout, kernel_size=7, padding=0)] + ([act] if act else [])


class ResnetBlock(nn.Module):
    """Parameter container with the keys of models/networks.py:554-593 (`conv_block.{1,2,5,6}`)."""

    def __init__(self, dim, padding_type, norm_layer, activation=nn.ReLU(True), use_dropout=False):
        super().__init__()
        if padding_type != 'reflect' or use_dropout:
            raise NotImplementedError('only reflect padding without dropout is used by vid2vid')
        self.conv_block = nn.Sequential(nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, kernel_size=3, padding=0),
                                        norm_layer(dim), activation,
                                        nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, kernel_size=3, padding=0),
                                        norm_layer(dim))


# ------------------------------------------------------------------------------------ lowering helpers
_ACTS = {nn.ReLU: (L.ACT_RELU, 0.0), nn.Tanh: (L.ACT_TANH, 0.0), nn.Sigmoid: (L.ACT_SIGMOID, 0.0)}


def _act_of(m):
    if isinstance(m, nn.LeakyReLU):
        return L.ACT_LRELU, m.negative_slope
    for k, v in _ACTS.items():
        if isinstance(m, k):
            return v
    return None


def _units(mods):
    """Group a flat layer list into units: ('conv', conv, pad_mode, pad, norm, act, slope) | ('res', block)."""
    units, i, pend = [], 0, None
    mods = list(mods)
    while i < len(mods):
        m = mods[i]
        if isinstance(m, nn.ReflectionPad2d):
            pend = m.padding[0]
            i += 1
        elif isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            norm, act, slope = None, L.ACT_NONE, 0.0
            j = i + 1
            if j < len(mods) and isinstance(mods[j], (nn.BatchNorm2d, nn.InstanceNorm2d)):
                norm = mods[j]
                j += 1
            if j < len(mods) and _act_of(mods[j]) is not None:
                act, slope = _act_of(mods[j])
                j += 1
            if pend is not None:
                units.append(('conv', m, L.PAD_REFLECT, pend, norm, act, slope))
            else:
                units.append(('conv', m, L.PAD_ZERO, None, norm, act, slope))
            pend, i = None, j
        elif isinstance(m, ResnetBlock):
            units.append(('res', m))
            i += 1
        else:
            raise NotImplementedError('cannot lower layer %r' % (m,))
    return units


def emit_seq(plan, mods, v, final_adds=(), defer_last=False):
    """Describe a Sequential on `plan` starting from value `v`.  `final_adds` are value ids summed
    into the last unit's output (branch merges / coarse-feature skips are fused into that unit's
    normalise pass).  With defer_last the last unit's normalise step is returned as a closure
    finish(adds) -> value so the caller can emit it more than once with different addends."""
    units = _units(mods)
    finish = None
    for k, u in enumerate(units):
        last = k == len(units) - 1
        adds = tuple(final_adds) if last else ()
        if u[0] == 'conv':
            _, conv, pmode, pad, norm, act, slope = u
            desc = conv_desc(conv, pmode, pad)
            if norm is None:
                if adds or (last and defer_last):
                    raise NotImplementedError('addends need a normalised unit')
                v = plan.conv_act(v, desc, act, slope)
            else:
                raw = plan.conv(v, desc)
                nd = norm_desc(norm)
                if last and defer_last:
                    finish = (lambda raw=raw, nd=nd, act=act, slope=slope: (lambda a: plan.norm_act(raw, nd, act, slope, a)))()
                else:
                    v = plan.norm_act(raw, nd, act, slope, adds)
        else:
            cb = u[1].conv_block
            raw1 = plan.conv(v, conv_desc(cb[1], L.PAD_REFLECT, 1))
            h = plan.norm_act(raw1, norm_desc(cb[2]), L.ACT_RELU, 0.0)
            raw2 = plan.conv(h, conv_desc(cb[5], L.PAD_REFLECT, 1))
            nd = norm_desc(cb[6])
            if last and defer_last:
                finish = (lambda raw2=raw2, nd=nd, v0=v: (lambda a: plan.norm_act(raw2, nd, L.ACT_NONE, 0.0, (v0,) + tuple(a))))()
            else:
                v = plan.norm_act(raw2, nd, L.ACT_NONE, 0.0, (v,) + adds)
    if defer_last:
        if finish is None:
            raise NotImplementedError('defer_last on an empty sequence')
        return finish
    return v


def emit_head(plan, mods, v, dst):
    """[ReflectionPad2d(3), Conv2d 7x7, (Tanh|Sigmoid)] -> fp32 NCHW planes of caller tensor slot `dst`
    = (slot, dst_C, scale)."""
    (u,) = _units(mods)
    _, conv, pmode, pad, norm, act, slope = u
    assert norm is None
    slot, dst_c, scale = dst
    plan.head(v, conv_desc(conv, pmode, pad), [(slot, j, dst_c, act, scale) for j in range(conv.out_channels)])


def emit_head_pair(plan, mods_a, dst_a, mods_b, dst_b, v):
    """Two heads that read the same value (model_final_flow + model_final_w, networks.py:182-183,212-213) as ONE
    convolution with the weights stacked along Cout: halves the activation traffic of the 7x7 heads."""
    (ua,), (ub,) = _units(mods_a), _units(mods_b)
    _, ca, pmode, pad, na, act_a, _ = ua
    _, cb, pmode_b, pad_b, nb, act_b, _ = ub
    assert na is None and nb is None and (pmode, pad) == (pmode_b, pad_b)
    chans = [(dst_a[0], j, dst_a[1], act_a, dst_a[2]) for j in range(ca.out_channels)]
    chans += [(dst_b[0], j, dst_b[1], act_b, dst_b[2]) for j in range(cb.out_channels)]
    plan.head(v, conv_desc(ca, pmode, pad, m2=cb), chans)


def emit_unit_pair(plan, mods_a, mods_b, v):
    """First units of two branches that read the same value with the same geometry (the 7x7 stems model_down_seg.1 and
    indv_down.1, networks.py:132,153) as ONE convolution with stacked weights; each half keeps its own norm layer.
    The small-N 7x7 stems are MMA-issue bound (a narrow MMA costs nearly what a wider one does), so sharing the
    instructions halves their cost.  Returns (value_a, value_b)."""
    (ua,), (ub,) = _units(mods_a), _units(mods_b)
    _, ca, pmode, pad, na, act_a, slope_a = ua
    _, cb, pmode_b, pad_b, nb, act_b, slope_b = ub
    assert na is not None and nb is not None and (pmode, pad) == (pmode_b, pad_b)
    raw = plan.conv(v, conv_desc(ca, pmode, pad, m2=cb))
    va = plan.norm_act(raw, norm_desc(na), act_a, slope_a, c_off=0, Cn=ca.out_channels)
    vb = plan.norm_act(raw, norm_desc(nb), act_b, slope_b, c_off=ca.out_channels, Cn=cb.out_channels)
    return va, vb


def _can_pair(mods_a, mods_b):
    ca, cb = mods_a[1], mods_b[1]
    return (isinstance(ca, nn.Conv2d) and isinstance(cb, nn.Conv2d) and ca.in_channels == cb.in_channels and
            ca.kernel_size == cb.kernel_size and ca.stride == cb.stride and ca.out_channels % 8 == 0)


class _PlanFunction(torch.autograd.Function):
    """Autograd node of one plan execution: forward = v2v_plan_run, backward = v2v_plan_backward (hand-written CUDA backward
    kernels over the plan's own buffers).  A plan holds the intermediates of its LAST run only: when another forward of the
    same plan happened in between (netD is called three times per loss, vid2vid_model_D.py:168-176), the backward first
    re-executes this node's forward (without the running-statistics side effect)."""

    @staticmethod
    def forward(ctx, owner, plan, io, in_slots, out_slots, fixed_slots, *args):
        # args = the input tensors that may need a gradient (slot order of in_slots) followed by the module parameters;
        # fixed_slots = every slot the caller supplied (inputs incl. masks): all other slots are outputs / internal tensors
        n_in = len(in_slots)
        ctx.plan, ctx.in_slots, ctx.out_slots, ctx.n_in, ctx.fixed = plan, in_slots, out_slots, n_in, set(fixed_slots)
        ctx.params = args[n_in:]
        plan.run(io, owner.use_cuda_graph)
        ctx.run_id = plan.run_id
        # The forward tensors the backward reads (inputs, masks AND the node's own outputs) go through save_for_backward: an
        # output kept as a plain ctx attribute is a reference cycle (output -> grad_fn -> ctx -> output) that only the cyclic
        # collector frees -- at cfg3 that held ~2.5 GB per training step until a generation-2 collection came by.
        ctx.n_slots = len(io)
        ctx.io_slots = [i for i, t_ in enumerate(io) if t_ is not None]
        ctx.save_for_backward(*[io[i] for i in ctx.io_slots])
        return tuple(io[s] for s in out_slots)

    @staticmethod
    def backward(ctx, *gouts):
        plan = ctx.plan
        io = [None] * ctx.n_slots
        for i, t_ in zip(ctx.io_slots, ctx.saved_tensors):
            io[i] = t_
        if plan.run_id != ctx.run_id:
            scratch = list(io)
            for s_ in range(len(scratch)):      # outputs of the re-execution go to scratch tensors (the originals are the user's)
                if s_ not in ctx.fixed and scratch[s_] is not None:
                    scratch[s_] = torch.empty_like(scratch[s_])
            plan.run(scratch, False, recompute=True)
            io = scratch
        gio = [None] * len(io)
        for s_, g in zip(ctx.out_slots, gouts):
            if g is not None:
                gio[s_] = g.contiguous().float()
        gin = []
        for k, s_ in enumerate(ctx.in_slots):
            if ctx.needs_input_grad[6 + k] and io[s_] is not None:
                gio[s_] = torch.zeros_like(io[s_])
                gin.append(gio[s_])
            else:
                gin.append(None)
        if os.environ.get('V2V_DEBUG_AUTOGRAD'):
            print('plan backward: in_slots', ctx.in_slots, 'needs', ctx.needs_input_grad[6:6 + ctx.n_in], 'gin', [g is not None for g in gin])
        # Parameter gradients.  The kernels ACCUMULATE into the tensors they are given, so a parameter that already owns a
        # .grad (the trainer's flat all-reduce buffer, or a previous backward) receives its gradient in place and autograd gets
        # None for it: no per-parameter zero fill, no per-parameter accumulate kernel (~1000 of each per step otherwise).  The
        # others share ONE zero-filled buffer.
        need = [bool(ctx.needs_input_grad[6 + ctx.n_in + j]) for j in range(len(ctx.params))]
        direct = [need[j] and p.grad is not None and p.grad.is_contiguous() and p.grad.dtype == torch.float32 and
                  p.grad.device == p.device for j, p in enumerate(ctx.params)]
        fresh = [j for j, p in enumerate(ctx.params) if need[j] and not direct[j]]
        pgrads, ret = [None] * len(ctx.params), [None] * len(ctx.params)
        if fresh:
            flat = torch.zeros(sum(ctx.params[j].numel() for j in fresh), device=ctx.params[fresh[0]].device, dtype=torch.float32)
            off = 0
            for j in fresh:
                n = ctx.params[j].numel()
                pgrads[j] = ret[j] = flat[off:off + n].view_as(ctx.params[j])
                off += n
        for j, p in enumerate(ctx.params):
            if direct[j]:
                pgrads[j] = p.grad
        plan.backward(io, gio, ctx.params, pgrads)
        return (None,) * 6 + tuple(gin) + tuple(ret)


# Arithmetic of the conv stack (include/v2v_b200.h V2V_PREC_*): 'precise' = split-bf16 3-MMA, fp32-class -- the mode
# the parity tests against the fp32 reference and the headline benchmark use; 'fast' = plain bf16 operands.
DEFAULT_PRECISION = os.environ.get('V2V_PRECISION', 'precise')


def set_default_precision(mode):
    global DEFAULT_PRECISION
    assert mode in ('fast', 'precise')
    DEFAULT_PRECISION = mode


class _Planned(nn.Module):
    """Caches one plan per input-shape key; re-packs weights when parameters were modified in place
    and rebuilds when their storage moved (.cuda(), .to())."""

    align_corners = False   # installed-PyTorch grid_sample default; True = PyTorch-0.4 semantics (App. B #2)
    use_cuda_graph = True
    precision = None        # None: DEFAULT_PRECISION at plan-build time; or 'fast' / 'precise' per module

    def _precision(self):
        return self.precision or DEFAULT_PRECISION

    def _plans(self):
        if '_plan_cache' not in self.__dict__:
            self.__dict__['_plan_cache'] = {}
        return self.__dict__['_plan_cache']

    def _signature(self):
        # (the tensor list is cached: walking the module tree costs ~0.6 ms per call, and a training step makes ~40 calls;
        # .cuda() / .to() / load_state_dict keep the Parameter objects, so the list stays valid)
        ts = self.__dict__.get('_sig_tensors')
        if ts is None:
            ts = self.__dict__['_sig_tensors'] = list(self.parameters()) + list(self.buffers())
        ptrs, ver = 0, 0
        for t in ts:
            ptrs = (ptrs * 1000003 + t.data_ptr()) & 0xFFFFFFFFFFFF
            ver += t._version
        return ptrs, ver

    def _wants_grad(self, *tensors):
        """Training plan (saved statistics, gradient buffers, autograd through the C-ABI backward) when autograd is
        recording and a parameter or an input asks for a gradient; the inference plan otherwise."""
        if not torch.is_grad_enabled():
            return False
        return any(p.requires_grad for p in self.parameters()) or any(t is not None and t.requires_grad for t in tensors)

    def _get_plan(self, key, device, build, train=False):
        ptrs, ver = self._signature()
        key = key + (('train',) if train else ()) + (self._precision(),)
        ent = self._plans().get(key)
        if ent is not None and ent['ptrs'] != ptrs:
            ent = None
        if ent is None:
            if os.environ.get('V2V_LOG_PLANS'):
                print('v2v: building plan %s for %s (cached: %d)' % (key, type(self).__name__, len(self._plans())), file=sys.stderr, flush=True)
            plan = Plan(device.index if device.index is not None else torch.cuda.current_device(),
                        precision=self._precision(), train=train)
            build(plan)
            plan.finalize()
            ent = {'plan': plan, 'ptrs': ptrs, 'ver': ver}
            self._plans()[key] = ent
        elif ent['ver'] != ver:
            ent['plan'].repack()
            ent['ver'] = ver
        return ent['plan']

    @staticmethod
    def _require_cuda(*ts):
        for t in ts:
            if t is not None and (not t.is_cuda or t.dtype != torch.float32):
                raise RuntimeError('vid2vid_b200 modules run on CUDA fp32 tensors only (no CPU fallback)')

    def conv_macs(self, *shape_key):
        """Algorithmic conv MACs of one forward for the given input shape (host-only; no GPU needed)."""
        plan = Plan(0)
        self._describe(plan, *shape_key)
        return plan.conv_macs


# IO slots of the composite generators
S_IN, S_PREV, S_MASK, S_FINAL, S_FLOW, S_W, S_RAW, S_IMGF, S_FLOWF, S_FGF, S_FG, S_CI, S_CF, S_CG, S_RAWC = range(15)


class CompositeGenerator(_Planned):
    """models/networks.py:117-232."""

    def __init__(self, opt, input_nc, output_nc, prev_output_nc, ngf, n_downsampling, n_blocks, use_fg_model=False,
                 no_flow=False, norm_layer=nn.BatchNorm2d, padding_type='reflect'):
        assert n_blocks >= 0
        super().__init__()
        self.opt = opt
        self.n_downsampling = n_downsampling
        self.use_fg_model = use_fg_model
        self.no_flow = no_flow
        self.input_nc, self.output_nc, self.prev_output_nc = input_nc, output_nc, prev_output_nc
        nd, mult = n_downsampling, 2 ** n_downsampling
        rb = lambda c: ResnetBlock(c, padding_type=padding_type, activation=nn.ReLU(True), norm_layer=norm_layer)

        if use_fg_model:
            c = ngf // 2 if nd > 2 else ngf
            indv_down = _stem(input_nc, c, norm_layer)
            for i in range(nd):
                indv_down += _down(c * 2 ** i, c * 2 ** (i + 1), norm_layer)
            indv_up = []
            for i in range(nd):
                indv_up += _up(c * 2 ** (nd - i), c * 2 ** (nd - i) // 2, norm_layer)
            self.indv_down = nn.Sequential(*indv_down)
            self.indv_res = nn.Sequential(*[rb(c * mult) for _ in range(n_blocks)])
            self.indv_up = nn.Sequential(*indv_up)
            self.indv_final = nn.Sequential(*_head(c, output_nc, nn.Tanh()))

        down_seg = _stem(input_nc, ngf, norm_layer)
        for i in range(nd):
            down_seg += _down(ngf * 2 ** i, ngf * 2 ** (i + 1), norm_layer)
        down_seg += [rb(ngf * mult) for _ in range(n_blocks - n_blocks // 2)]
        down_img = _stem(prev_output_nc, ngf, norm_layer) + copy.deepcopy(down_seg[4:])
        res_img = [rb(ngf * mult) for _ in range(n_blocks // 2)]
        up_img = []
        for i in range(nd):
            up_img += _up(ngf * 2 ** (nd - i), ngf * 2 ** (nd - i) // 2, norm_layer)

        self.model_down_seg = nn.Sequential(*down_seg)
        self.model_down_img = nn.Sequential(*down_img)
        self.model_res_img = nn.Sequential(*res_img)
        self.model_up_img = nn.Sequential(*up_img)
        self.model_final_img = nn.Sequential(*_head(ngf, output_nc, nn.Tanh()))
        if not no_flow:
            self.model_res_flow = copy.deepcopy(self.model_res_img)
            self.model_up_flow = copy.deepcopy(self.model_up_img)
            self.model_final_flow = nn.Sequential(*_head(ngf, 2))
            self.model_final_w = nn.Sequential(*_head(ngf, 1, nn.Sigmoid()))

    flow_multiplier = 20.0
    fuse_stems = True      # run model_down_seg.1 and indv_down.1 (same input, same 7x7 geometry) as one convolution
    # Set by Vid2VidModelG for the finest scale: `input` is encode_input's full-resolution one-hot + edge map (exact in
    # bf16), so precise plans need no lo half for it.  Leave False for arbitrary inputs (pose maps, pooled pyramid levels).
    input_exact_bf16 = False

    def _describe(self, plan, N, H, W, use_raw_only=False):
        v_in = plan.input(S_IN, N, self.input_nc, 0, self.input_nc, H, W, exact_bf16=self.input_exact_bf16)
        v_prev = plan.input(S_PREV, N, self.prev_output_nc, 0, self.prev_output_nc, H, W)
        fg0 = None
        if self.use_fg_model and self.fuse_stems and _can_pair(self.model_down_seg, self.indv_down):
            seg0, fg0 = emit_unit_pair(plan, list(self.model_down_seg)[:4], list(self.indv_down)[:4], v_in)
            seg = emit_seq(plan, list(self.model_down_seg)[4:], seg0)
        else:
            seg = emit_seq(plan, self.model_down_seg, v_in)
        down = emit_seq(plan, self.model_down_img, v_prev, final_adds=(seg,))              # networks.py:204
        img_feat = emit_seq(plan, self.model_up_img, emit_seq(plan, self.model_res_img, down))   # :205
        plan.export(img_feat, S_IMGF)
        emit_head(plan, self.model_final_img, img_feat, (S_RAW, self.output_nc, 1.0))     # :206
        if not self.no_flow:
            flow_feat = emit_seq(plan, self.model_up_flow, emit_seq(plan, self.model_res_flow, down))   # :210-211
            plan.export(flow_feat, S_FLOWF)
            emit_head_pair(plan, self.model_final_flow, (S_FLOW, 2, self.flow_multiplier),               # :212
                           self.model_final_w, (S_W, 1, 1.0), flow_feat)                                # :213
        if self.use_fg_model:
            fgd = emit_seq(plan, list(self.indv_down)[4:], fg0) if fg0 is not None else emit_seq(plan, self.indv_down, v_in)
            fg_feat = emit_seq(plan, self.indv_up, emit_seq(plan, self.indv_res, fgd))
            plan.export(fg_feat, S_FGF)                                                    # :225
            emit_head(plan, self.indv_final, fg_feat, (S_FG, self.output_nc, 1.0))         # :226
        self._emit_composite(plan, N, H, W, use_raw_only)

    def _emit_composite(self, plan, N, H, W, use_raw_only):
        warp = not (use_raw_only or self.no_flow)
        # training plans keep the head output in S_RAW (the backward needs it) and write the composited raw image to S_RAWC
        plan.composite(S_RAW, S_FLOW if warp else -1, S_W if warp else -1, S_PREV if warp else -1, self.prev_output_nc,
                       S_FG if self.use_fg_model else -1, S_MASK if self.use_fg_model else -1, S_FINAL, N, H, W, warp,
                       self.align_corners, s_raw_out=S_RAWC if (plan.train and self.use_fg_model) else -1)   # :216-230

    def _run(self, key, coarse, input, img_prev, mask, use_raw_only):
        self._require_cuda(input, img_prev, mask, *coarse)
        input, img_prev = input.contiguous(), img_prev.contiguous()
        N, _, H, W = input.shape
        if input.shape[1] != self.input_nc or img_prev.shape[1] != self.prev_output_nc or tuple(img_prev.shape[2:]) != (H, W):
            raise ValueError('netG input / img_prev shapes %s / %s do not match the module (%d / %d channels)' % (
                tuple(input.shape), tuple(img_prev.shape), self.input_nc, self.prev_output_nc))
        if self.use_fg_model and (mask is None or mask.numel() != N * H * W):
            raise ValueError('fg model needs a (N,1,H,W) mask')
        if self.output_nc != 3:
            raise NotImplementedError('the fused composite kernel handles 3 output channels')
        train = self._wants_grad(input, img_prev, *coarse)
        plan = self._get_plan(key + (N, H, W, bool(use_raw_only), bool(self.align_corners), bool(self.input_exact_bf16)), input.device,
                              lambda p: self._describe(p, N, H, W, use_raw_only), train=train)
        new = lambda c: torch.empty((N, c, H, W), device=input.device, dtype=torch.float32)
        io = [None] * 15
        io[S_IN], io[S_PREV] = input, img_prev
        io[S_FINAL], io[S_RAW], io[S_IMGF] = new(self.output_nc), new(self.output_nc), new(self._feat_c())
        if not self.no_flow:
            io[S_FLOW], io[S_W], io[S_FLOWF] = new(2), new(1), new(self._feat_c())
        if self.use_fg_model:
            io[S_MASK] = mask.contiguous()
            io[S_FGF], io[S_FG] = new(self._fg_feat_c()), new(self.output_nc)
        for s, t in zip((S_CI, S_CF, S_CG), coarse):
            io[s] = t.contiguous() if t is not None else None
        if not train:
            plan.run(io, self.use_cuda_graph)
            return io[S_FINAL], io[S_FLOW], io[S_W], io[S_RAW], io[S_IMGF], io[S_FLOWF], io[S_FGF]
        raw_slot = S_RAW
        if self.use_fg_model:
            io[S_RAWC] = new(self.output_nc)
            raw_slot = S_RAWC
        in_slots = [s for s in (S_IN, S_PREV, S_CI, S_CF, S_CG) if io[s] is not None]
        out_slots = [s for s in (S_FINAL, S_FLOW, S_W, raw_slot, S_IMGF, S_FLOWF, S_FGF) if io[s] is not None]
        fixed = [s for s in (S_IN, S_PREV, S_MASK, S_CI, S_CF, S_CG) if io[s] is not None]
        params = [p for p in self.parameters()]
        outs = _PlanFunction.apply(self, plan, io, tuple(in_slots), tuple(out_slots), tuple(fixed),
                                   *([io[s] for s in in_slots] + params))
        res = dict(zip(out_slots, outs))
        return (res.get(S_FINAL), res.get(S_FLOW), res.get(S_W), res.get(raw_slot), res.get(S_IMGF), res.get(S_FLOWF),
                res.get(S_FGF))

    def _feat_c(self):
        return self.model_final_img[1].in_channels

    def _fg_feat_c(self):
        return self.indv_final[1].in_channels

    def forward(self, input, img_prev, mask, img_feat_coarse, flow_feat_coarse, img_fg_feat_coarse, use_raw_only):
        return self._run(('G',), (), input, img_prev, mask, use_raw_only)


class CompositeLocalGenerator(CompositeGenerator):
    """models/networks.py:234-325."""

    def __init__(self, opt, input_nc, output_nc, prev_output_nc, ngf, n_downsampling, n_blocks_local,
                 use_fg_model=False, no_flow=False, norm_layer=nn.BatchNorm2d, padding_type='reflect', scale=1):
        _Planned.__init__(self)
        self.opt = opt
        self.use_fg_model = use_fg_model
        self.no_flow = no_flow
        self.scale = scale
        self.input_nc, self.output_nc, self.prev_output_nc = input_nc, output_nc, prev_output_nc
        rb = lambda c: ResnetBlock(c, padding_type=padding_type, activation=nn.ReLU(True), norm_layer=norm_layer)
        if use_fg_model:
            c = ngf // 2 if n_downsampling > 2 else ngf
            self.indv_down = nn.Sequential(*(_stem(input_nc, c, norm_layer) + _down(c, c * 2, norm_layer)))
            self.indv_up = nn.Sequential(*([rb(c * 2) for _ in range(n_blocks_local)] + _up(c * 2, c, norm_layer)))
            self.indv_final = nn.Sequential(*_head(c, output_nc, nn.Tanh()))
        self.model_down_seg = nn.Sequential(*(_stem(input_nc, ngf, norm_layer) + _down(ngf, ngf * 2, norm_layer)))
        self.model_down_img = nn.Sequential(*(_stem(prev_output_nc, ngf, norm_layer) + _down(ngf, ngf * 2, norm_layer)))
        self.model_up_img = nn.Sequential(*([rb(ngf * 2) for _ in range(n_blocks_local)] + _up(ngf * 2, ngf, norm_layer)))
        self.model_final_img = nn.Sequential(*_head(ngf, output_nc, nn.Tanh()))
        if not no_flow:
            self.model_up_flow = copy.deepcopy(self.model_up_img)
            self.model_final_flow = nn.Sequential(*_head(ngf, 2))
            self.model_final_w = nn.Sequential(*_head(ngf, 1, nn.Sigmoid()))

    def _describe(self, plan, N, H, W, use_raw_only=False):
        h2, w2 = H // 2, W // 2
        c2 = self.model_down_seg[4].out_channels
        v_in = plan.input(S_IN, N, self.input_nc, 0, self.input_nc, H, W, exact_bf16=self.input_exact_bf16)
        v_prev = plan.input(S_PREV, N, self.prev_output_nc, 0, self.prev_output_nc, H, W)
        ci = plan.input(S_CI, N, c2, 0, c2, h2, w2)
        fg0 = None
        if self.use_fg_model and self.fuse_stems and _can_pair(self.model_down_seg, self.indv_down):
            seg0, fg0 = emit_unit_pair(plan, list(self.model_down_seg)[:4], list(self.indv_down)[:4], v_in)
            seg = emit_seq(plan, list(self.model_down_seg)[4:], seg0)
        else:
            seg = emit_seq(plan, self.model_down_seg, v_in)
        fin = emit_seq(plan, self.model_down_img, v_prev, defer_last=True)      # down_img = seg + img (:298)
        img_feat = emit_seq(plan, self.model_up_img, fin((seg, ci)))             # :299
        plan.export(img_feat, S_IMGF)
        emit_head(plan, self.model_final_img, img_feat, (S_RAW, self.output_nc, 1.0))
        if not self.no_flow:
            cf = plan.input(S_CF, N, c2, 0, c2, h2, w2)
            flow_feat = emit_seq(plan, self.model_up_flow, fin((seg, cf)))       # :305
            plan.export(flow_feat, S_FLOWF)
            emit_head_pair(plan, self.model_final_flow, (S_FLOW, 2, 20.0 * (2 ** self.scale)),         # :297,306
                           self.model_final_w, (S_W, 1, 1.0), flow_feat)
        if self.use_fg_model:
            cg_c = self.indv_down[4].out_channels
            cg = plan.input(S_CG, N, cg_c, 0, cg_c, h2, w2)
            if fg0 is not None:
                fgd = emit_seq(plan, list(self.indv_down)[4:], fg0, final_adds=(cg,))
            else:
                fgd = emit_seq(plan, self.indv_down, v_in, final_adds=(cg,))
            fg_feat = emit_seq(plan, self.indv_up, fgd)                                                       # :319
            plan.export(fg_feat, S_FGF)
            emit_head(plan, self.indv_final, fg_feat, (S_FG, self.output_nc, 1.0))
        self._emit_composite(plan, N, H, W, use_raw_only)

    def forward(self, input, img_prev, mask, img_feat_coarse, flow_feat_coarse, img_fg_feat_coarse, use_raw_only):
        return self._run(('GL',), (img_feat_coarse, flow_feat_coarse, img_fg_feat_coarse), input, img_prev, mask,
                         use_raw_only)


class GlobalGenerator(_Planned):
    """models/networks.py:327-359 (first-frame generator under --use_single_G)."""

    def __init__(self, input_nc, output_nc, ngf=64, n_downsampling=3, n_blocks=9, norm_layer=nn.BatchNorm2d,
                 padding_type='reflect'):
        assert n_blocks >= 0
        super().__init__()
        cm = lambda c: min(1024, c)
        self.input_nc, self.output_nc = input_nc, output_nc
        model = _stem(input_nc, ngf, norm_layer)
        for i in range(n_downsampling):
            model += _down(cm(ngf * 2 ** i), cm(ngf * 2 ** (i + 1)), norm_layer)
        model += [ResnetBlock(cm(ngf * 2 ** n_downsampling), padding_type=padding_type, activation=nn.ReLU(True),
                              norm_layer=norm_layer) for _ in range(n_blocks)]
        for i in range(n_downsampling):
            m = 2 ** (n_downsampling - i)
            model += _up(cm(ngf * m), cm(int(ngf * m / 2)), norm_layer)
        model += _head(ngf, output_nc, nn.Tanh())
        self.model = nn.Sequential(*model)

    def _describe(self, plan, N, H, W):
        v = plan.input(0, N, self.input_nc, 0, self.input_nc, H, W)
        mods = list(self.model)
        v = emit_seq(plan, mods[:-3], v)
        emit_head(plan, mods[-3:], v, (1, self.output_nc, 1.0))

    def forward(self, input, feat=None):
        if feat is not None:
            input = torch.cat([input, feat], dim=1)
        self._require_cuda(input)
        input = input.contiguous()
        N, _, H, W = input.shape
        plan = self._get_plan(('GG', N, H, W), input.device, lambda p: self._describe(p, N, H, W))
        out = torch.empty((N, self.output_nc, H, W), device=input.device, dtype=torch.float32)
        plan.run([input, out], self.use_cuda_graph)
        return out


class Global_with_z(_Planned):
    """models/networks.py:421-467: a pix2pixHD global generator whose nz-channel feature map z is concatenated in at four
    places: with the input, in front of the residual blocks and of the upsampling path (z average-pooled n_downsample_G
    times), and in front of the 7x7 tanh head.  One plan: the input-side concatenation is the caller's torch.cat, the
    other three are concat nodes (forward only: the first-frame generator runs under no_grad)."""

    def __init__(self, input_nc, output_nc, nz, ngf=64, n_downsample_G=3, n_blocks=9, norm_layer=nn.BatchNorm2d,
                 padding_type='reflect'):
        super().__init__()
        self.n_downsample_G = n_downsample_G
        self.input_nc, self.output_nc, self.nz = input_nc, output_nc, nz
        cm = lambda c: min(1024, c)
        model_downsample = _stem(input_nc + nz, ngf, norm_layer)
        for i in range(n_downsample_G):
            model_downsample += _down(cm(ngf * 2 ** i), cm(ngf * 2 ** (i + 1)), norm_layer)
        mult = 2 ** n_downsample_G
        model_resnet = [ResnetBlock(cm(ngf * mult) + nz, padding_type=padding_type, norm_layer=norm_layer) for _ in range(n_blocks)]
        model_upsample = []
        for i in range(n_downsample_G):
            mult = 2 ** (n_downsample_G - i)
            model_upsample += _up(cm(ngf * mult) + (nz * 2 if i == 0 else 0), cm(ngf * mult // 2), norm_layer)
        self.model_downsample = nn.Sequential(*model_downsample)
        self.model_resnet = nn.Sequential(*model_resnet)
        self.model_upsample = nn.Sequential(*model_upsample)
        self.model_upsample_conv = nn.Sequential(*_head(ngf + nz, output_nc, nn.Tanh()))
        self.downsample = nn.AvgPool2d(3, stride=2, padding=[1, 1], count_include_pad=False)

    def _z_dims(self, H, W):
        for _ in range(self.n_downsample_G):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        return H, W

    def _describe(self, plan, N, H, W):
        """slot 0 = cat([x, z]) (N, input_nc + nz, H, W), slot 1 = z average-pooled n_downsample_G times, slot 2 = output."""
        cin = self.input_nc + self.nz
        v_xz = plan.input(0, N, cin, 0, cin, H, W)
        v_z = plan.input(0, N, cin, self.input_nc, self.nz, H, W)
        v_zd = plan.input(1, N, self.nz, 0, self.nz, *self._z_dims(H, W))
        down = emit_seq(plan, self.model_downsample, v_xz)                              # :461
        res = emit_seq(plan, self.model_resnet, plan.concat([down, v_zd]))              # :462
        up = emit_seq(plan, self.model_upsample, plan.concat([res, v_zd]))              # :463
        emit_head(plan, self.model_upsample_conv, plan.concat([up, v_z]), (2, self.output_nc, 1.0))   # :464

    def forward(self, x, z):
        from . import ops
        self._require_cuda(x, z)
        if self._wants_grad(x, z):
            raise NotImplementedError('Global_with_z has no backward (the first-frame generator runs under no_grad)')
        N, _, H, W = x.shape
        if x.shape[1] != self.input_nc or tuple(z.shape) != (N, self.nz, H, W) or H % 2 ** self.n_downsample_G or W % 2 ** self.n_downsample_G:
            raise ValueError('Global_with_z: x %s / z %s do not fit (%d + %d channels, sides divisible by %d)' % (
                tuple(x.shape), tuple(z.shape), self.input_nc, self.nz, 2 ** self.n_downsample_G))
        z = z.contiguous()
        z_down = z
        for _ in range(self.n_downsample_G):
            z_down = ops.avgpool3s2(z_down)
        xz = torch.cat([x, z], dim=1)
        plan = self._get_plan(('GZ', N, H, W), x.device, lambda p: self._describe(p, N, H, W))
        out = torch.empty((N, self.output_nc, H, W), device=x.device, dtype=torch.float32)
        plan.run([xz, z_down, out], self.use_cuda_graph)
        return out


class Encoder(_Planned):
    """models/networks.py:595-632: stem 7x7, n_downsampling stride-2 convs, as many transposed convs and a 7x7 tanh head
    (InstanceNorm throughout), then the instance-wise average pooling over the id map `inst` (ops.instance_mean, in place on
    the head output).  The ids must be integers in [0, n_ids): the face part maps hold 0 .. 6."""

    n_ids = 7        # face parts (data/face_dataset.py); a larger value only costs another pass per 8 ids

    def __init__(self, input_nc, output_nc, ngf=32, n_downsampling=4, norm_layer=nn.BatchNorm2d):
        super().__init__()
        self.input_nc, self.output_nc = input_nc, output_nc
        model = _stem(input_nc, ngf, norm_layer)
        for i in range(n_downsampling):
            model += _down(ngf * 2 ** i, ngf * 2 ** (i + 1), norm_layer)
        for i in range(n_downsampling):
            mult = 2 ** (n_downsampling - i)
            model += _up(ngf * mult, int(ngf * mult / 2), norm_layer)
        model += _head(ngf, output_nc, nn.Tanh())
        self.model = nn.Sequential(*model)

    def _describe(self, plan, N, H, W):
        mods = list(self.model)
        v = emit_seq(plan, mods[:-3], plan.input(0, N, self.input_nc, 0, self.input_nc, H, W))
        emit_head(plan, mods[-3:], v, (1, self.output_nc, 1.0))

    def forward(self, input, inst):
        from . import ops
        self._require_cuda(input, inst)
        if self._wants_grad(input):
            raise NotImplementedError('Encoder has no backward (the face first frame runs under no_grad)')
        input = input.contiguous()
        N, _, H, W = input.shape
        plan = self._get_plan(('E', N, H, W), input.device, lambda p: self._describe(p, N, H, W))
        out = torch.empty((N, self.output_nc, H, W), device=input.device, dtype=torch.float32)
        plan.run([input, out], self.use_cuda_graph)
        return ops.instance_mean(out, inst.contiguous(), self.n_ids, out=out)


# ------------------------------------------------------------------------------------ face features table
FACE_LABELS = 7          # face parts of the edge2face part map (data/face_dataset.py)


def synthetic_face_features(num_images, feat_num=16, seed=0, n_labels=FACE_LABELS):
    """A seeded stand-in for checkpoints/edge2face_single/features.npy: {label: (num_images, feat_num + 1) array}, the
    first feat_num columns uniform in [-1, 1] (the range of the Encoder's tanh means), the last (which the lookup never
    reads) the row index.  The values are fp32-exact, stored as float64 (numpy float64 scalars are Python floats, which the
    reference's element-wise copy into a FloatTensor accepts).  Depends only on the arguments."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for label in range(n_labels):
        f = torch.rand((num_images, feat_num), generator=g, dtype=torch.float64) * 2 - 1
        out[label] = torch.cat([f, torch.arange(num_images, dtype=torch.float64)[:, None]], 1).float().double().numpy()
    return out


def pack_face_features(features, feat_num):
    """features.npy's {label: (rows, feat_num + 1)} dict -> (table (n_labels, max_rows, feat_num + 1) fp32 CPU tensor, rows
    per label, num_images).  num_images is features[6].shape[0], as the reference takes it (vid2vid_model_G.py:298)."""
    labels = sorted(int(k) for k in features)
    if labels != list(range(len(labels))):
        raise ValueError('features table labels must be 0 .. n-1, got %s' % labels)
    arrs = [torch.as_tensor(features[k], dtype=torch.float32) for k in labels]
    if any(a.dim() != 2 or a.shape[1] < feat_num + 1 for a in arrs):
        raise ValueError('features table rows need feat_num + 1 = %d columns' % (feat_num + 1))
    rows = [a.shape[0] for a in arrs]
    table = torch.zeros(len(arrs), max(rows), feat_num + 1)
    for k, a in enumerate(arrs):
        table[k, :a.shape[0]] = a[:, :feat_num + 1]
    if len(rows) < FACE_LABELS:
        raise ValueError('features table has %d labels; the face parts are %d' % (len(rows), FACE_LABELS))
    return table, rows, rows[6]


class LocalEnhancer(_Planned):
    """models/networks.py:361-419."""

    def __init__(self, input_nc, output_nc, ngf=32, n_downsample_global=3, n_blocks_global=9, n_local_enhancers=1,
                 n_blocks_local=3, norm_layer=nn.BatchNorm2d, padding_type='reflect'):
        super().__init__()
        self.n_local_enhancers = n_local_enhancers
        self.input_nc, self.output_nc = input_nc, output_nc
        g = GlobalGenerator(input_nc, output_nc, ngf * (2 ** n_local_enhancers), n_downsample_global, n_blocks_global,
                            norm_layer).model
        self.model = nn.Sequential(*[g[i] for i in range(len(g) - 3)])
        for n in range(1, n_local_enhancers + 1):
            c = ngf * (2 ** (n_local_enhancers - n))
            down = _stem(input_nc, c, norm_layer) + _down(c, c * 2, norm_layer)
            up = [ResnetBlock(c * 2, padding_type=padding_type, norm_layer=norm_layer) for _ in range(n_blocks_local)]
            up += _up(c * 2, c, norm_layer)
            if n == n_local_enhancers:
                up += _head(ngf, output_nc, nn.Tanh())
            setattr(self, 'model%d_1' % n, nn.Sequential(*down))
            setattr(self, 'model%d_2' % n, nn.Sequential(*up))
        self.downsample = nn.AvgPool2d(3, stride=2, padding=[1, 1], count_include_pad=False)

    def _describe(self, plan, N, H, W):
        # pyramid level i of the input arrives in IO slot i (built by forward with the avg-pool kernel)
        L_ = self.n_local_enhancers
        dims = [(H, W)]
        for _ in range(L_):
            dims.append(((dims[-1][0] - 1) // 2 + 1, (dims[-1][1] - 1) // 2 + 1))
        out = emit_seq(plan, self.model, plan.input(L_, N, self.input_nc, 0, self.input_nc, *dims[L_]))
        for n in range(1, L_ + 1):
            lvl = L_ - n
            x = emit_seq(plan, getattr(self, 'model%d_1' % n),
                         plan.input(lvl, N, self.input_nc, 0, self.input_nc, *dims[lvl]), final_adds=(out,))
            mods = list(getattr(self, 'model%d_2' % n))
            if n == L_:
                out = emit_seq(plan, mods[:-3], x)
                emit_head(plan, mods[-3:], out, (L_ + 1, self.output_nc, 1.0))
            else:
                out = emit_seq(plan, mods, x)

    def forward(self, input, feat_map=None):
        from . import ops
        if feat_map is not None:
            input = torch.cat([input, feat_map], dim=1)
        self._require_cuda(input)
        pyr = [input.contiguous()]
        for _ in range(self.n_local_enhancers):
            pyr.append(ops.avgpool3s2(pyr[-1]))
        N, _, H, W = input.shape
        plan = self._get_plan(('LE', N, H, W), input.device, lambda p: self._describe(p, N, H, W))
        out = torch.empty((N, self.output_nc, H, W), device=input.device, dtype=torch.float32)
        plan.run(pyr + [out], self.use_cuda_graph)
        return out


# ------------------------------------------------------------------------------------ discriminators
class NLayerDiscriminator(nn.Module):
    """Parameter container with the keys of models/networks.py:679-725."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm_layer=nn.BatchNorm2d, getIntermFeat=False):
        super().__init__()
        self.getIntermFeat, self.n_layers = getIntermFeat, n_layers
        kw, padw = 4, 2
        seq = [[nn.Conv2d(input_nc, ndf, kernel_size=kw, stride=2, padding=padw), nn.LeakyReLU(0.2, True)]]
        nf = ndf
        for n in range(1, n_layers):
            nf_prev, nf = nf, min(nf * 2, 512)
            seq += [[nn.Conv2d(nf_prev, nf, kernel_size=kw, stride=2, padding=padw), norm_layer(nf),
                     nn.LeakyReLU(0.2, True)]]
        nf_prev, nf = nf, min(nf * 2, 512)
        seq += [[nn.Conv2d(nf_prev, nf, kernel_size=kw, stride=1, padding=padw), norm_layer(nf), nn.LeakyReLU(0.2, True)]]
        seq += [[nn.Conv2d(nf, 1, kernel_size=kw, stride=1, padding=padw)]]
        if getIntermFeat:
            for n in range(len(seq)):
                setattr(self, 'model' + str(n), nn.Sequential(*seq[n]))
        else:
            self.model = nn.Sequential(*[m for s in seq for m in s])


class MultiscaleDiscriminator(_Planned):
    """models/networks.py:634-675: num_D PatchGAN towers (NLayerDiscriminator, :679-725) on an avg-pool pyramid of the
    input; with getIntermFeat every layer output of every tower is returned (feature-matching loss,
    models/vid2vid_model_D.py:35-36).  Each tower is one plan: 4x4 s2 conv + bias + LeakyReLU epilogue, (n_layers - 1) x
    [4x4 s2 conv, norm, LeakyReLU], 4x4 s1 conv + norm + LeakyReLU, and the 1-channel 4x4 s1 head."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm_layer=nn.BatchNorm2d, num_D=3, getIntermFeat=False):
        super().__init__()
        self.num_D, self.n_layers, self.getIntermFeat = num_D, n_layers, getIntermFeat
        self.input_nc = input_nc
        for i in range(num_D):
            netD = NLayerDiscriminator(input_nc, min(64, ndf * (2 ** (num_D - 1 - i))), n_layers, norm_layer,
                                       getIntermFeat)
            if getIntermFeat:
                for j in range(n_layers + 2):
                    setattr(self, 'scale%d_layer%d' % (i, j), getattr(netD, 'model' + str(j)))
            else:
                setattr(self, 'layer' + str(i), netD.model)
        self.downsample = nn.AvgPool2d(3, stride=2, padding=[1, 1], count_include_pad=False)

    def _tower_layers(self, d):
        """List of per-layer module lists of tower d."""
        if self.getIntermFeat:
            return [list(getattr(self, 'scale%d_layer%d' % (d, j))) for j in range(self.n_layers + 2)]
        mods, layers, cur = list(getattr(self, 'layer' + str(d))), [], []
        for m in mods:
            if isinstance(m, nn.Conv2d) and cur:
                layers.append(cur)
                cur = []
            cur.append(m)
        layers.append(cur)
        return layers

    def _tower_params(self, d):
        return [p for mods in self._tower_layers(d) for m in mods for p in m.parameters()]

    def _describe(self, plan, d, N, H, W):
        layers = self._tower_layers(d)
        v = plan.input(0, N, self.input_nc, 0, self.input_nc, H, W)
        shapes = []
        for j, mods in enumerate(layers):
            last = j == len(layers) - 1
            conv = mods[0]
            oh = (H + 2 * conv.padding[0] - conv.kernel_size[0]) // conv.stride[0] + 1
            ow = (W + 2 * conv.padding[1] - conv.kernel_size[1]) // conv.stride[1] + 1
            if last:
                plan.head(v, conv_desc(conv), [(1 + j, 0, 1, L.ACT_NONE, 1.0)])      # 1-channel patch logits, fp32
            else:
                v = emit_seq(plan, mods, v)
                if self.getIntermFeat:
                    plan.export(v, 1 + j)
            shapes.append((conv.out_channels, oh, ow))
            H, W = oh, ow
        return shapes

    def _tower_forward(self, d, x):
        N, _, H, W = x.shape
        key = ('D', d, N, H, W)
        shapes_box = {}

        def build(p):
            shapes_box['s'] = self._describe(p, d, N, H, W)
        train = self._wants_grad(x)
        plan = self._get_plan(key, x.device, build, train=train)
        shapes = self._plans()[key + (('train',) if train else ()) + (self._precision(),)].setdefault('shapes', shapes_box.get('s'))
        outs = [torch.empty((N, c, h, w), device=x.device, dtype=torch.float32) for (c, h, w) in shapes]
        io = [x] + [o if (self.getIntermFeat or j == len(outs) - 1) else None for j, o in enumerate(outs)]
        if not train:
            plan.run(io, self.use_cuda_graph)
            return outs if self.getIntermFeat else [outs[-1]]
        out_slots = tuple(s for s in range(1, len(io)) if io[s] is not None)
        params = [p for p in self._tower_params(d)]
        res = _PlanFunction.apply(self, plan, io, (0,), out_slots, (0,), *([x] + params))
        return list(res)

    def forward(self, input):
        from . import ops
        self._require_cuda(input)
        result = []
        x = input.contiguous()
        for i in range(self.num_D):
            result.append(self._tower_forward(self.num_D - 1 - i, x))
            if i != self.num_D - 1:
                x = ops.avgpool3s2(x)            # autograd-aware (ops.AvgPool3s2Function) when x requires a gradient
        return result


def build_netG(opt, s):
    """netG{s} exactly as Vid2VidModelG.initialize builds it (models/vid2vid_model_G.py:30-43)."""
    input_nc = opt.label_nc if opt.label_nc != 0 else opt.input_nc
    netG_input_nc = input_nc * opt.n_frames_G + (opt.n_frames_G if opt.use_instance else 0)
    prev_output_nc = (opt.n_frames_G - 1) * opt.output_nc
    if s == 0:
        return define_G(netG_input_nc, opt.output_nc, prev_output_nc, opt.ngf, opt.netG, opt.n_downsample_G, opt.norm,
                        0, [], opt)
    return define_G(netG_input_nc, opt.output_nc, prev_output_nc, opt.ngf // (2 ** s), opt.netG + 'Local',
                    opt.n_downsample_G, opt.norm, s, [], opt)


class SequentialRunner(_Planned):
    """Runs a list of supported layer containers (conv / norm / activation units, ResnetBlocks, transposed
    convs; optionally a trailing small-Cout head) through the plan runtime: fp32 NCHW in -> fp32 NCHW out.
    Used by the per-kernel parity tests and handy for porting other vid2vid sub-networks."""

    def __init__(self, mods, head_mods=None, head_scale=1.0):
        super().__init__()
        self.seq = nn.Sequential(*mods)
        self.head = nn.Sequential(*head_mods) if head_mods else None
        self.head_scale = head_scale

    def _describe(self, plan, N, C, H, W):
        v = plan.input(0, N, C, 0, C, H, W)
        v = emit_seq(plan, self.seq, v)
        if self.head is not None:
            emit_head(plan, self.head, v, (1, self.head[1].out_channels, self.head_scale))
        else:
            plan.export(v, 1)

    def forward(self, x):
        self._require_cuda(x)
        x = x.contiguous()
        N, C, H, W = x.shape
        key = ('SR', N, C, H, W)
        plan = self._get_plan(key, x.device, lambda p: self._describe(p, N, C, H, W))
        if self.head is not None:
            oc, oh, ow = self.head[1].out_channels, H, W
            if len(self.seq):
                last = plan.describe()['values'][-1]
                oh, ow = last['H'], last['W']
        else:
            last = plan.describe()['values'][-1]
            oc, oh, ow = last['C'], last['H'], last['W']
        out = torch.empty((N, oc, oh, ow), device=x.device, dtype=torch.float32)
        if not self._wants_grad(x):
            plan.run([x, out], self.use_cuda_graph)
            return out
        tplan = self._get_plan(key, x.device, lambda p: self._describe(p, N, C, H, W), train=True)
        (res,) = _PlanFunction.apply(self, tplan, [x, out], (0,), (1,), (0,), *([x] + list(self.parameters())))
        return res


# ------------------------------------------------------------------------------------ VGG19 perceptual loss
VGG19_FILE = 'vgg19-dcbb9e9d.pth'      # torchvision's ImageNet VGG19 checkpoint, as its hub cache names it
_VGG_CFG = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512]   # -> features[0:30]
_VGG_SLICES = ((0, 2), (2, 7), (7, 12), (12, 21), (21, 30))    # slice k ends at relu{k}_1 (models/networks.py:849-858)


def vgg19_weights_path():
    return os.path.join(torch.hub.get_dir(), 'checkpoints', VGG19_FILE)


def vgg19_features():
    """torchvision's vgg19().features[0:30] as a list: the same layers at the same indices (3x3 convs with zero padding 1 and
    bias, ReLU, 2x2 max-pools).  Built with the global RNG state saved and restored: the weights are always replaced
    (load_vgg19_weights), and turning the loss on must not change the initialisation of anything created after it."""
    layers, c = [], 3
    with torch.random.fork_rng(devices=[]):
        for v in _VGG_CFG:
            if v == 'M':
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2, padding=0, dilation=1, ceil_mode=False))
            else:
                layers += [nn.Conv2d(c, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
                c = v
    return layers


def load_vgg19_weights(vgg, synthetic=False, seed=0):
    """Fill `vgg` (a Vgg19) from torchvision's cached ImageNet checkpoint, mapping its `features.{i}` keys to the slice keys.
    Nothing is ever downloaded.  Without the file: a seeded torchvision-style init (kaiming-normal fan_out weights, zero
    bias) when `synthetic`, FileNotFoundError otherwise."""
    path = vgg19_weights_path()
    if os.path.exists(path):
        sd = torch.load(path, map_location='cpu', weights_only=True)
        mapped = {}
        for k, (a, b) in enumerate(_VGG_SLICES):
            for i in range(a, b):
                for leaf in ('weight', 'bias'):
                    if 'features.%d.%s' % (i, leaf) in sd:
                        mapped['slice%d.%d.%s' % (k + 1, i, leaf)] = sd['features.%d.%s' % (i, leaf)]
        vgg.load_state_dict(mapped)
        return vgg
    if not synthetic:
        raise FileNotFoundError('VGG19 weights not found at %s (torchvision\'s ImageNet VGG19 checkpoint); copy the file '
                                'there, or set synthetic_weights for a seeded random init' % path)
    return vgg19_synthetic_(vgg, seed)


def vgg19_synthetic_(vgg, seed=0):
    """Seeded torchvision-style init of a Vgg19 in place: kaiming-normal (fan_out, ReLU gain) weights, zero bias.  Depends only
    on the seed (a private generator, the global RNG is untouched)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in vgg.state_dict().items():
            if name.endswith('.weight'):
                fan_out = t.shape[0] * t.shape[2] * t.shape[3]
                t.copy_(torch.randn(t.shape, generator=g) * (2.0 / fan_out) ** 0.5)
            else:
                t.zero_()
    return vgg


class Vgg19(_Planned):
    """models/networks.py:840-869: slice1 .. slice5 of VGG19's features, frozen, with the reference's module tree and
    state_dict keys (slice1.0.weight .. slice5.28.bias).  forward(X) returns the five relu{k}_1 maps; VGGLoss instead runs
    feature_l1(x, y), which never leaves the plan's buffers.  Each conv is a bias + ReLU unit on the wgmma conv kernel, each
    pool a max-pool node."""

    def __init__(self, requires_grad=False):
        super().__init__()
        feats = vgg19_features()
        for k, (a, b) in enumerate(_VGG_SLICES):
            s = nn.Sequential()
            for i in range(a, b):
                s.add_module(str(i), feats[i])
            setattr(self, 'slice%d' % (k + 1), s)
        if not requires_grad:
            for p in self.parameters():
                p.requires_grad = False

    def _branch(self, plan, v):
        outs = []
        for k in range(5):
            for m in getattr(self, 'slice%d' % (k + 1)):
                if isinstance(m, nn.Conv2d):
                    v = plan.conv_act(v, conv_desc(m), L.ACT_RELU, 0.0)      # (the ReLU that follows is fused)
                elif isinstance(m, nn.MaxPool2d):
                    v = plan.maxpool2(v)
            outs.append(v)
        return outs

    def _describe(self, plan, N, H, W):
        """The loss plan: slot 0 = x, slot 1 = y (the target), slot 2 = (5,) fp32 per-level mean |x_k - y_k|.  Both branches
        run the same frozen weights (packed once per branch); the y branch only feeds detached operands, so the backward
        skips it entirely."""
        fx = self._branch(plan, plan.input(0, N, 3, 0, 3, H, W))
        fy = self._branch(plan, plan.input(1, N, 3, 0, 3, H, W))
        for k in range(5):
            plan.feature_l1(fx[k], fy[k], 2, k)

    def _describe_features(self, plan, N, H, W):
        for k, v in enumerate(self._branch(plan, plan.input(0, N, 3, 0, 3, H, W))):
            plan.export(v, 1 + k)

    @staticmethod
    def feature_shapes(H, W):
        shapes = []
        for k, c in enumerate((64, 128, 256, 512, 512)):
            shapes.append((c, H, W))
            H, W = H // 2, W // 2
        return shapes

    def forward(self, X):
        """The five feature maps (inference only: VGGLoss differentiates through feature_l1)."""
        self._require_cuda(X)
        if self._wants_grad(X):
            raise NotImplementedError('Vgg19.forward has no backward; VGGLoss differentiates through Vgg19.feature_l1')
        X = X.contiguous()
        N, _, H, W = X.shape
        plan = self._get_plan(('VGGF', N, H, W), X.device, lambda p: self._describe_features(p, N, H, W))
        outs = [torch.empty((N, c, h, w), device=X.device, dtype=torch.float32) for c, h, w in self.feature_shapes(H, W)]
        plan.run([X] + outs, self.use_cuda_graph)
        return outs

    def feature_l1(self, x, y):
        """(5,) fp32 tensor of mean |vgg(x)_k - vgg(y)_k.detach()|, k = relu1_1 .. relu5_1.  Differentiable in x only."""
        self._require_cuda(x, y)
        x, y = x.contiguous(), y.detach().contiguous()
        if x.shape != y.shape or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError('VGG inputs must be two (N, 3, H, W) tensors of the same shape, got %s and %s' % (tuple(x.shape), tuple(y.shape)))
        N, _, H, W = x.shape
        train = self._wants_grad(x)
        plan = self._get_plan(('VGGL', N, H, W), x.device, lambda p: self._describe(p, N, H, W), train=train)
        out = torch.empty(5, device=x.device, dtype=torch.float32)
        io = [x, y, out]
        if not train:
            plan.run(io, self.use_cuda_graph)
            return out
        (res,) = _PlanFunction.apply(self, plan, io, (0,), (2,), (0, 1), *([x] + list(self.parameters())))
        return res


class AvgPool2(nn.Module):
    """nn.AvgPool2d(2, stride=2, count_include_pad=False) on the engine (ops.avgpool2, autograd-aware)."""

    kernel_size = stride = 2

    def forward(self, x):
        from . import ops
        return ops.avgpool2(x)


class VGGLoss(nn.Module):
    """models/networks.py:776-791: sum_k w_k * mean |vgg(x)_k - vgg(y)_k.detach()| with w = 1/32 .. 1, the images halved by
    a 2x2 mean while wider than 1024 pixels.  No ImageNet normalisation: the images go in as they are, in [-1, 1], as in
    the reference.  `vgg`, `weights` and `downsample` have the reference's meaning."""

    def __init__(self, gpu_id=0, synthetic=False, seed=0):
        super().__init__()
        self.vgg = load_vgg19_weights(Vgg19(), synthetic=synthetic, seed=seed).cuda(gpu_id)
        self.weights = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]
        self.downsample = AvgPool2()

    def forward(self, x, y):
        while x.size()[3] > 1024:
            x, y = self.downsample(x), self.downsample(y)
        levels = self.vgg.feature_l1(x, y)
        loss = 0
        for i in range(len(self.weights)):
            loss += self.weights[i] * levels[i]
        return loss
