"""H100 drop-ins for the reference optical-flow stack: FlowNet2 (models/flownet2_pytorch/models.py:30-160 with
FlowNetC / FlowNetS / FlowNetSD / FlowNetFusion, networks/*.py) and the vid2vid wrapper FlowNet
(models/flownet.py:12-62) that turns it into the (flow, confidence) training targets.

The torch.nn layers are parameter containers with the reference's state_dict keys (pinned by
tests/golden/flownet2_keys.json, the reference's own 220 keys / 162,518,834 parameters), so
FlowNet2_checkpoint.pth.tar loads unchanged.  forward() describes each sub-network once per input shape to the plan
runtime (wgmma convolutions in the precise split-bf16 mode -- FlowNet2 has no norm layers to absorb operand rounding --
bias + LeakyReLU(0.1) units, channel concatenation, the correlation op) and chains the plans with the stand-alone CUDA
operators (resample2d, channelnorm, x4 upsampling).  There is no PyTorch / cuDNN fallback.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib as L
from . import ops
from .networks import _Planned
from .plan import conv_desc, norm_desc

DIV_FLOW = 20.0
SLOPE = 0.1


def _conv(cin, cout, k=3, stride=1):
    """submodules.conv without batch norm (networks/submodules.py:7-21)."""
    return nn.Sequential(nn.Conv2d(cin, cout, k, stride=stride, padding=(k - 1) // 2, bias=True), nn.LeakyReLU(SLOPE, inplace=True))


def _i_conv(cin, cout):
    """submodules.i_conv (submodules.py:23-34): 3x3, bias, no activation (inside a Sequential like conv)."""
    return nn.Sequential(nn.Conv2d(cin, cout, 3, stride=1, padding=1, bias=True))


def _predict(cin):
    return nn.Conv2d(cin, 2, 3, stride=1, padding=1, bias=True)


def _deconv(cin, cout):
    return nn.Sequential(nn.ConvTranspose2d(cin, cout, 4, stride=2, padding=1, bias=True), nn.LeakyReLU(SLOPE, inplace=True))


def _upflow(bias):
    return nn.ConvTranspose2d(2, 2, 4, 2, 1, bias=bias)


class _Sub(nn.Module):
    """Shared lowering vocabulary of the four sub-networks (oracle/flownet2_oracle.py `_Net` is the CPU twin)."""

    def u_conv(self, plan, name, v, act=True):
        m = getattr(self, name)[0]
        raw = plan.conv(v, conv_desc(m))
        return plan.norm_act(raw, norm_desc(None), L.ACT_LRELU if act else L.ACT_NONE, SLOPE if act else 0.0)

    def u_predict(self, plan, name, v):
        raw = plan.conv(v, conv_desc(getattr(self, name)))
        return plan.norm_act(raw, norm_desc(None), L.ACT_NONE, 0.0)

    def u_deconv(self, plan, name, v):
        raw = plan.conv(v, conv_desc(getattr(self, name)[0]))
        return plan.norm_act(raw, norm_desc(None), L.ACT_LRELU, SLOPE)

    def u_upflow(self, plan, name, v):
        raw = plan.conv(v, conv_desc(getattr(self, name)))
        return plan.norm_act(raw, norm_desc(None), L.ACT_NONE, 0.0)

    def refine(self, plan, skips, top, inter=False):
        """The coarse-to-fine decoder (FlowNetC.py:100-126, FlowNetS.py:66-90, FlowNetSD.py:72-101)."""
        x = top
        flow = self.u_predict(plan, 'predict_flow6', x)
        for lvl in (5, 4, 3, 2):
            up = self.u_upflow(plan, 'upsampled_flow%d_to_%d' % (lvl + 1, lvl), flow)
            x = plan.concat([skips[lvl], self.u_deconv(plan, 'deconv%d' % lvl, x), up])
            flow = self.u_predict(plan, 'predict_flow%d' % lvl,
                                  self.u_conv(plan, 'inter_conv%d' % lvl, x, act=False) if inter else x)
        return flow

    def tail(self, plan, x):
        out = {}
        for lvl in (4, 5, 6):
            x = self.u_conv(plan, 'conv%d_1' % lvl, self.u_conv(plan, 'conv%d' % lvl, x))
            out[lvl] = x
        return out

    def _decoder_layers(self, with_bias_up, inter, pf):
        self.deconv5, self.deconv4 = _deconv(1024, 512), _deconv(1026, 256)
        self.deconv3, self.deconv2 = _deconv(770, 128), _deconv(386, 64)
        if inter:
            self.inter_conv5, self.inter_conv4 = _i_conv(1026, 512), _i_conv(770, 256)
            self.inter_conv3, self.inter_conv2 = _i_conv(386, 128), _i_conv(194, 64)
        for lvl, c in zip((6, 5, 4, 3, 2), pf):
            setattr(self, 'predict_flow%d' % lvl, _predict(c))
        for lvl in (6, 5, 4, 3):
            setattr(self, 'upsampled_flow%d_to_%d' % (lvl, lvl - 1), _upflow(with_bias_up))


class FlowNetC(_Sub):
    """networks/FlowNetC.py:14-131."""

    def __init__(self):
        super().__init__()
        self.conv1, self.conv2, self.conv3 = _conv(3, 64, 7, 2), _conv(64, 128, 5, 2), _conv(128, 256, 5, 2)
        self.conv_redir = _conv(256, 32, 1, 1)
        self.conv3_1 = _conv(473, 256)
        self.conv4, self.conv4_1 = _conv(256, 512, stride=2), _conv(512, 512)
        self.conv5, self.conv5_1 = _conv(512, 512, stride=2), _conv(512, 512)
        self.conv6, self.conv6_1 = _conv(512, 1024, stride=2), _conv(1024, 1024)
        self._decoder_layers(True, False, (1024, 1026, 770, 386, 194))

    def describe(self, plan, N, H, W):
        a = plan.input(0, N, 6, 0, 3, H, W)
        b = plan.input(0, N, 6, 3, 3, H, W)

        def stream(v):
            c2 = self.u_conv(plan, 'conv2', self.u_conv(plan, 'conv1', v))
            return c2, self.u_conv(plan, 'conv3', c2)
        c2a, c3a = stream(a)
        _, c3b = stream(b)
        corr = plan.correlation(c3a, c3b, 20, 1, 20, 1, 2, L.ACT_LRELU, SLOPE)          # FlowNetC.py:79-84
        c3 = self.u_conv(plan, 'conv3_1', plan.concat([self.u_conv(plan, 'conv_redir', c3a), corr]))
        t = self.tail(plan, c3)
        plan.export(self.refine(plan, {5: t[5], 4: t[4], 3: c3, 2: c2a}, t[6]), 1)


class FlowNetS(_Sub):
    """networks/FlowNetS.py:14-95 (12-channel evidence stack in)."""

    def __init__(self, input_channels=12):
        super().__init__()
        self.conv1, self.conv2, self.conv3 = _conv(input_channels, 64, 7, 2), _conv(64, 128, 5, 2), _conv(128, 256, 5, 2)
        self.conv3_1 = _conv(256, 256)
        self.conv4, self.conv4_1 = _conv(256, 512, stride=2), _conv(512, 512)
        self.conv5, self.conv5_1 = _conv(512, 512, stride=2), _conv(512, 512)
        self.conv6, self.conv6_1 = _conv(512, 1024, stride=2), _conv(1024, 1024)
        self._decoder_layers(False, False, (1024, 1026, 770, 386, 194))

    def describe(self, plan, N, H, W):
        # evidence stack (models.py:117): x (6) | resampled frame 1 (3) | flow / div_flow (2) | brightness error (1)
        stack = plan.concat([plan.input(0, N, 6, 0, 6, H, W), plan.input(1, N, 3, 0, 3, H, W), plan.input(2, N, 2, 0, 2, H, W),
                             plan.input(3, N, 1, 0, 1, H, W)])
        c2 = self.u_conv(plan, 'conv2', self.u_conv(plan, 'conv1', stack))
        c3 = self.u_conv(plan, 'conv3_1', self.u_conv(plan, 'conv3', c2))
        t = self.tail(plan, c3)
        plan.export(self.refine(plan, {5: t[5], 4: t[4], 3: c3, 2: c2}, t[6]), 4)


class FlowNetSD(_Sub):
    """networks/FlowNetSD.py:14-106."""

    def __init__(self):
        super().__init__()
        self.conv0 = _conv(6, 64)
        self.conv1, self.conv1_1 = _conv(64, 64, stride=2), _conv(64, 128)
        self.conv2, self.conv2_1 = _conv(128, 128, stride=2), _conv(128, 128)
        self.conv3, self.conv3_1 = _conv(128, 256, stride=2), _conv(256, 256)
        self.conv4, self.conv4_1 = _conv(256, 512, stride=2), _conv(512, 512)
        self.conv5, self.conv5_1 = _conv(512, 512, stride=2), _conv(512, 512)
        self.conv6, self.conv6_1 = _conv(512, 1024, stride=2), _conv(1024, 1024)
        self._decoder_layers(True, True, (1024, 512, 256, 128, 64))

    def describe(self, plan, N, H, W):
        c0 = self.u_conv(plan, 'conv0', plan.input(0, N, 6, 0, 6, H, W))
        c1 = self.u_conv(plan, 'conv1_1', self.u_conv(plan, 'conv1', c0))
        c2 = self.u_conv(plan, 'conv2_1', self.u_conv(plan, 'conv2', c1))
        c3 = self.u_conv(plan, 'conv3_1', self.u_conv(plan, 'conv3', c2))
        t = self.tail(plan, c3)
        plan.export(self.refine(plan, {5: t[5], 4: t[4], 3: c3, 2: c2}, t[6], inter=True), 1)


class FlowNetFusion(_Sub):
    """networks/FlowNetFusion.py:14-67 (11-channel stack in, full-resolution flow out)."""

    def __init__(self):
        super().__init__()
        self.conv0 = _conv(11, 64)
        self.conv1, self.conv1_1 = _conv(64, 64, stride=2), _conv(64, 128)
        self.conv2, self.conv2_1 = _conv(128, 128, stride=2), _conv(128, 128)
        self.deconv1, self.deconv0 = _deconv(128, 32), _deconv(162, 16)
        self.inter_conv1, self.inter_conv0 = _i_conv(162, 32), _i_conv(82, 16)
        self.predict_flow2, self.predict_flow1, self.predict_flow0 = _predict(128), _predict(32), _predict(16)
        self.upsampled_flow2_to_1, self.upsampled_flow1_to_0 = _upflow(True), _upflow(True)

    def describe(self, plan, N, H, W):
        # models.py:144: x[:, :3] | flownetsd_flow | flownets2_flow | |sd flow| | |s2 flow| | sd error | s2 error
        ins = [plan.input(0, N, 6, 0, 3, H, W), plan.input(1, N, 2, 0, 2, H, W), plan.input(2, N, 2, 0, 2, H, W)]
        ins += [plan.input(3 + i, N, 1, 0, 1, H, W) for i in range(4)]
        c0 = self.u_conv(plan, 'conv0', plan.concat(ins))
        c1 = self.u_conv(plan, 'conv1_1', self.u_conv(plan, 'conv1', c0))
        c2 = self.u_conv(plan, 'conv2_1', self.u_conv(plan, 'conv2', c1))
        flow2 = self.u_predict(plan, 'predict_flow2', c2)
        cat1 = plan.concat([c1, self.u_deconv(plan, 'deconv1', c2), self.u_upflow(plan, 'upsampled_flow2_to_1', flow2)])
        flow1 = self.u_predict(plan, 'predict_flow1', self.u_conv(plan, 'inter_conv1', cat1, act=False))
        cat0 = plan.concat([c0, self.u_deconv(plan, 'deconv0', cat1), self.u_upflow(plan, 'upsampled_flow1_to_0', flow1)])
        plan.export(self.u_predict(plan, 'predict_flow0', self.u_conv(plan, 'inter_conv0', cat0, act=False)), 7)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def resize(x, H, W, mode='bilinear', use_scale_factor=False, mul=1.0, pre_div=1.0, div=None):
    """F.interpolate(x * mul (or x / pre_div), size / scale_factor, mode) [, and the same / div]; (.., h, w) fp32 CUDA."""
    ops._chk(x)
    h, w = x.shape[-2:]
    planes = x.numel() // (h * w)
    out = torch.empty(tuple(x.shape[:-2]) + (H, W), device=x.device, dtype=torch.float32)
    out_div = torch.empty_like(out) if div is not None else None
    ops._ck(L.lib().v2v_resize(_p(x), _p(out), _p(out_div), planes, h, w, H, W, 0 if mode == 'bilinear' else 1,
                               int(use_scale_factor), mul, pre_div, div if div is not None else 1.0, L.current_stream_ptr()))
    return (out, out_div) if div is not None else out


class FlowNet2(_Planned):
    """models/flownet2_pytorch/models.py:30-160 (vid2vid instantiates it with batchNorm=False, div_flow=20, rgb_max=1)."""

    precision = 'precise'

    def __init__(self, args=None, batchNorm=False, div_flow=20.):
        super().__init__()
        if batchNorm:
            raise NotImplementedError('vid2vid uses FlowNet2 without batch norm (models.py:32)')
        self.div_flow = div_flow
        self.rgb_max = getattr(args, 'rgb_max', 1.0) if args is not None else 1.0
        self.flownetc = FlowNetC()
        self.flownets_1 = FlowNetS()
        self.flownets_2 = FlowNetS()
        self.flownets_d = FlowNetSD()
        self.flownetfusion = FlowNetFusion()
        for m in self.modules():                                      # models.py:68-77
            if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
                if m.bias is not None:
                    nn.init.uniform_(m.bias)
                nn.init.xavier_uniform_(m.weight)

    def _sub_plan(self, name, N, H, W, dev):
        sub = getattr(self, name)
        return self._get_plan((name, N, H, W), dev, lambda p: sub.describe(p, N, H, W))

    def _evidence(self, x, x1, flow):
        """models.py:113-116: frame 1 warped towards frame 0 and the brightness-error magnitude."""
        warped = ops.resample2d(x1, flow)
        b, _, h, w = x.shape
        diff = torch.empty_like(warped)
        ops._ck(L.lib().v2v_sub_channels(_p(x), _p(warped), _p(diff), b, 6, 0, 3, h, w, L.current_stream_ptr()))
        return warped, ops.channelnorm(diff)

    def forward_frames(self, f0, f1, bstride, cstride, B, H, W):
        dev = f0.device
        if H % 64 or W % 64:
            raise RuntimeError('FlowNet2 needs H and W divisible by 64 (got %dx%d)' % (H, W))
        new = lambda c, h, w: torch.empty((B, c, h, w), device=dev, dtype=torch.float32)
        x, x1, ws = new(6, H, W), new(3, H, W), torch.empty(B * 3, device=dev, dtype=torch.float32)
        ops._ck(L.lib().v2v_flownet_prep(_p(f0), _p(f1), bstride, cstride, _p(x), _p(x1), _p(ws), B, H, W, float(self.rgb_max),
                                         L.current_stream_ptr()))
        q = (H // 4, W // 4)
        flow2 = new(2, *q)
        self._sub_plan('flownetc', B, H, W, dev).run([x, flow2], self.use_cuda_graph)
        flow, flow_div = resize(flow2, H, W, 'bilinear', True, mul=self.div_flow, div=self.div_flow)     # models.py:106-107
        for name, mode in (('flownets_1', 'bilinear'), ('flownets_2', 'nearest')):
            warped, err = self._evidence(x, x1, flow)
            flow2 = new(2, *q)
            self._sub_plan(name, B, H, W, dev).run([x, warped, flow_div, err, flow2], self.use_cuda_graph)
            flow, flow_div = resize(flow2, H, W, mode, True, mul=self.div_flow, div=self.div_flow)       # :118-119 / :130-131
        flow_s = flow
        flow2 = new(2, *q)
        self._sub_plan('flownets_d', B, H, W, dev).run([x, flow2], self.use_cuda_graph)
        flow_sd = resize(flow2, H, W, 'nearest', True, pre_div=self.div_flow)                            # :142-143
        _, err_s = self._evidence(x, x1, flow_s)
        _, err_sd = self._evidence(x, x1, flow_sd)
        out = new(2, H, W)
        self._sub_plan('flownetfusion', B, H, W, dev).run(
            [x, flow_sd, flow_s, ops.channelnorm(flow_sd), ops.channelnorm(flow_s), err_sd, err_s, out], self.use_cuda_graph)
        return out

    def forward(self, inputs):
        """inputs (B, 3, 2, H, W) -> flow (B, 2, H, W) in pixels (models.py:96-160, eval mode)."""
        self._require_cuda(inputs)
        inputs = inputs.contiguous()
        B, _, _, H, W = inputs.shape
        hw = H * W
        f1 = inputs.view(-1)[hw:]
        return self.forward_frames(inputs, f1, 6 * hw, 2 * hw, B, H, W)


class FlowNet(nn.Module):
    """models/flownet.py:12-62: flowNet(input_A, input_B) -> (flow, conf), 4-D or 5-D inputs, always under no_grad."""

    def name(self):
        return 'FlowNet'

    def initialize(self, opt):
        self.opt = opt
        self.gpu_ids = getattr(opt, 'gpu_ids', [0])
        dev = torch.device('cuda', self.gpu_ids[0] if len(self.gpu_ids) else torch.cuda.current_device())
        self.flowNet = FlowNet2().to(dev)
        import os
        ckpt = 'models/flownet2_pytorch/FlowNet2_checkpoint.pth.tar'                  # flownet.py:19-20
        if os.path.exists(ckpt):
            self.flowNet.load_state_dict(torch.load(ckpt, map_location=dev)['state_dict'])
        elif not getattr(opt, 'synthetic_weights', False):
            raise FileNotFoundError('%s not found (set opt.synthetic_weights for random-weight benchmarking)' % ckpt)
        return self

    def forward(self, input_A, input_B):
        with torch.no_grad():
            size = input_A.size()
            assert len(size) in (4, 5)
            if len(size) == 5:
                b, n, c, h, w = size
                flow, conf = self.compute_flow_and_conf(input_A.contiguous().view(-1, c, h, w), input_B.contiguous().view(-1, c, h, w))
                return flow.view(b, n, 2, h, w), conf.view(b, n, 1, h, w)
            return self.compute_flow_and_conf(input_A, input_B)

    def compute_flow_and_conf(self, im1, im2):
        """flownet.py:43-58."""
        assert im1.size()[1] == 3 and im1.size() == im2.size()
        im1, im2 = im1.contiguous().float(), im2.contiguous().float()
        old_h, old_w = im1.size()[2], im1.size()[3]
        new_h, new_w = old_h // 64 * 64, old_w // 64 * 64
        if old_h != new_h:
            im1, im2 = resize(im1, new_h, new_w), resize(im2, new_h, new_w)
        B, _, H, W = im1.shape
        flow = self.flowNet.forward_frames(im1, im2, 3 * H * W, H * W, B, H, W)
        warped = ops.resample2d(im2, flow)
        conf = torch.empty((B, 1, H, W), device=im1.device, dtype=torch.float32)
        ops._ck(L.lib().v2v_flow_conf(_p(im1), _p(warped), _p(conf), B, 3, H, W, 0.02, L.current_stream_ptr()))
        if old_h != new_h:
            flow = resize(flow, old_h, old_w, mul=float(old_h) / new_h)
            conf = resize(conf, old_h, old_w)
        return flow, conf
