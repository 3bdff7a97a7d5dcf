"""TEST INFRASTRUCTURE -- not product code (only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import oracle/).

CPU restatement of the reference optical-flow network used to build the training targets (SURVEY 8 rows a14 / a15):
FlowNet2 = FlowNetC -> FlowNetS -> FlowNetS, in parallel FlowNetSD, merged by FlowNetFusion
(models/flownet2_pytorch/models.py:30-160), and the vid2vid wrapper that turns it into (flow, confidence)
(models/flownet.py:27-62).  Functional PyTorch over a reference-layout state_dict; the three native ops come from
oracle/flowops_oracle.c.  Pinned against the unmodified reference modules in tests/test_flownet2_oracle.py (build
container) and through tests/golden/flownet2_small.npz elsewhere.

Layer vocabulary of the reference (networks/submodules.py:7-41), all without batch norm as vid2vid instantiates it:
  conv(k, s)      Conv2d(k, stride s, padding (k-1)//2, bias) + LeakyReLU(0.1)      keys  <name>.0.weight / .0.bias
  i_conv          Conv2d(3, 1, 1, bias), no activation                               keys  <name>.0.weight / .0.bias
  predict_flow    Conv2d(C, 2, 3, 1, 1, bias)                                        keys  <name>.weight / .bias
  deconv          ConvTranspose2d(4, 2, 1, bias) + LeakyReLU(0.1)                    keys  <name>.0.weight / .0.bias
  upsampled_flow  ConvTranspose2d(2, 2, 4, 2, 1), bias only in FlowNetC / SD / Fusion
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import flowops

DIV_FLOW = 20.0      # models.py:32 (div_flow), FlowNetC.py:15
SLOPE = 0.1


def _np(t):
    return np.ascontiguousarray(t.detach().cpu().numpy(), dtype=np.float32)


def correlation(a, b):
    """FlowNetC.py:30: Correlation(pad_size=20, kernel_size=1, max_displacement=20, stride1=1, stride2=2)."""
    return torch.from_numpy(flowops.correlation(_np(a), _np(b), 20, 1, 20, 1, 2))


def resample2d(img, flow):
    """resample2d_package/resample2d.py:5-21 (kernel_size 1): bilinear backward warp of img by flow."""
    return torch.from_numpy(flowops.resample2d(_np(img), _np(flow), 1))


def channelnorm(x):
    """channelnorm_package/channelnorm.py:5-16 (norm_deg 2): L2 norm over channels, one output channel."""
    return torch.from_numpy(flowops.channelnorm(_np(x), 2))


class _Net:
    """Parameter view of one sub-network: sd keys under `prefix`."""

    def __init__(self, sd, prefix):
        self.sd, self.p = sd, prefix

    def _wb(self, key):
        return self.sd[self.p + key + '.weight'], self.sd.get(self.p + key + '.bias')

    def conv(self, name, x, stride=1, act=True):
        w, b = self._wb(name + '.0')
        y = F.conv2d(x, w, b, stride=stride, padding=(w.shape[-1] - 1) // 2)
        return F.leaky_relu(y, SLOPE) if act else y

    def predict(self, name, x):
        w, b = self._wb(name)
        return F.conv2d(x, w, b, stride=1, padding=1)

    def deconv(self, name, x):
        w, b = self._wb(name + '.0')
        return F.leaky_relu(F.conv_transpose2d(x, w, b, stride=2, padding=1), SLOPE)

    def up_flow(self, name, x):
        w, b = self._wb(name)
        return F.conv_transpose2d(x, w, b, stride=2, padding=1)

    def refine(self, skips, top, inter=False):
        """The coarse-to-fine decoder shared by FlowNetC / S / SD (FlowNetC.py:100-126, FlowNetS.py:66-90,
        FlowNetSD.py:72-101): starting from conv6, at every level concatenate (encoder skip, deconv of the running
        feature, 2x-upsampled flow) and predict the next flow -- through an inter_conv first in FlowNetSD."""
        x = top
        flow = self.predict('predict_flow6', x)
        for lvl in (5, 4, 3, 2):
            up = self.up_flow('upsampled_flow%d_to_%d' % (lvl + 1, lvl), flow)
            x = torch.cat((skips[lvl], self.deconv('deconv%d' % lvl, x), up), 1)
            flow = self.predict('predict_flow%d' % lvl, self.conv('inter_conv%d' % lvl, x, act=False) if inter else x)
        return flow

    def tail(self, x):
        """conv4 .. conv6_1 (stride-2 conv followed by a stride-1 conv at each level), returned per level."""
        out = {}
        for lvl in (4, 5, 6):
            x = self.conv('conv%d_1' % lvl, self.conv('conv%d' % lvl, x, stride=2))
            out[lvl] = x
        return out


def flownet_c(sd, prefix, x):
    """FlowNetC.forward (FlowNetC.py:66-131), eval mode: returns flow2 at 1/4 resolution."""
    n = _Net(sd, prefix)

    def stream(img):
        c1 = n.conv('conv1', img, stride=2)
        c2 = n.conv('conv2', c1, stride=2)
        return c2, n.conv('conv3', c2, stride=2)
    c2a, c3a = stream(x[:, 0:3])
    _, c3b = stream(x[:, 3:])
    corr = F.leaky_relu(correlation(c3a, c3b), SLOPE)
    c3 = n.conv('conv3_1', torch.cat((n.conv('conv_redir', c3a), corr), 1))
    t = n.tail(c3)
    return n.refine({5: t[5], 4: t[4], 3: c3, 2: c2a}, t[6])


def flownet_s(sd, prefix, x):
    """FlowNetS.forward (FlowNetS.py:58-95), eval mode."""
    n = _Net(sd, prefix)
    c2 = n.conv('conv2', n.conv('conv1', x, stride=2), stride=2)
    c3 = n.conv('conv3_1', n.conv('conv3', c2, stride=2))
    t = n.tail(c3)
    return n.refine({5: t[5], 4: t[4], 3: c3, 2: c2}, t[6])


def flownet_sd(sd, prefix, x):
    """FlowNetSD.forward (FlowNetSD.py:64-106), eval mode: small-displacement network, 3x3 filters throughout."""
    n = _Net(sd, prefix)
    c0 = n.conv('conv0', x)
    c1 = n.conv('conv1_1', n.conv('conv1', c0, stride=2))
    c2 = n.conv('conv2_1', n.conv('conv2', c1, stride=2))
    c3 = n.conv('conv3_1', n.conv('conv3', c2, stride=2))
    t = n.tail(c3)
    return n.refine({5: t[5], 4: t[4], 3: c3, 2: c2}, t[6], inter=True)


def flownet_fusion(sd, prefix, x):
    """FlowNetFusion.forward (FlowNetFusion.py:48-67): full-resolution flow from the 11-channel evidence stack."""
    n = _Net(sd, prefix)
    c0 = n.conv('conv0', x)
    c1 = n.conv('conv1_1', n.conv('conv1', c0, stride=2))
    c2 = n.conv('conv2_1', n.conv('conv2', c1, stride=2))
    flow2 = n.predict('predict_flow2', c2)
    cat1 = torch.cat((c1, n.deconv('deconv1', c2), n.up_flow('upsampled_flow2_to_1', flow2)), 1)
    flow1 = n.predict('predict_flow1', n.conv('inter_conv1', cat1, act=False))
    cat0 = torch.cat((c0, n.deconv('deconv0', cat1), n.up_flow('upsampled_flow1_to_0', flow1)), 1)
    return n.predict('predict_flow0', n.conv('inter_conv0', cat0, act=False))


def _evidence(x, flow):
    """Warp frame 1 towards frame 0 with `flow`; brightness error magnitude (models.py:113-116)."""
    warped = resample2d(x[:, 3:], flow)
    return warped, channelnorm(x[:, :3] - warped)


def flownet2(sd, inputs, rgb_max=1.0):
    """FlowNet2.forward (models.py:97-160).  inputs: (B, 3, 2, H, W) image pair, H and W multiples of 64."""
    b, c = inputs.shape[:2]
    mean = inputs.reshape(b, c, -1).mean(-1).view(b, c, 1, 1, 1)                 # per sample and colour, over both frames
    x = (inputs - mean) / rgb_max
    x = torch.cat((x[:, :, 0], x[:, :, 1]), 1)

    def up4(t, mode):
        return F.interpolate(t, scale_factor=4, mode=mode, **({'align_corners': False} if mode == 'bilinear' else {}))

    flow = up4(flownet_c(sd, 'flownetc.', x) * DIV_FLOW, 'bilinear')
    for name in ('flownets_1.', 'flownets_2.'):
        warped, err = _evidence(x, flow)
        stack = torch.cat((x, warped, flow / DIV_FLOW, err), 1)                   # 6 + 3 + 2 + 1 = 12 channels
        flow2 = flownet_s(sd, name, stack) * DIV_FLOW
        flow = up4(flow2, 'bilinear' if name == 'flownets_1.' else 'nearest')   # models.py:50,59 (upsample2 / upsample4)
    flow_s = flow
    flow_sd = up4(flownet_sd(sd, 'flownets_d.', x) / DIV_FLOW, 'nearest')        # models.py:142 divides here
    _, err_s = _evidence(x, flow_s)
    _, err_sd = _evidence(x, flow_sd)
    stack = torch.cat((x[:, :3], flow_sd, flow_s, channelnorm(flow_sd), channelnorm(flow_s), err_sd, err_s), 1)
    return flownet_fusion(sd, 'flownetfusion.', stack)


def flow_and_conf(sd, im1, im2):
    """FlowNet.compute_flow_and_conf (models/flownet.py:43-58): flow of im1 -> im2 and the 0/1 confidence mask
    |im1 - warp(im2, flow)|^2 < 0.02; inputs whose height is not a multiple of 64 are resized for the network and the
    flow scaled back by old_h / new_h (the reference keys both the test and the scale on the height only)."""
    old_h, old_w = im1.shape[2:]
    new_h, new_w = old_h // 64 * 64, old_w // 64 * 64
    if old_h != new_h:
        im1 = F.interpolate(im1, size=(new_h, new_w), mode='bilinear', align_corners=False)
        im2 = F.interpolate(im2, size=(new_h, new_w), mode='bilinear', align_corners=False)
    flow = flownet2(sd, torch.stack((im1, im2), 2))
    d = im1 - resample2d(im2, flow)
    conf = ((d * d).sum(1, keepdim=True) < 0.02).float()
    if old_h != new_h:
        flow = F.interpolate(flow, size=(old_h, old_w), mode='bilinear', align_corners=False) * old_h / new_h
        conf = F.interpolate(conf, size=(old_h, old_w), mode='bilinear', align_corners=False)
    return flow, conf


def det_state_dict(keys_shapes, seed=0):
    """Weights that depend only on (seed, key, shape): Xavier-uniform filters, as the reference initialises them
    (models.py:68-77), and small positive biases.  Lets a machine without the reference rebuild the exact 162 M parameters the golden fixture
    was produced with from the 220-entry key list in tests/golden/flownet2_keys.json."""
    import zlib
    sd = {}
    for name, shape in keys_shapes:
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(name.encode())) & 0x7FFFFFFF)
        if len(shape) == 4:
            rf = shape[2] * shape[3]
            a = (6.0 / ((shape[0] + shape[1]) * rf)) ** 0.5
            sd[name] = (torch.rand(shape, generator=g) * 2 - 1) * a
        else:
            sd[name] = torch.rand(shape, generator=g) * 0.1
    return sd
