"""GPU parity of the conv kernel configurations that product paths outside bench.py run and no other parity case reaches
(tests/product_plans.py lists the plans; tests/test_conv_census.py fails when one of their configurations goes uncovered or
a case here stops being needed): the face first frame's Encoder and Global_with_z, the pose training step with the face
discriminator (generator scales, netD / netD_f / netD_T towers), and the VGG19 loss.

Forward cases mirror a layer at the grid that reproduces its configuration, through test_gpu_conv's runner and tolerances:
fp64 in precise mode, bf16-emulated fp32 in fast mode.  Backward cases are smooth units as in test_gpu_backward_variants (conv,
conv + BatchNorm, transposed conv + BatchNorm; no activation gate that could flip between our forward and the reference's),
their input, weight and bias gradients held to float64 autograd at relative L2 <= 1e-4 and max|d| <= 1e-3 max|ref|.  The VGG
cases freeze their weights as Vgg19 does: the loss needs only the data gradient, and with no parameter asking for one the plan
launches no weight gradient."""
import pytest
import torch
import torch.nn as nn

import test_gpu_backward as TB
import test_gpu_backward_variants as TV
import test_gpu_conv as TC
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import make_opt

pytestmark = pytest.mark.gpu

BN = NW.get_norm_layer('batch')
IN = NW.get_norm_layer('instance')
MODES = TC.MODES


def _c(a, b, k, s, p):
    return nn.Conv2d(a, b, k, stride=s, padding=p)


def _vgg(a, b):
    return [_c(a, b, 3, 1, 1), nn.ReLU(True)]        # a Vgg19 conv: zero padding 1, bias, ReLU fused in the epilogue


LRELU = lambda: nn.LeakyReLU(0.2, True)


# name, layer list builder, head builder (None: no head), input shape, modes
FWD_CASES = [
    # face Encoder at 512x512 (instance norm throughout): the 64 -> 32 transposed conv at 128x128 on the epilogue warpgroup
    ('enc_up_64_32_128x128', lambda: NW._up(64, 32, IN), None, (1, 64, 128, 128), MODES),
    # its 16 -> 16 7x7 tanh head at 512x512: resident row tiles in precise mode, a 2-D patch of all 49 taps in fast mode
    ('enc_head_16_16_512x512', lambda: NW._up(32, 16, IN), lambda: NW._head(16, 16, nn.Tanh()), (1, 32, 256, 256), MODES),
    # Global_with_z's 31 -> 64 7x7 stem (15 input + 16 feature channels) at 512x512: M blocking 2, 32-channel K blocks; the
    # pose generator's finer 18 -> 64 training stem at 512x512 lowers the precise configuration too
    ('stem_31_64_mg2_kc32_512x512', lambda: NW._stem(31, 64, IN), None, (1, 31, 512, 512), MODES),
    # VGG19 at 1024x512: relu1_1 / conv1_2 (resident weights, 16- and 32-channel K blocks, epilogue warpgroup), conv2_1 on the
    # decoupled rings, and a 256 -> 512 conv4_1 on the rings at 64x128
    ('vgg_3_64_64_512x1024', lambda: _vgg(3, 64) + _vgg(64, 64), None, (1, 3, 512, 1024), ['precise']),
    ('vgg_64_128_ring2_256x512', lambda: _vgg(64, 128), None, (1, 64, 256, 512), ['precise']),
    ('vgg_256_512_ring2_64x128', lambda: _vgg(256, 512), None, (1, 256, 64, 128), ['precise']),
    # netD's tower 1 at 512x512 (256x256 input): the 9 -> 64 first layer at 129x129 with resident weights
    ('d_first_9_64_129x129', lambda: [_c(9, 64, 4, 2, 2), LRELU()], None, (1, 9, 256, 256), ['precise']),
    # netD_f / netD tower 0: the 512 -> 1 logit head at 19x19, too small a grid for the kx-GEMM head
    ('d_logit_head_512_1_19x19', lambda: [_c(256, 512, 4, 1, 2), BN(512), LRELU()], lambda: [_c(512, 1, 4, 1, 2)], (1, 256, 17, 17),
     ['precise']),
]


@pytest.mark.parametrize('name,build,head,shape,mode', [c[:4] + (m,) for c in FWD_CASES for m in c[4]],
                         ids=['%s-%s' % (c[0], m) for c in FWD_CASES for m in c[4]])
def test_product_conv(name, build, head, shape, mode):
    if head is None:
        out, ref = TC._run(build(), TC._x(*shape), mode=mode)
        TC._check(out, ref, name, mode=mode)
    else:
        out, ref = TC._run(build(), TC._x(*shape), head(), 1.0, mode=mode)
        TC._check(out, ref, name, ulps=4.0, mean_tol=5e-3, mode=mode)       # test_gpu_conv's head tolerance


# name, layer list builder, input shape, weights frozen
BWD_CASES = [
    # the pose generator at 512x512: the coarser scale's 18 -> 128 stem at 256x256
    ('g_stem_18_128_256x256', lambda: [nn.ReflectionPad2d(3), _c(18, 128, 7, 1, 0), BN(128)], (1, 18, 256, 256), False),
    # its 1024-channel layers at 32x32: stride-2 512 -> 1024, a residual block's 1024 -> 1024 3x3 and the 1024 -> 512
    # transposed conv, whose weight gradients take a whole 32-pixel-row K chunk per unit (no K split)
    ('g_1024_32x32_s2_c3_up', lambda: [_c(512, 1024, 3, 2, 1), BN(1024), nn.ReflectionPad2d(1), _c(1024, 1024, 3, 1, 0), BN(1024),
                                       TV._t(1024, 512), BN(512)], (1, 512, 64, 64), False),
    # netD_f on the 128x128 face crop (and netD's tower 0 at 128x128): 128 -> 256 stride 2 at 17x17, 256 -> 512 at 18x18 and
    # the 512 -> 1 logit at 19x19, every weight gradient with a ragged last row segment
    ('d_crop_128_256_512_1', lambda: [_c(128, 256, 4, 2, 2), BN(256), _c(256, 512, 4, 1, 2), BN(512), _c(512, 1, 4, 1, 2)],
     (1, 128, 33, 33), False),
    # netD's tower 2 at 512x512: the 512 -> 1 logit at 67x67, whose data gradient is a 4-tap row-tile conv
    ('d2_256_512_1_67x67', lambda: [_c(256, 512, 4, 1, 2), BN(512), _c(512, 1, 4, 1, 2)], (1, 256, 65, 65), False),
    # VGG19 at 1024x512: the data gradients of conv1_1 (into the generated image) and conv2_1
    ('vgg_3_64_dgrad_512x1024', lambda: [_c(3, 64, 3, 1, 1)], (1, 3, 512, 1024), True),
    ('vgg_64_128_dgrad_256x512', lambda: [_c(64, 128, 3, 1, 1)], (1, 64, 256, 512), True),
]


@pytest.mark.parametrize('name,build,shape,frozen', BWD_CASES, ids=[c[0] for c in BWD_CASES])
def test_product_backward(name, build, shape, frozen):
    runner = TV._runner(build, None, 1.0, False)
    if frozen:
        runner.requires_grad_(False)
    names, ours, refs, out, ref = TB._grads(runner, TV._input(shape, False))
    TB._cmp(name + ' forward', out.detach(), ref.detach(), tol=3e-4, l2=1e-4)
    if frozen:
        assert all(p.grad is None for p in runner.parameters()), name
        names, ours, refs = names[:1], ours[:1], refs[:1]
    bad = []
    for n, o, r in zip(names, ours, refs):
        if n.endswith('.bias') and r.abs().max().item() < 1e-6:
            # zero in the reference (a conv bias in front of a norm): ours is fp32 cancellation noise, held to MAX relative to
            # the same layer's weight gradient, as test_gpu_backward_variants holds it
            w = refs[names.index(n[:-len('bias')] + 'weight')].abs().max().item()
            assert o.abs().max().item() <= TV.MAX * w, (n, o.abs().max().item(), w)
            continue
        try:
            TB._cmp('%s d/d %s' % (name, n), o, r, tol=TV.MAX, l2=TV.L2)
        except AssertionError as e:
            bad.append(str(e)[:160])
    assert not bad, bad


@pytest.mark.parametrize('mode', MODES)
def test_first_frame_networks_follow_the_default_precision(mode):
    """The first-frame generators pin no arithmetic mode: they build their plans in the mode every generator defaults to."""
    saved = NW.DEFAULT_PRECISION
    NW.set_default_precision(mode)
    try:
        enc = NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []).cuda()
        opt = make_opt(dataset_mode='face', label_nc=0, input_nc=15, feat_num=16, gpu_ids=[0])
        gz = NW.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt).cuda()
        inst = torch.zeros(1, 1, 64, 64, device='cuda')
        with torch.no_grad():
            z = enc(TC._x(1, 3, 64, 64).cuda(), inst)
            gz(TC._x(1, 15, 64, 64).cuda(), z)
        for net in (enc, gz):
            keys = list(net._plans())
            assert keys and all(k[-1] == mode for k in keys), (type(net).__name__, keys)
    finally:
        NW.set_default_precision(saved)
