"""GPU parity of the convolution path, one unit at a time, through the C-ABI plan runtime, in both arithmetic modes.
  precise (split-bf16, 3 MMAs; the default product mode): reference = the same layers evaluated by PyTorch in fp64
          with no rounding anywhere; tolerance |d| <= 2e-4 * max(1, |ref|), mean |d| <= 3e-5 (fp32-class).
  fast    (bf16 operands): reference = PyTorch fp32 with bf16 rounding at the points where the CUDA path stores bf16
          (tests/bf16_emul.py); agreement must be within ~1 bf16 ulp (tolerance written below)."""
import os

import pytest
import torch
import torch.nn as nn

import bf16_emul as E
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import det_fill_

pytestmark = pytest.mark.gpu

BN = NW.get_norm_layer('batch')
IN = NW.get_norm_layer('instance')


SIMT = os.environ.get('V2V_CONV_IMPL') == 'simt'   # cross-check kernel: statistics come from the bf16-stored raws


PRECISE_TOL, PRECISE_MEAN = 2e-4, 3e-5


def _check(out, ref, name, ulps=2.0, mean_tol=2e-3, mode='fast', scale=1.0):
    if SIMT:
        ulps, mean_tol = ulps * 3, mean_tol * 3
    out, ref = out.double().cpu(), ref.double().cpu()
    assert out.shape == ref.shape, (out.shape, ref.shape)
    assert torch.isfinite(out).all(), name + ': non-finite output'
    diff = (out - ref).abs()
    if mode == 'precise':
        tol = PRECISE_TOL * scale * torch.clamp(ref.abs(), min=1.0)
        worst = (diff / tol).max().item()
        print('%-28s [precise] max|d|=%.3e mean|d|=%.3e worst/tol=%.2f' % (name, diff.max().item(), diff.mean().item(), worst))
        assert diff.mean().item() < PRECISE_MEAN * scale, name
        assert worst <= 1.0, '%s: max |d| %.3e beyond the fp32-class tolerance' % (name, diff.max().item())
        return
    tol = ulps * (2.0 ** -8) * torch.clamp(ref.abs(), min=1.0)     # bf16 has 8 significand bits
    worst = (diff / tol).max().item()
    print('%-28s max|d|=%.3e mean|d|=%.3e worst/tol=%.2f' % (name, diff.max().item(), diff.mean().item(), worst))
    assert diff.mean().item() < mean_tol, name
    frac_bad = (diff > tol).float().mean().item()
    assert frac_bad < (2e-2 if SIMT else 1e-3), '%s: %.4f%% of elements beyond %.1f bf16 ulp' % (name, 100 * frac_bad, ulps)


def _run(mods, x, head=None, head_scale=1.0, seed=1, mode='fast', exact=False):
    runner = det_fill_(NW.SequentialRunner(mods, head, head_scale), seed=seed).cuda()
    runner.precision = mode
    runner.input_exact_bf16 = exact
    xd = x.cuda()
    E.ROUND[0] = (mode == 'fast')
    try:
        with torch.no_grad():
            out = runner(xd)
            out2 = runner(xd)          # second call replays the CUDA graph
            xr = E.r16(xd)
            ref = E.run_units(list(runner.seq), xr)
            if head is not None:
                ref = E.run_head(list(runner.head), ref, head_scale)
    finally:
        E.ROUND[0] = True
    assert torch.equal(out, out2), 'graph replay differs from eager run'
    return out, ref


def _x(n, c, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, c, h, w, generator=g)


def _label_x(n, c, h, w, seed=0):
    """What encode_input feeds the finest scale: per frame, a one-hot map over 35 labels and a 0/1 instance-edge channel
    (c = 36 x frames).  Every element is exact in bf16."""
    assert c % 36 == 0
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(n, c // 36, 36, h, w)
    x.scatter_(2, torch.randint(0, 35, (n, c // 36, 1, h, w), generator=g), 1.0)
    x[:, :, 35] = (torch.rand(n, c // 36, h, w, generator=g) < 0.2).float()
    return x.view(n, c, h, w)


CASES = [
    # name, layer list builder, input shape
    ('c3s1_reflect_64_128_32x64', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 128, 3), BN(128), nn.ReLU(True)], (1, 64, 32, 64)),
    ('c3s1_rowtile_R3_8x160', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)], (1, 64, 8, 160)),
    ('c7_stem_R7_108_32', lambda: NW._stem(108, 32, BN), (1, 108, 12, 136)),
    ('c7_stem_small_map', lambda: NW._stem(6, 32, BN), (1, 6, 16, 32)),
    ('c3s2_zero_64_128', lambda: NW._down(64, 128, BN), (1, 64, 32, 64)),
    ('c3s2_odd_extent', lambda: NW._down(32, 64, BN), (1, 32, 18, 30)),
    ('deconv_128_64', lambda: NW._up(128, 64, BN), (1, 128, 16, 32)),
    ('deconv_wide', lambda: NW._up(64, 32, BN), (1, 64, 8, 80)),
    ('resblock_128', lambda: [NW.ResnetBlock(128, 'reflect', BN)], (1, 128, 16, 32)),
    ('resblock_x2_instance', lambda: [NW.ResnetBlock(64, 'reflect', IN), NW.ResnetBlock(64, 'reflect', IN)], (2, 64, 16, 16)),
    ('batch2_bn', lambda: NW._down(64, 64, BN) + [NW.ResnetBlock(64, 'reflect', BN)], (2, 64, 16, 32)),
    ('cout_16_cin_16', lambda: NW._stem(16, 16, BN) + NW._down(16, 32, BN), (1, 16, 16, 40)),
    ('d_first_layer_lrelu', lambda: [nn.Conv2d(39, 64, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True)], (2, 39, 32, 48)),
    ('c3_1024_1024_32x64', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(1024, 1024, 3), BN(1024), nn.ReLU(True)], (1, 1024, 32, 64)),
    ('c3_512_512_16x32', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(512, 512, 3), BN(512), nn.ReLU(True)], (1, 512, 16, 32)),
    # persistent paths: more tiles than SMs, resident / streamed weights, weight-set changes inside a CTA
    ('mt_deconv_resident', lambda: NW._up(64, 32, BN), (1, 64, 64, 320)),
    ('mt_c3_resident_R3', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)], (1, 64, 96, 256)),
    ('mt_c3_stream_R3', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 96, 256)),
    ('mt_c3_two_ntiles_resident', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 256, 3), BN(256), nn.ReLU(True)], (1, 64, 96, 256)),
    ('mt_s2', lambda: NW._down(32, 64, BN), (1, 32, 160, 512)),
    ('mt_stem_R7', lambda: NW._stem(108, 32, BN), (1, 108, 80, 256)),
    ('mt_stem_R7_cout128', lambda: NW._stem(108, 128, BN), (1, 108, 80, 256)),
    ('mt_batch2_resblock', lambda: [NW.ResnetBlock(64, 'reflect', BN)], (2, 64, 48, 256)),
    # streamed weights with M blocking (several accumulators per weight pass), incl. a unit that straddles two images
    ('mg2_stream_c128', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 160, 512)),
    ('mg4_stem', lambda: NW._stem(108, 32, BN), (1, 108, 256, 640)),
    ('mg2_stem_batch2_straddle', lambda: NW._stem(108, 16, BN), (2, 108, 107, 384)),
    ('mg4_stem_108_48', lambda: NW._stem(108, 48, BN), (1, 108, 160, 512)),
    ('mg2_bn96_stem_108_96', lambda: NW._stem(108, 96, BN), (1, 108, 160, 512)),
    ('mg_stem_batch2_instance', lambda: NW._stem(108, 32, IN), (2, 108, 80, 512)),
    ('mg_stem_108_192_ntiles', lambda: NW._stem(108, 192, BN), (1, 108, 160, 512)),
    # 16- and 32-channel K blocks (32-byte / 64-byte swizzled rows), with and without tap reuse
    ('kc16_stem_R7', lambda: NW._stem(6, 32, BN), (1, 6, 12, 136)),
    ('kc16_stem_R7_mt', lambda: NW._stem(6, 32, BN), (1, 6, 80, 256)),
    ('kc32_c3_R3', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(32, 32, 3), BN(32), nn.ReLU(True)], (1, 32, 8, 160)),
    ('kc32_resblock_mt', lambda: [NW.ResnetBlock(32, 'reflect', BN)], (1, 32, 96, 256)),
    ('kc16_s2_then_kc32_deconv', lambda: NW._down(16, 32, BN) + NW._up(32, 16, BN), (1, 16, 32, 64)),
    ('kc16_resblock_small', lambda: [NW.ResnetBlock(16, 'reflect', BN)], (1, 16, 16, 32)),
    ('kc32_s2_mt', lambda: NW._down(32, 64, BN), (1, 32, 160, 512)),
    # 2-D patch mode (16x8 tiles, one patch for all taps): ragged edges, batch straddle, halved N tile with resident
    # weights, 64-byte rows with streamed weights, 49 taps from one patch
    ('p2d_ragged_c64', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)], (1, 64, 30, 52)),
    ('p2d_batch2_c32_zero_pad', lambda: [nn.Conv2d(32, 64, 3, padding=1), BN(64), nn.ReLU(True)], (2, 32, 48, 72)),
    ('p2d_bn64_resident_c128', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(128, 128, 3), BN(128), nn.ReLU(True)], (1, 128, 192, 512)),
    ('p2d_stream_kc32_c256', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(256, 256, 3), BN(256), nn.ReLU(True)], (1, 256, 32, 64)),
    ('p2d_c7_cin16_mt', lambda: NW._stem(16, 64, BN), (1, 16, 96, 256)),
    ('p2d_resblock_instance_batch2', lambda: [NW.ResnetBlock(64, 'reflect', IN)], (2, 64, 32, 40)),
]


MODES = ['precise', 'fast']


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name,build,shape', CASES, ids=[c[0] for c in CASES])
def test_conv_unit(name, build, shape, mode):
    out, ref = _run(build(), _x(*shape), mode=mode)
    _check(out, ref, name, mode=mode)


HEADS = [
    ('head_tanh_64_3', lambda: NW._stem(32, 64, BN), lambda: NW._head(64, 3, nn.Tanh()), 1.0, (1, 32, 12, 136)),
    ('head_flow_x20', lambda: NW._stem(32, 64, BN), lambda: NW._head(64, 2), 20.0, (1, 32, 16, 32)),
    ('head_sigmoid', lambda: NW._stem(32, 32, BN), lambda: NW._head(32, 1, nn.Sigmoid()), 1.0, (2, 32, 16, 140)),
    ('mt_head', lambda: NW._stem(32, 64, BN), lambda: NW._head(64, 3, nn.Tanh()), 1.0, (1, 32, 80, 256)),
    ('kc32_head_mt', lambda: NW._stem(32, 32, BN), lambda: NW._head(32, 3, nn.Tanh()), 1.0, (1, 32, 80, 256)),
    ('kc16_head', lambda: NW._stem(32, 16, BN), lambda: NW._head(16, 3, nn.Tanh()), 1.0, (1, 32, 12, 136)),
]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('name,build,head,scale,shape', HEADS, ids=[c[0] for c in HEADS])
def test_head(name, build, head, scale, shape, mode):
    out, ref = _run(build(), _x(*shape), head(), scale, mode=mode)
    # head outputs are fp32; inputs differ by <= 1 bf16 ulp of the previous activation
    _check(out, ref, name, ulps=4.0 * max(1.0, scale), mean_tol=5e-3 * max(1.0, scale), mode=mode, scale=max(1.0, scale))


# Kernel configurations that the benchmark's plans lower (cfg4 / cfg2 / cfg3 generators, the cfg3 image and temporal
# discriminators, FlowNet2) and the cases above do not reach, each at the smallest shape that selects it on 132 SMs.
# tests/test_conv_census.py fails when one of them goes missing or stops being needed.
# name, layer list builder, input shape, modes, input = one-hot labels + 0/1 edges declared exact in bf16 (_label_x)
# FlowNet2's units are conv + bias + LeakyReLU(0.1) lowered as a conv with the raw + statistics epilogue (bias-free) and a
# normalise pass that adds the bias (plan.cu, G_NORM_ACT without a norm).  A batch norm in its place gives the conv kernel the
# same epilogue; the bias pass is checked by tests/test_gpu_flownet2.py.
LR01 = lambda: nn.LeakyReLU(0.1, True)
VARIANT_CASES = [
    ('stem_6_128_ring2_tb4', lambda: NW._stem(6, 128, BN), (1, 6, 160, 512), ['precise'], False),
    ('stem_6_128_kc16_bn128', lambda: NW._stem(6, 128, BN), (1, 6, 256, 512), ['fast'], False),
    ('stem_6_64_mg2_kc16', lambda: NW._stem(6, 64, BN), (1, 6, 512, 1024), MODES, False),
    ('stem_108_48_exact_mg2', lambda: NW._stem(108, 48, BN), (1, 108, 160, 512), ['precise'], True),
    ('stem_108_96_exact_kc32', lambda: NW._stem(108, 96, BN), (1, 108, 160, 512), ['precise'], True),
    ('s2_16_32_resident_kc16', lambda: NW._down(16, 32, BN), (1, 16, 1024, 2048), MODES, False),
    ('s2_64_128_resident', lambda: NW._down(64, 128, BN), (1, 64, 160, 512), ['fast'], False),
    ('deconv_32_16_resident', lambda: NW._up(32, 16, BN), (1, 32, 160, 128), MODES, False),
    ('deconv_128_64_resident', lambda: NW._up(128, 64, BN), (1, 128, 160, 128), ['fast'], False),
    ('deconv_1024_512_stream', lambda: NW._up(1024, 512, BN), (1, 1024, 8, 16), MODES, False),
    # temporal discriminator's first layer (13 channels, 4x4 stride 2, bias + LeakyReLU epilogue)
    ('d_first_13_stream', lambda: [nn.Conv2d(13, 64, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True)], (1, 13, 64, 128), ['precise'], False),
    ('d_first_13_resident', lambda: [nn.Conv2d(13, 64, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True)], (1, 13, 256, 512), ['precise'], False),
    # FlowNet2: flow upsampling (2 -> 2 4x4 transposed), flow predictors, odd concatenated channel counts
    ('fn_upflow_stream', lambda: [nn.ConvTranspose2d(2, 2, 4, 2, 1), BN(2), LR01()], (1, 2, 8, 16), ['precise'], False),
    ('fn_upflow_resident', lambda: [nn.ConvTranspose2d(2, 2, 4, 2, 1), BN(2), LR01()], (1, 2, 128, 256), ['precise'], False),
    ('fn_predict_1026_p2d', lambda: [nn.Conv2d(1026, 2, 3, padding=1), BN(2), LR01()], (1, 1026, 16, 32), ['precise'], False),
    ('fn_predict_194_p2d_ring2', lambda: [nn.Conv2d(194, 2, 3, padding=1), BN(2), LR01()], (1, 194, 128, 256), ['precise'], False),
    ('fn_6_64_2_kc16_resident', lambda: [nn.Conv2d(6, 64, 3, padding=1), BN(64), LR01(), nn.Conv2d(64, 2, 3, padding=1), BN(2), LR01()],
     (1, 6, 128, 256), ['precise'], False),
    ('fn_194_64_ring2_tb2', lambda: [nn.Conv2d(194, 64, 3, padding=1), BN(64), LR01()], (1, 194, 128, 256), ['precise'], False),
    ('fn_162_32_stream', lambda: [nn.Conv2d(162, 32, 3, padding=1), BN(32), LR01()], (1, 162, 256, 512), ['precise'], False),
    ('fn_16_2_kc16_resident', lambda: [nn.Conv2d(16, 2, 3, padding=1), BN(2), LR01()], (1, 16, 512, 1024), ['precise'], False),
    # large grids: enough units per CTA for the epilogue warpgroup (async_epi), at the sizes the benchmark runs the layers
    ('d_first_39_async_512x1024', lambda: [nn.Conv2d(39, 64, 4, stride=2, padding=2), nn.LeakyReLU(0.2, True)], (1, 39, 512, 1024),
     ['precise'], False),
    ('d_k4_256_512_ring2_tb1', lambda: [nn.Conv2d(256, 512, 4, stride=1, padding=2), BN(512), nn.LeakyReLU(0.2, True)], (1, 256, 33, 65),
     ['precise'], False),
    ('g1_64_128_s2_256x512', lambda: NW._down(64, 128, BN), (1, 64, 512, 1024), MODES, False),
    ('g2_res32_512x1024', lambda: [NW.ResnetBlock(32, 'reflect', BN)], (1, 32, 512, 1024), MODES, False),
    ('fn_c1_3_64_k7s2_async', lambda: [nn.Conv2d(3, 64, 7, stride=2, padding=3), BN(64), LR01()], (1, 3, 512, 1024), ['precise'], False),
    ('fn_6_64_s2_async_512x1024', lambda: [nn.Conv2d(6, 64, 3, padding=1), BN(64), LR01(), nn.Conv2d(64, 64, 3, stride=2, padding=1), BN(64),
                                            LR01()], (1, 6, 512, 1024), ['precise'], False),
]


@pytest.mark.parametrize('name,build,shape,mode,exact', [(c[0], c[1], c[2], m, c[4]) for c in VARIANT_CASES for m in c[3]],
                         ids=['%s-%s' % (c[0], m) for c in VARIANT_CASES for m in c[3]])
def test_conv_variant(name, build, shape, mode, exact):
    x = _label_x(*shape) if exact else _x(*shape)
    out, ref = _run(build(), x, mode=mode, exact=exact)
    _check(out, ref, name, mode=mode)


# name, layer list builder, head builder, head scale, input shape, modes
VARIANT_HEADS = [
    # the finest scale's 16 -> 3 image head: kx-GEMM with a 16-channel K block, resident weights
    ('head_16_3_headkx_kc16', lambda: NW._stem(8, 16, BN), lambda: NW._head(16, 3, nn.Tanh()), 1.0, (1, 8, 1024, 2048), MODES),
    # the discriminators' last two layers: 4x4 stride-1 conv on the decoupled rings, then the 1-channel 4x4 logit head
    ('d_last_layers_k4_headkx', lambda: [nn.Conv2d(256, 512, 4, stride=1, padding=2), BN(512), nn.LeakyReLU(0.2, True)],
     lambda: [nn.Conv2d(512, 1, 4, stride=1, padding=2)], 1.0, (1, 256, 33, 129), ['precise']),
    # the cfg4 generators' encoder / decoder paths at the benchmark's grids, where most layers run the async epilogue
    ('g0_128_enc_dec_256x512', lambda: NW._down(128, 256, BN) + NW._down(256, 512, BN) + NW._up(512, 256, BN) + NW._up(256, 128, BN),
     lambda: NW._head(128, 3, nn.Tanh()), 1.0, (1, 128, 256, 512), MODES),
    ('g0_128_64_up_head_128x256', lambda: NW._up(128, 64, BN), lambda: NW._head(64, 3, nn.Tanh()), 1.0, (1, 128, 128, 256), ['precise']),
    ('g2_6_32_res64_1024x2048', lambda: NW._stem(6, 32, BN) + NW._down(32, 64, BN) + [NW.ResnetBlock(64, 'reflect', BN)] + NW._up(64, 32, BN),
     lambda: NW._head(32, 3, nn.Tanh()), 1.0, (1, 6, 1024, 2048), MODES),
]


@pytest.mark.parametrize('name,build,head,scale,shape,mode', [c[:5] + (m,) for c in VARIANT_HEADS for m in c[5]],
                         ids=['%s-%s' % (c[0], m) for c in VARIANT_HEADS for m in c[5]])
def test_head_variant(name, build, head, scale, shape, mode):
    out, ref = _run(build(), _x(*shape), head(), scale, mode=mode)
    _check(out, ref, name, ulps=4.0 * max(1.0, scale), mean_tol=5e-3 * max(1.0, scale), mode=mode, scale=max(1.0, scale))


def test_running_stats_side_effect():
    """nn.BatchNorm2d in train mode updates running_mean/var/num_batches_tracked (SURVEY App. B #1)."""
    mods = [nn.Conv2d(64, 64, 3, padding=1), BN(64), nn.ReLU(True)]
    runner = det_fill_(NW.SequentialRunner(mods), seed=3).cuda()
    x = _x(2, 64, 16, 16).cuda()
    ref_conv, ref_bn = nn.Conv2d(64, 64, 3, padding=1).cuda(), nn.BatchNorm2d(64).cuda()
    ref_conv.load_state_dict(runner.seq[0].state_dict())
    ref_bn.load_state_dict(runner.seq[1].state_dict())
    with torch.no_grad():
        runner(x)
        ref_bn.train()
        ref_bn(ref_conv(x))
    torch.cuda.synchronize()
    assert int(runner.seq[1].num_batches_tracked.item()) == 1
    assert torch.allclose(runner.seq[1].running_mean, ref_bn.running_mean, atol=2e-3)
    assert torch.allclose(runner.seq[1].running_var, ref_bn.running_var, rtol=2e-2, atol=1e-3)


def test_repack_after_weight_update():
    mods = [nn.ReflectionPad2d(1), nn.Conv2d(64, 64, 3), BN(64), nn.ReLU(True)]
    runner = det_fill_(NW.SequentialRunner(mods), seed=4).cuda()
    runner.precision = 'fast'
    x = _x(1, 64, 16, 32).cuda()
    with torch.no_grad():
        a = runner(x)
        runner.seq[1].weight.mul_(-1.0)          # in-place update, as an optimiser step would do
        b = runner(x)
        ref = E.run_units(list(runner.seq), E.r16(x))
    assert not torch.equal(a, b)
    _check(b, ref, 'after_repack')


@pytest.mark.parametrize('mode', ['fast', 'precise'])
def test_caller_provided_workspace(mode):
    """v2v_plan_finalize_ws: the plan's arena in caller-owned memory gives bit-identical results; the size is known beforehand."""
    from vid2vid_b200.plan import Plan
    mods = [nn.ReflectionPad2d(1), nn.Conv2d(32, 64, 3), BN(64), nn.ReLU(True)] + NW._down(64, 64, BN) + NW._up(64, 32, BN)
    runner = det_fill_(NW.SequentialRunner(mods), seed=9).cuda()
    runner.precision = mode
    x = _x(2, 32, 24, 40).cuda()
    with torch.no_grad():
        ref = runner(x)
    p = Plan(x.device.index, precision=mode)
    runner._describe(p, *x.shape)
    need = p.workspace_bytes
    assert need > 0
    ws = torch.empty(need + 1024, dtype=torch.uint8, device=x.device)
    with pytest.raises(ValueError):
        p.finalize(workspace=ws[:need // 2])
    p.finalize(workspace=ws)
    out = torch.empty_like(ref)
    p.run([x, out], use_graph=False)
    p.run([x, out], use_graph=True)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
