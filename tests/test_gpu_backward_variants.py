"""GPU parity of the tensor-core backward at the configurations cfg3's training step runs (tests/test_conv_census.py
fails when one of them is reached by no case).  Each case mirrors benchmark layers -- channels, kernel, stride, padding and
grid -- as smooth units (conv, conv + BatchNorm, transposed conv + BatchNorm, the tanh image head; no ReLU / LeakyReLU), so no
activation gate can flip between our forward and the reference's, and the gradients are compared with PyTorch autograd in
float64 at a tight bound: relative L2 <= 1e-4 and max|d| <= 1e-3 * max|ref| per tensor.  The precise path's split-bf16
products are fp32-class and each weight-gradient unit sums its K chunk (chunks_per_unit x KP pixels) in the tensor-core
accumulator, the K splits meeting through fp32 atomics; measured on an H100 SXM (700 W) every tensor here stays at or below
~2e-5, while dropping one split-bf16 cross term moves a gradient by ~2^-9.  The bound holds only while a unit's K chunk stays
moderate: the G1 image head's weight gradient at the full 512 x 1024 grid (87k pixels per unit, a sum that grows linearly
because tanh-head gradient and activation are correlated) measured 3e-4, so its case runs at 128 x 256, which keeps its
configuration (KP 64, K split) with 5.5k pixels per unit.

The finest stem's case declares its one-hot input exact in bf16 (as cfg3's finest scale does): the forward reads only the hi
half of that input, and the weight gradient reads the lo half, which the import never writes."""
import pytest
import torch
import torch.nn as nn

import bf16_emul as E
import test_gpu_backward as TB
import test_gpu_conv as TC
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import det_fill_

pytestmark = pytest.mark.gpu

BN = NW.get_norm_layer('batch')
L2, MAX = 1e-4, 1e-3


def _c(a, b, k, s, p):
    return nn.Conv2d(a, b, k, stride=s, padding=p)


def _t(a, b):
    return nn.ConvTranspose2d(a, b, 3, stride=2, padding=1, output_padding=1)


def _tanh(c):
    return lambda: NW._head(c, 3, nn.Tanh())


# name, layer list builder, input shape, head builder, head scale, input exact in bf16 (one-hot labels + 0/1 edges)
CASES = [
    # cfg3 G0 (256 x 512): the finest-branch stem (exact input), stride-2 / transposed weight gradients with 128-wide N tiles
    ('g0_stem_108_192_exact', lambda: [nn.ReflectionPad2d(3), _c(108, 192, 7, 1, 0), BN(192)], (1, 108, 256, 512), None, 1.0, True),
    ('g0_stem_6_128_s2_up_head', lambda: [nn.ReflectionPad2d(3), _c(6, 128, 7, 1, 0), BN(128), _c(128, 256, 3, 2, 1), BN(256),
                                          _t(256, 128), BN(128)], (1, 6, 256, 512), _tanh(128), 1.0, False),
    ('g0_512_1024_s2_up_up', lambda: [_c(512, 1024, 3, 2, 1), BN(1024), _t(1024, 512), BN(512), _t(512, 256), BN(256)],
     (1, 512, 64, 128), None, 1.0, False),
    ('g0_64_128_s2_up_head', lambda: [_c(64, 128, 3, 2, 1), BN(128), _t(128, 64), BN(64)], (1, 64, 256, 512), _tanh(64), 1.0, False),
    # cfg3 G1 (512 x 1024): the 6 -> 64 stem's weight gradient (16-channel N side, 32-byte rows, K split)
    ('g1_stem_6_64', lambda: [nn.ReflectionPad2d(3), _c(6, 64, 7, 1, 0), BN(64)], (1, 6, 64, 256), None, 1.0, False),
    # cfg3 G1's encoder / decoder and image head
    ('g1_32_64_s2_c3_up_head', lambda: [_c(32, 64, 3, 2, 1), BN(64), nn.ReflectionPad2d(1), _c(64, 64, 3, 1, 0), BN(64), _t(64, 32),
                                        BN(32)], (1, 32, 128, 256), _tanh(32), 1.0, False),
    # cfg3's image discriminator: tower 2 at 512 x 1024 (ragged 64-pixel row segments), tower 1's last layers, tower 0's
    # 32-pixel K chunks
    ('d2_39_tower', lambda: [_c(39, 64, 4, 2, 2), _c(64, 128, 4, 2, 2), BN(128), _c(128, 256, 4, 2, 2), BN(256), _c(256, 512, 4, 1, 2),
                             BN(512), _c(512, 1, 4, 1, 2)], (1, 39, 512, 1024), None, 1.0, False),
    ('d1_256_512_1', lambda: [_c(256, 512, 4, 1, 2), BN(512), _c(512, 1, 4, 1, 2)], (1, 256, 33, 65), None, 1.0, False),
    ('d0_128_256_s2', lambda: [_c(128, 256, 4, 2, 2), BN(256)], (1, 128, 32, 64), None, 1.0, False),
    # cfg3's temporal discriminator's first layer at tower 0: 13 channels (16 padded)
    ('dt0_13_64', lambda: [_c(13, 64, 4, 2, 2)], (1, 13, 128, 256), None, 1.0, False),
]


def _runner(build, head, scale, exact):
    r = det_fill_(NW.SequentialRunner(build(), head() if head else None, scale), seed=5).cuda()
    r.precision = 'precise'
    r.input_exact_bf16 = exact
    return r


def _input(shape, exact):
    return (TC._label_x(*shape, seed=1) if exact else TC._x(*shape, seed=1)).cuda()


@pytest.mark.parametrize('name,build,shape,head,scale,exact', CASES, ids=[c[0] for c in CASES])
def test_backward_variant(name, build, shape, head, scale, exact):
    runner = _runner(build, head, scale, exact)
    names, ours, refs, out, ref = TB._grads(runner, _input(shape, exact))
    TB._cmp(name + ' forward', out.detach(), ref.detach(), tol=3e-4, l2=1e-4)
    bad = []
    for n, o, r in zip(names, ours, refs):
        if n.endswith('.bias') and r.abs().max().item() < 1e-6:
            # zero in the reference: a conv bias in front of a norm, or a norm's shift whose output feeds a conv and another
            # norm (the shift cancels).  Ours is fp32 cancellation noise of a sum with as many terms as the same layer's
            # weight gradient, so it is held to MAX relative to that gradient's scale.
            w = refs[names.index(n[:-len('bias')] + 'weight')].abs().max().item()
            assert o.abs().max().item() <= MAX * w, (n, o.abs().max().item(), w)
            continue
        try:
            TB._cmp('%s d/d %s' % (name, n), o, r, tol=MAX, l2=L2)
        except AssertionError as e:
            bad.append(str(e)[:160])
    assert not bad, bad


def test_device_reference_matches_cpu():
    """The fp64 reference runs on the device to keep the cases fast; at a small shape it equals the CPU's."""
    runner = _runner(lambda: [_c(39, 64, 4, 2, 2), _c(64, 128, 4, 2, 2), BN(128), _t(128, 64), BN(64)], None, 1.0, False)
    x = TC._x(1, 39, 24, 40, seed=1).double()
    grads = []
    E.ROUND[0], E.GRAD[0] = False, True
    try:
        for dev in ('cpu', 'cuda'):
            mods = [m.to(dev).double() for m in runner.seq]
            for p in runner.parameters():
                p.grad = None
            xd = x.to(dev).clone().requires_grad_(True)
            out = E.run_units(mods, xd)
            g = torch.randn(out.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
            (out * g.to(dev)).sum().backward()
            grads.append([t.to('cpu', copy=True) for t in [xd.grad] + [p.grad for p in runner.parameters() if p.grad is not None]])
    finally:
        E.ROUND[0], E.GRAD[0] = True, False
    assert len(grads[0]) == len(grads[1]) > 1
    for a, b in zip(*grads):
        assert ((a - b).norm() / max(b.norm().item(), 1e-30)).item() < 1e-12


def _backward_records(describe):
    """The plan's description on the host, and read from what finalize built."""
    p = Plan(0, precision='precise', train=True)
    describe(p)
    before = p.describe()
    p.finalize()
    return before, p.describe()


def test_describe_matches_finalized_backward():
    """The description v2v_plan_describe derives on the host equals the one read from the plan finalize built: the backward
    units, and the forward launch list's layout and epilogue records (imports, packs, statistics, tail finalisations and
    normalise passes)."""
    runner = _runner(lambda: [nn.ReflectionPad2d(3), _c(6, 64, 7, 1, 0), BN(64), _c(64, 128, 3, 2, 1), BN(128), _t(128, 64), BN(64)],
                     _tanh(64), 1.0, False)
    before, after = _backward_records(lambda p: runner._describe(p, 1, 6, 32, 64))
    assert len(before['backward']) == 4 and {b['mode'] for b in before['backward']} == {1, 2, 3}, before['backward']
    assert {r['kind'] for r in before['epilogue_forward']} == {'stats', 'finalize', 'apply'}, before['epilogue_forward']
    assert {'import', 'pack'} <= {r['kind'] for r in before['layout']}, before['layout']
    assert before == after
    d = NW.define_D(39, 64, 3, 'batch', 1, True, []).cuda()
    before, after = _backward_records(lambda p: d._describe(p, 0, 1, 64, 128))
    assert len(before['backward']) >= 4 and any(b['wgrad'] for b in before['backward']), before['backward']
    assert before == after
