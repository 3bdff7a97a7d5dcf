"""GPU parity of conv_umma_kernel's epilogue warpgroups, which store each work unit while the consumers multiply the next one.
The cases are the layers whose CTAs pass the most units through the staging-tile handoff, at the sizes the benchmark runs
them: 64->64 at 512x1024, a layer with two 64-column handoffs per unit, the finest kx-GEMM image head at 1024x2048, and a
batch-2 InstanceNorm layer whose CTAs flush the statistics of one image and go on with the next; and the exact-input
108->48 finest stem, whose M-blocked units keep the consumers' epilogue.  Each is checked against the references and
tolerances of tests/test_gpu_conv.py, its running statistics (written by the last CTA's finalisation) against PyTorch's
train-mode norm layer, and two independent runs must agree bit for bit."""
import copy

import pytest
import torch
import torch.nn as nn

import test_gpu_conv as TC
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import det_fill_

pytestmark = pytest.mark.gpu

BN = NW.get_norm_layer('batch')
IN = NW.get_norm_layer('instance')


def _c3(c, norm):
    return [nn.ReflectionPad2d(1), nn.Conv2d(c, c, 3), norm(c), nn.ReLU(True)]


def _handoffs(c):
    return c['MG'] * ((c['BN'] + 63) // 64)


# name, layer list builder, head builder, input shape, exact one-hot input, what the first conv's configuration must show
CASES = [
    ('c64_512x1024', lambda: _c3(64, BN), None, (1, 64, 512, 1024), False,
     lambda c: c['async_epi'] == 1 and c['units'] >= 8 * c['ctas']),
    ('stem_108_48_exact_1024x2048', lambda: NW._stem(108, 48, BN), None, (1, 108, 1024, 2048), True,
     lambda c: c['async_epi'] == 0 and c['MG'] == 2 and c['BNt'] == 48),
    ('c128_256x512_two_handoffs', lambda: _c3(128, BN), None, (1, 128, 256, 512), False,
     lambda c: c['async_epi'] == 1 and _handoffs(c) == 2 and c['units'] >= 4 * c['ctas']),
    ('head_16_3_headkx_1024x2048', lambda: NW._stem(8, 16, BN), lambda: NW._head(16, 3, nn.Tanh()), (1, 8, 1024, 2048), False,
     lambda c: c['async_epi'] == 1),
    ('c64_instance_batch2', lambda: _c3(64, IN), None, (2, 64, 128, 256), False,
     lambda c: c['async_epi'] == 1 and c['units'] >= 2 * c['ctas']),
]


def _norm(m):
    return isinstance(m, (nn.BatchNorm2d, nn.InstanceNorm2d))


def _once(build, head, x, mode, exact):
    runner = det_fill_(NW.SequentialRunner(build(), head() if head else None), seed=1).cuda()
    runner.precision = mode
    runner.input_exact_bf16 = exact
    # PyTorch's train-mode forward up to the first norm layer, from the same weights and running statistics
    mods = list(runner.seq)
    first = next(i for i, m in enumerate(mods) if _norm(m))
    ref = copy.deepcopy(nn.Sequential(*mods[:first + 1])).train()
    with torch.no_grad():
        out = runner(x)
        ref(x)
    torch.cuda.synchronize()
    stats = [t.clone() for m in runner.modules() if _norm(m) for t in (m.running_mean, m.running_var)]
    return out, stats, (mods[first], ref[first])


@pytest.mark.parametrize('mode', TC.MODES)
@pytest.mark.parametrize('name,build,head,shape,exact,want', CASES, ids=[c[0] for c in CASES])
def test_async_epilogue(name, build, head, shape, exact, want, mode):
    r = NW.SequentialRunner(build(), head() if head else None)
    r.input_exact_bf16 = exact
    p = Plan(0, precision=mode)
    r._describe(p, *shape)
    convs = p.describe()['convs']
    assert want(convs[0]), convs[0]
    if head is not None:
        assert convs[-1]['headkx'] > 0, convs[-1]
    x = TC._label_x(*shape) if exact else TC._x(*shape)
    out, ref = TC._run(build(), x, head() if head else None, mode=mode, exact=exact)
    if head is not None:
        TC._check(out, ref, name, ulps=4.0, mean_tol=5e-3, mode=mode)
    else:
        TC._check(out, ref, name, mode=mode)
    del ref
    xd = x.cuda()
    a, sa, (ours, theirs) = _once(build, head, xd, mode, exact)
    assert torch.allclose(ours.running_mean, theirs.running_mean, atol=2e-3), name + ': running mean'
    assert torch.allclose(ours.running_var, theirs.running_var, rtol=2e-2, atol=1e-3), name + ': running variance'
    b, sb, _ = _once(build, head, xd, mode, exact)
    assert torch.equal(a, b), name + ': two runs differ'
    assert sa and len(sa) == len(sb)
    for u, v in zip(sa, sb):
        assert torch.equal(u, v), name + ': running statistics differ between two runs'
