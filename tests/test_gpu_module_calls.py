"""How a planned module call picks its plan: the modules without a backward refuse autograd instead of returning tensors
without a gradient, per-sample-statistics discriminators run, and the plan cache keys keep the layout bench.py and
tools/time_vgg.py read (key[0] the module tag, 'train' in training keys, key[-1] the precision)."""
import pytest
import torch

import cases as C
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import networks as NW

pytestmark = pytest.mark.gpu


def _x(*shape):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(0)).cuda()


def _no_backward_calls():
    gg = C.build_module(C.CASES['global_small']).cuda()
    le = C.build_module(C.CASES['local_small']).cuda()
    enc = NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []).cuda()
    gz = NW.define_G(15, 3, 0, 16, 'global_with_features', 3, 'instance', 0, [], C.make_opt(n_blocks=2, feat_num=16)).cuda()
    vgg = NW.Vgg19(requires_grad=True).cuda()
    flow = FN.FlowNet2().cuda()
    return [('GlobalGenerator', lambda: gg(_x(1, 35, 32, 64))),
            ('LocalEnhancer', lambda: le(_x(1, 35, 64, 64))),
            ('Encoder', lambda: enc(_x(1, 3, 64, 64), torch.zeros(1, 1, 64, 64, device='cuda'))),
            ('Global_with_z', lambda: gz(_x(1, 15, 64, 64), _x(1, 16, 64, 64))),
            ('Vgg19', lambda: vgg(_x(1, 3, 64, 64))),
            ('FlowNet2', lambda: flow(_x(1, 3, 2, 64, 64)))]


def test_modules_without_a_backward_refuse_autograd():
    for name, call in _no_backward_calls():
        with pytest.raises(NotImplementedError, match=name + '.forward has no backward'):
            call()


def test_sample_stats_discriminator_runs_without_autograd():
    c = C.CASES['D_small']
    x = _x(c['batch'], c['input_nc'], c['h'], c['w'])
    ref = C.build_module(c).cuda()
    net = C.build_module(c).cuda()
    net.sample_stats = True
    with torch.no_grad():
        a, b = ref(x), net(x)
    assert [[t.shape for t in tower] for tower in a] == [[t.shape for t in tower] for tower in b]
    assert all('sample_stats' in k for k in net._plans())


def test_plan_cache_keys():
    c = C.CASES['g0_small']
    g = C.build_module(c).cuda()
    g.precision = 'precise'
    inp, prev, mask = (t.cuda() for t in C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed']))
    with torch.no_grad():
        g(inp, prev, mask, None, None, None, False)
    g(inp, prev, mask, None, None, None, False)
    assert list(g._plans()) == [('G', 1, 32, 64, False, False, False, 'precise'),
                                ('G', 1, 32, 64, False, False, False, 'train', 'precise')]

    d = NW.define_D(6, 16, 2, 'batch', 2, True, []).cuda()
    d.precision = 'fast'
    x = _x(1, 6, 64, 96)
    with torch.no_grad():
        d(x)
    d(x.requires_grad_())
    assert list(d._plans()) == [('D', 1, 1, 64, 96, 'fast'), ('D', 0, 1, 32, 48, 'fast'),
                                ('D', 1, 1, 64, 96, 'train', 'fast'), ('D', 0, 1, 32, 48, 'train', 'fast')]

    vgg = NW.Vgg19().cuda()
    vgg.precision = 'precise'
    y = _x(1, 3, 64, 128)
    vgg.feature_l1(y.clone().requires_grad_(), y)
    with torch.no_grad():
        vgg(y)
    assert list(vgg._plans()) == [('VGGL', 1, 64, 128, 'train', 'precise'), ('VGGF', 1, 64, 128, 'precise')]
