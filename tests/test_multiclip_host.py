"""Host-side checks of per-sample-statistics plans (v2v_plan_set_sample_stats), no GPU needed: the switch is refused on
training plans, and a per-sample plan of B clips lowers every conv with the kernel configuration of the batch-1 plan (that
configuration fixes each pixel's accumulation order, which is what keeps every clip bit-identical to its own run)."""
import pytest

import bench
import product_plans as PP
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan

# the launch quantities that scale with the number of images, and the epilogue placement chosen from them (the epilogue
# only stores results: it does not change any sum; tests/test_conv_census.py keys configurations by it)
PER_LAUNCH = ('units', 'm_total', 'ctas', 'async_epi')


def test_sample_stats_is_refused_on_a_training_plan():
    p = Plan(0, precision='precise', train=True)
    with pytest.raises(RuntimeError, match='per-sample statistics are for inference plans'):
        L.check(L.lib().v2v_plan_set_sample_stats(p._h, 1))


def test_training_is_refused_on_a_sample_stats_plan():
    p = Plan(0, precision='precise', sample_stats=True)
    with pytest.raises(RuntimeError, match='per-sample-statistics plan cannot train'):
        L.check(L.lib().v2v_plan_set_training(p._h, 1))


def test_sample_stats_module_refuses_autograd():
    opt = bench.make_opt_for('cfg2')
    opt.gpu_ids = []
    net = NW.build_netG(opt, 0)
    net.sample_stats = True
    with pytest.raises(RuntimeError, match='per-sample statistics are for inference plans'):
        net._get_plan(('G',), __import__('torch').device('cuda', 0), lambda p: None, train=True)


def _convs(net, N, H, W, mode, sample_stats):
    d = PP.describe(PP.PlanSpec('multiclip', 'B=%d' % N, lambda p: net._describe(p, N, H, W), mode, sample_stats=sample_stats))
    assert d['sample_stats'] == int(sample_stats)
    return d['convs']


@pytest.mark.parametrize('mode', ['precise', 'fast'])
@pytest.mark.parametrize('wl', list(PP.TM.WORKLOADS))
def test_per_sample_plan_keeps_the_batch1_configuration(wl, mode):
    W = PP.TM.WORKLOADS[wl]
    for net, h, w in PP.scales(PP.clip_opt(W), W['H'], W['W']):
        one = _convs(net, 1, h, w, mode, False)
        four = _convs(net, 4, h, w, mode, True)
        assert len(one) == len(four)
        for a, b in zip(one, four):
            assert {k: v for k, v in a.items() if k not in PER_LAUNCH} == {k: v for k, v in b.items() if k not in PER_LAUNCH}
            assert b['m_total'] == 4 * a['m_total'] and b['units'] == 4 * a['units']
