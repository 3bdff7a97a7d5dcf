"""Host-side checks of per-sample-statistics plans (v2v_plan_set_sample_stats), no GPU needed: the switch is refused on
training plans, and a per-sample plan of B clips lowers every conv with the kernel configuration of the batch-1 plan (that
configuration fixes each pixel's accumulation order, which is what keeps every clip bit-identical to its own run)."""
import os
import sys

import pytest

import bench
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import time_multiclip as TM     # noqa: E402

# the launch quantities that scale with the number of images, and the epilogue placement chosen from them (the epilogue
# only stores results: it does not change any sum; tests/test_multiclip_census.py keys configurations by it)
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
    p = Plan(0, precision=mode, sample_stats=sample_stats)
    net._describe(p, N, H, W)
    d = p.describe()
    assert d['sample_stats'] == int(sample_stats)
    return d['convs']


@pytest.mark.parametrize('mode', ['precise', 'fast'])
@pytest.mark.parametrize('wl', list(TM.WORKLOADS))
def test_per_sample_plan_keeps_the_batch1_configuration(wl, mode):
    W = TM.WORKLOADS[wl]
    o = dict(W['opt'])
    opt = make_opt(gpu_ids=[], synthetic_weights=True, **o)
    S = opt.n_scales_spatial
    for s in range(S):
        sc = 2 ** (S - 1 - s)
        net = NW.build_netG(opt, s)
        net.input_exact_bf16 = s == S - 1 and opt.label_nc != 0
        h, w = W['H'] // sc, W['W'] // sc
        one = _convs(net, 1, h, w, mode, False)
        four = _convs(net, 4, h, w, mode, True)
        assert len(one) == len(four)
        for a, b in zip(one, four):
            assert {k: v for k, v in a.items() if k not in PER_LAUNCH} == {k: v for k, v in b.items() if k not in PER_LAUNCH}
            assert b['m_total'] == 4 * a['m_total'] and b['units'] == 4 * a['units']
