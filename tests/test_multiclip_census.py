"""CPU-only census of the conv kernel configurations that several clips per GPU run: every configuration the plans of
tools/time_multiclip.py lower (each workload, both arithmetic modes, every clip count B, per-sample plans for B > 1) must be
lowered by a GPU parity case that compares it with fp64 (or bf16-emulated fp32): the cases tests/test_conv_variant_census.py
collects, or the per-sample cases of tests/test_gpu_multiclip.py.  The configuration is keyed as that census keys it
(including async_epi: more clips mean more work units, which can move a conv onto the epilogue-warpgroup instantiation)."""
import collections
import functools
import os
import sys

import pytest
import torch

import test_conv_variant_census as CEN
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import time_multiclip as TM     # noqa: E402


@pytest.fixture(autouse=True)
def _h100_sxm():
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != CEN.H100_SXM_SMS:
        pytest.skip('the census describes a %d-SM H100 SXM' % CEN.H100_SXM_SMS)


def _variants(describe, mode, sample_stats):
    p = Plan(0, precision=mode, sample_stats=sample_stats)
    describe(p)
    return [CEN.variant(c) for c in p.describe()['convs']]


@functools.lru_cache(maxsize=None)
def multiclip_variants():
    """{variant: one time_multiclip conv that uses it}."""
    found = collections.OrderedDict()
    for wl, w in TM.WORKLOADS.items():
        o = dict(w['opt'])
        opt = make_opt(use_single_G=False, use_real_img=not o.get('no_first_img', False), gpu_ids=[], synthetic_weights=True, **o)
        S = opt.n_scales_spatial
        for s in range(S):
            net = NW.build_netG(opt, s)
            net.input_exact_bf16 = s == S - 1 and opt.label_nc != 0      # as Vid2VidModelG.initialize sets it
            h, w_ = w['H'] // 2 ** (S - 1 - s), w['W'] // 2 ** (S - 1 - s)
            for mode in ('precise', 'fast'):
                for b in w['bs']:
                    for v in _variants(lambda p: net._describe(p, b, h, w_), mode, b > 1):
                        found.setdefault(v, '%s %s G%d B=%d' % (wl, mode, s, b))
    return found


@functools.lru_cache(maxsize=None)
def multiclip_case_variants():
    import test_gpu_multiclip as TMC
    out = {}
    for name, build, shape, modes in TMC.CONV_CASES:
        r = NW.SequentialRunner(build())
        out[name] = {v for m in modes for v in _variants(lambda p: r._describe(p, *shape), m, True)}
    return out


def test_every_multiclip_conv_configuration_has_a_unit_case():
    reached = set().union(*CEN.unit_variants().values(), *multiclip_case_variants().values())
    missing = [(v, where) for v, where in multiclip_variants().items() if v not in reached]
    assert not missing, '%d kernel configurations of the multi-clip plans are not reached by any GPU parity case:\n%s' % (
        len(missing), '\n'.join('  %s  e.g. %s' % (v, where) for v, where in missing))


def test_every_multiclip_case_is_needed():
    """Each per-sample case reaches a multi-clip configuration that no other parity case reaches."""
    cases, mv = multiclip_case_variants(), set(multiclip_variants())
    base = set().union(*CEN.unit_variants().values())
    for name, vs in cases.items():
        others = base.union(*(o for k, o in cases.items() if k != name))
        assert vs & mv - others, '%s reaches no multi-clip configuration of its own' % name


def test_multiclip_census_is_not_vacuous():
    mv = multiclip_variants()
    assert len(mv) >= 50, len(mv)
    assert any(v.async_epi for v in mv) and any(not v.split for v in mv) and any(v.patch for v in mv)
