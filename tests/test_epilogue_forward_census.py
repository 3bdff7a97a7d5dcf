"""CPU-only census of the forward epilogue of the norm layers: the statistics accumulation in conv_umma_kernel's epilogue, their
finalisation (the last CTA's tail of the conv launch, or stats_finalize_kernel) with the train-mode side effects, and the
normalise pass (norm_apply_rows_kernel / norm_apply_kernel).  Every path the products run must also be run by a case of
tests/test_gpu_epilogue_forward.py, which holds it to an fp64 reference with a bound derived from the kernels' arithmetic.

v2v_plan_describe reports, for every plan, an "epilogue_forward" array (stats / finalize / apply records) with the choices
finalize_sites and norm_apply_launch make -- the host functions the plan's emission calls -- without a GPU and assuming the
H100 SXM's 132 SMs.  Each record is reduced to the fields that select a code path or change the summation order."""
import collections
import functools
import os
import sys

import pytest

import bench
import product_plans as PP
import test_backward_variant_census as BC
from test_conv_variant_census import _h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import time_multiclip as TM     # noqa: E402
import time_slots as TS         # noqa: E402

# stats: which threads run the epilogue (async_epi), tiles per unit (MG), several phases (transposed convs: the key, and so the
# flushed accumulator, changes with the phase), whether one CTA accumulates several units (and so flushes at key changes inside
# its run), several images (a flush per image), and the finalising tail slots.  N tile and K
# block choose the kernel instantiation, which tests/test_conv_variant_census.py already requires a parity case for.
StatsKey = collections.namedtuple('StatsKey', 'impl async_epi MG multi_phase multi_unit multi_image sites')
FinKey = collections.namedtuple('FinKey', 'site stats flags running bias mean_rstd c_off multi_image')
# apply: the kernel and its template (PREC, NADD), idle threads and a ragged last row segment, the halo (reflect pads 1 and 3
# map different rows), the parity split, the scale source, a second layout and a repeated pass.
ApplyKey = collections.namedtuple('ApplyKey', 'kernel prec nadd idle ragged pad_mode pad parity scale layout repeat')


def keys_of(d):
    """{key: record} of one plan description."""
    out = collections.OrderedDict()
    for r in d['epilogue_forward']:
        if r['kind'] == 'stats':
            per_cta = -(-r['units'] // r['ctas'])
            k = StatsKey(r['impl'], r['async_epi'], r['MG'], int(r['phases'] > 1), int(per_cta > 1), int(r['N'] > 1), len(r['fin']))
        elif r['kind'] == 'finalize':
            k = FinKey(r['site'], r['stats'], r['flags'], r['running'], r['bias'], r['mean_rstd'], int(r['c_off'] != 0),
                       int(r['N'] > 1))
        else:
            k = ApplyKey(r['kernel'], r['prec'], r['nadd'], r['idle'], r['ragged'], r['pad_mode'], max(r['pads']), r['parity'],
                         r['scale'], int(r['layout'] > 0), r['repeat'])
        out.setdefault(k, r)
    return out


def _where(tag, r):
    if r['kind'] == 'stats':
        return '%s: conv -> %d ch @ %dx%d (N %d)' % (tag, r['C'], r['H'], r['W'], r['N'])
    if r['kind'] == 'finalize':
        return '%s: %d ch at %d' % (tag, r['C'], r['c_off'])
    return '%s: %d ch @ %dx%d layout %d' % (tag, r['Cvalid'], r['H'], r['W'], r['layout'])


def _plan_describe(describe, precision, train=False, sample_stats=False, flags=False):
    p = Plan(0, precision=precision, train=train, sample_stats=sample_stats)
    if flags:
        p.set_image_flags(NW.S_FLAGS)
    describe(p)
    return p.describe()


def _net_describe(net, N, H, W):
    return functools.partial(lambda net, N, H, W, p: net._describe(p, N, H, W), net, N, H, W)


def _product_describes():
    """(tag, describe, plan options) over the products' plans."""
    out = []
    # bench.py: cfg4 / cfg2 inference in both modes; cfg3's training step (generator scales, D and D_T towers); FlowNet2
    for wl in ('cfg4', 'cfg2'):
        W = bench.WORKLOADS[wl]
        opt = bench.make_opt_for(wl)
        opt.gpu_ids = []
        for s in range(W['n_scales']):
            sc = 2 ** (W['n_scales'] - 1 - s)
            net = NW.build_netG(opt, s)
            net.input_exact_bf16 = s == W['n_scales'] - 1 and opt.label_nc != 0
            for mode in ('fast', 'precise'):
                out.append(('%s %s G%d' % (wl, mode, s), _net_describe(net, 1, W['H'] // sc, W['W'] // sc), dict(precision=mode)))
    out += [(tag, d, dict(precision='precise', train=True)) for tag, d in BC._benchmark_describes()]
    W = bench.WORKLOADS['flownet2']
    f = FN.FlowNet2()
    for name in ('flownetc', 'flownets_1', 'flownets_2', 'flownets_d', 'flownetfusion'):
        out.append(('flownet2 ' + name, functools.partial(lambda sub, p: sub.describe(p, 1, W['H'], W['W']), getattr(f, name)),
                    dict(precision=FN.FlowNet2.precision)))
    # tests/product_plans.py: the first-frame generators, the pose step (the VGG plans have no norm layer: asserted below)
    for tag, d in PP.first_frame():
        out += [(tag + ' ' + mode, d, dict(precision=mode)) for mode in ('fast', 'precise')]
    out += [(tag, d, dict(precision='precise', train=True)) for tag, d in PP.pose_step()]
    # tools/time_multiclip.py's per-sample plans for every clip count, tools/time_slots.py's flag-reading slot plans
    for tools, flags in ((TM, False), (TS, True)):
        for wl, w in tools.WORKLOADS.items():
            o = dict(w['opt'])
            if tools is TM:
                o = dict(use_single_G=False, use_real_img=not o.get('no_first_img', False), **o)
            opt = make_opt(gpu_ids=[], synthetic_weights=True, **o)
            S = opt.n_scales_spatial
            for s in range(S):
                net = NW.build_netG(opt, s)
                net.input_exact_bf16 = s == S - 1 and opt.label_nc != 0
                h, w_ = w['H'] // 2 ** (S - 1 - s), w['W'] // 2 ** (S - 1 - s)
                for mode in ('precise', 'fast'):
                    for b in w['bs']:
                        if flags or b > 1:
                            out.append(('%s %s %s G%d B=%d' % ('slots' if flags else 'multiclip', wl, mode, s, b),
                                        _net_describe(net, b, h, w_), dict(precision=mode, sample_stats=True, flags=flags)))
    return out


@functools.lru_cache(maxsize=None)
def product_keys():
    found = collections.OrderedDict()
    for tag, describe, kw in _product_describes():
        for k, r in keys_of(_plan_describe(describe, **kw)).items():
            found.setdefault(k, _where(tag, r))
    return found


@functools.lru_cache(maxsize=None)
def case_keys():
    """{case id: keys} over the GPU cases, described from the same builders the GPU test runs (modules on the CPU)."""
    import test_gpu_epilogue_forward as EF
    out = collections.OrderedDict()
    for name, spec in EF.CASES:
        out[name] = set()
        for mode in spec.modes:
            out[name] |= set(keys_of(_plan_describe(lambda p: EF.build(p, spec, 'cpu'), **EF.plan_options(spec, mode))))
    return out


# The paths GPU cases run although no product plan reaches them, each with the reason.
UNREACHED = {
    ApplyKey('rows', 0, 0, 0, 1, 0, 0, 0, 'none', 0, 0): 'a fast-mode norm-less pass without bias: the cases read a stride-2 '
                                                         '(parity) layout back through one; only FlowNet2 (precise) has such passes',
}


def test_census_is_not_vacuous():
    keys = product_keys()
    st = [k for k in keys if isinstance(k, StatsKey)]
    fin = [k for k in keys if isinstance(k, FinKey)]
    ap = [k for k in keys if isinstance(k, ApplyKey)]
    assert {k.sites for k in st} == {1, 2}, 'both tail slots'
    assert any(k.multi_phase for k in st), 'transposed convs (four phases, a flush per phase)'
    assert {k.async_epi for k in st} == {0, 1} and any(k.multi_unit for k in st) and any(k.MG > 1 for k in st)
    assert any(k.multi_image for k in st) and any(k.flags and k.multi_image for k in fin)
    assert {k.site for k in fin} == {'tail0', 'tail1'} and any(k.mean_rstd for k in fin) and any(k.stats == 'instance' for k in fin)
    assert {k.nadd for k in ap} == {0, 1, 2} and {k.prec for k in ap} == {0, 1}
    assert {k.pad for k in ap if k.pad_mode == 2} >= {1, 3} and any(k.parity for k in ap) and any(k.idle for k in ap)
    assert any(k.scale == 'bias' for k in ap) and any(k.repeat for k in ap)


def test_vgg_plans_have_no_norm():
    for tag, d in PP.vgg():
        for train in (False, True):
            assert _plan_describe(d, 'precise', train=train)['epilogue_forward'] == [], tag


def test_every_product_epilogue_key_has_a_gpu_case():
    cases = case_keys()
    reached = set().union(*cases.values())
    keys = product_keys()
    print('%d forward epilogue keys in the products' % len(keys))
    for k, where in keys.items():
        by = [n for n, ks in cases.items() if k in ks]
        print('  %s  (%s)  reached by %s' % (tuple(k), where, by[0] if by else 'NONE'))
    missing = [(k, where) for k, where in keys.items() if k not in reached]
    assert not missing, '%d forward epilogue paths of the products are reached by no GPU case:\n%s' % (
        len(missing), '\n'.join('  %s  e.g. %s' % (tuple(k), where) for k, where in missing))


def test_unreached_keys_are_listed():
    """Every listed path is run by a GPU case and reached by no product; every case key is a product key or listed."""
    prod = set(product_keys())
    reached = set().union(*case_keys().values())
    assert not set(UNREACHED) & prod, sorted(set(UNREACHED) & prod)
    assert set(UNREACHED) <= reached, sorted(set(UNREACHED) - reached)
    unlisted = sorted((name, tuple(k)) for name, ks in case_keys().items() for k in ks - prod - set(UNREACHED))
    assert not unlisted, 'case keys no product reaches and UNREACHED does not list: %s' % unlisted


def test_every_gpu_case_is_needed():
    """Each case reaches a key no other case reaches: a product key or a listed unreached one."""
    wanted = set(product_keys()) | set(UNREACHED)
    cases = case_keys()
    for name, keys in cases.items():
        others = set().union(*(k for n, k in cases.items() if n != name))
        assert (keys & wanted) - others, '%s reaches no key of its own: %s' % (name, sorted(keys))
