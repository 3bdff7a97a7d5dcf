"""CPU-only census of the conv kernels' code paths: every conv_umma_kernel configuration, every data-gradient and every
wgrad_umma_kernel configuration that the products' plans (tests/product_plans.py) lower must also be lowered by a GPU parity
case that compares it with fp64 (or bf16-emulated fp32 in fast mode), and the convs whose backward stays on the fp32 SIMT
kernels are pinned with the reason.

The host picks one configuration per convolution (fill_conv_params in csrc/conv_lower.cu): 2-D patch or row tiles and the taps
per patch, single or multi-phase (transposed) tiling, N tile, K block, M blocking, resident or streamed weights, the coupled
stages or the decoupled operand rings (with taps per weight chunk), precise or fast arithmetic, the exact-bf16 input shortcut,
the kx-GEMM head and the epilogue warpgroup.  For each live conv of a training plan choose_backward_unit
(csrc/plan_backward.cu) picks the data-gradient mode (1 stride-1 conv, 2 transposed conv, 3 stride-2 conv as a cropped
transposed conv), the sub-plan's forward conv on conv_umma_kernel and the wgrad_umma_kernel launch.  v2v_plan_describe reports
both choices without a GPU.

The census is layered: each level's product keys may be reached only by the case lists at or below it, so that a case checking
a configuration closely is not made redundant by a later case that reaches it through a looser check.

  bench                    bench.py's plans        test_gpu_conv's CASES, HEADS and VARIANT_*; test_gpu_backward's UNITS,
                                                   TENSOR_UNITS and HEADS (each compares the plan's forward with fp64)
  multiclip                multi-clip, slot plans  + test_gpu_multiclip.CONV_CASES
  product                  first frame, VGG, pose  + test_gpu_product_variants.FWD_CASES
  cfg3 weight / data       cfg3's training step    test_gpu_backward's units held to a strict bound (not DEEP: their only
  gradient                                         gradient check is a flip-tolerant relative L2, which a defect confined to
                                                   one configuration's path would pass) and HEADS; test_gpu_backward_variants
  product weight / data    the pose step; VGG's    + test_gpu_product_variants.BWD_CASES
  gradient                 data gradients

A data gradient's sub-plan conv runs conv_umma_kernel like any forward conv, so a forward case of the same configuration counts
for it too: a bench-level case on the cfg3 level, any forward case on the product level."""
import collections
import functools

import census as C
import product_plans as PP
from product_plans import h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)
from vid2vid_b200 import networks as NW

Variant = collections.namedtuple('Variant', 'kind patch R multi_phase BN kc MG resident split a_exact ring2 TB headkx async_epi')
WgradVariant = collections.namedtuple('WgradVariant', 'mode swap Mblocks Nblocks BN b_row KP split ksplit partial_m partial_n ragged')
DgradVariant = collections.namedtuple('DgradVariant', 'mode conv')
DGRAD_MODES = (1, 2, 3)


def variant(c):
    """The fields of a described conv that select a code path of the kernel (the stage / commit-group / unit counts CG, SG,
    SBr and units only tune it; async_epi selects the 640-thread instantiation whose epilogue warpgroup stores each unit
    while the consumers multiply the next)."""
    return Variant(c['kind'], c['p2d'], c['R'], int(c['phases'] > 1), c['BN'], c['kc'], c['MG'], c['resident'], c['split'],
                   c['a_exact'], c['ring2'], c['TB'], c['headkx'], c['async_epi'])


def wgrad_variant(b):
    """The fields of a weight-gradient launch that select a code path of wgrad_umma_kernel: operand roles, tile shapes, the
    split-K atomics, partial M / N tiles and a row segment shorter than KP pixels."""
    w = b['wgrad']
    return WgradVariant(b['mode'], w['swap'], w['Mblocks'], w['Nblocks'], w['BN'], w['b_row'], w['KP'], w['split'],
                        int(w['ksplit'] > 1), int(w['Mp'] % (64 * w['Mblocks']) != 0), int(w['Np'] % w['BN'] != 0),
                        int(w['gw'] % w['KP'] != 0))


def _where(tag, c):
    return '%s: %d->%d %dx%d stride %d%s, grid %dx%d' % (tag, c['Cin'], c['Cout'], c['k'][0], c['k'][1], c['stride'],
                                                       ' transposed' if c['transposed'] else '', c['grid'][0], c['grid'][1])


def forward(specs):
    return C.first_where((variant(c), _where(s.tag, c)) for s in specs for c in PP.describe(s)['convs'])


def backward(specs):
    """({weight-gradient variant: where}, {data-gradient variant: where}, [(conv, reason)] of the SIMT fallbacks) of training
    plans."""
    wg, dg, simt = [], [], []
    for s in specs:
        d = PP.describe(s)
        fwd = [c for c in d['convs'] if c['grad']]      # one backward record per live conv, in graph order
        assert len(fwd) == len(d['backward']), (s.tag, len(fwd), len(d['backward']))
        for c, b in zip(fwd, d['backward']):
            where = _where(s.tag, c)
            if not b['mode']:
                simt.append((where, b['simt']))
                continue
            dg.append((DgradVariant(b['mode'], variant(b['conv'])), where))
            if b['wgrad'] is None:
                simt.append((where + ' (weight gradient)', b['wgrad_simt']))
            elif not s.frozen:      # no parameter asks for a gradient: the plan launches no weight gradient
                wg.append((wgrad_variant(b), where))
    return C.first_where(wg), C.first_where(dg), simt


@functools.lru_cache(maxsize=None)
def product_backward(level):
    groups = {'cfg3': ('bench',), 'product': ('pose_step', 'vgg')}[level]
    return backward([s for s in PP.group(*groups) if s.train])


def _case(name, build, shape, modes, head=None, scale=1.0, exact=False, train=False, sample_stats=False, frozen=False):
    def describe(p):
        r = NW.SequentialRunner(build(), head() if head else None, scale)
        r.input_exact_bf16 = exact
        r._describe(p, *shape)
    return name, [PP.PlanSpec('case', name, describe, m, train, sample_stats, frozen=frozen) for m in modes]


@functools.lru_cache(maxsize=None)
def cases():
    """{list: [(case id, its plans)]} over the GPU parity cases, described from the same builders the GPU tests run."""
    import test_gpu_backward as TB
    import test_gpu_backward_variants as TV
    import test_gpu_conv as TC
    import test_gpu_multiclip as TMC
    import test_gpu_product_variants as TP
    P = ('precise',)
    units = {u[0]: _case('test_gpu_backward::' + u[0], u[1], u[2], P, *u[3:], train=True) for u in TB.UNITS + TB.TENSOR_UNITS}
    heads = [_case('test_gpu_backward::head_' + n, b, s, P, h, k, train=True) for n, b, h, k, s in TB.HEADS]
    return {
        'fwd_bench': [_case('test_gpu_conv::' + n, b, s, TC.MODES) for n, b, s in TC.CASES] +
                     [_case('test_gpu_conv::' + n, b, s, TC.MODES, h, k) for n, b, h, k, s in TC.HEADS] +
                     list(units.values()) + heads,
        'fwd_variant': [_case('test_gpu_conv::' + n, b, s, m, exact=e) for n, b, s, m, e in TC.VARIANT_CASES] +
                       [_case('test_gpu_conv::' + n, b, s, m, h, k) for n, b, h, k, s, m in TC.VARIANT_HEADS],
        'fwd_multiclip': [_case('test_gpu_multiclip::' + n, b, s, m, sample_stats=True) for n, b, s, m in TMC.CONV_CASES],
        'fwd_product': [_case('test_gpu_product_variants::' + n, b, s, m, h) for n, b, h, s, m in TP.FWD_CASES],
        'bwd_bench': [c for n, c in units.items() if n not in TB.DEEP] + heads,
        'bwd_variant': [_case('test_gpu_backward_variants::' + n, b, s, P, h, k, e, train=True) for n, b, s, h, k, e in TV.CASES],
        'bwd_product': [_case('test_gpu_product_variants::' + n, b, s, P, train=True, frozen=f) for n, b, s, f in TP.BWD_CASES],
    }


def _union(*levels):
    out = collections.defaultdict(set)
    for level in levels:
        for name, keys in level.items():
            out[name] |= keys
    return out


@functools.lru_cache(maxsize=None)
def levels():
    """{level: (product keys {key: where}, cases {case id: keys})}, each level counting the case lists at or below it."""
    cs = cases()
    fwd = {k: {name: set(forward(specs)) for name, specs in cs[k]} for k in cs if k.startswith('fwd')}
    wg, dg = {}, {}
    for k in ('bwd_bench', 'bwd_variant', 'bwd_product'):
        keys = {name: backward(specs) for name, specs in cs[k]}
        wg[k], dg[k] = ({name: set(b[i]) for name, b in keys.items()} for i in (0, 1))
    f1 = _union(fwd['fwd_bench'], fwd['fwd_variant'])
    f2 = _union(f1, fwd['fwd_multiclip'])
    f3 = _union(f2, fwd['fwd_product'])
    as_dgrad = lambda f: {name: {DgradVariant(m, v) for v in keys for m in DGRAD_MODES} for name, keys in f.items()}
    w1, d1 = _union(wg['bwd_bench'], wg['bwd_variant']), _union(dg['bwd_bench'], dg['bwd_variant'])
    return {
        'bench': (forward(PP.group('bench')), f1),
        'multiclip': (forward(PP.group('multiclip', 'slots')), f2),
        'product': (forward(PP.group('first_frame', 'vgg', 'pose_step')), f3),
        'cfg3 weight gradient': (product_backward('cfg3')[0], w1),
        'cfg3 data gradient': (product_backward('cfg3')[1], _union(d1, as_dgrad(f1))),
        'product weight gradient': (product_backward('product')[0], _union(w1, wg['bwd_product'])),
        'product data gradient': (product_backward('product')[1], _union(d1, dg['bwd_product'], as_dgrad(f3))),
    }


def test_every_bench_configuration_has_a_case():
    C.assert_reached('bench configurations', *levels()['bench'])


def test_every_multiclip_configuration_has_a_case():
    C.assert_reached('multiclip configurations', *levels()['multiclip'])


def test_every_product_configuration_has_a_case():
    C.assert_reached('product configurations', *levels()['product'])


def test_every_cfg3_weight_gradient_configuration_has_a_case():
    C.assert_reached('cfg3 weight-gradient configurations', *levels()['cfg3 weight gradient'])


def test_every_cfg3_data_gradient_configuration_has_a_case():
    C.assert_reached('cfg3 data-gradient configurations', *levels()['cfg3 data gradient'])


def test_every_product_weight_gradient_configuration_has_a_case():
    C.assert_reached('product weight-gradient configurations', *levels()['product weight gradient'])


def test_every_product_data_gradient_configuration_has_a_case():
    C.assert_reached('product data-gradient configurations', *levels()['product data gradient'])


# Each case a census added must reach a configuration of its own level that no other case at or below that level reaches:
# the lists stay minimal, and deleting a case fails the census.
def _assert_needed(added, *level_names):
    C.assert_needed([name for name, _ in cases()[added]], [levels()[level] for level in level_names])


def test_every_variant_case_is_needed():
    _assert_needed('fwd_variant', 'bench')


def test_every_multiclip_case_is_needed():
    _assert_needed('fwd_multiclip', 'multiclip')


def test_every_backward_variant_case_is_needed():
    _assert_needed('bwd_variant', 'cfg3 weight gradient', 'cfg3 data gradient')


def test_every_product_case_is_needed():
    _assert_needed('fwd_product', 'product')
    _assert_needed('bwd_product', 'product weight gradient', 'product data gradient')


def test_bench_census_is_not_vacuous():
    bv, f1 = levels()['bench']
    assert len(bv) >= 50, len(bv)
    known = {
        'precise 7x7 stem on the decoupled rings, 4 taps per weight chunk': lambda v: v.ring2 and v.TB == 4 and v.R == 7,
        'exact-bf16 input, M blocking': lambda v: v.a_exact and v.MG == 2,
        'kx-GEMM 7x7 head': lambda v: v.headkx == 7,
        'kx-GEMM 4x4 logit head': lambda v: v.headkx == 4,
        'multi-phase transposed conv': lambda v: v.multi_phase,
        '2-D patch': lambda v: v.patch,
        'fast mode': lambda v: not v.split,
    }
    for name, pred in known.items():
        assert any(pred(v) for v in bv), name
    assert len(set().union(*f1.values())) >= len(bv)


def test_multiclip_census_is_not_vacuous():
    mv = levels()['multiclip'][0]
    assert len(mv) >= 50, len(mv)
    assert any(v.async_epi for v in mv) and any(not v.split for v in mv) and any(v.patch for v in mv)


def test_backward_census_is_not_vacuous():
    wg, dg, _ = product_backward('cfg3')
    assert len(wg) >= 15 and len(dg) >= 15, (len(wg), len(dg))
    assert {v.mode for v in wg} == set(DGRAD_MODES)
    assert any(v.swap for v in wg) and any(v.ksplit for v in wg) and any(v.ragged for v in wg) and any(v.partial_m for v in wg)


def test_product_census_is_not_vacuous():
    pv = levels()['product'][0]
    wg, dg, _ = product_backward('product')
    assert len(pv) >= 40 and len(wg) >= 15 and len(dg) >= 15, (len(pv), len(wg), len(dg))
    known = {
        'face Encoder head: 2-D patch of 49 taps, fast': lambda v: v.kind == 4 and v.patch and v.R == 49 and not v.split,
        'Global_with_z stem: M blocking 2, 32-channel K blocks': lambda v: v.R == 7 and v.MG == 2 and v.kc == 32,
        'VGG conv2_1 on the decoupled rings with the epilogue warpgroup': lambda v: v.ring2 and v.TB == 1 and v.async_epi,
    }
    for name, pred in known.items():
        assert any(pred(v) for v in pv), name
    assert any(v.Mblocks == 2 and v.Nblocks == 2 and v.BN == 128 and v.KP == 32 and not v.ksplit for v in wg), 'no-K-split wgrad'
    assert any(v.ragged and v.swap for v in wg), 'ragged swapped logit wgrad'
    # the street first-frame generators are listed, in both modes
    tags = [s.tag for s in PP.group('first_frame')]
    assert sum(t.startswith('City') for t in tags) == 3 * len(PP.MODES) and any('netE' in t for t in tags)


# The convs of cfg3's training step and of the product training plans whose backward (or only its weight gradient) runs on
# the fp32 SIMT kernels, as (conv, reason): none today.  A new entry is a visible slowdown of the training step, not a silent one.
SIMT_FALLBACKS = {'cfg3': set(), 'product': set()}


def _assert_simt_pinned(level):
    simt = set(product_backward(level)[2])
    assert simt == SIMT_FALLBACKS[level], sorted(simt ^ SIMT_FALLBACKS[level])


def test_cfg3_simt_fallbacks_are_pinned():
    _assert_simt_pinned('cfg3')


def test_product_simt_fallbacks_are_pinned():
    _assert_simt_pinned('product')


def test_simt_switch_is_honoured(monkeypatch):
    monkeypatch.setenv('V2V_BWD', 'simt')
    _, (spec,) = _case('simt', lambda: NW._down(64, 128, NW.get_norm_layer('batch')), (1, 64, 16, 80), ('precise',), train=True)
    recs = PP.describe(spec)['backward']
    assert recs and all(b['mode'] == 0 and b['simt'] == 'V2V_BWD=simt' and b['wgrad'] is None for b in recs), recs


def test_vgg_weight_gradients_are_not_launched():
    """The VGG loss plan describes a weight-gradient launch for its convs, but Vgg19 freezes its parameters, so the backward
    is handed no weight-gradient buffer and launches none (plan_backward.cu: need_w): the census does not ask for cases."""
    recs = [b for s in PP.group('vgg') if s.train for b in PP.describe(s)['backward']]
    assert recs and any(b['wgrad'] for b in recs) and all(s.frozen for s in PP.group('vgg'))
    assert not any(p.requires_grad for p in NW.Vgg19().parameters())
