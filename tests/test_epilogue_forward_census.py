"""CPU-only census of the forward epilogue of the norm layers: the statistics accumulation in conv_umma_kernel's epilogue, their
finalisation (the last CTA's tail of the conv launch, or stats_finalize_kernel) with the train-mode side effects, and the
normalise pass (norm_apply_rows_kernel / norm_apply_kernel).  Every path the products' plans (every group of
tests/product_plans.py) run must also be run by a case of tests/test_gpu_epilogue_forward.py, which holds it to an fp64
reference with a bound derived from the kernels' arithmetic.

v2v_plan_describe reports, for every plan, an "epilogue_forward" array (stats / finalize / apply records) with the choices
finalize_sites and norm_apply_launch make -- the host functions the plan's emission calls -- without a GPU and assuming the
H100 SXM's 132 SMs.  Each record is reduced to the fields that select a code path or change the summation order."""
import collections
import functools

import census as C
import product_plans as PP
from product_plans import h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)

# stats: which threads run the epilogue (async_epi), tiles per unit (MG), several phases (transposed convs: the key, and so the
# flushed accumulator, changes with the phase), whether one CTA accumulates several units (and so flushes at key changes inside
# its run), several images (a flush per image), and the finalising tail slots.  N tile and K
# block choose the kernel instantiation, which tests/test_conv_census.py already requires a parity case for.
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


@functools.lru_cache(maxsize=None)
def product_keys():
    """{key: where} over every plan of the inventory."""
    return C.first_where((k, _where(s.tag, r)) for s in PP.plans() for k, r in keys_of(PP.describe(s)).items())


@functools.lru_cache(maxsize=None)
def case_keys():
    """{case id: keys} over the GPU cases, described from the same builders the GPU test runs (modules on the CPU)."""
    import test_gpu_epilogue_forward as EF
    return {name: set().union(*(keys_of(PP.describe(PP.PlanSpec('case', name, functools.partial(EF.build, spec=spec, device='cpu'),
                                                                **EF.plan_options(spec, mode)))) for mode in spec.modes))
            for name, spec in EF.CASES}


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
    vgg = PP.group('vgg')
    assert {s.train for s in vgg} == {False, True}
    for s in vgg:
        assert PP.describe(s)['epilogue_forward'] == [], s.tag


def test_every_product_epilogue_key_has_a_gpu_case():
    C.assert_reached('forward epilogue paths of the products', product_keys(), case_keys())


def test_unreached_keys_are_listed():
    """Every listed path is run by a GPU case and reached by no product; every case key is a product key or listed."""
    C.assert_unreached_listed(product_keys(), case_keys(), UNREACHED)


def test_every_gpu_case_is_needed():
    """Each case reaches a key no other case reaches: a product key or a listed unreached one."""
    import test_gpu_epilogue_forward as EF
    C.assert_needed([name for name, _ in EF.CASES], [({**product_keys(), **UNREACHED}, case_keys())])
