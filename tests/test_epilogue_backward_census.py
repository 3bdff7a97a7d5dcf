"""CPU-only census of the CUDA-core epilogue backward (csrc/backward.cu): every launch path of the norm backward, the conv_act /
head backward and the bias gradient that cfg3's training step or the pose training step runs must also be run by a case of
tests/test_gpu_epilogue_backward.py, which holds it to an fp64 reference with a derived bound.

v2v_plan_describe reports, for training plans, one "epilogue_backward" record per live G_NORM_ACT / G_CONV_ACT / G_HEAD with
the launch shape norm_bwd_launch / bias_grad_blocks choose (the same host functions the launches call), without a GPU and
assuming the H100 SXM's 132 SMs.  Each record is reduced to the fields that select a code path or change the summation order."""
import collections
import functools

import census as C
import product_plans as PP
from product_plans import h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)

NormKey = collections.namedtuple('NormKey', 'reduce ppb1 multi_block ragged c_off adds act twice raw_f32 batch_stats multi_image')
BiasKey = collections.namedtuple('BiasKey', 'kind acts split multi_block')


def keys_of(d):
    """{key: record} of one plan description.  A raw slice normalised by more than one pass (CompositeLocalGenerator's
    defer_last) accumulates into draw / dgamma / dbeta once per pass; it is a key field of every such pass."""
    recs = d['epilogue_backward']
    passes = collections.Counter((r['raw'], r['c_off']) for r in recs if r['kind'] == 'norm_act')
    out = collections.OrderedDict()
    for r in recs:
        if r['kind'] == 'norm_act':
            vec = r['reduce'] == 'vec'
            k = NormKey(r['reduce'], int(vec and r['ppb'] == 1), int(r['grid'][0] > 1 if vec else r['grid'][2] > 1),
                        int(vec and (r['H'] * r['W']) % r['chunk'] != 0), int(r['c_off'] != 0), r['adds'], r['act'],
                        int(passes[(r['raw'], r['c_off'])] > 1), r['raw_f32'], r['batch_stats'], int(r['N'] > 1))
        else:
            k = BiasKey(r['kind'], tuple(sorted(set(r['acts']))), int(r['C1'] < r['C']), int(r['bias_grid'][1] > 1))
        out.setdefault(k, r)
    return out


@functools.lru_cache(maxsize=None)
def product_keys():
    """{key: where} over cfg3's training step (generator scales, D and D_T towers, as bench.py runs it) and the pose step with
    the face discriminator: the training plans of the inventory's bench and pose_step groups."""
    return C.first_where((k, '%s: %s %d ch @ %dx%d' % (s.tag, r['kind'], r['C'], r['H'], r['W']))
                         for s in PP.group('bench', 'pose_step') if s.train for k, r in keys_of(PP.describe(s)).items())


@functools.lru_cache(maxsize=None)
def case_keys():
    """{case id: keys} over the GPU cases, described from the same builders the GPU test runs (modules on the CPU)."""
    import test_gpu_epilogue_backward as EB
    return {name: set(keys_of(PP.describe(PP.PlanSpec('case', name, functools.partial(EB.build, spec=spec, device='cpu'),
                                                      EB.precision(spec), True))))
            for name, spec in EB.CASES}


# The launch paths GPU cases run although no product plan reaches them, each with the reason.  They are listed key by key, so
# that each one stays a path some case must run.
_K = NormKey
UNREACHED = {
    _K('scalar', 0, 0, 0, 0, 0, 1, 0, 1, 1, 0): 'scalar reduce, one pixel slice per channel: every product norm layer has '
                                                'C % 4 == 0 and C <= 1024',
    _K('scalar', 0, 1, 0, 0, 0, 1, 0, 1, 1, 0): 'scalar reduce, pixel slices meeting in global atomics (C > 1024): as above',
    _K('vec', 0, 1, 1, 0, 0, 2, 0, 1, 0, 1): 'InstanceNorm: cfg3 and the pose step train BatchNorm only (--norm batch)',
    _K('vec', 0, 1, 0, 0, 1, 1, 0, 0, 1, 0): 'bf16 raw: training runs precise plans, whose raw conv outputs are fp32',
    _K('vec', 0, 1, 1, 0, 1, 1, 0, 1, 1, 1): 'N > 1: the training steps run one clip per step',
}


def test_every_product_epilogue_key_has_a_gpu_case():
    C.assert_reached('epilogue backward launch paths of the products', product_keys(), case_keys())


def test_unreached_keys_are_listed():
    """Every listed path is run by a GPU case and reached by no product; every case key is a product key or listed."""
    C.assert_unreached_listed(product_keys(), case_keys(), UNREACHED)


def test_every_gpu_case_is_needed():
    """Each case reaches a key no other case reaches: a product key or a listed unreached one."""
    import test_gpu_epilogue_backward as EB
    C.assert_needed([name for name, _ in EB.CASES], [({**product_keys(), **UNREACHED}, case_keys())])


def test_census_is_not_vacuous():
    keys = product_keys()
    norm = [k for k in keys if isinstance(k, NormKey)]
    assert len(norm) >= 10 and len(keys) - len(norm) >= 4, (len(norm), len(keys))
    assert any(k.ppb1 for k in norm) and any(k.ragged for k in norm) and any(k.c_off for k in norm) and any(k.twice for k in norm)
    assert {k.adds for k in norm} == {0, 1, 2} and {k.act for k in norm} == {0, 1, 2}

