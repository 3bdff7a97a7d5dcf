"""CPU-only census of the conv kernel configurations that product paths outside bench.py run (tests/product_plans.py): the
first-frame generators (both arithmetic modes), the VGG19 loss and the pose training step with the face discriminator
(precise mode).  Every forward configuration must be lowered by a GPU parity case against fp64 (or bf16-emulated fp32), every
weight- and data-gradient configuration by a strict backward case, and the convs whose backward falls back to the SIMT kernels
are pinned.  Configurations are keyed as tests/test_conv_variant_census.py and tests/test_backward_variant_census.py key them;
the cases they count stay counted, and the cases of tests/test_gpu_product_variants.py are added."""
import collections
import functools

import test_backward_variant_census as BC
import test_conv_variant_census as CEN
import test_multiclip_census as MC
import product_plans as PP
from test_conv_variant_census import _h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)
from vid2vid_b200 import networks as NW

# The convs of the pose step whose backward (or only its weight gradient) runs on the fp32 SIMT kernels: none at 512x512.
SIMT_FALLBACKS = set()


def _forward(found, describes, modes, train):
    for tag, describe in describes:
        for mode in modes:
            for c in CEN._convs(describe, mode, train):
                found.setdefault(CEN.variant(c), CEN._where('%s %s' % (tag, mode), c))


@functools.lru_cache(maxsize=None)
def product_variants():
    """{variant: one product conv that uses it}."""
    found = collections.OrderedDict()
    _forward(found, PP.first_frame(), ('precise', 'fast'), False)
    _forward(found, PP.vgg(), ('precise',), True)
    _forward(found, PP.vgg(), ('precise',), False)
    _forward(found, PP.pose_step(), ('precise',), True)
    return found


@functools.lru_cache(maxsize=None)
def product_backward():
    """(weight-gradient variants, data-gradient variants, SIMT fallbacks) of the training plans: the pose step, and the VGG
    loss's data gradients (its weight-gradient records are described but never launched: see
    test_vgg_weight_gradients_are_not_launched)."""
    wg, dg, simt = BC._collect(PP.pose_step())
    _, vgg_dg, vgg_simt = BC._collect(PP.vgg())
    for v, where in vgg_dg.items():
        dg.setdefault(v, where)
    return wg, dg, simt + vgg_simt


@functools.lru_cache(maxsize=None)
def new_cases():
    """{case id: (forward variants, weight-gradient variants, data-gradient variants)} of test_gpu_product_variants."""
    import test_gpu_product_variants as TP
    out = {}
    for name, build, head, shape, modes in TP.FWD_CASES:
        out[name] = (CEN._case_variants(build, shape, modes, head), set(), set())
    for name, build, shape, frozen in TP.BWD_CASES:
        wg, dg, _ = BC._collect([(name, BC._runner_describe(build, shape))])
        # a frozen case gives the plan no weight to differentiate: its weight-gradient records are never launched
        out[name] = (set(), set() if frozen else set(wg), set(dg))
    return out


def _existing_forward():
    return set().union(*CEN.unit_variants().values(), *MC.multiclip_case_variants().values())


def _existing_backward():
    cases = BC.case_backward()
    return set().union(*(w for w, _ in cases.values())), set().union(*(d for _, d in cases.values()))


def _report(what, missing):
    return '%d %s configurations of the product plans are reached by no GPU parity case:\n%s' % (
        len(missing), what, '\n'.join('  %s  e.g. %s' % (v, where) for v, where in missing))


def test_every_product_conv_configuration_has_a_unit_case():
    reached = _existing_forward().union(*(f for f, _, _ in new_cases().values()))
    missing = [(v, where) for v, where in product_variants().items() if v not in reached]
    assert not missing, _report('forward', missing)


def test_every_product_weight_gradient_variant_has_a_case():
    wg, _, _ = product_backward()
    reached = _existing_backward()[0].union(*(w for _, w, _ in new_cases().values()))
    missing = [(tuple(v), where) for v, where in wg.items() if v not in reached]
    assert not missing, _report('weight-gradient', missing)


def test_every_product_data_gradient_variant_has_a_case():
    _, dg, _ = product_backward()
    bwd = _existing_backward()[1].union(*(d for _, _, d in new_cases().values()))
    fwd = _existing_forward().union(*(f for f, _, _ in new_cases().values()))
    missing = [((v.mode,) + tuple(v.conv), where) for v, where in dg.items() if not BC._dgrad_reached(v, bwd, fwd)]
    assert not missing, _report('data-gradient', missing)


def test_vgg_weight_gradients_are_not_launched():
    """The VGG loss plan describes a weight-gradient launch for its convs, but Vgg19 freezes its parameters, so the backward
    is handed no weight-gradient buffer and launches none (plan_backward.cu: need_w): the census does not ask for cases."""
    recs = [b for _, describe in PP.vgg() for b in BC._describe(describe)['backward']]
    assert recs and any(b['wgrad'] for b in recs)
    assert not any(p.requires_grad for p in NW.Vgg19().parameters())


def test_simt_fallbacks_are_pinned():
    _, _, simt = product_backward()
    assert set(simt) == SIMT_FALLBACKS, sorted(set(simt) ^ SIMT_FALLBACKS)


def test_product_census_is_not_vacuous():
    pv = product_variants()
    wg, dg, _ = product_backward()
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
    tags = [t for t, _ in PP.first_frame()]
    assert sum(t.startswith('City') for t in tags) == 3 and any('netE' in t for t in tags)


def test_every_product_case_is_needed():
    """Each case of test_gpu_product_variants reaches a product configuration that no other parity case reaches."""
    pv, (wg, dg, _) = set(product_variants()), product_backward()
    base_f, (base_w, base_d) = _existing_forward(), _existing_backward()
    cases = new_cases()
    for name, (f, w, d) in cases.items():
        others = [c for k, c in cases.items() if k != name]
        of = base_f.union(*(c[0] for c in others))
        ow = base_w.union(*(c[1] for c in others))
        od = base_d.union(*(c[2] for c in others))
        own = (f & pv - of) | (w & set(wg) - ow) | {v for v in d & set(dg) if not BC._dgrad_reached(v, od, of)}
        assert own, '%s reaches no product configuration of its own' % name
