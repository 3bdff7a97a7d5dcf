"""CPU-only census of the tensor-core backward: every data-gradient and weight-gradient configuration that cfg3's training
step runs must also be run by a GPU parity case against fp64 (test_gpu_backward_variants / test_gpu_backward), and the convs
whose backward stays on the fp32 SIMT kernels are pinned with the reason.

choose_backward_unit (csrc/plan_backward.cu) picks, for each live conv of a training plan, the data-gradient mode (1 stride-1 conv,
2 transposed conv, 3 stride-2 conv as a cropped transposed conv), the sub-plan's forward conv on conv_umma_kernel and the
wgrad_umma_kernel launch; v2v_plan_describe reports that choice under "backward" without a GPU, assuming the H100 SXM's
132 SMs as the forward lowering does."""
import collections
import functools

import pytest

import bench
import test_conv_variant_census as CEN
from test_conv_variant_census import _h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan

WgradVariant = collections.namedtuple('WgradVariant', 'mode swap Mblocks Nblocks BN b_row KP split ksplit partial_m partial_n ragged')
DgradVariant = collections.namedtuple('DgradVariant', 'mode conv')


def wgrad_variant(b):
    """The fields of a weight-gradient launch that select a code path of wgrad_umma_kernel: operand roles, tile shapes, the
    split-K atomics, partial M / N tiles and a row segment shorter than KP pixels."""
    w = b['wgrad']
    return WgradVariant(b['mode'], w['swap'], w['Mblocks'], w['Nblocks'], w['BN'], w['b_row'], w['KP'], w['split'],
                        int(w['ksplit'] > 1), int(w['Mp'] % (64 * w['Mblocks']) != 0), int(w['Np'] % w['BN'] != 0),
                        int(w['gw'] % w['KP'] != 0))


def _describe(describe):
    p = Plan(0, precision='precise', train=True)
    describe(p)
    return p.describe()


def _walk(describe, tag, add):
    d = _describe(describe)
    fwd = [c for c in d['convs'] if c['grad']]      # one backward record per live conv, in graph order
    assert len(fwd) == len(d['backward']), (tag, len(fwd), len(d['backward']))
    for c, b in zip(fwd, d['backward']):
        add(tag, c, b)


def _collect(describes):
    """{variant: where} for the weight- and data-gradient variants, and [(where, reason)] for the SIMT fallbacks."""
    wg, dg, simt = collections.OrderedDict(), collections.OrderedDict(), []

    def add(tag, c, b):
        where = CEN._where(tag, c)
        if not b['mode']:
            simt.append((where, b['simt']))
            return
        dg.setdefault(DgradVariant(b['mode'], CEN.variant(b['conv'])), where)
        if b['wgrad'] is None:
            simt.append((where + ' (weight gradient)', b['wgrad_simt']))
        else:
            wg.setdefault(wgrad_variant(b), where)
    for tag, describe in describes:
        _walk(describe, tag, add)
    return wg, dg, simt


def _benchmark_describes():
    """cfg3's training step as bench.py runs it: the generator scales (the finest reads the exact one-hot + edge input) and the
    image / temporal discriminator towers at the avg-pool pyramid levels Vid2VidModelD feeds them."""
    W = bench.WORKLOADS['cfg3']
    opt = bench.make_opt_for('cfg3')
    opt.gpu_ids = []
    out = []
    for s in range(W['n_scales']):
        sc = 2 ** (W['n_scales'] - 1 - s)
        net = NW.build_netG(opt, s)
        net.input_exact_bf16 = s == W['n_scales'] - 1 and opt.label_nc != 0
        out.append(('cfg3 G%d' % s, functools.partial(lambda net, h, w, p: net._describe(p, 1, h, w), net, W['H'] // sc, W['W'] // sc)))
    num_D, n_frames_D = 3, 3
    for name, nc in (('D', opt.label_nc + int(opt.use_instance) + opt.output_nc), ('D_T', opt.output_nc * n_frames_D + 2 * (n_frames_D - 1))):
        d = NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, num_D, not opt.no_ganFeat, [])
        h, w = W['H'], W['W']
        for i in range(num_D):
            tower = num_D - 1 - i
            out.append(('cfg3 %s tower %d' % (name, tower), functools.partial(lambda d, t, h, w, p: d._describe(p, t, 1, h, w), d, tower, h, w)))
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return out


@functools.lru_cache(maxsize=None)
def benchmark_backward():
    return _collect(_benchmark_describes())


def _runner_describe(build, shape, head=None, scale=1.0, exact=False):
    def describe(p):
        r = NW.SequentialRunner(build(), head() if head else None, scale)
        r.input_exact_bf16 = exact
        r._describe(p, *shape)
    return describe


@functools.lru_cache(maxsize=None)
def case_backward():
    """{case id: (weight-gradient variants, data-gradient variants)} over the GPU backward parity cases whose gradients are held
    to a strict bound.  The DEEP units of test_gpu_backward are left out: their only gradient check is the flip-tolerant
    relative L2 <= 8e-2, which a defect confined to one configuration's path would pass."""
    import test_gpu_backward as TB
    import test_gpu_backward_variants as TV
    out = {}
    strict = [u for u in TB.UNITS if u[0] not in TB.DEEP] + TB.TENSOR_UNITS
    cases = [('test_gpu_backward::' + u[0], _runner_describe(u[1], u[2], *u[3:])) for u in strict]
    cases += [('test_gpu_backward::head_' + h[0], _runner_describe(h[1], h[4], h[2], h[3])) for h in TB.HEADS]
    cases += [('test_gpu_backward_variants::' + c[0], _runner_describe(c[1], c[2], c[3], c[4], c[5])) for c in TV.CASES]
    for key, describe in cases:
        wg, dg, _ = _collect([(key, describe)])
        out[key] = (set(wg), set(dg))
    return out


def _dgrad_reached(v, bwd_dg, fwd):
    # the sub-plan conv runs conv_umma_kernel like any forward conv: a forward parity case of the same configuration counts
    return v in bwd_dg or v.conv in fwd


def test_every_weight_gradient_variant_has_a_case():
    wg, _, _ = benchmark_backward()
    reached = set().union(*(w for w, _ in case_backward().values()))
    missing = [(v, where) for v, where in wg.items() if v not in reached]
    assert not missing, '%d weight-gradient configurations of cfg3 are reached by no GPU parity case:\n%s' % (
        len(missing), '\n'.join('  %s  e.g. %s' % (v, where) for v, where in missing))


def test_every_data_gradient_variant_has_a_case():
    _, dg, _ = benchmark_backward()
    bwd_dg = set().union(*(d for _, d in case_backward().values()))
    fwd = set().union(*CEN.unit_variants().values())
    missing = [(v, where) for v, where in dg.items() if not _dgrad_reached(v, bwd_dg, fwd)]
    assert not missing, '%d data-gradient configurations of cfg3 are reached by no GPU parity case:\n%s' % (
        len(missing), '\n'.join('  %s  e.g. %s' % (v, where) for v, where in missing))


# The convs of cfg3's training step whose backward (or only its weight gradient) runs on the fp32 SIMT kernels, as
# (conv, reason): none today.  A new entry is a visible slowdown of the training step, not a silent one.
SIMT_FALLBACKS = set()


def test_simt_fallbacks_are_pinned():
    _, _, simt = benchmark_backward()
    assert set(simt) == SIMT_FALLBACKS, sorted(set(simt) ^ SIMT_FALLBACKS)


def test_backward_census_is_not_vacuous():
    wg, dg, _ = benchmark_backward()
    assert len(wg) >= 15 and len(dg) >= 15, (len(wg), len(dg))
    assert {v.mode for v in wg} == {1, 2, 3}
    assert any(v.swap for v in wg) and any(v.ksplit for v in wg) and any(v.ragged for v in wg) and any(v.partial_m for v in wg)


def test_simt_switch_is_honoured(monkeypatch):
    monkeypatch.setenv('V2V_BWD', 'simt')
    recs = _describe(_runner_describe(lambda: NW._down(64, 128, NW.get_norm_layer('batch')), (1, 64, 16, 80)))['backward']
    assert recs and all(b['mode'] == 0 and b['simt'] == 'V2V_BWD=simt' and b['wgrad'] is None for b in recs), recs


def test_every_backward_variant_case_is_needed():
    """Each case of test_gpu_backward_variants reaches a cfg3 backward configuration that no other case reaches."""
    import test_gpu_backward_variants as TV
    wg, dg, _ = benchmark_backward()
    cases = case_backward()
    fwd = set().union(*CEN.unit_variants().values())
    for name in [c[0] for c in TV.CASES]:
        key = 'test_gpu_backward_variants::' + name
        w_others = set().union(*(w for k, (w, _) in cases.items() if k != key))
        d_others = set().union(*(d for k, (_, d) in cases.items() if k != key))
        own_w = cases[key][0] & set(wg) - w_others
        own_d = {v for v in cases[key][1] & set(dg) if not _dgrad_reached(v, d_others, fwd)}
        assert own_w or own_d, '%s reaches no cfg3 backward configuration of its own' % name


def main():
    wg, dg, simt = benchmark_backward()
    cases = case_backward()
    fwd_cases = CEN.unit_variants()
    print('cfg3 weight-gradient variants: %d' % len(wg))
    for v, where in wg.items():
        by = [k for k, (w, _) in cases.items() if v in w]
        print('  %-100s %s\n      reached by: %s' % (tuple(v), where, by[0] if by else 'NONE'))
    print('cfg3 data-gradient variants: %d' % len(dg))
    for v, where in dg.items():
        by = [k for k, (_, d) in cases.items() if v in d] + [k for k, f in fwd_cases.items() if v.conv in f]
        print('  mode %d %-96s %s\n      reached by: %s' % (v.mode, tuple(v.conv), where, by[0] if by else 'NONE'))
    print('SIMT fallbacks:')
    for where, why in simt:
        print('  %s: %s' % (where, why))


if __name__ == '__main__':
    main()
