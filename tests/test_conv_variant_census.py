"""CPU-only census of conv_umma_kernel's code paths: every kernel configuration that the benchmark's plans lower must also be
lowered by a GPU parity case (test_gpu_conv / test_gpu_backward), where it is compared with an fp64 (or bf16-emulated)
evaluation of the same layers at unit tolerance.

The host picks one configuration per convolution (fill_conv_params in csrc/conv_lower.cu): 2-D patch or row tiles and the taps per
patch, single or multi-phase (transposed) tiling, N tile, K block, M blocking, resident or streamed weights, the coupled
stages or the decoupled operand rings (with taps per weight chunk), precise or fast arithmetic, the exact-bf16 input
shortcut and the kx-GEMM head.  v2v_plan_describe reports that choice without a GPU.  The choice depends on the SM count:
with no device the lowering assumes the H100 SXM's 132 SMs, and on a GPU host the census runs only on a 132-SM device."""
import collections
import functools

import pytest
import torch

import bench
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan

H100_SXM_SMS = 132

Variant = collections.namedtuple('Variant', 'kind patch R multi_phase BN kc MG resident split a_exact ring2 TB headkx async_epi')


def variant(c):
    """The fields of a described conv that select a code path of the kernel (the stage / commit-group / unit counts CG, SG,
    SBr and units only tune it; async_epi selects the 640-thread instantiation whose epilogue warpgroup stores each unit
    while the consumers multiply the next)."""
    return Variant(c['kind'], c['p2d'], c['R'], int(c['phases'] > 1), c['BN'], c['kc'], c['MG'], c['resident'], c['split'],
                   c['a_exact'], c['ring2'], c['TB'], c['headkx'], c['async_epi'])


@pytest.fixture(autouse=True)
def _h100_sxm():
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != H100_SXM_SMS:
        pytest.skip('the census describes a %d-SM H100 SXM; this device has %d SMs' % (
            H100_SXM_SMS, torch.cuda.get_device_properties(0).multi_processor_count))


def _convs(describe, mode, train=False):
    p = Plan(0, precision=mode, train=train)
    describe(p)
    return p.describe()['convs']


def _where(tag, c):
    return '%s: %d->%d %dx%d stride %d%s, grid %dx%d' % (tag, c['Cin'], c['Cout'], c['k'][0], c['k'][1], c['stride'],
                                                       ' transposed' if c['transposed'] else '', c['grid'][0], c['grid'][1])


@functools.lru_cache(maxsize=None)
def benchmark_variants():
    """{variant: one benchmark conv that uses it} over the plans bench.py runs."""
    found = collections.OrderedDict()

    def add(tag, convs):
        for c in convs:
            found.setdefault(variant(c), _where(tag, c))
    # generators: inference workloads in both modes, the training step in precise mode; the finest scale reads the exact
    # one-hot + edge input (Vid2VidModelG.initialize sets input_exact_bf16 there when label_nc != 0)
    for wl, modes, train in (('cfg4', ('fast', 'precise'), False), ('cfg2', ('fast', 'precise'), False), ('cfg3', ('precise',), True)):
        W = bench.WORKLOADS[wl]
        opt = bench.make_opt_for(wl)
        opt.gpu_ids = []
        for s in range(W['n_scales']):
            sc = 2 ** (W['n_scales'] - 1 - s)
            net = NW.build_netG(opt, s)
            net.input_exact_bf16 = s == W['n_scales'] - 1 and opt.label_nc != 0
            for mode in modes:
                add('%s %s G%d' % (wl, mode, s), _convs(lambda p: net._describe(p, 1, W['H'] // sc, W['W'] // sc), mode, train))
    # cfg3's image and temporal discriminators at the shapes Vid2VidModelD feeds them: one clip per GPU, one generated frame
    # per step, each tower on its level of the avg-pool pyramid
    W = bench.WORKLOADS['cfg3']
    opt = bench.make_opt_for('cfg3')
    num_D, n_frames_D = 3, 3                     # bench.py's training options
    for name, nc in (('D', opt.label_nc + int(opt.use_instance) + opt.output_nc), ('D_T', opt.output_nc * n_frames_D + 2 * (n_frames_D - 1))):
        d = NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, num_D, not opt.no_ganFeat, [])
        h, w = W['H'], W['W']
        for i in range(num_D):
            tower = num_D - 1 - i
            add('cfg3 %s tower %d' % (name, tower), _convs(lambda p: d._describe(p, tower, 1, h, w), 'precise', True))
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    # FlowNet2 on one frame pair (the flownet2 workload, and cfg3's reference flow at the same size)
    W = bench.WORKLOADS['flownet2']
    f = FN.FlowNet2()
    for name in ('flownetc', 'flownets_1', 'flownets_2', 'flownets_d', 'flownetfusion'):
        sub = getattr(f, name)
        add('flownet2 ' + name, _convs(lambda p: sub.describe(p, 1, W['H'], W['W']), FN.FlowNet2.precision))
    return found


def _case_variants(build, shape, modes, head=None, scale=1.0, exact=False, train=False):
    r = NW.SequentialRunner(build(), head() if head else None, scale)
    r.input_exact_bf16 = exact
    return {variant(c) for mode in modes for c in _convs(lambda p: r._describe(p, *shape), mode, train)}


@functools.lru_cache(maxsize=None)
def unit_variants():
    """{case id: variants its forward lowers} over the GPU parity cases."""
    import test_gpu_backward as TB
    import test_gpu_conv as TC
    out = {}
    for name, build, shape in TC.CASES:
        out['test_gpu_conv::' + name] = _case_variants(build, shape, TC.MODES)
    for name, build, head, scale, shape in TC.HEADS:
        out['test_gpu_conv::' + name] = _case_variants(build, shape, TC.MODES, head, scale)
    for name, build, shape, modes, exact in TC.VARIANT_CASES:
        out['test_gpu_conv::' + name] = _case_variants(build, shape, modes, exact=exact)
    for name, build, head, scale, shape, modes in TC.VARIANT_HEADS:
        out['test_gpu_conv::' + name] = _case_variants(build, shape, modes, head, scale)
    # the backward tests run precise training plans; each compares the plan's forward output with fp64 before its gradients
    for u in TB.UNITS + TB.TENSOR_UNITS:
        out['test_gpu_backward::' + u[0]] = _case_variants(u[1], u[2], ('precise',), *u[3:], train=True)
    for name, build, head, scale, shape in TB.HEADS:
        out['test_gpu_backward::head_' + name] = _case_variants(build, shape, ('precise',), head, scale, train=True)
    return out


def test_every_benchmark_conv_configuration_has_a_unit_case():
    reached = set().union(*unit_variants().values())
    missing = [(v, where) for v, where in benchmark_variants().items() if v not in reached]
    assert not missing, '%d kernel configurations the benchmark runs are not reached by any GPU parity case:\n%s' % (
        len(missing), '\n'.join('  %s  e.g. %s' % (v, where) for v, where in missing))


def test_census_is_not_vacuous():
    bv = benchmark_variants()
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
    assert len(set().union(*unit_variants().values())) >= len(bv)


def test_every_variant_case_is_needed():
    """Each case added for the census reaches a benchmark configuration that no other case reaches: the list stays minimal,
    and deleting a case fails the census."""
    import test_gpu_conv as TC
    units, bv = unit_variants(), set(benchmark_variants())
    for name in [c[0] for c in TC.VARIANT_CASES + TC.VARIANT_HEADS]:
        key = 'test_gpu_conv::' + name
        others = set().union(*(vs for k, vs in units.items() if k != key))
        assert units[key] & bv - others, '%s reaches no benchmark configuration of its own' % name
