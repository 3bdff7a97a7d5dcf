"""CPU-only census of the layout kernels (csrc/layout.cu, the gradient layout of csrc/backward.cu, fold_add and unstage of
csrc/wgrad_umma.cu): every layout launch path a product plan takes must also be taken by a case of tests/test_gpu_layout.py,
which holds it to bit equality.

v2v_plan_describe reports one "layout" record per import, export, concat copy and weight pack a plan launches, with the choice
import_tile_channels / pack_weights_tiling / grad_layout_tiled make (the host functions the launches call); training plans add
the gradient import and export of every output and input, and per tensor-core backward unit its fold, dgrad pack and unstage.
Each record is reduced to the fields that select a code path.  Training plans also key the data gradients the fp32 SIMT
kernel computes (mode 0 units), whose reflect fold the integer cases check."""
import collections
import functools

import census as C
import product_plans as PP
from product_plans import h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)

Import = collections.namedtuple('Import', 'kind CT pad_mode parity split skip_lo act window wide')
Export = collections.namedtuple('Export', 'kind split wide ragged direct')
Copy = collections.namedtuple('Copy', 'kind pad_mode split odd_c_off parity')
Pack = collections.namedtuple('Pack', 'kind TC dgrad w2 headkx transposed split')
GradLayout = collections.namedtuple('GradLayout', 'kind tiled window hw_ragged c_ragged')
Fold = collections.namedtuple('Fold', 'kind mode reflect crop overlap')
Unstage = collections.namedtuple('Unstage', 'kind swap dw2 multi_tap')
SimtDgrad = collections.namedtuple('SimtDgrad', 'kind k stride transposed why')


# Every key starts with its kind, so that keys of different kinds never compare equal as tuples.
def _key(r):
    k = r['kind']
    if k == 'import':
        return Import('import', r['CT'], r['pad_mode'], r['parity'], r['split'], r['skip_lo'], r['act'],
                      int(r['c_off'] != 0 or r['C_src'] != r['Cvalid']), int(r['Wpad'] > 128))
    if k == 'export':
        return Export('export', r['split'], int(r['W'] > 128), int(r['Cvalid'] % 32 != 0), r['direct'])
    if k == 'copy':
        return Copy('copy', r['pad_mode'], r['split'], r['c_off'] % 2, r['parity'])
    if k == 'pack':
        return Pack('pack', r['TC'], r['dgrad'], r['w2'], int(r['headkx'] > 0), r['transposed'], r['split'])
    if k in ('grad_import', 'grad_export'):
        return GradLayout(k, r['tiled'], int(r['c_off'] != 0 or r['C_src'] != r['C']), int(r['H'] * r['W'] % 32 != 0),
                          int(r['C'] % 32 != 0))
    if k == 'fold':
        return Fold('fold', r['mode'], r['reflect'], r['crop'], r['overlap'])
    assert k == 'unstage', k
    return Unstage('unstage', r['swap'], int(r['R1'] < r['R']), int(r['taps'] > 1))


def keys_of(d):
    """{key: record} of one plan description."""
    out = collections.OrderedDict()
    for r in d['layout']:
        out.setdefault(_key(r), r)
    live = [c for c in d['convs'] if c['grad']]          # the backward units, one per live conv, in graph order
    for c, u in zip(live, d.get('backward', [])):
        if u['mode'] == 0:
            out.setdefault(SimtDgrad('simt_dgrad', tuple(c['k']), c['stride'], c['transposed'], u['simt'].split(':')[0]), u)
    return out


@functools.lru_cache(maxsize=None)
def product_keys():
    """{key: where} over every plan of the inventory."""
    return C.first_where((k, '%s: %s' % (s.tag, r['kind'] if 'kind' in r else 'backward unit %d' % r['gop']))
                         for s in PP.plans() for k, r in keys_of(PP.describe(s)).items())


def checked(spec, key):
    """Whether the GPU test of `spec` holds the launch path `key` to bit equality: a case family counts only the kernels its
    test decodes (the integer conv units: the fold, the dgrad packing, the unstage and the SIMT data gradient)."""
    import test_gpu_layout as GL
    families = {GL.Imports: (Import, Export), GL.Corr: (Import, Export), GL.Cat: (Copy, Export), GL.Pack: (Pack,),
                GL.Grad: (GradLayout,), GL.Int: (Fold, Unstage, Pack, SimtDgrad)}
    if isinstance(spec, GL.Int) and isinstance(key, Pack):
        return bool(key.dgrad)
    return isinstance(key, families[type(spec)])


@functools.lru_cache(maxsize=None)
def case_keys():
    """{case id: keys} over the GPU cases, described from the same builders the GPU test runs (modules on the CPU)."""
    import test_gpu_layout as GL
    return {name: {k for k in keys_of(PP.describe(PP.PlanSpec('case', name, functools.partial(GL.build, spec=spec, device='cpu'),
                                                              GL.precision(spec), GL.is_train(spec)))) if checked(spec, k)}
            for name, spec in GL.CASES}


_NARROW = 'export of a ragged channel tile from a buffer at most 128 pixels wide: the products export ragged tiles only from wider ' \
          'buffers'
_WINDOW = 'gradient of a caller channel window: no product reads a training input through a window'
UNREACHED = {
    Export('export', 0, 0, 1, 0): _NARROW,
    Export('export', 1, 0, 1, 0): _NARROW,
    GradLayout('grad_export', 1, 1, 1, 1): _WINDOW,
    GradLayout('grad_export', 0, 1, 1, 1): _WINDOW,
    GradLayout('grad_import', 0, 0, 1, 1): 'scalar gradient import (C < 8): the products\' training plans export only wide values',
    GradLayout('grad_import', 0, 0, 0, 1): 'scalar gradient import (C < 8): as above',
    GradLayout('grad_import', 1, 0, 0, 1): 'tiled gradient import of a ragged channel tile: every product training export is 32k wide',
    GradLayout('grad_import', 1, 0, 1, 1): 'tiled gradient import of a ragged channel tile: as above',
    GradLayout('grad_export', 1, 0, 1, 0): 'tiled gradient export with HW % 32 != 0: the products\' training inputs are 32-pixel multiples',
    Fold('fold', 1, 1, 0, 1): 'reflect halo so deep that both mirrors reach one pixel: no product conv runs on so small an input',
    SimtDgrad('simt_dgrad', (3, 3), 2, 0, 'stride-2 conv behind a reflect halo'):
        'no product has a stride-2 conv behind ReflectionPad2d; the tensor-core backward would crop its mirrored halo',
    SimtDgrad('simt_dgrad', (7, 7), 1, 0, 'bf16 plan'): 'fast-mode training: the products train precise plans only',
    SimtDgrad('simt_dgrad', (3, 3), 2, 0, 'bf16 plan'): 'fast-mode training: as above',
    SimtDgrad('simt_dgrad', (4, 4), 2, 0, 'bf16 plan'): 'fast-mode training: as above',
    SimtDgrad('simt_dgrad', (3, 3), 2, 1, 'bf16 plan'): 'fast-mode training: as above',
}


def test_every_product_layout_key_has_a_gpu_case():
    C.assert_reached('layout launch paths of the products', product_keys(), case_keys())


def test_unreached_keys_are_listed():
    """Every listed path is run by a GPU case and reached by no product; every case key is a product key or listed."""
    C.assert_unreached_listed(product_keys(), case_keys(), UNREACHED)


def test_every_gpu_case_is_needed():
    """Each case reaches a key no other case reaches: a product key or a listed unreached one."""
    import test_gpu_layout as GL
    C.assert_needed([name for name, _ in GL.CASES], [({**product_keys(), **UNREACHED}, case_keys())])


def test_census_is_not_vacuous():
    keys = product_keys()
    of = lambda t: [k for k in keys if isinstance(k, t)]
    imp, pack = of(Import), of(Pack)
    assert {k.CT for k in imp} == {16, 64} and any(k.pad_mode == 2 for k in imp) and any(k.parity for k in imp)
    assert any(k.skip_lo for k in imp) and any(k.act == 2 for k in imp)
    assert {k.TC for k in pack} >= {0, 4, 32} and any(k.dgrad and k.w2 for k in pack) and any(k.headkx for k in pack)
    assert any(k.transposed for k in pack)
    grad = of(GradLayout)
    assert {k.tiled for k in grad} == {0, 1}
    assert any(k.reflect for k in of(Fold)) and any(k.swap for k in of(Unstage))
