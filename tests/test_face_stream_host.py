"""Host-side checks of the edge2face and pose2body streams, no GPU needed: inference_stream's argument errors for dense and
face streams, and a census of the plans those streams add.  The batch-B Encoder and Global_with_z of batched face first
frames are per-sample plans that must lower every conv with the configuration of the batch-1 plan (that configuration fixes
each pixel's accumulation order, which is what keeps every clip bit-identical to its own run), and every conv configuration
the plans of tools/time_face_stream.py lower must be reached by a GPU parity case against fp64: one of tests/test_conv_census.py's
or one of tests/test_gpu_face_stream.CONV_CASES, each of which must reach a configuration no other case reaches."""
import types

import pytest
import torch

import census as C
import product_plans as PP
import test_conv_census as TCC
from product_plans import h100_sxm  # noqa: F401  (autouse: the census describes a 132-SM device)
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.utils import make_opt

# the launch quantities that scale with the number of images, and the epilogue placement chosen from them
PER_LAUNCH = ('units', 'm_total', 'ctas', 'async_epi')


# ----------------------------------------------------------------------------- argument checks
def _model(face=True, **o):
    """A stand-in model with no stream running: _stream_frames reads only the options and the stream state."""
    kw = dict(label_nc=0, input_nc=15, dataset_mode='face', use_single_G=True) if face else dict(label_nc=0, input_nc=6,
                                                                                                    no_first_img=True)
    kw.update(o)
    opt = make_opt(gpu_ids=[], **kw)
    return types.SimpleNamespace(opt=opt, use_single_G=opt.use_single_G, _win_A=None, _win_n=0, _DT=Vid2VidModelG._DT)


def _check(m, label, inst=None, real=None):
    return Vid2VidModelG._stream_frames(m, label, inst, real)


def test_dense_frames_and_their_channel_count():
    pose = _model(face=False)
    assert _check(pose, torch.zeros(6, 16, 8)) == (1, 16, 8, False, True)
    assert _check(pose, torch.zeros(2, 6, 16, 8)) == (2, 16, 8, True, True)
    for bad in (torch.zeros(5, 16, 8), torch.zeros(2, 7, 16, 8), torch.zeros(16, 8), torch.zeros(6, 16, 8, dtype=torch.float64)):
        with pytest.raises(ValueError, match=r'dense \(6, H, W\) or \(B, 6, H, W\) float32'):
            _check(pose, bad)
    with pytest.raises(ValueError, match='face streams only'):
        _check(pose, torch.zeros(6, 16, 8), real=torch.zeros(3, 16, 8))


def test_face_fill_needs_the_real_frame_and_the_part_map():
    face = _model()
    x, real, part = torch.zeros(15, 16, 8), torch.zeros(3, 16, 8), torch.zeros(16, 8, dtype=torch.uint8)
    assert _check(face, x, part, real) == (1, 16, 8, False, True)
    with pytest.raises(ValueError, match='needs real_frame on each of its first 2 calls'):
        _check(face, x, part, None)
    with pytest.raises(ValueError, match=r'needs inst_frame \(the part map\) on each'):
        _check(face, x, None, real)
    with pytest.raises(ValueError, match=r'needs real_frame and inst_frame \(the part map\)'):
        _check(face, x)
    # the window still filling (one frame in): still required; once tG - 1 frames are in: ignored
    face._win_A, face._win_n = torch.zeros(1, 3, 15, 16, 8), 1
    with pytest.raises(ValueError, match='needs real_frame'):
        _check(face, x, part, None)
    face._win_n = 2
    assert _check(face, x) == (1, 16, 8, False, False)
    # other frame sizes start a new window, which fills again
    with pytest.raises(ValueError, match='needs real_frame'):
        _check(face, torch.zeros(15, 32, 8))


def test_face_frame_shapes_must_match():
    face = _model()
    x, real, part = torch.zeros(3, 15, 16, 8), torch.zeros(3, 3, 16, 8), torch.zeros(3, 16, 8, dtype=torch.int32)
    assert _check(face, x, part, real) == (3, 16, 8, True, True)
    for bad_real in (torch.zeros(3, 16, 8), torch.zeros(2, 3, 16, 8), torch.zeros(3, 3, 16, 16)):
        with pytest.raises(ValueError, match='real_frame .* does not match label_frame'):
            _check(face, x, part, bad_real)
    for bad_part in (torch.zeros(16, 8), torch.zeros(3, 1, 16, 8), torch.zeros(3, 8, 16)):
        with pytest.raises(ValueError, match='inst_frame .* does not match label_frame'):
            _check(face, x, bad_part, real)
    with pytest.raises(TypeError, match='inst_frame uint8, int32 or float32'):
        _check(face, x, part.long(), real)
    with pytest.raises(TypeError, match='real_frame must be floating point'):
        _check(face, x, part, real.to(torch.uint8))


def test_clip_count_is_fixed_for_a_stream():
    for m, frame in ((_model(face=False), torch.zeros(6, 16, 8)), (_model(), torch.zeros(15, 16, 8))):
        m._win_A, m._win_n = torch.zeros(3, 3, m.opt.input_nc, 16, 8), 5
        with pytest.raises(ValueError, match='started with 3 clip'):
            _check(m, frame)
        with pytest.raises(ValueError, match='started with 3 clip'):
            _check(m, frame.expand(2, *frame.shape))


# ----------------------------------------------------------------------------- conv census
FACE_BS = (2, 4)


def _face_nets():
    """(netE, netG_i) of the edge2face demo (Vid2VidModelG.load_single_G) and the frame size of tools/time_face_stream.py."""
    import time_face_stream as TFS
    netG, netE = PP._single_G(**TFS.WORKLOADS['face_512']['opt'])
    return (('netE', netE), ('netG_i', netG)), TFS.WORKLOADS['face_512']['H'], TFS.WORKLOADS['face_512']['W']


@pytest.mark.parametrize('mode', PP.MODES)
def test_batched_first_frame_plans_keep_the_batch1_configuration(mode):
    nets, H, W = _face_nets()
    for name, net in nets:
        one = PP.describe(PP.PlanSpec('face_stream', '%s B=1' % name, PP._net(net, 1, H, W), mode))['convs']
        for b in FACE_BS:
            d = PP.describe(PP.PlanSpec('face_stream', '%s B=%d' % (name, b), PP._net(net, b, H, W), mode, sample_stats=True))
            assert d['sample_stats'] == 1 and len(d['convs']) == len(one)
            for a, c in zip(one, d['convs']):
                assert {k: v for k, v in a.items() if k not in PER_LAUNCH} == {k: v for k, v in c.items() if k not in PER_LAUNCH}
                assert c['m_total'] == b * a['m_total'] and c['units'] == b * a['units']


def _stream_plans():
    """The PlanSpecs of tools/time_face_stream.py in both arithmetic modes: the face first-frame networks and generator at
    every B (per-sample plans for B > 1) and the pose generator scales."""
    import time_face_stream as TFS
    out = []
    nets, H, W = _face_nets()
    for wl, w in TFS.WORKLOADS.items():
        opt = make_opt(**dict(w['opt'], gpu_ids=[]))
        gens = [('G%d' % s, net, h, w_) for s, (net, h, w_) in enumerate(PP.scales(opt, w['H'], w['W']))]
        if wl == 'face_512':
            gens += [(name, net, H, W) for name, net in nets]
        out += [PP.PlanSpec('face_stream', '%s %s %s B=%d' % (wl, name, mode, b), PP._net(net, b, h, w_), mode, sample_stats=b > 1)
                for name, net, h, w_ in gens for mode in PP.MODES for b in w['bs']]
    return out


def _cases():
    """{case id: keys} of tests/test_conv_census.py's forward cases and of this product's own cases."""
    import test_gpu_face_stream as TG
    cases = {}
    for level in ('bench', 'multiclip', 'product'):
        cases.update(TCC.levels()[level][1])
    own = [TCC._case('test_gpu_face_stream::' + n, b, s, m, sample_stats=True) for n, b, s, m in TG.CONV_CASES]
    cases.update({name: set(TCC.forward(specs)) for name, specs in own})
    return cases, [name for name, _ in own]


def test_every_face_stream_configuration_has_a_case():
    keys = TCC.forward(_stream_plans())
    cases, own = _cases()
    assert len(keys) >= 30, len(keys)
    C.assert_reached('face / pose stream configurations', keys, cases)
    C.assert_needed(own, [(keys, cases)])
