"""Several clips at once on one GPU: a per-sample-statistics plan (v2v_plan_set_sample_stats, _Planned.sample_stats) over B
independent clips must give every clip exactly what its own batch-1 run gives, bit for bit, and leave the running
statistics as B batch-1 forwards in clip order would.  The clips get different inputs, so any mixing of statistics shows."""
import copy

import pytest
import torch
import torch.nn as nn

import bf16_emul as E
import cases as C
import test_gpu_conv as TC
from vid2vid_b200 import networks as NW
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.utils import det_fill_, make_opt, synth_label_sequence

pytestmark = pytest.mark.gpu

B = 3
MODES = ('precise', 'fast')
# fg on / fg off / no_flow CompositeGenerator, and the CompositeLocalGenerator
GEN_CASES = ('g0_small', 'g0_nofg_nd2', 'g0_noflow', 'gl_small_s1')


def _clip_inputs(net, c, k):
    inp, prev, mask = C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed'] + 100 * k)
    coarse = (None, None, None)
    if c['kind'] == 'compositeLocal':
        g = torch.Generator().manual_seed(c['seed'] + 100 * k + 5)
        h2, w2 = c['h'] // 2, c['w'] // 2
        c2 = net.model_down_seg[4].out_channels
        cg = net.indv_down[4].out_channels if net.use_fg_model else None
        coarse = (torch.randn(1, c2, h2, w2, generator=g), torch.randn(1, c2, h2, w2, generator=g),
                  torch.randn(1, cg, h2, w2, generator=g) if cg else None)
    return [t.cuda() if t is not None else None for t in (inp, prev, mask) + coarse]


def _forward(net, x):
    return net(x[0], x[1], x[2], x[3], x[4], x[5], False)


def _running(net):
    return {k: v.clone() for k, v in net.state_dict().items() if 'running' in k or 'num_batches' in k}


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', GEN_CASES)
def test_per_sample_forward_equals_batch1_forwards(case, mode):
    c = C.CASES[case]
    net = det_fill_(C.build_module(c), seed=c['seed']).cuda()
    net.precision = mode
    ref = copy.deepcopy(net)
    clips = [_clip_inputs(net, c, k) for k in range(B)]
    batched = [torch.cat([x[i] for x in clips]) if clips[0][i] is not None else None for i in range(6)]
    net.sample_stats = True
    with torch.no_grad():
        outs = _forward(net, batched)
        singles = [_forward(ref, x) for x in clips]
    torch.cuda.synchronize()
    n_out = 0
    for name, o, *s in zip(C.GEN_OUT_NAMES, outs, *singles):
        assert (o is None) == (s[0] is None), name
        if o is None:
            continue
        n_out += 1
        for k in range(B):
            assert torch.equal(o[k:k + 1], s[k]), '%s of clip %d differs from its batch-1 forward (max |d| %.3g)' % (
                name, k, (o[k:k + 1] - s[k]).abs().max().item())
    assert n_out >= 4
    # the running statistics: B momentum updates in clip order, each as a batch-1 plan makes it
    rn, rr = _running(net), _running(ref)
    assert rn
    for k in rn:
        assert torch.equal(rn[k], rr[k]), k


# --------------------------------------------------------------------------------------- conv configurations vs fp64
# Kernel configurations that the plans of tools/time_multiclip.py lower and no other GPU parity case reaches, each at a small
# shape that selects it on 132 SMs, run as a per-sample plan over N images and checked against the same layers evaluated
# image by image in fp64 (precise) or bf16-emulated fp32 (fast) at tests/test_gpu_conv.py's tolerances.
# tests/test_conv_census.py fails when a configuration goes uncovered or a case stops being needed.
# name, layer list builder, input shape (N, C, H, W), modes
BN = NW.get_norm_layer('batch')
CONV_CASES = [
    # 1024->1024 3x3 at 32x48 per image: 2-D patch, 32-channel K blocks; three images give the epilogue warpgroup its units
    ('c3_1024_p2d_kc32_async', lambda: [nn.ReflectionPad2d(1), nn.Conv2d(1024, 1024, 3), BN(1024), nn.ReLU(True)],
     (3, 1024, 32, 48), ['fast']),
    # the pose model's fused 18-channel 7x7 stems (model_down_seg + indv_down: 128 + 64, and 64 + 32 at the finer scale)
    ('stem_18_192_async', lambda: NW._stem(18, 192, BN), (3, 18, 128, 128), TC.MODES),
    ('stem_18_96_ring2_tb4_async', lambda: NW._stem(18, 96, BN), (3, 18, 256, 128), ['precise']),
    # its 6-channel previous-frame stem: 16-channel K blocks with a 128-wide N tile, on one image and on three
    ('stem_6_128_kc16', lambda: NW._stem(6, 128, BN), (1, 6, 256, 128), TC.MODES),
    ('stem_6_128_kc16_async', lambda: NW._stem(6, 128, BN), (3, 6, 256, 128), ['precise']),
    ('deconv_128_64_async', lambda: NW._up(128, 64, BN), (3, 128, 64, 64), ['fast']),
]


def _per_sample_runner(build, mode, seed=1):
    r = det_fill_(NW.SequentialRunner(build()), seed=seed).cuda()
    r.precision = mode
    r.sample_stats = True
    return r


@pytest.mark.parametrize('name,build,shape,mode', [(c[0], c[1], c[2], m) for c in CONV_CASES for m in c[3]],
                         ids=['%s-%s' % (c[0], m) for c in CONV_CASES for m in c[3]])
def test_per_sample_conv_configuration_vs_fp64(name, build, shape, mode):
    runner = _per_sample_runner(build, mode)
    x = TC._x(*shape).cuda()
    E.ROUND[0] = (mode == 'fast')
    try:
        with torch.no_grad():
            out = runner(x)
            out2 = runner(x)           # second call replays the CUDA graph
            xr = E.r16(x)
            ref = torch.cat([E.run_units(list(runner.seq), xr[k:k + 1]) for k in range(shape[0])])
    finally:
        E.ROUND[0] = True
    assert torch.equal(out, out2), 'graph replay differs from eager run'
    TC._check(out, ref, name, mode=mode)


# ------------------------------------------------------------------------------------------------- Vid2VidModelG
N_FRAMES = 8


def _street(use_real_img=False):
    c = C.CASES['infer_s3']
    opt = C.inference_opt(c)
    opt.gpu_ids = [0]
    opt.use_real_img = use_real_img
    m = Vid2VidModelG()
    m.use_single_G = opt.use_single_G = False          # build without checkpoints, then attach the seeded first-frame net
    m.initialize(opt)
    opt.use_single_G = m.use_single_G = True
    m.netG_i = det_fill_(NW.define_G(c['label_nc'], 3, 0, 16, 'global', 2, 'instance', 0, [], opt), seed=c['seed'] + 100).cuda()
    for s in range(c['n_scales']):
        det_fill_(getattr(m, 'netG%d' % s), seed=c['seed'] + s)
        C.condition_flow_heads(getattr(m, 'netG%d' % s), c['flow_weight_scale'])
    tG = opt.n_frames_G

    def clip(k):
        seq = synth_label_sequence(N_FRAMES + tG - 1, c['h'], c['w'], label_nc=c['label_nc'], block=8, seed=c['seed'] + 7 * k)
        real = torch.rand(1, N_FRAMES + tG - 1, 3, c['h'], c['w'], generator=torch.Generator().manual_seed(60 + k)) * 2 - 1
        return seq, (real if use_real_img else None), seq
    return m, clip


def _pose():
    opt = make_opt(label_nc=0, input_nc=6, n_scales_spatial=2, no_first_img=True, fg=True, fg_labels=[2], ngf=16, n_blocks=3,
                   n_blocks_local=2, n_downsample_G=2, dataroot='datasets/pose/', gpu_ids=[0])
    m = Vid2VidModelG().initialize(opt)
    for s in range(2):
        det_fill_(getattr(m, 'netG%d' % s), seed=40 + s)
        C.condition_flow_heads(getattr(m, 'netG%d' % s), 0.05)
    H, W = 128, 64

    def clip(k):
        g = torch.Generator().manual_seed(50 + k)
        A = torch.rand(1, N_FRAMES + opt.n_frames_G - 1, 6, H, W, generator=g) * 2 - 1
        A[..., :, :H // 4, :] = 0                  # background rows
        return A, None, None
    return m, clip


def _face():
    from oracle import face_oracle as FO
    opt = FO.face_opt(gpu_ids=[0], synthetic_weights=True)
    m = Vid2VidModelG().initialize(opt)
    seeds = FO.infer_seeds()
    det_fill_(m.netE, seed=seeds['netE'])
    det_fill_(m.netG_i, seed=seeds['netG_i'])
    det_fill_(m.netG0, seed=seeds['netG0'])
    FO.condition(m)
    m.load_face_features(features=FO.synthetic_features())
    H = W = FO.INFER_SIZE
    nF = N_FRAMES + opt.n_frames_G - 1

    def clip(k):
        s = FO.SEED + 20 + 3 * k
        return FO.edge_maps(nF, H, W, s), FO.real_images(nF, H, W, s), FO.part_map(nF, H, W, s)
    return m, clip


def _window(x, t, tG):
    return x[:, t:t + tG] if x is not None else None


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('model', ['street', 'street_use_real_img', 'pose', 'face'])
def test_inference_of_b_clips_equals_each_clip(model, mode):
    NW.set_default_precision(mode)
    try:
        m, clip = {'street': _street, 'street_use_real_img': lambda: _street(True), 'pose': _pose, 'face': _face}[model]()
        tG = m.opt.n_frames_G
        clips = [clip(k) for k in range(B)]
        cat = lambda i: torch.cat([c[i] for c in clips]) if clips[0][i] is not None else None
        both = [cat(i) for i in range(3)]
        batched = []
        for t in range(N_FRAMES):
            fake_B, _ = m.inference(*[_window(x, t, tG) for x in both])
            assert fake_B.shape[0] == B
            batched.append(fake_B.clone())
        # per-sample plans only for the duration of a call: the modules build batch-statistics / training plans afterwards
        assert not any(getattr(m, 'netG%d' % s).sample_stats for s in range(m.n_scales))
        for k in range(B):
            m.reset_stream()
            for t in range(N_FRAMES):
                fake_B, _ = m.inference(*[_window(x, t, tG) for x in clips[k]])
                assert torch.equal(batched[t][k:k + 1], fake_B), 'clip %d frame %d: max |d| %.3g' % (
                    k, t, (batched[t][k:k + 1] - fake_B).abs().max().item())
    finally:
        NW.set_default_precision('precise')


def test_inference_stream_of_b_clips_equals_each_stream():
    m, clip = _street()
    tG = m.opt.n_frames_G
    labels = [clip(k)[0][0, :, 0].to(torch.uint8) for k in range(B)]      # (frames, H, W) uint8 id maps per clip
    H, W = labels[0].shape[-2:]
    n = labels[0].shape[0]
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device='cuda')
    got = []
    for t in range(n):
        r = m.inference_stream(torch.stack([lab[t] for lab in labels]), torch.stack([lab[t] for lab in labels]), out_u8=out)
        assert (r is None) == (t < tG - 1)
        if r is not None:
            got.append(out.clone())
    with pytest.raises(ValueError, match='started with 3 clip'):
        m.inference_stream(labels[0][0], labels[0][0])
    with pytest.raises(NotImplementedError, match='running batch'):
        m.reset_stream(clips=[1])
    one = torch.empty(H, W, 3, dtype=torch.uint8, device='cuda')
    for k in range(B):
        m.reset_stream()
        j = 0
        for t in range(n):
            if m.inference_stream(labels[k][t], labels[k][t], out_u8=one) is not None:
                assert torch.equal(got[j][k], one), 'clip %d step %d' % (k, t)
                j += 1
        assert j == len(got)


def test_inference_refuses_a_different_clip_count():
    m, clip = _street()
    tG = m.opt.n_frames_G
    A = torch.cat([clip(k)[0] for k in range(B)])
    m.inference(A[:, :tG], None, A[:, :tG])
    with pytest.raises(ValueError, match='started with 3 clip'):
        m.inference(A[:2, 1:tG + 1], None, A[:2, 1:tG + 1])
