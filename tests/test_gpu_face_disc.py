"""The pose demo's face discriminator on the GPU (--add_face_disc): the face_region kernel against the oracle's fp32 predicate,
Vid2VidModelD.forward(0, ...) against the reference's stored losses and the oracle, and pose training steps (label_nc 0,
input_nc 6, with and without no_first_img and openpose_only) against the oracle chain of tests/test_gpu_train_step.py: losses
and gradients with its flip-tolerant criterion and thresholds."""
import pytest
import torch

from oracle import face_disc_oracle as FD
from oracle import flownet2_oracle as FO
from oracle import generator_oracle as GO
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import ops
from vid2vid_b200.model_d import Vid2VidModelD
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.trainer import Trainer
from vid2vid_b200.utils import det_fill_, make_opt

pytestmark = pytest.mark.gpu
F32 = FD.F32


# ------------------------------------------------------------------------------------------------ face_region
def _check_region(x, openpose_only=False):
    ours = ops.face_region(x.cuda(), openpose_only).get()
    assert ours == FD.face_box(x, openpose_only), (tuple(x.shape), openpose_only, ours, FD.face_box(x, openpose_only))
    return ours


def _background(N, H, W, g, C=6):
    """Maps in which no pixel satisfies either predicate."""
    x = torch.rand(N, C, H, W, generator=g) * 2 - 1
    x[:, 2] = x[:, 2] * 0.9 - 0.1
    x[:, 1] = x[:, 1] * 0.99 + 0.01
    return x


def _paint(x, m, openpose_only):
    """Make the pixels of mask m (N, H, W) face pixels of the selected predicate."""
    if openpose_only:
        x[:, 0][m], x[:, 1][m], x[:, 2][m] = 0.2, -0.995, -0.6
    else:
        x[:, 2][m] = 0.95
    return x


@pytest.mark.parametrize('openpose_only', [False, True])
def test_face_region_random_masks(openpose_only):
    g = torch.Generator().manual_seed(11 + openpose_only)
    for (N, H, W), p in [((1, 37, 53), 0.3), ((3, 64, 128), 0.01), ((2, 257, 300), 1e-4), ((4, 16, 16), 0.05), ((2, 512, 512), 2e-6),
                         ((2, 1, 1000), 0.002), ((1, 1000, 1), 0.002), ((8, 96, 128), 1e-5)]:
        x = _background(N, H, W, g)
        m = torch.rand(N, H, W, generator=g) < p
        _check_region(_paint(x, m, openpose_only), openpose_only)


def test_face_region_single_pixel_last_image_and_borders():
    g = torch.Generator().manual_seed(3)
    N, H, W = 3, 70, 90
    for openpose_only in (False, True):
        for n, y, x in [(0, 33, 41), (2, 5, 7), (1, 0, 0), (2, H - 1, W - 1), (0, 0, W - 1), (1, H - 1, 0)]:
            m = torch.zeros(N, H, W, dtype=torch.bool)
            m[n, y, x] = True
            assert _check_region(_paint(_background(N, H, W, g), m, openpose_only), openpose_only) == (y, y, x, x)
        # a face only in the last image of the batch
        m = torch.zeros(N, H, W, dtype=torch.bool)
        m[N - 1, 20:31, 40:52] = True
        assert _check_region(_paint(_background(N, H, W, g), m, openpose_only), openpose_only) == (20, 30, 40, 51)
        # every border: whole first / last row and column, in different images
        for sl in [(0, 0, slice(None)), (1, H - 1, slice(None)), (2, slice(None), 0), (0, slice(None), W - 1)]:
            m = torch.zeros(N, H, W, dtype=torch.bool)
            m[sl] = True
            _check_region(_paint(_background(N, H, W, g), m, openpose_only), openpose_only)
        # no face
        assert _check_region(_background(N, H, W, g), openpose_only) is None


def test_face_region_fp32_boundaries():
    """Pixels exactly on the fp32-rounded constants: a comparison in double would accept c0 == float32(0.21) and
    c1 == float32(-0.99); the reference (fp32 tensor vs Python float) does not, and neither must the kernel."""
    g = torch.Generator().manual_seed(7)
    N, H, W = 2, 40, 60
    cases = [
        (False, (2,), (F32(0.9),), None),                        # c2 > 0.9: float32(0.9) < 0.9, not a face
        (False, (2,), (float(torch.nextafter(torch.tensor(F32(0.9)), torch.tensor(2.0))),), (5, 5, 6, 6)),
        (True, (0, 1, 2), (F32(0.21), -1.0, -0.6), None),
        (True, (0, 1, 2), (F32(0.19), -1.0, -0.6), None),
        (True, (0, 1, 2), (0.2, F32(-0.99), -0.6), None),
        (True, (0, 1, 2), (0.2, -1.0, F32(-0.61)), None),
        (True, (0, 1, 2), (0.2, -1.0, F32(-0.59)), None),
        (True, (0, 1, 2), (float(torch.nextafter(torch.tensor(F32(0.21)), torch.tensor(0.0))), -1.0, -0.6), (5, 5, 6, 6)),
        (True, (0, 1, 2), (0.2, float(torch.nextafter(torch.tensor(F32(-0.99)), torch.tensor(-2.0))), -0.6), (5, 5, 6, 6)),
    ]
    for openpose_only, chans, vals, want in cases:
        x = _background(N, H, W, g)
        for c, v in zip(chans, vals):
            x[1, c, 5, 6] = v
        assert _check_region(x, openpose_only) == want, (openpose_only, vals)
    # both predicates' boundary pixels together, around a real face: the box is the face's
    x = FD.case_inputs('openpose')[3]
    assert _check_region(x, True) == FD.face_box(x, True) != FD.face_box(x.double(), True)


def test_face_region_needs_three_channels():
    with pytest.raises(RuntimeError, match='channels'):
        ops.face_region(torch.zeros(1, 2, 8, 8, device='cuda'))


# ------------------------------------------------------------------------------------------------ Vid2VidModelD.forward
def _model_d(name, flag=True):
    opt = FD.case_opt(name)
    opt.add_face_disc, opt.n_scales_temporal = flag, 1
    D = Vid2VidModelD().initialize(opt)
    det_fill_(D.netD, seed=FD.D_SEED)
    if flag:
        det_fill_(D.netD_f, seed=FD.D_F_SEED)
    return opt, D


def _gold():
    import numpy as np
    import os
    with np.load(os.path.join(os.path.dirname(__file__), 'golden', 'face_disc.npz')) as z:
        return {k: z[k] for k in z.files}


def _close(a, b, rel=2e-3):
    a, b = a.detach().cpu().double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    return (a - b).abs().max().item() <= rel * max(1.0, b.abs().max().item())


@pytest.mark.parametrize('name', sorted(FD.CASES))
def test_forward_losses_match_reference_and_oracle(name):
    gold = _gold()
    opt, D = _model_d(name)
    inputs = FD.case_inputs(name)
    cu = [t.cuda() if t is not None else None for t in inputs]
    sd_D = {k: v.detach().cpu().clone() for k, v in D.netD.state_dict().items()}
    sd_f = {k: v.detach().cpu().clone() for k, v in D.netD_f.state_dict().items()}
    stats = FD.running_stats(sd_f)
    with torch.no_grad():
        ref = FD.face_disc_losses(sd_D, sd_f, stats, inputs, opt)
    ours = D(0, cu)
    torch.cuda.synchronize()
    assert len(ours) == 13
    for n, o, r in zip(D.loss_names, ours, ref):
        print('%-13s ours %.6f oracle %.6f' % (n, float(o.flatten()[0]), float(r.flatten()[0])))
        assert _close(o, gold['%s/loss/%s' % (name, n)]), (name, n)
        assert _close(o, r), (name, n)
    window = D.get_face_region(cu[3])
    want = [None] * 4 if name == 'none' else gold['%s/window' % name].tolist()
    assert list(window) == want
    after = D.netD_f.state_dict()
    if name == 'none':
        assert all(float(o.abs().max()) == 0.0 for o in ours[9:])
        assert all(torch.equal(after[k].cpu(), sd_f[k]) for k in sd_f)            # netD_f never ran
    else:
        for layer, (rm, rv) in stats.items():
            for leaf, v in (('running_mean', rm), ('running_var', rv)):
                k = layer + '.' + leaf
                assert _close(after[k], gold['%s/stats/%s' % (name, k)]) and _close(after[k], v), k

    # the nine losses without the face discriminator: bit-identical on the same weights and inputs
    _, D_off = _model_d(name, flag=False)
    off = D_off(0, cu)
    assert len(off) == 9
    for n, a, b in zip(D_off.loss_names, ours[:9], off):
        assert torch.equal(a, b), n


# ------------------------------------------------------------------------------------------------ pose training step
def _setup(openpose_only, H=128, W=128, seed=3, no_first_img=True):
    opt = make_opt(label_nc=0, input_nc=6, use_instance=False, fg=False, n_scales_spatial=2, ngf=16, n_downsample_G=2, n_blocks=4,
                   n_blocks_local=2, num_D=3, ndf=16, n_scales_temporal=2, isTrain=True, no_vgg=True, gpu_ids=[0], n_frames_total=12,
                   no_first_img=no_first_img, add_face_disc=True, openpose_only=openpose_only, fineSize=256, dataroot='datasets/pose',
                   dataset_mode='pose')
    G = Vid2VidModelG().initialize(opt)
    D = Vid2VidModelD().initialize(opt)
    for s in range(2):
        det_fill_(getattr(G, 'netG%d' % s), seed=seed + s)
    det_fill_(D.netD, seed=seed + 10)
    det_fill_(D.netD_f, seed=seed + 30)
    for s in range(2):
        det_fill_(getattr(D, 'netD_T%d' % s), seed=seed + 20 + s)
    flow = FN.FlowNet().initialize(opt)
    A, B = FD.pose_clip(8, H, W, seed, blob_rows=(40, 58), blob_cols=(50, 70), openpose_only=openpose_only)
    return opt, G, D, flow, A, B


def _biases_before_norm(module, prefix=''):
    """Names of the conv / transposed-conv biases that feed a BatchNorm directly.  Their exact gradient is zero (the norm
    subtracts the batch mean): ours must be exactly zero, and the fp32 oracle's value is rounding noise, which with dense
    real-valued pose inputs can exceed the 1e-5-of-the-largest-gradient cut tests/test_gpu_train_step.py uses to recognise it."""
    names = set()
    for mname, m in module.named_modules():
        if isinstance(m, torch.nn.Sequential):
            kids = list(m.named_children())
            for (n, a), (_, b) in zip(kids, kids[1:]):
                if isinstance(a, (torch.nn.Conv2d, torch.nn.ConvTranspose2d)) and a.bias is not None and isinstance(b, torch.nn.BatchNorm2d):
                    names.add(prefix + (mname + '.' if mname else '') + n + '.bias')
    return names


def _check_grads(ours, ref, max_rel, med_rel, what, zero):
    """tests/test_gpu_train_step.py's criterion: every tensor within max_rel relative L2, the median within med_rel.  The biases
    in `zero` (exact gradient zero) must be exactly zero here and are not compared with the oracle's rounding noise."""
    rels = []
    for k, r in ref.items():
        if k in zero:
            assert ours[k].abs().max().item() == 0, (what, k)
            continue
        if r.abs().max().item() < 1e-9:
            continue
        rel = ((ours[k] - r).norm() / r.norm()).item()
        rels.append(rel)
        assert rel <= max_rel, (what, k, rel)
    rels.sort()
    print('%s gradients: %d tensors, median rel L2 %.2e, max %.2e' % (what, len(rels), rels[len(rels) // 2], rels[-1]))
    assert rels[len(rels) // 2] <= med_rel, what


def _pose_step(openpose_only, no_first_img):
    """The first pose training step (Trainer.losses, then loss_G and loss_D backward as Trainer.step does) and the oracle chain
    of tests/test_gpu_train_step.py with the face terms.  Returns ours and the oracle's losses and gradients."""
    opt, G, D, flow, A, B = _setup(openpose_only, no_first_img=no_first_img)
    tr = Trainer(opt, G, D, flow, world=1)
    tG = opt.n_frames_G
    a, b = A[:, :tG].cuda(), B[:, :tG].cuda()
    loss_G, loss_D, loss_D_T, ld, ldT = tr.losses(a, b, a)
    assert not loss_D_T
    tr.grads.zero()
    loss_G.backward()
    ours = {'G': {k: p.grad.detach().cpu().double().clone() for s in range(2) for k, p in
                  (('%d.%s' % (s, n), q) for n, q in getattr(G, 'netG%d' % s).named_parameters())}}
    tr.grads.zero(1)
    loss_D.backward()
    ours['D'] = {n: p.grad.detach().cpu().double().clone() for n, p in D.netD.named_parameters()}
    ours['D_f'] = {n: p.grad.detach().cpu().double().clone() for n, p in D.netD_f.named_parameters()}

    leaf = lambda net: {k: v.detach().cpu().clone().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
                        for k, v in net.state_dict().items()}
    sds = [leaf(getattr(G, 'netG%d' % s)) for s in range(2)]
    sdD, sdDf = leaf(D.netD), leaf(D.netD_f)
    stats = FD.running_stats({k: v.detach() for k, v in sdDf.items()})
    sdF = {k: v.detach().cpu() for k, v in flow.flowNet.state_dict().items()}
    orc = GO.ModelGOracle(opt, sds)
    fake_B, raws, flows, weights, real_A, real_Bp, _ = orc.train_forward(A[:, :tG], B[:, :tG], A[:, :tG], None, n_frames_load=1)
    real_B_prev, real_B = real_Bp[:, :-1], real_Bp[:, 1:]
    with torch.no_grad():
        flow_ref, conf_ref = FO.flow_and_conf(sdF, real_B[:, 0], real_B_prev[:, 0])
    m = lambda t: t.reshape(-1, *t.shape[2:]) if t is not None else None
    assert FD.face_box(m(real_A), openpose_only) is not None
    lo = FD.face_disc_losses(sdD, sdDf, stats, [m(real_B), m(fake_B), m(raws), m(real_A), m(real_B_prev), m(real_B_prev[:, 0:1]),
                                                m(flows), m(weights), flow_ref, conf_ref], opt)
    od = dict(zip(D.loss_names, [torch.mean(x) for x in lo]))
    oG = sum(od[n] for n in ('G_GAN', 'G_GAN_Feat', 'G_VGG', 'G_Warp', 'F_Flow', 'F_Warp', 'W', 'G_f_GAN', 'G_f_GAN_Feat'))
    oD = (od['D_fake'] + od['D_real']) * 0.5 + (od['D_f_fake'] + od['D_f_real']) * 0.5
    oG.backward(retain_graph=True)
    ref = {'G': {'%d.%s' % (s, k): v.grad.double().clone() for s in range(2) for k, v in sds[s].items() if v.grad is not None}}
    for v in list(sdD.values()) + list(sdDf.values()):
        v.grad = None
    oD.backward()
    ref['D'] = {k: v.grad.double() for k, v in sdD.items() if v.grad is not None}
    ref['D_f'] = {k: v.grad.double() for k, v in sdDf.items() if v.grad is not None}
    zero = {'G': set().union(*(_biases_before_norm(getattr(G, 'netG%d' % s), '%d.' % s) for s in range(2))),
            'D': _biases_before_norm(D.netD), 'D_f': _biases_before_norm(D.netD_f)}
    return ld, od, D.loss_names, ours, ref, zero


def _check_losses(ld, od, names):
    for n in names:
        o, r = float(ld[n]), float(od[n])
        print('%-13s ours %.6f oracle %.6f' % (n, o, r))
        assert abs(o - r) <= 2e-3 * max(1.0, abs(r)), n
    assert float(od['D_f_real']) > 0 and float(od['G_f_GAN']) > 0


@pytest.mark.parametrize('openpose_only', [False, True])
def test_first_pose_training_step_vs_oracle(openpose_only):
    """Dense pose inputs with the real first frames given (no --no_first_img): losses, and the G, D and D_f gradients under
    tests/test_gpu_train_step.py's criterion and thresholds -- the generator gradients include the face terms' path through
    netD_f's input gradient and the crop."""
    ld, od, names, ours, ref, zero = _pose_step(openpose_only, no_first_img=False)
    _check_losses(ld, od, names)
    _check_grads(ours['G'], ref['G'], 0.15, 3e-2, 'G', zero['G'])
    _check_grads(ours['D'], ref['D'], 0.1, 2e-2, 'D', zero['D'])
    _check_grads(ours['D_f'], ref['D_f'], 0.1, 2e-2, 'D_f', zero['D_f'])


@pytest.mark.parametrize('openpose_only', [False, True])
def test_first_pose_training_step_no_first_img_vs_oracle(openpose_only):
    """--no_first_img, as the pose recipes train: losses and the D and D_f gradients.  The generator gradients are checked in
    the xfail test below."""
    ld, od, names, ours, ref, zero = _pose_step(openpose_only, no_first_img=True)
    _check_losses(ld, od, names)
    _check_grads(ours['D'], ref['D'], 0.1, 2e-2, 'D', zero['D'])
    _check_grads(ours['D_f'], ref['D_f'], 0.1, 2e-2, 'D_f', zero['D_f'])


@pytest.mark.xfail(strict=True, reason='known engine defect (DESIGN.md section 6): with --no_first_img the previous frames of the '
                   'first step are zeros, so the first convs of the generators\' image branch see spatially constant inputs and '
                   'their BatchNorm variance is far below mean^2.  Our gradients differ from an fp64 oracle by a median 7 % (the fp32 '
                   'oracle by 0.6 %); with the SIMT conv path they agree within the thresholds, so the error lies in the wgmma conv '
                   'path, most likely its one-pass fixed-point (sum, sumsq) norm statistics')
def test_first_pose_training_step_no_first_img_generator_gradients():
    ld, od, names, ours, ref, zero = _pose_step(False, no_first_img=True)
    _check_grads(ours['G'], ref['G'], 0.15, 3e-2, 'G', zero['G'])


def test_pose_training_steps_update_face_discriminator():
    opt, G, D, flow, A, B = _setup(False, seed=5)
    tr = Trainer(opt, G, D, flow, world=1)
    assert [id(p) for p in tr.grads.groups[1]] == [id(p) for grp in D.optimizer_D.param_groups for p in grp['params']]
    assert len(tr.grads.groups[1]) == len(list(D.netD.parameters())) + len(list(D.netD_f.parameters()))
    tG = opt.n_frames_G
    before = {n: p.detach().clone() for n, p in D.netD_f.named_parameters()}
    for i in range(6):
        a, b = A[:, i:i + tG].cuda(), B[:, i:i + tG].cuda()
        ld, ldT = tr.step(a, b, a)
        assert len(ld) == 13 and all(torch.isfinite(torch.tensor(v)) for v in ld.values()), ld
        assert ld['D_f_real'] > 0
        for d in ldT:
            assert all(torch.isfinite(torch.tensor(v)) for v in d.values()), d
    moved = max((p.detach() - before[n]).abs().max().item() for n, p in D.netD_f.named_parameters())
    assert moved > 0
