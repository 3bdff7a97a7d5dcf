"""TEST INFRASTRUCTURE -- not product code (only tests/ and tools/ may import oracle/).

CPU restatement of the pose demo's face discriminator (models/vid2vid_model_D.py:38-40,149-162,215-230,249-256) on top of
losses_oracle.spatial_losses, the seeded pose-like inputs its checks use, and the recipe that pins it against the
unmodified reference.

    face_box(real_A, openpose_only)        the pixel search of get_face_region: (ymin, ymax, xmin, xmax) or None
    face_window(box, h, w, fineSize)       the crop (ys, ye, xs, xe) around it
    face_terms(sd_f, stats_f, ...)         [G_f_GAN, G_f_GAN_Feat, D_f_real, D_f_fake] (compute_loss_D on netD_f, with the
                                           reference's 1 / num_D weighting of netD's tower count); netD_f's batch-norm
                                           running statistics in stats_f advance once per tower call, as in train mode
    face_disc_losses(...)                  the 13 losses of Vid2VidModelD.forward(0, ...) with --add_face_disc

    python -m oracle.face_disc_oracle [OUT_DIR]   # writes face_disc_keys.json and face_disc.npz (default tests/golden/)

The recipe runs the reference's own Vid2VidModelD (add_face_disc=True) and Vid2VidModelG (pose mode) on the CPU through
ref_shim, with det_fill_ weights.  ref_shim's shims are process-wide: run the recipe in its own process.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import generator_oracle as GO                       # noqa: E402
from oracle import losses_oracle as LO                          # noqa: E402
from vid2vid_b200.utils import make_opt, det_fill_              # noqa: E402

SEED = 61
D_SEED, D_F_SEED = 71, 72
FACE_WEIGHT = 2
# (a)-(e): Vid2VidModelD.forward(0, ...) cases: name -> (h, w, openpose_only, face blob (frame, y0, y1, x0, x1) or None,
# boundary decoys, with fake_B_raw)
CASES = {
    'interior': (96, 128, False, (0, 30, 41, 50, 67), False, True),
    'corner': (96, 128, False, (1, 80, 96, 110, 128), False, False),
    'none': (96, 128, False, None, False, True),
    'openpose': (96, 128, True, (1, 20, 29, 70, 90), True, False),
    'short': (48, 128, False, (0, 10, 30, 20, 40), False, True),
}
LOSS_NAMES = ['G_VGG', 'G_GAN', 'G_GAN_Feat', 'D_real', 'D_fake', 'G_Warp', 'F_Flow', 'F_Warp', 'W',
              'G_f_GAN', 'G_f_GAN_Feat', 'D_f_real', 'D_f_fake']
STAT_KEYS = ('running_mean', 'running_var')


# ----------------------------------------------------------------------------- restatement
def face_mask(real_A, openpose_only):
    """The face predicate of get_face_region (vid2vid_model_D.py:217-220): fp32 tensors against Python floats."""
    if not openpose_only:
        return real_A[:, 2] > 0.9
    return (real_A[:, 0] > 0.19) & (real_A[:, 0] < 0.21) & (real_A[:, 1] < -0.99) & (real_A[:, 2] > -0.61) & (real_A[:, 2] < -0.59)


def face_box(real_A, openpose_only):
    face = face_mask(real_A, openpose_only).nonzero()
    if not face.size(0):
        return None
    y, x = face[:, 1], face[:, 2]
    return int(y.min()), int(y.max()), int(x.min()), int(x.max())


def face_window(box, h, w, fineSize):
    """vid2vid_model_D.py:224-229."""
    if box is None:
        return None
    ys, ye, xs, xe = box
    yc, ylen = (ys + ye) // 2, fineSize // 32 * 8
    xc, xlen = (xs + xe) // 2, fineSize // 32 * 8
    yc = max(ylen // 2, min(h - 1 - ylen // 2, yc))
    xc = max(xlen // 2, min(w - 1 - xlen // 2, xc))
    return yc - ylen // 2, yc + ylen // 2, xc - xlen // 2, xc + xlen // 2


def running_stats(sd):
    """{norm layer prefix: [running_mean, running_var]} copies of a discriminator state_dict's batch-norm buffers."""
    return {k[:-len('.running_mean')]: [sd[k].clone(), sd[k[:-len('mean')] + 'var'].clone()]
            for k in sd if k.endswith('.running_mean')}


def tracked_discriminator(sd, stats, inp, *, num_D, n_layers=3):
    """generator_oracle.multiscale_discriminator with batch norm in train mode that also advances the running statistics in
    `stats` (nn.BatchNorm2d, momentum 0.1, unbiased variance), as every netD_f.forward of the reference does."""
    result = []
    x = inp
    for i in range(num_D):
        d = num_D - 1 - i
        feats = []
        h = x
        for j in range(n_layers + 2):
            p = 'scale%d_layer%d' % (d, j)
            h = GO._conv(h, sd, p + '.0', stride=2 if j < n_layers else 1, padding=2)
            if 0 < j < n_layers + 1:
                rm, rv = stats[p + '.1']
                h = F.batch_norm(h, rm, rv, sd[p + '.1.weight'], sd[p + '.1.bias'], True, 0.1, GO.EPS)
            if j < n_layers + 1:
                h = F.leaky_relu(h, 0.2)
            feats.append(h)
        result.append(feats)
        if i != num_D - 1:
            x = GO.avgpool3s2(x)
    return result


def face_terms(sd_f, stats_f, real_A, real_B, fake_B, window, *, num_D, n_layers_D=3, lambda_feat=10.0):
    """vid2vid_model_D.py:149-158 with compute_loss_D (:168-179) on netD_f (max(1, num_D - 2) towers): three tower calls
    (real, detached fake, fake), GAN_and_FM_loss weighted by netD's num_D.  Returns [G_f_GAN, G_f_GAN_Feat, D_f_real,
    D_f_fake], each (1, 1); zeros and no tower call without a face."""
    if window is None:
        z = torch.zeros(())
        return [z.reshape(1, 1)] * 4
    ys, ye, xs, xe = window
    crop = lambda t: t[:, :, ys:ye, xs:xe]
    real_AB, fake_AB = torch.cat((crop(real_A), crop(real_B)), 1), torch.cat((crop(real_A), crop(fake_B)), 1)
    kw = dict(num_D=max(1, num_D - 2), n_layers=n_layers_D)
    pred_real = tracked_discriminator(sd_f, stats_f, real_AB, **kw)
    pred_fake = tracked_discriminator(sd_f, stats_f, fake_AB.detach(), **kw)
    d_real, d_fake = LO.gan_loss(pred_real, True), LO.gan_loss(pred_fake, False)
    pred_fake = tracked_discriminator(sd_f, stats_f, fake_AB, **kw)
    g_gan, g_fm = LO.gan_and_fm_loss(pred_real, pred_fake, n_layers_D=n_layers_D, num_D=num_D, lambda_feat=lambda_feat)
    return [t.reshape(1, 1) for t in (g_gan * FACE_WEIGHT, g_fm * FACE_WEIGHT, d_real, d_fake)]


def face_disc_losses(sd_D, sd_f, stats_f, inputs, opt):
    """The 13 losses of Vid2VidModelD.forward(0, inputs) with --add_face_disc, --no_vgg (forward values)."""
    real_B, fake_B, fake_B_raw, real_A, real_B_prev, fake_B_prev, flow, weight, flow_ref, conf_ref = inputs
    lo = LO.spatial_losses(sd_D, real_B, fake_B, fake_B_raw, real_A, real_B_prev, fake_B_prev, flow, weight, flow_ref, conf_ref,
                           lambda_F=opt.lambda_F, lambda_T=opt.lambda_T, lambda_feat=opt.lambda_feat,
                           n_scales_spatial=opt.n_scales_spatial, no_first_img=opt.no_first_img, num_D=opt.num_D,
                           n_layers_D=opt.n_layers_D, norm=opt.norm)
    window = face_window(face_box(real_A, opt.openpose_only), *real_A.shape[-2:], opt.fineSize)
    return lo + face_terms(sd_f, stats_f, real_A, real_B, fake_B, window, num_D=opt.num_D, n_layers_D=opt.n_layers_D,
                           lambda_feat=opt.lambda_feat)


# ----------------------------------------------------------------------------- seeded pose-like inputs
F32 = lambda v: float(np.float32(v))


def pose_maps(N, H, W, seed, blob=None, openpose_only=False, decoys=False, block=1):
    """(N, 6, H, W) dense maps in [-1, 1] standing in for the pose demo's DensePose + OpenPose channels.  Outside the blob
    no pixel satisfies either face predicate (channel 2 <= 0.85, channel 1 >= -0.98); blob = (frame, y0, y1, x0, x1) gets
    pixels that satisfy the predicate selected by openpose_only.  decoys: pixels far from the blob that sit exactly on
    the fp32 boundaries (c0 == float32(0.21), c1 == float32(-0.99), c2 == float32(0.9)) and so match neither predicate in
    fp32, although two of them would match a double comparison.  block > 1: noise on an H / block x W / block grid,
    bilinearly upsampled (smooth maps, closer to rendered pose channels than per-pixel noise)."""
    g = torch.Generator().manual_seed(seed)
    if block > 1:
        x = F.interpolate(torch.rand(N, 6, H // block, W // block, generator=g) * 2 - 1, size=(H, W), mode='bilinear',
                          align_corners=False)
    else:
        x = torch.rand(N, 6, H, W, generator=g) * 2 - 1
    x[:, 2] = x[:, 2] * 0.925 - 0.075                      # [-1, 0.85]
    x[:, 1] = x[:, 1] * 0.99 + 0.01                        # [-0.98, 1]
    if blob is not None:
        n, y0, y1, x0, x1 = blob
        if openpose_only:
            x[n, 0, y0:y1, x0:x1], x[n, 1, y0:y1, x0:x1], x[n, 2, y0:y1, x0:x1] = 0.2, -1.0, -0.6
        else:
            x[n, 2, y0:y1, x0:x1] = 0.95
    if decoys:
        x[0, 0, H - 2, 2], x[0, 1, H - 2, 2], x[0, 2, H - 2, 2] = F32(0.21), -1.0, -0.6          # c0 < 0.21 fails in fp32
        x[0, 0, 1, W - 3], x[0, 1, 1, W - 3], x[0, 2, 1, W - 3] = 0.2, F32(-0.99), -0.6          # c1 < -0.99 fails in fp32
        x[N - 1, 2, H - 3, W - 2] = F32(0.9)                                                      # c2 > 0.9 fails
    return x


def _rand(shape, g, lo=-1.0, hi=1.0):
    return torch.rand(shape, generator=g) * (hi - lo) + lo


def case_opt(name):
    h, w, openpose_only, _, _, _ = CASES[name]
    return make_opt(label_nc=0, input_nc=6, use_instance=False, isTrain=True, gpu_ids=[0], n_gpus_gen=1, no_vgg=True,
                    add_face_disc=True, openpose_only=openpose_only, no_flow=openpose_only, no_first_img=True, num_D=3, ndf=16,
                    n_scales_spatial=2, fineSize=256, dataroot='datasets/pose', dataset_mode='pose')


def case_inputs(name, N=2):
    """The input list of Vid2VidModelD.forward(0, ...) for case `name` (merged batch of N frames; no flow under
    openpose_only, whose generator has none)."""
    h, w, openpose_only, blob, decoys, with_raw = CASES[name]
    g = torch.Generator().manual_seed(SEED + sorted(CASES).index(name))
    real_B, fake_B, real_B_prev, fake_B_prev = (_rand((N, 3, h, w), g) for _ in range(4))
    fake_B_raw = _rand((N, 3, h, w), g) if with_raw else None
    real_A = pose_maps(N, h, w, SEED + 7 * sorted(CASES).index(name), blob, openpose_only, decoys)
    flow, flow_ref = _rand((N, 2, h, w), g, -3, 3), _rand((N, 2, h, w), g, -3, 3)
    weight = _rand((N, 1, h, w), g, 0, 1)
    conf = (_rand((N, 1, h, w), g) > 0).float()
    if openpose_only:
        flow = weight = None
    return [real_B, fake_B, fake_B_raw, real_A, real_B_prev, fake_B_prev, flow, weight, flow_ref, conf]


def pose_clip(T, H, W, seed, blob_rows=(8, 16), blob_cols=(24, 40), openpose_only=False):
    """(1, T, 6, H, W) smooth pose maps with a face blob drifting one pixel right per frame, and (1, T, 3, H, W) low-pass
    real frames in [-1, 1]."""
    A = torch.stack([pose_maps(1, H, W, seed + t, (0, blob_rows[0], blob_rows[1], blob_cols[0] + t, blob_cols[1] + t),
                               openpose_only, block=8)[0] for t in range(T)]).unsqueeze(0)
    g = torch.Generator().manual_seed(seed + 100)
    coarse = torch.rand(T, 3, H // 8, W // 8, generator=g) * 2 - 1
    B = F.interpolate(coarse, size=(H, W), mode='bilinear', align_corners=False).unsqueeze(0)
    return A, B


def pose_g_opt(**kw):
    o = dict(label_nc=0, input_nc=6, use_instance=False, fg=False, n_scales_spatial=2, ngf=8, n_blocks=2, n_blocks_local=1,
             n_downsample_G=2, gpu_ids=[0], n_gpus_gen=1, isTrain=True, no_first_img=True, max_frames_per_gpu=2, batchSize=1,
             dataroot='datasets/pose', dataset_mode='pose')
    o.update(kw)
    return make_opt(**o)


G_SEEDS = (81, 82)
G_CLIP = (6, 32, 64)                 # frames, H, W of the generator case: two calls of two frames


def g_call_inputs(A, B, opt, call):
    sl = slice(call * 2, call * 2 + 2 + opt.n_frames_G - 1)
    return A[:, sl].contiguous(), B[:, sl].contiguous()


def condition(net):
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import cases
    cases.condition_flow_heads(net, 0.05)
    return net


# ----------------------------------------------------------------------------- recipe
def ref_model_D(opt):
    import contextlib
    import io
    from oracle import ref_shim
    ref_shim.install()
    from models.vid2vid_model_D import Vid2VidModelD          # noqa (reference module)
    m = Vid2VidModelD()
    with contextlib.redirect_stdout(io.StringIO()):
        m.initialize(opt)
    det_fill_(m.netD, seed=D_SEED)
    det_fill_(m.netD_f, seed=D_F_SEED)
    return m


def make_golden(out_dir=os.path.join(ROOT, 'tests', 'golden')):
    import json
    from oracle import ref_shim
    written = []
    torch.manual_seed(0)
    # state_dict keys of netD_f as the pose 512p (num_D 3: one tower) and 1024p (num_D 4: two towers) recipes build it
    keys = {}
    for num_D in (3, 4):
        m = ref_model_D(make_opt(label_nc=0, input_nc=6, use_instance=False, isTrain=True, gpu_ids=[0], n_gpus_gen=1, no_vgg=True,
                                 add_face_disc=True, num_D=num_D, n_scales_temporal=1))
        keys['num_D_%d' % num_D] = [[n, list(v.shape)] for n, v in m.netD_f.state_dict().items()]
    path = os.path.join(out_dir, 'face_disc_keys.json')
    with open(path, 'w') as f:
        json.dump(keys, f)
        f.write('\n')
    written.append(path)

    out = {}
    with torch.no_grad():
        for name in CASES:
            opt = case_opt(name)
            m = ref_model_D(opt)
            inputs = case_inputs(name)
            box = m.get_face_region(inputs[3])
            out['%s/window' % name] = np.asarray([-1 if v is None else v for v in box], dtype=np.int64)
            for n, v in zip(LOSS_NAMES, m.forward(0, inputs)):
                out['%s/loss/%s' % (name, n)] = v.numpy()
            for k, v in m.netD_f.state_dict().items():
                if k.rsplit('.', 1)[-1] in STAT_KEYS:
                    out['%s/stats/%s' % (name, k)] = v.numpy()
        # (f) Vid2VidModelG.forward in pose mode: two calls continuing from the returned fake_B_prev pyramid
        opt = pose_g_opt()
        g = ref_shim.make_model_G(opt)
        for s in range(2):
            condition(det_fill_(getattr(g, 'netG%d' % s), seed=G_SEEDS[s]))
        A, B = pose_clip(*G_CLIP, SEED + 50)
        prev = None
        for call in range(2):
            a, b = g_call_inputs(A, B, opt, call)
            r = g.forward(a, b, a, prev)
            for n, v in zip(['fake_B', 'fake_B_raw', 'flow', 'weight', 'real_A', 'real_B'], r[:6]):
                out['g/%d/%s' % (call, n)] = v.numpy()
            prev = r[6]
    path = os.path.join(out_dir, 'face_disc.npz')
    np.savez_compressed(path, **out)
    written.append(path)
    return written


if __name__ == '__main__':
    for p in make_golden(*sys.argv[1:2]):
        print(p)
