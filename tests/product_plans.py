"""The plans that product paths outside bench.py lower, as (tag, describe(plan)) lists for the CPU censuses
(tests/test_product_census.py).  Each list is built from the path's own definitions, so it follows them when they change:

  first_frame    the first-frame generators of Vid2VidModelG.load_single_G: netG_i for City at loadSize 512 / 1024 / 2048
                 (2:1 frames), and for face the Encoder plus Global_with_z at tools/time_face.py's size.  They run under
                 no_grad in whichever arithmetic mode the generators use: neither Vid2VidModelG nor these networks pin a mode,
                 so all of them follow networks.DEFAULT_PRECISION.
  vgg            the VGG19 loss plan at the sizes tools/time_vgg.py times, after VGGLoss's halving of images wider than 1024
                 pixels; a training plan (the generator's output needs its gradient) and the inference plan.
  pose_step      tools/time_face_disc.py's training step: the pose generator scales, netD, the temporal netD_T towers and
                 netD_f (--add_face_disc) at the shapes Vid2VidModelD feeds them.  Precise mode, as training runs."""
import functools
import os
import sys
from types import SimpleNamespace

from vid2vid_b200 import networks as NW
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.utils import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import time_face as TF             # noqa: E402
import time_face_disc as TFD       # noqa: E402
import time_vgg as TV              # noqa: E402

CITY_LOAD_SIZES = (512, 1024, 2048)     # the loadSizes load_single_G has a City generator for; frames are W x W / 2


def _describe(net, *shape):
    return functools.partial(lambda net, shape, p: net._describe(p, *shape), net, shape)


def _single_G(**kw):
    """(netG_i, netE or None) as Vid2VidModelG.load_single_G builds them: weights and the features table are not loaded."""
    host = SimpleNamespace(opt=make_opt(gpu_ids=[], synthetic_weights=True, **kw), device_='cpu')
    host._load = lambda net, path: net
    host.load_face_features = lambda path: None
    netG = Vid2VidModelG.load_single_G(host)
    return netG, getattr(host, 'netE', None)


@functools.lru_cache(maxsize=None)
def first_frame():
    out = []
    for load in CITY_LOAD_SIZES:
        netG, _ = _single_G(dataroot='datasets/Cityscapes/', loadSize=load, label_nc=35)
        out.append(('City %d netG_i' % load, _describe(netG, 1, load // 2, load)))
    netG, netE = _single_G(dataroot='datasets/face/', dataset_mode='face', label_nc=0, input_nc=15)
    out.append(('face %d netE' % TF.SIZE, _describe(netE, 1, TF.SIZE, TF.SIZE)))
    out.append(('face %d netG_i' % TF.SIZE, _describe(netG, 1, TF.SIZE, TF.SIZE)))
    return out


def vgg_sizes():
    """The (H, W) the loss plans run at: VGGLoss.forward halves the images while they are wider than 1024 pixels."""
    sizes = []
    for H, W in TV.LOSS_SIZES:
        while W > 1024:
            H, W = H // 2, W // 2
        if (H, W) not in sizes:
            sizes.append((H, W))
    return sizes


@functools.lru_cache(maxsize=None)
def vgg():
    net = NW.Vgg19()
    return [('VGG %dx%d' % (W, H), _describe(net, 1, H, W)) for H, W in vgg_sizes()]


def pose_opt():
    return make_opt(gpu_ids=[], add_face_disc=True, fineSize=TFD.SIZE, loadSize=TFD.SIZE, **TFD.OPT)


def _towers(tag, d, num_D, H, W):
    """Tower k of a num_D-tower discriminator on level num_D - 1 - k of the avg-pool pyramid (MultiscaleDiscriminator)."""
    out = []
    for i in range(num_D):
        tower = num_D - 1 - i
        out.append(('%s tower %d' % (tag, tower), functools.partial(lambda d, t, h, w, p: d._describe(p, t, 1, h, w), d, tower, H, W)))
        H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    return out


@functools.lru_cache(maxsize=None)
def pose_step():
    opt = pose_opt()
    H = W = TFD.SIZE
    S = opt.n_scales_spatial
    out = []
    for s in range(S):
        sc = 2 ** (S - 1 - s)
        net = NW.build_netG(opt, s)
        net.input_exact_bf16 = s == S - 1 and opt.label_nc != 0      # as Vid2VidModelG.initialize sets it
        out.append(('pose G%d' % s, _describe(net, 1, H // sc, W // sc)))
    # Vid2VidModelD.initialize: netD and netD_f see the input maps plus the image; netD_f has two towers fewer and runs on the
    # fineSize // 32 * 8 square around the face (Vid2VidModelD.face_window); every temporal scale's netD_T sees
    # n_frames_D images and the flows between them
    input_nc = (opt.label_nc if opt.label_nc != 0 else opt.input_nc) + int(opt.use_instance)
    nc_t = opt.output_nc * opt.n_frames_D + 2 * (opt.n_frames_D - 1)
    num_D_f = max(1, opt.num_D - 2)
    crop = opt.fineSize // 32 * 8
    for tag, nc, num_D, h, w in (('pose D', input_nc + opt.output_nc, opt.num_D, H, W),
                                 ('pose D_f', input_nc + opt.output_nc, num_D_f, crop, crop),
                                 ('pose D_T', nc_t, opt.num_D, H, W)):
        d = NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, num_D, not opt.no_ganFeat, [])
        out += _towers(tag, d, num_D, h, w)
    return out
