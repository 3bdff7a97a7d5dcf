"""The plans the products lower: one inventory of PlanSpec records for the CPU censuses (tests/test_conv_census.py,
tests/test_epilogue_forward_census.py, tests/test_epilogue_backward_census.py).  Each group is built from the product's own
definitions, so it follows them when they change:

  bench        bench.py: cfg4 and cfg2 inference in both arithmetic modes; cfg3's training step in precise mode (the generator
               scales, and the image and temporal discriminators' towers at the shapes Vid2VidModelD feeds them); FlowNet2's
               five sub-plans on one frame pair (the flownet2 workload, and cfg3's reference flow at the same size).
  first_frame  the first-frame generators of Vid2VidModelG.load_single_G: netG_i for City at loadSize 512 / 1024 / 2048
               (2:1 frames), and for face the Encoder plus Global_with_z at tools/time_face.py's size.  They run under
               no_grad in whichever arithmetic mode the generators use: neither Vid2VidModelG nor these networks pin a mode,
               so all of them are listed in both.
  vgg          the VGG19 loss plan at the sizes tools/time_vgg.py times, after VGGLoss's halving of images wider than 1024
               pixels; a training plan (the generator's output needs its gradient) and the inference plan.  Vgg19 freezes its
               weights (frozen): the backward launches no weight gradient.
  pose_step    tools/time_face_disc.py's training step: the pose generator scales, netD, the temporal netD_T towers and
               netD_f (--add_face_disc) at the shapes Vid2VidModelD feeds them.  Precise mode, as training runs.
  multiclip    tools/time_multiclip.py: every workload's generator scales in both modes at every clip count B, per-sample
               plans for B > 1.
  slots        tools/time_slots.py: the generator scales of the slot streams, per-sample plans reading per-image flags.

The lowering depends on the SM count: with no device it assumes the H100 SXM's 132 SMs, and on a GPU host the censuses run
only on a 132-SM device (h100_sxm)."""
import collections
import functools
import os
import sys
from types import SimpleNamespace

import pytest
import torch

import bench
from vid2vid_b200 import flownet as FN
from vid2vid_b200 import networks as NW
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.plan import Plan
from vid2vid_b200.utils import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import time_face as TF             # noqa: E402
import time_face_disc as TFD       # noqa: E402
import time_multiclip as TM        # noqa: E402
import time_slots as TS            # noqa: E402
import time_vgg as TV              # noqa: E402

H100_SXM_SMS = 132
MODES = ('fast', 'precise')
CITY_LOAD_SIZES = (512, 1024, 2048)     # the loadSizes load_single_G has a City generator for; frames are W x W / 2

# describe(plan) lowers the plan's graph onto `plan`, which is created with the remaining fields.  sample_stats: per-image
# norm statistics; flags: the plan reads per-image flags; frozen: no parameter asks for a gradient.
PlanSpec = collections.namedtuple('PlanSpec', 'group tag describe precision train sample_stats flags frozen',
                                  defaults=(False, False, False, False))


@pytest.fixture(autouse=True)
def h100_sxm():
    """Imported by a test module, skips its tests on a GPU whose SM count is not the H100 SXM's."""
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != H100_SXM_SMS:
        pytest.skip('the census describes a %d-SM H100 SXM; this device has %d SMs' % (
            H100_SXM_SMS, torch.cuda.get_device_properties(0).multi_processor_count))


@functools.lru_cache(maxsize=None)
def describe(spec):
    """v2v_plan_describe of one plan, lowered once per process."""
    p = Plan(0, precision=spec.precision, train=spec.train, sample_stats=spec.sample_stats)
    if spec.flags:
        p.set_image_flags(NW.S_FLAGS)
    spec.describe(p)
    return p.describe()


def _net(net, *shape):
    return lambda p: net._describe(p, *shape)


def scales(opt, H, W):
    """[(netG{s}, h, w)] of a workload's generator scales (networks.build_netGs) at its H x W frames."""
    S = opt.n_scales_spatial
    return [(net, H // 2 ** (S - 1 - s), W // 2 ** (S - 1 - s)) for s, net in enumerate(NW.build_netGs(opt))]


def clip_opt(w):
    """The options of a tools/time_multiclip.py or tools/time_slots.py workload, as time_multiclip builds its model."""
    o = w['opt']
    return make_opt(**{'use_single_G': False, 'use_real_img': not o.get('no_first_img', False), 'gpu_ids': [],
                       'synthetic_weights': True, **o})


def _discriminators(group, tag, opt, H, W, face=False):
    """Vid2VidModelD.initialize's netD (the input maps plus the image), every temporal scale's netD_T (n_frames_D images and
    the flows between them) and with face netD_f: netD's input on two towers fewer, on the fineSize // 32 * 8 square around
    the face (Vid2VidModelD.face_window).  Tower k of a num_D-tower discriminator runs on level num_D - 1 - k of the avg-pool
    pyramid (MultiscaleDiscriminator); one clip, one generated frame."""
    input_nc = (opt.label_nc if opt.label_nc != 0 else opt.input_nc) + int(opt.use_instance)
    crop = opt.fineSize // 32 * 8
    ds = [('D', input_nc + opt.output_nc, opt.num_D, H, W)]
    if face:
        ds.append(('D_f', input_nc + opt.output_nc, max(1, opt.num_D - 2), crop, crop))
    ds.append(('D_T', opt.output_nc * opt.n_frames_D + 2 * (opt.n_frames_D - 1), opt.num_D, H, W))
    out = []
    for name, nc, num_D, h, w in ds:
        d = NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, num_D, not opt.no_ganFeat, [])
        for i in range(num_D):
            tower = num_D - 1 - i
            out.append(PlanSpec(group, '%s %s tower %d' % (tag, name, tower),
                                functools.partial(lambda d, t, h, w, p: d._describe(p, t, 1, h, w), d, tower, h, w), 'precise', True))
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return out


def _bench():
    out = []
    for wl, modes, train in (('cfg4', MODES, False), ('cfg2', MODES, False), ('cfg3', ('precise',), True)):
        W = bench.WORKLOADS[wl]
        for s, (net, h, w) in enumerate(scales(bench.make_opt_for(wl), W['H'], W['W'])):
            out += [PlanSpec('bench', '%s %s G%d' % (wl, mode, s), _net(net, 1, h, w), mode, train) for mode in modes]
    opt, W = bench.make_opt_for('cfg3'), bench.WORKLOADS['cfg3']
    opt.num_D = opt.n_frames_D = 3                  # bench.py's training options
    out += _discriminators('bench', 'cfg3', opt, W['H'], W['W'])
    W, f = bench.WORKLOADS['flownet2'], FN.FlowNet2()
    for name in ('flownetc', 'flownets_1', 'flownets_2', 'flownets_d', 'flownetfusion'):
        out.append(PlanSpec('bench', 'flownet2 ' + name, functools.partial(lambda sub, p: sub.describe(p, 1, W['H'], W['W']),
                                                                           getattr(f, name)), FN.FlowNet2.precision))
    return out


def _single_G(**kw):
    """(netG_i, netE or None) as Vid2VidModelG.load_single_G builds them: weights and the features table are not loaded."""
    host = SimpleNamespace(opt=make_opt(gpu_ids=[], synthetic_weights=True, **kw), device_='cpu')
    host._load = lambda net, path: net
    host.load_face_features = lambda path: None
    netG = Vid2VidModelG.load_single_G(host)
    return netG, getattr(host, 'netE', None)


def _first_frame():
    nets = []
    for load in CITY_LOAD_SIZES:
        netG, _ = _single_G(dataroot='datasets/Cityscapes/', loadSize=load, label_nc=35)
        nets.append(('City %d netG_i' % load, netG, load // 2, load))
    netG, netE = _single_G(dataroot='datasets/face/', dataset_mode='face', label_nc=0, input_nc=15)
    nets += [('face %d netE' % TF.SIZE, netE, TF.SIZE, TF.SIZE), ('face %d netG_i' % TF.SIZE, netG, TF.SIZE, TF.SIZE)]
    return [PlanSpec('first_frame', '%s %s' % (tag, mode), _net(net, 1, h, w), mode) for tag, net, h, w in nets for mode in MODES]


def vgg_sizes():
    """The (H, W) the loss plans run at: VGGLoss.forward halves the images while they are wider than 1024 pixels."""
    sizes = []
    for H, W in TV.LOSS_SIZES:
        while W > 1024:
            H, W = H // 2, W // 2
        if (H, W) not in sizes:
            sizes.append((H, W))
    return sizes


def _vgg():
    net = NW.Vgg19()
    return [PlanSpec('vgg', 'VGG %dx%d%s' % (W, H, ' train' if train else ''), _net(net, 1, H, W), 'precise', train, frozen=True)
            for H, W in vgg_sizes() for train in (True, False)]


def pose_opt():
    return make_opt(gpu_ids=[], add_face_disc=True, fineSize=TFD.SIZE, loadSize=TFD.SIZE, **TFD.OPT)


def _pose_step():
    opt = pose_opt()
    out = [PlanSpec('pose_step', 'pose G%d' % s, _net(net, 1, h, w), 'precise', True)
           for s, (net, h, w) in enumerate(scales(opt, TFD.SIZE, TFD.SIZE))]
    return out + _discriminators('pose_step', 'pose', opt, TFD.SIZE, TFD.SIZE, face=True)


def _clips(group, workloads, flags):
    out = []
    for wl, w in workloads.items():
        for s, (net, h, w_) in enumerate(scales(clip_opt(w), w['H'], w['W'])):
            out += [PlanSpec(group, '%s %s %s G%d B=%d' % (group, wl, mode, s, B), _net(net, B, h, w_), mode,
                             sample_stats=flags or B > 1, flags=flags) for mode in MODES for B in w['bs']]
    return out


@functools.lru_cache(maxsize=None)
def plans():
    """Every PlanSpec of the products."""
    return tuple(_bench() + _first_frame() + _vgg() + _pose_step() + _clips('multiclip', TM.WORKLOADS, False) +
                 _clips('slots', TS.WORKLOADS, True))


def group(*names):
    return [s for s in plans() if s.group in names]
