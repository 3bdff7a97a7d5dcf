"""Seeded inputs and options of the checks against the reference whose outputs are stored in
tests/golden/reference*.npz and tests/golden/host_schedule.json (written by
`python -m oracle.make_golden reference_checks`).  Shared by that recipe and the tests, so both sides
see the same inputs; weights are regenerated from seeds with det_fill_ / flownet2_oracle.det_state_dict."""
import os
import types

import torch
import torch.nn as nn

from vid2vid_b200.utils import make_opt, synth_label_sequence

GOLD = os.path.join(os.path.dirname(__file__), 'golden')

COMPOSITE_VARIANTS = [(True, False, 3), (False, False, 2), (True, True, 3)]      # (fg, no_flow, n_downsampling)
TRAIN_OUT_NAMES = ['fake_B', 'fake_B_raw', 'flow', 'weight', 'real_A', 'real_B']
LOSS_NAMES = ['G_VGG', 'G_GAN', 'G_GAN_Feat', 'D_real', 'D_fake', 'G_Warp', 'F_Flow', 'F_Warp', 'W']
LOSS_NAMES_T = ['G_T_GAN', 'G_T_GAN_Feat', 'D_T_real', 'D_T_fake', 'G_T_Warp']
# spatial losses: (no_first_img, with fake_B_raw); temporal losses: the default options
LOSS_MODELS = {'raw': dict(n_scales_spatial=2, no_first_img=False), 'no_first_img': dict(n_scales_spatial=2, no_first_img=True),
               'temporal': dict(no_first_img=False)}
D_SEED, D_T_SEED = 41, 42
FLOWNET_SEED = 3
FLOWNET_WRAPPER_SIZES = ((64, 64), (70, 64))
SCHEDULE_EPOCHS = (11, 15, 20)
SCHEDULE_RATIOS = range(1, 6)


def golden():
    """{key: array} of the stored reference outputs (tests/golden/reference.npz and its parts)."""
    import cases
    return cases.load_golden('reference')


def composite_key(fg, no_flow, nd):
    return 'composite_fg%d_noflow%d_nd%d' % (int(fg), int(no_flow), nd)


def gen_inputs(nc, h, w, seed=0):
    from oracle import generator_oracle as GO
    g = torch.Generator().manual_seed(seed)
    lab = synth_label_sequence(3, h, w, label_nc=nc - 1, block=4, seed=seed)
    real_A = GO.encode_input(lab, lab, nc - 1, True)
    inp = real_A.view(1, -1, h, w)
    img_prev = torch.rand(1, 6, h, w, generator=g) * 2 - 1
    mask = (lab[:, -1] == 2).float()
    return inp, img_prev, mask


def local_coarse():
    g = torch.Generator().manual_seed(5)
    return tuple(torch.randn(1, c, 8, 16, generator=g) for c in (8, 8, 4))


def single_image_input():
    return torch.rand(1, 5, 32, 64, generator=torch.Generator().manual_seed(3))


def discriminator_input():
    return torch.randn(2, 9, 32, 48, generator=torch.Generator().manual_seed(6))


def inference_opt():
    return make_opt(label_nc=5, use_instance=True, fg=True, fg_labels=[2], n_scales_spatial=2, ngf=8, n_blocks=2, n_blocks_local=1,
                    use_single_G=True, n_downsample_G=2, gpu_ids=[], dataroot='City')


def inference_sequence():
    return synth_label_sequence(5, 32, 64, label_nc=5, block=4, seed=3)


def train_opt(no_first_img):
    return make_opt(label_nc=5, use_instance=True, fg=True, fg_labels=[2], n_scales_spatial=2, ngf=8, n_blocks=2, n_blocks_local=1,
                    n_downsample_G=2, gpu_ids=[0], n_gpus_gen=1, isTrain=True, no_first_img=no_first_img, max_frames_per_gpu=2,
                    batchSize=1, dataroot='City')


def train_clip(opt):
    T = 2 * 2 + opt.n_frames_G - 1
    seq = synth_label_sequence(T, 32, 64, label_nc=5, block=4, seed=4)
    real = torch.rand(1, T, 3, 32, 64, generator=torch.Generator().manual_seed(6)) * 2 - 1
    return seq, real


def train_call_inputs(seq, real, opt, call):
    """The contiguous clip of training call `call` (two generated frames per call)."""
    sl = slice(call * 2, call * 2 + 2 + opt.n_frames_G - 1)
    return seq[:, sl].contiguous(), real[:, sl].contiguous()


def objective(outs, cot):
    return sum((o * c).sum() for o, c in zip(outs, cot) if o is not None)


def cotangents(outs):
    g = torch.Generator().manual_seed(9)
    return [torch.randn(o.shape, generator=g) if o is not None else None for o in outs]


def loss_opt(**kw):
    return make_opt(label_nc=35, use_instance=True, isTrain=True, gpu_ids=[0], n_gpus_gen=1, no_vgg=True, **kw)


def _rand(shape, g, lo=-1.0, hi=1.0):
    return torch.rand(shape, generator=g) * (hi - lo) + lo


def spatial_loss_inputs(opt, no_first_img, with_raw):
    """The input list of Vid2VidModelD.forward(0, ...)."""
    g = torch.Generator().manual_seed(1)
    h, w = 48, 64
    real_B, fake_B, real_B_prev, fake_B_prev = (_rand((1, 3, h, w), g) for _ in range(4))
    fake_B_raw = _rand((1, 3, h, w), g) if with_raw else None
    real_A = (_rand((1, 36, h, w), g) > 0.8).float()
    flow, flow_ref = _rand((1, 2, h, w), g, -3, 3), _rand((1, 2, h, w), g, -3, 3)
    weight = _rand((1, 1, h, w), g, 0, 1)
    conf = (_rand((1, 1, h, w), g) > 0).float()
    return [real_B, fake_B, fake_B_raw, real_A, real_B_prev, fake_B_prev, flow, weight, flow_ref, conf]


def temporal_loss_inputs(opt):
    """The input list of Vid2VidModelD.forward(1, ...)."""
    g = torch.Generator().manual_seed(2)
    h, w, tD = 48, 64, opt.n_frames_D
    real_B, fake_B = _rand((1, tD, 3, h, w), g), _rand((1, tD, 3, h, w), g)
    flow_ref = _rand((1, tD - 1, 2, h, w), g, -40, 40)
    conf = (_rand((1, tD - 1, 1, h, w), g) > 0).float()
    return [real_B, fake_B, flow_ref, conf]


def flownet_inputs():
    g = torch.Generator().manual_seed(13)
    return {'pair': torch.rand(2, 3, 2, 64, 64, generator=g), 'x6': torch.rand(1, 6, 64, 128, generator=g) - 0.5,
            'x12': torch.rand(1, 12, 64, 128, generator=g) - 0.5, 'xf': torch.rand(1, 11, 64, 64, generator=g)}


def flownet_wrapper_inputs(h, w):
    im1 = torch.rand(1, 3, h, w, generator=torch.Generator().manual_seed(h * 1000 + w))
    return im1, torch.roll(im1, shifts=(1, 1), dims=(2, 3))


def flownet_pair_128x192():
    base = torch.rand(1, 3, 128, 192, generator=torch.Generator().manual_seed(8))
    return torch.stack([base, torch.roll(base, shifts=(1, 2), dims=(2, 3)) * 0.9 + 0.05], 2)


def schedule_opt(tmp):
    return types.SimpleNamespace(checkpoints_dir=str(tmp), name='run', lr=2e-4, niter=10, niter_decay=10, beta1=0.5,
                                 max_frames_backpropagate=4, max_frames_per_gpu=8)


def schedule_state(opt, cls):
    """A model object of class `cls` in the state BaseModel's schedule helpers expect."""
    torch.manual_seed(0)
    m = cls()
    m.opt = opt
    m.old_lr = opt.lr
    m.n_scales = 2
    m.netG0, m.netG1 = nn.Linear(3, 2), nn.Linear(2, 2)
    m.optimizer_G = torch.optim.Adam(list(m.netG1.parameters()), lr=opt.lr, betas=(opt.beta1, 0.999))
    m.n_gpus, m.n_frames_per_gpu, m.n_frames_load, m.n_frames_bp = 1, 1, 1, 1
    m.finetune_all = False
    return m
