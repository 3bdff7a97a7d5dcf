"""Pins oracle/losses_oracle.py (SURVEY 8 row a13: warp / flow / GAN / feature-matching losses of the training step)
against the unmodified reference Vid2VidModelD.forward (models/vid2vid_model_D.py:92-197) on CPU, --no_vgg: its loss
values on seeded inputs, with discriminators filled by det_fill_, are stored in tests/golden/reference*.npz."""
import pytest
import torch

import reference_inputs as RI
from oracle import losses_oracle as LO
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import det_fill_

GOLD = RI.golden()


def _discriminators(opt):
    """netD and netD_T0 as Vid2VidModelD builds them (vid2vid_model_D.py:33-46), with the weights of the stored run."""
    input_nc = opt.label_nc + (1 if opt.use_instance else 0) + opt.output_nc
    nc_t = opt.output_nc * opt.n_frames_D + 2 * (opt.n_frames_D - 1)
    netD = det_fill_(NW.define_D(input_nc, opt.ndf, opt.n_layers_D, opt.norm, opt.num_D, not opt.no_ganFeat, []), seed=RI.D_SEED)
    netD_T = det_fill_(NW.define_D(nc_t, opt.ndf, opt.n_layers_D, opt.norm, opt.num_D, not opt.no_ganFeat, []), seed=RI.D_T_SEED)
    return netD, netD_T


@pytest.mark.parametrize('no_first_img,with_raw', [(False, True), (True, False)])
def test_spatial_losses_match_reference(no_first_img, with_raw):
    tag = 'raw' if with_raw else 'no_first_img'
    opt = RI.loss_opt(**RI.LOSS_MODELS[tag])
    assert opt.no_first_img == no_first_img
    netD, _ = _discriminators(opt)
    with torch.no_grad():
        ours = LO.spatial_losses(netD.state_dict(), *RI.spatial_loss_inputs(opt, no_first_img, with_raw), lambda_F=opt.lambda_F,
                                 lambda_T=opt.lambda_T, lambda_feat=opt.lambda_feat, n_scales_spatial=opt.n_scales_spatial,
                                 no_first_img=no_first_img, num_D=opt.num_D, n_layers_D=opt.n_layers_D, norm=opt.norm)
    assert len(ours) == len(RI.LOSS_NAMES)
    for n, a in zip(RI.LOSS_NAMES, ours):
        b = torch.from_numpy(GOLD['losses/%s/%s' % (tag, n)])
        # (G_VGG under --no_vgg and W without --no_first_img are zeros_like(weight): H*W rows of zeros in both)
        assert a.shape == b.shape, (n, a.shape, b.shape)
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), (n, float(a.abs().max()), float(b.abs().max()))
        if n in ('G_GAN', 'G_GAN_Feat', 'D_real', 'D_fake', 'G_Warp', 'F_Flow', 'F_Warp'):
            assert a.shape == (1, 1) and float(a) > 0


def test_temporal_losses_match_reference():
    opt = RI.loss_opt(**RI.LOSS_MODELS['temporal'])
    _, netD_T = _discriminators(opt)
    with torch.no_grad():
        ours = LO.temporal_losses(netD_T.state_dict(), *RI.temporal_loss_inputs(opt), n_frames_D=opt.n_frames_D, output_nc=3,
                                  lambda_feat=opt.lambda_feat, num_D=opt.num_D, n_layers_D=opt.n_layers_D, norm=opt.norm)
    assert len(ours) == len(RI.LOSS_NAMES_T)
    for n, a in zip(RI.LOSS_NAMES_T, ours):
        b = torch.from_numpy(GOLD['losses/temporal/' + n])
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), (n, float(a), float(b))
