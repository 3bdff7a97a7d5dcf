"""TEST INFRASTRUCTURE -- not product code (only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import oracle/).

CPU restatement of the per-frame training losses of the reference's discriminator-side model (SURVEY 8 row a13 and the
loss half of the training step): Vid2VidModelD.forward / compute_loss_D / compute_loss_D_T / GAN_and_FM_loss
(models/vid2vid_model_D.py:92-213) with the criteria of models/networks.py:731-812 (LSGAN, masked L1, feature
matching).  The VGG perceptual term needs downloaded weights and is outside the hot path (DESIGN.md section 5): it is
reported as zero, as the reference does under --no_vgg.  Pinned against the unmodified reference in
tests/test_losses_oracle.py.

Everything here is forward arithmetic on CPU tensors; the discriminator towers are generator_oracle.multiscale_discriminator.
"""
import torch
import torch.nn.functional as F

from . import generator_oracle as GO


def gan_loss(preds, target_is_real):
    """GANLoss.__call__ with use_lsgan truthy (networks.py:764-774; vid2vid_model_D.py:62 passes the gan_mode string as
    use_lsgan): for every tower, mean squared distance of its LAST output to the constant label 1 (real) / 0 (fake)."""
    label = 1.0 if target_is_real else 0.0
    total = 0
    for tower in preds:
        total = total + torch.mean((tower[-1] - label) ** 2)
    return total


# Sign source of every L1 term here.  None: mean |a - b|.  A callable sign(a, b) -> tensor shaped like a (entries +-1 or 0):
# the term becomes mean(sign * (a - b)), which has the same value wherever the sign is that of a - b and the same gradient
# away from a = b, but takes its kinks from the caller -- a gradient comparison with another implementation passes that
# implementation's signs, so that elements where the two sit on opposite sides of a = b do not count as differences.
L1_SIGN = None


def l1_mean(a, b):
    """mean |a - b| (nn.L1Loss), or mean(s * (a - b)) with s = L1_SIGN(a, b) when a sign source is set."""
    if L1_SIGN is None:
        return torch.mean(torch.abs(a - b))
    return torch.mean(L1_SIGN(a.detach(), b.detach()) * (a - b))


def masked_l1(inp, target, mask):
    """MaskedL1Loss.forward (networks.py:809-812): L1 over input*mask vs target*mask, mask broadcast over channels,
    averaged over ALL elements (masked-out pixels count as zeros, they are not excluded from the mean)."""
    m = mask.expand(-1, inp.size(1), -1, -1)
    return l1_mean(inp * m, target * m)


def gan_and_fm_loss(pred_real, pred_fake, *, n_layers_D=3, num_D=2, lambda_feat=10.0, no_ganFeat=False):
    """GAN_and_FM_loss (vid2vid_model_D.py:199-213): generator LSGAN term on the fake predictions plus the discriminator
    feature-matching term: L1 between every intermediate feature map (all but the last output) of each tower, weighted
    4 / (n_layers_D + 1) * 1 / num_D * lambda_feat."""
    g_gan = gan_loss(pred_fake, True)
    fm = torch.zeros_like(g_gan)
    if not no_ganFeat:
        w = (4.0 / (n_layers_D + 1)) * (1.0 / num_D) * lambda_feat
        for i in range(min(len(pred_fake), num_D)):
            for j in range(len(pred_fake[i]) - 1):
                fm = fm + w * l1_mean(pred_fake[i][j], pred_real[i][j])
    return g_gan, fm


def discriminator_losses(sd, real_cond, real_img, fake_img, *, num_D=2, n_layers_D=3, norm='batch', lambda_feat=10.0,
                         no_ganFeat=False):
    """compute_loss_D (vid2vid_model_D.py:166-177): the towers see (condition, image) stacked along channels.  Forward
    values only: the reference's second fake pass differs from the first by .detach(), not numerically -- but with batch
    norm in train mode each call updates running statistics, which do not feed the outputs."""
    d = dict(num_D=num_D, n_layers=n_layers_D, norm=norm, getIntermFeat=True)
    cat = (lambda a, b: torch.cat((a, b), 1)) if real_cond is not None else (lambda a, b: b)
    pred_real = GO.multiscale_discriminator(sd, cat(real_cond, real_img), **d)
    pred_fake = GO.multiscale_discriminator(sd, cat(real_cond, fake_img), **d)
    g_gan, fm = gan_and_fm_loss(pred_real, pred_fake, n_layers_D=n_layers_D, num_D=num_D, lambda_feat=lambda_feat,
                                no_ganFeat=no_ganFeat)
    return gan_loss(pred_real, True), gan_loss(pred_fake, False), g_gan, fm


def spatial_losses(sd_D, real_B, fake_B, fake_B_raw, real_A, real_B_prev, fake_B_prev, flow, weight, flow_ref, conf_ref, *,
                   lambda_F=10.0, lambda_T=10.0, lambda_feat=10.0, n_scales_spatial=1, no_first_img=False, num_D=2,
                   n_layers_D=3, norm='batch', no_ganFeat=False, align_corners=False):
    """Vid2VidModelD.forward for scale_T == 0 (vid2vid_model_D.py:117-164), --no_vgg, no face discriminator.  Returns the
    reference's loss_list order: [G_VGG, G_GAN, G_GAN_Feat, D_real, D_fake, G_Warp, F_Flow, F_Warp, W], each (1, 1)."""
    if flow is not None:
        f_flow = masked_l1(flow, flow_ref, conf_ref) * lambda_F / (2 ** (n_scales_spatial - 1))
        # the real previous frame warped by the PREDICTED flow should land on the real current frame
        f_warp = masked_l1(GO.resample(real_B_prev, flow, align_corners), real_B, conf_ref) * lambda_T
        w_loss = torch.zeros_like(weight)
        if no_first_img:
            w_loss = masked_l1(weight, torch.zeros_like(weight), conf_ref)
    else:
        f_flow = f_warp = w_loss = torch.zeros_like(conf_ref)
    g_vgg = torch.zeros_like(w_loss)
    kw = dict(num_D=num_D, n_layers_D=n_layers_D, norm=norm, lambda_feat=lambda_feat, no_ganFeat=no_ganFeat)
    d_real, d_fake, g_gan, g_fm = discriminator_losses(sd_D, real_A, real_B, fake_B, **kw)
    # the generated frame should agree with the previous GENERATED frame warped by the REFERENCE flow
    g_warp = masked_l1(fake_B, GO.resample(fake_B_prev, flow_ref, align_corners), conf_ref) * lambda_T
    if fake_B_raw is not None:
        r = discriminator_losses(sd_D, real_A, real_B, fake_B_raw, **kw)
        d_real, d_fake, g_gan, g_fm = d_real + r[0], d_fake + r[1], g_gan + r[2], g_fm + r[3]
    return [t.reshape(-1, 1) for t in (g_vgg, g_gan, g_fm, d_real, d_fake, g_warp, f_flow, f_warp, w_loss)]


def temporal_losses(sd_DT, real_B, fake_B, flow_ref, conf_ref, *, n_frames_D=3, output_nc=3, lambda_feat=10.0, num_D=2,
                    n_layers_D=3, norm='batch', no_ganFeat=False):
    """Vid2VidModelD.forward for scale_T > 0 -> compute_loss_D_T (vid2vid_model_D.py:103-115,179-197): the temporal
    towers see n_frames_D consecutive frames stacked along channels, followed by the n_frames_D - 1 reference flows
    (divided by 20 by the caller in the reference; done here).  Returns [G_T_GAN, G_T_GAN_Feat, D_T_real, D_T_fake,
    G_T_Warp (always zero)]."""
    h, w = real_B.shape[-2:]
    real = real_B.reshape(-1, output_nc * n_frames_D, h, w)
    fake = fake_B.reshape(-1, output_nc * n_frames_D, h, w)
    if flow_ref is not None:
        fl = (flow_ref / 20).reshape(-1, 2 * (n_frames_D - 1), h, w)
        real, fake = torch.cat((real, fl), 1), torch.cat((fake, fl), 1)
    d_real, d_fake, g_gan, g_fm = discriminator_losses(sd_DT, None, real, fake, num_D=num_D, n_layers_D=n_layers_D, norm=norm,
                                                       lambda_feat=lambda_feat, no_ganFeat=no_ganFeat)
    return [t.reshape(-1, 1) for t in (g_gan, g_fm, d_real, d_fake, torch.zeros_like(g_gan))]
