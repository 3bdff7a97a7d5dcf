"""Seeded synthetic cases shared by oracle/make_golden.py (which runs the *reference* on them
and writes tests/golden/<case>.npz) and by the parity tests (which rebuild the same weights
and inputs from the seeds and compare the oracle / the CUDA path with the stored outputs).

Weights never travel: `det_fill_` regenerates them from (seed, parameter name, shape)."""
import os

import numpy as np
import torch

from vid2vid_b200.utils import make_opt, synth_label_sequence

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def load_golden(name):
    """{key: array} of the fixture tests/golden/<name>.npz and its parts <name>_2.npz, <name>_3.npz, ... (files are kept
    under 1 MB: oracle/make_golden.py splits larger fixtures by array)."""
    out, k, path = {}, 1, os.path.join(GOLD, name + '.npz')
    while os.path.exists(path):
        with np.load(path) as z:
            out.update({key: z[key] for key in z.files})
        k += 1
        path = os.path.join(GOLD, '%s_%d.npz' % (name, k))
    assert out, 'no fixture %s' % name
    return out

GEN_OUT_NAMES = ['img_final', 'flow', 'weight', 'img_raw', 'img_feat', 'flow_feat', 'img_fg_feat']


def onehot_input(label_nc, h, w, seed, block=4, n_frames=3):
    """(1, n_frames*(label_nc+1), h, w) one-hot + edge input, plus the label sequence."""
    lab = synth_label_sequence(n_frames, h, w, label_nc=label_nc, block=block, seed=seed)
    oh = torch.zeros(1, n_frames, label_nc, h, w)
    oh.scatter_(2, lab.long(), 1.0)
    t = lab
    edge = torch.zeros(t.size(), dtype=torch.bool)
    edge[..., :, 1:] |= (t[..., :, 1:] != t[..., :, :-1])
    edge[..., :, :-1] |= (t[..., :, 1:] != t[..., :, :-1])
    edge[..., 1:, :] |= (t[..., 1:, :] != t[..., :-1, :])
    edge[..., :-1, :] |= (t[..., 1:, :] != t[..., :-1, :])
    real_A = torch.cat([oh, edge.float()], dim=2)
    return real_A.view(1, -1, h, w), lab


def gen_inputs(label_nc, h, w, seed, fg_label=2, block=4):
    g = torch.Generator().manual_seed(seed + 77)
    inp, lab = onehot_input(label_nc, h, w, seed, block)
    # low-pass noise (SURVEY 8d): coarse U(-1,1) field, bilinearly upsampled
    coarse = torch.rand(1, 6, max(2, h // 8), max(2, w // 8), generator=g) * 2 - 1
    img_prev = torch.nn.functional.interpolate(coarse, size=(h, w), mode='bilinear', align_corners=False)
    mask = (lab[:, -1] == fg_label).float()
    return inp, img_prev, mask


# name -> dict(kind, args...) ; every entry is a reference forward whose outputs are stored.
CASES = {
    # CompositeGenerator, full structure (nd 3, 9 blocks, fg) at toy width
    'g0_small': dict(kind='composite', label_nc=35, ngf=16, nd=3, n_blocks=9, fg=True, no_flow=False,
                     h=32, w=64, seed=11),
    'g0_small_ac': dict(kind='composite', label_nc=35, ngf=16, nd=3, n_blocks=9, fg=True, no_flow=False,
                        h=32, w=64, seed=11, align_corners=True),
    'g0_nofg_nd2': dict(kind='composite', label_nc=5, ngf=32, nd=2, n_blocks=4, fg=False, no_flow=False,
                        h=24, w=40, seed=12),
    'g0_noflow': dict(kind='composite', label_nc=5, ngf=16, nd=3, n_blocks=3, fg=True, no_flow=True,
                      h=32, w=32, seed=13),
    # CompositeLocalGenerator scale 1 / 2
    'gl_small_s1': dict(kind='compositeLocal', label_nc=35, ngf=16, nd=3, n_blocks_local=3, fg=True,
                        scale=1, h=32, w=64, seed=14),
    'gl_small_s2': dict(kind='compositeLocal', label_nc=5, ngf=8, nd=3, n_blocks_local=2, fg=True,
                        scale=2, h=48, w=80, seed=15),
    # first-frame generators (InstanceNorm)
    'global_small': dict(kind='global', input_nc=35, ngf=16, nd=3, n_blocks=4, h=32, w=64, seed=16),
    'local_small': dict(kind='local', input_nc=35, ngf=8, nd=3, n_blocks=3, n_blocks_local=3,
                        h=64, w=64, seed=17),
    # discriminator towers
    'D_small': dict(kind='D', input_nc=39, ndf=16, n_layers=3, num_D=3, batch=2, h=64, w=96, seed=18),
    # BASELINE config 1: full-width CompositeGenerator forward at 256x128 (W x H)
    'cfg1': dict(kind='composite', label_nc=35, ngf=128, nd=3, n_blocks=9, fg=True, no_flow=False,
                 h=128, w=256, seed=21, block=8, subsample=8),
    # Vid2VidModelG.inference, 3 scales, --fg --use_single_G, 4 generated frames
    'infer_s3': dict(kind='inference', label_nc=35, ngf=16, nd=2, n_blocks=4, n_blocks_local=2,
                     n_scales=3, h=128, w=256, n_gen=4, seed=31, flow_weight_scale=0.05),
}


def inference_opt(c):
    return make_opt(label_nc=c['label_nc'], use_instance=True, fg=True, fg_labels=[2],
                    n_scales_spatial=c['n_scales'], ngf=c['ngf'], n_blocks=c['n_blocks'],
                    n_blocks_local=c['n_blocks_local'], use_single_G=True, n_downsample_G=c['nd'],
                    gpu_ids=[], dataroot='City')


def build_module(c):
    """Our (vid2vid_b200.networks) module for a case, constructed like the reference constructs its own
    in oracle/make_golden.py."""
    from vid2vid_b200 import networks as NW
    kind = c['kind']
    if kind in ('composite', 'compositeLocal'):
        nc = 3 * (c['label_nc'] + 1)
        opt = make_opt(ngf=c['ngf'], n_blocks=c.get('n_blocks', 9), n_blocks_local=c.get('n_blocks_local', 3),
                       fg=c['fg'], no_flow=c.get('no_flow', False), n_downsample_G=c['nd'], gpu_ids=[])
        return NW.define_G(nc, 3, 6, c['ngf'], kind, c['nd'], 'batch', c.get('scale', 0), [], opt)
    if kind in ('global', 'local'):
        opt = make_opt(n_blocks=c['n_blocks'], n_blocks_local=c.get('n_blocks_local', 3), gpu_ids=[])
        return NW.define_G(c['input_nc'], 3, 0, c['ngf'], kind, c['nd'], 'instance', 0, [], opt)
    if kind == 'D':
        return NW.define_D(c['input_nc'], c['ndf'], c['n_layers'], 'batch', c['num_D'], True, [])
    raise ValueError(kind)


# module configurations whose state_dict key/shape lists are pinned in tests/golden/state_dict_keys.json
KEY_CASES = {
    'G0_street': dict(kind='composite', label_nc=35, ngf=128, nd=3, n_blocks=9, fg=True, no_flow=False),
    'G1_street': dict(kind='compositeLocal', label_nc=35, ngf=64, nd=3, n_blocks_local=3, fg=True, scale=1),
    'G2_street': dict(kind='compositeLocal', label_nc=35, ngf=32, nd=3, n_blocks_local=3, fg=True, scale=2),
    'G0_noflow_nofg': dict(kind='composite', label_nc=5, ngf=16, nd=2, n_blocks=5, fg=False, no_flow=True),
    'single_512': dict(kind='global', input_nc=35, ngf=64, nd=3, n_blocks=9),
    'single_2048': dict(kind='local', input_nc=35, ngf=32, nd=4, n_blocks=9, n_blocks_local=3),
    'D_img': dict(kind='D', input_nc=39, ndf=64, n_layers=3, num_D=3),
}


def condition_flow_heads(net, scale):
    """Random N(0,0.02) flow heads times the x20*2^s output scale give noise-like multi-pixel flows, which turn the
    warp into an error amplifier no trained model has; the inference case shrinks the flow-head weights instead."""
    import torch
    with torch.no_grad():
        if hasattr(net, 'model_final_flow'):
            net.model_final_flow[1].weight.mul_(scale)
            net.model_final_flow[1].bias.mul_(scale)
