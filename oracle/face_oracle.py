"""TEST INFRASTRUCTURE -- not product code (only tests/ and tools/ may import oracle/).

CPU restatement of the edge2face first-frame generator (models/vid2vid_model_G.py:231-320) and the recipe that pins it
against the unmodified reference.

    encoder(sd, x, inst)                    Encoder.forward (models/networks.py:595-632): conv stack + instance-wise mean
    face_features(pooled, inst, features)   get_face_features + dists_min (vid2vid_model_G.py:290-320, base_model.py:136-144)
                                            with labels absent from the part map contributing nothing to the distance
    global_with_z(sd, x, z)                 Global_with_z.forward (models/networks.py:421-467)

All run in the inputs' dtype (fp32 or fp64); the instance means and the distances are taken in fp64.

    python -m oracle.face_oracle [OUT_DIR]  # writes face_keys.json and face_*.npz (default tests/golden/)

The recipe runs the reference's own define_G(..., 'encoder' | 'global_with_features') modules and Vid2VidModelG's
get_face_features / inference on the CPU through ref_shim, with det_fill_ weights and a seeded synthetic features.npy written
into a temporary working directory (the reference reads the relative path checkpoints/edge2face_single/features.npy).  Two
harness shims, neither touching arithmetic: np.load gets allow_pickle=True (current numpy refuses to unpickle the dict
otherwise), and load_single_G is stubbed to return the seeded Global_with_z with netE set.  ref_shim's shims are
process-wide: run the recipe in its own process (tests/test_face_oracle.py does).
"""
import contextlib
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle.generator_oracle import _norm, _conv, _deconv, _resblock      # noqa: E402
from vid2vid_b200.utils import make_opt, det_fill_                        # noqa: E402

N_LABELS, FEAT_NUM = 7, 16
SEED = 41
# fixtures: the Encoder / lookup / Global_with_z case at 256x256, the inference case at 128x128
SIZE, INFER_SIZE = 256, 128
NUM_IMAGES = 24                      # rows of the synthetic features table
GZ_CFG = dict(ngf=32, n_blocks=3)    # Global_with_z of the 256x256 case (528 -> 272 channels keeps the CPU run short)
INFER_CFG = dict(ngf=16, n_blocks=2, n_frames=3)


# ----------------------------------------------------------------------------- restatement
def _stem(x, sd, p, kind='instance'):
    return F.relu(_norm(_conv(F.pad(x, (3, 3, 3, 3), mode='reflect'), sd, p + '.1'), sd, p + '.2', kind))


def _conv_stack(x, sd, p, i, n_down, n_up, kind='instance'):
    """n_down [Conv3x3 s2, norm, ReLU] then n_up [ConvTranspose3x3 s2, norm, ReLU] starting at index i of Sequential p."""
    for _ in range(n_down):
        x = F.relu(_norm(_conv(x, sd, '%s.%d' % (p, i), stride=2, padding=1), sd, '%s.%d' % (p, i + 1), kind))
        i += 3
    for _ in range(n_up):
        x = F.relu(_norm(_deconv(x, sd, '%s.%d' % (p, i)), sd, '%s.%d' % (p, i + 1), kind))
        i += 3
    return x, i


def _cast(sd, dtype):
    return {k: v.to(dtype) for k, v in sd.items()}


def instance_mean(out, inst):
    """networks.py:617-632 with the per-instance means taken in fp64."""
    res = out.clone()
    ids = inst.round().long()
    for b in range(out.shape[0]):
        for i in torch.unique(ids[b]).tolist():
            m = (ids[b, 0] == i)
            for j in range(out.shape[1]):
                res[b, j][m] = out[b, j][m].double().mean().to(out.dtype)
    return res


def encoder(sd, x, inst, n_downsampling=4, pool=True):
    sd = _cast(sd, x.dtype)
    h = _stem(x, sd, 'model')
    h, i = _conv_stack(h, sd, 'model', 4, n_downsampling, n_downsampling)
    h = torch.tanh(_conv(F.pad(h, (3, 3, 3, 3), mode='reflect'), sd, 'model.%d' % (i + 1)))
    return instance_mean(h, inst) if pool else h


def first_pixels(inst):
    """{label: (n, y, x) of its first pixel in flat (n, y, x) order} (idx[0] of (inst == label).nonzero())."""
    ids = inst.round().long()[:, 0]
    out = {}
    for label in torch.unique(ids).tolist():
        n, y, x = (ids == label).nonzero()[0].tolist()
        out[label] = (n, y, x)
    return out


def face_dists(pooled, inst, features, feat_num=FEAT_NUM):
    """dists[m] in fp64 over the labels present (vid2vid_model_G.py:297-309, base_model.py:136-137), num_images = rows of 6."""
    num_images = features[6].shape[0]
    d = torch.zeros(num_images, dtype=torch.float64)
    for label, (n, y, x) in first_pixels(inst).items():
        ori = pooled[n, :feat_num, y, x].double()
        ref = torch.as_tensor(np.asarray(features[label])[:num_images, :feat_num], dtype=torch.float64)
        d += ((ori[None, :] - ref) ** 2).sum(1)
    return d


def paint(inst, features, chosen, feat_num=FEAT_NUM, dtype=torch.float32):
    """vid2vid_model_G.py:312-318: every pixel gets its label's row min(chosen, rows - 1), first feat_num columns."""
    ids = inst.round().long()
    N, _, H, W = inst.shape
    out = torch.zeros(N, feat_num, H, W, dtype=dtype)
    for label in torch.unique(ids).tolist():
        f = torch.as_tensor(np.asarray(features[label])[:, :-1], dtype=dtype)
        row = f[min(chosen, f.shape[0] - 1), :feat_num]
        m = (ids == label).expand(N, feat_num, H, W)
        out[m] = row[None, :, None, None].expand(N, feat_num, H, W)[m]
    return out


def face_features(pooled, inst, features, feat_num=FEAT_NUM):
    """(feat_map, chosen, dists)."""
    d = face_dists(pooled, inst, features, feat_num)
    chosen = int(torch.argmin(d).item())          # torch.argmin returns the first minimum
    return paint(inst, features, chosen, feat_num, pooled.dtype), chosen, d


def global_with_z(sd, x, z, n_downsample_G=3, n_blocks=9):
    sd = _cast(sd, x.dtype)
    z_down = z
    for _ in range(n_downsample_G):
        z_down = F.avg_pool2d(z_down, 3, 2, 1, count_include_pad=False)
    h = _stem(torch.cat([x, z], 1), sd, 'model_downsample')
    h, _ = _conv_stack(h, sd, 'model_downsample', 4, n_downsample_G, 0)
    h = torch.cat([h, z_down], 1)
    for b in range(n_blocks):
        h = _resblock(h, sd, 'model_resnet.%d' % b, 'instance')
    h, _ = _conv_stack(torch.cat([h, z_down], 1), sd, 'model_upsample', 0, 0, n_downsample_G)
    return torch.tanh(_conv(F.pad(torch.cat([h, z], 1), (3, 3, 3, 3), mode='reflect'), sd, 'model_upsample_conv.1'))


# ----------------------------------------------------------------------------- seeded inputs
def part_map(n_frames, H, W, seed):
    """(1, n_frames, 1, H, W) float part labels 0..6 in 16-pixel blocks, every label present in every frame (a band of
    the seven labels along the top rows), drifting by one block per frame."""
    from vid2vid_b200.utils import synth_label_sequence
    lab = synth_label_sequence(n_frames, H, W, label_nc=N_LABELS, block=16, seed=seed)
    for label in range(N_LABELS):
        lab[..., :16, 16 * label:16 * (label + 1)] = float(label)
    return lab


def real_images(n_frames, H, W, seed):
    """(1, n_frames, 3, H, W) low-pass images in [-1, 1]."""
    g = torch.Generator().manual_seed(seed + 3)
    coarse = torch.rand(n_frames, 3, H // 16, W // 16, generator=g) * 2 - 1
    return F.interpolate(coarse, size=(H, W), mode='bilinear', align_corners=False).unsqueeze(0)


def edge_maps(n_frames, H, W, seed, nc=15):
    """(1, n_frames, nc, H, W) sparse 0/1 maps standing in for the face edge channels."""
    g = torch.Generator().manual_seed(seed + 5)
    return (torch.rand(1, n_frames, nc, H, W, generator=g) < 0.1).float()


def synthetic_features(seed=SEED, num_images=NUM_IMAGES):
    from vid2vid_b200.networks import synthetic_face_features
    return synthetic_face_features(num_images, FEAT_NUM, seed)


def face_opt(**kw):
    o = dict(dataset_mode='face', dataroot='datasets/face/', label_nc=0, input_nc=15, use_single_G=True, feat_num=FEAT_NUM,
             ngf=INFER_CFG['ngf'], n_blocks=INFER_CFG['n_blocks'], n_frames_G=3, gpu_ids=[], use_instance=False, fg=False)
    o.update(kw)
    return make_opt(**o)


def encoder_state(module):
    return det_fill_(module, seed=SEED + 1)


def gz_state(module):
    return det_fill_(module, seed=SEED + 2)


def infer_seeds():
    return dict(netE=SEED + 11, netG_i=SEED + 12, netG0=SEED + 13)


def condition(m):
    """Shrink the flow heads of netG0 as the street inference case does (tests/cases.condition_flow_heads)."""
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import cases
    cases.condition_flow_heads(m.netG0, 0.05)


# ----------------------------------------------------------------------------- recipe
@contextlib.contextmanager
def _features_dir(features):
    import tempfile
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, 'checkpoints', 'edge2face_single'))
        np.save(os.path.join(tmp, 'checkpoints', 'edge2face_single', 'features.npy'), features, allow_pickle=True)
        os.chdir(tmp)
        orig = np.load
        np.load = lambda *a, **k: orig(*a, **dict(k, allow_pickle=True))
        try:
            yield
        finally:
            np.load = orig
            os.chdir(cwd)


def chosen_of(feat_map, inst, features):
    """The row index the reference painted (recovered from its feature map at label 0's first pixel)."""
    n, y, x = first_pixels(inst)[0]
    v = feat_map[n, :, y, x].double()
    rows = torch.as_tensor(np.asarray(features[0])[:, :FEAT_NUM], dtype=torch.float64)
    hit = ((rows - v[None]).abs().max(1).values == 0).nonzero()
    return int(hit[0, 0])


def make_golden(out_dir=os.path.join(ROOT, 'tests', 'golden')):
    import json
    from oracle import ref_shim
    RN = ref_shim.networks()
    written = []
    torch.manual_seed(0)
    opt_full = face_opt(n_blocks=9)
    keys = {'encoder': RN.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []),
            'global_with_z': RN.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt_full)}
    path = os.path.join(out_dir, 'face_keys.json')
    with open(path, 'w') as f:
        json.dump({k: [[n, list(v.shape)] for n, v in m.state_dict().items()] for k, m in keys.items()}, f)
        f.write('\n')
    written.append(path)

    features = synthetic_features()
    out = {}
    with torch.no_grad(), _features_dir(features):
        # Encoder + nearest-neighbour lookup at 256x256
        netE = encoder_state(RN.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []))
        B = real_images(1, SIZE, SIZE, SEED)[:, 0]
        inst = part_map(1, SIZE, SIZE, SEED)[:, 0]
        pooled = netE(B, inst)
        out['pooled_means'] = np.stack([pooled[0, :, y, x].numpy() for _, (n, y, x) in sorted(first_pixels(inst).items())])
        out['pooled_sub'] = pooled[:, :, ::16, ::16].numpy()
        m = ref_shim.make_model_G(face_opt(), None)
        m.netE = netE
        feat_map = m.get_face_features(B, inst)
        out['chosen'] = np.int64(chosen_of(feat_map, inst, features))
        out['feat_sub'] = feat_map[:, :, ::8, ::8].numpy()
        # Global_with_z at 256x256 on the painted features
        opt = face_opt(**GZ_CFG)
        gz = gz_state(RN.define_G(15, 3, 0, GZ_CFG['ngf'], 'global_with_features', 3, 'instance', 0, [], opt))
        x = edge_maps(1, SIZE, SIZE, SEED)[:, 0]
        out['gz_out'] = gz(x, feat_map).numpy()
    path = os.path.join(out_dir, 'face_256.npz')
    np.savez_compressed(path, **out)
    written.append(path)

    # Vid2VidModelG.inference in face mode: the first call builds the two first frames with the single-image generator
    out = {}
    H = W = INFER_SIZE
    nF = INFER_CFG['n_frames'] + 2
    A, Bs, I = edge_maps(nF, H, W, SEED + 20), real_images(nF, H, W, SEED + 20), part_map(nF, H, W, SEED + 20)
    with torch.no_grad(), _features_dir(features):
        torch.manual_seed(0)
        opt = face_opt()
        seeds = infer_seeds()
        single = det_fill_(RN.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt), seed=seeds['netG_i'])
        m = ref_shim.make_model_G(opt, single)
        m.netE = det_fill_(RN.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []), seed=seeds['netE'])
        det_fill_(m.netG0, seed=seeds['netG0'])
        condition(m)
        firsts, chosen = [], []
        orig_gff, orig_gf = m.generate_first_frame, m.get_face_features

        def gff(*a, **k):
            r = orig_gff(*a, **k)
            firsts.append(r[0].clone())
            return r

        def gf(real_image, inst):
            r = orig_gf(real_image, inst)
            chosen.append(chosen_of(r, inst, features))
            return r
        m.generate_first_frame, m.get_face_features = gff, gf
        for t in range(INFER_CFG['n_frames']):
            fake_B, _ = m.inference(A[:, t:t + 3], Bs[:, t:t + 3], I[:, t:t + 3])
            out['fake_B_%d' % t] = fake_B.numpy()
    out['first_frames'] = firsts[0].numpy()
    out['first_chosen'] = np.asarray(chosen, dtype=np.int64)
    path = os.path.join(out_dir, 'face_infer.npz')
    np.savez_compressed(path, **out)
    written.append(path)
    return written


if __name__ == '__main__':
    for p in make_golden(*sys.argv[1:2]):
        print(p)
