"""TEST INFRASTRUCTURE -- not product code (only tests/ and tools/ may import oracle/).

CPU restatement of the reference's VGG19 perceptual loss (VGGLoss / Vgg19, models/networks.py:776-791,840-869) and the
recipe that pins it against the unmodified reference.

    vgg_loss(sd, x, y)   sum_k w_k * mean |f_k(x) - f_k(y)|, w = 1/32 .. 1, f_k = relu{k}_1 of VGG19's features, the images
                         halved by a 2x2 mean while wider than 1024 pixels; no ImageNet normalisation (the images go in as
                         they are).  sd: a Vgg19 state_dict (slice keys).  Runs in the inputs' dtype (fp32 or fp64).

    python -m oracle.vgg_oracle [OUT_DIR]   # writes vgg19_keys.json and vgg_*.npz (default tests/golden/)

The recipe runs the reference's own VGGLoss.__init__ / forward and Vgg19 on the CPU, imported through ref_shim (the tree
named by V2V_REFERENCE_ROOT, else oracle/_ref; its shims make .cuda() the identity).  One more shim, applied only while the
reference module is built: torchvision.models.vgg19 returns a weights=None model filled with
vid2vid_b200.networks.vgg19_synthetic_, so nothing is downloaded.  ref_shim's shims are process-wide: run the recipe in its
own process (tests/test_vgg_oracle.py does).
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WEIGHTS = (1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0)
SLICES = ((0, 2), (2, 7), (7, 12), (12, 21), (21, 30))
POOLS = (4, 9, 18, 27)
SEED = 7
# (name, N, H, W): the small case keeps every level but relu5_1 on row tiles; the wide one runs the downsample loop twice
CASES = (('vgg_small', 1, 96, 160), ('vgg_wide', 1, 64, 2080))
N_GRAD_SAMPLES = 4096


def _slice_of(i):
    for k, (a, b) in enumerate(SLICES):
        if a <= i < b:
            return k + 1
    raise KeyError(i)


def features(sd, x):
    """The five relu{k}_1 maps of x."""
    outs = []
    for i in range(30):
        k = _slice_of(i)
        w = sd.get('slice%d.%d.weight' % (k, i))
        if w is not None:
            x = F.conv2d(x, w.to(x.dtype), sd['slice%d.%d.bias' % (k, i)].to(x.dtype), padding=1)
        elif i in POOLS:
            x = F.max_pool2d(x, 2, 2)
        else:
            x = F.relu(x)
        if i + 1 == SLICES[k - 1][1]:
            outs.append(x)
    return outs


def vgg_loss(sd, x, y, weights=WEIGHTS, levels=False):
    while x.size(3) > 1024:
        x, y = F.avg_pool2d(x, 2, 2), F.avg_pool2d(y, 2, 2)
    fx, fy = features(sd, x), features(sd, y)
    per = [torch.mean(torch.abs(a - b.detach())) for a, b in zip(fx, fy)]
    loss = 0
    for w, l in zip(weights, per):
        loss = loss + w * l
    return (loss, per) if levels else loss


def case_inputs(N, H, W, seed=SEED):
    """Seeded image pair in [-1, 1] (as the generator's tanh head produces it)."""
    g = torch.Generator().manual_seed(seed * 7919 + H * 31 + W)
    x = torch.rand((N, 3, H, W), generator=g) * 2 - 1
    y = torch.rand((N, 3, H, W), generator=g) * 2 - 1
    return x, y


def grad_sample_index(numel, seed=SEED):
    g = torch.Generator().manual_seed(seed + numel)
    return torch.randperm(numel, generator=g)[:min(N_GRAD_SAMPLES, numel)].sort().values


def synthetic_state(seed=SEED):
    sys.path.insert(0, ROOT)
    from vid2vid_b200.networks import Vgg19, vgg19_synthetic_
    return vgg19_synthetic_(Vgg19(), seed).state_dict()


def reference_vgg_loss(seed=SEED):
    """The reference's VGGLoss module (unmodified code from oracle/_ref), built on the CPU with seeded weights."""
    import torchvision
    from oracle import ref_shim
    RN = ref_shim.networks()                     # the reference's models/networks.py
    sd = synthetic_state(seed)
    tv_vgg19 = torchvision.models.vgg19             # (RN.models is torchvision.models itself)

    def vgg19(pretrained=False, **kw):
        m = tv_vgg19(weights=None)
        with torch.no_grad():
            for name, t in sd.items():
                _, i, leaf = name.split('.')
                getattr(m.features[int(i)], leaf).copy_(t)
        return m

    saved_vgg = RN.models.vgg19
    RN.models.vgg19 = vgg19
    try:
        crit = RN.VGGLoss(0)
    finally:
        RN.models.vgg19 = saved_vgg
    return crit, sd


def make_golden(out_dir=os.path.join(ROOT, 'tests', 'golden')):
    import json
    crit, _ = reference_vgg_loss()
    written = [os.path.join(out_dir, 'vgg19_keys.json')]
    with open(written[0], 'w') as f:                 # the reference Vgg19's state_dict keys and shapes
        json.dump([[k, list(v.shape)] for k, v in crit.vgg.state_dict().items()], f)
        f.write('\n')
    for name, N, H, W in CASES:
        x, y = case_inputs(N, H, W)
        x = x.clone().requires_grad_(True)
        loss = crit(x, y)
        loss.backward()
        idx = grad_sample_index(x.numel())
        path = os.path.join(out_dir, name + '.npz')
        np.savez(path, loss=np.float32(loss.item()), grad_index=idx.numpy().astype(np.int64),
                 grad=x.grad.reshape(-1)[idx].numpy().astype(np.float32))
        written.append(path)
    return written


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    for p in make_golden(*sys.argv[1:2]):
        print(p)
