"""TEST INFRASTRUCTURE -- not product code (only tests/ and tools/ may import oracle/).

The generator oracle's training forward with the reference's two detach points, and the recipe that pins them against the
unmodified reference:

    BPTTModelGOracle.train_forward(..., n_frames_bp=None, finetune_all=True)
        vid2vid_model_G.py:167-168: frame t's previous frames are detached when t % n_frames_bp == 0 (None: never, the
        graph of GO.ModelGOracle.train_forward); :181-186: with finetune_all=False every scale but the finest has its
        outputs detached.  Forward values do not depend on either.

    python -m oracle.bptt_oracle [OUT_DIR]   # writes bptt.npz (default tests/golden/)

The recipe runs the reference's own Vid2VidModelG.forward (training, two scales, --fg, two generated frames per call) on the
CPU through ref_shim with det_fill_ weights, sets n_frames_bp / finetune_all on it as update_training_batch /
initialize do, and stores the parameter gradients of one random-cotangent objective over fake_B, fake_B_raw, flow and
weight for each variant in VARIANTS.  ref_shim's shims are process-wide: run the recipe in its own process.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import generator_oracle as GO                       # noqa: E402
from vid2vid_b200.utils import det_fill_                        # noqa: E402

G_SEEDS = (91, 92)
# name -> (n_frames_bp, finetune_all)
VARIANTS = {'bp2': (2, True), 'fixed_global': (1, False)}


class BPTTModelGOracle(GO.ModelGOracle):
    def train_forward(self, input_A, input_B, inst_A, fake_B_prev=None, n_frames_load=1, n_frames_bp=None, finetune_all=True):
        self._bp, self._finetune_all, self._calls = n_frames_bp, finetune_all, 0
        return super().train_forward(input_A, input_B, inst_A, fake_B_prev, n_frames_load)

    def _generate(self, s, a, prevs, mask, feats, raw_only):
        # the base class calls this once per (frame t, scale s), t-major, with frame t's previous frames of scale s
        t = self._calls // self.n_scales
        self._calls += 1
        if self._bp is not None and t % self._bp == 0:                                   # :167-168
            prevs = prevs.detach()
        out = super()._generate(s, a, prevs, mask, feats, raw_only)
        if s != self.n_scales - 1 and not self._finetune_all:                           # :181-186
            out = tuple(o.detach() if o is not None else None for o in out)
        return out


def _tests_path():
    sys.path.insert(0, os.path.join(ROOT, 'tests'))


def case_opt():
    _tests_path()
    import reference_inputs as RI
    return RI.train_opt(False)


def case_inputs(opt):
    """(A, B): the first training call's clip (two generated frames)."""
    _tests_path()
    import reference_inputs as RI
    seq, real = RI.train_clip(opt)
    return RI.train_call_inputs(seq, real, opt, 0)


def condition(net):
    _tests_path()
    import cases
    cases.condition_flow_heads(net, 0.05)
    return net


def cotangents(outs):
    g = torch.Generator().manual_seed(17)
    return [torch.randn(o.shape, generator=g) for o in outs]


def make_golden(out_dir=os.path.join(ROOT, 'tests', 'golden')):
    from oracle import ref_shim
    opt = case_opt()
    A, B = case_inputs(opt)
    out = {}
    for name, (n_frames_bp, finetune_all) in VARIANTS.items():
        m = ref_shim.make_model_G(opt)
        for s in range(2):
            condition(det_fill_(getattr(m, 'netG%d' % s), seed=G_SEEDS[s]))
        m.n_frames_bp, m.finetune_all = n_frames_bp, finetune_all
        r = m.forward(A, B, A, None)
        outs = list(r[:4])
        sum((o * c).sum() for o, c in zip(outs, cotangents(outs))).backward()
        for s in range(2):
            for k, p in getattr(m, 'netG%d' % s).named_parameters():
                if p.grad is not None:
                    out['%s/%d.%s' % (name, s, k)] = p.grad.numpy()
    path = os.path.join(out_dir, 'bptt.npz')
    np.savez_compressed(path, **out)
    return [path]


if __name__ == '__main__':
    for p in make_golden(*sys.argv[1:2]):
        print(p)
