"""CPU: where a training step's gradient is cut (vid2vid_model_G.py:167-168 and :181-186).  The detach-aware oracle
(oracle/bptt_oracle.py) against the unmodified reference's parameter gradients (tests/golden/bptt.npz) and against the plain
oracle, and Vid2VidModelG.init_train's frame budget and optimizer (vid2vid_model_G.py:57-84)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import bptt_oracle as BO
from oracle.bptt_oracle import BPTTModelGOracle
from vid2vid_b200 import networks
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.utils import det_fill_, make_opt, synth_label_sequence


def _opt(**kw):
    base = dict(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=2, ngf=16, n_downsample_G=2, n_blocks=4,
                n_blocks_local=2, isTrain=True, gpu_ids=[0], n_frames_total=12, max_frames_per_gpu=2, max_frames_backpropagate=2)
    base.update(kw)
    return make_opt(**base)


def _case(H=32, W=64, seed=3):
    opt = _opt()
    nets = [det_fill_(networks.build_netG(opt, s), seed=seed + s) for s in range(2)]
    T = opt.n_frames_G + 1                                               # two generated frames
    A = synth_label_sequence(T, H, W, label_nc=35, block=8, seed=seed)
    B = torch.rand(1, T, 3, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    return opt, nets, A, B


def _grads(opt, nets, A, B, frames=(0, 1), **kw):
    """Parameter gradients of a random-cotangent objective over the outputs of `frames` (zero where none arrives)."""
    sds = [{k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
            for k, v in n.state_dict().items()} for n in nets]
    out = BPTTModelGOracle(opt, sds).train_forward(A, B, A, None, n_frames_load=2, **kw)
    g = torch.Generator().manual_seed(11)
    J = sum((o[:, list(frames)] * torch.randn(o[:, list(frames)].shape, generator=g)).sum() for o in out[:4])
    J.backward()
    return out, {'%d.%s' % (s, k): v.grad if v.grad is not None else torch.zeros_like(v) for s in range(2)
                 for k, v in sds[s].items() if v.requires_grad}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bptt.npz')


def _fixture_case_grads(n_frames_bp, finetune_all):
    """The oracle on the recipe's case: parameter gradients of its objective, only where a gradient arrives."""
    opt = BO.case_opt()
    A, B = BO.case_inputs(opt)
    sds = [{k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and k.split('.')[-1] in ('weight', 'bias'))
            for k, v in BO.condition(det_fill_(networks.build_netG(opt, s), seed=BO.G_SEEDS[s])).state_dict().items()}
           for s in range(2)]
    out = BPTTModelGOracle(opt, sds).train_forward(A, B, A, None, n_frames_load=2, n_frames_bp=n_frames_bp, finetune_all=finetune_all)
    outs = list(out[:4])
    sum((o * c).sum() for o, c in zip(outs, BO.cotangents(outs))).backward()
    return {'%d.%s' % (s, k): v.grad for s in range(2) for k, v in sds[s].items() if v.grad is not None}


@pytest.mark.parametrize('variant', list(BO.VARIANTS))
def test_detach_points_match_the_reference(variant):
    gold = np.load(GOLD)
    ref = {k[len(variant) + 1:]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith(variant + '/')}
    ours = _fixture_case_grads(*BO.VARIANTS[variant])
    assert set(ours) == set(ref)                  # fixed_global: no gradient reaches netG0 in either
    for k, r in ref.items():
        scale = max(1.0, r.abs().max().item())
        assert (ours[k] - r).abs().max().item() <= 2e-4 * scale, (k, (ours[k] - r).abs().max().item(), scale)
    if variant == 'bp2':                          # the fixture tells the cut apart: without it frame 1 reaches frame 0
        cut = _fixture_case_grads(1, True)
        for s in range(2):
            rels = sorted(_rel(cut.get(k, torch.zeros_like(r)), r) for k, r in ref.items() if k.startswith('%d.' % s) and r.norm() > 0)
            assert rels[len(rels) // 2] > 0.1, (s, rels[len(rels) // 2])


def test_golden_regenerates_byte_identical(tmp_path):
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip('no reference tree (oracle/_ref or V2V_REFERENCE_ROOT)')
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
    subprocess.run([sys.executable, '-m', 'oracle.bptt_oracle', str(tmp_path)], cwd=root, check=True, capture_output=True)
    with open(GOLD, 'rb') as a, open(str(tmp_path / 'bptt.npz'), 'rb') as b:
        assert a.read() == b.read()
    assert os.path.getsize(GOLD) < 1 << 20


def test_detach_points_leave_the_forward_and_the_default_graph_unchanged():
    opt, nets, A, B = _case()
    sds = [{k: v.detach().clone() for k, v in n.state_dict().items()} for n in nets]
    from oracle import generator_oracle as GO
    with torch.no_grad():
        ref = GO.ModelGOracle(opt, sds).train_forward(A, B, A, None, n_frames_load=2)
        for kw in ({}, dict(n_frames_bp=1), dict(n_frames_bp=2, finetune_all=False)):
            ours = BPTTModelGOracle(opt, sds).train_forward(A, B, A, None, n_frames_load=2, **kw)
            for o, r in zip(ours[:6], ref[:6]):
                assert torch.equal(o, r), kw
    # with two frames per step, n_frames_bp = 2 cuts nothing: the same gradients as no detach point at all
    _, g_none = _grads(opt, nets, A, B)
    _, g_bp2 = _grads(opt, nets, A, B, n_frames_bp=2)
    for k in g_none:
        assert torch.equal(g_none[k], g_bp2[k]), k


def test_previous_frame_gradient_flows_only_past_the_cut():
    opt, nets, A, B = _case()
    _, g1 = _grads(opt, nets, A, B, n_frames_bp=1)
    _, g2 = _grads(opt, nets, A, B, n_frames_bp=2)
    # frame 0's own outputs do not see the cut ...
    _, f1 = _grads(opt, nets, A, B, frames=(0,), n_frames_bp=1)
    _, f2 = _grads(opt, nets, A, B, frames=(0,), n_frames_bp=2)
    for k in f1:
        assert torch.allclose(f1[k], f2[k], rtol=1e-5, atol=1e-7), k
    # ... frame 1's reach frame 0's generator at both scales only without it
    rels = sorted(_rel(g1[k], g2[k]) for k in g2 if g2[k].norm() > 1e-6 * max(v.norm() for v in g2.values()))
    print('n_frames_bp 1 vs 2: median rel L2 %.3f, max %.3f over %d tensors' % (rels[len(rels) // 2], rels[-1], len(rels)))
    assert rels[len(rels) // 2] > 0.1
    for s in range(2):
        assert max(_rel(g1[k], g2[k]) for k in g2 if k.startswith('%d.' % s) and g2[k].norm() > 0) > 0.1, s


def test_fixed_global_scales_get_no_gradient_and_the_finest_scale_is_unchanged():
    opt, nets, A, B = _case()
    _, ga = _grads(opt, nets, A, B, n_frames_bp=2)
    _, gf = _grads(opt, nets, A, B, n_frames_bp=2, finetune_all=False)
    for k in ga:
        if k.startswith('0.'):
            assert not gf[k].any(), k
        else:
            assert torch.allclose(gf[k], ga[k], rtol=1e-5, atol=1e-8), k


def _model(**kw):
    m = Vid2VidModelG()
    m.opt = _opt(**kw)
    m.n_scales = 2
    for s in range(2):
        setattr(m, 'netG%d' % s, networks.build_netG(m.opt, s))
    return m.init_train()


def test_init_train_starts_at_one_backpropagated_frame_and_fixes_the_global_scales():
    m = _model()
    assert (m.n_frames_bp, m.n_frames_per_gpu, m.n_frames_load, m.finetune_all) == (1, 2, 2, True)
    ids = lambda opt_: [id(p) for g in opt_.param_groups for p in g['params']]
    all_ids = lambda m: sorted(id(p) for s in range(2) for p in getattr(m, 'netG%d' % s).parameters())
    assert sorted(ids(m.optimizer_G)) == all_ids(m)
    for ttur in (False, True):
        m = _model(niter_fix_global=1, TTUR=ttur)
        assert not m.finetune_all
        assert ids(m.optimizer_G) == [id(p) for p in m.netG1.parameters()]                 # the finest scale only (:72-77)
        assert m.optimizer_G.param_groups[0]['betas'] == ((0, 0.9) if ttur else (0.5, 0.999))
        assert m.optimizer_G.param_groups[0]['lr'] == (m.opt.lr / 2 if ttur else m.opt.lr)
        m.update_training_batch(1)
        assert m.n_frames_bp == 2
        m.update_fixed_params()
        assert m.finetune_all and sorted(ids(m.optimizer_G)) == all_ids(m)
