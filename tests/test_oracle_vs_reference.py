"""Pins oracle/generator_oracle.py against the unmodified reference: its outputs (and gradients) on seeded inputs are
stored in tests/golden/reference*.npz (oracle/make_golden.py reference_checks); the weights are regenerated here with
det_fill_ on our own modules, whose state_dict keys and shapes equal the reference's (tests/test_oracle_vs_golden.py)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from oracle import generator_oracle as GO                     # noqa: E402
from vid2vid_b200 import networks as NW                        # noqa: E402
from vid2vid_b200.utils import make_opt, det_fill_             # noqa: E402
import cases                                                  # noqa: E402
import reference_inputs as RI                                 # noqa: E402

GOLD = RI.golden()


def _close(a, key, tol=2e-5):
    b = torch.from_numpy(GOLD[key])
    assert a.shape == b.shape, (key, a.shape, b.shape)
    assert (a - b).abs().max().item() <= tol, (key, (a - b).abs().max().item())


def _close_all(prefix, names, outs):
    for n, o in zip(names, outs):
        key = prefix + '/' + n
        assert (o is None) == (key not in GOLD), key
        if o is not None:
            _close(o, key)


@pytest.mark.parametrize('fg,no_flow,nd', RI.COMPOSITE_VARIANTS)
def test_composite_generator(fg, no_flow, nd):
    opt = make_opt(ngf=8, n_blocks=3, fg=fg, no_flow=no_flow, n_downsample_G=nd, gpu_ids=[])
    sd = det_fill_(NW.define_G(18, 3, 6, 8, 'composite', nd, 'batch', 0, [], opt), seed=1).state_dict()
    inp, img_prev, mask = RI.gen_inputs(6, 16, 32)
    with torch.no_grad():
        out = GO.composite_generator(sd, inp, img_prev, mask, False, n_downsampling=nd, n_blocks=3, use_fg_model=fg, no_flow=no_flow)
    _close_all(RI.composite_key(fg, no_flow, nd), cases.GEN_OUT_NAMES, out)


def test_composite_local_generator():
    opt = make_opt(ngf=8, n_blocks_local=2, fg=True, gpu_ids=[])
    sd = det_fill_(NW.define_G(18, 3, 6, 4, 'compositeLocal', 3, 'batch', 1, [], opt), seed=2).state_dict()
    inp, img_prev, mask = RI.gen_inputs(6, 16, 32)
    c1, c2, c3 = RI.local_coarse()
    with torch.no_grad():
        out = GO.composite_local_generator(sd, inp, img_prev, mask, c1, c2, c3, False, n_blocks_local=2, scale=1)
    _close_all('composite_local', cases.GEN_OUT_NAMES, out)


def test_single_image_generators():
    opt = make_opt(n_blocks=2, n_blocks_local=2, gpu_ids=[])
    x = RI.single_image_input()
    sdg = det_fill_(NW.define_G(5, 3, 0, 8, 'global', 2, 'instance', 0, [], opt), seed=3).state_dict()
    sdl = det_fill_(NW.define_G(5, 3, 0, 4, 'local', 2, 'instance', 0, [], opt), seed=4).state_dict()
    with torch.no_grad():
        _close(GO.global_generator(sdg, x, n_downsampling=2, n_blocks=2), 'single/global')
        _close(GO.local_enhancer(sdl, x, n_downsample_global=2, n_blocks_global=2, n_blocks_local=2), 'single/local')


def test_discriminator():
    sd = det_fill_(NW.define_D(9, 8, 3, 'batch', 2, True, []), seed=5).state_dict()
    with torch.no_grad():
        out = GO.multiscale_discriminator(sd, RI.discriminator_input(), num_D=2, n_layers=3)
    n = 0
    for i, tower in enumerate(out):
        for j, t in enumerate(tower):
            _close(t, 'D/t%d_l%d' % (i, j))
            n += 1
    assert n == sum(1 for k in GOLD if k.startswith('D/'))


def test_model_G_inference_multiscale():
    opt = RI.inference_opt()
    single = det_fill_(NW.define_G(5, 3, 0, 8, 'global', 2, 'instance', 0, [], opt), seed=9)
    sds = [det_fill_(NW.build_netG(opt, s), seed=10 + s).state_dict() for s in range(2)]
    orc = GO.ModelGOracle(opt, sds, single.state_dict(), 'global', 2)
    seq = RI.inference_sequence()
    for t in range(3):
        A = seq[:, t:t + 3]
        o_B, o_A = orc.inference(A, A)
        _close(o_B, 'inference/%d/fake_B' % t)
        _close(o_A, 'inference/%d/real_A' % t)


@pytest.mark.parametrize('no_first_img', [False, True])
def test_model_G_training_forward(no_first_img):
    """Vid2VidModelG.forward / generate_frame_train (vid2vid_model_G.py:114-196): two frames per call, two calls (the
    second continues from the returned fake_B_prev pyramid), two spatial scales, foreground branch.  Batch 1, as the
    reference trains: its build_pyr `.view`s a time slice of the clip, which only works for one clip per batch."""
    opt = RI.train_opt(no_first_img)
    nets = [det_fill_(NW.build_netG(opt, s), seed=20 + s) for s in range(2)]
    for net in nets:
        cases.condition_flow_heads(net, 0.05)
    orc = GO.ModelGOracle(opt, [net.state_dict() for net in nets])
    seq, real = RI.train_clip(opt)
    prev = None
    for call in range(2):
        prefix = 'train_forward/%d/%d' % (int(no_first_img), call)
        with torch.no_grad():
            A, B = RI.train_call_inputs(seq, real, opt, call)
            o = orc.train_forward(A, B, A, prev, n_frames_load=2)
        _close_all(prefix, RI.TRAIN_OUT_NAMES, o[:6])
        assert o[0].shape == (1, 2, 3, 32, 64)
        _close_all(prefix, ['prev_%d' % i for i in range(len(o[6]))], o[6])
        prev = o[6]


def test_oracle_gradients_match_reference():
    """The oracle is plain differentiable PyTorch over the state_dict tensors, so autograd through it is the CPU
    reference for the backward kernels (dgrad / wgrad / norm / warp) of the training rows: for one scalar objective
    built from every output of the coarse generator, d/d(parameters), d/d(previous frames) and d/d(input) must agree
    with the gradients the reference module produces."""
    opt = make_opt(ngf=8, n_blocks=2, fg=True, n_downsample_G=2, gpu_ids=[])
    net = det_fill_(NW.define_G(18, 3, 6, 8, 'composite', 2, 'batch', 0, [], opt), seed=31)
    cases.condition_flow_heads(net, 0.05)
    inp, img_prev, mask = RI.gen_inputs(6, 16, 32, seed=2)
    params = {k for k, _ in net.named_parameters()}
    assert params == {k[len('grad/'):] for k in GOLD if k.startswith('grad/')} - {'input', 'img_prev'}
    sd = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and k in params) for k, v in net.state_dict().items()}
    x_o, p_o = inp.clone().requires_grad_(True), img_prev.clone().requires_grad_(True)
    out = GO.composite_generator(sd, x_o, p_o, mask, False, n_downsampling=2, n_blocks=2, use_fg_model=True)
    RI.objective(out, RI.cotangents(out)).backward()
    for k in params:
        gr = torch.from_numpy(GOLD['grad/' + k])
        scale = max(1.0, float(gr.abs().max()))
        assert sd[k].grad is not None, k
        assert float((sd[k].grad - gr).abs().max()) <= 2e-4 * scale, (k, float((sd[k].grad - gr).abs().max()), scale)
    for a, key in ((x_o.grad, 'grad/input'), (p_o.grad, 'grad/img_prev')):
        b = torch.from_numpy(GOLD[key])
        assert float((a - b).abs().max()) <= 2e-4 * max(1.0, float(b.abs().max()))
