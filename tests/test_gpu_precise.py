"""Parity of the precise (split-bf16 x3, fp32-class) product mode with the fp32 oracle at the BASELINE configurations:

* cfg4: one steady-state frame at 2048x1024, all three scales chained through Vid2VidModelG.inference (ngf 128),
  against oracle.generator_oracle.ModelGOracle on identical weights / inputs / previous frames;
* cfg2: 32 recurrent frames at 512x256 with UN-shrunken random flow heads.  The recurrence with random weights is
  chaotic (tools/precision_study.py, on the CPU: the oracle evaluated with
  fp32-rounded operands diverges from its own fp64 evaluation by x2-x60 per frame and saturates within 4-16 frames),
  so a free-running comparison of ANY two implementations is ill-posed after a few frames.  Two well-posed forms:
    - every checked frame of the 32-frame recurrent run is compared with the oracle stepped from OUR recurrent state
      (same previous frames): the single-step error must stay below the same bound at frame 31 as at frame 0;
    - free-running, at a size where the oracle can also be run in fp64: our divergence from the fp64 truth must stay
      within a constant factor of the fp32 oracle's own divergence from it, at every frame.

Stated tolerances (precise mode; images in [-1,1], flow in pixels incl. the x20*2^s head scale):
   images max|d| <= 5e-3, features max|d| <= 1e-3 * max(1,|ref|) rms-relative 1e-3, flow max|d| <= 0.02 px.
"""
import os

import numpy as np
import pytest
import torch

import cases as C
from oracle import generator_oracle as GO
from vid2vid_b200 import networks as NW
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.utils import det_fill_, make_opt, synth_label_sequence

pytestmark = pytest.mark.gpu

IMG_MAX, FLOW_MAX_PX, FEAT_REL = 5e-3, 0.02, 1e-3
# Single recurrent steps from GENERATED previous frames: with random weights the previous frame is noise-like (gradients of
# O(1) per pixel), so the warp turns the <= 0.02 px flow tolerance into up to 0.02 of image error at isolated pixels.
IMG_STEP_MAX, IMG_STEP_MEAN = 2e-2, 1e-3


def _model(opt, seed, flow_scale=1.0):
    m = Vid2VidModelG()
    single = opt.use_single_G
    opt.use_single_G = False                 # no checkpoints/ on the box: previous frames are supplied by the test
    m.initialize(opt)
    opt.use_single_G = single
    sds = []
    for s in range(opt.n_scales_spatial):
        net = getattr(m, 'netG%d' % s)
        det_fill_(net, seed=seed + s)
        if flow_scale != 1.0:
            C.condition_flow_heads(net, flow_scale)
        net.precision = 'precise'
        sds.append({k: v.detach().cpu().clone() for k, v in net.state_dict().items()})
    return m, sds


def _prev_pyramid(H, W, n_scales, seed):
    """Low-pass noise 'previous frames' (SURVEY 8d) for every scale: list over scales of (2, 3, h, w)."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(2, 3, H // 16, W // 16, generator=g) * 2 - 1
    full = torch.nn.functional.interpolate(coarse, size=(H, W), mode='bilinear', align_corners=False)
    pyr = [full]
    for _ in range(1, n_scales):
        pyr.append(GO.avgpool3s2(pyr[-1]))
    return pyr


def _cmp(name, ours, ref, lim, rel=False):
    ours, ref = ours.double().cpu(), ref.double()
    d = (ours - ref).abs()
    rms = ref.pow(2).mean().sqrt().item()
    mx, mn = d.max().item(), d.mean().item()
    print('%-22s max|d|=%.3e mean|d|=%.3e ref rms=%.3f' % (name, mx, mn, rms))
    assert torch.isfinite(ours).all(), name
    if rel:
        assert mx <= lim * max(1.0, ref.abs().max().item()), (name, mx)
        assert mn <= lim * rms * 0.2 + 1e-7, (name, mn, rms)
    else:
        assert mx <= lim, (name, mx)
    return mx


def test_cfg4_steady_state_frame_vs_oracle():
    """BASELINE config 4: 2048x1024, n_scales_spatial 3, --fg, ngf 128: one steady-state frame through inference()."""
    H, W, S = 1024, 2048, 3
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=S, ngf=128, use_single_G=True,
                   loadSize=2048, dataroot='datasets/Cityscapes/', gpu_ids=[0])
    m, sds = _model(opt, seed=61)
    seq = synth_label_sequence(3, H, W, label_nc=35, block=64, seed=5)
    prev = _prev_pyramid(H, W, S, seed=9)
    m.fake_B_prev = [p.cuda() for p in prev]
    orc = GO.ModelGOracle(opt, sds)
    orc.fake_B_prev = [p.clone() for p in prev]
    torch.set_num_threads(min(32, os.cpu_count()))
    with torch.no_grad():
        fb_ref, _ = orc.inference(seq, seq)
    fb, _ = m.inference(seq, None, seq)
    _cmp('cfg4 fake_B (scale 2)', fb, fb_ref, IMG_MAX)
    for si in range(S):
        _cmp('cfg4 state scale %d' % si, m.fake_B_prev[si][-1], orc.fake_B_prev[si][-1], IMG_MAX)
    # second call replays the CUDA graphs of all three scales: same state in -> bit-identical frame out
    m.fake_B_prev = [p.cuda() for p in prev]
    fb2, _ = m.inference(seq, None, seq)
    assert torch.equal(fb, fb2)


def test_cfg4_each_scale_all_outputs_vs_oracle():
    """All seven outputs of every scale at cfg4 size (flow in px, features), scale s fed with the ORACLE's coarse features
    so each generator is checked on identical inputs."""
    H, W, S = 1024, 2048, 3
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=S, ngf=128, gpu_ids=[0])
    torch.set_num_threads(min(32, os.cpu_count()))
    feats = (None, None, None)
    for s in range(S):
        h, w = H >> (S - 1 - s), W >> (S - 1 - s)
        net = det_fill_(NW.build_netG(opt, s), seed=71 + s)
        net.precision = 'precise'
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        inp, img_prev, mask = C.gen_inputs(35, h, w, seed=80 + s, fg_label=26, block=max(8, 64 >> (S - 1 - s)))
        with torch.no_grad():
            if s == 0:
                ref = GO.composite_generator(sd, inp, img_prev, mask, False, n_downsampling=3, n_blocks=9, use_fg_model=True)
            else:
                ref = GO.composite_local_generator(sd, inp, img_prev, mask, *feats, False, n_blocks_local=3, use_fg_model=True, scale=s)
            net = net.cuda()
            cf = tuple(f.cuda() if f is not None else None for f in feats)
            out = net(inp.cuda(), img_prev.cuda(), mask.cuda(), *cf, False)
        for key, o, r in zip(C.GEN_OUT_NAMES, out, ref):
            if key == 'flow':
                _cmp('cfg4 G%d %s' % (s, key), o, r, FLOW_MAX_PX)
            elif key.endswith('feat'):
                _cmp('cfg4 G%d %s' % (s, key), o, r, FEAT_REL, rel=True)
            else:
                _cmp('cfg4 G%d %s' % (s, key), o, r, IMG_MAX)
        feats = (ref[4], ref[5], ref[6])


def test_cfg2_32_recurrent_frames_single_step_error_does_not_grow():
    """BASELINE config 2 geometry (512x256, S=1, ngf 128, fg), un-shrunken random flow heads, 32 recurrent frames on the
    GPU.  At the checked frames the oracle is stepped from our own recurrent state; the bound is the same for all."""
    H, W = 256, 512
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=1, ngf=128, use_single_G=True,
                   loadSize=512, dataroot='datasets/Cityscapes/', gpu_ids=[0])
    m, sds = _model(opt, seed=91)
    n = 32
    seq = synth_label_sequence(n + 2, H, W, label_nc=35, block=16, seed=6)
    m.fake_B_prev = [p.cuda() for p in _prev_pyramid(H, W, 1, seed=10)]
    orc = GO.ModelGOracle(opt, sds)
    torch.set_num_threads(min(32, os.cpu_count()))
    checked = {0, 1, 2, 3, 7, 15, 23, 31}
    worst = []
    for t in range(n):
        A = seq[:, t:t + 3]
        if t in checked:
            orc.fake_B_prev = [p.cpu().clone() for p in m.fake_B_prev]
            with torch.no_grad():
                ref, _ = orc.inference(A, A)
        fb, _ = m.inference(A, None, A)
        if t in checked:
            worst.append(_cmp('cfg2 frame %2d (single step)' % t, fb, ref, IMG_STEP_MAX))
            assert (fb.cpu() - ref).abs().mean().item() <= IMG_STEP_MEAN
    # no growth: the last checked frames are not worse than 3x the early generated-state ones (independent single steps)
    assert max(worst[-3:]) <= 3 * max(worst[1:4]) + 1e-4, worst


def test_free_running_divergence_tracks_the_fp32_noise_floor():
    """Free-running 24 recurrent frames (un-shrunken flow heads) at a size where the oracle also runs in fp64.  Truth =
    oracle in fp64; floor(t) = |oracle fp32 - truth|; ours(t) = |GPU precise - truth|.  Chaos amplifies both alike; the
    statement that survives is ours(t) <= 32 * floor(t) + 1e-4 for every frame (until the floor itself saturates)."""
    H, W, n = 64, 128, 24
    opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=1, ngf=32, use_single_G=True,
                   loadSize=512, dataroot='datasets/Cityscapes/', gpu_ids=[0])
    m, sds = _model(opt, seed=95)
    seq = synth_label_sequence(n + 2, H, W, label_nc=35, block=8, seed=7)
    prev = _prev_pyramid(H, W, 1, seed=11)
    m.fake_B_prev = [p.cuda() for p in prev]
    o32 = GO.ModelGOracle(opt, sds)
    o32.fake_B_prev = [p.clone() for p in prev]
    sds64 = [{k: v.double() for k, v in sd.items()} for sd in sds]
    o64 = GO.ModelGOracle(opt, sds64)
    o64.fake_B_prev = [p.double() for p in prev]
    ratios = []
    for t in range(n):
        A = seq[:, t:t + 3]
        with torch.no_grad():
            r32, _ = o32.inference(A, A)
            torch.set_default_dtype(torch.float64)
            try:
                r64, _ = o64.inference(A.double(), A.double())
            finally:
                torch.set_default_dtype(torch.float32)
        fb, _ = m.inference(A, None, A)
        floor = (r32.double() - r64).abs().mean().item()
        ours = (fb.double().cpu() - r64).abs().mean().item()
        print('frame %2d  floor(fp32 oracle vs fp64) mean|d|=%.3e   ours vs fp64 mean|d|=%.3e' % (t, floor, ours))
        if floor > 0.02:          # saturated: both trajectories have decorrelated from the truth
            break
        assert ours <= 32 * floor + 1e-4, (t, ours, floor)
        ratios.append(ours / max(floor, 1e-9))
    assert len(ratios) >= 3
