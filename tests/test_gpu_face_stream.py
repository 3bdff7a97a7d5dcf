"""Streaming the edge2face and pose2body demos on the GPU: the per-image face-feature lookup (v2v_face_features_per_image)
against oracle/face_oracle.py applied image by image, batched face first frames (each clip bit-identical to its own b = 1
run), face and dense (pose) streams through Vid2VidModelG.inference_stream against inference() on the same 5-D tensors, and
the conv configurations that only these products' plans lower, against fp64 (tests/test_face_stream_host.py censuses them).
"""
import os
import sys

import pytest
import torch

import bf16_emul as E
import test_gpu_conv as TC
import test_gpu_multiclip as TMC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from oracle import face_oracle as FO                     # noqa: E402
from vid2vid_b200 import networks as NW, ops             # noqa: E402

pytestmark = pytest.mark.gpu
N_FRAMES = 8


@pytest.fixture(autouse=True)
def _precise():
    saved = NW.DEFAULT_PRECISION
    NW.set_default_precision('precise')
    yield
    NW.set_default_precision(saved)


# ----------------------------------------------------------------------------- per-image face_features
def _image(H, W, seed, drop=(), repeat=None):
    """(pooled (1, 16, H, W), part map (1, 1, H, W)) of one image: labels in `drop` replaced by 0 (absent), or every label
    folded onto `repeat` labels (the others absent, the kept ones repeated over more blocks)."""
    g = torch.Generator().manual_seed(seed)
    inst = FO.part_map(1, H, W, seed)[:, 0]
    for d in drop:
        inst[inst == d] = 0.0
    if repeat:
        inst = torch.remainder(inst, repeat)
    return FO.instance_mean(torch.rand(1, 16, H, W, generator=g) * 2 - 1, inst), inst


# per batch: one (seed, drop, repeat) per image; the images share labels, miss some and repeat others
BATCHES = {
    'one': [(3, (), None)],
    'two_missing': [(4, (), None), (5, (2, 5), None)],
    'three_repeat': [(6, (), None), (7, (), 3), (8, (1,), None)],
    'four_mixed': [(9, (6,), None), (10, (), 2), (11, (), None), (12, (3, 4), None)],
}


@pytest.mark.parametrize('batch', list(BATCHES))
def test_per_image_lookup_matches_oracle_image_by_image(batch):
    H, W = 128, 144
    imgs = [_image(H, W, s, d, r) for s, d, r in BATCHES[batch]]
    pooled, inst = torch.cat([p for p, _ in imgs]), torch.cat([i for _, i in imgs])
    feats = FO.synthetic_features(seed=9, num_images=40)
    table, rows, num = NW.pack_face_features(feats, 16)
    out, chosen = ops.face_features(pooled.cuda(), inst.cuda(), table.cuda(), rows, num, per_image=True)
    out, chosen = out.cpu(), chosen.cpu().tolist()
    assert len(chosen) == len(imgs)
    for n, (p, i) in enumerate(imgs):
        ref_map, ref_idx, d = FO.face_features(p, i, feats)
        srt = torch.sort(d).values
        assert (srt[1] - srt[0]).item() > 1e-4, n          # a clear margin (the oracle's distances are fp64)
        assert chosen[n] == ref_idx, (n, chosen, ref_idx)
        assert torch.equal(out[n:n + 1], ref_map), n
    if len(imgs) > 1:
        assert len(set(chosen)) > 1, chosen               # the images' own rows differ: one row for all would fail


def test_per_image_lookup_at_one_image_equals_whole_batch_lookup():
    pooled, inst = _image(128, 160, 21, (6, 3))
    table, rows, num = NW.pack_face_features(FO.synthetic_features(seed=2, num_images=20), 16)
    args = (pooled.cuda(), inst.cuda(), table.cuda(), rows, num)
    a, ca = ops.face_features(*args)
    b, cb = ops.face_features(*args, per_image=True)
    assert torch.equal(ca, cb) and torch.equal(a, b)


def test_per_image_lookup_rejects_invalid_ids():
    pooled, inst = _image(64, 64, 5)
    pooled, inst = pooled.repeat(2, 1, 1, 1), inst.repeat(2, 1, 1, 1)
    inst[1, 0, 3, 7] = 7.0
    table, rows, num = NW.pack_face_features(FO.synthetic_features(seed=2, num_images=20), 16)
    with pytest.raises(RuntimeError, match='not an integer'):
        ops.face_features(pooled.cuda(), inst.cuda(), table.cuda(), rows, num, per_image=True)


def test_per_image_lookup_under_graph_capture_flags_only_the_bad_image():
    pooled, inst = _image(64, 64, 5)
    pooled, inst = pooled.repeat(2, 1, 1, 1).cuda(), inst.repeat(2, 1, 1, 1)
    inst[1, 0, 3, 7] = 2.5
    inst = inst.cuda()
    table, rows, num = NW.pack_face_features(FO.synthetic_features(seed=2, num_images=20), 16)
    table = table.cuda()
    good, good_c = ops.face_features(pooled[:1], inst[:1], table, rows, num, per_image=True)
    graph, res = torch.cuda.CUDAGraph(), {}
    with torch.cuda.graph(graph):                 # the capture cannot wait for the check: the bad image is flagged instead
        res['out'], res['chosen'] = ops.face_features(pooled, inst, table, rows, num, per_image=True)
    graph.replay()
    torch.cuda.synchronize()
    assert res['chosen'].tolist() == [int(good_c.item()), -1]
    assert torch.equal(res['out'][:1], good) and torch.isnan(res['out'][1]).all()


# ----------------------------------------------------------------------------- batched face first frames
B = 3


def _face_model():
    m, clip = TMC._face()
    return m, [clip(k) for k in range(B)]


def _chosen_recorder(m):
    rec = []
    for name in ('get_face_features', 'get_face_features_per_clip'):
        orig = getattr(m, name)

        def wrap(real_image, inst, orig=orig):
            r = orig(real_image, inst)
            rec.append(m.face_chosen.cpu().tolist())
            return r
        setattr(m, name, wrap)
    return rec


def test_batched_face_first_frames_equal_each_clip():
    m, clips = _face_model()
    tG = m.opt.n_frames_G
    rec = _chosen_recorder(m)
    both = [torch.cat([c[i] for c in clips]) for i in range(3)]
    batched = [m.inference(*[x[:, t:t + tG] for x in both])[0].clone() for t in range(N_FRAMES)]
    assert len(rec) == tG - 1 and all(len(r) == B for r in rec)          # one lookup per first frame, one row per clip
    per_clip = [[r[k] for r in rec] for k in range(B)]
    assert not (m.netE.sample_stats or m.netG_i.sample_stats)
    for k in range(B):
        m.reset_stream()
        del rec[:]
        for t in range(N_FRAMES):
            fake_B, _ = m.inference(*[x[:, t:t + tG] for x in clips[k]])
            assert torch.equal(batched[t][k:k + 1], fake_B), 'clip %d frame %d: max |d| %.3g' % (
                k, t, (batched[t][k:k + 1] - fake_B).abs().max().item())
        assert [r[0] for r in rec] == per_clip[k], (k, rec, per_clip[k])


# ----------------------------------------------------------------------------- face streams
def _stream(m, A, Bs, I, u8=False):
    """Feeds (b, T, ...) clips to inference_stream frame by frame (the real frames and part maps only while the window
    fills); b == 1 passes unbatched frames.  Returns the generated frames, or with u8 the uint8 images."""
    tG, b = m.opt.n_frames_G, A.shape[0]
    sq = (lambda x: x[0]) if b == 1 else (lambda x: x)
    H, W = A.shape[-2:]
    out = torch.empty(((b,) if b > 1 else ()) + (H, W, 3), dtype=torch.uint8, device='cuda') if u8 else None
    got = []
    for t in range(A.shape[1]):
        fill = Bs is not None and t < tG - 1
        kw = dict(real_frame=sq(Bs[:, t]), inst_frame=sq(I[:, t, 0]).to(torch.uint8)) if fill else {}
        r = m.inference_stream(sq(A[:, t]), out_u8=out, **kw)
        assert (r is None) == (t < tG - 1)
        if r is not None:
            got.append(r.clone())
    return got


def _inference(m, A, Bs, I):
    tG = m.opt.n_frames_G
    m.reset_stream()
    return [m.inference(A[:, t:t + tG], Bs[:, t:t + tG] if Bs is not None else None,
                        I[:, t:t + tG] if I is not None else None)[0].clone() for t in range(A.shape[1] - tG + 1)]


def _tensor2im(frame):
    import ctypes
    from vid2vid_b200 import _lib as L
    out = torch.empty(frame.shape[-2], frame.shape[-1], 3, dtype=torch.uint8, device='cuda')
    L.check(L.lib().v2v_tensor2im_u8(ctypes.c_void_p(frame.data_ptr()), ctypes.c_void_p(out.data_ptr()), 1, 3, frame.shape[-2],
                                     frame.shape[-1], L.current_stream_ptr()))
    return out


def test_face_stream_equals_inference():
    m, clips = _face_model()
    A, Bs, I = clips[0]
    ref = _inference(m, A, Bs, I)
    m.reset_stream()
    got = _stream(m, A, Bs, I)
    assert len(got) == len(ref) == N_FRAMES
    for t, (g, r) in enumerate(zip(got, ref)):
        assert torch.equal(g, r), 'frame %d: max |d| %.3g' % (t, (g - r).abs().max().item())
    m.reset_stream()
    images = _stream(m, A, Bs, I, u8=True)
    for t, (im, r) in enumerate(zip(images, ref)):
        assert torch.equal(im, _tensor2im(r)), t
    # reset_stream() and a new clip reproduce a fresh run of that clip
    m.reset_stream()
    A2, B2, I2 = clips[1]
    again = _stream(m, A2, B2, I2)
    fresh = _inference(m, A2, B2, I2)
    assert len(again) == len(fresh) and all(torch.equal(a, f) for a, f in zip(again, fresh))


def test_face_stream_of_b_clips_equals_each_stream():
    m, clips = _face_model()
    both = [torch.cat([c[i] for c in clips]) for i in range(3)]
    m.reset_stream()
    batched = _stream(m, *both)
    with pytest.raises(ValueError, match='started with 3 clip'):
        m.inference_stream(clips[0][0][0, 0])
    for k in range(B):
        m.reset_stream()
        one = _stream(m, *clips[k])
        assert len(one) == len(batched)
        for t, (g, r) in enumerate(zip(batched, one)):
            assert torch.equal(g[k:k + 1], r), 'clip %d frame %d' % (k, t)


# ----------------------------------------------------------------------------- pose (dense) streams
@pytest.mark.parametrize('b', [1, 2])
def test_pose_stream_equals_inference(b):
    m, clip = TMC._pose()
    A = torch.cat([clip(k)[0] for k in range(b)])
    ref = _inference(m, A, None, None)
    m.reset_stream()
    got = _stream(m, A, None, None)
    assert len(got) == len(ref) == N_FRAMES
    for t, (g, r) in enumerate(zip(got, ref)):
        assert torch.equal(g, r), 'frame %d: max |d| %.3g' % (t, (g - r).abs().max().item())


# ----------------------------------------------------------------------------- conv configurations vs fp64
# Kernel configurations that tools/time_face_stream.py's plans lower and no other GPU parity case reaches, at the shape that
# selects them on 132 SMs, checked against the same layers in fp64 (precise) or bf16-emulated fp32 (fast) image by image.
# name, layer list builder, input shape (N, C, H, W), modes
BN = NW.get_norm_layer('batch')
CONV_CASES = [
    # the face Encoder's second stride-2 conv at 512x512 on four clips: the epilogue warpgroup gets enough units
    ('enc_down_32_64_async', lambda: NW._down(32, 64, BN), (4, 32, 256, 256), TC.MODES),
    # the 1024x512 pose model's 18-channel label stems: the coarsest scale (ngf 128) and the finest (ngf 32)
    ('pose_stem_18_128', lambda: NW._stem(18, 128, BN), (1, 18, 256, 128), TC.MODES),
    ('pose_stem_18_32', lambda: NW._stem(18, 32, BN), (1, 18, 1024, 512), TC.MODES),
]


@pytest.mark.parametrize('name,build,shape,mode', [(c[0], c[1], c[2], m) for c in CONV_CASES for m in c[3]],
                         ids=['%s-%s' % (c[0], m) for c in CONV_CASES for m in c[3]])
def test_face_stream_conv_configuration_vs_fp64(name, build, shape, mode):
    runner = TMC._per_sample_runner(build, mode)
    x = TC._x(*shape).cuda()
    E.ROUND[0] = (mode == 'fast')
    try:
        with torch.no_grad():
            out = runner(x)
            out2 = runner(x)
            xr = E.r16(x)
            ref = torch.cat([E.run_units(list(runner.seq), xr[k:k + 1]) for k in range(shape[0])])
    finally:
        E.ROUND[0] = True
    assert torch.equal(out, out2), 'graph replay differs from eager run'
    TC._check(out, ref, name, mode=mode)
