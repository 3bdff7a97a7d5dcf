"""Face discriminator of the pose demo, host side: the CPU oracle (oracle/face_disc_oracle.py) against the unmodified reference's
stored results (tests/golden/face_disc.npz), the module tree of netD_f, and its checkpoint file."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from oracle import face_disc_oracle as FD                # noqa: E402
from oracle import generator_oracle as GO                # noqa: E402
from vid2vid_b200 import networks as NW                  # noqa: E402
from vid2vid_b200.utils import det_fill_                 # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
FILES = ['face_disc_keys.json', 'face_disc.npz']


def _gold():
    with np.load(os.path.join(GOLD, 'face_disc.npz')) as z:
        return {k: z[k] for k in z.files}


def _discriminators(opt):
    nc = opt.input_nc + opt.output_nc
    netD = det_fill_(NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, opt.num_D, True, []), seed=FD.D_SEED)
    netD_f = det_fill_(NW.define_D(nc, opt.ndf, opt.n_layers_D, opt.norm, max(1, opt.num_D - 2), True, []), seed=FD.D_F_SEED)
    return netD.state_dict(), netD_f.state_dict()


@pytest.mark.parametrize('name', sorted(FD.CASES))
def test_oracle_matches_reference(name):
    g = _gold()
    opt = FD.case_opt(name)
    sd_D, sd_f = _discriminators(opt)
    stats = FD.running_stats(sd_f)
    inputs = FD.case_inputs(name)
    window = FD.face_window(FD.face_box(inputs[3], opt.openpose_only), *inputs[3].shape[-2:], opt.fineSize)
    assert list(window or (-1,) * 4) == g['%s/window' % name].tolist()
    with torch.no_grad():
        losses = FD.face_disc_losses(sd_D, sd_f, stats, inputs, opt)
    assert len(losses) == len(FD.LOSS_NAMES) == 13
    for n, a in zip(FD.LOSS_NAMES, losses):
        b = torch.from_numpy(g['%s/loss/%s' % (name, n)])
        assert a.shape == b.shape, (n, a.shape, b.shape)
        assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item()), (name, n, a.flatten()[:1], b.flatten()[:1])
    keys = [k for k in g if k.startswith(name + '/stats/')]
    assert len(keys) == 2 * len(stats)
    for k in keys:
        layer, leaf = k[len(name + '/stats/'):].rsplit('.', 1)
        ours = stats[layer][FD.STAT_KEYS.index(leaf)]
        assert (ours - torch.from_numpy(g[k])).abs().max().item() <= 1e-5, k
        if window is None:                          # no face: netD_f never ran
            assert torch.equal(ours, sd_f[layer + '.' + leaf])


def test_boundary_pixels_decide_the_box():
    """The decoys of the openpose case sit exactly on float32(0.21) / float32(-0.99): in fp32 they are not face pixels (the
    stored window agrees), in double two of them would be and would stretch the box across the image."""
    real_A = FD.case_inputs('openpose')[3]
    box = FD.face_box(real_A, True)
    d = real_A.double()
    m64 = (d[:, 0] > 0.19) & (d[:, 0] < 0.21) & (d[:, 1] < -0.99) & (d[:, 2] > -0.61) & (d[:, 2] < -0.59)
    assert int(m64.sum()) == int(FD.face_mask(real_A, True).sum()) + 2
    blob = FD.CASES['openpose'][3]
    assert box == (blob[1], blob[2] - 1, blob[3], blob[4] - 1)


def test_oracle_pose_generator_matches_reference():
    """Vid2VidModelG.forward in pose mode (label_nc 0, input_nc 6, no_first_img, two scales), two calls."""
    g = _gold()
    opt = FD.pose_g_opt()
    nets = [FD.condition(det_fill_(NW.build_netG(opt, s), seed=FD.G_SEEDS[s])) for s in range(2)]
    orc = GO.ModelGOracle(opt, [n.state_dict() for n in nets])
    A, B = FD.pose_clip(*FD.G_CLIP, FD.SEED + 50)
    prev = None
    for call in range(2):
        a, b = FD.g_call_inputs(A, B, opt, call)
        with torch.no_grad():
            o = orc.train_forward(a, b, a, prev, n_frames_load=2)
        for n, v in zip(['fake_B', 'fake_B_raw', 'flow', 'weight', 'real_A', 'real_B'], o[:6]):
            ref = torch.from_numpy(g['g/%d/%s' % (call, n)])
            assert v.shape == ref.shape and (v - ref).abs().max().item() <= 2e-5, (call, n)
        prev = o[6]


def test_golden_regenerates_byte_identical(tmp_path):
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip('no reference tree (oracle/_ref or V2V_REFERENCE_ROOT)')
    root = os.path.join(os.path.dirname(__file__), '..')
    subprocess.run([sys.executable, '-m', 'oracle.face_disc_oracle', str(tmp_path)], cwd=root, check=True, capture_output=True)
    for f in FILES:
        with open(os.path.join(GOLD, f), 'rb') as a, open(str(tmp_path / f), 'rb') as b:
            assert a.read() == b.read(), f
        assert os.path.getsize(os.path.join(GOLD, f)) < 1 << 20, f


def _model_d(monkeypatch, tmp_path, **kw):
    """Vid2VidModelD.initialize on the host: device moves are skipped (the module tree, the optimizer's parameter list and the
    checkpoint files do not depend on the device)."""
    from vid2vid_b200.model_d import Vid2VidModelD
    monkeypatch.setattr(torch.nn.Module, 'to', lambda self, *a, **k: self)
    opt = FD.case_opt('interior')
    opt.checkpoints_dir, opt.name, opt.n_scales_temporal, opt.ndf = str(tmp_path), 'pose', 1, 64
    for k, v in kw.items():
        setattr(opt, k, v)
    return Vid2VidModelD().initialize(opt)


@pytest.mark.parametrize('num_D', [3, 4])
def test_model_d_keys_losses_and_optimizer(monkeypatch, tmp_path, num_D):
    with open(os.path.join(GOLD, 'face_disc_keys.json')) as f:
        ref = [(n, tuple(s)) for n, s in json.load(f)['num_D_%d' % num_D]]
    m = _model_d(monkeypatch, tmp_path, num_D=num_D)
    assert [(k, tuple(v.shape)) for k, v in m.netD_f.state_dict().items()] == ref
    assert m.netD_f.num_D == max(1, num_D - 2)
    assert m.loss_names[9:] == ['G_f_GAN', 'G_f_GAN_Feat', 'D_f_real', 'D_f_fake']
    params = [p for grp in m.optimizer_D.param_groups for p in grp['params']]
    assert [id(p) for p in params] == [id(p) for p in list(m.netD.parameters()) + list(m.netD_f.parameters())]


def test_model_d_without_flag_is_unchanged(monkeypatch, tmp_path):
    m = _model_d(monkeypatch, tmp_path, add_face_disc=False)
    assert not hasattr(m, 'netD_f') and len(m.loss_names) == 9
    assert [id(p) for grp in m.optimizer_D.param_groups for p in grp['params']] == [id(p) for p in m.netD.parameters()]


def test_face_window_matches_reference_rule():
    """vid2vid_model_D.py:224-229 on a few boxes, with the expected windows worked out by hand (fineSize 256: 64 x 64)."""
    from vid2vid_b200.model_d import Vid2VidModelD
    m = Vid2VidModelD()
    m.opt = FD.case_opt('interior')
    for box, h, w, want in [((30, 40, 50, 66), 96, 128, (3, 67, 26, 90)), ((80, 95, 110, 127), 96, 128, (31, 95, 63, 127)),
                            ((0, 0, 0, 0), 96, 128, (0, 64, 0, 64)), ((10, 29, 20, 39), 48, 128, (0, 64, 0, 64))]:
        assert m.face_window(box, h, w) == want == FD.face_window(box, h, w, 256)
    assert m.face_window(None, 96, 128) == (None,) * 4


def test_save_writes_face_discriminator(monkeypatch, tmp_path):
    m = _model_d(monkeypatch, tmp_path)
    m.save('latest')
    path = tmp_path / 'pose' / 'latest_net_D_f.pth'
    assert path.exists()
    sd = torch.load(str(path))
    assert list(sd) == list(m.netD_f.state_dict())
    assert all(torch.equal(sd[k], v) for k, v in m.netD_f.state_dict().items())
