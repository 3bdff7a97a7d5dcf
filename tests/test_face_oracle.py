"""edge2face first frame, host side: the CPU oracle (oracle/face_oracle.py) against the unmodified reference's stored results,
the module trees, the plan MAC counts, and offline loading of the weights and the features table."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from oracle import face_oracle as FO                     # noqa: E402
from vid2vid_b200 import networks as NW                  # noqa: E402
from vid2vid_b200.utils import det_fill_                 # noqa: E402
import cases                                             # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
FILES = ['face_keys.json', 'face_256.npz', 'face_infer.npz']


def _gold(name):
    with np.load(os.path.join(GOLD, name)) as z:
        return {k: z[k] for k in z.files}


def _encoder():
    return FO.encoder_state(NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []))


def test_oracle_encoder_and_lookup_match_reference():
    g = _gold('face_256.npz')
    sd = _encoder().state_dict()
    B = FO.real_images(1, FO.SIZE, FO.SIZE, FO.SEED)[:, 0]
    inst = FO.part_map(1, FO.SIZE, FO.SIZE, FO.SEED)[:, 0]
    with torch.no_grad():
        pooled = FO.encoder(sd, B, inst)
    means = np.stack([pooled[0, :, y, x].numpy() for _, (n, y, x) in sorted(FO.first_pixels(inst).items())])
    assert np.abs(means - g['pooled_means']).max() <= 1e-5
    assert np.abs(pooled[:, :, ::16, ::16].numpy() - g['pooled_sub']).max() <= 1e-5
    feat, chosen, d = FO.face_features(pooled, inst, FO.synthetic_features())
    assert chosen == int(g['chosen'])
    srt = torch.sort(d).values
    assert (srt[1] - srt[0]).item() > 1e-3              # the fixture's choice is not a near tie
    assert np.array_equal(feat[:, :, ::8, ::8].numpy(), g['feat_sub'])


def test_oracle_global_with_z_matches_reference():
    g = _gold('face_256.npz')
    opt = FO.face_opt(**FO.GZ_CFG)
    sd = FO.gz_state(NW.define_G(15, 3, 0, FO.GZ_CFG['ngf'], 'global_with_features', 3, 'instance', 0, [], opt)).state_dict()
    inst = FO.part_map(1, FO.SIZE, FO.SIZE, FO.SEED)[:, 0]
    z = FO.paint(inst, FO.synthetic_features(), int(g['chosen']))
    x = FO.edge_maps(1, FO.SIZE, FO.SIZE, FO.SEED)[:, 0]
    with torch.no_grad():
        out = FO.global_with_z(sd, x, z, 3, FO.GZ_CFG['n_blocks'])
    assert np.abs(out.numpy() - g['gz_out']).max() <= 1e-4


def test_oracle_first_frames_match_reference():
    """The reference inference's two first frames: Encoder -> lookup -> Global_with_z per frame, restated."""
    g = _gold('face_infer.npz')
    H = W = FO.INFER_SIZE
    nF = FO.INFER_CFG['n_frames'] + 2
    A, Bs, I = FO.edge_maps(nF, H, W, FO.SEED + 20), FO.real_images(nF, H, W, FO.SEED + 20), FO.part_map(nF, H, W, FO.SEED + 20)
    seeds = FO.infer_seeds()
    opt = FO.face_opt()
    sdE = det_fill_(NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []), seed=seeds['netE']).state_dict()
    sdG = det_fill_(NW.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], opt), seed=seeds['netG_i']).state_dict()
    feats = FO.synthetic_features()
    with torch.no_grad():
        for i in range(2):
            pooled = FO.encoder(sdE, Bs[:, i], I[:, i])
            fm, chosen, _ = FO.face_features(pooled, I[:, i], feats)
            assert chosen == int(g['first_chosen'][i])
            out = FO.global_with_z(sdG, A[:, i], fm, 3, opt.n_blocks)
            assert np.abs(out.numpy() - g['first_frames'][i:i + 1]).max() <= 1e-4


def test_golden_regenerates_byte_identical(tmp_path):
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip('no reference tree (oracle/_ref or V2V_REFERENCE_ROOT)')
    root = os.path.join(os.path.dirname(__file__), '..')
    subprocess.run([sys.executable, '-m', 'oracle.face_oracle', str(tmp_path)], cwd=root, check=True, capture_output=True)
    for f in FILES:
        with open(os.path.join(GOLD, f), 'rb') as a, open(str(tmp_path / f), 'rb') as b:
            assert a.read() == b.read(), f
        assert os.path.getsize(os.path.join(GOLD, f)) < 1 << 20, f


def test_state_dict_keys_match_reference():
    with open(os.path.join(GOLD, 'face_keys.json')) as f:
        ref = {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}
    enc = NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, [])
    gz = NW.define_G(15, 3, 0, 64, 'global_with_features', 3, 'instance', 0, [], FO.face_opt(n_blocks=9))
    for name, m in (('encoder', enc), ('global_with_z', gz)):
        assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == ref[name]
        # a reference-layout checkpoint loads strictly
        m.load_state_dict({k: torch.zeros(s) if not k.endswith('num_batches_tracked') else torch.zeros(s, dtype=torch.long)
                           for k, s in ref[name]}, strict=True)


def test_local_with_features_still_raises():
    with pytest.raises(NotImplementedError):
        NW.define_G(15, 3, 0, 32, 'local_with_features', 3, 'instance', 0, [], FO.face_opt())


def _conv_macs(H, W, layers):
    """Independent count: layers = [(kind, cin, cout, k, scale_before)] walked over the resolution (conv s2 halves it,
    transposed conv doubles it and counts its input pixels)."""
    total, h, w = 0, H, W
    for kind, cin, cout, k in layers:
        if kind == 'down':
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            total += h * w * cin * cout * 9
        elif kind == 'up':
            total += h * w * cin * cout * 9
            h, w = 2 * h, 2 * w
        else:
            total += h * w * cin * cout * k * k
    return total


@pytest.mark.parametrize('H,W', [(256, 256), (512, 512), (128, 192)])
def test_plan_macs(H, W):
    ngf, nd = 16, 4
    enc = [('conv', 3, ngf, 7)] + [('down', ngf * 2 ** i, ngf * 2 ** (i + 1), 3) for i in range(nd)]
    enc += [('up', ngf * 2 ** (nd - i), ngf * 2 ** (nd - i) // 2, 3) for i in range(nd)] + [('conv', ngf, 16, 7)]
    assert NW.define_G(3, 16, 0, ngf, 'encoder', nd, 'instance', 0, []).conv_macs(1, H, W) == _conv_macs(H, W, enc)
    ngf, nd, nz, nb = 64, 3, 16, 9
    gz = [('conv', 15 + nz, ngf, 7)] + [('down', ngf * 2 ** i, ngf * 2 ** (i + 1), 3) for i in range(nd)]
    gz += [('conv', 512 + nz, 512 + nz, 3)] * (2 * nb)
    gz += [('up', ngf * 2 ** (nd - i) + (2 * nz if i == 0 else 0), ngf * 2 ** (nd - i) // 2, 3) for i in range(nd)]
    gz += [('conv', ngf + nz, 3, 7)]
    m = NW.define_G(15, 3, 0, ngf, 'global_with_features', nd, 'instance', 0, [], FO.face_opt(n_blocks=nb))
    assert m.conv_macs(1, H, W) == _conv_macs(H, W, gz)


def _model(tmp_path, monkeypatch, synthetic):
    from vid2vid_b200.model_g import Vid2VidModelG
    monkeypatch.chdir(tmp_path)
    opt = FO.face_opt(synthetic_weights=synthetic)
    m = Vid2VidModelG()
    m.opt, m.device_ = opt, torch.device('cpu')
    return m


def test_missing_files_raise_and_synthetic_loads_offline(tmp_path, monkeypatch):
    m = _model(tmp_path, monkeypatch, False)
    with pytest.raises(FileNotFoundError, match='checkpoints/edge2face_single/latest_net_E.pth'):
        m.load_single_G()
    with pytest.raises(FileNotFoundError, match='checkpoints/edge2face_single/features.npy'):
        m.load_face_features()
    m = _model(tmp_path, monkeypatch, True)
    g = m.load_single_G()
    assert isinstance(g, NW.Global_with_z) and isinstance(m.netE, NW.Encoder) and m.opt.feat_num == 16
    assert m.face_table.shape == (7, 16, 17) and m.face_rows == [16] * 7 and m.face_num_images == 16
    # a features.npy in the reference's pickled-dict layout is read from the local path
    feats = FO.synthetic_features(seed=5, num_images=9)
    os.makedirs(tmp_path / 'checkpoints' / 'edge2face_single')
    np.save(str(tmp_path / 'checkpoints' / 'edge2face_single' / 'features.npy'), feats, allow_pickle=True)
    m.load_face_features()
    assert m.face_num_images == 9 and torch.equal(m.face_table[3, :9], torch.as_tensor(feats[3]).float())
    # checkpoints in the reference layout load when present
    torch.save(NW.define_G(3, 16, 0, 16, 'encoder', 4, 'instance', 0, []).state_dict(),
               str(tmp_path / 'checkpoints' / 'edge2face_single' / 'latest_net_E.pth'))
    m = _model(tmp_path, monkeypatch, False)
    with pytest.raises(FileNotFoundError, match='latest_net_G.pth'):
        m.load_single_G()


def test_pack_face_features():
    feats = {k: np.arange(12, dtype=np.float64).reshape(3, 4) + k for k in range(7)}
    feats[2] = feats[2][:2]
    table, rows, num = NW.pack_face_features(feats, 3)
    assert table.shape == (7, 3, 4) and rows == [3, 3, 2, 3, 3, 3, 3] and num == 3
    assert torch.equal(table[2, 2], torch.zeros(4))
