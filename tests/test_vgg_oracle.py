"""VGG19 perceptual loss, host side: the CPU oracle (oracle/vgg_oracle.py) against the unmodified reference's stored results,
the module tree, the plan's MAC count and backward liveness, and offline weight loading."""
import json
import os
import subprocess
import sys
import urllib.request

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
from oracle import vgg_oracle as VO                      # noqa: E402
from vid2vid_b200 import networks as NW                  # noqa: E402
from vid2vid_b200.utils import make_opt                  # noqa: E402
import cases                                             # noqa: E402

MAC_PER_PIXEL = 361152       # VGG19 features[0:30] (13 3x3 convs) per input pixel


@pytest.mark.parametrize('name,N,H,W', VO.CASES)
def test_oracle_matches_reference(name, N, H, W):
    """Loss value and sampled input gradient of the oracle against the reference's VGGLoss (same seeded weights), fp32."""
    gold = cases.load_golden(name)
    sd = VO.synthetic_state()
    x, y = VO.case_inputs(N, H, W)
    x = x.clone().requires_grad_(True)
    loss = VO.vgg_loss(sd, x, y)
    loss.backward()
    assert abs(loss.item() - float(gold['loss'])) <= 1e-5 * abs(float(gold['loss']))
    g = x.grad.reshape(-1)[torch.from_numpy(gold['grad_index'])]
    ref = torch.from_numpy(gold['grad'])
    # fp32 round-off of two different summation orders; the gradient is sign(.) / numel times conv transposes
    assert (g - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


def test_golden_regenerates_byte_identical(tmp_path):
    """oracle/vgg_oracle.py rewrites the committed fixtures bit for bit from the unmodified reference (in its own process:
    ref_shim's shims are process-wide)."""
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip('no reference tree (oracle/_ref or V2V_REFERENCE_ROOT)')
    root = os.path.join(os.path.dirname(__file__), '..')
    subprocess.run([sys.executable, '-m', 'oracle.vgg_oracle', str(tmp_path)], cwd=root, check=True, capture_output=True)
    gd = os.path.join(os.path.dirname(__file__), 'golden')
    for f in ['vgg19_keys.json'] + [c[0] + '.npz' for c in VO.CASES]:
        with open(os.path.join(gd, f), 'rb') as a, open(str(tmp_path / f), 'rb') as b:
            assert a.read() == b.read(), f


def test_golden_files_small():
    gd = os.path.join(os.path.dirname(__file__), 'golden')
    for f in os.listdir(gd):
        if f.startswith('vgg'):
            assert os.path.getsize(os.path.join(gd, f)) < 1 << 20, f


def test_state_dict_keys_match_reference():
    with open(os.path.join(os.path.dirname(__file__), 'golden', 'vgg19_keys.json')) as f:
        ref = [(k, tuple(s)) for k, s in json.load(f)]
    ours = [(k, tuple(v.shape)) for k, v in NW.Vgg19().state_dict().items()]
    assert ours == ref
    assert not any(p.requires_grad for p in NW.Vgg19().parameters())


@pytest.mark.parametrize('N,H,W', [(1, 512, 1024), (2, 96, 160), (1, 64, 128)])
def test_plan_macs(N, H, W):
    """The loss plan runs two branches (x and the target y) of 361,152 MAC per input pixel each."""
    assert NW.Vgg19().conv_macs(N, H, W) == 2 * MAC_PER_PIXEL * N * H * W


def _describe(module, *shape):
    from vid2vid_b200.plan import Plan
    p = Plan(0)
    module._describe(p, *shape)
    return p.describe()


def test_target_branch_is_forward_only():
    """The y branch feeds only the detached operands of the feature-L1 nodes: its 13 convs get no backward and its values
    (input, 13 conv outputs, 4 pools) no gradient buffer; the x branch keeps all of its backward."""
    d = _describe(NW.Vgg19(), 1, 64, 128)
    grads = [c['grad'] for c in d['convs']]
    assert grads == [1] * 13 + [0] * 13
    assert d['detached_values'] == 18
    assert d['backward_ops'] == d['ops'] - 18          # the y input, its 13 convs and 4 pools


def test_existing_plans_keep_every_backward_op():
    """Without feature-L1 nodes no value is detached: generator, discriminator and FlowNet2 plans keep every op in the
    backward walk (the same backward kernels as before the liveness rule)."""
    opt = make_opt(ngf=8, n_blocks=3, fg=True, gpu_ids=[])
    plans = [
        _describe(NW.define_G(18, 3, 6, 8, 'composite', 3, 'batch', 0, [], opt), 1, 64, 128),
        _describe(NW.define_G(18, 3, 6, 4, 'compositeLocal', 3, 'batch', 1, [], opt), 1, 64, 128),
    ]
    D = NW.define_D(21, 8, 3, 'batch', 2, True, [])
    plans += [_describe(D, d, 1, 64, 128) for d in range(2)]
    from vid2vid_b200 import flownet as FN
    from vid2vid_b200.plan import Plan
    fn = FN.FlowNet2()
    for name in ('flownetc', 'flownets_1', 'flownets_2', 'flownets_d', 'flownetfusion'):
        p = Plan(0)
        getattr(fn, name).describe(p, 1, 64, 128)
        plans.append(p.describe())
    for d in plans:
        assert d['detached_values'] == 0
        assert d['backward_ops'] == d['ops']
        assert all(c['grad'] == 1 for c in d['convs'])


def test_weights_offline(tmp_path, monkeypatch):
    """The loader reads torchvision's cached checkpoint if present and never touches the network."""
    def no_network(*a, **k):
        raise AssertionError('network access')
    monkeypatch.setattr(torch.hub, 'load_state_dict_from_url', no_network)
    monkeypatch.setattr(urllib.request, 'urlopen', no_network)
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError, match=NW.VGG19_FILE):
        NW.load_vgg19_weights(NW.Vgg19())
    a = NW.load_vgg19_weights(NW.Vgg19(), synthetic=True, seed=3).state_dict()
    b = NW.vgg19_synthetic_(NW.Vgg19(), 3).state_dict()
    assert all(torch.equal(a[k], b[k]) for k in a)
    w = a['slice5.28.weight']
    assert abs(w.std().item() - (2.0 / (512 * 9)) ** 0.5) < 1e-3 and a['slice5.28.bias'].abs().max() == 0
    # a checkpoint in torchvision's layout (features.{i}.*) is mapped to the slice keys
    ck = {'features.%d.%s' % (int(k.split('.')[1]), k.split('.')[2]): v + 1 for k, v in a.items()}
    os.makedirs(tmp_path / 'checkpoints')
    torch.save(ck, str(tmp_path / 'checkpoints' / NW.VGG19_FILE))
    c = NW.load_vgg19_weights(NW.Vgg19()).state_dict()
    assert all(torch.equal(c[k], a[k] + 1) for k in a)


def test_no_pretrained_anywhere():
    """No file of the feature asks torchvision for pretrained weights."""
    root = os.path.join(os.path.dirname(__file__), '..')
    for rel in ('vid2vid_b200/networks.py', 'vid2vid_b200/model_d.py', 'oracle/vgg_oracle.py', 'tools/time_vgg.py',
                'tests/test_gpu_vgg.py'):
        src = open(os.path.join(root, rel)).read()
        assert 'pretrained=True' not in src and 'weights=IMAGENET' not in src.upper(), rel
