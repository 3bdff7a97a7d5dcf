"""CPU-only checks of the host side: C-ABI surface, conv lowering (tap groups / padding / parity /
transposed phases) emulated in numpy against torch convolutions, algorithmic MAC counts against
BASELINE.md, and state_dict compatibility with the reference.  No compute call touches a GPU."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from vid2vid_b200 import _lib as L
from vid2vid_b200 import networks as NW
from vid2vid_b200.utils import make_opt

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


def test_abi_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, 'include', 'v2v_b200.h')).read()
    declared = set(re.findall(r'\b(v2v_[a-z0-9_]+)\s*\(', hdr))
    lib = L.lib()
    for name in declared:
        assert hasattr(lib, name), 'symbol %s declared in include/v2v_b200.h is not exported' % name
    assert declared == set(L.SYMBOLS), declared ^ set(L.SYMBOLS)
    assert lib.v2v_version() >= 100


def _tap_table(desc, H, W, reuse):
    ia = lambda n: (C.c_int * n)()
    ng, nph, par, mul = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    R = ia(2)
    plane, dy, dx, tap0 = ia(64), ia(64), ia(64), ia(64)
    pb, oya, oxa, pads, ghw, ohw = ia(5), ia(4), ia(4), ia(4), ia(2), ia(2)
    L.check(L.lib().v2v_conv_tap_table(C.byref(desc), H, W, int(reuse), C.byref(ng), R, plane, dy, dx, tap0,
                                       C.byref(nph), pb, oya, oxa, pads, C.byref(par), ghw, ohw, C.byref(mul)))
    return dict(groups=[(plane[i], dy[i], dx[i], tap0[i]) for i in range(ng.value)], R=R[0], RW=R[1],
                phases=[(pb[i], pb[i + 1], oya[i], oxa[i]) for i in range(nph.value)], pads=list(pads), parity=par.value,
                grid=tuple(ghw), out=tuple(ohw), mul=mul.value)


def _emulate(x, w, t, kh, kw, transposed, reflect):
    """What the kernel computes from a tap table: x (C,H,W), w torch-layout weights."""
    Cin, H, W = x.shape
    pt, pl, pb, pr = t['pads']
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr)), mode='reflect' if reflect else 'constant')
    if t['parity']:
        Hp, Wp = (xp.shape[1] + 1) // 2, (xp.shape[2] + 1) // 2
        planes = np.zeros((4, Cin, Hp + 8, Wp + 8), np.float64)
        for py in range(2):
            for px in range(2):
                s = xp[:, py::2, px::2]
                planes[py * 2 + px, :, :s.shape[1], :s.shape[2]] = s
    else:
        planes = np.zeros((1, Cin, xp.shape[1] + 8, xp.shape[2] + 8), np.float64)
        planes[0, :, :xp.shape[1], :xp.shape[2]] = xp
    Cout = w.shape[1] if transposed else w.shape[0]
    gh, gw = t['grid']
    out = np.zeros((Cout, t['out'][0], t['out'][1]))
    for (b, e, oya, oxa) in t['phases']:
        acc = np.zeros((Cout, gh, gw))
        for (plane, dy, dx, tap0) in t['groups'][b:e]:
            for r in range(t['R']):
                ky, kx = divmod(tap0 + r, kw)
                ry, rx = divmod(r, t['RW'])          # tap r reads the patch shifted by ry rows, rx columns
                a = planes[plane, :, dy + ry:dy + ry + gh, dx + rx:dx + rx + gw]
                wk = w[:, :, ky, kx].T if transposed else w[:, :, ky, kx]      # (Cout, Cin)
                acc += np.einsum('oc,chw->ohw', wk, a)
        out[:, oya::t['mul'], oxa::t['mul']] = acc
    return out


@pytest.mark.parametrize('kh,stride,pad,reflect,transposed,op,H,W,reuse', [
    (3, 1, 1, True, False, 0, 6, 10, True),
    (3, 1, 1, True, False, 0, 5, 130, True),     # row tiles: taps served from one patch (R = 3)
    (7, 1, 3, True, False, 0, 9, 140, True),     # R = 7
    (7, 1, 3, True, False, 0, 9, 140, False),
    (3, 1, 1, True, False, 0, 32, 24, True),     # 16x8 tiles, one 18x10 patch serves all nine taps
    (7, 1, 3, True, False, 0, 16, 16, True),     # 22x14 patch, 49 taps
    (3, 1, 1, False, False, 0, 30, 17, True),    # 2-D patch with ragged edges
    (3, 2, 1, False, False, 0, 8, 12, True),
    (3, 2, 1, False, False, 0, 7, 9, True),      # odd extents
    (4, 2, 2, False, False, 0, 8, 10, True),     # discriminator
    (4, 1, 2, False, False, 0, 5, 6, True),
    (5, 2, 2, False, False, 0, 8, 8, True),      # FlowNet2
    (1, 1, 0, False, False, 0, 4, 4, True),
    (3, 2, 1, False, True, 1, 5, 7, True),       # generator deconv
    (4, 2, 1, False, True, 0, 4, 6, True),       # FlowNet2 deconv
])
def test_tap_table_matches_torch_conv(kh, stride, pad, reflect, transposed, op, H, W, reuse):
    g = torch.Generator().manual_seed(kh * 100 + stride * 10 + pad)
    Cin, Cout = 3, 4
    x = torch.randn(1, Cin, H, W, generator=g, dtype=torch.float64)
    d = L.ConvDesc()
    d.Cin, d.Cout, d.kh, d.kw, d.stride, d.pad = Cin, Cout, kh, kh, stride, pad
    d.pad_mode = L.PAD_REFLECT if reflect else L.PAD_ZERO
    d.transposed, d.output_padding = int(transposed), op
    t = _tap_table(d, H, W, reuse)
    if transposed:
        w = torch.randn(Cin, Cout, kh, kh, generator=g, dtype=torch.float64)
        ref = F.conv_transpose2d(x, w, stride=stride, padding=pad, output_padding=op)
    else:
        w = torch.randn(Cout, Cin, kh, kh, generator=g, dtype=torch.float64)
        xin = F.pad(x, (pad,) * 4, mode='reflect') if reflect else x
        ref = F.conv2d(xin, w, stride=stride, padding=0 if reflect else pad)
    assert tuple(ref.shape[2:]) == t['out']
    if reuse and not transposed and stride == 1 and W > 64 and kh > 1:
        assert t['R'] in (kh, kh * kh)                  # row tiles with horizontal reuse, or one 2-D patch for all taps
        assert t['RW'] == kh
    out = _emulate(x[0].numpy(), w.numpy(), t, kh, kh, transposed, reflect)
    np.testing.assert_allclose(out, ref[0].numpy(), rtol=1e-10, atol=1e-10)


# ---- algorithmic MACs (BASELINE.md section 2; SURVEY 8d) -------------------------------------------
def _street_opt(**kw):
    return make_opt(label_nc=35, use_instance=True, fg=True, gpu_ids=[], **kw)


def test_conv_macs_match_baseline():
    opt = _street_opt(n_scales_spatial=3)
    g0, g1, g2 = (NW.build_netG(opt, s) for s in range(3))
    assert g0.conv_macs(1, 128, 256) == 264373272576                          # cfg1
    m0 = g0.conv_macs(1, 256, 512)
    assert m0 == 1057493090304                                                # cfg2 / cfg4-G0
    m1 = g1.conv_macs(1, 512, 1024)
    m2 = g2.conv_macs(1, 1024, 2048)
    assert m1 == 592957145088 and m2 == 881508483072
    assert m0 + m1 + m2 == 2531958718464                                      # cfg4 frame
    assert g0.conv_macs(1, 256, 512) + g1.conv_macs(1, 512, 1024) == 1650450235392   # cfg3 (S=2)


def test_conv_macs_first_frame_generators():
    opt = make_opt(gpu_ids=[])
    g512 = NW.define_G(35, 3, 0, 64, 'global', 3, 'instance', 0, [], opt)
    g2048 = NW.define_G(35, 3, 0, 32, 'local', 4, 'instance', 0, [], opt)
    assert abs(g512.conv_macs(1, 256, 512) / 1e9 - 117.1) < 0.1
    assert abs(g2048.conv_macs(1, 1024, 2048) / 1e9 - 743.0) < 0.1


# ---- state_dict compatibility ------------------------------------------------------------------------
def test_state_dict_keys_match_reference_fixture():
    gold = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'state_dict_keys.json')))
    for name, c in cases.KEY_CASES.items():
        ours = [[k, list(v.shape)] for k, v in cases.build_module(c).state_dict().items()]
        assert ours == gold[name], name


def test_plan_describe_layouts():
    opt = _street_opt()
    g0 = NW.build_netG(opt, 0)
    from vid2vid_b200.plan import Plan
    p = Plan(0)
    g0._describe(p, 1, 256, 512)
    d = p.describe()
    assert d['conv_macs'] == 1057493090304
    # every value consumed by a stride-2 conv is parity split; reflect-3 layouts feed the 7x7 convs
    convs = d['convs']
    assert sum(1 for c in convs if c['k'] == [7, 7]) == 2 + 3          # stems (seg+fg fused, img) + heads (flow+weight fused)
    assert all(c['TH'] * c['TW'] == 128 for c in convs)
    assert any(c['R'] == 7 for c in convs) and any(c['phases'] == 4 for c in convs)


def _cfg4_convs(scale, h, w):
    from vid2vid_b200.plan import Plan
    g = NW.build_netG(_street_opt(n_scales_spatial=3), scale)
    p = Plan(0)
    g._describe(p, 1, h, w)
    return p.describe()['convs']


def test_kernel_configuration_choices():
    """The tiling / K-block / M-blocking decisions DESIGN.md describes, as the lowering makes them for cfg4."""
    def pick(convs, **kw):
        out = [c for c in convs if all(c[k] == v for k, v in kw.items())]
        assert out, kw
        return out
    c0, c2 = _cfg4_convs(0, 256, 512), _cfg4_convs(2, 1024, 2048)
    # 1024->1024 3x3 @32x64: 2-D patch (16x8 tiles, all 9 taps from one patch), weights streamed in 32-channel K blocks
    for c in pick(c0, Cin=1024, Cout=1024):
        assert (c['TH'], c['TW'], c['R'], c['kc'], c['BN'], c['resident'], c['MG']) == (16, 8, 9, 32, 128, 0, 1)
        assert c['units'] == 128                       # 16 M tiles x 8 N tiles: one wave on 132 SMs
    # 64->64 3x3 @512x1024: 2-D patch with resident weights
    for c in pick(c2, Cin=64, Cout=64, stride=1):
        assert (c['TH'], c['TW'], c['R'], c['kc'], c['resident']) == (16, 8, 9, 64, 1)
    # the 7x7 stems over the 108-channel input: row tiles, streamed weights, 2 x-adjacent tiles per weight pass
    for c in pick(c2, Cin=108, Cout=48) + pick(c0, Cin=108, Cout=192):
        assert (c['TH'], c['TW'], c['R'], c['MG'], c['resident'], c['BN'], c['kc']) == (1, 128, 7, 2, 0, 64, 64)
    for c in pick(_cfg4_convs(1, 512, 1024), Cin=108, Cout=96):
        assert (c['MG'], c['BN'], c['kc']) == (1, 96, 32)          # exact N tile for 96 output channels
    # every configuration respects the register budget of the accumulators: MG tiles x max(32, BN) columns <= 128
    for c in c0 + c2:
        assert c['MG'] * max(32, c['BN']) <= 128 and c['EG'] == 1 and c['CG'] >= 1 and c['SG'] >= 2


def test_conv_macs_discriminators():
    """BASELINE.md: image D (39 ch) 42.54 GMAC and temporal D (13 ch) 37.93 GMAC per forward at 1024x512, num_D 3."""
    from vid2vid_b200.plan import Plan
    for nc, want in ((39, 42.54), (13, 37.93)):
        d = NW.define_D(nc, 64, 3, 'batch', 3, True, [])
        tot, h, w = 0.0, 512, 1024
        for i in range(3):
            p = Plan(0)
            d._describe(p, 2 - i, 1, h, w)
            tot += p.conv_macs
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        assert abs(tot / 1e9 - want) < 0.01, (nc, tot)


def test_flownet2_state_dict_keys_match_reference():
    """vid2vid_b200.flownet.FlowNet2 exposes exactly the reference's 220 parameters (names and shapes), so
    FlowNet2_checkpoint.pth.tar loads unchanged (models/flownet.py:19-21)."""
    import json
    from vid2vid_b200 import flownet as FN
    keys = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'flownet2_keys.json')))
    sd = FN.FlowNet2().state_dict()
    ours = {k: list(v.shape) for k, v in sd.items()}
    ref = {k: s for k, s in keys}
    assert ours == ref, (sorted(set(ours) ^ set(ref))[:10], [k for k in ref if k in ours and ours[k] != ref[k]][:10])
    assert [k for k, _ in keys] == list(sd.keys())


def test_workspace_bytes_is_known_before_finalize():
    """include/v2v_b200.h: v2v_plan_workspace_bytes lays the arena out on the host, so a caller can allocate it and hand it to
    v2v_plan_finalize_ws (no GPU involved in the sizing)."""
    from vid2vid_b200.plan import Plan
    opt = _street_opt()
    g0 = NW.build_netG(opt, 0)
    sizes = []
    for mode in ('fast', 'precise'):
        for (h, w) in ((128, 256), (256, 512)):
            p = Plan(0, precision=mode)
            g0._describe(p, 1, h, w)
            assert not p.finalized
            sizes.append(p.workspace_bytes)
            assert p.workspace_bytes == sizes[-1]                     # idempotent
    assert all(s > 0 and s % 1024 == 0 for s in sizes)
    assert sizes[1] > sizes[0] and sizes[3] > sizes[2] and sizes[2] > sizes[0]      # grows with the frame and with the precise mode


def test_pending_losses_round_trip_on_cpu():
    """trainer.PendingLosses: the stacked loss vector comes back as the per-dictionary Python floats (host logic; on CUDA the copy
    is asynchronous and get() waits for its event only)."""
    import torch
    from vid2vid_b200.trainer import PendingLosses
    keys = [(None, 'G_GAN'), (None, 'D_real'), (0, 'G_T_GAN'), (1, 'D_T_fake')]
    p = PendingLosses(keys, torch.tensor([1.5, 2.5, 3.5, 4.5]), 2)
    out, out_T = p.get()
    assert out == {'G_GAN': 1.5, 'D_real': 2.5} and out_T == [{'G_T_GAN': 3.5}, {'D_T_fake': 4.5}]


def test_bench_prints_exactly_one_json_line_on_stdout():
    """The driver parses bench.py's stdout: whatever libraries print there (NCCL's version banner, for one) is routed to
    stderr, the JSON line goes to the real stdout."""
    import json
    import subprocess
    import sys
    code = ("import os, sys; sys.argv = ['bench.py', '--impl', 'reference', '--workload', 'cfg3']; import bench; "
            "bench.main.__globals__['run_reference'] = (lambda a, r, w: (os.write(1, b'noise on fd 1\\n'), print('noise via print'), "
            "bench.emit({'impl': 'reference', 'ok': 1}))); bench.main()")
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-500:]
    lines = r.stdout.splitlines()
    assert len(lines) == 1 and json.loads(lines[0]) == {'impl': 'reference', 'ok': 1}
    assert 'noise on fd 1' in r.stderr and 'noise via print' in r.stderr


def test_bench_dump_outputs_writes_float_arrays_and_a_fixed_sample(tmp_path):
    """bench.dump_outputs: small arrays whole, arrays above DUMP_MAX_ELEMS as the same seeded sample on every call, loss values
    float64; the training step's (loss dict, [temporal loss dicts]) as Trainer.step returns it goes through loss_arrays."""
    import sys
    sys.path.insert(0, ROOT)
    import bench
    from vid2vid_b200.trainer import PendingLosses
    small = torch.arange(12, dtype=torch.float32).view(3, 4)
    big = np.arange(bench.DUMP_MAX_ELEMS + 12345, dtype=np.float32)
    out, out_T = PendingLosses([(None, 'G_GAN'), (0, 'D_T_fake')], torch.tensor([1.5, 4.5]), 1).get()
    arrays = dict(small=small, big=big, **bench.loss_arrays(out, out_T))
    assert sorted(arrays) == ['big', 'loss_G_GAN', 'loss_T0_D_T_fake', 'small']
    for d in ('a', 'b'):
        bench.dump_outputs(str(tmp_path / d), arrays)
    a = {f[:-4]: np.load(str(tmp_path / 'a' / f)) for f in os.listdir(str(tmp_path / 'a'))}
    assert sorted(a) == sorted(arrays)
    assert a['small'].dtype == np.float32 and np.array_equal(a['small'], small.numpy())
    assert a['loss_G_GAN'].dtype == np.float64 and float(a['loss_G_GAN']) == 1.5 and float(a['loss_T0_D_T_fake']) == 4.5
    s = a['big']
    assert s.dtype == np.float32 and s.size == bench.DUMP_MAX_ELEMS
    assert np.all(np.diff(s) > 0) and np.all(np.isin(s, big))                 # sorted distinct elements of the array
    assert np.array_equal(s, np.load(str(tmp_path / 'b' / 'big.npy')))        # the same sample again
    assert sum(os.path.getsize(str(tmp_path / 'a' / f)) for f in os.listdir(str(tmp_path / 'a'))) < 64 << 20


def test_bench_dump_outputs_and_steps_arguments():
    """--dump-outputs DIR and --steps K reach the workload runner; --steps 0 is rejected."""
    import subprocess
    import sys
    code = ("import sys; sys.argv = ['bench.py'] + sys.argv[1:]; import bench; "
            "bench.main.__globals__['run_ours'] = (lambda a, r, w, lr: bench.emit({'dump': a.dump_outputs, 'steps': a.steps})); "
            "bench.main()")
    r = subprocess.run([sys.executable, '-c', code, '--steps', '7', '--dump-outputs', 'some/dir'], cwd=ROOT, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-500:]
    assert json.loads(r.stdout.splitlines()[-1]) == {'dump': 'some/dir', 'steps': 7}
    r = subprocess.run([sys.executable, '-c', code, '--steps', '0'], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and '--steps' in r.stderr
