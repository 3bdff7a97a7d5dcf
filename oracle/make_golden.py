"""TEST INFRASTRUCTURE.  Generates tests/golden/*.npz by running the UNMODIFIED reference
(imported through oracle/ref_shim.py, V2V_REFERENCE_ROOT) on the seeded cases of
tests/cases.py.  Run where the reference tree is available:   python -m oracle.make_golden [case ...]

The fixtures are what pins oracle/generator_oracle.py, oracle/losses_oracle.py, the host helpers
and the CUDA path: the tests regenerate the weights and inputs from the seeds and compare with them.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
from oracle import ref_shim                                     # noqa: E402
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import cases as C                                               # noqa: E402
from vid2vid_b200.utils import make_opt, det_fill_, synth_label_sequence   # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')


def _np(t):
    return t.detach().cpu().numpy().astype(np.float32)


def coarse_feats(c):
    g = torch.Generator().manual_seed(c['seed'] + 5)
    h2, w2, ngf = c['h'] // 2, c['w'] // 2, c['ngf']
    return (torch.randn(1, 2 * ngf, h2, w2, generator=g), torch.randn(1, 2 * ngf, h2, w2, generator=g),
            torch.randn(1, ngf, h2, w2, generator=g))


def run_case(name, c):
    N = ref_shim.networks()
    kind = c['kind']
    out = {}
    torch.manual_seed(0)
    if c.get('align_corners'):
        # original PyTorch-0.4 semantics (SURVEY App. B #2): force the flag the reference omits
        import torch.nn.functional as F
        orig = F.grid_sample
        F.grid_sample = lambda *a, **k: orig(*a, **{**k, 'align_corners': True})
    try:
        with torch.no_grad():
            if kind in ('composite', 'compositeLocal'):
                nc = 3 * (c['label_nc'] + 1)
                opt = make_opt(ngf=c['ngf'], n_blocks=c.get('n_blocks', 9), n_blocks_local=c.get('n_blocks_local', 3),
                               fg=c['fg'], no_flow=c.get('no_flow', False), n_downsample_G=c['nd'], gpu_ids=[])
                net = det_fill_(N.define_G(nc, 3, 6, c['ngf'], kind, c['nd'], 'batch', c.get('scale', 0), [], opt),
                                seed=c['seed'])
                inp, img_prev, mask = C.gen_inputs(c['label_nc'], c['h'], c['w'], c['seed'], block=c.get('block', 4))
                if kind == 'composite':
                    res = net(inp, img_prev, mask, None, None, None, False)
                else:
                    res = net(inp, img_prev, mask, *coarse_feats(c), False)
                ss = c.get('subsample', 1)
                for nme, t in zip(C.GEN_OUT_NAMES, res):
                    if t is None:
                        continue
                    if ss > 1 and t.shape[1] > 3:     # big feature maps: keep a strided sample + channel means
                        out[nme + '_sub'] = _np(t[:, :, ::ss, ::ss])
                        out[nme + '_cmean'] = _np(t.mean(dim=(2, 3)))
                    else:
                        out[nme] = _np(t)
            elif kind in ('global', 'local'):
                opt = make_opt(n_blocks=c['n_blocks'], n_blocks_local=c.get('n_blocks_local', 3), gpu_ids=[])
                net = det_fill_(N.define_G(c['input_nc'], 3, 0, c['ngf'], kind, c['nd'], 'instance', 0, [], opt),
                                seed=c['seed'])
                g = torch.Generator().manual_seed(c['seed'] + 1)
                lab = synth_label_sequence(1, c['h'], c['w'], label_nc=c['input_nc'], block=4, seed=c['seed'])
                x = torch.zeros(1, c['input_nc'], c['h'], c['w']).scatter_(1, lab[:, 0].long(), 1.0)
                out['out'] = _np(net(x))
            elif kind == 'D':
                net = det_fill_(N.define_D(c['input_nc'], c['ndf'], c['n_layers'], 'batch', c['num_D'], True, []),
                                seed=c['seed'])
                g = torch.Generator().manual_seed(c['seed'] + 1)
                x = torch.randn(c['batch'], c['input_nc'], c['h'], c['w'], generator=g)
                for i, tower in enumerate(net(x)):
                    for j, t in enumerate(tower):
                        out['t%d_l%d' % (i, j)] = _np(t)
            elif kind == 'inference':
                opt = C.inference_opt(c)
                single = det_fill_(N.define_G(c['label_nc'], 3, 0, 16, 'global', 2, 'instance', 0, [], opt),
                                   seed=c['seed'] + 100)
                m = ref_shim.make_model_G(opt, single)
                for s in range(c['n_scales']):
                    det_fill_(getattr(m, 'netG%d' % s), seed=c['seed'] + s)
                    C.condition_flow_heads(getattr(m, 'netG%d' % s), c['flow_weight_scale'])
                tG = opt.n_frames_G
                seq = synth_label_sequence(c['n_gen'] + tG - 1, c['h'], c['w'], label_nc=c['label_nc'], block=8,
                                           seed=c['seed'])
                for t in range(c['n_gen']):
                    A = seq[:, t:t + tG]
                    fake_B, real_A = m.inference(A, None, A)
                    out['fake_B_%d' % t] = _np(fake_B)
                for si in range(c['n_scales']):
                    out['prev_state_%d' % si] = _np(m.fake_B_prev[si])
            else:
                raise ValueError(kind)
    finally:
        if c.get('align_corners'):
            F.grid_sample = orig
    save_fixture(name, out)


PART_BYTES = 900 * 1024


def save_fixture(name, arrays):
    """tests/golden/<name>.npz, continued in <name>_2.npz, ... so that no file exceeds 1 MB (tests/cases.load_golden)."""
    os.makedirs(OUT, exist_ok=True)
    parts, cur, size = [], {}, 0
    for k, v in arrays.items():
        if cur and size + v.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, part in enumerate(parts):
        path = os.path.join(OUT, name + ('.npz' if i == 0 else '_%d.npz' % (i + 1)))
        np.savez_compressed(path, **part)
        print('%-14s %7.1f KB  %s' % (os.path.basename(path), os.path.getsize(path) / 1024, sorted(part)))


def dump_keys():
    """state_dict key / shape lists of the reference modules -> tests/golden/state_dict_keys.json."""
    import json
    N = ref_shim.networks()
    out = {}
    for name, c in C.KEY_CASES.items():
        kind = c['kind']
        if kind in ('composite', 'compositeLocal'):
            opt = make_opt(ngf=c['ngf'], n_blocks=c.get('n_blocks', 9), n_blocks_local=c.get('n_blocks_local', 3),
                           fg=c['fg'], no_flow=c.get('no_flow', False), n_downsample_G=c['nd'], gpu_ids=[])
            net = N.define_G(3 * (c['label_nc'] + 1), 3, 6, c['ngf'], kind, c['nd'], 'batch', c.get('scale', 0), [], opt)
        elif kind in ('global', 'local'):
            opt = make_opt(n_blocks=c['n_blocks'], n_blocks_local=c.get('n_blocks_local', 3), gpu_ids=[])
            net = N.define_G(c['input_nc'], 3, 0, c['ngf'], kind, c['nd'], 'instance', 0, [], opt)
        else:
            net = N.define_D(c['input_nc'], c['ndf'], c['n_layers'], 'batch', c['num_D'], True, [])
        out[name] = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(OUT, 'state_dict_keys.json'), 'w') as f:
        json.dump(out, f)
    print('state_dict_keys.json', {k: len(v) for k, v in out.items()})


def flownet2_golden():
    """Reference FlowNet2 (with the op stand-ins of ref_shim.install_flownet2_ops) and the FlowNet wrapper's
    compute_flow_and_conf on seeded inputs, with the deterministic weights of flownet2_oracle.det_state_dict ->
    tests/golden/flownet2_keys.json + flownet2_small.npz."""
    import json
    import types
    from oracle import flownet2_oracle as FO
    F2 = ref_shim.flownet2_class()
    net = F2().eval()
    keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(OUT, 'flownet2_keys.json'), 'w') as f:
        json.dump(keys, f)
    net.load_state_dict(FO.det_state_dict(keys, seed=7))
    g = torch.Generator().manual_seed(11)
    pair = torch.rand(1, 3, 2, 64, 128, generator=g)
    base = torch.rand(1, 3, 80, 64, generator=g)                    # height 80: exercises the resize-to-64 path
    im1, im2 = base, torch.roll(base, shifts=(1, 2), dims=(2, 3)) * 0.9 + 0.05
    from models.flownet import FlowNet                              # noqa (reference module)
    from models.flownet2_pytorch.networks.resample2d_package.resample2d import Resample2d   # noqa
    stub = types.SimpleNamespace(flowNet=net, resample=Resample2d())
    stub.norm = lambda t: FlowNet.norm(stub, t)
    with torch.no_grad():
        flow = net(pair)
        wflow, wconf = FlowNet.compute_flow_and_conf(stub, im1, im2)
    out = dict(pair=_np(pair), flow=_np(flow), im1=_np(im1), im2=_np(im2), wflow=_np(wflow), wconf=_np(wconf))
    path = os.path.join(OUT, 'flownet2_small.npz')
    np.savez_compressed(path, **out)
    print('flownet2_small %7.1f KB flow rms %.3f wflow rms %.3f conf mean %.3f' % (
        os.path.getsize(path) / 1024, float(flow.pow(2).mean().sqrt()), float(wflow.pow(2).mean().sqrt()), float(wconf.mean())))


def reference_checks():
    """Reference outputs (and gradients) on the seeded inputs of tests/test_oracle_vs_reference.py,
    tests/test_losses_oracle.py, tests/test_flownet2_oracle.py and tests/test_gpu_integration.py -> tests/golden/reference*.npz,
    and the reference BaseModel's schedule / checkpoint behaviour of tests/test_host_schedule.py -> host_schedule.json.
    Every module is filled with det_fill_ (FlowNet2: flownet2_oracle.det_state_dict), so the tests rebuild the same
    weights on their own modules."""
    import json
    import tempfile
    import types
    from oracle import generator_oracle as GO
    import reference_inputs as RI
    N = ref_shim.networks()
    out = {}

    def put(prefix, tensors):
        for k, t in tensors.items():
            if t is not None:
                out[prefix + '/' + k] = _np(t)

    with torch.no_grad():
        for fg, no_flow, nd in RI.COMPOSITE_VARIANTS:
            opt = make_opt(ngf=8, n_blocks=3, fg=fg, no_flow=no_flow, n_downsample_G=nd, gpu_ids=[])
            net = det_fill_(N.define_G(18, 3, 6, 8, 'composite', nd, 'batch', 0, [], opt), seed=1)
            inp, img_prev, mask = RI.gen_inputs(6, 16, 32)
            put(RI.composite_key(fg, no_flow, nd), dict(zip(C.GEN_OUT_NAMES, net(inp, img_prev, mask, None, None, None, False))))
        opt = make_opt(ngf=8, n_blocks_local=2, fg=True, gpu_ids=[])
        net = det_fill_(N.define_G(18, 3, 6, 4, 'compositeLocal', 3, 'batch', 1, [], opt), seed=2)
        inp, img_prev, mask = RI.gen_inputs(6, 16, 32)
        put('composite_local', dict(zip(C.GEN_OUT_NAMES, net(inp, img_prev, mask, *RI.local_coarse(), False))))
        opt = make_opt(n_blocks=2, n_blocks_local=2, gpu_ids=[])
        x = RI.single_image_input()
        put('single', {'global': det_fill_(N.define_G(5, 3, 0, 8, 'global', 2, 'instance', 0, [], opt), seed=3)(x),
                       'local': det_fill_(N.define_G(5, 3, 0, 4, 'local', 2, 'instance', 0, [], opt), seed=4)(x)})
        net = det_fill_(N.define_D(9, 8, 3, 'batch', 2, True, []), seed=5)
        put('D', {'t%d_l%d' % (i, j): t for i, tower in enumerate(net(RI.discriminator_input())) for j, t in enumerate(tower)})
        # Vid2VidModelG.inference, two scales, --fg --use_single_G
        opt = RI.inference_opt()
        single = det_fill_(N.define_G(5, 3, 0, 8, 'global', 2, 'instance', 0, [], opt), seed=9)
        m = ref_shim.make_model_G(opt, single)
        det_fill_(m.netG0, seed=10)
        det_fill_(m.netG1, seed=11)
        seq = RI.inference_sequence()
        for t in range(3):
            A = seq[:, t:t + 3]
            fake_B, real_A = m.inference(A, None, A)
            put('inference/%d' % t, {'fake_B': fake_B, 'real_A': real_A})
        # Vid2VidModelG.forward (training), two calls continuing from the returned fake_B_prev pyramid
        for no_first_img in (False, True):
            opt = RI.train_opt(no_first_img)
            m = ref_shim.make_model_G(opt)
            det_fill_(m.netG0, seed=20)
            det_fill_(m.netG1, seed=21)
            C.condition_flow_heads(m.netG0, 0.05)
            C.condition_flow_heads(m.netG1, 0.05)
            seq, real = RI.train_clip(opt)
            prev = None
            for call in range(2):
                A, B = RI.train_call_inputs(seq, real, opt, call)
                r = m.forward(A, B, A, prev)
                put('train_forward/%d/%d' % (int(no_first_img), call), dict(zip(RI.TRAIN_OUT_NAMES, r[:6])))
                put('train_forward/%d/%d' % (int(no_first_img), call), {'prev_%d' % i: t for i, t in enumerate(r[6])})
                prev = r[6]
    # gradients of one scalar objective over every output of a coarse generator
    opt = make_opt(ngf=8, n_blocks=2, fg=True, n_downsample_G=2, gpu_ids=[])
    net = det_fill_(N.define_G(18, 3, 6, 8, 'composite', 2, 'batch', 0, [], opt), seed=31)
    C.condition_flow_heads(net, 0.05)
    inp, img_prev, mask = RI.gen_inputs(6, 16, 32, seed=2)
    x_r, p_r = inp.clone().requires_grad_(True), img_prev.clone().requires_grad_(True)
    outs = net(x_r, p_r, mask, None, None, None, False)
    RI.objective(outs, RI.cotangents(outs)).backward()
    put('grad', {k: v.grad for k, v in net.named_parameters()})
    put('grad', {'input': x_r.grad, 'img_prev': p_r.grad})
    # training losses of Vid2VidModelD.forward (--no_vgg)
    ref_shim.install()
    from models.vid2vid_model_D import Vid2VidModelD          # noqa (reference module)
    for tag, kw in RI.LOSS_MODELS.items():
        opt = RI.loss_opt(**kw)
        opt.add_face_disc = False
        m = Vid2VidModelD()
        m.initialize(opt)
        det_fill_(m.netD, seed=RI.D_SEED)
        det_fill_(m.netD_T0, seed=RI.D_T_SEED)
        with torch.no_grad():
            if tag == 'temporal':
                put('losses/' + tag, dict(zip(RI.LOSS_NAMES_T, m.forward(1, RI.temporal_loss_inputs(opt)))))
            else:
                put('losses/' + tag, dict(zip(RI.LOSS_NAMES, m.forward(0, RI.spatial_loss_inputs(opt, kw['no_first_img'], tag == 'raw')))))
    # FlowNet2: the network, its sub-networks and the vid2vid wrapper on deterministic weights
    from oracle import flownet2_oracle as FO
    F2 = ref_shim.flownet2_class()
    fnet = F2().eval()
    fnet.load_state_dict(FO.det_state_dict([[k, list(v.shape)] for k, v in fnet.state_dict().items()], seed=RI.FLOWNET_SEED))
    from models.flownet import FlowNet                                                        # noqa (reference module)
    from models.flownet2_pytorch.networks.resample2d_package.resample2d import Resample2d     # noqa
    stub = types.SimpleNamespace(flowNet=fnet, resample=Resample2d())
    stub.norm = lambda t: FlowNet.norm(stub, t)
    fi = RI.flownet_inputs()
    with torch.no_grad():
        put('flownet2', {'pair': fnet(fi['pair']), 'c': fnet.flownetc(fi['x6'])[0], 's': fnet.flownets_1(fi['x12'])[0],
                         'sd': fnet.flownets_d(fi['x6'])[0], 'fusion': fnet.flownetfusion(fi['xf'])})
        for h, w in RI.FLOWNET_WRAPPER_SIZES:
            f, c = FlowNet.compute_flow_and_conf(stub, *RI.flownet_wrapper_inputs(h, w))
            put('flownet2', {'wrapper_flow_%dx%d' % (h, w): f, 'wrapper_conf_%dx%d' % (h, w): c})
        fnet.load_state_dict(FO.det_state_dict([[k, list(v.shape)] for k, v in fnet.state_dict().items()], seed=7))
        put('flownet2', {'pair_128x192': fnet(RI.flownet_pair_128x192())})
    save_fixture('reference', out)

    # BaseModel: learning-rate schedule, frame-count schedule, fixed-parameter release, checkpoint file
    ref_shim.install()
    from models.base_model import BaseModel                   # noqa (reference module)
    with tempfile.TemporaryDirectory() as tmp:
        opt = RI.schedule_opt(tmp)
        ref = RI.schedule_state(opt, BaseModel)
        ref.save_dir = os.path.join(tmp, 'ref')
        os.makedirs(ref.save_dir)
        rec = {'lr': [], 'batch': []}
        for epoch in RI.SCHEDULE_EPOCHS:
            ref.update_learning_rate(epoch, 'G')
            rec['lr'].append([ref.old_lr, [g['lr'] for g in ref.optimizer_G.param_groups]])
        for ratio in RI.SCHEDULE_RATIOS:
            ref.update_training_batch(ratio)
            rec['batch'].append([ref.n_frames_bp, ref.n_frames_per_gpu, ref.n_frames_load])
        ref.update_fixed_params()
        rec['finetune_all'] = bool(ref.finetune_all)
        rec['n_params_after_release'] = sum(p.numel() for g in ref.optimizer_G.param_groups for p in g['params'])
        rec['lr_after_release'] = ref.optimizer_G.param_groups[0]['lr']
        ref.save_network(ref.netG1, 'G1', 'latest', [])
        rec['checkpoint_files'] = sorted(os.listdir(ref.save_dir))
        saved = torch.load(os.path.join(ref.save_dir, 'latest_net_G1.pth'))
        rec['checkpoint'] = {k: {'shape': list(v.shape), 'values': v.flatten().tolist()} for k, v in saved.items()}
    with open(os.path.join(OUT, 'host_schedule.json'), 'w') as f:
        json.dump(rec, f, indent=1)
    print('host_schedule.json', rec)


if __name__ == '__main__':
    names = sys.argv[1:] or (list(C.CASES) + ['keys'])
    for n in names:
        if n == 'keys':
            dump_keys()
        elif n == 'flownet2':
            flownet2_golden()
        elif n == 'reference_checks':
            reference_checks()
        else:
            run_case(n, C.CASES[n])
