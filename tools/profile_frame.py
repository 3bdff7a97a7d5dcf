"""Per-kernel device-time breakdown of one steady-state frame (CUDA events after every kernel,
v2v_plan_profile).  Usage: python tools/profile_frame.py [workload] [out_prefix]"""
import json
import os
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import torch                                       # noqa: E402
import bench                                       # noqa: E402
from vid2vid_b200.model_g import Vid2VidModelG     # noqa: E402
from vid2vid_b200.utils import synth_label_sequence   # noqa: E402

KINDS = {0: 'import', 1: 'conv', 2: 'rawstats', 3: 'finalize', 4: 'apply', 5: 'export', 6: 'composite', 7: 'memset'}


def main():
    wl_name = sys.argv[1] if len(sys.argv) > 1 else 'cfg4'
    prefix = sys.argv[2] if len(sys.argv) > 2 else os.path.join(tempfile.gettempdir(), 'profile_' + wl_name)
    wl = bench.WORKLOADS[wl_name]
    opt = bench.make_opt_for(wl_name)
    torch.manual_seed(0)
    model = Vid2VidModelG().initialize(opt)
    seq = synth_label_sequence(8, wl['H'], wl['W'], label_nc=35, block=64, seed=0).cuda()
    for t in range(4):
        model.inference(seq[:, t:t + 3], None, seq[:, t:t + 3])
    torch.cuda.synchronize()
    rows = []
    for s in range(wl['n_scales']):
        net = getattr(model, 'netG%d' % s)
        for ent in net._plans().values():
            plan = ent['plan']
            convs = plan.describe()['convs']
            ci = 0
            best = None
            for rep in range(3):
                prof = plan.profile()
                if best is None:
                    best = [list(p) for p in prof]
                else:
                    for b, p in zip(best, prof):
                        b[1] = min(b[1], p[1])
            for kind, ms, macs in best:
                r = {'scale': s, 'op': KINDS[kind], 'ms': ms}
                if kind == 1:
                    c = convs[ci]
                    ci += 1
                    r.update(c)
                    r['macs'] = macs
                    r['tflops'] = 2 * macs / (ms * 1e-3) / 1e12 if ms > 0 else 0
                rows.append(r)
    total = sum(r['ms'] for r in rows)
    lines = ['total %.3f ms over %d kernels' % (total, len(rows))]
    bykind = {}
    for r in rows:
        bykind[r['op']] = bykind.get(r['op'], 0) + r['ms']
    lines.append('by kind: ' + ', '.join('%s %.3f' % kv for kv in sorted(bykind.items(), key=lambda kv: -kv[1])))
    agg = {}
    for r in rows:
        if r['op'] != 'conv':
            continue
        key = (r['scale'], r['Cin'], r['Cout'], tuple(r['k']), r['stride'], r['transposed'], tuple(r['grid']), r['R'], r['TH'], r['TW'])
        a = agg.setdefault(key, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += r['ms']
        a[2] += r['macs']
    lines.append('%-5s %-5s %-5s %-6s %-2s %-2s %-11s %-2s %-7s %5s %9s %8s %8s' % ('scale', 'Cin', 'Cout', 'k', 's', 'T', 'grid', 'R', 'tile', 'n', 'ms', 'GMAC', 'TFLOP/s'))
    for key, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        s, cin, cout, k, st, tr, grid, R, TH, TW = key
        lines.append('%-5d %-5d %-5d %-6s %-2d %-2d %-11s %-2d %-7s %5d %9.3f %8.2f %8.1f' % (
            s, cin, cout, '%dx%d' % k, st, tr, '%dx%d' % grid, R, '%dx%d' % (TH, TW), a[0], a[1], a[2] / 1e9, 2 * a[2] / (a[1] * 1e-3) / 1e12))
    txt = '\n'.join(lines)
    print(txt)
    os.makedirs(os.path.dirname(prefix), exist_ok=True)
    open(prefix + '.txt', 'w').write(txt + '\n')
    json.dump(rows, open(prefix + '.json', 'w'))


if __name__ == '__main__':
    main()
