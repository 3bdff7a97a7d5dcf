"""Host-only: print the kernel configuration (tile, K block, N tile, stages) the plan runtime picks for every distinct
convolution of a workload in both arithmetic modes.  python tools/dump_configs.py [workload]"""
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import bench                                  # noqa: E402
from vid2vid_b200 import networks as NW       # noqa: E402
from vid2vid_b200.plan import Plan            # noqa: E402

wl = sys.argv[1] if len(sys.argv) > 1 else 'cfg4'
W = bench.WORKLOADS[wl]
opt = bench.make_opt_for(wl)
opt.gpu_ids = []
for mode in ('fast', 'precise'):
    print(mode)
    seen = set()
    for s, net in enumerate(NW.build_netGs(opt)):
        sc = 2 ** (W['n_scales'] - 1 - s)
        plan = Plan(0, precision=mode)
        net._describe(plan, 1, W['H'] // sc, W['W'] // sc)
        for c in plan.describe()['convs']:
            key = (s, c['Cin'], c['Cout'], tuple(c['k']), c['stride'], c['transposed'], tuple(c['grid']))
            if key in seen:
                continue
            seen.add(key)
            print(' s%d %4d->%4d k%d s%d T%d grid %-12s tile %2dx%-3d R%-2d BN%-3d kc%d MG%d CG%-2d SG%d res%d units %d' % (
                s, c['Cin'], c['Cout'], c['k'][0], c['stride'], c['transposed'], c['grid'], c['TH'], c['TW'], c['R'], c['BN'],
                c['kc'], c['MG'], c['CG'], c['SG'], c['resident'], c['units']))
