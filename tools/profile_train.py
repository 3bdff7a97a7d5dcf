"""Kernel-time breakdown of one training step (torch.profiler / CUPTI): python tools/profile_train.py [workload] [out.txt]"""
import os, sys, tempfile
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import torch
import bench
from vid2vid_b200 import flownet as FN
from vid2vid_b200.model_d import Vid2VidModelD
from vid2vid_b200.model_g import Vid2VidModelG
from vid2vid_b200.trainer import Trainer
from vid2vid_b200.utils import make_opt, synth_label_sequence

wl_name = sys.argv[1] if len(sys.argv) > 1 else 'cfg3'
out_path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(tempfile.gettempdir(), 'profile_train_%s.txt' % wl_name)
wl = bench.WORKLOADS[wl_name]
H, Wd = wl['H'], wl['W']
opt = make_opt(label_nc=35, use_instance=True, fg=True, fg_labels=[26], n_scales_spatial=wl['n_scales'], ngf=wl['ngf'], num_D=3,
               n_scales_temporal=2, n_frames_D=3, isTrain=True, no_vgg=True, gpu_ids=[0], n_frames_total=30, dataroot='datasets/Cityscapes/', loadSize=Wd)
torch.manual_seed(1234)
G = Vid2VidModelG().initialize(opt); D = Vid2VidModelD().initialize(opt); F = FN.FlowNet().initialize(opt)
tr = Trainer(opt, G, D, F, world=1)
tG = opt.n_frames_G
T = 12
A = synth_label_sequence(T, H, Wd, label_nc=35, block=64, seed=0).cuda()
g = torch.Generator().manual_seed(77)
coarse = torch.rand(T, 3, H // 16, Wd // 16, generator=g) * 2 - 1
B = torch.nn.functional.interpolate(coarse, size=(H, Wd), mode='bilinear', align_corners=False).view(1, T, 3, H, Wd).cuda()
NW_ = int(os.environ.get('PROFILE_WARMUP', '5'))
for t in range(NW_):
    tr.step(A[:, t % 9:t % 9 + tG], B[:, t % 9:t % 9 + tG], A[:, t % 9:t % 9 + tG])
torch.cuda.synchronize()
if os.environ.get('PROFILE_CPU'):
    import cProfile, pstats, time
    pr = cProfile.Profile()
    t0 = time.time()
    pr.enable()
    pend = [tr.step_async(A[:, t:t + tG], B[:, t:t + tG], A[:, t:t + tG]) for t in range(5, 8)]
    pr.disable()
    t1 = time.time()
    torch.cuda.synchronize()
    print('host issue time of 3 steps: %.1f ms each (then %.1f ms until the GPU was done)' % ((t1 - t0) / 3 * 1e3, (time.time() - t1) * 1e3))
    print('3 steps wall %.1f ms each' % ((time.time() - t0) / 3 * 1e3))
    st = pstats.Stats(pr)
    st.sort_stats('cumulative').print_stats(45)
    st.sort_stats('tottime').print_stats(30)
    sys.exit(0)
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    t = 5
    tr.step(A[:, t:t + tG], B[:, t:t + tG], A[:, t:t + tG])
    torch.cuda.synchronize()
rows = sorted(prof.key_averages(), key=lambda r: -r.device_time_total)
tot = sum(r.device_time_total for r in rows)
with open(out_path, 'w') as f:
    f.write('one %s training step: %.1f ms of kernel time over %d launches\n' % (wl_name, tot / 1e3, sum(r.count for r in rows)))
    for r in rows[:40]:
        f.write('%8.2f ms %5.1f %% %6d x  %s\n' % (r.device_time_total / 1e3, 100 * r.device_time_total / tot, r.count, r.key[:110]))
print(open(out_path).read())
# per-launch durations of the weight-gradient kernel in launch order (pair with the V2V_WG_LOG=1 lines on stderr)
evs = [e for e in prof.events() if 'wgrad_umma_kernel' in e.name]
evs.sort(key=lambda e: e.time_range.start)
print('WGRAD_US ' + ' '.join('%.0f' % e.device_time for e in evs))
evs = [e for e in prof.events() if 'conv_umma_kernel' in e.name]
evs.sort(key=lambda e: e.time_range.start)
print('CONV_US ' + ' '.join('%.0f' % e.device_time for e in evs))
