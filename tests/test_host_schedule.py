"""CPU: the host-side checkpoint / schedule helpers (vid2vid_b200/base_model.py) against the reference's BaseModel
(models/base_model.py:43-48,154-181) run on the same state: what it did is stored in tests/golden/host_schedule.json
(oracle/make_golden.py reference_checks)."""
import json
import os

import torch

import reference_inputs as RI
from vid2vid_b200.base_model import HostScheduleMixin


class _Ours(HostScheduleMixin):
    pass


REF = json.load(open(os.path.join(RI.GOLD, 'host_schedule.json')))


def test_schedules_match_the_reference(tmp_path):
    opt = RI.schedule_opt(tmp_path)
    ours = RI.schedule_state(opt, _Ours)
    for epoch, (old_lr, lrs) in zip(RI.SCHEDULE_EPOCHS, REF['lr']):
        ours.update_learning_rate(epoch, 'G')
        assert ours.old_lr == old_lr
        assert [g['lr'] for g in ours.optimizer_G.param_groups] == lrs
    for ratio, batch in zip(RI.SCHEDULE_RATIOS, REF['batch']):          # train.py:121-123: every niter_step epochs
        ours.update_training_batch(ratio)
        assert [ours.n_frames_bp, ours.n_frames_per_gpu, ours.n_frames_load] == batch
    assert ours.n_frames_per_gpu == 8
    ours.update_fixed_params()
    assert ours.finetune_all and REF['finetune_all']
    n_ours = sum(p.numel() for g in ours.optimizer_G.param_groups for p in g['params'])
    assert n_ours == REF['n_params_after_release'] == sum(p.numel() for m in (ours.netG0, ours.netG1) for p in m.parameters())
    assert ours.optimizer_G.param_groups[0]['lr'] == REF['lr_after_release'] == ours.old_lr


def test_save_network_writes_the_reference_file_and_keeps_the_parameters_in_place(tmp_path):
    opt = RI.schedule_opt(tmp_path)
    ours = RI.schedule_state(opt, _Ours)
    ptrs = [p.data_ptr() for p in ours.netG1.parameters()]
    path = ours.save_network(ours.netG1, 'G1', 'latest', [])
    assert [os.path.basename(path)] == REF['checkpoint_files'] and os.path.dirname(path) == os.path.join(opt.checkpoints_dir, opt.name)
    a = torch.load(path)
    assert list(a) == list(REF['checkpoint'])                              # the reference's file: same keys, same order ...
    for k, ref in REF['checkpoint'].items():                               # ... and the tensors it saved for the same module
        assert a[k].device.type == 'cpu' and torch.equal(a[k], torch.tensor(ref['values'], dtype=torch.float32).view(ref['shape'])), k
    assert ptrs == [p.data_ptr() for p in ours.netG1.parameters()]          # no .cpu() / .cuda() round trip of the module
