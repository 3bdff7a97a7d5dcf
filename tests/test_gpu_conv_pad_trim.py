"""GPU parity of the convs whose padded channels conv_umma_kernel skips (tests/test_conv_pad_trim.py): the 108-channel 7x7
stems at shapes that lower the benchmark's tilings (tail N tiles of 48 of 64 and 64 of 128 columns, a last K block of 1 or 3
of its k16 steps; coupled, M-blocked and ring2 paths), and a resident-weight transposed conv with 162 input and 16 output
channels.  References and tolerances as in tests/test_gpu_conv.py: fp64 (precise), bf16-emulated fp32 (fast)."""
import pytest
import torch.nn as nn

import test_gpu_conv as TC
from test_conv_pad_trim import STEMS
from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan

pytestmark = pytest.mark.gpu

BN = NW.get_norm_layer('batch')
FIELDS = ('BN', 'BNt', 'kc', 'kmma', 'kmma_last')

# name, layer list builder, input shape, exact one-hot input, {mode: (BN, BNt, kc, kmma, kmma_last, MG, ring2, resident)}
CASES = [
    # a band of rows at the full 2048 width keeps m_tiles >= 4 x SMs, as the cfg4 finest stem has
    ('stem_108_48_band', lambda: NW._stem(108, 48, BN), (1, 108, 40, 2048), True,
     {m: STEMS[(m, 2, 48)] + (2, 0, 0) for m in ('fast', 'precise')}),
    ('stem_108_96', lambda: NW._stem(108, 96, BN), (1, 108, 80, 1024), False,
     {'fast': STEMS[('fast', 1, 96)] + (1, 0, 0), 'precise': STEMS[('precise', 1, 96)] + (1, 1, 0)}),
    ('stem_108_192', lambda: NW._stem(108, 192, BN), (1, 108, 160, 512), False,
     {'fast': STEMS[('fast', 0, 192)] + (2, 0, 0), 'precise': STEMS[('precise', 0, 192)] + (1, 1, 0)}),
    ('deconv_162_16_resident', lambda: [nn.ConvTranspose2d(162, 16, 4, 2, 1), BN(16), nn.LeakyReLU(0.1, True)], (1, 162, 128, 256),
     False, {m: (32, 32, 64, 4, 3, 1, 0, 1) for m in ('fast', 'precise')}),
]


@pytest.mark.parametrize('mode', TC.MODES)
@pytest.mark.parametrize('name,build,shape,exact,want', CASES, ids=[c[0] for c in CASES])
def test_padded_channel_trim(name, build, shape, exact, want, mode):
    mods = build()
    r = NW.SequentialRunner(mods)
    r.input_exact_bf16 = exact
    p = Plan(0, precision=mode)
    r._describe(p, *shape)
    c = p.describe()['convs'][0]
    assert tuple(c[k] for k in FIELDS + ('MG', 'ring2', 'resident')) == want[mode], c
    x = TC._label_x(*shape) if exact else TC._x(*shape)
    out, ref = TC._run(mods, x, mode=mode, exact=exact)
    TC._check(out, ref, name, mode=mode)
