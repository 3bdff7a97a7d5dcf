"""CPU-only: the lowering halves the 128-wide N tile of a precise conv whose work units would fit in one round over the SMs
(the 512->512 and 1024->1024 3x3 convs at the coarsest cfg4 scale), and leaves other layers alone.  With no device the lowering
assumes the H100 SXM's 132 SMs; on a GPU host the test runs only on a 132-SM device."""
import pytest
import torch
import torch.nn as nn

from vid2vid_b200 import networks as NW
from vid2vid_b200.plan import Plan

BN = NW.get_norm_layer('batch')


@pytest.fixture(autouse=True)
def _h100_sxm():
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip('describes a 132-SM H100 SXM')


def _conv(cin, cout, shape, mode, stride=1):
    layers = [nn.ReflectionPad2d(1), nn.Conv2d(cin, cout, 3, stride=stride), BN(cout), nn.ReLU(True)]
    r = NW.SequentialRunner(layers)
    p = Plan(0, precision=mode)
    r._describe(p, *shape)
    (c,) = p.describe()['convs']
    return c


def test_precise_512_conv_at_32x64_splits_its_n_tile():
    c = _conv(512, 512, (1, 512, 32, 64), 'precise')
    assert (c['BN'], c['units'], c['ring2'], c['resident']) == (64, 128, 0, 0), c


def test_precise_1024_conv_at_32x64_splits_its_n_tile():
    c = _conv(1024, 1024, (1, 1024, 32, 64), 'precise')
    assert (c['BN'], c['units'], c['SG'], c['ring2'], c['resident']) == (64, 256, 3, 0, 0), c


def test_precise_strided_256_to_512_splits_its_n_tile():
    c = _conv(256, 512, (1, 256, 64, 128), 'precise', stride=2)
    assert (c['BN'], c['units']) == (64, 128), c


@pytest.mark.parametrize('cin,cout,shape,mode,bn,units', [
    (1024, 1024, (1, 1024, 64, 64), 'precise', 128, 256),    # more units than SMs
    (512, 512, (1, 512, 32, 64), 'fast', 128, 64),           # fast plans keep their tiling
    (128, 128, (1, 128, 256, 512), 'precise', 128, 1024),    # many units
])
def test_other_layers_keep_their_n_tile(cin, cout, shape, mode, bn, units):
    c = _conv(cin, cout, shape, mode)
    assert (c['BN'], c['units']) == (bn, units), c
