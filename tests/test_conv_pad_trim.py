"""CPU: the tensor-core work conv_umma_kernel skips on padded channels, as v2v_plan_describe reports it.

kmma_last: k16 MMA steps of the last K block, only those that reach an input channel below Cin (the packed weights of the
padded channels [Cin, Cp) are zero).  BNt: MMA width of the last N tile, its valid output columns rounded up to 16, where
the kernel has an instantiation of that width.  The 7x7 stems over the 108-channel label input (3 frames x 35 one-hot
labels + 1 edge channel, padded to 128) are the layers these matter for."""
import pytest

import product_plans as PP
from product_plans import h100_sxm  # noqa: F401  (autouse: the tilings below are those of a 132-SM H100 SXM)


def _cfg4_convs(mode):
    """[describe() convs of scale s] of the cfg4 generators, as bench.py lowers them."""
    return [PP.describe(s)['convs'] for s in PP.group('bench') if s.tag.startswith('cfg4 ') and s.precision == mode]


# mode, scale, Cout -> (BN, BNt, kc, kmma, kmma_last)
STEMS = {
    ('fast', 0, 192): (64, 64, 64, 4, 3),
    ('fast', 1, 96): (96, 96, 32, 2, 1),
    ('fast', 2, 48): (64, 48, 64, 4, 3),
    ('precise', 0, 192): (128, 64, 64, 4, 3),
    ('precise', 1, 96): (96, 96, 64, 4, 3),
    ('precise', 2, 48): (64, 48, 32, 2, 1),
}


@pytest.mark.parametrize('mode', ['fast', 'precise'])
def test_cfg4_stems_issue_only_valid_columns_and_k_steps(mode):
    convs = _cfg4_convs(mode)
    for (m, s, cout), want in STEMS.items():
        if m != mode:
            continue
        stems = [c for c in convs[s] if c['Cin'] == 108 and c['k'] == [7, 7]]
        assert len(stems) == 1 and stems[0]['Cout'] == cout, (s, [(c['Cin'], c['Cout']) for c in stems])
        c = stems[0]
        assert (c['BN'], c['BNt'], c['kc'], c['kmma'], c['kmma_last']) == want, (mode, s, c)


@pytest.mark.parametrize('mode', ['fast', 'precise'])
def test_unpadded_convs_keep_full_widths(mode):
    n = 0
    for convs in _cfg4_convs(mode):
        for c in convs:
            if c['Cin'] % 16 == 0 and c['Cin'] == c['Cp'] and c['Cout'] % c['BN'] == 0:
                assert c['kmma_last'] == c['kmma'] and c['BNt'] == c['BN'], c
                n += 1
            assert 1 <= c['kmma_last'] <= c['kmma'] and 16 <= c['BNt'] <= c['BN'], c
    assert n >= 10, n
