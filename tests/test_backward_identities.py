"""CPU: the algebra the tensor-core backward rests on (csrc/plan_backward.cu:build_backward_units), checked with PyTorch autograd in
fp64.  The data gradient of every conv of a training plan is evaluated as a FORWARD conv of the output gradient:

  mode 1  stride-1 conv, pad p (reflect or zero)  -> stride-1 conv of dY with zero pad k - 1 and transposed + flipped weights; the
                                                     result lives on the padded input extent and the halo is folded back
  mode 2  transposed conv (stride 2)              -> stride-2 conv of dY with the SAME weight tensor
  mode 3  stride-2 conv                           -> transposed conv of dY with the SAME weight tensor, asked for 2 oh x 2 ow outputs
                                                     (output_padding 2 + 2p - k) and cropped to the input extent

and the weight gradient as sum over pixels of dY[pixel] (x) X[pixel @ tap] with the tap -> (parity plane, offset) table of the
forward conv.  The GPU tests compare the kernels with fp64 autograd; these tests pin the identities themselves."""
import pytest
import torch
import torch.nn.functional as F


def _fold_reflect(gpad, p):
    """Adjoint of ReflectionPad2d(p): fold the halo of a gradient on the padded extent back onto the interior."""
    H, W = gpad.shape[-2] - 2 * p, gpad.shape[-1] - 2 * p
    # rows first (over the full padded width, so the corners travel with them), then columns
    rows = gpad.clone()
    for i in range(1, p + 1):
        rows[..., p + i, :] += gpad[..., p - i, :]
        rows[..., p + H - 1 - i, :] += gpad[..., p + H - 1 + i, :]
    out = rows[..., p:p + H, p:p + W].clone()
    for j in range(1, p + 1):
        out[..., :, j] += rows[..., p:p + H, p - j]
        out[..., :, W - 1 - j] += rows[..., p:p + H, p + W - 1 + j]
    return out


@pytest.mark.parametrize('k,p,reflect', [(3, 1, True), (7, 3, True), (4, 2, False), (3, 1, False)])
def test_mode1_stride1_data_gradient_is_a_forward_conv(k, p, reflect):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 9, 11, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(7, 5, k, k, generator=g, dtype=torch.float64)
    xp = F.pad(x, (p, p, p, p), mode='reflect') if reflect else F.pad(x, (p, p, p, p))
    y = F.conv2d(xp, w)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, x, dy)
    wt = w.transpose(0, 1).flip(2, 3)                                    # [Cin][Cout][k][k], taps flipped
    gpad = F.conv2d(F.pad(dy, (k - 1,) * 4), wt)                         # gradient on the padded input extent
    assert gpad.shape[-2:] == (x.shape[-2] + 2 * p, x.shape[-1] + 2 * p)
    ours = _fold_reflect(gpad, p) if reflect else gpad[..., p:p + x.shape[-2], p:p + x.shape[-1]]
    assert torch.allclose(ours, ref, atol=1e-10)


def test_mode2_transposed_conv_data_gradient_is_a_stride2_conv_with_the_same_weights():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 6, 5, 7, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(6, 4, 3, 3, generator=g, dtype=torch.float64)        # ConvTranspose2d weight [Cin][Cout][k][k]
    y = F.conv_transpose2d(x, w, stride=2, padding=1, output_padding=1)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, x, dy)
    ours = F.conv2d(dy, w, stride=2, padding=1)                          # the same tensor read as [Cout' = Cin][Cin' = Cout][k][k]
    assert torch.allclose(ours, ref, atol=1e-10)


@pytest.mark.parametrize('k,p,H,W', [(3, 1, 8, 12), (3, 1, 9, 13), (4, 2, 8, 12), (4, 2, 10, 16)])
def test_mode3_stride2_conv_data_gradient_is_a_cropped_transposed_conv(k, p, H, W):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 5, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(6, 5, k, k, generator=g, dtype=torch.float64)
    y = F.conv2d(x, w, stride=2, padding=p)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, x, dy)
    oh, ow = y.shape[-2:]
    # the kernel is asked for 2 oh x 2 ow outputs: (oh - 1) * 2 - 2p + k + op with op = 2 + 2p - k (2 for 4x4 / pad 2, which
    # nn.ConvTranspose2d rejects, so the extra rows are produced here by zero-extending dY)
    full = F.conv_transpose2d(F.pad(dy, (0, 1, 0, 1)), w, stride=2, padding=p)
    assert full.shape[-2] >= 2 * oh and 2 * oh >= H and 2 * ow >= W
    assert torch.allclose(full[..., :H, :W], ref, atol=1e-10)


@pytest.mark.parametrize('k,p,s', [(3, 1, 1), (7, 3, 1), (3, 1, 2), (4, 2, 2)])
def test_weight_gradient_as_a_sum_over_pixels_with_the_tap_table(k, p, s):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 10, 14, generator=g, dtype=torch.float64)
    w = torch.randn(6, 4, k, k, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(F.pad(x, (p,) * 4), w, stride=s)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, w, dy)
    xp = F.pad(x, (p,) * 4)
    Hp, Wp = xp.shape[-2:]
    oh, ow = y.shape[-2:]
    ours = torch.zeros_like(ref)
    if s == 1:
        for ky in range(k):
            for kx in range(k):                                          # IN buffer coordinate of grid pixel (y, x): (y + ky, x + kx)
                win = xp[..., ky:ky + oh, kx:kx + ow]
                ours[:, :, ky, kx] = torch.einsum('nohw,nihw->oi', dy, win)
    else:
        # parity planes of the padded input: plane (ky & 1, kx & 1), offset (ky >> 1, kx >> 1)
        planes = {(a, b): xp[..., a::2, b::2] for a in (0, 1) for b in (0, 1)}
        for ky in range(k):
            for kx in range(k):
                pl = planes[(ky & 1, kx & 1)]
                win = pl[..., (ky >> 1):(ky >> 1) + oh, (kx >> 1):(kx >> 1) + ow]
                ours[:, :, ky, kx] = torch.einsum('nohw,nihw->oi', dy, win)
    assert torch.allclose(ours, ref, atol=1e-9)
