"""Stand-alone operators: thin Python wrappers over group (1) of the C ABI, mirroring the reference's
operator surface (same class names / argument meaning / output-ownership rules):

  Correlation / Resample2d / ChannelNorm  <- models/flownet2_pytorch/networks/*_package/*.py
  resample(image, flow)                   <- BaseModel.resample (models/base_model.py:189-196)
  onehot_edges / avgpool3s2 / fg_mask     <- Vid2VidModelG.encode_input / build_pyr / compute_mask
  instance_mean / face_features           <- Encoder.forward's pooling / Vid2VidModelG.get_face_features (edge2face)
  face_region                             <- Vid2VidModelD.get_face_region's pixel search (pose face discriminator)

CUDA fp32 contiguous tensors only; errors from the library raise RuntimeError (the reference's
wrapper raises via AT_ERROR, correlation_cuda.cc:81-83).  No CPU fallback.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib as L


def _chk(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda or t.dtype != torch.float32:
            raise RuntimeError('vid2vid_b200 ops need CUDA float32 tensors (no CPU fallback)')
        if not t.is_contiguous():
            raise RuntimeError('vid2vid_b200 ops need contiguous tensors')   # resample2d.py:9-10, channelnorm.py:9


def _ck(rc):
    L.check(rc)
    L.LAUNCHES[0] += 1


def _on(t):
    """Context for a launch on tensor t's device (correlation.py:21 `with torch.cuda.device_of(input1)`); pair it with
    _st(t), the caller's current stream on THAT device."""
    return torch.cuda.device_of(t)


def _st(t):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def correlation(input1, input2, pad_size=20, kernel_size=1, max_displacement=20, stride1=1, stride2=2,
                corr_multiply=1):
    """CorrelationFunction.forward (correlation.py:18-30)."""
    _chk(input1, input2)
    n, c, h, w = input1.shape
    oc, oh, ow = C.c_int(), C.c_int(), C.c_int()
    L.check(L.lib().v2v_correlation_out_shape(h, w, pad_size, kernel_size, max_displacement, stride1, stride2,
                                              C.byref(oc), C.byref(oh), C.byref(ow)))
    out = torch.empty((n, oc.value, oh.value, ow.value), device=input1.device, dtype=torch.float32)
    with torch.cuda.device_of(input1):
        _ck(L.lib().v2v_correlation_forward(_p(input1), _p(input2), _p(out), n, c, h, w, pad_size, kernel_size,
                                                max_displacement, stride1, stride2, corr_multiply, _st(input1)))
    return out


class Correlation(nn.Module):
    """correlation.py:47-61."""

    def __init__(self, pad_size=0, kernel_size=0, max_displacement=0, stride1=1, stride2=2, corr_multiply=1):
        super().__init__()
        self.pad_size, self.kernel_size, self.max_displacement = pad_size, kernel_size, max_displacement
        self.stride1, self.stride2, self.corr_multiply = stride1, stride2, corr_multiply

    def forward(self, input1, input2):
        return correlation(input1.contiguous(), input2.contiguous(), self.pad_size, self.kernel_size,
                           self.max_displacement, self.stride1, self.stride2, self.corr_multiply)


def resample2d(input1, input2, kernel_size=1):
    """Resample2dFunction.forward (resample2d.py:8-21)."""
    _chk(input1, input2)
    _, d, ih, iw = input1.shape
    b, _, h, w = input2.shape
    out = torch.empty((b, d, h, w), device=input1.device, dtype=torch.float32)
    with torch.cuda.device_of(input1):
        _ck(L.lib().v2v_resample2d_forward(_p(input1), _p(input2), _p(out), b, d, h, w, ih, iw, kernel_size, _st(input1)))
    return out


class Resample2d(nn.Module):
    """resample2d.py:38-46."""

    def __init__(self, kernel_size=1):
        super().__init__()
        self.kernel_size = kernel_size

    def forward(self, input1, input2):
        return resample2d(input1.contiguous(), input2.contiguous(), self.kernel_size)


def channelnorm(input1, norm_deg=2):
    """ChannelNormFunction.forward (channelnorm.py:7-17)."""
    _chk(input1)
    b, c, h, w = input1.shape
    out = torch.empty((b, 1, h, w), device=input1.device, dtype=torch.float32)
    with torch.cuda.device_of(input1):
        _ck(L.lib().v2v_channelnorm_forward(_p(input1), _p(out), b, c, h, w, norm_deg, _st(input1)))
    return out


class ChannelNorm(nn.Module):
    """channelnorm.py:31-38."""

    def __init__(self, norm_deg=2):
        super().__init__()
        self.norm_deg = norm_deg

    def forward(self, input1):
        return channelnorm(input1.contiguous(), self.norm_deg)


def _resample_fwd(image, flow, align_corners):
    image, flow = image.contiguous(), flow.contiguous()
    _chk(image, flow)
    b, c, h, w = image.shape
    out = torch.empty_like(image)
    with _on(image):
        _ck(L.lib().v2v_resample_forward(_p(image), _p(flow), _p(out), b, c, h, w, int(align_corners), _st(image)))
    return out


class ResampleFunction(torch.autograd.Function):
    """resample with gradients wrt image and flow (the warp losses differentiate through it, vid2vid_model_D.py:123)."""

    @staticmethod
    def forward(ctx, image, flow, align_corners):
        image, flow = image.detach().contiguous(), flow.detach().contiguous()
        ctx.save_for_backward(image, flow)
        ctx.ac = int(align_corners)
        return _resample_fwd(image, flow, align_corners)

    @staticmethod
    def backward(ctx, g):
        image, flow = ctx.saved_tensors
        b, c, h, w = image.shape
        g = g.contiguous()
        gi = torch.zeros_like(image) if ctx.needs_input_grad[0] else None
        gf = torch.empty_like(flow) if ctx.needs_input_grad[1] else None
        _ck(L.lib().v2v_resample_backward(_p(image), _p(flow), _p(g), _p(gi), _p(gf), b, c, h, w, ctx.ac, L.current_stream_ptr()))
        return gi, gf, None


def resample(image, flow, align_corners=False):
    """BaseModel.resample / BaseNetwork.resample (base_model.py:189-196, networks.py:108-115)."""
    if torch.is_grad_enabled() and (image.requires_grad or flow.requires_grad):
        return ResampleFunction.apply(image, flow, align_corners)
    return _resample_fwd(image, flow, align_corners)


def onehot_edges(label_map, inst_map, label_nc, use_instance):
    """encode_input + get_edges (vid2vid_model_G.py:86-112, base_model.py:146-152).
    label_map / inst_map: (b, t, 1, H, W) float ids -> (b, t, label_nc [+1], H, W)."""
    label_map = label_map.contiguous()
    inst = inst_map.contiguous() if use_instance else None
    _chk(label_map, inst)
    b, t, _, h, w = label_map.shape
    out = torch.empty((b, t, label_nc + int(bool(use_instance)), h, w), device=label_map.device, dtype=torch.float32)
    with _on(label_map):
        _ck(L.lib().v2v_onehot_edges(_p(label_map), _p(inst), _p(out), b * t, label_nc, int(bool(use_instance)), h, w, _st(label_map)))
    return out


class AvgPool3s2Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.shape = x.shape
        return _avgpool3s2_fwd(x.detach())

    @staticmethod
    def backward(ctx, g):
        h, w = ctx.shape[-2:]
        g = g.contiguous()
        gin = torch.empty(ctx.shape, device=g.device, dtype=torch.float32)
        _ck(L.lib().v2v_avgpool3s2_backward(_p(g), _p(gin), gin.numel() // (h * w), h, w, L.current_stream_ptr()))
        return gin


def avgpool3s2(x):
    """AvgPool2d(3, stride=2, padding=1, count_include_pad=False) over the last two dims (autograd-aware)."""
    if torch.is_grad_enabled() and x.requires_grad:
        return AvgPool3s2Function.apply(x)
    return _avgpool3s2_fwd(x)


def _avgpool3s2_fwd(x):
    x = x.contiguous()
    _chk(x)
    h, w = x.shape[-2:]
    planes = x.numel() // (h * w)
    out = torch.empty(tuple(x.shape[:-2]) + ((h - 1) // 2 + 1, (w - 1) // 2 + 1), device=x.device, dtype=torch.float32)
    with _on(x):
        _ck(L.lib().v2v_avgpool3s2(_p(x), _p(out), planes, h, w, _st(x)))
    return out


def _avgpool2_fwd(x):
    x = x.contiguous()
    _chk(x)
    h, w = x.shape[-2:]
    out = torch.empty(tuple(x.shape[:-2]) + (h // 2, w // 2), device=x.device, dtype=torch.float32)
    with _on(x):
        _ck(L.lib().v2v_avgpool2(_p(x), _p(out), x.numel() // (h * w), h, w, _st(x)))
    return out


class AvgPool2Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.shape = x.shape
        return _avgpool2_fwd(x.detach())

    @staticmethod
    def backward(ctx, g):
        h, w = ctx.shape[-2:]
        g = g.contiguous()
        gin = torch.empty(ctx.shape, device=g.device, dtype=torch.float32)
        with _on(g):
            _ck(L.lib().v2v_avgpool2_backward(_p(g), _p(gin), gin.numel() // (h * w), h, w, _st(g)))
        return gin


def avgpool2(x):
    """AvgPool2d(2, stride=2, count_include_pad=False) over the last two dims (VGGLoss's downsample, networks.py:782-786);
    autograd-aware."""
    if torch.is_grad_enabled() and x.requires_grad:
        return AvgPool2Function.apply(x)
    return _avgpool2_fwd(x)


def instance_mean(x, inst, n_ids, out=None):
    """Encoder.forward's instance-wise average pooling (models/networks.py:617-632): x (N, C, H, W), inst (N, 1, H, W) float
    ids, integers in [0, n_ids) (anything else raises).  Returns `out` (a new tensor, or x itself for an in-place pass) with
    every value replaced by the mean of its channel over the pixels of its image that share its id.  Deterministic."""
    _chk(x, inst, out)
    N, C, H, W = x.shape
    if inst.numel() != N * H * W:
        raise ValueError('instance_mean: id map %s does not match features %s' % (tuple(inst.shape), tuple(x.shape)))
    if out is None:
        out = torch.empty_like(x)
    with _on(x):
        _ck(L.lib().v2v_instance_mean(_p(x), _p(inst), _p(out), N, C, H, W, int(n_ids), _st(x)))
    return out


def face_features(pooled, inst, table, rows, num_images):
    """get_face_features's nearest-neighbour lookup (models/vid2vid_model_G.py:290-320): pooled (N, feat_num, H, W) Encoder
    output, inst (N, 1, H, W) part labels, table (n_labels, max_rows, feat_num + 1) the packed features.npy, rows the
    per-label row counts (host ints).  Returns (feat_map (N, feat_num, H, W), chosen (1,) int32 device tensor)."""
    _chk(pooled, inst, table)
    N, F_, H, W = pooled.shape
    n_labels, max_rows, stride = table.shape
    if inst.numel() != N * H * W or len(rows) != n_labels:
        raise ValueError('face_features: part map %s / rows %d do not match features %s / table %s' % (
            tuple(inst.shape), len(rows), tuple(pooled.shape), tuple(table.shape)))
    out = torch.empty_like(pooled)
    chosen = torch.empty(1, dtype=torch.int32, device=pooled.device)
    arr = (C.c_int * n_labels)(*[int(r) for r in rows])
    with _on(pooled):
        _ck(L.lib().v2v_face_features(_p(pooled), _p(inst), _p(table), arr, n_labels, max_rows, int(num_images), F_, stride, _p(out),
                                      C.c_void_p(chosen.data_ptr()), N, H, W, _st(pooled)))
    return out, chosen


class FaceRegion:
    """The face box of ops.face_region on its way to the host: one 20-byte copy into pinned memory, queued behind the
    search kernel.  get() waits for that copy only (not for work queued after it) and returns (ymin, ymax, xmin, xmax) as
    host ints, inclusive, or None when no pixel matched."""

    def __init__(self, box):
        self.host = torch.empty(5, dtype=torch.int32, pin_memory=True)
        self.host.copy_(box, non_blocking=True)
        self.event = torch.cuda.Event()
        self.event.record(torch.cuda.current_stream(box.device))

    def get(self):
        self.event.synchronize()
        found, ymin, ymax, xmin, xmax = self.host.tolist()
        return (ymin, ymax, xmin, xmax) if found else None


def face_region(real_A, openpose_only=False):
    """The pixel search of Vid2VidModelD.get_face_region (models/vid2vid_model_D.py:215-230) over the whole batch real_A
    (N, C >= 3, H, W): face pixels are real_A[:, 2] > 0.9, or with openpose_only 0.19 < c0 < 0.21, c1 < -0.99,
    -0.61 < c2 < -0.59 (fp32 comparisons).  Launches the kernel and the copy of its result; returns a FaceRegion."""
    real_A = real_A.contiguous()
    _chk(real_A)
    N, Ch, H, W = real_A.shape
    box = torch.empty(5, dtype=torch.int32, device=real_A.device)
    with _on(real_A):
        _ck(L.lib().v2v_face_region(_p(real_A), N, Ch, H, W, int(bool(openpose_only)), C.c_void_p(box.data_ptr()), _st(real_A)))
        return FaceRegion(box)


def fg_mask(real_As, ts, fg_labels):
    """compute_mask (vid2vid_model_G.py:322-330): (b, T, C, h, w) -> (b, 1, h, w)."""
    real_As = real_As.contiguous()
    _chk(real_As)
    b, T, c, h, w = real_As.shape
    out = torch.empty((b, 1, h, w), device=real_As.device, dtype=torch.float32)
    arr = (C.c_int * len(fg_labels))(*fg_labels)
    with _on(real_As):
        _ck(L.lib().v2v_fg_mask(_p(real_As), _p(out), b, T, c, h, w, ts, arr, len(fg_labels), _st(real_As)))
    return out


# ------------------------------------------------------------------------------------------------ training losses
def _scalar_ws(dev):
    return torch.zeros(1, device=dev, dtype=torch.float64), torch.empty(1, device=dev, dtype=torch.float32)


class L1LossFunction(torch.autograd.Function):
    """mean |a*m - b*m| (MaskedL1Loss, networks.py:804-812) / mean |a - b| (nn.L1Loss) with m = None; b may be None (= 0)."""

    @staticmethod
    def forward(ctx, a, b, mask):
        a = a.detach().contiguous()
        b = b.detach().contiguous() if b is not None else None
        mask = mask.detach().contiguous() if mask is not None else None
        _chk(a, b, mask)
        a4 = a if a.dim() == 4 else a.reshape(-1, a.shape[-3], a.shape[-2], a.shape[-1])
        ctx.dims = a4.shape
        ws, out = _scalar_ws(a.device)
        n, c, h, w = a4.shape
        _ck(L.lib().v2v_l1_loss_forward(_p(a), _p(b), _p(mask), n, c, h, w, C.c_void_p(ws.data_ptr()), _p(out), L.current_stream_ptr()))
        ctx.save_for_backward(a, b, mask)
        return out.reshape(())

    @staticmethod
    def backward(ctx, g):
        a, b, mask = ctx.saved_tensors
        n, c, h, w = ctx.dims
        g = g.reshape(1).contiguous().float()
        ga = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        gb = torch.empty_like(b) if (b is not None and ctx.needs_input_grad[1]) else None
        if ga is None and gb is None:
            return None, None, None
        _ck(L.lib().v2v_l1_loss_backward(_p(a), _p(b), _p(mask), n, c, h, w, _p(g), _p(ga), _p(gb), L.current_stream_ptr()))
        return ga, gb, None


def l1_loss(a, b=None, mask=None):
    return L1LossFunction.apply(a, b, mask)


class MseConstFunction(torch.autograd.Function):
    """mean (x - target)^2 against a constant label: GANLoss with use_lsgan (networks.py:764-774)."""

    @staticmethod
    def forward(ctx, x, target):
        x = x.detach().contiguous()
        _chk(x)
        ctx.t = float(target)
        ws, out = _scalar_ws(x.device)
        _ck(L.lib().v2v_mse_const_forward(_p(x), x.numel(), ctx.t, C.c_void_p(ws.data_ptr()), _p(out), L.current_stream_ptr()))
        ctx.save_for_backward(x)
        return out.reshape(())

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        g = g.reshape(1).contiguous().float()
        gx = torch.empty_like(x)
        _ck(L.lib().v2v_mse_const_backward(_p(x), x.numel(), ctx.t, _p(g), _p(gx), L.current_stream_ptr()))
        return gx, None


def mse_to_const(x, target):
    return MseConstFunction.apply(x, target)
