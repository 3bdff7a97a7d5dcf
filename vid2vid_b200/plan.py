"""Python face of the plan runtime (include/v2v_b200.h group (2)): describe a module once as a
graph of logical values and convolution units, finalize, then run per call against caller tensors."""
import ctypes as C
import json
import os

import torch
import torch.nn as nn

from . import _lib as L


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def conv_desc(m, pad_mode=L.PAD_ZERO, pad=None, m2=None):
    """v2v_conv_desc for an nn.Conv2d / nn.ConvTranspose2d parameter container.  `pad`/`pad_mode`
    override the module's own zero padding when a ReflectionPad2d precedes it."""
    d = L.ConvDesc()
    tr = isinstance(m, nn.ConvTranspose2d)
    d.Cin, d.Cout = m.in_channels, m.out_channels
    d.kh, d.kw = m.kernel_size
    assert m.stride[0] == m.stride[1] and m.padding[0] == m.padding[1]
    d.stride = m.stride[0]
    d.pad = m.padding[0] if pad is None else pad
    d.pad_mode = pad_mode
    d.transposed = int(tr)
    d.output_padding = m.output_padding[0] if tr else 0
    d.weight = m.weight.data_ptr()
    d.bias = m.bias.data_ptr() if m.bias is not None else None
    if m2 is not None:       # second conv with the same geometry stacked along Cout (fused heads)
        assert (m2.in_channels, m2.kernel_size, m2.stride, m2.padding) == (m.in_channels, m.kernel_size, m.stride, m.padding)
        assert (m2.bias is None) == (m.bias is None)
        d.Cout = m.out_channels + m2.out_channels
        d.Cout2 = m2.out_channels
        d.weight2 = m2.weight.data_ptr()
        d.bias2 = m2.bias.data_ptr() if m2.bias is not None else None
    return d


def norm_desc(m):
    d = L.NormDesc()
    if m is None:
        d.kind = L.NORM_NONE
        return d
    d.kind = L.NORM_BATCH if isinstance(m, nn.BatchNorm2d) else L.NORM_INSTANCE
    d.gamma = m.weight.data_ptr() if getattr(m, 'weight', None) is not None else None
    d.beta = m.bias.data_ptr() if getattr(m, 'bias', None) is not None else None
    if getattr(m, 'running_mean', None) is not None:
        d.running_mean = m.running_mean.data_ptr()
        d.running_var = m.running_var.data_ptr()
        d.num_batches_tracked = m.num_batches_tracked.data_ptr()
    d.momentum = m.momentum if m.momentum is not None else 0.1
    d.eps = m.eps
    return d


class Plan:
    def __init__(self, device=0, impl=None, precision='fast', train=False, sample_stats=False):
        if impl is None:
            impl = L.IMPL_SIMT if os.environ.get('V2V_CONV_IMPL') == 'simt' else L.IMPL_UMMA
        self._h = C.c_void_p()
        self.device = device
        self.precision = precision
        L.check(L.lib().v2v_plan_create(device, impl, C.byref(self._h)))
        L.check(L.lib().v2v_plan_set_precision(self._h, {'fast': L.PREC_BF16, 'precise': L.PREC_BF16X3}[precision]))
        self.train = bool(train)
        if train:
            L.check(L.lib().v2v_plan_set_training(self._h, 1))
        # per-sample statistics: image n of the batch is normalised with its own statistics (independent clips)
        self.sample_stats = bool(sample_stats)
        if sample_stats:
            L.check(L.lib().v2v_plan_set_sample_stats(self._h, 1))
        self.run_id = 0
        self._keep = []
        self.finalized = False
        self.n_slots = 0
        self._graph_ok = False
        self.outs = None        # {slot: shape} of the tensors a run writes, as the module that described the plan reports it

    def __del__(self):
        try:
            if self._h:
                L.lib().v2v_plan_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def set_image_flags(self, slot):
        """Per-image flags (v2v_plan_set_image_flags; per-sample inference plans): IO slot `slot` holds an int32 (N,) device
        tensor read at run time -- IMAGE_ACTIVE (the image updates the running statistics) | IMAGE_RAW_ONLY (its composite
        takes the raw image) -- so a captured graph serves every combination."""
        L.check(L.lib().v2v_plan_set_image_flags(self._h, slot))
        self.n_slots = max(self.n_slots, slot + 1)

    # ---- description
    def input(self, slot, N, C_src, c_off, Cn, H, W, exact_bf16=False):
        v = C.c_int()
        L.check(L.lib().v2v_g_input(self._h, slot, N, C_src, c_off, Cn, H, W, 1 if exact_bf16 else 0, C.byref(v)))
        self.n_slots = max(self.n_slots, slot + 1)
        return v.value

    def conv(self, vin, desc):
        r = C.c_int()
        self._keep.append(desc)
        L.check(L.lib().v2v_g_conv(self._h, vin, C.byref(desc), C.byref(r)))
        return r.value

    def norm_act(self, raw, ndesc, act=L.ACT_NONE, slope=0.0, adds=(), c_off=0, Cn=None):
        v = C.c_int()
        if len(adds) > 2:
            raise NotImplementedError('at most two addends per normalise pass')
        adds = list(adds) + [-1, -1]
        self._keep.append(ndesc)
        if Cn is None:
            L.check(L.lib().v2v_g_norm_act(self._h, raw, C.byref(ndesc), act, slope, adds[0], adds[1], C.byref(v)))
        else:
            L.check(L.lib().v2v_g_norm_act_slice(self._h, raw, c_off, Cn, C.byref(ndesc), act, slope, adds[0], adds[1],
                                                 C.byref(v)))
        return v.value

    def conv_act(self, vin, desc, act=L.ACT_NONE, slope=0.0):
        v = C.c_int()
        self._keep.append(desc)
        L.check(L.lib().v2v_g_conv_act(self._h, vin, C.byref(desc), act, slope, C.byref(v)))
        return v.value

    def head(self, vin, desc, channels):
        """channels: list of (slot, channel, dst_C, act, scale), one per output channel."""
        arr = (L.HeadChannel * len(channels))()
        for i, (slot, ch, dst_c, act, scale) in enumerate(channels):
            arr[i].slot, arr[i].channel, arr[i].dst_C, arr[i].act, arr[i].scale = slot, ch, dst_c, act, scale
            self.n_slots = max(self.n_slots, slot + 1)
        self._keep += [desc, arr]
        L.check(L.lib().v2v_g_head(self._h, vin, C.byref(desc), arr))

    def concat(self, values):
        arr = (C.c_int * len(values))(*values)
        v = C.c_int()
        L.check(L.lib().v2v_g_concat(self._h, arr, len(values), C.byref(v)))
        return v.value

    def correlation(self, va, vb, pad_size=20, kernel_size=1, max_displacement=20, stride1=1, stride2=2, act=L.ACT_NONE,
                    slope=0.0):
        v = C.c_int()
        L.check(L.lib().v2v_g_correlation(self._h, va, vb, pad_size, kernel_size, max_displacement, stride1, stride2, act, slope,
                                          C.byref(v)))
        return v.value

    def maxpool2(self, vin):
        v = C.c_int()
        L.check(L.lib().v2v_g_maxpool2(self._h, vin, C.byref(v)))
        return v.value

    def feature_l1(self, vx, vy, slot, index):
        """io[slot][index] = mean |x - y|; y is detached (no gradient, no backward work for what only feeds it)."""
        L.check(L.lib().v2v_g_feature_l1(self._h, vx, vy, slot, index))
        self.n_slots = max(self.n_slots, slot + 1)

    def export(self, v, slot):
        L.check(L.lib().v2v_g_export(self._h, v, slot))
        self.n_slots = max(self.n_slots, slot + 1)

    def composite(self, s_raw, s_flow, s_weight, s_prev, prev_C, s_fg, s_mask, s_final, N, H, W, use_warp,
                  align_corners, s_raw_out=-1):
        L.check(L.lib().v2v_g_composite(self._h, s_raw, s_flow, s_weight, s_prev, prev_C, s_fg, s_mask, s_final, s_raw_out,
                                        N, H, W, int(use_warp), int(align_corners)))
        self.n_slots = max(self.n_slots, s_raw + 1, s_flow + 1, s_weight + 1, s_prev + 1, s_fg + 1, s_mask + 1,
                           s_final + 1, s_raw_out + 1)

    # ---- execution
    def _stream(self):
        """The caller's current stream ON THE PLAN'S DEVICE (which need not be PyTorch's current device)."""
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def finalize(self, workspace=None):
        """workspace: optional caller-owned uint8 CUDA tensor of at least workspace_bytes + 1024 bytes that holds the plan's arena
        (v2v_plan_finalize_ws); the plan keeps a reference so that it outlives the kernels."""
        if workspace is None:
            L.check(L.lib().v2v_plan_finalize(self._h, self._stream()))
        else:
            need = self.workspace_bytes
            base = (workspace.data_ptr() + 1023) // 1024 * 1024
            avail = workspace.data_ptr() + workspace.numel() * workspace.element_size() - base
            if avail < need:
                raise ValueError('workspace holds %d usable bytes, the plan needs %d' % (avail, need))
            self._workspace = workspace
            L.check(L.lib().v2v_plan_finalize_ws(self._h, C.c_void_p(base), need, self._stream()))
        self.finalized = True

    def repack(self):
        L.check(L.lib().v2v_plan_repack(self._h, self._stream()))

    def _io_array(self, io):
        arr = (C.c_void_p * self.n_slots)()
        for i in range(self.n_slots):
            t = io[i] if i < len(io) else None
            arr[i] = t.data_ptr() if t is not None else None
        return arr

    def run(self, io, use_graph=True, recompute=False):
        """io: list indexed by slot of tensors (or None).  recompute: eager re-execution before a backward, without the
        running-statistics side effect."""
        arr = self._io_array(io)
        # the first execution is eager (lazy module loading, attribute setup); graphs from the second on
        g = 2 if recompute else int(use_graph and self._graph_ok)
        L.check(L.lib().v2v_plan_run(self._h, arr, self.n_slots, g, self._stream()))
        L.LAUNCHES[0] += self.num_kernels
        if not recompute:
            self._graph_ok = True
        self.last_io = io
        self.run_id += 1

    def backward(self, io, gio, params, grads):
        """Backward of the last run: io = its forward tensors, gio[slot] = incoming gradient (outputs) / gradient destination
        (inputs), params / grads = parameter tensors and the tensors their gradients are accumulated into."""
        n = len(params)
        pa, ga = (C.c_void_p * max(n, 1))(), (C.c_void_p * max(n, 1))()
        for i, (p_, g_) in enumerate(zip(params, grads)):
            pa[i], ga[i] = p_.data_ptr(), (g_.data_ptr() if g_ is not None else None)
        L.check(L.lib().v2v_plan_backward(self._h, self._io_array(io), self._io_array(gio), self.n_slots, pa, ga, n,
                                          self._stream()))
        L.LAUNCHES[0] += 3 * self.num_kernels

    def profile(self, io=None):
        """Eager run with a CUDA event after every kernel -> list of (kind, ms, conv_macs)."""
        arr = self._io_array(io if io is not None else self.last_io)
        n = self.num_kernels + 4
        kinds, ms, macs, cnt = (C.c_int * n)(), (C.c_float * n)(), (C.c_double * n)(), C.c_int()
        L.check(L.lib().v2v_plan_profile(self._h, arr, self.n_slots, self._stream(), n, kinds, ms, macs,
                                         C.byref(cnt)))
        return [(kinds[i], ms[i], macs[i]) for i in range(cnt.value)]

    # ---- introspection
    @property
    def num_kernels(self):
        return L.lib().v2v_plan_num_kernels(self._h)

    @property
    def conv_macs(self):
        return L.lib().v2v_plan_conv_macs(self._h)

    @property
    def workspace_bytes(self):
        return L.lib().v2v_plan_workspace_bytes(self._h)

    def describe(self):
        n = L.lib().v2v_plan_describe(self._h, None, 0)
        buf = C.create_string_buffer(int(n))
        L.lib().v2v_plan_describe(self._h, buf, n)
        return json.loads(buf.value.decode())
