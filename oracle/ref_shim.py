"""TEST INFRASTRUCTURE -- not product code.

Imports the *unmodified* reference (NVIDIA/vid2vid: the tree named by V2V_REFERENCE_ROOT, else the
copy oracle/make_ref.py made in the git-ignored oracle/_ref/) on CPU under the installed PyTorch with the
harness-level shims of SURVEY.md 8(c).  Used by oracle/make_golden.py to produce the committed fixtures in
tests/golden/, by the GPU integration tests that run the reference's own modules, and by bench.py's
reference arm (the reference's own modules on the host cores).

Shims (none changes reference arithmetic):
  1. Tensor.cuda / Module.cuda -> identity  (reference hard-codes .cuda(gpu_id),
     models/networks.py:93,113,219,228; models/vid2vid_model_G.py:90,100,110)
  2. torch.cuda.FloatTensor/ByteTensor -> CPU tensor types (vid2vid_model_G.py:94,
     base_model.py:14,147)
  3. fractions.gcd = math.gcd (models/models.py:7-8)
  4. Tensor.get_device() on CPU returns -1 already; `.cuda(-1)` is swallowed by shim 1.
"""
import os
import sys
import math
import fractions

_VENDORED = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')
REF_ROOT = os.environ.get('V2V_REFERENCE_ROOT') or _VENDORED


def available():
    return os.path.isdir(os.path.join(REF_ROOT, 'models'))


_installed = False


def install():
    """Apply the shims and put the reference on sys.path.  Idempotent."""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError('reference tree not found at %s' % REF_ROOT)
    import torch
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.cuda.FloatTensor = torch.FloatTensor
    torch.cuda.ByteTensor = torch.ByteTensor
    if not hasattr(fractions, 'gcd'):
        fractions.gcd = math.gcd
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    _installed = True


def networks():
    install()
    import models.networks as ref_networks   # noqa  (reference module)
    return ref_networks


def model_G_class():
    install()
    from models.vid2vid_model_G import Vid2VidModelG
    return Vid2VidModelG


def make_model_G(opt, single_G=None):
    """Build the reference Vid2VidModelG without touching disk: load_network and
    load_single_G are stubbed (SURVEY 8c shim 4).  `single_G` is the module returned by
    the stubbed load_single_G (the caller builds it with networks().define_G)."""
    cls = model_G_class()
    import contextlib
    import io

    class _M(cls):
        def load_network(self, *a, **k):
            return None

        def load_single_G(self):
            return single_G

    m = _M()
    with contextlib.redirect_stdout(io.StringIO()):
        m.initialize(opt)
    return m


def install_flownet2_ops():
    """Harness-level stand-ins for the three pybind11 extensions the reference's FlowNet2 imports (`correlation_cuda`,
    `resample2d_cuda`, `channelnorm_cuda`: CUDA only, they do not build against the installed torch): the same
    `forward(...)` entry points, computed by oracle/flowops_oracle.c on CPU tensors.  Also replaces
    `Correlation.forward`, which instantiates a legacy (non-static) autograd Function that current PyTorch refuses to
    run (networks/correlation_package/correlation.py:6-30,56-60); the replacement performs the identical single call.
    No reference arithmetic outside those extensions is touched."""
    install()
    import types
    import numpy as np
    import torch
    from oracle import flowops

    def _np(t):
        return np.ascontiguousarray(t.detach().cpu().numpy(), dtype=np.float32)

    corr = types.ModuleType('correlation_cuda')

    def corr_forward(in1, in2, rbot1, rbot2, out, pad, k, max_disp, s1, s2, corr_type):
        r = torch.from_numpy(flowops.correlation(_np(in1), _np(in2), pad, k, max_disp, s1, s2))
        out.resize_(r.shape).copy_(r)
        return 1
    corr.forward = corr_forward
    res = types.ModuleType('resample2d_cuda')

    def res_forward(in1, in2, out, kernel_size):
        out.copy_(torch.from_numpy(flowops.resample2d(_np(in1), _np(in2), kernel_size)))
        return 1
    res.forward = res_forward
    cn = types.ModuleType('channelnorm_cuda')

    def cn_forward(in1, out, norm_deg):
        out.copy_(torch.from_numpy(flowops.channelnorm(_np(in1), norm_deg)))
        return 1
    cn.forward = cn_forward
    sys.modules.setdefault('correlation_cuda', corr)
    sys.modules.setdefault('resample2d_cuda', res)
    sys.modules.setdefault('channelnorm_cuda', cn)

    from models.flownet2_pytorch.networks.correlation_package import correlation as ref_corr   # noqa (reference module)

    def forward(self, input1, input2):
        out = input1.new()
        sys.modules['correlation_cuda'].forward(input1, input2, input1.new(), input2.new(), out, self.pad_size, self.kernel_size,
                                                self.max_displacement, self.stride1, self.stride2, self.corr_multiply)
        return out
    ref_corr.Correlation.forward = forward


def flownet2_class():
    install_flownet2_ops()
    from models.flownet2_pytorch import models as ref_models   # noqa (reference module)
    return ref_models.FlowNet2
