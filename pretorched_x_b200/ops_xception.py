"""The launching entry Xception adds: the depthwise half of its separable convolutions, which reads ReLU(x) and applies no affine
(b2_dwconv3x3_relu_in_ndhwc, dwconv3x3_kernel<1, 4, true>).

Kept out of ``ops`` because every launching entry of ``ops`` is held by the whole-forward audit's own tables
(tests/model_audit.py); this module's entry is audited by tests/xception_audit.py, which plugs it into the same auditor, and
tests/test_xception_cpu.py holds every launching function of this module to that table.  Call sites reach the entry through the
module attribute (``ops_xception.dwconv3x3_relu_in(...)``) so that the audit's patch sees every launch.
"""
import torch

from . import _lib, ops
from .ops import Act


@ops._on_device
def dwconv3x3_relu_in(a, w9, out=None):
    """y = depthwise 3x3 convolution (stride 1, padding 1) of max(x, 0), no affine (b2_dwconv3x3_relu_in_ndhwc): the ReLU that
    opens each separable convolution of an Xception block (xception.py:74-101) and its SeparableConv2d.conv1.  ``w9``: fp32 [9][C]
    taps (kh * 3 + kw).  The output has ``a``'s shape and pitch, channels [C, ld) zero.  ``out``: see ``ops.conv``."""
    if a.C % 8 or a.T != 1:
        raise ValueError("the depthwise pass takes images with C %% 8 == 0, got %r" % (a,))
    if tuple(w9.shape) != (9, a.C) or w9.dtype != torch.float32 or not w9.is_contiguous():
        raise ValueError("w9 must be a contiguous fp32 [9][%d] tap matrix, got %s %s" % (a.C, w9.dtype, tuple(w9.shape)))
    ops._require_cuda(a.data, "input")
    if w9.device != a.data.device:
        raise ValueError("w9 lives on %s, the input on %s" % (w9.device, a.data.device))
    y = ops._out_rows(out, a.M, a.ld) if out is not None else torch.empty((a.M, a.ld), dtype=torch.float16, device=a.data.device)
    with ops._timed("dwconv", "dwconv 3x3 s1 C%d M=%d relu_in" % (a.C, a.M), 18.0 * a.M * a.C, 2.0 * a.C * 2 * a.M):
        _lib.check(_lib.load().b2_dwconv3x3_relu_in_ndhwc(ops._ptr(a.data), ops._ptr(w9), ops._ptr(y), a.N, a.H, a.W, a.C, a.ld,
                                                          ops._stream()), "b2_dwconv3x3_relu_in_ndhwc")
    return Act(y, a.N, 1, a.H, a.W, a.C)
