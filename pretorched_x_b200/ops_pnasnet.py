"""The launching entries PNASNet-5-Large's cells need (pretorched/models/pnasnet.py:49-146): the depthwise half of a separable
branch, a K x K depthwise pass (K = 3, 5, 7; stride 1 or 2) that reads ReLU(x), applies no affine and writes a column slice
(b2_dwconv_kxk_relu_in_ndhwc, dwconv_kxk_kernel<K, S, R>), and the strided pixel gather with a grid offset that path_2 of
FactorizedReduction reads (b2_shortcut_a_offset_ndhwc).

Kept out of ``ops`` because every launching entry of ``ops`` is held by the whole-forward audit's own tables (tests/model_audit.py).
Call sites reach the entries through the module attribute (``ops_pnasnet.dwconv_kxk_relu_in(...)``) so that an audit's patch sees
every launch.
"""
import torch

from . import _lib, ops
from .ops import Act


def _rows_view(t, what):
    """(pointer, pitch, columns) of an fp16 2-D matrix or column slice ``m[:, c0:c0 + cols]``: 16-byte aligned, contiguous columns,
    a pitch that is a multiple of 8."""
    p, ld, cols = ops._slice_view(t, what)
    if ld % 8:
        raise ValueError("%s has a row pitch of %d, not a multiple of 8" % (what, ld))
    return p, ld, cols


@ops._on_device
def dwconv_kxk_relu_in(a, wk, k, stride, pad, Ho, Wo, out=None):
    """y = depthwise k x k convolution (stride 1 or 2, top / left padding ``pad``, output extent Ho x Wo, taps outside the map
    zero) of max(x, 0), no affine (b2_dwconv_kxk_relu_in_ndhwc): relu_1 / relu_2 and depthwise_conv2d of PNASNet's
    BranchSeparables (pnasnet.py:67-97).  ``a.data`` may be a column slice of a wider matrix (``m[:, c0:c0 + C]``: its rows of pitch
    ``a.data.stride(0)`` are read); ``wk``: fp32 [k * k][C] taps (kh * k + kw).  ``out``: an fp16 [N * Ho * Wo][C] matrix or column
    slice to write (columns [0, C) of each row, nothing else); a fresh [N * Ho * Wo][C] matrix when None."""
    if a.T != 1 or a.C % 8 or a.data.shape[1] != a.C:
        raise ValueError("the depthwise pass takes images whose data holds exactly C %% 8 == 0 channels, got %r" % (a,))
    if k not in (3, 5, 7) or stride not in (1, 2):
        raise ValueError("the depthwise pass covers k in (3, 5, 7) at stride 1 or 2, got k %r stride %r" % (k, stride))
    if tuple(wk.shape) != (k * k, a.C) or wk.dtype != torch.float32 or not wk.is_contiguous():
        raise ValueError("wk must be a contiguous fp32 [%d][%d] tap matrix, got %s %s" % (k * k, a.C, wk.dtype, tuple(wk.shape)))
    ops._require_cuda(a.data, "input")
    if wk.device != a.data.device:
        raise ValueError("wk lives on %s, the input on %s" % (wk.device, a.data.device))
    xp, ldx, _ = _rows_view(a.data, "depthwise input")
    M = a.N * Ho * Wo
    y = out if out is not None else torch.empty((M, a.C), dtype=torch.float16, device=a.data.device)
    yp, ldy, cols = _rows_view(y, "depthwise output")
    if y.shape[0] != M or cols != a.C:
        raise ValueError("depthwise output %s does not fit %d rows of %d channels" % (tuple(y.shape), M, a.C))
    with ops._timed("dwconv", "dwconv %dx%d s%d p%d C%d M=%d relu_in" % (k, k, stride, pad, a.C, M), 2.0 * k * k * M * a.C,
                    2.0 * a.C * (a.M + M)):
        _lib.check(_lib.load().b2_dwconv_kxk_relu_in_ndhwc(xp, ldx, ops._ptr(wk), yp, ldy, a.N, a.H, a.W, a.C, k, stride, pad, Ho, Wo,
                                                           ops._stream()), "b2_dwconv_kxk_relu_in_ndhwc")
    return Act(y, a.N, 1, Ho, Wo, a.C)


@ops._on_device
def gather_offset(a, stride, offset, relu=False):
    """y[n, i, j] = x[n, stride * i + offset, stride * j + offset] (max(x, 0) with ``relu``), zero past the map's far edge, for i < (H - 1) // stride + 1
    (b2_shortcut_a_offset_ndhwc): path_1 (offset 0) and path_2 (offset 1) of FactorizedReduction (pnasnet.py:117-146), whose 1x1
    convolutions then run as GEMMs.  The output has ``a``'s pitch, channels [C, ld) zero."""
    if a.T != 1:
        raise ValueError("the offset gather takes images, got %r" % (a,))
    ops._require_cuda(a.data, "input")
    if not a.data.is_contiguous():
        raise ValueError("the offset gather reads a dense [rows][ld] matrix")
    Ho, Wo = (a.H - 1) // stride + 1, (a.W - 1) // stride + 1
    y = torch.empty((a.N * Ho * Wo, a.ld), dtype=torch.float16, device=a.data.device)
    with ops._timed("gather", "gather s%d +%d C%d M=%d->%d%s" % (stride, offset, a.ld, a.M, y.shape[0], " relu" if relu else ""), 0.0,
                    4.0 * a.ld * y.shape[0]):
        _lib.check(_lib.load().b2_shortcut_a_offset_ndhwc(ops._ptr(a.data), ops._ptr(y), a.N, a.H, a.W, a.ld, stride, offset, int(relu),
                                                          a.ld, ops._stream()), "b2_shortcut_a_offset_ndhwc")
    return Act(y, a.N, 1, Ho, Wo, a.C)
