"""The launching entries of the grouped-convolution backward (fine-tuning ResNeXt-101): the input gradient on the group-aware
kernel with the ReLU-derivative mask (b2_conv_grouped_ndhwc_dgrad) and the diagonal-block weight gradient (b2_conv_wgrad_grouped).

Kept out of ``ops`` because every launching entry of ``ops`` is held by the whole-forward audit's own tables (tests/model_audit.py);
these run in the backward only and are held element by element to fp64 by tests/test_gpu_grouped_backward.py.
"""
import ctypes

import torch

from . import _lib, ops
from .ops import Act


@ops._on_device
def conv_grouped_dgrad(z, pc, mask):
    """Input gradient of a grouped convolution (b2_conv_grouped_ndhwc_dgrad): the stride-1 ``PackedGroupedConv`` ``pc`` (filter
    transposed within each group, flipped, BN-scaled) over the (zero-inserted) gradient ``z``, zeroed where the Act ``mask`` <= 0."""
    if z.ld != pc.C or pc.s != (1, 1, 1):
        raise ValueError("the grouped input gradient is a stride-1 convolution over a gradient of pitch %d" % pc.C)
    kt, kh, kw = pc.k
    To, Ho, Wo = (ops._out_dim(z.T, kt, 1, pc.p[0]), ops._out_dim(z.H, kh, 1, pc.p[1]), ops._out_dim(z.W, kw, 1, pc.p[2]))
    M = z.N * To * Ho * Wo
    if mask.M != M or mask.ld < pc.K:
        raise ValueError("mask rows %d / pitch %d do not match the %d x %d output" % (mask.M, mask.ld, M, pc.K))
    y = torch.empty((M, pc.K), dtype=torch.float16, device=z.data.device)
    args = ops.ConvArgs()
    args.x, args.w, args.scale, args.shift = ops._ptr(z.data), ops._ptr(pc.w), ops._ptr(pc.scale), ops._ptr(pc.shift)
    args.y, args.mask, args.ldm = ops._ptr(y), ops._ptr(mask.data), mask.ld
    args.N, args.T, args.H, args.W, args.C = z.N, z.T, z.H, z.W, z.ld
    args.K, args.ldy = pc.K, pc.K
    args.kt, args.kh, args.kw = kt, kh, kw
    args.st, args.sh, args.sw = pc.s
    args.pt, args.ph, args.pw = pc.p
    args.mode = ops.B2_CONV_AUTO
    taps = kt * kh * kw
    with ops._timed("conv", "gconv-dgrad %dx%dx%d C%d g%d M=%d" % (kt, kh, kw, pc.K, pc.groups, M), 2.0 * M * pc.K * pc.Cin * taps,
                2.0 * (z.M * z.C + 2 * M * pc.K + pc.K * pc.Cin * taps)):
        _lib.check(_lib.load().b2_conv_grouped_ndhwc_dgrad(ctypes.byref(args), pc.groups, ops._stream()), "b2_conv_grouped_ndhwc_dgrad")
    return Act(y, z.N, To, Ho, Wo, pc.K)


def wgrad_grouped_plan(N, T, H, W, C, groups, stride):
    """(executed, algorithmic multiply-accumulates, splits) of ``conv_wgrad_grouped``'s plan (host arithmetic)."""
    e, a, sp = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    _lib.check(_lib.load().b2_conv_wgrad_grouped_plan(N, T, H, W, C, groups, stride, ctypes.byref(e), ctypes.byref(a), ctypes.byref(sp)),
               "b2_conv_wgrad_grouped_plan")
    return e.value, a.value, sp.value


@ops._on_device
def conv_wgrad_grouped(g, x, groups, stride, weight=None, scale=None, inv_loss_scale=None):
    """Weight gradient of a grouped 3x3 convolution, C == K, padding 1 (b2_conv_wgrad_grouped): g = Act gradient at its output,
    x = Act input.  Returns (dw fp32 [C][C / groups][1][3][3] scaled by ``scale[k]`` and ``inv_loss_scale``, and, with
    ``weight``, wdot[k] = <weight[k], G[k]> * inv_loss_scale)."""
    C, cg = x.C, x.C // groups
    dev = g.data.device
    lib = _lib.load()
    n = lib.b2_conv_wgrad_grouped_workspace_elems(x.N, x.T, x.H, x.W, C, groups, stride)
    ws = torch.empty(max(int(n), 1), dtype=torch.float32, device=dev)
    dw = torch.empty((C, cg, 1, 3, 3), dtype=torch.float32, device=dev)
    w = weight.detach().float().contiguous() if weight is not None else None
    wdot = torch.empty(C, dtype=torch.float32, device=dev) if weight is not None else None
    with ops._timed("wgrad", "wgrad-grouped 1x3x3 s%d C%d g%d M=%d" % (stride, C, groups, g.M), 2.0 * g.M * C * cg * 9,
                2.0 * (g.M * C + x.M * C) + 4.0 * C * cg * 9):
        _lib.check(lib.b2_conv_wgrad_grouped(ops._ptr(g.data), g.ld, ops._ptr(x.data), x.ld, ops._ptr(w), ops._ptr(scale), ops._ptr(inv_loss_scale), ops._ptr(dw),
                                             ops._ptr(wdot), ops._ptr(ws), ws.numel(), x.N, x.T, x.H, x.W, C, groups, stride, ops._stream()),
                   "b2_conv_wgrad_grouped")
    return dw, wdot
