"""GPU (-m gpu): the PNASNet-5 kernels against fp64.

1. The k x k ReLU-on-input depthwise pass (b2_dwconv_kxk_relu_in_ndhwc) within the per-element bound of tests/kernel_ref.py for
   every (K, stride, pad, C, map) PNASNet-5-Large runs at 331^2 (tests/pnasnet_kernel_ref.network_cases), with the kernel that ran
   pinned (KID 20, info {K, stride, pad, columns per thread}); the input read as a column slice of a wider matrix and the output
   written into a column slice whose neighbouring columns and rows stay untouched; 54 / 108 channels at pitches 56 / 112 with zero
   taps in the pad channels (which come out exactly zero); ragged, non-square maps at both strides.
2. The K = 3, stride 1, padding 1 instance equal bit for bit to b2_dwconv3x3_relu_in_ndhwc: the same taps in the same order.
3. The offset gather (b2_shortcut_a_offset_ndhwc) equal to its reference on odd and even maps, and at offset 0 to
   b2_shortcut_a_ndhwc bit for bit.
"""
import ctypes

import pytest
import torch

from pretorched_x_b200 import _lib, ops, ops_pnasnet, ops_xception
from tests.conftest import has_h100
from tests.kernel_ref import where_worst, worst_ratio
from tests import pnasnet_kernel_ref as PR

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
KID_DWCONV_KXK = 20                # csrc/b2_host.h


def _last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _run(x, wk, k, stride, pad, Ho, Wo, zero_channels=0):
    """x fp16 [B, H, W, C] on the CPU.  The input is a column slice (8 columns in) of a wider matrix, the output a column slice of a
    NaN-filled one; checks the bound, KID 20, the untouched columns and rows, and returns the output."""
    B, H, W, C = x.shape
    M = B * Ho * Wo
    wide = torch.full((B * H * W, C + 24), float("nan"), dtype=torch.float16)
    wide[:, 8:8 + C] = x.reshape(-1, C)
    a = ops.Act(wide.to(dev)[:, 8:8 + C], B, 1, H, W, C)
    rows = 3
    buf = torch.full((M + 2 * rows, C + 32), float("nan"), dtype=torch.float16, device=dev)
    out = buf[rows:rows + M, 16:16 + C]
    y = ops_pnasnet.dwconv_kxk_relu_in(a, wk.to(dev), k, stride, pad, Ho, Wo, out=out)
    torch.cuda.synchronize()
    R = 2 if stride == 2 else (6 if k == 3 else 4)
    assert _last_kernel() == (KID_DWCONV_KXK, [k, stride, pad, R, 0])
    assert (y.N, y.T, y.H, y.W, y.C) == (B, 1, Ho, Wo, C)
    assert torch.isnan(buf[:rows].float()).all() and torch.isnan(buf[rows + M:].float()).all(), "rows outside the slice written"
    assert torch.isnan(buf[:, :16].float()).all() and torch.isnan(buf[:, 16 + C:].float()).all(), "columns outside the slice written"
    got = out.cpu()
    ref, A = PR.dw_kxk_relu_in_ref(x, wk, k, stride, pad, Ho, Wo, device=dev)
    r = worst_ratio(got, ref.cpu(), A.cpu(), True)
    tag = "K%d s%d p%d C%-4d %3dx%-3d -> %3dx%-3d" % (k, stride, pad, C, H, W, Ho, Wo)
    print("[pnasnet-dw] %s worst err/bound %.4f" % (tag, r))
    assert r <= 1.0, "%s: err/bound %.3f at %s" % (tag, r, where_worst(got, ref.cpu(), A.cpu(), True))
    if zero_channels:
        assert torch.all(got[:, C - zero_channels:] == 0), "pad channels with zero taps are not zero"
    again = ops_pnasnet.dwconv_kxk_relu_in(a, wk.to(dev), k, stride, pad, Ho, Wo)
    torch.cuda.synchronize()
    assert torch.equal(again.data.cpu().view(torch.int16), got.view(torch.int16)), "two identical calls differ"
    return got


def _operands(B, H, W, C, k, seed, zero_channels=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, W, C, generator=g) * 3).half()          # signed: the ReLU on load matters
    wk = torch.randn(k * k, C, generator=g) * 0.3
    if zero_channels:
        x[..., C - zero_channels:] = 0
        wk[:, C - zero_channels:] = 0
    return x, wk


@pytest.mark.parametrize("case", PR.network_cases(), ids=lambda c: "K%d-s%d-p%d-C%d-%d" % c[:5])
def test_depthwise_kxk_network_shapes_against_fp64(case):
    k, stride, pad, C, hw, Ho = case
    zero = {56: 2, 112: 4}.get(C, 0)            # 54 / 108 channels at pitch 56 / 112, zero taps in the pad channels
    x, wk = _operands(2, hw, hw, C, k, seed=hash(case) % 100000, zero_channels=zero)
    _run(x, wk, k, stride, pad, Ho, Ho, zero_channels=zero)


@pytest.mark.parametrize("k", (3, 5, 7))
@pytest.mark.parametrize("stride", (1, 2))
def test_depthwise_kxk_ragged_maps_against_fp64(k, stride):
    for H, W in ((13, 17), (7, 5), (1, 9), (k, k + 1)):
        for pad in range(k // 2 + 1):
            Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
            # also the extent whose last window runs past the bottom / right edge (the ceil rule of the zero-pad form)
            for ho, wo in {(Ho, Wo), (Ho + 1, Wo + 1)}:
                if ho <= 0 or wo <= 0 or (ho - 1) * stride - pad >= H or (wo - 1) * stride - pad >= W:
                    continue
                x, wk = _operands(3, H, W, 24, k, seed=H * 100 + W * 10 + pad)
                _run(x, wk, k, stride, pad, ho, wo)


def test_k3_stride1_equals_the_xception_pass_bitwise():
    for hw, C in ((42, 216), (11, 864), (19, 728)):
        x, wk = _operands(2, hw, hw, C, 3, seed=hw)
        a = ops.Act(x.reshape(-1, C).to(dev), 2, 1, hw, hw, C)
        y = ops_pnasnet.dwconv_kxk_relu_in(a, wk.to(dev), 3, 1, 1, hw, hw)
        z = ops_xception.dwconv3x3_relu_in(a, wk.to(dev))
        torch.cuda.synchronize()
        assert torch.equal(y.data.view(torch.int16), z.data.view(torch.int16))


@pytest.mark.parametrize("hw", (165, 83, 42, 21, 11))
@pytest.mark.parametrize("C", (96, 272, 1080))
def test_offset_gather_against_reference(hw, C):
    g = torch.Generator().manual_seed(hw * C)
    x = torch.randn(2, hw, hw, C, generator=g).half()
    a = ops.Act(x.reshape(-1, C).to(dev), 2, 1, hw, hw, C)
    for off in (0, 1):
        y = ops_pnasnet.gather_offset(a, 2, off)
        torch.cuda.synchronize()
        Ho = (hw - 1) // 2 + 1
        assert (y.H, y.W, y.C, y.ld) == (Ho, Ho, C, C)
        assert torch.equal(y.data.cpu(), PR.gather_offset_ref(x, 2, off))
        if off == 0:
            assert torch.equal(y.data, ops.shortcut_a(a, 2, C).data)
