"""fp64 references of the PNASNet-5 kernels (pretorched_x_b200/ops_pnasnet.py) and the shapes PNASNet-5-Large runs them at.

``dw_kxk_relu_in_ref`` and ``gather_offset_ref`` restate the C entries' contracts (include/b2_pretorched.h) on plain tensors;
tests/test_pnasnet_kernels_cpu.py pins both, in fp64, to the reference model's own formulation (ZeroPad2d -> convolution -> crop,
FactorizedReduction's pad / crop / AvgPool2d(1, 2)), and tests/test_gpu_pnasnet_kernels.py holds the kernels to them within the
per-element bound of tests/kernel_ref.py.
"""
import torch
import torch.nn.functional as F

from tests import kernel_ref as KR


def dw_kxk_relu_in_ref(x, wk, k, stride, pad, Ho, Wo, device="cpu"):
    """fp64 reference of b2_dwconv_kxk_relu_in_ndhwc: x fp16 [B, H, W, C], wk fp32 [k * k][C] (tap kh * k + kw).
    y[n, i, j, c] = sum max(x[n, i*stride + kh - pad, j*stride + kw - pad, c], 0) * wk[kh*k + kw][c], taps outside the map zero.
    Returns (ref, A), fp64 [B * Ho * Wo, C], A = sum |max(x, 0) * w|."""
    x = x.double().to(device).clamp(min=0.0)
    B, H, W, C = x.shape
    xt = x.permute(0, 3, 1, 2)
    bottom = max(0, (Ho - 1) * stride + k - pad - H)
    right = max(0, (Wo - 1) * stride + k - pad - W)
    xt = F.pad(xt, (pad, right, pad, bottom))
    wt = wk.double().to(device).t().reshape(C, 1, k, k)
    acc = F.conv2d(xt, wt, stride=stride, groups=C)[:, :, :Ho, :Wo]
    mag = F.conv2d(xt.abs(), wt.abs(), stride=stride, groups=C)[:, :, :Ho, :Wo]
    return acc.permute(0, 2, 3, 1).reshape(-1, C), mag.permute(0, 2, 3, 1).reshape(-1, C)


def gather_offset_ref(x, stride, offset):
    """Reference of b2_shortcut_a_offset_ndhwc on x [B, H, W, C]: x[:, stride*i + offset, stride*j + offset], zero past the far
    edge, i < (H - 1) // stride + 1.  Returns [B * Ho * Wo, C] in x's dtype."""
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    y = x.new_zeros((B, Ho, Wo, C))
    sub = x[:, offset::stride, offset::stride]
    y[:, :sub.shape[1], :sub.shape[2]] = sub[:, :Ho, :Wo]
    return y.reshape(-1, C)


def check_dw_kxk(y, ref, A):
    """Worst err / bound of the used channels against the fp64 reference (KR.worst_ratio's metric)."""
    return KR.worst_ratio(y, ref, A, True)


# The depthwise passes of PNASNet-5-Large at 331^2 as (K, stride, pad, C, H, Ho), C the channels the kernel sees (54 and 108 at
# their padded pitches 56 and 112).  Stride 1: every separable branch's second pass, and comb_iter_3_left's first.  Stride 2: the
# first pass of a reduction branch -- CellStem0 from conv_0's 165^2 (96 channels from x_left, 56 from x_right), cell_stem_1 from
# 83^2, cell_4's zero-pad form from 42^2 (pad K // 2 - 1, ceil extent), cell_8 from 21^2.
def network_cases():
    cases = []
    for k in (3, 5, 7):
        p = k // 2
        for C, hw in ((56, 83), (112, 42), (216, 42), (432, 21), (864, 11)):
            cases.append((k, 1, p, C, hw, hw))
        cases += [(k, 2, p, 96, 165, 83), (k, 2, p, 56, 165, 83), (k, 2, p, 112, 83, 42), (k, 2, p - 1, 432, 42, 21),
                  (k, 2, p, 864, 21, 11)]
    return cases
