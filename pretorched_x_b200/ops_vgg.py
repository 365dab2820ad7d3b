"""The two launching entries VGG and AlexNet add: AlexNet's space-to-depth stem input (b2_space_to_depth4_nchw) and the split-K
GEMM of the fully connected classifiers (b2_gemm_splitk_f16, pgemm_kernel<BN, 0, 5> + its reduction pass).

Kept out of ``ops`` because every launching entry of ``ops`` is held by the whole-forward audit's own tables
(tests/model_audit.py); this module's entries are audited by tests/vgg_audit.py, which plugs them into the same auditor, and
tests/test_vgg_cpu.py holds every launching function of this module to that table.  Call sites reach the entries through the
module attribute (``ops_vgg.gemm_splitk(...)``) so that the audit's patch sees every launch.
"""
import ctypes

import torch

from . import _lib, ops
from .ops import Act


def s2d_extent(H, W):
    """(Ho, Wo, Hs, Ws): the output map of nn.Conv2d(3, 64, 11, stride=4, padding=2) on an H x W image and the space-to-depth
    image (Ho + 2) x (Wo + 2) that the equivalent valid 3x3 convolution reads."""
    Ho, Wo = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    return Ho, Wo, Ho + 2, Wo + 2


@ops._on_device
def space_to_depth4(x):
    """fp32 NCHW images [N][3][H][W] -> the Act [N*Hs*Ws][48] (b2_space_to_depth4_nchw): channel (dh * 4 + dw) * 3 + c of pixel
    (hs, ws) is x[c][4 hs + dh - 2][4 ws + dw - 2], zero outside the image.  AlexNet's conv1 (11x11, stride 4, padding 2) is the
    valid 3x3 stride-1 convolution of this image with ``s2d_filter`` of its weight."""
    ops._require_cuda(x, "input")
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError("space_to_depth4 takes [N][3][H][W] images, got %s" % (tuple(x.shape),))
    N, _, H, W = x.shape
    if H < 7 or W < 7:
        raise ValueError("the 11x11 stride-4 filter needs images of at least 7x7, got %dx%d" % (H, W))
    x = x.contiguous().float()
    _, _, Hs, Ws = s2d_extent(H, W)
    y = torch.empty((N * Hs * Ws, 48), dtype=torch.float16, device=x.device)
    with ops._timed("layout", "space_to_depth4 %dx%d M=%d" % (H, W, N * Hs * Ws), 0.0, 4.0 * x.numel() + 2.0 * y.numel()):
        _lib.check(_lib.load().b2_space_to_depth4_nchw(ops._ptr(x), ops._ptr(y), N, H, W, ops._stream()), "b2_space_to_depth4_nchw")
    return Act(y, N, 1, Hs, Ws, 48)


def s2d_filter(weight):
    """nn.Conv2d(3, K, 11) weight [K][3][11][11] -> the [K][48][3][3] filter of the valid 3x3 convolution over ``space_to_depth4``'s
    image: W3[k][(dh * 4 + dw) * 3 + c][a][b] = W[k][c][4 a + dh][4 b + dw], zero where 4 a + dh or 4 b + dw reaches 11."""
    K, C, kh, kw = weight.shape
    if (C, kh, kw) != (3, 11, 11):
        raise ValueError("s2d_filter regroups an 11x11 filter over 3 channels, got %s" % (tuple(weight.shape),))
    w12 = weight.new_zeros((K, 3, 12, 12))
    w12[:, :, :11, :11] = weight
    # [K][c][a][dh][b][dw] -> [K][dh][dw][c][a][b]
    return w12.reshape(K, 3, 3, 4, 3, 4).permute(0, 3, 5, 1, 2, 4).reshape(K, 48, 3, 3).contiguous()


def splitk_plan(M, N, Kd, sm_count=None):
    """The splits b2_gemm_splitk_plan picks for an M x N x Kd product (host arithmetic; ``sm_count`` defaults to the current
    device's)."""
    if sm_count is None:
        sm_count = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    s = _lib.load().b2_gemm_splitk_plan(M, N, Kd, sm_count)
    if s < 1:
        raise ValueError("split-K plan of M=%d N=%d K=%d on %d SMs: %s" % (M, N, Kd, sm_count, _lib.last_error()))
    return s


@ops._on_device
def gemm_splitk(a2d, b2d, scale, shift, M, N, Kd, splits, relu=False, out_f32=False):
    """D[M][N] = act(scale * A[M][Kd] . B[N][Kd]^T + shift) with the K blocks split ``splits`` ways (b2_gemm_splitk_f16): each
    split's fp32 partial product goes to its own workspace slice, a second pass sums them in split order and applies the affine
    and ReLU.  fp16 [M][round_up(N, 8)] out, or fp32 [M][N] with ``out_f32``.  Bitwise repeatable."""
    dev = a2d.device
    ldd = N if out_f32 else ops._round_up(N, 8)
    out = torch.empty((M, ldd), dtype=torch.float32 if out_f32 else torch.float16, device=dev)
    lib = _lib.load()
    n_ws = lib.b2_gemm_splitk_workspace_elems(M, N, splits)
    ws = torch.empty(max(int(n_ws), 1), dtype=torch.float32, device=dev)
    g = ops.GemmArgs()
    g.a, g.b, g.scale, g.shift = ops._ptr(a2d), ops._ptr(b2d), ops._ptr(scale), ops._ptr(shift)
    g.d = ops._ptr(out)
    g.M, g.N, g.Kd = M, N, Kd
    g.lda, g.ldb, g.ldd = a2d.stride(0), b2d.stride(0), ldd
    g.relu, g.out_f32 = int(relu), int(out_f32)
    with ops._timed("gemm_splitk", "gemm splitk M=%d N=%d K=%d S=%d" % (M, N, Kd, splits), 2.0 * M * N * Kd,
                    2.0 * (M * Kd + N * Kd) + out.element_size() * M * N + 8.0 * n_ws):
        _lib.check(lib.b2_gemm_splitk_f16(ctypes.byref(g), splits, ops._ptr(ws), n_ws, ops._stream()), "b2_gemm_splitk_f16")
    return out
