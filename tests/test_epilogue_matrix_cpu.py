"""CPU: the generator-epilogue references of tests/kernel_ref.py (per-sample affine, fused upsample, upsampled / pre-affine residual,
second output, input affine) and the elementwise bound tests/test_gpu_epilogue_matrix.py holds the kernels to.  The exact result
rounded once to fp16 passes; each fault a kernel could make in these epilogues fails."""
import torch
import torch.nn.functional as F

from tests.kernel_ref import (conv_acc, epilogue, gemm_acc, in_affine_acc, in_affine_operand, nearest_up2, per_row, second_output,
                              upconv_acc, upconv_fold, worst_ratio)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def affines(g, N, K, pitch=None):
    pitch = pitch or K
    sc = torch.rand(N, pitch, generator=g) + 0.5
    sh = torch.randn(N, pitch, generator=g) * 0.3
    return sc, sh


def gemm_problem(seed, N=3, rows=128, C=64, K=48):
    g = gen(seed)
    x = torch.randn(N * rows, C, generator=g).half()
    w = (torch.randn(K, C, generator=g) / C ** 0.5).half()
    return g, x, w


def exact(v):
    return v.half()


def test_per_sample_affine_exact_passes_and_neighbour_tile_fails():
    g, x, w = gemm_problem(1, N=3, rows=256)
    M, K = x.shape[0], w.shape[0]
    sc, sh = affines(g, 3, K, pitch=K + 4)
    acc, mag = gemm_acc(x, w)
    v, A = epilogue(acc, mag, per_row(sc, 256, M, K), per_row(sh, 256, M, K), relu=True)
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    # the second 128-row tile of sample 0 scaled with sample 1's affine row
    bad_sc, bad_sh = per_row(sc, 256, M, K).clone(), per_row(sh, 256, M, K).clone()
    bad_sc[128:256], bad_sh[128:256] = sc[1, :K].double(), sh[1, :K].double()
    bad, _ = epilogue(acc, mag, bad_sc, bad_sh, relu=True)
    assert worst_ratio(exact(bad), v, A, True) > 1.0


def test_per_sample_affine_indexed_by_plane_fails():
    """3-D per-sample case: 2 samples x 3 output planes of 4 x 4; a kernel that indexes the affine by plane instead of sample."""
    g = gen(2)
    N, T, H, W, C, K = 2, 3, 4, 4, 16, 24
    x = torch.randn(N, T, H, W, C, generator=g).half()
    w = (torch.randn(K, 27, C, generator=g) / (27 * C) ** 0.5).half()
    sc, sh = affines(g, N * T, K)                      # rows beyond N: what a plane index would read
    acc, mag = conv_acc(x, w, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    M, rows = acc.shape[0], T * H * W
    v, A = epilogue(acc, mag, per_row(sc[:N], rows, M, K), per_row(sh[:N], rows, M, K))
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    bad, _ = epilogue(acc, mag, per_row(sc, H * W, M, K), per_row(sh, H * W, M, K))
    assert worst_ratio(exact(bad), v, A, True) > 1.0


def test_upsample_reference_is_the_3x3_conv_of_the_upsampled_image_and_swapped_phases_fail():
    g = gen(3)
    N, H, W, C, K = 2, 5, 7, 16, 24
    x = torch.randn(N, H, W, C, generator=g).half()
    w3 = torch.randn(K, C, 3, 3, generator=g) / (9 * C) ** 0.5
    fold, _ = upconv_fold(w3)
    acc, mag = upconv_acc(x, fold)
    # the phase decomposition is exactly conv3x3(up2(x)) with the unfolded filter
    up = x.double().permute(0, 3, 1, 2).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    direct = F.conv2d(up, w3.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, K)
    assert torch.allclose(acc, direct, rtol=0, atol=1e-12)
    sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    v, A = epilogue(acc, mag, sc, sh, relu=True)
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    # phases (0, 0) and (0, 1) of every output pixel pair swapped
    bad = v.reshape(N, 2 * H, 2 * W, K).clone()
    bad[:, 0::2, 0::2], bad[:, 0::2, 1::2] = bad[:, 0::2, 1::2].clone(), bad[:, 0::2, 0::2].clone()
    assert worst_ratio(exact(bad.reshape(-1, K)), v, A, True) > 1.0


def test_upconv_fold_bound_passes_rounded_fold_and_fails_a_dropped_tap():
    w3 = torch.randn(32, 24, 3, 3, generator=gen(4))
    fold, wsum = upconv_fold(w3)
    bnd = 2.0 ** -11 * fold.abs() + 2.0 ** -22 * wsum
    assert float(((fold.half().double() - fold).abs() / bnd).max()) <= 1.0
    w_drop = w3.clone()
    w_drop[:, :, 1, 2] = 0                                # one 3x3 tap missing from every fold it feeds
    bad, _ = upconv_fold(w_drop)
    assert float(((bad.half().double() - fold).abs() / bnd).max()) > 1.0


def test_residual_up_neighbouring_low_res_column_fails():
    g, x, w = gemm_problem(5, N=2, rows=128)            # 2 images of 8 x 16
    N, H, W, K = 2, 8, 16, 40
    w = w[:K]
    skip = torch.randn(N * (H // 2) * (W // 2), 48, generator=g).half()   # channel drop: 48 -> 40
    acc, mag = gemm_acc(x, w)
    sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    r = nearest_up2(skip, N, H, W, K)
    v, A = epilogue(acc, mag, sc, sh, residual=r)
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    shifted = skip.reshape(N, H // 2, W // 2, 48).roll(-1, dims=2).reshape(-1, 48)   # low-res column w/2 + 1
    bad, _ = epilogue(acc, mag, sc, sh, residual=nearest_up2(shifted, N, H, W, K))
    assert worst_ratio(exact(bad), v, A, True) > 1.0


def test_residual_pre_after_the_affine_fails():
    g, x, w = gemm_problem(6)
    M, K = x.shape[0], w.shape[0]
    r = torch.randn(M, K, generator=g).half().double()
    sc, sh = torch.rand(K, generator=g) + 1.5, torch.randn(K, generator=g)
    acc, mag = gemm_acc(x, w)
    v, A = epilogue(acc, mag, sc, sh, residual=r, pre=True, relu=True)
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    bad, _ = epilogue(acc, mag, sc, sh, residual=r, pre=False, relu=True)
    assert worst_ratio(exact(bad), v, A, True) > 1.0


def test_second_output_from_the_rounded_first_output_fails():
    g, x, w = gemm_problem(7, N=2)
    M, K = x.shape[0], w.shape[0]
    sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    s2, t2 = affines(g, 2, K)
    s2 = s2 * 64                                          # a large second scale magnifies the first rounding
    acc, mag = gemm_acc(x, w)
    v, A = epilogue(acc, mag, sc, sh)
    ref2, A2 = second_output(v, A, per_row(s2, 128, M, K), per_row(t2, 128, M, K))
    assert worst_ratio(exact(ref2), ref2, A2, True) <= 1.0
    bad2, _ = second_output(v.half().double(), A, per_row(s2, 128, M, K), per_row(t2, 128, M, K))
    assert worst_ratio(exact(bad2), ref2, A2, True) > 1.0


def test_input_affine_exact_passes_and_missing_relu_or_wrong_sample_fails():
    g, x, w = gemm_problem(8, N=2, C=64, K=32)
    M, K = x.shape[0], w.shape[0]
    isc, ish = affines(g, 2, 64, pitch=68)
    acc, mag = in_affine_acc(x, w, isc, ish, 128)
    sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    v, A = epilogue(acc, mag, sc, sh)
    assert worst_ratio(exact(v), v, A, True) <= 1.0
    # no ReLU on the operand
    xn = (x.double() * per_row(isc, 128, M, 64) + per_row(ish, 128, M, 64)).half()
    bad, _ = epilogue(*gemm_acc(xn, w), sc, sh)
    assert worst_ratio(exact(bad), v, A, True) > 1.0
    # affine rows of the other sample
    swapped = torch.stack([isc[1], isc[0]]), torch.stack([ish[1], ish[0]])
    bad, _ = epilogue(*in_affine_acc(x, w, *swapped, 128), sc, sh)
    assert worst_ratio(exact(bad), v, A, True) > 1.0


def test_input_affine_midpoint_operands_are_flagged_and_covered():
    """An operand whose fp64 value sits on an fp16 rounding midpoint may round either way in the kernel: both outcomes pass."""
    x = torch.tensor([[1.0, 0.5, 2.0, 1.0]], dtype=torch.float16)
    sc = torch.tensor([[1.0 + 2.0 ** -11, 1.0, 1.0, 1.0]])  # 1 + 2^-11: the midpoint between 1 and 1 + 2^-10
    sh = torch.zeros(1, 4)
    xq, other = in_affine_operand(x, sc, sh, 1)
    assert other[0, 0] > 0 and bool((other[0, 1:] == 0).all())
    w = torch.ones(8, 4, dtype=torch.float16)
    acc, mag = in_affine_acc(x, w, sc, sh, 1)
    v, A = epilogue(acc, mag, torch.ones(8), torch.zeros(8))
    for first in (1.0, 1.0 + 2.0 ** -10):
        got = first + 0.5 + 2.0 + 1.0
        assert worst_ratio(torch.full((1, 8), got).half(), v, A, True) <= 1.0


def test_residual_in_the_padding_columns_fails():
    """y[:, K:ldy] must be exactly zero: a residual copied into the padding is caught by the bound on those columns (ref 0, A 0)."""
    g, x, w = gemm_problem(9, C=64, K=60)
    M, K, ldy = x.shape[0], 60, 64
    r = torch.randn(M, 72, generator=g).half()         # a wider skip tensor: columns [60, 72) hold data
    sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
    acc, mag = gemm_acc(x, w)
    v, A = epilogue(acc, mag, sc, sh, residual=r[:, :K].double())
    full_ref = torch.cat([v, torch.zeros(M, ldy - K, dtype=torch.float64)], dim=1)
    full_A = torch.cat([A, torch.zeros(M, ldy - K, dtype=torch.float64)], dim=1)
    good = torch.cat([v.half(), torch.zeros(M, ldy - K, dtype=torch.float16)], dim=1)
    assert worst_ratio(good, full_ref, full_A, True) <= 1.0
    bad = good.clone()
    bad[:, K:] = r[:, K:ldy]
    assert worst_ratio(bad, full_ref, full_A, True) > 1.0
