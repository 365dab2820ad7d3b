"""GPU (-m gpu): the transposed four-row stem convolution (b2_stemconv.cuh, kT: the filter as the m64 operand, one N = 112 MMA
per output row and slab row), with the instance pinned through the last-kernel record.  Each case is checked bitwise against the
four-row instance with positions along M (forced through the knob; both accumulate every output element in the same order:
temporal tap, slab row, K step), against the CUDA-core cross-check, and against an fp64 conv + BN + ReLU (+ max-pool) on the host
within the stem tolerance."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_stem import POOL_FULL, POOL_TH, TOL_F16, make_stem, rel

pytestmark = pytest.mark.gpu

STEM = 1
FORCE_T = 4 | 16


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_set_stem_rows.argtypes = [ctypes.c_int]
    yield lib
    lib.b2_debug_set_stem_rows(-1)


def run_stem(lib, force, conv, bn, a, pooled):
    """The stem (+ the (T, H) pool pass when pooled) under the force knob; returns the output and (kernel id, G, transposed)."""
    from pretorched_x_b200 import engine, ops
    lib.b2_debug_set_stem_rows(force)
    try:
        y = engine.conv_bn_act(conv, bn, a, relu=True, pool_w=pooled)
        torch.cuda.synchronize()
        info = (ctypes.c_int * 5)()
        kid = lib.b2_debug_last_kernel(info)
    finally:
        lib.b2_debug_set_stem_rows(-1)
    return (ops.maxpool3d(y, *POOL_TH) if pooled else y), (kid, info[0], info[1])


def fp64_ref(x, conv, bn, k, p, pooled):
    """conv + BN (eval) + ReLU (+ MaxPool3d(3, 2, 1)) in fp64 on the host, as [positions][channels]."""
    y = F.conv3d(x.double(), conv.weight.detach().double().cpu(), stride=(1, 2, 2), padding=p)
    y = F.batch_norm(y, bn.running_mean.double().cpu(), bn.running_var.double().cpu(), bn.weight.detach().double().cpu(),
                     bn.bias.detach().double().cpu(), training=False, eps=bn.eps).clamp_min(0.0)
    if pooled:
        y = F.max_pool3d(y, *POOL_FULL)
    return y.permute(0, 2, 3, 4, 1).reshape(-1, y.shape[1])


T_CASES = [
    # name, N, T, H, W, K, kernel, padding, pooled
    ("resnet3d50_stem_b1", 1, 16, 224, 224, 64, (7, 7, 7), (3, 3, 3), True),
    ("resnet3d50_stem_b2_unpooled", 2, 16, 224, 224, 64, (7, 7, 7), (3, 3, 3), False),
    ("ho16_mod4_0_wo32", 1, 4, 32, 64, 64, (7, 7, 7), (3, 3, 3), True),
    ("ho17_mod4_1_wo56", 1, 4, 34, 112, 64, (7, 7, 7), (3, 3, 3), False),
    ("ho18_mod4_2_wo111", 1, 3, 36, 222, 64, (7, 7, 7), (3, 3, 3), True),
    ("ho19_mod4_3_wo109", 2, 2, 38, 218, 64, (7, 7, 7), (3, 3, 3), False),
    ("t_below_kt_both_ends", 2, 3, 22, 40, 64, (7, 7, 7), (3, 3, 3), True),
    ("slowfast_5x7x7_to_8", 2, 8, 32, 64, 8, (5, 7, 7), (2, 3, 3), True),
    ("kt3_kh3_to_40_unpooled", 1, 5, 30, 100, 40, (3, 3, 7), (1, 1, 3), False),
]


@pytest.mark.parametrize("case", T_CASES, ids=[c[0] for c in T_CASES])
def test_transposed_stem(lib, case):
    from pretorched_x_b200 import engine, ops
    name, N, T, H, W, K, k, p, pooled = case
    x, a, conv, bn = make_stem(torch.device("cuda:0"), N, T, H, W, K, k, p, sum(map(ord, name)))
    got, ran = run_stem(lib, -1, conv, bn, a, pooled)
    assert ran == (STEM, 4, 1)                                        # the rule takes the transposed instance
    forced, ran_t = run_stem(lib, FORCE_T, conv, bn, a, pooled)
    assert ran_t == (STEM, 4, 1) and torch.equal(forced.data, got.data)
    m_op, ran4 = run_stem(lib, 4, conv, bn, a, pooled)
    assert ran4 == (STEM, 4, 0)
    assert torch.equal(got.data, m_op.data)                           # same accumulation order: bit-identical
    ref = engine.conv_bn_act(conv, bn, a, relu=True, simt=True)
    if pooled:
        ref = ops.maxpool3d(ref, *POOL_FULL)
    assert (got.N, got.T, got.H, got.W, got.C) == (ref.N, ref.T, ref.H, ref.W, ref.C)
    assert rel(got.data[:, :K].float(), ref.data[:, :K].float()) <= TOL_F16
    if got.ld > K:                                                    # channel padding stays exactly zero
        assert float(got.data[:, K:].abs().max()) == 0.0
    if N * T * H * W <= 2 * 4 * 40 * 224:                             # fp64 on the host for the small shapes
        assert rel(got.data[:, :K].cpu(), fp64_ref(x, conv, bn, k, p, pooled)) <= TOL_F16
