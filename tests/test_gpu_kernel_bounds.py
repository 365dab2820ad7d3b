"""GPU (-m gpu): the stem convolution (every instance, with and without its fused W max-pool), the max-pool kernels, the temporal
stack kernel with the full-layer convolution shapes, the depthwise 3x3 kernel and the weight-gradient kernels, element by element
against fp64 references built from exactly the operands each kernel reads (tests/kernel_ref.py).  Every element is held to
2^-11 |ref| + b A + 2^-24 (b = 2^-14, or the accumulation-chain coefficient of the weight gradient); every case asserts which
kernel, instance or plan produced it.  Worst err / bound ratios are printed per case (pytest -s).

The per-tensor metrics of the older tests (rel <= 2e-3, cosine) cannot see errors confined to small elements: a slab row dropped
at a border, a pool window shifted at the right edge in a channel with a small BN scale, split partials kept in fp16;
tests/test_kernel_bounds_cpu.py shows each of those passing the old metric and failing these bounds."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import functional as OF
from tests.conftest import has_h100
from tests.kernel_ref import (conv_ref, dw_ref, pool_w, stem_operands, wdot_ref, wgrad_bound, wgrad_ref, where_worst, where_worst_of,
                              worst_ratio, worst_ratio_of)
from tests.test_gpu_kernel_matrix import (DENSEM, IGEMM, KIND, KNOB_ENV, PGEMM, SLAB, STEM, TSTACK, Problem, last_kernel,
                                          plan_info, rup, run_f16, seed_of, slab_plan)
from tests.test_gpu_kernels import CONV_CASES, TSTACK_CASES

STEM_ENV = ("B2_STEM_ROWS", "B2_STEM_PAIR")

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV + STEM_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV + STEM_ENV)),
]

FORCE_T = 4 | 16                 # b2_debug_set_stem_rows: the transposed four-row instance
STEM_FORCES = (-1, 2, 4, FORCE_T)
POOL_TH = ((3, 3, 1), (2, 2, 1), (1, 1, 0))     # what remains of MaxPool3d(3, 2, 1) once the stem pooled along W


def _lib():
    from pretorched_x_b200 import _lib as L
    return L


def reset_knobs(lib):
    lib.b2_debug_set_stem_rows(-1)
    lib.b2_debug_set_tstack(-1)
    lib.b2_debug_set_densem(-1, 0)
    lib.b2_debug_set_conv_algo(0)
    lib.b2_debug_set_gemm_algo(0)
    lib.b2_debug_set_slab_mt(0)
    lib.b2_debug_set_slab_wide(-1)
    lib.b2_debug_set_slabts(-1)
    lib.b2_debug_set_attention_algo(0)


@pytest.fixture(autouse=True)
def lib():
    """The knobs are process-global and the other GPU files run in the same process: put every one back to its rule."""
    lib = _lib().load()
    lib.b2_debug_set_stem_rows.argtypes = [ctypes.c_int]
    try:
        yield lib
    finally:
        reset_knobs(lib)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def report(name, ratio):
    print("[kernel-bounds] %-66s worst err/bound %.4f" % (name, ratio))


def check_bound(name, got, ref, bnd):
    r = worst_ratio_of(got, ref, bnd)
    report(name, r)
    assert r <= 1.0, "%s: err/bound %.3f at %s" % (name, r, where_worst_of(got, ref, bnd))


# ---------------------------------------------------------------------------------------------
# 1. stem convolution
# ---------------------------------------------------------------------------------------------
# name, N, T, H, W, K, kernel, padding, pooled, (kernel id, G, transposed) the rule picks.  Ho = ceil(H / 2) for kh = 7, Wo = W / 2.
STEM_CASES = [
    ("ho16_mod4_0_wo56_pooled", 1, 4, 32, 112, 64, (7, 7, 7), (3, 3, 3), True, (STEM, 4, 1)),
    ("ho17_mod4_1_wo109_t2_below_kt_pooled", 2, 2, 34, 218, 64, (7, 7, 7), (3, 3, 3), True, (STEM, 4, 1)),
    ("ho18_mod4_2_wo111", 1, 3, 36, 222, 64, (7, 7, 7), (3, 3, 3), False, (STEM, 4, 1)),
    ("ho19_mod4_3_wo112_pooled", 1, 2, 38, 224, 64, (7, 7, 7), (3, 3, 3), True, (STEM, 4, 1)),
    ("ho13_wo113_k40_pooled", 1, 2, 26, 226, 40, (7, 7, 7), (3, 3, 3), True, (STEM, 4, 0)),
    ("slowfast_5x7x7_k8_ho15_wo120_pooled", 2, 4, 30, 240, 8, (5, 7, 7), (2, 3, 3), True, (STEM, 4, 0)),
    ("kt3_kh3_k40_wo50", 1, 5, 30, 100, 40, (3, 3, 7), (1, 1, 3), False, (STEM, 4, 1)),
    ("bn128_k110_wo56_pooled", 1, 3, 20, 112, 110, (3, 7, 7), (1, 3, 3), True, (STEM, 1, 0)),
    ("bn128_k128_wo113_t2_below_kt", 2, 2, 14, 226, 128, (7, 7, 7), (3, 3, 3), False, (STEM, 1, 0)),
    ("pair_odd_planes_112_k110", 1, 3, 20, 112, 110, (1, 7, 7), (0, 3, 3), False, (STEM, 1, 0)),
    ("pair_2d_7x7_k64_three_planes", 3, 1, 48, 96, 64, (1, 7, 7), (0, 3, 3), False, (STEM, 2, 0)),
    ("stem2d_7x7_k64_wo112_pooled", 2, 1, 64, 224, 64, (1, 7, 7), (0, 3, 3), True, (STEM, 2, 0)),
    # tall filters: a single operand ring stage
    ("one_stage_kh13_k64_pooled", 2, 4, 40, 64, 64, (3, 13, 7), (1, 6, 3), True, (STEM, 2, 0)),
    ("one_stage_kh9_bn128", 1, 4, 40, 64, 128, (3, 9, 7), (1, 4, 3), False, (STEM, 1, 0)),
    # resnet3d50's stem on two clips: more items than SMs under every instance, the operand ring and staging tiles wrap
    ("resnet3d50_stem_224_two_clips_pooled", 2, 4, 224, 224, 64, (7, 7, 7), (3, 3, 3), True, (STEM, 4, 1)),
]


def stem_geometry(case):
    _, N, T, H, W, K, k, p, pooled, _ = case
    To = T + 2 * p[0] - k[0] + 1
    Ho = (H + 2 * p[1] - k[1]) // 2 + 1
    Wo = (W - 1) // 2 + 1
    pair = int(k[0] == 1 and p[0] == 0 and Wo <= 60 and not pooled and W <= 120)
    return To, Ho, Wo, pair


def stem_expect(lib, case):
    """{force: (kernel id, G, transposed)} of a STEM_CASES case from the host-only b2_debug_stem_plan (K > 64: the BN = 128
    instance, G = 1, whatever is forced)."""
    K, k = case[5], case[6]
    _, _, Wo, pair = stem_geometry(case)
    out = (ctypes.c_int * 2)()
    exp = {}
    try:
        for f in STEM_FORCES:
            lib.b2_debug_set_stem_rows(f)
            assert lib.b2_debug_stem_plan(K, k[0], k[1], Wo, pair, out) == 0
            exp[f] = (STEM, 1, 0) if K > 64 else (STEM, out[0], out[1])
    finally:
        lib.b2_debug_set_stem_rows(-1)
    return exp


def stem_problem(dev, case):
    from pretorched_x_b200 import ops
    name, N, T, H, W, K, k, p, pooled, _ = case
    g = torch.Generator().manual_seed(seed_of(name))
    x = torch.randn(N, 3, T, H, W, generator=g)
    conv = nn.Conv3d(3, K, k, stride=(1, 2, 2), padding=p, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / (3 * k[0] * k[1] * k[2]) ** 0.5)
    bn = OF.randomize_bn_(nn.BatchNorm3d(K), seed_of(name) + 1).eval()
    with torch.no_grad():                    # one channel with a small BN scale: its errors are invisible to a per-tensor metric
        bn.weight[K // 3] = bn.weight[K // 3] * 2.0 ** -8
    pc = ops.PackedConv(conv.weight.to(dev), None, bn.to(dev), stride=(1, 2, 2), padding=p, stem=True)
    a = ops.from_ncdhw(x.to(dev))
    x4, w4 = stem_operands(x, conv.weight)
    assert torch.equal(a.data.cpu().view(-1, 4), x4.view(-1, 4))
    return pc, a, x4, w4


def run_stem(lib, pc, a, M, ldy, pooled, force):
    """The stem under ``force`` into a row range of a NaN-filled buffer; checks the sentinel rows, the zero padding channels and
    a bitwise-identical second call.  Returns (out rows, (kernel id, G, transposed))."""
    from pretorched_x_b200 import ops
    lib.b2_debug_set_stem_rows(force)
    pad = 3
    buf = torch.full((M + 2 * pad, ldy), float("nan"), dtype=torch.float16, device=a.data.device)
    out = buf[pad:pad + M]
    ops.conv(a, pc, relu=True, pool_w=pooled, out=out)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    again = torch.empty_like(out)
    ops.conv(a, pc, relu=True, pool_w=pooled, out=again)
    torch.cuda.synchronize()
    lib.b2_debug_set_stem_rows(-1)
    assert torch.isnan(buf[:pad].float()).all() and torch.isnan(buf[pad + M:].float()).all(), "rows outside out= were written"
    if ldy > pc.K:
        assert torch.all(out[:, pc.K:].cpu() == 0), "padding channels [K, ldy) not zero"
    assert torch.equal(again.view(torch.int16), out.view(torch.int16)), "two identical calls differ"
    return out, (kid, info[0], info[1])


@pytest.mark.parametrize("case", STEM_CASES, ids=[c[0] for c in STEM_CASES])
def test_stem_every_instance_against_fp64(dev, lib, case):
    from pretorched_x_b200 import ops
    name, N, T, H, W, K, k, p, pooled, want_rule = case
    To, Ho, Wo, _ = stem_geometry(case)
    exp = stem_expect(lib, case)
    assert exp[-1] == want_rule, exp
    pc, a, x4, w4 = stem_problem(dev, case)
    ref, A = conv_ref(x4, w4, pc.scale, pc.shift, k, (1, 2, 2), p, relu=True)
    if pooled:
        ref, bnd = pool_w(ref, A, Wo)
        Wout = (Wo - 1) // 2 + 1
    else:
        bnd, Wout = None, Wo
    M, ldy = N * To * Ho * Wout, rup(K, 8)
    seen = {}
    for f in STEM_FORCES:
        want = exp[f]
        if want in seen:                     # the same instance computes the same bits: no need to hold it to the bound twice
            continue
        out, ran = run_stem(lib, pc, a, M, ldy, pooled, f)
        assert ran == want, (f, ran, want)
        seen[want] = out
        label = "stem G%d%s %s%s" % (ran[1], "t" if ran[2] else "", name, " (rule)" if f == -1 else "")
        if pooled:
            check_bound(label, out[:, :K], ref, bnd)
            th = ops.maxpool3d(ops.Act(out, N, To, Ho, Wout, K), *POOL_TH)
            torch.cuda.synchronize()
            want_th = F.max_pool3d(out.double().cpu().view(N, To, Ho, Wout, ldy).permute(0, 4, 1, 2, 3), *POOL_TH)
            assert torch.equal(th.data.double().cpu(), want_th.permute(0, 2, 3, 4, 1).reshape(-1, ldy)), "(T, H) pool pass differs"
        else:
            r = worst_ratio(out[:, :K], ref, A, True)
            report(label, r)
            assert r <= 1.0, "%s: err/bound %.3f at %s" % (label, r, where_worst(out[:, :K], ref, A, True))


# general max-pool kernel and the two fixed-window ones: bit-exact against F.max_pool3d of the same fp16 tensor in fp64
# N, C, ld, T, H, W, kernel, stride, padding
POOL_CASES = [
    (2, 24, 32, 5, 13, 11, (3, 3, 3), (2, 2, 2), (1, 1, 1)),          # the stem pool's fixed-window kernel, odd sizes
    (3, 40, 48, 4, 9, 7, (3, 3, 1), (2, 2, 1), (1, 1, 0)),            # the (T, H) pass, ragged
    (1, 8, 8, 1, 1, 1, (3, 3, 1), (2, 2, 1), (1, 1, 0)),
    (2, 16, 24, 3, 10, 9, (1, 3, 3), (1, 2, 2), (0, 1, 1)),           # the general kernel from here on
    (2, 64, 64, 7, 5, 6, (3, 1, 1), (2, 1, 1), (1, 0, 0)),
    (1, 200, 208, 4, 6, 5, (2, 2, 2), (2, 2, 2), (0, 0, 0)),
    (3, 8, 16, 2, 7, 7, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
]


@pytest.mark.parametrize("case", POOL_CASES, ids=["N%dC%dld%d_T%dH%dW%d_k%s_s%s" % (c[:6] + ("".join(map(str, c[6])), "".join(map(str, c[7]))))
                                                  for c in POOL_CASES])
def test_maxpool_kernels_bit_exact(dev, case):
    from pretorched_x_b200 import ops
    N, C, ld, T, H, W, k, s, p = case
    g = torch.Generator().manual_seed(N * 1000 + C + T)
    data = torch.zeros(N * T * H * W, ld, dtype=torch.float16)
    data[:, :C] = torch.randn(N * T * H * W, C, generator=g).half()      # signed: the -65504 start of the max is never the answer
    y = ops.maxpool3d(ops.Act(data.to(dev), N, T, H, W, C), k, s, p)
    torch.cuda.synchronize()
    want = F.max_pool3d(data.double().view(N, T, H, W, ld).permute(0, 4, 1, 2, 3), k, s, p)
    assert (y.T, y.H, y.W) == tuple(want.shape[2:])
    assert torch.equal(y.data.double().cpu(), want.permute(0, 2, 3, 4, 1).reshape(-1, ld))


# ---------------------------------------------------------------------------------------------
# 2. temporal stack kernel and the full-layer convolution shapes of tests/test_gpu_kernels.py
# ---------------------------------------------------------------------------------------------
TSTACK_RULE_CASE = ("tstack_rule_c144_to_64_t16_28x28_res", 6, 144, 16, 28, 28, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), True, True,
                    False, True)


def layer_problem(dev, case):
    name, N, Cin, T, H, W, K, k, s, p, res, relu, bias, bn = case
    return Problem(dev, name, N, Cin, T, H, W, K, k, s, p, bias_only=bias and not bn)


@pytest.mark.parametrize("case", TSTACK_CASES + [TSTACK_RULE_CASE], ids=[c[0] for c in TSTACK_CASES] + [TSTACK_RULE_CASE[0]])
def test_tstack_against_fp64(dev, lib, case):
    if case is not TSTACK_RULE_CASE:
        lib.b2_debug_set_tstack(1)           # below the kernel's one-item-per-SM rule: forced
    pb = layer_problem(dev, case)
    kid, _ = run_f16(dev, lib, pb, residual=case[10], relu=case[11])
    assert kid == TSTACK and lib.b2_debug_last_conv_path() == 1


# The kernel the rule picks today for every non-stem CONV_CASES shape through ops.conv (the strided 1x1x1 projections run as
# gathers here: engine.conv_bn_act subsamples them first).  The slabts_* shapes resolve to the slab kernel (see
# tests/test_gpu_kernel_matrix.py::test_slabts_and_slab_against_fp64).
RULE_KID = {
    "1x1x1_tma": PGEMM, "1x1x1_reduce": PGEMM, "3x3x3_s1": DENSEM, "3x3x3_s1_ragged_rows": DENSEM, "3x3x3_s2": DENSEM,
    "3x3x3_T1_all_temporal_padding": DENSEM, "shortcutB_1x1x1_s2": IGEMM, "r2p1d_spatial_144": DENSEM,
    "r2p1d_temporal_from_144": DENSEM, "r2p1d_temporal7_from_110": DENSEM, "r2p1d_spatial_s2_odd_230": DENSEM,
    "r2p1d_temporal_s2_from_230": DENSEM, "nonlocal_theta_bias_no_bn": PGEMM, "single_output_pixel": DENSEM,
    "slab_layer1_56x56": SLAB, "slab_layer2_28x28_res": SLAB, "slab_layer3_14x14": SLAB, "slab_odd_sizes_200ch": DENSEM,
    "slab_s2_56_to_28": DENSEM, "slab_s2_odd_input_7x7": DENSEM, "slab_2d_3x3_s2_resnet18": DENSEM, "slab_temporal7_wide": SLAB,
    "flexn_144_56x56": IGEMM, "flexn_288_28x28_res": SLAB, "flexn_576_14x14_3tiles": DENSEM, "flexn_460_s2": DENSEM,
    "wide_row_chunks_3x3": SLAB, "wide_row_chunks_3x3_s2": DENSEM, "temporal3_chunked_28x28_res": SLAB,
    "temporal3_14x14_from_576": SLAB, "temporal5_ragged_positions": DENSEM,
    "projection_1x1x1_s2_subsample": IGEMM, "densem_4x4_1152_split": DENSEM, "densem_temporal_1152_512_res": DENSEM,
    "densem_3x3x3_s2_odd_200ch": DENSEM, "densem_tiny_m_3": DENSEM, "slabts_c64_t5_res": SLAB, "slabts_c32_to_48_t7_odd": SLAB,
    "slabts_c128_to_64_t3": SLAB, "slabts_temporal_3x1x1_to_64": SLAB, "slabts_wide_rows_chunked": SLAB,
    "slab_multiplane_7x7_192": SLAB, "slab_multiplane_7x7_T1_3x3x3": SLAB, "slab_multiplane_5x6_c512_256wide": SLAB,
}
LAYER_CASES = [c + (RULE_KID.get(c[0]),) for c in CONV_CASES if not c[0].startswith("stem")]


def layer_slab_case(case):
    """The (name, N, Cin, pitch, T, H, W, K, kernel, stride, padding) form slab_plan reads."""
    name, N, Cin, T, H, W, K, k, s, p = case[:10]
    return (name, N, Cin, rup(Cin, 8), T, H, W, K, k, s, p)


@pytest.mark.parametrize("case", LAYER_CASES, ids=[c[0] for c in LAYER_CASES])
def test_full_layer_shapes_against_fp64(dev, lib, case):
    pb = layer_problem(dev, case[:14])
    kid, info = run_f16(dev, lib, pb, residual=case[10], relu=case[11])
    assert kid == case[14], (KIND[kid], info)
    if kid == SLAB:
        assert info == plan_info(slab_plan(lib, layer_slab_case(case)))


# ---------------------------------------------------------------------------------------------
# 3. depthwise 3x3 (dwconv3x3_kernel<1, 4> at stride 1, <2, 2> at stride 2: the instance is fixed by the stride)
# ---------------------------------------------------------------------------------------------
def _dw_cases():
    from tests.test_gpu_mobilenet import DW_CASES
    extra = [
        # B, C, H, W, stride, ld, clamp_in, relu6
        (3, 8, 7, 9, 1, 16, True, True),          # Wo % 4 == 1, C = 8, ld > C
        (3, 1000, 5, 10, 1, 1008, True, True),    # Wo % 4 == 2, C not a multiple of 64
        (2, 960, 6, 11, 1, 960, False, True),     # Wo % 4 == 3, signed input
        (3, 40, 9, 13, 2, 48, True, True),        # stride 2, Wo = 7
        (2, 1000, 7, 9, 2, 1000, False, False),   # stride 2, Wo = 5, signed, no activation
        (4, 24, 5, 3, 1, 24, True, True),         # Wo = 3 < R
        (3, 64, 4, 1, 2, 72, True, True),         # W = 1 at stride 2: Wo = 1 < R
        (3, 16, 1, 6, 1, 16, False, False),       # H = 1
        (2, 32, 1, 1, 1, 40, True, True),         # H = W = 1
    ]
    return DW_CASES + extra


DWB_CASES = _dw_cases()


@pytest.mark.parametrize("case", DWB_CASES, ids=["B%dC%dH%dW%ds%dld%d%s%s" % (c[:6] + ("_clamp" if c[6] else "", "_relu6" if c[7] else ""))
                                                 for c in DWB_CASES])
def test_depthwise_against_fp64(dev, case):
    from pretorched_x_b200 import ops
    B, C, H, W, stride, ld, clamp_in, relu6 = case
    g = torch.Generator().manual_seed(B * 7919 + C * 31 + H * 7 + W + stride)
    x = torch.randn(B, H, W, C, generator=g) * 3
    x = (x.relu() if clamp_in else x).half()             # producers that stored ReLU(x) feed clamp_in; the others are signed
    w9 = torch.randn(9, C, generator=g) * 0.3
    scale = torch.rand(C, generator=g) + 0.5
    shift = torch.randn(C, generator=g) * 0.5
    data = torch.zeros(B * H * W, ld, dtype=torch.float16)
    data[:, :C] = x.reshape(-1, C)
    a = ops.Act(data.to(dev), B, 1, H, W, C)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    M, pad = B * Ho * Wo, 2
    buf = torch.full((M + 2 * pad, ld), float("nan"), dtype=torch.float16, device=dev)
    out = buf[pad:pad + M]
    wd, sd, hd = w9.to(dev), scale.to(dev), shift.to(dev)
    y = ops.dwconv3x3(a, wd, sd, hd, stride, clamp_in=clamp_in, relu6=relu6, out=out)
    again = ops.dwconv3x3(a, wd, sd, hd, stride, clamp_in=clamp_in, relu6=relu6)
    torch.cuda.synchronize()
    assert (y.N, y.T, y.H, y.W, y.C, y.ld) == (B, 1, Ho, Wo, C, ld)
    assert torch.isnan(buf[:pad].float()).all() and torch.isnan(buf[pad + M:].float()).all(), "rows outside out= were written"
    assert torch.all(out[:, C:].cpu() == 0), "padding channels [C, ld) not zero"
    assert torch.equal(again.data.view(torch.int16), out.view(torch.int16)), "two identical calls differ"
    ref, A = dw_ref(x, w9, scale, shift, stride, clamp_in, relu6)
    r = worst_ratio(out[:, :C], ref, A, True)
    report("dwconv s%d %s" % (stride, case), r)
    assert r <= 1.0, "err/bound %.3f at %s" % (r, where_worst(out[:, :C], ref, A, True))


# ---------------------------------------------------------------------------------------------
# 4. weight gradient (wgrad_kernel + wgrad_reduce_kernel) and <w, G>
# ---------------------------------------------------------------------------------------------
def _wgrad_cases():
    """(name, N, T, H, W, Cin, Cout, (kt, kh, kw), (st, s), x sign, ldx, ldg, with_w, with_scale, with_inv); x sign: 'relu',
    'signed' or 'positive' (x, g and w all >= 0: every product adds, the accumulation budget is as small as it gets)."""
    from tests.test_gpu_finetune import WGRAD_CASES
    from tests.test_gpu_finetune_2d import THW_CASES
    out = []
    for N, T, H, W, Cin, Cout, k, s in WGRAD_CASES:
        out.append(("wgrad_%dx%dx%dx%d_%d-%d_k%d_s%d" % (N, T, H, W, Cin, Cout, k, s), N, T, H, W, Cin, Cout, (k, k, k), (s, s),
                    "relu", Cin, Cout, True, True, True))
    for N, T, H, W, Cin, Cout, k, (st, s) in THW_CASES:
        out.append(("thw_%dx%dx%dx%d_%d-%d_k%s_s%d%d" % (N, T, H, W, Cin, Cout, "".join(map(str, k)), st, s), N, T, H, W, Cin,
                    Cout, k, (st, s), "relu", Cin, Cout, True, True, True))
    out += [
        ("ho7_wo9_signed", 2, 3, 7, 9, 24, 72, (3, 3, 3), (1, 1), "signed", 24, 72, True, True, True),
        ("ho8_wo17_pitches_no_weight", 1, 2, 8, 17, 72, 24, (1, 3, 3), (1, 1), "signed", 80, 40, False, True, True),
        ("ho17_wo1_no_scale", 2, 4, 17, 1, 200, 8, (3, 3, 3), (1, 1), "signed", 200, 16, True, False, True),
        ("h1_w1_t5_no_inv", 3, 5, 1, 1, 64, 200, (3, 3, 3), (1, 1), "signed", 72, 200, True, True, False),
        ("t1_kt3_c8", 2, 1, 9, 9, 8, 72, (3, 3, 3), (1, 1), "signed", 8, 72, True, True, True),
        ("st2_odd_t5", 2, 5, 8, 8, 72, 200, (3, 3, 3), (2, 1), "signed", 72, 208, True, True, True),
        ("st2_even_t6_ho9_wo7", 1, 6, 9, 7, 24, 24, (3, 3, 3), (2, 1), "signed", 32, 24, True, True, True),
        ("s2_odd_17x15", 2, 2, 17, 15, 200, 72, (1, 3, 3), (1, 2), "signed", 200, 72, True, True, True),
        ("s2_even_16x18_1x1", 2, 2, 16, 18, 8, 200, (1, 1, 1), (1, 2), "signed", 16, 200, True, True, True),
        ("many_splits_1x1_c256", 4, 8, 28, 28, 256, 256, (1, 1, 1), (1, 1), "signed", 256, 256, True, True, True),
        ("positive_1x1x1", 2, 2, 9, 9, 72, 64, (1, 1, 1), (1, 1), "positive", 72, 64, True, True, True),
        ("positive_1x3x3", 2, 1, 16, 16, 64, 72, (1, 3, 3), (1, 1), "positive", 64, 72, True, True, True),
        ("positive_3x3x3", 1, 4, 8, 8, 24, 200, (3, 3, 3), (1, 1), "positive", 24, 200, True, True, True),
        ("no_weight_no_scale_no_inv", 1, 3, 9, 8, 24, 24, (3, 3, 3), (1, 1), "signed", 24, 24, False, False, False),
    ]
    return out


WGRAD_BOUND_CASES = _wgrad_cases()


def wgrad_splits(lib, case):
    """(splits, position blocks) of a WGRAD_BOUND_CASES case, from the workspace query (host only)."""
    _, N, T, H, W, Cin, Cout, k, (st, s) = case[:9]
    pt, p = k[0] // 2, k[1] // 2
    n = lib.b2_conv_wgrad_thw_workspace_elems(N, T, H, W, Cin, Cout, k[0], k[1], k[2], st, s, pt, p)
    taps = k[0] * k[1] * k[2]
    assert n % (taps * Cout * Cin) == 0
    To, Ho, Wo = (T + 2 * pt - k[0]) // st + 1, (H + 2 * p - k[1]) // s + 1, (W + 2 * p - k[2]) // s + 1
    return n // (taps * Cout * Cin), N * To * -(-Ho // 8) * -(-Wo // 8)


@pytest.mark.parametrize("case", WGRAD_BOUND_CASES, ids=[c[0] for c in WGRAD_BOUND_CASES])
def test_wgrad_against_fp64(dev, lib, case):
    from pretorched_x_b200 import ops
    name, N, T, H, W, Cin, Cout, k, (st, s), sign, ldx, ldg, with_w, with_scale, with_inv = case
    pad = (k[0] // 2, k[1] // 2, k[2] // 2)
    stride = (st, s, s)
    To, Ho, Wo = ((n + 2 * pp - kk) // ss + 1 for n, kk, ss, pp in zip((T, H, W), k, stride, pad))
    gen = torch.Generator().manual_seed(seed_of(name))
    x = torch.randn(N, Cin, T, H, W, generator=gen)
    g = torch.randn(N, Cout, To, Ho, Wo, generator=gen)
    w = torch.randn((Cout, Cin) + tuple(k), generator=gen) * 0.05
    if sign == "relu":
        x = x.relu()
    elif sign == "positive":
        x, g, w = x.abs(), g.abs(), w.abs()
    x16, g16 = x.half(), g.half()
    scale = torch.rand(Cout, generator=gen) + 0.5 if with_scale else None
    inv = torch.tensor([2.0 ** -3]) if with_inv else None
    xa = ops.from_ncdhw(x16.to(dev), pitch=ldx)
    ga = ops.from_ncdhw(g16.to(dev), pitch=ldg)
    splits, nbox = wgrad_splits(lib, case)
    kw = dict(weight=w.to(dev) if with_w else None, scale=scale.to(dev) if with_scale else None,
              inv_loss_scale=inv.to(dev) if with_inv else None)
    dw, dot = ops.conv_wgrad(ga, xa, k, stride, pad, **kw)
    dw2, dot2 = ops.conv_wgrad(ga, xa, k, stride, pad, **kw)
    torch.cuda.synchronize()
    assert tuple(dw.shape) == (Cout, Cin) + tuple(k)
    assert torch.equal(dw.view(torch.int32), dw2.view(torch.int32)), "weight gradient is not bitwise repeatable"
    G, Mg, ref, A = wgrad_ref(x16, g16, k, stride, pad, scale, inv)
    label = "wgrad %s splits %d nbox %d" % (name, splits, nbox)
    check_bound(label, dw, ref, wgrad_bound(A, nbox, splits))
    if with_w:
        assert torch.equal(dot.view(torch.int32), dot2.view(torch.int32)), "<w, G> is not bitwise repeatable"
        dref, dbnd = wdot_ref(G, Mg, w, inv, nbox, splits)
        check_bound("wdot " + label, dot, dref, dbnd)
    else:
        assert dot is None
