"""CPU: the per-element references of tests/kernel_ref.py that tests/test_gpu_kernel_bounds.py holds the stem (with its fused W
max-pool), depthwise 3x3 and weight-gradient kernels to.  For each, the exact result rounded the way the kernel's output is
rounded passes, and a concrete fault that the kernel's older per-tensor metric lets through fails -- both halves asserted.  Also
host-only: the dispatch knobs, the stem instance plan of every GPU stem case and the weight-gradient workspace query behave as
the GPU file assumes."""
import ctypes

import torch
import torch.nn.functional as F

from pretorched_x_b200 import _lib
from tests.kernel_ref import (FLOOR, bound, conv_ref, dw_ref, pool_w, stem_operands, wdot_ref, wgrad_b, wgrad_bound, wgrad_ref,
                              worst_ratio, worst_ratio_of)


def rel(got, ref):
    """The per-tensor metric of the older stem / depthwise / weight-gradient tests: max |got - ref| / max |ref|."""
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def cos(got, ref):
    return float(F.cosine_similarity(got.double().reshape(-1), ref.double().reshape(-1), dim=0))


# ---------------------------------------------------------------------------------------------
# stem
# ---------------------------------------------------------------------------------------------
SMALL = 5                      # the channel with a small BN scale (and no shift): its values are 2^-10 of the others'


def stem_problem(seed, T=3, H=12, W=22, K=16, k=(3, 7, 7), p=(1, 3, 3)):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 3, T, H, W, generator=g)
    weight = torch.randn((K, 3) + k, generator=g) / (3 * k[0] * k[1] * k[2]) ** 0.5
    scale = torch.rand(K, generator=g) + 0.5
    shift = torch.randn(K, generator=g) * 0.1
    scale[SMALL], shift[SMALL] = 2.0 ** -10, 0.0
    x4, w4 = stem_operands(x, weight)
    ref, A = conv_ref(x4, w4, scale, shift, k, (1, 2, 2), p, relu=True)
    To, Ho, Wo = T + 2 * p[0] - k[0] + 1, (H + 2 * p[1] - k[1]) // 2 + 1, (W + 6 - 7) // 2 + 1
    return x4, w4, scale, shift, ref, A, (To, Ho, Wo), k, p


def test_stem_operands_are_the_fp16_filter_and_ndhwc4_input():
    x = torch.randn(2, 3, 2, 4, 6)
    w = torch.randn(8, 3, 1, 7, 7)
    x4, w4 = stem_operands(x, w)
    assert x4.dtype == w4.dtype == torch.float16
    assert torch.all(x4[..., 3] == 0) and torch.all(w4[..., 3] == 0)
    assert torch.equal(x4[..., :3], x.half().permute(0, 2, 3, 4, 1))
    assert torch.equal(w4[:, 7 * 2 + 5, :3], w.half()[:, :, 0, 2, 5])            # tap (dt, dh, dw) = (0, 2, 5)


def test_stem_exact_result_rounded_once_to_fp16_passes():
    *_, ref, A, (To, Ho, Wo), _, _ = stem_problem(1)
    assert worst_ratio(ref.half(), ref, A, True) <= 1.0
    pref, pbnd = pool_w(ref, A, Wo)
    assert worst_ratio_of(pool_w(ref.half().double(), A, Wo)[0], pref, pbnd) <= 1.0   # pooling the rounded values


def test_stem_dropped_slab_row_at_a_border_output_in_a_small_scale_channel():
    """Output row 0 (top border: slab rows above the image are padding) loses its first in-image slab row, in the channel with a
    small BN scale.  Its error is ~2^-10 of the tensor's largest value: inside the 2e-3 per-tensor metric, far outside the bound."""
    x4, w4, sc, sh, ref, A, (To, Ho, Wo), k, p = stem_problem(2)
    xb = x4.clone()
    xb[:, :, 0] = 0                                           # input row 0 is the first in-image slab row of output row 0
    bad, _ = conv_ref(xb, w4, sc, sh, k, (1, 2, 2), p, relu=True)
    got = ref.clone().reshape(To, Ho, Wo, -1)
    got[:, 0, :, SMALL] = bad.reshape(To, Ho, Wo, -1)[:, 0, :, SMALL]
    got = got.reshape(ref.shape).half()
    assert rel(got, ref) <= 2e-3
    assert worst_ratio(got, ref, A, True) > 1.0


def test_stem_pool_window_shifted_at_the_right_edge():
    """The last pooled column of every row takes the window {Wo - 3, Wo - 2, Wo - 1} instead of {Wo - 2, Wo - 1} (odd Wo: the
    window's third column is past the row), in the small-scale channel: passes the per-tensor metric, fails the bound."""
    *_, ref, A, (To, Ho, Wo), _, _ = stem_problem(3, W=22)
    assert Wo % 2 == 1
    pref, pbnd = pool_w(ref, A, Wo)
    got = pool_w(ref.half().double(), A, Wo)[0]
    K = ref.shape[1]
    r16 = ref.half().double().reshape(-1, Wo, K)
    Wp = (Wo - 1) // 2 + 1
    g = got.reshape(-1, Wp, K)
    g[:, Wp - 1, SMALL] = r16[:, Wo - 3:Wo, SMALL].amax(dim=1)
    assert bool((g.reshape(pref.shape) != pref.half().double()).any())
    assert rel(got, pref) <= 2e-3
    assert worst_ratio_of(got, pref, pbnd) > 1.0


def test_pooled_bound_is_the_window_maximum_of_the_element_bounds():
    ref = torch.tensor([[0.0], [1.0], [3.0], [2.0], [5.0]], dtype=torch.float64)
    A = torch.tensor([[1.0], [2.0], [0.5], [8.0], [1.0]], dtype=torch.float64)
    pref, pbnd = pool_w(ref, A, 5)
    assert pref.reshape(-1).tolist() == [1.0, 3.0, 5.0]
    b = bound(ref, A, True).reshape(-1)
    assert pbnd.reshape(-1).tolist() == [max(b[0], b[1]), max(b[1], b[2], b[3]), max(b[3], b[4])]


# ---------------------------------------------------------------------------------------------
# depthwise 3x3
# ---------------------------------------------------------------------------------------------
def dw_problem(seed, B=2, H=9, W=11, C=24, stride=1, clamp_in=True):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, W, C, generator=g) * 3).relu().half()
    w9 = torch.randn(9, C, generator=g) * 0.3
    scale = torch.rand(C, generator=g) + 0.5
    shift = torch.randn(C, generator=g) * 0.5
    scale[SMALL], shift[SMALL] = 2.0 ** -10, 0.0
    return x, w9, scale, shift


def test_dw_exact_result_rounded_once_to_fp16_passes():
    for stride, clamp_in, relu6 in ((1, True, True), (2, False, True), (2, True, False)):
        x, w9, sc, sh = dw_problem(4)
        ref, A = dw_ref(x, w9, sc, sh, stride, clamp_in, relu6)
        assert worst_ratio(ref.half(), ref, A, True) <= 1.0


def test_dw_clamp_in_is_applied_before_the_taps():
    x = torch.full((1, 1, 1, 8), 10.0).half()
    w9 = torch.zeros(9, 8)
    w9[4] = 1.0
    ref, _ = dw_ref(x, w9, torch.ones(8), torch.zeros(8), 1, True, False)
    assert torch.all(ref == 6.0)


def test_dw_dropped_right_edge_tap_in_a_small_scale_channel():
    """The last output column of each row (the ragged end of a run of R = 4 columns when Wo = 11) loses its left tap column in the
    small-scale channel: inside the 2e-3 per-tensor metric, outside the bound."""
    x, w9, sc, sh = dw_problem(5)
    ref, A = dw_ref(x, w9, sc, sh, 1, True, True)
    w_bad = w9.clone()
    w_bad[[0, 3, 6], SMALL] = 0                                # kw = 0 of every row
    bad, _ = dw_ref(x, w_bad, sc, sh, 1, True, True)
    B, Ho, Wo, C = 2, 9, 11, 24
    got = ref.clone().reshape(B, Ho, Wo, C)
    got[:, :, Wo - 1, SMALL] = bad.reshape(B, Ho, Wo, C)[:, :, Wo - 1, SMALL]
    got = got.reshape(ref.shape).half()
    assert rel(got, ref) <= 2e-3
    assert worst_ratio(got, ref, A, True) > 1.0


# ---------------------------------------------------------------------------------------------
# weight gradient and <w, G>
# ---------------------------------------------------------------------------------------------
def wg_problem(seed, positive, N=1, T=4, H=8, W=8, Cin=16, Cout=24, k=(3, 3, 3)):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, T, H, W, generator=g).half()
    gr = torch.randn(N, Cout, T, H, W, generator=g).half()
    w = torch.randn((Cout, Cin) + k, generator=g) * 0.05
    if positive:
        x, gr, w = x.abs(), gr.abs(), w.abs()
    scale = torch.rand(Cout, generator=g) + 0.5
    return x, gr, w, scale


def old_wgrad_metric_passes(got, ref):
    """The older weight-gradient test: rel <= 1e-3 and cosine >= 0.999999."""
    return rel(got, ref) <= 1e-3 and cos(got, ref) >= 0.999999


def test_wgrad_exact_result_rounded_once_to_fp32_passes():
    for positive in (False, True):
        x, gr, w, sc = wg_problem(6, positive)
        inv = torch.tensor(0.25)
        G, M, dW, A = wgrad_ref(x, gr, (3, 3, 3), 1, 1, sc, inv)
        assert worst_ratio_of(dW.float(), dW, wgrad_bound(A, 4, 2)) <= 1.0
        ref, bnd = wdot_ref(G, M, w, inv, 4, 2)
        assert worst_ratio_of(ref.float(), ref, bnd) <= 1.0
    G, M, dW, A = wgrad_ref(x, gr, (3, 3, 3), 1, 1)                  # scale = inv = None
    assert torch.equal(dW, G) and torch.equal(A, M)


def test_wgrad_b_grows_with_the_accumulation_chain():
    assert wgrad_b(4, 2) == 2.0 ** -14
    assert wgrad_b(4000, 1) == (64 * 4000 + 3) * FLOOR
    assert wgrad_b(4001, 2) == (64 * 2001 + 4) * FLOOR


def test_wgrad_split_partials_rounded_to_fp16_fail():
    """Each split's partial G kept in fp16 instead of fp32 (all-positive problem, 4 position blocks = 4 frames of 8 x 8 in 2
    splits): relative errors ~2^-12 pass rel <= 1e-3 and cosine >= 0.999999 and fail the bound."""
    x, gr, w, sc = wg_problem(7, True)
    inv = torch.tensor(0.25)
    G, M, dW, A = wgrad_ref(x, gr, (3, 3, 3), 1, 1, sc, inv)
    parts = []
    for frames in ((0, 1), (2, 3)):                             # split j: position blocks (= frames) [2j, 2j + 2)
        gj = torch.zeros_like(gr)
        gj[:, :, list(frames)] = gr[:, :, list(frames)]
        parts.append(wgrad_ref(x, gj, (3, 3, 3), 1, 1)[0].half().double())
    got = (parts[0] + parts[1]) * 0.25 * sc.double().view(-1, 1, 1, 1, 1)
    assert old_wgrad_metric_passes(got, dW)
    assert worst_ratio_of(got, dW, wgrad_bound(A, 4, 2)) > 1.0


def test_wgrad_inverse_loss_scale_in_fp16_fails():
    """inv = 1/3 applied after rounding to fp16 (a relative change of 2^-12): a uniform scale, so the cosine is exactly 1 and the
    relative error stays under 1e-3 -- for dW and for <w, G> alike; both fail the bound on an all-positive problem."""
    x, gr, w, sc = wg_problem(8, True)
    inv = torch.tensor(1.0 / 3.0)
    inv16 = inv.half().float()
    G, M, dW, A = wgrad_ref(x, gr, (3, 3, 3), 1, 1, sc, inv)
    bad = wgrad_ref(x, gr, (3, 3, 3), 1, 1, sc, inv16)[2]
    assert old_wgrad_metric_passes(bad, dW)
    assert worst_ratio_of(bad, dW, wgrad_bound(A, 4, 2)) > 1.0
    ref, bnd = wdot_ref(G, M, w, inv, 4, 2)
    bad_dot = wdot_ref(G, M, w, inv16, 4, 2)[0]
    assert old_wgrad_metric_passes(bad_dot, ref)
    assert worst_ratio_of(bad_dot, ref, bnd) > 1.0


# ---------------------------------------------------------------------------------------------
# host-only: knobs, stem instance plans, weight-gradient workspace
# ---------------------------------------------------------------------------------------------
def test_every_full_layer_shape_has_a_recorded_kernel():
    """A shape added to tests/test_gpu_kernels.py::CONV_CASES needs the kernel the rule picks for it recorded beside it."""
    from tests.test_gpu_kernel_bounds import LAYER_CASES
    assert all(c[-1] is not None for c in LAYER_CASES), [c[0] for c in LAYER_CASES if c[-1] is None]


def test_knobs_and_host_plans_work_without_a_gpu():
    from tests.test_gpu_kernel_bounds import STEM_CASES, WGRAD_BOUND_CASES, reset_knobs, stem_expect, wgrad_splits
    lib = _lib.load()
    lib.b2_debug_set_stem_rows.argtypes = [ctypes.c_int]
    try:
        for v in (-1, 2, 4, 4 | 16):
            assert lib.b2_debug_set_stem_rows(v) == 0
        assert lib.b2_debug_set_tstack(1) == 0 and lib.b2_debug_set_densem(-1, 0) == 0
        out = (ctypes.c_int * 2)()
        lib.b2_debug_set_stem_rows(2)                          # forcing is visible in the host plan
        assert lib.b2_debug_stem_plan(64, 7, 7, 56, 0, out) == 0 and tuple(out) == (2, 0)
        lib.b2_debug_set_stem_rows(4 | 16)
        lib.b2_debug_stem_plan(64, 7, 7, 56, 0, out)
        assert tuple(out) == (4, 1)
        lib.b2_debug_stem_plan(64, 7, 7, 113, 0, out)          # past the 112-column transposed tile
        assert tuple(out) == (4, 0)
        lib.b2_debug_stem_plan(64, 1, 7, 56, 1, out)           # pair mode keeps two rows whatever is forced
        assert tuple(out) == (2, 0)
        lib.b2_debug_set_stem_rows(4)
        lib.b2_debug_stem_plan(64, 3, 13, 56, 0, out)          # kh = 13: no room for G = 4's ring
        assert tuple(out) == (2, 0)
    finally:
        reset_knobs(lib)
    # every GPU stem case: the instances its forcings resolve to, and each case's reason to exist
    seen = set()
    for c in STEM_CASES:
        exp = stem_expect(lib, c)
        assert set(exp) == {-1, 2, 4, 4 | 16}
        seen.update(exp.values())
        name, N, T, H, W, K, k, p, pooled, want_rule = c
        assert exp[-1] == want_rule, (name, exp[-1])
    assert {(1, 1, 0), (1, 2, 0), (1, 4, 0), (1, 4, 1)} <= seen
    # the weight-gradient workspace query: splits from the host plan, and the three split regimes all covered
    kinds = set()
    for c in WGRAD_BOUND_CASES:
        splits, nbox = wgrad_splits(lib, c)
        assert 1 <= splits <= 64 and splits <= max(1, nbox // 4)
        kinds.add("1" if splits == 1 else ("even" if nbox % splits == 0 else "ragged"))
    assert kinds == {"1", "even", "ragged"}
