"""CPU: the elementwise bound of tests/kernel_ref.py (which tests/test_gpu_kernel_matrix.py holds every kernel variant to) fails
on the faults a max-relative metric lets through and passes the exact result rounded once to fp16; the library exports the
kernel probe and the knobs that test relies on, and they work without a GPU."""
import ctypes

import torch

from pretorched_x_b200 import _lib
from tests.kernel_ref import conv_ref, worst_ratio

K, C = 48, 64


def problem(seed=0, positive=False):
    """A 3x3x3 convolution with ragged borders: x [1, 3, 5, 7, C], packed filter [K, 27, C], folded affine."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 3, 5, 7, C, generator=g).half()
    w = (torch.randn(K, 27, C, generator=g) / (27 * C) ** 0.5).half()
    if positive:                     # every product has the same sign: the accumulation error budget is as small as it gets
        x, w = x.abs(), w.abs()
    scale = (torch.rand(K, generator=g) + 0.5).float()
    shift = (torch.randn(K, generator=g) * 0.1).float()
    return x, w, scale, shift


def ref_of(x, w, scale, shift, **kw):
    return conv_ref(x, w, scale, shift, (3, 3, 3), (1, 1, 1), (1, 1, 1), **kw)


def test_exact_result_rounded_once_to_fp16_passes():
    x, w, sc, sh = problem()
    r = torch.randn(105, K, generator=torch.Generator().manual_seed(3)).half()
    ref, A = ref_of(x, w, sc, sh, residual=r, relu=True)
    assert worst_ratio(ref.half(), ref, A, True) <= 1.0
    assert worst_ratio(ref.float(), ref, A, False) <= 1.0


def test_dropped_tap_chunk_at_one_border_position_fails():
    x, w, sc, sh = problem(1)
    ref, A = ref_of(x, w, sc, sh)
    # output (t=0, h=0, w=6): the corner; drop tap (dt=1, dh=1, dw=0) for channels [0, 64) -- one K block of the gather loop
    xb = x.clone()
    xb[0, 0, 0, 5, :] = 0
    bad, _ = ref_of(xb, w, sc, sh)
    got = ref.clone()
    row = (0 * 5 + 0) * 7 + 6
    got[row] = bad[row]
    got = got.half()
    assert worst_ratio(got, ref, A, True) > 1.0


def test_stale_ragged_tail_row_fails():
    x, w, sc, sh = problem(2)
    ref, A = ref_of(x, w, sc, sh, relu=True)
    x2, _, _, _ = problem(5)
    stale, _ = ref_of(x2, w, sc, sh, relu=True)   # what the buffer held from an earlier call
    got = ref.clone()
    got[-1] = stale[-1]                             # M = 105: the last row of the last (partial) 128-row tile
    assert worst_ratio(got.half(), ref, A, True) > 1.0


def test_scale_rounded_to_fp16_fails():
    x, w, sc, sh = problem(3, positive=True)
    sc = torch.full((K,), 1.0 + 3 * 2.0 ** -13)      # the fp16 grid at 1 is 2^-10: rounding moves it by 3 * 2^-13
    ref, A = ref_of(x, w, sc, sh)
    bad, _ = ref_of(x, w, sc.half().float(), sh)
    assert worst_ratio(bad.float(), ref, A, False) > 1.0


def test_dropped_eight_channel_chunk_fails():
    x, w, sc, sh = problem(4)
    ref, A = ref_of(x, w, sc, sh)
    xb = x.clone()
    xb[..., 40:48] = 0                             # one 16-byte chunk of every pixel
    bad, _ = ref_of(xb, w, sc, sh)
    assert worst_ratio(bad.half(), ref, A, True) > 1.0


def test_nan_in_output_fails():
    x, w, sc, sh = problem(6)
    ref, A = ref_of(x, w, sc, sh)
    got = ref.clone()
    got[17, 3] = float("nan")
    assert worst_ratio(got.half(), ref, A, True) == float("inf")


def test_kernel_probe_and_knobs_work_without_a_gpu():
    lib = _lib.load()
    info = (ctypes.c_int * 5)(*([7] * 5))
    args = _lib.ConvArgs()                         # all-null: refused before any launch
    assert lib.b2_conv_ndhwc_fprop(ctypes.byref(args), None) != 0
    assert lib.b2_debug_last_kernel(info) == 0 and list(info) == [0] * 5
    assert lib.b2_debug_last_kernel(None) == 0
    try:
        for v in (-1, 0, 1):
            assert lib.b2_debug_set_slabts(v) == 0
        assert lib.b2_debug_set_conv_algo(1) == 0 and lib.b2_debug_set_gemm_algo(1) == 0
        assert lib.b2_debug_set_densem(100, 2) == 0 and lib.b2_debug_set_slab_mt(2) == 0
        assert lib.b2_debug_set_slab_wide(1) == 0 and lib.b2_debug_set_tstack(1) == 0
        assert lib.b2_debug_set_attention_algo(1) == 0
    finally:
        lib.b2_debug_set_conv_algo(0)
        lib.b2_debug_set_gemm_algo(0)
        lib.b2_debug_set_densem(-1, 0)
        lib.b2_debug_set_slab_mt(0)
        lib.b2_debug_set_slab_wide(-1)
        lib.b2_debug_set_tstack(-1)
        lib.b2_debug_set_slabts(-1)
        lib.b2_debug_set_attention_algo(0)


def test_slab_plan_of_the_gpu_matrix_shapes():
    """The slab shapes of the GPU matrix exercise the plan each is named for (fixed / runtime N tile, W chunks, temporal
    remap), checked on the host plan so a re-fit of the constants shows here first."""
    from tests.test_gpu_kernel_matrix import PLAN_KEYS, SLAB_CASES, slab_plan
    lib = _lib.load()
    for c in SLAB_CASES:
        plan = slab_plan(lib, c)
        key, want = c[12]
        assert plan[0] == 1, c[0]
        assert (plan[PLAN_KEYS[key]] >= want if key == "wchunks" else plan[PLAN_KEYS[key]] == want), (c[0], plan)
