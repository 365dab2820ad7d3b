"""GPU (-m gpu): the slab kernels with register accumulators (b2_slabconv.cuh, b2_slabts.cuh).  Every launch here has more than
3 x SM-count work items, so each persistent CTA hands many items to its epilogue through the single accumulator tile; each compiled
N width of the consumer loop runs, MT * N reaches the register bound (kSlabAccCols = 192 columns), multi-plane items use the
largest plane count the planner allows, and residuals are added on ragged last M tiles."""
import ctypes

import pytest
import torch

from .test_gpu_kernels import check_conv_case, dev  # noqa: F401  (dev: fixture)

pytestmark = pytest.mark.gpu

ACC_COLS = 192      # kSlabAccCols


def slab_plan(N, C, T, H, W, K, k):
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_slab_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K = N, T, H, W, (C + 7) // 8 * 8, K
    a.ldy = (K + 7) // 8 * 8
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = 1, 1, 1
    a.pt, a.ph, a.pw = k[0] // 2, k[1] // 2, k[2] // 2
    out = (ctypes.c_int * 10)()
    assert lib.b2_debug_slab_plan(ctypes.byref(a), out) == 0
    return dict(zip("applies BN MT R PW WC wchunks items flex remap".split(), list(out)))


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# name, N, Cin, T, H, W, K, kernel, residual, expected N tile, expected MT (None: any)
MANY_ITEM_CASES = [
    ("n64_res_ragged_56x56", 4, 64, 8, 56, 56, 64, (3, 3, 3), True, 64, None),       # 3248 positions per plane: ragged last tile
    ("n128_28x28", 8, 128, 8, 28, 28, 128, (3, 3, 3), False, 128, 1),
    ("n16_rgb_head_mt3", 8, 64, 32, 28, 28, 3, (1, 3, 3), True, 16, 3),
    ("n144_res_28x28", 4, 64, 16, 28, 28, 144, (1, 3, 3), True, 144, 1),
    ("n160_28x28", 4, 64, 16, 28, 28, 160, (1, 3, 3), False, 160, 1),
    ("n176_7x7_res", 64, 128, 8, 7, 7, 176, (1, 3, 3), True, 176, 1),
    ("n192_7x7", 64, 128, 8, 7, 7, 192, (1, 3, 3), False, 192, 1),
    ("multiplane_7x7_n64", 128, 128, 8, 7, 7, 64, (1, 3, 3), True, 64, 2),
]


@pytest.mark.parametrize("case", MANY_ITEM_CASES, ids=[c[0] for c in MANY_ITEM_CASES])
def test_slab_many_items_per_cta(dev, case):  # noqa: F811
    name, N, C, T, H, W, K, k, res, bn, mt = case
    p = slab_plan(N, C, T, H, W, K, k)
    items = p["items"] // p["MT"] if H * (W + 2) <= 128 else p["items"]       # (the debug plan counts planes, not plane groups)
    assert p["applies"] and p["BN"] == bn and items > 3 * sm_count()
    assert p["MT"] * p["BN"] <= ACC_COLS and (mt is None or p["MT"] == mt)
    check_conv_case(dev, (name, N, C, T, H, W, K, k, (1, 1, 1), tuple(x // 2 for x in k), res, True, False, True), False)


def test_slab_mt_at_register_bound(dev):  # noqa: F811
    """MT * N = 192, the whole register budget of the consumers: N = 64 with MT forced to 3 (multi-plane 7x7 items, the only MT = 3
    slab of N = 64 that fits in shared memory next to the accumulator tile; 401 planes leave the last group partial, residual)."""
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_set_slab_mt(3)
    try:
        p = slab_plan(401, 128, 1, 7, 7, 64, (1, 3, 3))
        assert p["applies"] and p["BN"] == 64 and p["MT"] * p["BN"] == ACC_COLS
        check_conv_case(dev, ("mt3_n64_multiplane_res", 401, 128, 1, 7, 7, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), True, True, False, True),
                        False)
    finally:
        lib.b2_debug_set_slab_mt(0)


def test_slab_multiplane_largest_group(dev):  # noqa: F811
    """Small planes at N = 16: the planner groups four planes per item, the most the item decode allows; odd plane count."""
    p = slab_plan(401, 128, 1, 7, 7, 16, (1, 3, 3))
    assert p["applies"] and p["BN"] == 16 and p["MT"] == 4
    check_conv_case(dev, ("mp4_n16_res", 401, 128, 1, 7, 7, 16, (1, 3, 3), (1, 1, 1), (0, 1, 1), True, True, False, True), False)


def test_slabts_many_items_per_cta(dev):  # noqa: F811
    """The temporal-group kernel (no residual, Cout <= 64) over 6 clips of layer1 shape: 26 tiles x 3 frame groups x 6 clips."""
    check_conv_case(dev, ("slabts_many_items", 6, 64, 8, 56, 56, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), False, True, False, True),
                    False)
