"""Host logic (no GPU): where the slab kernel's 64-wide transposed form (slab_t_kernel<64, NP>, b2_slab_t128.cuh) is taken, and that
its plans are ones the kernel can run -- the compiled width, and shared memory within 227 KB."""
import ctypes

import pytest

NP = 168
SMEM = 227 * 1024
KEYS = "taken applies NP R items smem slab_items slab_MT sms".split()


@pytest.fixture(scope="module")
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_slab_t64_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    lib.b2_debug_set_slab_t64.argtypes = [ctypes.c_int]
    lib.b2_debug_set_slab_mt.argtypes = [ctypes.c_int]
    lib.b2_debug_set_slab_t64(-1)
    yield lib
    lib.b2_debug_set_slab_t64(-1)


def plan(lib, N, C, T, H, W, K, k, s=(1, 1, 1), residual=False, aff_ld=0):
    from pretorched_x_b200 import _lib
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K = N, T, H, W, (C + 7) // 8 * 8, K
    a.ldy = (K + 7) // 8 * 8
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = s
    a.pt, a.ph, a.pw = k[0] // 2, k[1] // 2, k[2] // 2
    if residual:
        a.residual, a.ldr = 16, a.ldy            # never dereferenced by the host-only plan
    a.aff_ld = aff_ld
    out = (ctypes.c_int * 9)()
    assert lib.b2_debug_slab_t64_plan(ctypes.byref(a), out) == 0
    return dict(zip(KEYS, list(out)))


K333, K133 = (3, 3, 3), (1, 3, 3)
# 64 -> 64 3x3 convolutions on 56 x 56 planes at the benchmark batch sizes: conv2 of layer1's bottlenecks in resnet3d50 (32 clips of
# 16 frames), nonlocal50 (8 clips of 32 frames) and TRN's resnet50 (32 clips x 8 segments = 256 images); conv1 of resnet18's
# layer1 BasicBlocks (256 images)
LAYER1 = [
    ("r3d50_layer1", (32, 64, 8, 56, 56, 64, K333)),
    ("nonlocal50_layer1", (8, 64, 16, 56, 56, 64, K333)),
    ("trn_r50_layer1", (256, 64, 1, 56, 56, 64, K133)),
    ("resnet18_layer1_conv1", (256, 64, 1, 56, 56, 64, K133)),
]


@pytest.mark.parametrize("name,shape", LAYER1, ids=[t[0] for t in LAYER1])
def test_rule_takes_layer1(lib, name, shape):
    p = plan(lib, *shape)
    assert p["taken"] == 1 and p["applies"] == 1, p
    assert p["NP"] == NP and p["smem"] <= SMEM, p
    N, T = shape[0], shape[2]
    assert p["items"] == N * T * -(-56 * 58 // (2 * NP)), p


# the slab kernel's own 64-wide cases, which tests pin to it (test_gpu_slab_n64.py, test_gpu_kernel_matrix.py), and the layer1 shapes
# with what the form does not take
DECLINED = [
    ("n64_r3d50_layer1_b2", (2, 64, 8, 56, 56, 64, K333)),
    ("n64_ragged", (1, 64, 3, 17, 20, 64, K333)),
    ("n64_c128_in", (1, 128, 3, 14, 15, 64, K333)),
    ("n64_2d_3x3", (4, 64, 1, 28, 28, 64, K133)),
    ("n64_stride2", (1, 64, 4, 17, 17, 64, K333, (2, 2, 2))),
    ("slab_fixed64_3x3x3", (1, 64, 3, 9, 11, 64, K333)),
    ("r3d50_layer1_residual", (32, 64, 8, 56, 56, 64, K333), dict(residual=True)),
    ("r3d50_layer1_per_sample_affine", (32, 64, 8, 56, 56, 64, K333), dict(aff_ld=64)),
    ("r3d50_layer1_k96", (32, 64, 8, 56, 56, 96, K333)),
    ("r3d50_layer1_c72", (32, 72, 8, 56, 56, 64, K333)),
    ("r3d50_layer1_1x1x1", (32, 64, 8, 56, 56, 64, (1, 1, 1))),
]


@pytest.mark.parametrize("case", DECLINED, ids=[d[0] for d in DECLINED])
def test_rule_declines(lib, case):
    kw = case[2] if len(case) > 2 else {}
    assert plan(lib, *case[1], **kw)["taken"] == 0


def test_forced_mt_declines(lib):
    try:
        lib.b2_debug_set_slab_mt(2)
        assert plan(lib, 32, 64, 8, 56, 56, 64, K333)["taken"] == 0
    finally:
        lib.b2_debug_set_slab_mt(0)
    assert plan(lib, 32, 64, 8, 56, 56, 64, K333)["taken"] == 1


def test_force_and_off(lib):
    shape = (2, 64, 8, 56, 56, 64, K333)                   # eligible, but too few items for the rule
    try:
        lib.b2_debug_set_slab_t64(1)
        p = plan(lib, *shape)
        assert p["taken"] == 1 and p["NP"] == NP and p["smem"] <= SMEM, p
        lib.b2_debug_set_slab_t64(0)
        assert plan(lib, 32, 64, 8, 56, 56, 64, K333)["taken"] == 0
    finally:
        lib.b2_debug_set_slab_t64(-1)


def test_every_eligible_plan_fits(lib):
    """Over planes of 4 ... 80 rows, both strides and output widths up to 64: a plan the form accepts always uses the compiled
    width, covers its items' slab rows in one TMA box and fits in shared memory."""
    try:
        lib.b2_debug_set_slab_t64(1)
        seen = 0
        for H in range(4, 81):
            for s in (1, 2):
                for K in (8, 40, 64):
                    p = plan(lib, 2, 64, 3, H, H + 3, K, K333, (s, s, s))
                    if not p["applies"]:
                        continue
                    seen += 1
                    Ho, Wo = (H - 1) // s + 1, (H + 2) // s + 1
                    PW = Wo + (2 if s == 1 else 1)
                    assert p["NP"] == NP and p["smem"] <= SMEM and s * (p["R"] - 1) + 1 <= 256, (H, s, K, p)
                    To = (3 - 1) // s + 1
                    assert p["items"] == 2 * To * -(-Ho * PW // (2 * NP)), (H, s, K, p)
        assert seen > 300
    finally:
        lib.b2_debug_set_slab_t64(-1)
