"""Host logic (no GPU): where the slab kernel's 128-wide transposed form (b2_slab_t128.cuh) is taken, and that its plans are ones the
kernel can run -- a compiled item width that holds the item's whole rows, and shared memory within 227 KB."""
import ctypes

import pytest

WIDTHS = (216, 224, 256)
SMEM = 227 * 1024
KEYS = "taken applies NP rows R items smem slab_items slab_MT sms".split()


@pytest.fixture(scope="module")
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_slab_t128_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    lib.b2_debug_set_slab_t128.argtypes = [ctypes.c_int]
    lib.b2_debug_set_slab_t128(-1)
    yield lib
    lib.b2_debug_set_slab_t128(-1)


def plan(lib, N, C, T, H, W, K, k, s=(1, 1, 1), residual=False):
    from pretorched_x_b200 import _lib
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K = N, T, H, W, (C + 7) // 8 * 8, K
    a.ldy = (K + 7) // 8 * 8
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = s
    a.pt, a.ph, a.pw = k[0] // 2, k[1] // 2, k[2] // 2
    if residual:
        a.residual, a.ldr = 16, a.ldy            # never dereferenced by the host-only plan
    out = (ctypes.c_int * 10)()
    assert lib.b2_debug_slab_t128_plan(ctypes.byref(a), out) == 0
    return dict(zip(KEYS, list(out)))


K333, K133 = (3, 3, 3), (1, 3, 3)
# conv2 of the bottlenecks of layers 2-3 at the benchmark batch sizes: resnet3d50 (32 clips of 16 frames), nonlocal50 (8 clips of 32
# frames: layer2), TRN on resnet50 (32 clips x 8 segments = 256 images); stride 1 and the strided first block of each layer
TAKEN = [
    ("r3d50_layer2", (32, 128, 4, 28, 28, 128, K333)),
    ("r3d50_layer2.0_s2", (32, 128, 8, 56, 56, 128, K333, (2, 2, 2))),
    ("r3d50_layer3", (32, 256, 2, 14, 14, 256, K333)),
    ("r3d50_layer3.0_s2", (32, 256, 4, 28, 28, 256, K333, (2, 2, 2))),
    ("nonlocal50_layer2", (8, 128, 8, 28, 28, 128, K333)),
    ("nonlocal50_layer2.0_s2", (8, 128, 16, 56, 56, 128, K333, (2, 2, 2))),
    ("trn_r50_layer2", (256, 128, 1, 28, 28, 128, K133)),
    ("trn_r50_layer2.0_s2", (256, 128, 1, 56, 56, 128, K133, (1, 2, 2))),
    ("trn_r50_layer3", (256, 256, 1, 14, 14, 256, K133)),
    ("trn_r50_layer3.0_s2", (256, 256, 1, 28, 28, 256, K133, (1, 2, 2))),
]
# the slab shapes of the existing kernel tests: C = 72, too few items to fill the SMs, multi-plane items, the temporal remap, a
# residual, 64 output channels
DECLINED = [
    ("slab_fixed128_s2_c72", (1, 72, 3, 13, 13, 128, K333, (2, 2, 2))),
    ("slab_wide_256", (2, 64, 1, 10, 12, 256, K133)),
    ("slab_layer3_14x14", (3, 256, 2, 14, 14, 256, K333)),
    ("slab_multiplane_7x7_192", (9, 128, 3, 7, 7, 192, K133)),
    ("slab_multiplane_7x7_T1_3x3x3", (23, 128, 1, 7, 7, 128, K333)),
    ("slab_multiplane_5x6_c512_256wide", (41, 512, 1, 5, 6, 256, K133)),
    ("temporal3_14x14_from_576", (2, 576, 4, 14, 14, 256, (3, 1, 1))),
    ("slab_layer2_28x28_res", (2, 128, 3, 28, 28, 128, K333), True),
    ("slab_s2_56_to_28", (2, 128, 4, 56, 56, 128, K333, (2, 2, 2))),
    ("r3d50_layer1", (32, 64, 8, 56, 56, 64, K333)),
    ("r3d50_layer4", (32, 512, 1, 7, 7, 512, K333)),
    ("nonlocal50_layer3", (8, 256, 4, 14, 14, 256, K333)),      # 64 items: one round either way, and a longer one
]


@pytest.mark.parametrize("name,shape", TAKEN, ids=[t[0] for t in TAKEN])
def test_rule_takes_bottleneck_layers(lib, name, shape):
    p = plan(lib, *shape)
    assert p["taken"] == 1 and p["applies"] == 1, p
    assert p["NP"] in WIDTHS and p["smem"] <= SMEM, p
    N, C, T, H, W, K, k = shape[:7]
    s = shape[7] if len(shape) > 7 else (1, 1, 1)
    Ho, Wo = (H - 1) // s[1] + 1, (W - 1) // s[2] + 1
    PW = Wo + (2 if s[1] == 1 else 1)                      # halo columns of the padded rows
    assert p["NP"] == min(w for w in WIDTHS if w >= p["rows"] * PW), p
    To = (T - 1) // s[0] + 1
    assert p["items"] == N * To * -(-Ho // p["rows"]) * (K // 128), p
    sms = p["sms"]                                         # the SM count of the device the rule planned for (132 without one)
    assert -(-p["items"] // sms) * p["NP"] <= -(-p["slab_items"] // sms) * p["slab_MT"] * 128, p


@pytest.mark.parametrize("case", DECLINED, ids=[d[0] for d in DECLINED])
def test_rule_declines_slab_test_shapes(lib, case):
    name, shape = case[0], case[1]
    p = plan(lib, *shape, residual=len(case) > 2)
    assert p["taken"] == 0, p


def test_force_and_off(lib):
    shape = (2, 128, 2, 28, 28, 128, K333)                 # eligible, but too few items for the rule
    assert plan(lib, *shape)["taken"] == 0
    try:
        lib.b2_debug_set_slab_t128(1)
        p = plan(lib, *shape)
        assert p["taken"] == 1 and p["NP"] == 216 and p["rows"] == 7 and p["smem"] <= SMEM, p
        lib.b2_debug_set_slab_t128(0)
        assert plan(lib, 32, 128, 4, 28, 28, 128, K333)["taken"] == 0
    finally:
        lib.b2_debug_set_slab_t128(-1)


def test_every_eligible_plan_fits(lib):
    """Over planes of 4 ... 64 rows and both strides: a plan the form accepts always holds its rows and fits in shared memory."""
    try:
        lib.b2_debug_set_slab_t128(1)
        seen = 0
        for H in range(4, 65):
            for s in (1, 2):
                p = plan(lib, 2, 128, 3, H, H, 256, K333, (s, s, s))
                if not p["applies"]:
                    continue
                seen += 1
                Wo = (H - 1) // s + 1
                PW = Wo + (2 if s == 1 else 1)
                assert p["NP"] in WIDTHS and p["rows"] * PW <= p["NP"] and p["smem"] <= SMEM, (H, s, p)
        assert seen > 40
    finally:
        lib.b2_debug_set_slab_t128(-1)
