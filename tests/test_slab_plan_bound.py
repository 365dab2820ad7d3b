"""Host logic (no GPU): the slab kernel's tile planner never picks a plan whose accumulators exceed what the consumer warpgroups hold
in registers, MT x N <= kSlabAccCols = 192 columns (b2_slabconv.cuh)."""
import ctypes

ACC_COLS = 192      # kSlabAccCols


def _plan(lib, N, C, T, H, W, K, k, s=(1, 1, 1)):
    from pretorched_x_b200 import _lib
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K = N, T, H, W, (C + 7) // 8 * 8, K
    a.ldy = (K + 7) // 8 * 8
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = s
    a.pt, a.ph, a.pw = k[0] // 2, k[1] // 2, k[2] // 2
    out = (ctypes.c_int * 10)()
    assert lib.b2_debug_slab_plan(ctypes.byref(a), out) == 0
    return dict(zip("applies BN MT R PW WC wchunks items flex remap".split(), list(out)))


def test_slab_plans_fit_register_accumulators():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_slab_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    shapes = [
        # BASELINE layers: R(2+1)D-34 at batch 16, resnet3d50 at batch 32, resnet18 / BigGAN-like 2-D 3x3 convolutions
        (16, 64, 16, 28, 28, 144, (1, 3, 3)), (16, 144, 16, 28, 28, 64, (3, 1, 1)), (16, 128, 8, 14, 14, 288, (1, 3, 3)),
        (16, 288, 8, 14, 14, 128, (3, 1, 1)), (16, 256, 4, 7, 7, 576, (1, 3, 3)), (16, 576, 4, 7, 7, 256, (3, 1, 1)),
        (16, 512, 2, 4, 4, 1152, (1, 3, 3)), (16, 1152, 2, 4, 4, 512, (3, 1, 1)), (16, 110, 32, 56, 56, 64, (7, 1, 1)),
        (32, 64, 8, 56, 56, 64, (3, 3, 3)), (32, 128, 4, 28, 28, 128, (3, 3, 3)), (32, 256, 2, 14, 14, 256, (3, 3, 3)),
        (32, 512, 1, 7, 7, 512, (3, 3, 3)), (64, 64, 1, 56, 56, 64, (1, 3, 3)), (64, 512, 1, 7, 7, 512, (1, 3, 3)),
        (8, 1024, 1, 32, 32, 1024, (1, 3, 3)), (8, 128, 1, 256, 256, 3, (1, 3, 3)),
    ]
    for c in range(16, 1153, 8):                                 # channel counts 16 ... 1152
        shapes += [(4, c, 4, 14, 14, c, (1, 3, 3)), (8, 64, 1, 7, 7, c, (1, 3, 3)), (2, c, 8, 28, 28, 64, (3, 3, 3)),
                   (2, c, 4, 28, 28, c, (3, 1, 1))]
    taken = 0
    for sh in shapes:
        p = _plan(lib, *sh)
        if p["applies"]:
            taken += 1
            assert p["MT"] * p["BN"] <= ACC_COLS, (sh, p)
    assert taken > len(shapes) // 2

