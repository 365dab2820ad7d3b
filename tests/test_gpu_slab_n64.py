"""GPU (-m gpu): the slab kernel's 64-wide output tile (b2_slabconv.cuh), which computes the transposed product -- the weight stage
as the m64 A operand, the item's slab positions as a K-major B operand of N = 64 MT -- against fp64 with the bound of
tests/kernel_ref.py.  Every case pins KID_SLAB and the plan ({64, MT, 0, wchunks, remapped}); run_f16 also checks the zero padding
columns, the untouched rows around the output and that two identical calls are bitwise equal."""
import pytest

from tests.conftest import has_h100
from tests.test_gpu_kernel_matrix import SLAB, dev, lib, make, plan_info, run_f16, slab_plan  # noqa: F401 (fixtures)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

S1, P3, P133 = (1, 1, 1), (1, 1, 1), (0, 1, 1)
# (name, N, Cin, pitch, T, H, W, K, k, s, p, residual, forced MT or 0, check(plan) -> bool)
CASES = [
    # resnet3d50 layer1 (64 -> 64, 8 x 56 x 56) at batch 2 instead of 32
    ("n64_r3d50_layer1_b2", 2, 64, 64, 8, 56, 56, 64, (3, 3, 3), S1, P3, False, 0, lambda pl: True),
    ("n64_r3d50_layer1_b2_res", 2, 64, 64, 8, 56, 56, 64, (3, 3, 3), S1, P3, True, 0, lambda pl: True),
    # padded rows of 22, MT = 2 (256 positions per item): 17 x 22 = 374 = one item + 118 (the last item has mt_valid 1 of 2: the
    # second warpgroup's whole half lies past the plane); 20 x 22 = 440 = one item + 184 (mt_valid 2, the second tile part-filled)
    ("n64_ragged_mtvalid1", 1, 64, 64, 3, 17, 20, 64, (3, 3, 3), S1, P3, False, 2, lambda pl: True),
    ("n64_ragged_mtvalid2", 1, 64, 64, 3, 20, 20, 64, (3, 3, 3), S1, P3, True, 2, lambda pl: True),
    ("n64_forced_mt1", 1, 64, 64, 3, 24, 20, 64, (3, 3, 3), S1, P3, False, 1, lambda pl: True),
    ("n64_forced_mt2", 1, 64, 64, 3, 24, 20, 64, (3, 3, 3), S1, P3, False, 2, lambda pl: True),
    # fewer output channels: rows [K, 64) of the weight tile are TMA zero fill; ldy 48 > K = 44 checks the zero padding columns
    ("n64_cout48", 1, 64, 64, 3, 16, 18, 48, (3, 3, 3), S1, P3, True, 0, lambda pl: True),
    ("n64_cout44_pad", 1, 40, 40, 3, 16, 18, 44, (3, 3, 3), S1, P3, False, 0, lambda pl: True),
    ("n64_c128_in", 1, 128, 128, 3, 14, 15, 64, (3, 3, 3), S1, P3, True, 0, lambda pl: True),
    # rows longer than a TMA box: W chunks, each with its own halo
    ("n64_wchunks_300", 1, 64, 64, 1, 5, 300, 64, (1, 3, 3), S1, P133, True, 0, lambda pl: pl[6] >= 2),
    # 7 x 7 planes (63 padded positions): MT consecutive planes per item, one m64n64k16 per plane chunk.  MT = 3 fits only here
    # (a plane's slab is small); 15 planes = five items of three, 14 = a last item with 2 of 3 planes
    ("n64_multiplane_7x7_mt3", 5, 64, 64, 3, 7, 7, 64, (1, 3, 3), S1, P133, True, 3, lambda pl: True),
    ("n64_multiplane_7x7_mt3_ragged", 7, 64, 64, 2, 7, 7, 64, (1, 3, 3), S1, P133, False, 3, lambda pl: True),
    ("n64_multiplane_8x6_mt2", 3, 64, 64, 3, 8, 6, 64, (1, 3, 3), S1, P133, True, 2, lambda pl: True),
    ("n64_2d_3x3", 4, 64, 64, 1, 28, 28, 64, (1, 3, 3), S1, P133, True, 0, lambda pl: True),
    ("n64_stride2", 1, 64, 64, 4, 17, 17, 64, (3, 3, 3), (2, 2, 2), P3, False, 0, lambda pl: True),
    # (3,1,1) over 144 channels to 64: run as a (1,3,1) filter over frames x (H*W) once the temporal stack kernel is off
    ("n64_remap_3x1x1", 2, 144, 144, 6, 10, 10, 64, (3, 1, 1), S1, (1, 0, 0), True, 0, lambda pl: pl[9] == 1),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_slab_n64_against_fp64(dev, lib, case):  # noqa: F811
    name, residual, mt, check = case[0], case[11], case[12], case[13]
    geo = case[:11]
    lib.b2_debug_set_densem(0, 0)                 # small planes: keep them off the dense-M kernel
    lib.b2_debug_set_tstack(0)
    if mt:
        lib.b2_debug_set_slab_mt(mt)
    plan = slab_plan(lib, geo)
    assert plan[0] == 1 and plan[1] == 64 and plan[8] == 0, (name, plan)
    assert (not mt or plan[2] == mt) and check(plan), (name, plan)
    pb = make(dev, geo)
    kid, info = run_f16(dev, lib, pb, residual=residual, relu=True)
    assert kid == SLAB and info == plan_info(plan), (name, kid, info, plan)
