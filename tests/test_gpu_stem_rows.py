"""GPU (-m gpu): the four-output-row instance of the stem convolution (b2_stemconv.cuh, G = 4: 512 threads, one N = 64 MMA per
output row and slab row, one staging tile) against the CUDA-core cross-check, and bitwise against the two-row instance it replaces:
both accumulate every output element in the same order (temporal tap, slab row, K step)."""
import ctypes

import pytest
import torch

from tests.test_gpu_stem import POOL_FULL, POOL_TH, TOL_F16, make_stem, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    lib.b2_debug_set_stem_rows.argtypes = [ctypes.c_int]
    yield lib
    lib.b2_debug_set_stem_rows(-1)


def run_stem(lib, rows, conv, bn, a, pooled, out=None):
    from pretorched_x_b200 import engine, ops
    lib.b2_debug_set_stem_rows(rows)
    try:
        y = engine.conv_bn_act(conv, bn, a, relu=True, pool_w=pooled, out=out)
        torch.cuda.synchronize()
        ran = lib.b2_debug_last_stem_rows()
    finally:
        lib.b2_debug_set_stem_rows(-1)
    return (ops.maxpool3d(y, *POOL_TH) if pooled else y), ran


ROW_CASES = [
    # name, N, T, H, W, kernel, padding, pooled
    ("ho16_mod4_0", 1, 4, 32, 64, (7, 7, 7), (3, 3, 3), True),
    ("ho17_mod4_1", 1, 4, 34, 64, (7, 7, 7), (3, 3, 3), True),
    ("ho18_mod4_2", 1, 4, 36, 64, (7, 7, 7), (3, 3, 3), False),
    ("ho19_mod4_3", 1, 4, 38, 64, (7, 7, 7), (3, 3, 3), False),
    ("t_below_kt", 2, 3, 22, 40, (7, 7, 7), (3, 3, 3), True),
    ("items_above_sm_count", 2, 16, 224, 224, (7, 7, 7), (3, 3, 3), True),      # 896 items: the ring and staging tile wrap
    ("resnet3d50_stem_b1", 1, 16, 224, 224, (7, 7, 7), (3, 3, 3), True),
    ("nonlocal50_stem_b1", 1, 32, 224, 224, (7, 7, 7), (3, 3, 3), True),
    ("resnet18_stem_b8", 8, 1, 224, 224, (1, 7, 7), (0, 3, 3), True),
    ("three_column_tiles_unpooled", 1, 2, 18, 500, (7, 7, 7), (3, 3, 3), False),
    ("slowfast_5x7x7", 2, 8, 32, 64, (5, 7, 7), (2, 3, 3), True),
]


@pytest.mark.parametrize("case", ROW_CASES, ids=[c[0] for c in ROW_CASES])
def test_four_row_stem(lib, case):
    from pretorched_x_b200 import engine, ops
    name, N, T, H, W, k, p, pooled = case
    K = 8 if name.startswith("slowfast") else 64
    _, a, conv, bn = make_stem(torch.device("cuda:0"), N, T, H, W, K, k, p, sum(map(ord, name)))
    got, ran4 = run_stem(lib, 4, conv, bn, a, pooled)
    two, ran2 = run_stem(lib, 2, conv, bn, a, pooled)
    assert (ran4, ran2) == (4, 2)
    assert torch.equal(got.data, two.data)                          # same accumulation order: bit-identical to G = 2
    ref = engine.conv_bn_act(conv, bn, a, relu=True, simt=True)
    if pooled:
        ref = ops.maxpool3d(ref, *POOL_FULL)
    assert (got.N, got.T, got.H, got.W, got.C) == (ref.N, ref.T, ref.H, ref.W, ref.C)
    assert rel(got.data[:, :K].float(), ref.data[:, :K].float()) <= TOL_F16


def test_four_row_stem_out_rows(lib):
    """out=: one clip written into its row range of a whole-batch buffer by the G = 4 instance (the rule's choice for a 7x7x7 stem)
    equals the whole-batch call."""
    from pretorched_x_b200 import engine, ops
    x, a, conv, bn = make_stem(torch.device("cuda:0"), 3, 5, 50, 96, 64, (7, 7, 7), (3, 3, 3), 11)
    lib.b2_debug_set_stem_rows(-1)
    whole = engine.conv_bn_act(conv, bn, a, relu=True, pool_w=True)
    rows = whole.data.shape[0] // 3
    buf = torch.full_like(whole.data, 7.0)
    engine.conv_bn_act(conv, bn, ops.from_ncdhw(x[1:2].to(a.data.device)), relu=True, pool_w=True, out=buf[rows:2 * rows])
    torch.cuda.synchronize()
    assert lib.b2_debug_last_stem_rows() == 4
    assert torch.equal(buf[rows:2 * rows], whole.data[rows:2 * rows])
    assert bool((buf[:rows] == 7.0).all()) and bool((buf[2 * rows:] == 7.0).all())


@pytest.mark.parametrize("force", [-1, 4])
def test_stems_that_keep_two_rows(lib, force):
    """kh = 13 leaves no room for G = 4's three ring stages and narrow (1, 7, 7) images run in pair mode: both keep G = 2 even when
    G = 4 is requested.  A wide 2-D stem (kt = 1, one tap per item) keeps G = 2 under the rule."""
    from pretorched_x_b200 import engine
    dev = torch.device("cuda:0")
    cases = [((1, 4, 40, 64, 64, (3, 13, 7), (1, 6, 3)), False), ((2, 4, 56, 56, 64, (1, 7, 7), (0, 3, 3)), False)]
    if force == -1:
        cases.append(((4, 1, 64, 224, 64, (1, 7, 7), (0, 3, 3)), True))
    for shape, pooled in cases:
        _, a, conv, bn = make_stem(dev, *shape, 3)
        lib.b2_debug_set_stem_rows(force)
        try:
            engine.conv_bn_act(conv, bn, a, relu=True, pool_w=pooled)
            torch.cuda.synchronize()
            assert lib.b2_debug_last_stem_rows() == 2, shape
        finally:
            lib.b2_debug_set_stem_rows(-1)
