"""GPU (-m gpu): the stem convolution kernel (b2_stemconv.cuh: register accumulators, operand ring, double-buffered fp16 staging
tiles) on shapes the model-level tests do not reach, against the CUDA-core cross-check (simt=True) followed by a stand-alone
max-pool.  Tolerance: 2e-3 of max|reference| (fp32 accumulation, one fp16 rounding of the result)."""
import pytest
import torch
import torch.nn as nn

from oracle import functional as OF

pytestmark = pytest.mark.gpu

TOL_F16 = 2e-3
POOL_TH = ((3, 3, 1), (2, 2, 1), (1, 1, 0))          # what remains of MaxPool3d(3, 2, 1) once the stem pooled along W
POOL_FULL = ((3, 3, 3), (2, 2, 2), (1, 1, 1))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    from pretorched_x_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def make_stem(dev, N, T, H, W, K, k, p, seed):
    from pretorched_x_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, T, H, W, generator=g).half().float()
    conv = nn.Conv3d(3, K, k, stride=(1, 2, 2), padding=p, bias=False)
    with torch.no_grad():
        conv.weight.copy_((torch.randn(conv.weight.shape, generator=g) / (3 * k[0] * k[1] * k[2]) ** 0.5).half().float())
    bn = OF.randomize_bn_(nn.BatchNorm3d(K), seed).eval()
    return x, ops.from_ncdhw(x.to(dev)), conv.to(dev), bn.to(dev)


def rel(got, ref):
    return (got.double() - ref.double()).abs().max().item() / max(ref.abs().max().item(), 1e-12)


def check(dev, N, T, H, W, K, k, p, pooled, seed):
    from pretorched_x_b200 import engine, ops
    _, a, conv, bn = make_stem(dev, N, T, H, W, K, k, p, seed)
    if pooled:
        run = lambda: ops.maxpool3d(engine.conv_bn_act(conv, bn, a, relu=True, pool_w=True), *POOL_TH)
        ref = ops.maxpool3d(engine.conv_bn_act(conv, bn, a, relu=True, simt=True), *POOL_FULL)
    else:
        run = lambda: engine.conv_bn_act(conv, bn, a, relu=True)
        ref = engine.conv_bn_act(conv, bn, a, relu=True, simt=True)
    got, again = run(), run()
    assert (got.N, got.T, got.H, got.W, got.C) == (ref.N, ref.T, ref.H, ref.W, ref.C)
    assert torch.equal(got.data, again.data)                       # deterministic: no accumulation-order freedom
    assert rel(got.data[:, :K].float(), ref.data[:, :K].float()) <= TOL_F16
    if got.ld > K:                                                 # channel padding stays exactly zero
        assert float(got.data[:, K:].abs().max()) == 0.0


STEM_CASES = [
    # name, N, T, H, W, K, kernel, padding, pooled
    # 2 x 16 x 56 items: every CTA wraps the operand ring and both staging tiles many times
    ("many_items_2x16x224", 2, 16, 224, 224, 64, (7, 7, 7), (3, 3, 3), True),
    ("ho_odd_15_rows", 1, 4, 30, 64, 64, (7, 7, 7), (3, 3, 3), True),                 # the last item has one valid output row
    ("t_below_kt", 2, 3, 20, 40, 64, (7, 7, 7), (3, 3, 3), True),                     # temporal taps outside the clip everywhere
    ("three_column_tiles_unpooled", 1, 2, 14, 500, 64, (7, 7, 7), (3, 3, 3), False),   # Wo = 250: 3 column tiles, the last ragged
    ("bn128_256_channels", 1, 3, 26, 96, 256, (7, 7, 7), (3, 3, 3), True),            # two 128-wide N tiles, G = 1
    ("bn128_unpooled_200_channels", 2, 2, 17, 252, 200, (3, 7, 7), (1, 3, 3), False),  # ragged second N tile, 2 column tiles
    ("slowfast_5x7x7_to_8", 2, 8, 32, 64, 8, (5, 7, 7), (2, 3, 3), True),             # SlowFast fast-path stem
    # tall filters: a single operand ring slot, each temporal tap's slot released before the next tap is loaded
    ("one_stage_bn128_kh9", 2, 4, 40, 64, 128, (3, 9, 7), (1, 4, 3), False),
    ("one_stage_bn64_kh13", 3, 4, 40, 64, 64, (3, 13, 7), (1, 6, 3), True),
]


@pytest.mark.parametrize("case", STEM_CASES, ids=[c[0] for c in STEM_CASES])
def test_stem_matches_crosscheck(dev, case):
    check(dev, *case[1:], seed=sum(map(ord, case[0])))


def test_stem_chunked_out_rows(dev):
    """out=: one clip's pooled stem written into its row range of a whole-batch buffer equals the whole-batch call, and the
    rows around it are untouched."""
    from pretorched_x_b200 import engine, ops
    x, a, conv, bn = make_stem(dev, 3, 5, 48, 96, 64, (7, 7, 7), (3, 3, 3), 5)
    whole = engine.conv_bn_act(conv, bn, a, relu=True, pool_w=True)
    rows = whole.data.shape[0] // 3
    buf = torch.full_like(whole.data, 7.0)
    part = engine.conv_bn_act(conv, bn, ops.from_ncdhw(x[1:2].to(dev)), relu=True, pool_w=True, out=buf[rows:2 * rows])
    assert part.data.data_ptr() == buf[rows:].data_ptr()
    assert torch.equal(buf[rows:2 * rows], whole.data[rows:2 * rows])
    assert bool((buf[:rows] == 7.0).all()) and bool((buf[2 * rows:] == 7.0).all())
    ref = ops.maxpool3d(engine.conv_bn_act(conv, bn, a, relu=True, simt=True), *POOL_FULL)
    got = ops.maxpool3d(whole, *POOL_TH)
    assert rel(got.data.float(), ref.data.float()) <= TOL_F16


def test_stem_refuses_temporal_padding_not_below_kt(dev):
    """pt >= kt leaves output frames without any input frame; the stem kernel refuses such a call instead of running it."""
    from pretorched_x_b200 import engine
    _, a, conv, bn = make_stem(dev, 1, 3, 20, 40, 64, (1, 7, 7), (1, 3, 3), 3)
    with pytest.raises(RuntimeError, match="temporal padding"):
        engine.conv_bn_act(conv, bn, a, relu=True)
    torch.cuda.synchronize()
