"""GPU (-m gpu): the group-aware convolution kernel (csrc/b2_groupconv.cuh, b2_conv_grouped_ndhwc_fprop) -- its filter packing
against ``ops.dense_from_grouped``, the kernel against fp64 under the kernel matrix's elementwise bound (tests/kernel_ref.py),
the grouped route against the dense-packed route, and ResNeXt-3D end to end on it (golden forward, packed-weight memory, CUDA
graph replay)."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import functional as OF
import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200.graph import GraphedForward
from tests.kernel_ref import bound, where_worst, worst_ratio

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "resnext3d50_b1_t8_64.pt")
KID_GROUPCONV = 10
# (channels per group, groups): two 64-channel slices each, except the last (four slices, ResNeXt's own layer2 width)
WIDTHS = [(4, 32), (8, 16), (16, 8), (32, 4), (8, 32)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


def f16_values(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).half().float()


def last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), tuple(info)


def make_case(dev, cg, groups, kt, stride, N, T, H, W, seed):
    C = cg * groups
    w = f16_values((C, cg, kt, 3, 3), seed, 0.1)                        # fp16-representable: packing rounds nothing
    x = f16_values((N, T, H, W, C), seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    scale = torch.rand(C, generator=g) + 0.5
    shift = torch.randn(C, generator=g)
    s, p = (stride if kt == 3 else 1, stride, stride), (kt // 2, 1, 1)
    pc = ops.PackedGroupedConv(w.to(dev), groups, stride=s, padding=p)
    pc.scale, pc.shift = scale.to(dev), shift.to(dev)
    a = ops.Act(x.reshape(-1, C).half().to(dev), N, T, H, W, C)
    return dict(w=w, x=x, scale=scale, shift=shift, s=s, p=p, pc=pc, a=a, groups=groups, C=C)


def grouped_ref(c, residual=None, relu=False):
    """fp64 reference and magnitude sum of the kernel's own operands (kernel_ref.conv_ref with ``groups``)."""
    xt = c["x"].double().permute(0, 4, 1, 2, 3)
    wt = c["w"].double()
    acc = F.conv3d(xt, wt, stride=c["s"], padding=c["p"], groups=c["groups"]).permute(0, 2, 3, 4, 1).reshape(-1, c["C"])
    mag = F.conv3d(xt.abs(), wt.abs(), stride=c["s"], padding=c["p"], groups=c["groups"]).permute(0, 2, 3, 4, 1).reshape(-1, c["C"])
    ref = acc * c["scale"].double() + c["shift"].double()
    A = mag * c["scale"].double().abs() + c["shift"].double().abs()
    if residual is not None:
        ref, A = ref + residual.double(), A + residual.double().abs()
    return (ref.clamp_min(0.0) if relu else ref), A


def assert_within(name, got, ref, A):
    r = worst_ratio(got, ref, A, True)
    assert r <= 1.0, "%s: err/bound %.3f at %s" % (name, r, where_worst(got, ref, A, True))


@pytest.mark.parametrize("kt", [1, 3])
@pytest.mark.parametrize("cg,groups", WIDTHS)
def test_packed_filter_is_the_diagonal_chunks_of_the_dense_filter(dev, cg, groups, kt):
    C = cg * groups
    G = 32 if cg == 32 else 16
    w = f16_values((C, cg, kt, 3, 3), 7 * cg + kt, 0.1)
    pc = ops.PackedGroupedConv(w.to(dev), groups, stride=(1, 1, 1), padding=(kt // 2, 1, 1))
    taps = kt * 9
    assert pc.w.numel() == C * G * taps
    got = pc.w.cpu().reshape(C // 64, taps, G, 4, 16)
    dense = ops.dense_from_grouped(w, groups).reshape(C, C, taps).half()            # [K][C][tap]
    r, j, kk = torch.meshgrid(torch.arange(G), torch.arange(4), torch.arange(16), indexing="ij")
    o_local = 16 * j + r if G == 16 else 32 * (j // 2) + r
    for sl in range(C // 64):
        want = dense[64 * sl + o_local, 64 * sl + 16 * j + kk]                      # [G][4][16][tap]
        assert torch.equal(got[sl], want.permute(3, 0, 1, 2)), sl
        off_group = ((64 * sl + o_local) // cg) != ((64 * sl + 16 * j + kk) // cg)
        assert bool((got[sl][:, off_group] == 0).all())                             # exact zeros off the group blocks
    assert int((got != 0).sum()) == int((dense != 0).sum())                         # every filter coefficient is in a chunk


def test_grouped_entry_refuses_extras_and_shapes_outside_the_contract(dev):
    lib = _lib.load()
    c = make_case(dev, 4, 32, 3, 1, 1, 2, 6, 6, 11)
    y = torch.empty((2 * 36, 128), dtype=torch.float16, device=dev)

    def call(groups=32, **over):
        args = _lib.ConvArgs()
        args.x, args.w, args.scale, args.shift, args.y = (ctypes.c_void_p(t.data_ptr()) for t in
                                                          (c["a"].data, c["pc"].w, c["pc"].scale, c["pc"].shift, y))
        args.N, args.T, args.H, args.W, args.C, args.K, args.ldy = 1, 2, 6, 6, 128, 128, 128
        args.kt = args.kh = args.kw = 3
        args.st = args.sh = args.sw = 1
        args.pt = args.ph = args.pw = 1
        for k, v in over.items():
            setattr(args, k, v)
        return lib.b2_conv_grouped_ndhwc_fprop(ctypes.byref(args), groups, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

    assert call() == 0
    assert call(mode=1) == -1
    assert call(out_f32=1) == -1
    assert call(upsample=1) == -1
    assert call(in_scale=ctypes.c_void_p(c["pc"].scale.data_ptr())) == -1
    assert call(mask=ctypes.c_void_p(y.data_ptr()), ldm=128) == -1
    assert call(aff_ld=128) == -1
    assert call(groups=64) == -3            # 2 channels per group
    assert call(K=64, ldy=64) == -3         # C != K
    assert call(pw=0) == -3
    torch.cuda.synchronize()


CASES = [(cg, groups, kt, stride) for cg, groups in WIDTHS[:4] for kt in (1, 3) for stride in (1, 2)]


@pytest.mark.parametrize("cg,groups,kt,stride", CASES)
def test_kernel_against_fp64(dev, cg, groups, kt, stride):
    """Every width, stride 1 and 2, 3x3x3 and 1x3x3; 14 x 14 planes (224 padded-row positions: not a multiple of the 128-row tile),
    two clips, ReLU alternating."""
    relu = bool((cg // 4 + kt + stride) & 1)
    c = make_case(dev, cg, groups, kt, stride, 2, 3, 14, 14, 100 + cg + 3 * kt + stride)
    out = ops.conv(c["a"], c["pc"], relu=relu)
    kid, info = last_kernel()
    assert kid == KID_GROUPCONV and info[0] == (32 if cg == 32 else 16), (kid, info)
    ref, A = grouped_ref(c, relu=relu)
    assert out.data.shape == ref.shape
    assert_within("gconv cg%d kt%d s%d" % (cg, kt, stride), out.data, ref, A)


@pytest.mark.parametrize("name,cg,groups,kt,stride,N,T,H,W", [
    ("t1_plane", 16, 8, 3, 1, 2, 1, 10, 10),          # T = 1: the temporal taps that see only padding are skipped
    ("t1_strided", 32, 4, 3, 2, 1, 1, 9, 9),          # odd extent, stride 2, T = 1
    ("layer1_plane", 4, 32, 3, 1, 1, 3, 56, 56),      # several position tiles per plane, several M tiles per item
    ("small_planes", 8, 32, 3, 1, 2, 8, 7, 7),        # planes below one tile (several planes per item), four slices
    ("wide_rows", 8, 16, 1, 1, 1, 2, 6, 300),         # rows longer than a TMA box: W chunks
])
def test_kernel_shapes_against_fp64(dev, name, cg, groups, kt, stride, N, T, H, W):
    c = make_case(dev, cg, groups, kt, stride, N, T, H, W, 300 + H + W)
    out = ops.conv(c["a"], c["pc"], relu=True)
    assert last_kernel()[0] == KID_GROUPCONV
    ref, A = grouped_ref(c, relu=True)
    assert_within(name, out.data, ref, A)


def test_residual_and_out_row_range(dev):
    c = make_case(dev, 8, 16, 3, 2, 2, 4, 12, 12, 500)
    M = 2 * 2 * 6 * 6
    res = f16_values((M, 128), 501)
    ract = ops.Act(res.half().to(dev), 2, 2, 6, 6, 128)
    big = torch.full((M + 64, 128), 7.0, dtype=torch.float16, device=dev)
    out = ops.conv(c["a"], c["pc"], residual=ract, relu=True, out=big[32:32 + M])
    assert out.data.data_ptr() == big[32:].data_ptr()
    ref, A = grouped_ref(c, residual=res, relu=True)
    assert_within("gconv residual out=", big[32:32 + M], ref, A)
    assert bool((big[:32] == 7.0).all()) and bool((big[32 + M:] == 7.0).all())     # rows outside the range untouched
    again = torch.empty((M, 128), dtype=torch.float16, device=dev)
    ops.conv(c["a"], c["pc"], residual=ract, relu=True, out=again)
    assert torch.equal(again, big[32:32 + M])                                       # fixed summation order: bit-identical reruns


@pytest.mark.parametrize("cg,groups,kt,stride", [(4, 32, 3, 1), (8, 16, 3, 2), (16, 8, 1, 1), (32, 4, 3, 2)])
def test_grouped_route_matches_dense_route(dev, cg, groups, kt, stride):
    """Both routes round the same fp32 sum once to fp16; the sums differ in summation order (and the dense one adds exact zeros).
    Bound used: twice the kernel matrix's elementwise bound, i.e. each route within it of the fp64 value."""
    c = make_case(dev, cg, groups, kt, stride, 2, 3, 14, 14, 700 + cg)
    dense = ops.PackedConv(ops.dense_from_grouped(c["w"], groups).to(dev), stride=c["s"], padding=c["p"])
    dense.scale, dense.shift = c["pc"].scale, c["pc"].shift
    yd = ops.conv(c["a"], dense, relu=True)
    assert last_kernel()[0] != KID_GROUPCONV
    yg = ops.conv(c["a"], c["pc"], relu=True)
    ref, A = grouped_ref(c, relu=True)
    excess = (yg.data.double().cpu() - yd.data.double().cpu()).abs() - 2.0 * bound(ref, A, True)
    assert float(excess.max()) <= 0.0


def conv2_packs(model):
    return [blk.conv2.__dict__["_b2_cache"]["pc"][1] for ln in ("layer1", "layer2", "layer3", "layer4") for blk in getattr(model, ln)]


@pytest.mark.timeout(240, method="thread")
def test_resnext3d50_golden_on_the_grouped_kernel(dev):
    fx = torch.load(GOLDEN, weights_only=False)
    torch.manual_seed(fx["seeds"]["init"])
    m = getattr(P, fx["arch"])(**fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    m = m.eval().to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        logits = m(x)
    packs = conv2_packs(m)
    assert len(packs) == 16 and all(type(pc) is ops.PackedGroupedConv for pc in packs)
    err = ((logits.cpu().double() - fx["logits"].double()).abs() / fx["logits"].abs().max().item()).max().item()
    assert err <= 5e-3, err
    assert torch.equal(logits.argmax(1).cpu(), fx["logits"].argmax(1))
    # the CUDA-core cross-check reads the dense layout: it packs its own copy and leaves the grouped pack in place
    blk = m.layer1[0]
    a = engine.run_stem(m, x)
    with torch.no_grad():
        h = engine.conv_bn_act(blk.conv1, blk.bn1, a, relu=True)
        fast = engine.conv_bn_act(blk.conv2, blk.bn2, h, relu=True)
        slow = engine.conv_bn_act(blk.conv2, blk.bn2, h, relu=True, simt=True)
    assert type(blk.conv2.__dict__["_b2_cache"]["pc"][1]) is ops.PackedGroupedConv
    scale = float(slow.data.abs().max())
    assert float((fast.data.float() - slow.data.float()).abs().max()) <= 4e-3 * scale


@pytest.mark.timeout(240, method="thread")
def test_resnext3d101_packed_conv2_filters_fit_in_32_mb(dev):
    torch.manual_seed(0)
    m = P.resnext3d101(num_classes=10).eval().to(dev)
    with torch.no_grad():
        m(OF.seeded_input((1, 3, 8, 64, 64), 3).to(dev))
    packs = conv2_packs(m)
    assert len(packs) == 33 and all(type(pc) is ops.PackedGroupedConv for pc in packs)
    nbytes = sum(pc.w.numel() * pc.w.element_size() for pc in packs)
    dense_bytes = sum(2 * pc.K * pc.K * 27 for pc in packs)
    assert nbytes <= 32 << 20 and dense_bytes >= 400 << 20, (nbytes, dense_bytes)     # ~17 MB against ~0.5 GB block-diagonal dense
    m.invalidate()
    assert all("_b2_cache" not in blk.conv2.__dict__ for blk in m.layer3)


@pytest.mark.timeout(240, method="thread")
def test_graphed_forward_replays_bit_identically(dev):
    torch.manual_seed(1)
    m = P.resnext3d50(num_classes=10)
    OF.randomize_bn_(m, 2)
    m = m.eval().to(dev)
    x = OF.seeded_input((2, 3, 8, 64, 64), 4).to(dev)
    with torch.no_grad():
        eager = m(x).clone()
    g = GraphedForward(m, x)
    assert torch.equal(g(x), eager)
    assert torch.equal(g(x), eager)
