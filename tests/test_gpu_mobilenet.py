"""GPU (-m gpu): MobileNetV2 on the engine -- the depthwise 3x3 kernel against an fp64 grouped convolution, the whole network
and a TRN on its features against the reference's fixtures (tests/golden, kinds "mobilenetv2" / "trn_mobilenetv2"), CUDA-graph
replay, and a trainable head on the frozen features.

Tolerances (DESIGN.md section 6; relative to max |reference| of the tensor): depthwise kernel 2e-3; per-stage samples 1e-2,
logits 5e-3, equal arg-max."""
import ctypes
import glob
import os

import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200 import functions as Fn
from pretorched_x_b200.ops import Act
from oracle import functional as OF
from oracle import mobilenet as OM
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIX = sorted(glob.glob(os.path.join(GOLDEN, "mobilenetv2_*.pt")))
TRN_FIX = os.path.join(GOLDEN, "trn_mobilenetv2_TRN.pt")


def _load(path):
    return torch.load(path, weights_only=False)


# ---------------------------------------------------------------------------------------------
# 1. depthwise kernel
# ---------------------------------------------------------------------------------------------
DW_CASES = [
    # B, C, H, W, stride, ld, clamp_in, relu6
    # every depthwise layer of MobileNetV2 at 224 x 224
    (2, 32, 112, 112, 1, 32, True, True),
    (2, 96, 112, 112, 2, 96, True, True),
    (2, 144, 56, 56, 1, 144, True, True),
    (2, 144, 56, 56, 2, 144, True, True),
    (2, 192, 28, 28, 1, 192, True, True),
    (2, 192, 28, 28, 2, 192, True, True),
    (2, 384, 14, 14, 1, 384, True, True),
    (2, 576, 14, 14, 1, 576, True, True),
    (2, 576, 14, 14, 2, 576, True, True),
    (2, 960, 7, 7, 1, 960, True, True),
    # odd sizes, 1 x 1 and 1 x W maps, C = 8, C not a multiple of 64, ld > C, several images, clamp and activation off
    (3, 24, 13, 11, 2, 24, True, True),
    (3, 24, 13, 11, 1, 24, False, True),
    (2, 64, 1, 1, 1, 64, True, True),
    (2, 64, 1, 1, 2, 64, True, True),
    (2, 40, 1, 9, 2, 40, True, True),
    (4, 8, 5, 7, 1, 8, True, True),
    (2, 72, 9, 10, 2, 72, False, False),
    (3, 24, 6, 5, 1, 40, True, True),
    (2, 48, 3, 2, 2, 64, False, True),
]


def _dw_case(B, C, H, W, stride, ld, clamp_in, relu6, seed=0):
    gen = torch.Generator().manual_seed(seed + C * 7 + H)
    x = ((torch.randn((B, C, H, W), generator=gen) * 3).relu()).half()           # ~2 % of the inputs above 6
    w = torch.randn((C, 1, 3, 3), generator=gen) * 0.3
    scale = torch.rand(C, generator=gen) + 0.5
    shift = torch.randn(C, generator=gen) * 0.5
    data = torch.zeros((B * H * W, ld), dtype=torch.float16)
    data[:, :C] = x.permute(0, 2, 3, 1).reshape(-1, C)
    a = Act(data.to(dev), B, 1, H, W, C)
    xin = x.double().clamp(max=6) if clamp_in else x.double()
    ref = F.conv2d(xin, w.double(), stride=stride, padding=1, groups=C) * scale.double()[:, None, None] + shift.double()[:, None, None]
    if relu6:
        ref = ref.clamp(0, 6)
    w9 = w.reshape(C, 9).t().contiguous().to(dev)
    return a, w9, scale.to(dev), shift.to(dev), ref


@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "B%dC%dH%dW%ds%dld%d%s%s" % (c[:6] + ("_clamp" if c[6] else "", "_relu6" if c[7] else "")))
def test_depthwise_kernel_matches_fp64_grouped_conv(case):
    B, C, H, W, stride, ld, clamp_in, relu6 = case
    a, w9, scale, shift, ref = _dw_case(*case)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.full((B * Ho * Wo, ld), 1.0, dtype=torch.float16, device=dev)     # padding channels must be overwritten with 0
    y = ops.dwconv3x3(a, w9, scale, shift, stride, clamp_in=clamp_in, relu6=relu6, out=out)
    y2 = ops.dwconv3x3(a, w9, scale, shift, stride, clamp_in=clamp_in, relu6=relu6)
    torch.cuda.synchronize()
    assert (y.N, y.T, y.H, y.W, y.C, y.ld) == (B, 1, Ho, Wo, C, ld)
    assert torch.equal(y.data, y2.data), "depthwise kernel is not bitwise repeatable"
    got = y.data.cpu()
    assert torch.equal(got[:, C:], torch.zeros_like(got[:, C:]))
    got = got[:, :C].double().reshape(B, Ho, Wo, C).permute(0, 3, 1, 2)
    err = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
    assert err <= 2e-3, err
    if relu6:
        assert got.max().item() <= 6.0 and got.min().item() >= 0.0


def test_relu6_inplace():
    gen = torch.Generator().manual_seed(5)
    data = torch.zeros((37, 24), dtype=torch.float16)
    data[:, :20] = (torch.randn((37, 20), generator=gen) * 8).half()
    a = Act(data.to(dev), 1, 1, 37, 1, 20)
    ops.relu6_(a)
    assert torch.equal(a.data.cpu(), data.clamp(0, 6))


# ---------------------------------------------------------------------------------------------
# 2. the stem's 3-channel 3x3 stride-2 convolution
# ---------------------------------------------------------------------------------------------
def test_stem_convolution_runs_on_the_slab_kernel():
    """Pitch-8 input, 32 outputs, 3x3 stride 2 at B = 2, 224 x 224 (M = 25088): the slab kernel takes it (it records neither a
    temporal-stack nor a GEMM-family launch); at 96 x 64 (M = 3072) the dense small-M kernel does."""
    lib = _lib.load()
    for fn in (lib.b2_debug_last_conv_path, lib.b2_debug_last_gemm_path):
        fn.restype = ctypes.c_int
    lib.b2_debug_slab_plan.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.mobilenetv2(num_classes=10, pretrained=None), 1).eval().to(dev)
    stem = m.features[0]
    for (H, W), path in (((224, 224), (0, 0)), ((96, 64), (0, 1))):
        x = torch.randn((2, 3, H, W), generator=torch.Generator().manual_seed(1))
        a = ops.from_ncdhw(x.to(dev), pitch=8)
        args = _lib.ConvArgs()
        args.N, args.T, args.H, args.W, args.C, args.K, args.ldy = 2, 1, H, W, 8, 32, 32
        args.kt, args.kh, args.kw, args.st, args.sh, args.sw, args.pt, args.ph, args.pw = 1, 3, 3, 1, 2, 2, 0, 1, 1
        plan = (ctypes.c_int * 10)()
        lib.b2_debug_slab_plan(ctypes.byref(args), plan)
        with torch.no_grad():
            y = engine._conv_bn_relu6_body(stem, a)
        torch.cuda.synchronize()
        assert (lib.b2_debug_last_conv_path(), lib.b2_debug_last_gemm_path()) == path, (H, W)
        assert plan[0] == 1
        sd = {k: v.cpu() for k, v in m.state_dict().items()}
        want = OM.conv_bn(x.half().float(), sd, "features.0", 2)
        got = ops.to_ncdhw(y).squeeze(2).cpu()
        assert (got - want).abs().max().item() <= 5e-3 * want.abs().max().item()


# ---------------------------------------------------------------------------------------------
# 3. whole network against the reference's fixtures
# ---------------------------------------------------------------------------------------------
def staged(m, x):
    """The engine walk of ``run_mobilenet_features`` with every block output kept, then the head."""
    outs = {}
    with torch.no_grad():
        a = ops.from_ncdhw(x, pitch=8)
        mods = list(m.features)
        for i, blk in enumerate(mods):
            if hasattr(blk, "use_res_connect"):
                a = Fn.frozen(lambda t, o: engine._inverted_residual_body(blk, t, o), a)
            else:
                a = Fn.frozen(lambda t, o: engine._conv_bn_relu6_body(blk, t, i == len(mods) - 1), a)
            outs["features.%d" % i] = a
        logits = m.logits(a)
    return outs, logits


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-3] for p in FIX])
def test_staged_forward_matches_reference_golden(path):
    fx = _load(path)
    m = OM.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    outs, logits = staged(m, x)
    for name, ref in fx["stages"].items():
        if name == "logits":
            continue
        t = ops.to_ncdhw(outs[name]).squeeze(2)
        assert tuple(t.shape) == tuple(ref["shape"]), name
        t = t.reshape(-1)[::ref["step"]][:ref["sample"].numel()].cpu().double()
        err = (t - ref["sample"].double()).abs().max().item() / max(ref["absmax"], 1e-12)
        print("%-14s %.2e" % (name, err))
        assert err <= 1e-2, (name, err)
    err = (logits.cpu().double() - fx["logits"].double()).abs().max().item() / fx["logits"].abs().max().item()
    print("%-14s %.2e" % ("logits", err))
    assert err <= 5e-3, err
    assert torch.equal(logits.argmax(1).cpu(), fx["logits"].argmax(1))
    with torch.no_grad():
        assert torch.equal(m(x), logits)                     # the public forward is the staged walk
        feat = m.features(x)
    assert feat.dtype == torch.float32 and tuple(feat.shape) == tuple(fx["stages"]["features.18"]["shape"])


def test_graph_replay_is_bit_identical():
    from pretorched_x_b200.graph import GraphedForward
    fx = _load([p for p in FIX if p.endswith("_224.pt")][0])
    m = OM.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        eager = m(x).clone()
    g = GraphedForward(m, x)
    x2 = OF.seeded_input(fx["input_shape"], 9).to(dev)
    with torch.no_grad():
        eager2 = m(x2).clone()
    assert torch.equal(g(x2).clone(), eager2)
    assert torch.equal(g(x).clone(), eager)


def test_trn_on_mobilenetv2_matches_reference_golden():
    fx = _load(TRN_FIX)
    m = OM.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
    for got, ref in ((feats, fx["features"]), (logits, fx["logits"])):
        err = (got.cpu().double() - ref.double()).abs().max().item() / ref.abs().max().item()
        assert err <= 5e-3, err
    assert torch.equal(logits.argmax(-1).cpu(), fx["logits"].argmax(-1))


# ---------------------------------------------------------------------------------------------
# 4. a trainable head on the frozen features
# ---------------------------------------------------------------------------------------------
def test_trainable_head_on_frozen_features():
    fx = _load([p for p in FIX if p.endswith("96x64.pt")][0])
    m = OM.build_package_model(P, fx).to(dev)
    for p in m.features.parameters():
        p.requires_grad_(False)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    loss = F.cross_entropy(m(x), torch.tensor([1, 2], device=dev))
    loss.backward()
    assert m.last_linear.weight.grad is not None and m.last_linear.weight.grad.abs().sum().item() > 0
    assert m.last_linear.bias.grad is not None
    assert all(p.grad is None for p in m.features.parameters())
    # reference: the same head on the engine's pooled features through torch autograd
    with torch.no_grad():
        pooled = ops.avgpool_global(m.features_act(x))[:, :1280].float()
    w = m.last_linear.weight.detach().clone().requires_grad_(True)
    F.cross_entropy(F.linear(pooled, w, m.last_linear.bias.detach()), torch.tensor([1, 2], device=dev)).backward()
    err = (m.last_linear.weight.grad - w.grad).abs().max().item() / w.grad.abs().max().item()
    assert err <= 1e-2, err
    # a swapped head receives the pooled fp32 features
    m.last_linear = torch.nn.Identity()
    with torch.no_grad():
        feats = m(x)
    assert feats.dtype == torch.float32 and tuple(feats.shape) == (2, 1280)
    # a frozen model receives no gradient at all
    frozen = OM.build_package_model(P, fx).to(dev)
    for p in frozen.parameters():
        p.requires_grad_(False)
    out = frozen(x)
    assert not out.requires_grad
