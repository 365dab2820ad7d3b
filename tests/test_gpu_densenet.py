"""GPU (-m gpu): the DenseNets and TRN on densenet121.

1. b2_gemm_preact_f16 against fp64 under the kernel-matrix bound of tests/kernel_ref.py (the in-affine operand rounded to fp16
   once, as tests/kernel_ref.in_affine_acc models it), the kernel pinned (persistent GEMM, generator instance): the ragged input
   widths of the dense layers (C_L = 64 .. 2112, N = 128 and 192), M not a multiple of 128, positive shifts t1, the block
   matrix's columns >= C_L filled with NaN (never read from A) and the filter stored at a wider pitch with NaN past C_L (never
   read from B either: both tensor maps span C_L columns).
2. The growth-rate 3x3 convolutions (128 -> 32, 192 -> 48 at 56 / 28 / 14 / 7) into a sentinel-filled block matrix, on the
   64-wide tile (b2_conv_ndhwc_fprop_slice) and on the k-wide tile (b2_conv_ndhwc_fprop_slice_narrow), each pinned: within the fp64
   bound, every column outside the slice bit-for-bit unchanged, and the two tiles' outputs bitwise equal.
3. The transition pool (BatchNorm + ReLU + 2x2 average, odd extents included) and the head pool (affine + ReLU + global mean)
   against fp64.
4. Every dense block and transition of densenet121 / densenet161 against the fp64 oracle on the engine's fp16 input.
5. Both networks and TRN-MSTRN on densenet121 against the reference's fixtures, CUDA-graph replay bit-identical to the eager
   forward, a trainable last_linear on the frozen trunk against fp64, and the refusal of a final map other than 7x7.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200.graph import GraphedForward
from pretorched_x_b200.ops import Act
from oracle import densenet as OD
from oracle import functional as OF
from oracle.make_golden import sample_of
from tests import kernel_ref as KR
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
KID_PGEMM, KID_SLAB_SLICE, KID_POOL = 6, 13, 14   # csrc/b2_host.h
SENTINEL = -12345


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------
# 1. pre-activated GEMM
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_L,N", [(64, 128), (96, 128), (160, 128), (224, 128), (992, 128), (96, 192), (144, 192), (2112, 192)])
@pytest.mark.parametrize("M", [1000, 6272])
def test_preact_gemm(C_L, N, M):
    g = _gen(C_L + N + M)
    pitch = ops._round_up(C_L + 40, 8)
    blk = torch.full((M, pitch), float("nan"), dtype=torch.float16)
    blk[:, :C_L] = torch.randn(M, C_L, generator=g).half()
    w = (torch.randn(N, C_L, generator=g) * C_L ** -0.5).half()
    wpad = torch.full((N, C_L + 64), float("nan"), dtype=torch.float16)     # filter rows at a wider pitch, NaN past C_L
    wpad[:, :C_L] = w
    s1 = torch.rand(C_L, generator=g) + 0.5
    t1 = torch.rand(C_L, generator=g) * 0.5 + 0.05              # shifts > 0, as after BatchNorm
    kpad = ops._round_up(C_L, 64)
    s1p, t1p = torch.zeros(kpad), torch.zeros(kpad)
    s1p[:C_L], t1p[:C_L] = s1, t1
    s2, t2 = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    out = ops.gemm_preact(blk.to(dev), wpad.to(dev), s2.to(dev), t2.to(dev), s1p.to(dev), t1p.to(dev), M, N, C_L, relu=True)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    assert kid == KID_PGEMM and info[:3] == [128, 0, 1], (kid, info)
    acc, mag = KR.in_affine_acc(blk[:, :C_L], w, s1, t1, M)
    ref, A = KR.epilogue(acc, mag, s2, t2, relu=True)
    got = out[:, :N]
    assert KR.worst_ratio(got, ref, A, True) <= 1.0, KR.where_worst(got, ref, A, True)


# ---------------------------------------------------------------------------------------------
# 2. growth-rate 3x3 convolutions into the block matrix
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,K", [(128, 32), (192, 48)])
@pytest.mark.parametrize("H", [56, 28, 14, 7])
def test_growth_conv_into_block_slice(C, K, H):
    g = _gen(C + K + H)
    N = 4
    x = torch.rand(N, 1, H, H, C, generator=g).half()
    w = torch.randn(K, C, 3, 3, generator=g) * (9 * C) ** -0.5
    pc = ops.PackedConv(w.to(dev), None, None, (1, 1, 1), (0, 1, 1), in_pitch=C)
    M, c0, width = N * H * H, 96 + K, 96 + 3 * K
    ref, A = KR.conv_ref(x, pc.w.view(K, 9, C).cpu(), pc.scale.cpu(), pc.shift.cpu(), (1, 3, 3), (1, 1, 1), (0, 1, 1))
    outs = []
    for narrow in (False, True):
        blk = torch.full((M, width), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
        ops.conv_slice(Act(x.reshape(M, C).to(dev), N, 1, H, H, C), pc, blk[:, c0:c0 + K], relu=False, narrow=narrow)
        torch.cuda.synchronize()
        kid, info = _last_kernel()
        assert kid == KID_SLAB_SLICE and info[0] == (K if narrow else 64) and info[2] == int(narrow), (narrow, kid, info)
        b = blk.view(torch.int16)
        assert bool((b[:, :c0] == SENTINEL).all()) and bool((b[:, c0 + K:] == SENTINEL).all())
        got = blk[:, c0:c0 + K]
        assert KR.worst_ratio(got, ref, A, True) <= 1.0, KR.where_worst(got, ref, A, True)
        outs.append(got.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "the k-wide tile differs from the 64-wide tile"


# ---------------------------------------------------------------------------------------------
# 3. transition pool, head pool
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,C", [(56, 56, 256), (14, 14, 1056), (15, 9, 64), (7, 7, 1024)])
def test_transition_pool(H, W, C):
    g = _gen(H * W + C)
    N, ldx = 2, C + 16
    x = torch.randn(N * H * W, ldx, generator=g).half()
    s, t = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    Ho, Wo = H // 2, W // 2
    y = torch.full((N * Ho * Wo, C + 32), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
    ops.bn_relu_avgpool2(Act(x.to(dev)[:, :ldx], N, 1, H, W, C), s.to(dev), t.to(dev), y[:, 16:16 + C])
    torch.cuda.synchronize()
    assert _last_kernel() == (KID_POOL, [3, 0, 0, 0, 0])
    b = y.view(torch.int16)
    assert bool((b[:, :16] == SENTINEL).all()) and bool((b[:, 16 + C:] == SENTINEL).all())
    xd = x[:, :C].double().view(N, H, W, C).permute(0, 3, 1, 2)
    v = (xd * s.double().view(1, C, 1, 1) + t.double().view(1, C, 1, 1)).clamp_min(0.0)
    want = F.avg_pool2d(v, 2, 2).permute(0, 2, 3, 1).reshape(-1, C)
    mag = F.avg_pool2d((xd * s.double().view(1, C, 1, 1)).abs() + t.double().abs().view(1, C, 1, 1), 2, 2).permute(0, 2, 3, 1).reshape(-1, C)
    bnd = KR.U_F16 * want.abs() + 2.0 ** -20 * mag + KR.FLOOR
    err = (y[:, 16:16 + C].double().cpu() - want).abs()
    assert float((err / bnd).max()) <= 1.0


@pytest.mark.parametrize("S,C", [(49, 1024), (49, 2208), (9, 64)])
def test_head_pool(S, C):
    g = _gen(S + C)
    N = 3
    x = torch.randn(N * S, C, generator=g).half()
    s, t = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    y = ops.avgpool_global_affine(Act(x.to(dev), N, 1, 1, S, C), s.to(dev), t.to(dev))
    torch.cuda.synchronize()
    assert _last_kernel() == (KID_POOL, [4, 0, 0, 0, 0])
    xd = x.double().view(N, S, C)
    want = (xd * s.double() + t.double()).clamp_min(0.0).mean(1)
    mag = ((xd * s.double()).abs() + t.double().abs()).mean(1)
    bnd = KR.U_F16 * want.abs() + 2.0 ** -18 * mag + KR.FLOOR
    err = (y.double().cpu() - want).abs()
    assert float((err / bnd).max()) <= 1.0


# ---------------------------------------------------------------------------------------------
# 4. blocks and transitions against the fp64 oracle
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models():
    out = {}
    for arch in ("densenet121", "densenet161"):
        torch.manual_seed(0)
        m = P.__dict__[arch](pretrained=None)
        OF.randomize_bn_(m, 1)
        out[arch] = m.eval().to(dev)
    return out


@pytest.mark.parametrize("arch", ["densenet121", "densenet161"])
@pytest.mark.parametrize("b", [1, 2, 3, 4])
def test_block_and_transition_match_oracle(models, arch, b):
    m = models[arch]
    feats = m.features
    block = getattr(feats, "denseblock%d" % b)
    layers = list(block.children())
    C0 = layers[0].conv1.in_channels
    Cf = C0 + sum(l.conv2.out_channels for l in layers)
    H = 56 >> (b - 1)
    N = 2
    x = torch.rand((N, C0, H, H), generator=_gen(b)).half()
    blk = Act(torch.empty((N * H * H, Cf), dtype=torch.float16, device=dev), N, 1, H, H, Cf)
    blk.data[:, :C0] = x.permute(0, 2, 3, 1).reshape(-1, C0).to(dev)
    with torch.no_grad():
        for layer in layers:
            engine._dense_layer(layer, blk)
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    want = OD.block(x.double(), sd, "features.denseblock%d." % b)
    got = blk.data.double().cpu().view(N, H, H, Cf).permute(0, 3, 1, 2)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "denseblock%d: rel err %.3e" % (b, err)
    if b == 4:
        return
    tr = getattr(feats, "transition%d" % b)
    C2 = tr.conv.out_channels
    nxt = torch.full((N * (H // 2) ** 2, C2 + 64), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
    with torch.no_grad():
        engine._dense_transition(tr, blk, nxt[:, :C2])
    assert bool((nxt[:, C2:].view(torch.int16) == SENTINEL).all())
    want = OD.transition(got, sd, "features.transition%d." % b)
    got = nxt[:, :C2].double().cpu().view(N, H // 2, H // 2, C2).permute(0, 3, 1, 2)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "transition%d: rel err %.3e" % (b, err)


# ---------------------------------------------------------------------------------------------
# 5. models against the reference fixtures
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["densenet121", "densenet161"])
def test_model_matches_reference_fixture(arch):
    fx = _load("%s_b2_224.pt" % arch)
    m = OD.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
        whole = m(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == tuple(fx["features"]["shape"]) and feats.dtype == torch.float32
    s, step = sample_of(feats.cpu())
    assert step == fx["features"]["step"]
    err = (s.double() - fx["features"]["sample"].double()).abs().max().item() / fx["features"]["absmax"]
    assert err <= 1e-2, "features: rel err %.3e" % err
    want = fx["logits"].double()
    for got in (logits, whole):
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= 5e-3, "logits: rel err %.3e" % err
        assert torch.equal(got.argmax(1).cpu(), want.argmax(1))
    g = GraphedForward(m, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_densenet121_MSTRN.pt")
    m = OD.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        np.random.seed(fx["seeds"]["tuples"])
        feats = m.features(x)
        logits = m.logits(feats)
    for got, want, tol in ((feats, fx["features"], 1e-2), (logits, fx["logits"], 5e-3)):
        want = want.double()
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= tol, "rel err %.3e" % err
    assert int(logits.argmax()) == int(fx["logits"].argmax())
    np.random.seed(fx["seeds"]["tuples"])
    with torch.no_grad():
        m(x)
        eager = m(x)
    np.random.seed(fx["seeds"]["tuples"])
    g = GraphedForward(m, x, warmup=1)
    assert torch.equal(g(x).clone(), eager), "graph replay differs from the eager forward"


@pytest.mark.parametrize("arch", ["densenet121", "densenet161"])
def test_trainable_last_linear_on_frozen_trunk(models, arch):
    model = models[arch]
    C = model.last_linear.in_features
    head = torch.nn.Linear(C, 7).to(dev)
    old = model.last_linear
    model.last_linear = head
    try:
        x = torch.rand((2, 3, 224, 224), generator=_gen(4)).to(dev)
        model(x).square().sum().backward()
        with torch.no_grad():
            pooled = F.relu(model.features(x)).double().mean((2, 3))
        out = pooled @ head.weight.double().t() + head.bias.double()
        want = 2.0 * out.t() @ pooled
        err = (head.weight.grad.double() - want).abs().max().item() / want.abs().max().item()
        assert err <= 1e-2, "dW rel err %.3e" % err
        assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith("last_linear"))
    finally:
        model.last_linear = old


@pytest.mark.parametrize("arch", ["densenet121", "densenet161"])
def test_final_map_other_than_7x7_is_refused(models, arch):
    x = torch.rand((1, 3, 256, 256), device=dev)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="7x7"):
        models[arch](x)
