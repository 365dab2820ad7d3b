"""VGG and AlexNet on the H100 (-m gpu):

1. ``ops_vgg.space_to_depth4`` bit for bit against the rearrangement built with torch, and AlexNet's conv1 through it against the
   per-element fp64 bound of the 11x11 stride-4 convolution (tests/kernel_ref.py);
2. ``ops_vgg.gemm_splitk`` against the per-element fp64 bound at the classifier shapes and at ragged M / N, fp16 and fp32 output,
   with and without ReLU, with the kernel and splits pinned, bitwise repeatability and every refusal;
3. the nine models and TRN against the reference fixtures;
4. tests/vgg_audit.audit over every forward at 256 images (TRN-MSTRN: 16 videos x 8 segments), a CUDA-graph replay bitwise equal to
   the audited output, and the launches per forward;
5. the trainable ``last_linear``'s gradients against fp64.
"""
import ctypes
import functools
import os
import time

import numpy as np
import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, ops, ops_vgg
from pretorched_x_b200.graph import GraphedForward
from oracle import functional as OF
from tests import kernel_ref as KR
from tests.conftest import has_h100
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report
from tests.test_vgg_cpu import trn_as_reference
from tests.vgg_audit import audit, check_gemm_splitk, s2d_ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)
ARCHS = ("vgg11", "vgg11_bn", "vgg13", "vgg13_bn", "vgg16", "vgg16_bn", "vgg19", "vgg19_bn", "alexnet")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 8)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _sms():
    return torch.cuda.get_device_properties(dev).multi_processor_count


# ---------------------------------------------------------------------------------------------
# 1. space-to-depth
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W", [(3, 224, 224), (2, 227, 227), (2, 199, 241)])
def test_space_to_depth4_bitwise(N, H, W):
    x = torch.randn((N, 3, H, W), generator=torch.Generator().manual_seed(H + W))
    a = ops_vgg.space_to_depth4(x.to(dev))
    torch.cuda.synchronize()
    want = s2d_ref(x)
    assert (a.N, a.H, a.W, a.C, a.ld) == (N, ops_vgg.s2d_extent(H, W)[2], ops_vgg.s2d_extent(H, W)[3], 48, 48)
    assert torch.equal(a.data.cpu().view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("H,W", [(224, 224), (227, 227), (199, 241)])
def test_alexnet_conv1_through_space_to_depth_against_fp64(H, W):
    g = torch.Generator().manual_seed(5)
    x = torch.randn((2, 3, H, W), generator=g)
    w = torch.randn((64, 3, 11, 11), generator=g) / 20
    bias = torch.randn(64, generator=g) * 0.1
    pc = ops.PackedConv(ops_vgg.s2d_filter(w).to(dev), bias.to(dev), None, (1, 1, 1), (0, 0, 0), in_pitch=48)
    y = ops.conv(ops_vgg.space_to_depth4(x.to(dev)), pc, relu=True)
    torch.cuda.synchronize()
    x16, w16 = x.half().double(), w.half().double()
    ref = torch.nn.functional.conv2d(x16, w16, bias.double(), stride=4, padding=2).clamp_min(0)
    A = torch.nn.functional.conv2d(x16.abs(), w16.abs(), bias.double().abs(), stride=4, padding=2)
    got = y.data.cpu().double().reshape(2, y.H, y.W, 64).permute(0, 3, 1, 2)
    assert got.shape == ref.shape
    err = (got - ref).abs() / KR.bound(ref, A, True)
    assert float(err.max()) <= 1.0


# ---------------------------------------------------------------------------------------------
# 2. the split-K GEMM
# ---------------------------------------------------------------------------------------------
def _gemm_case(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = (torch.rand((M, K), generator=g) * 2).half().to(dev)
    b = (torch.randn((N, K), generator=g) / K ** 0.5).half().to(dev)
    sc = (torch.rand(N, generator=g) + 0.5).to(dev)
    sh = (torch.randn(N, generator=g) * 0.1).to(dev)
    return a, b, sc, sh


SHAPES = [(M, N, K) for M in (2, 16, 128, 256) for (N, K) in ((4096, 25088), (4096, 9216), (4096, 4096), (1000, 4096), (365, 4096))]
SHAPES += [(77, 1003, 1000), (300, 130, 2112), (5, 36, 640)]


@pytest.mark.parametrize("M,N,K", SHAPES, ids=["%dx%dx%d" % c for c in SHAPES])
def test_gemm_splitk_against_fp64(M, N, K):
    a, b, sc, sh = _gemm_case(M, N, K, seed=M + N + K)
    i = SHAPES.index((M, N, K))
    relu, out_f32 = bool(i % 2), bool((i // 2) % 2)
    splits = max(2, ops_vgg.splitk_plan(M, N, K, _sms())) if (K + 63) // 64 >= 2 else 1
    d = ops_vgg.gemm_splitk(a, b, sc, sh, M, N, K, splits, relu=relu, out_f32=out_f32)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    assert kid == 17 and info[:2] == [64 if ops._round_up(N, 8) <= 64 else 128, splits]
    ratio, where = check_gemm_splitk(a, b, sc, sh, M, N, K, d, relu=relu, out_f32=out_f32)
    assert ratio <= 1.0, where
    again = ops_vgg.gemm_splitk(a, b, sc, sh, M, N, K, splits, relu=relu, out_f32=out_f32)
    assert torch.equal(again.view(torch.int16), d.view(torch.int16)), "a second call differs"


def test_gemm_splitk_refuses_calls_outside_its_contract():
    M, N, K = 16, 256, 1024
    a, b, sc, sh = _gemm_case(M, N, K, seed=3)
    d = torch.empty((M, N), dtype=torch.float16, device=dev)
    lib = _lib.load()
    n_ws = lib.b2_gemm_splitk_workspace_elems(M, N, 4)
    ws = torch.empty(n_ws, dtype=torch.float32, device=dev)

    def call(splits=4, ws_elems=n_ws, **kw):
        g = ops.GemmArgs()
        g.a, g.b, g.scale, g.shift, g.d = ops._ptr(a), ops._ptr(b), ops._ptr(sc), ops._ptr(sh), ops._ptr(d)
        g.M, g.N, g.Kd, g.lda, g.ldb, g.ldd = M, N, K, K, K, N
        for k, v in kw.items():
            setattr(g, k, v)
        return lib.b2_gemm_splitk_f16(ctypes.byref(g), splits, ops._ptr(ws), ws_elems, ops._stream())

    assert call() == 0
    torch.cuda.synchronize()
    assert call(residual=ops._ptr(d), ldr=N) == -1 and call(mask=ops._ptr(d), ldm=N) == -1 and call(per_row=1) == -1
    assert call(aff_ld=N, aff_rows=128) == -1 and call(d2=ops._ptr(d)) == -1 and call(accumulate=1, out_f32=1) == -1
    assert call(splits=0) == -1 and call(splits=17) == -1 and call(ws_elems=n_ws - 1) == -1


# ---------------------------------------------------------------------------------------------
# 3. the models and TRN against the reference fixtures
# ---------------------------------------------------------------------------------------------
def _fixture_model(fx):
    torch.manual_seed(fx["seeds"]["init"])
    m = getattr(P, fx["arch"])(pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval().to(dev)


@pytest.mark.parametrize("arch", ("vgg16", "vgg16_bn", "vgg11", "alexnet"))
def test_model_matches_reference_fixture(arch):
    fx = _load("%s_b2_224.pt" % arch)
    m = _fixture_model(fx)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
        whole = m(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == (2, 4096) and feats.dtype == torch.float32
    for got, want in ((feats, fx["features"]), (logits, fx["logits"])):
        want = want.double()
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= 1e-2, "%s: rel err %.3e" % (arch, err)
    assert torch.equal(logits.argmax(1).cpu(), fx["logits"].argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(m, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


@pytest.mark.parametrize("arch", ("vgg16", "alexnet"))
def test_trn_mstrn_matches_reference_fixture(arch):
    fx = _load("trn_%s_MSTRN.pt" % arch)
    m = trn_as_reference(arch, fx)
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    m = m.eval().to(dev)
    assert m.frame_feature_dim == 4096
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        np.random.seed(fx["seeds"]["tuples"])
        feats = m.features(x)
        logits = m.logits(feats)
    for got, want in ((feats, fx["features"]), (logits, fx["logits"])):
        want = want.double()
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= 1e-2, "rel err %.3e" % err


# ---------------------------------------------------------------------------------------------
# 4. every launch of the forwards at their measured batch against fp64
# ---------------------------------------------------------------------------------------------
def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _expected_launches(m, B):
    """Launches of one forward: the input pass, one per convolution and pool, and per classifier GEMM two when it runs split-K."""
    trunk = 1 + sum(isinstance(l, (torch.nn.Conv2d, torch.nn.MaxPool2d)) for l in m._features)
    C, H = (256, 6) if isinstance(m, P.models.vgg.AlexNet) else (512, 7)
    gemms = [(B, 4096, C * H * H), (B, 4096, 4096), (B, m.last_linear.out_features, 4096)]
    return trunk + 1 + sum(2 if ops_vgg.splitk_plan(*s, _sms()) > 1 else 1 for s in gemms)


AUDITS = [(a, functools.partial(getattr(P, a), pretrained=None), (256, 3, 224, 224)) for a in ARCHS]
AUDITS += [("trn_%s_MSTRN" % a, functools.partial(P.TRN, 10, num_segments=8, arch=a, consensus="MSTRN", pretrained=None, **TRN_KW),
            (16, 8, 3, 224, 224)) for a in ("vgg16", "alexnet")]


@pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV), reason="a dispatch override is set in the environment")
@pytest.mark.timeout(2400, method="thread")
@pytest.mark.parametrize("name,make,shape", AUDITS, ids=[a[0] for a in AUDITS])
def test_forward_every_launch_against_fp64(name, make, shape):
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    m = make()
    OF.randomize_bn_(m, 1)
    m = m.eval().to(dev)
    for mod in m.modules():
        if hasattr(mod, "sample_tuples"):
            np.random.seed(0)
            picks = mod.sample_tuples()
            mod.sample_tuples = functools.partial(lambda p: p, picks)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1000)).to(dev)
    t0 = time.time()
    rep = audit(lambda: m(x))
    _report("%s_B%d" % (name, shape[0]), rep, time.time() - t0)
    _assert_clean(name, rep)
    want = rep.output.clone()
    rep = None
    c0 = _lib.launch_count()
    with torch.no_grad():
        again = m(x)
    torch.cuda.synchronize()
    if not name.startswith("trn"):                  # once the filters are packed
        assert _lib.launch_count() - c0 == _expected_launches(m, shape[0])
    assert torch.equal(_bits(again), _bits(want)), "a second eager forward differs from the audited one"
    got = GraphedForward(m, x, warmup=1)()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"


# ---------------------------------------------------------------------------------------------
# 5. the trainable head
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ("vgg16", "alexnet"))
def test_last_linear_gradients_against_fp64(arch):
    torch.manual_seed(0)
    m = getattr(P, arch)(pretrained=None).eval().to(dev)
    x = torch.randn((4, 3, 224, 224), generator=torch.Generator().manual_seed(7)).to(dev)
    with torch.no_grad():
        f = m.features(x)
    out = m.logits(f)
    gy = torch.randn(out.shape, generator=torch.Generator().manual_seed(8)).to(dev) / 4
    out.backward(gy)
    x16 = torch.relu(f).half().double()
    gw = gy.double().t() @ x16
    gb = gy.double().sum(0)
    A = gy.double().abs().t() @ x16.abs()
    assert float(((m.last_linear.weight.grad.double() - gw).abs() / (2 ** -8 * A + 2 ** -24)).max()) <= 1.0
    assert float(((m.last_linear.bias.grad.double() - gb).abs() / (2 ** -20 * gy.double().abs().sum(0) + 2 ** -24)).max()) <= 1.0
