"""GPU (-m gpu): SE-ResNet / SE-ResNeXt on the engine.

1. b2_gemm_sample_affine_f16 element by element against fp64 under the kernel-matrix bound of tests/kernel_ref.py
   (2^-11 |ref| + 2^-14 A + 2^-24, A = |scale| sum |a w| + |shift| + |r|), at every rows-per-sample of the 224^2 networks and
   at ones that do not divide a 128-row tile, with the persistent kernel pinned and the pitch contract asserted.
2. b2_se_excite against an fp64 restatement of SEModule (unfolded: conv3 + bn3, avgpool, fc1, fc2) under the bound derived in
   ``tests/kernel_ref.excite_bound``.
3. The ceil-mode stem pool bit-exact against F.max_pool2d(..., ceil_mode=True).
4. Every SE block kind against the fp64 oracle block (oracle/senet.py) on the engine's own fp16 input: 5e-3 of max |ref|.
5. se_resnet50 / se_resnext50_32x4d / TRN-MSTRN against the reference's fixtures (per-stage samples 1e-2, logits 5e-3 of
   max |ref|, equal arg-max), and CUDA-graph replay bit-identical to the eager forward.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200 import functions as Fn
from pretorched_x_b200.graph import GraphedForward
from pretorched_x_b200.models import senet as PS
from pretorched_x_b200.ops import Act
from oracle import functional as OF
from oracle import senet as OS
from oracle.make_golden import sample_of
from tests import kernel_ref as KR
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PGEMM = 6          # KID_PGEMM of csrc/b2_host.h


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 5)()
    kid = _lib.load().b2_debug_last_kernel(info)
    return kid, list(info)


# ---------------------------------------------------------------------------------------------
# 1. per-sample-affine GEMM at any rows per sample
# ---------------------------------------------------------------------------------------------
GEMM_CASES = [
    # rows per sample, samples, N, Kd, residual, ldd extra columns
    (3136, 2, 256, 64, True, 0),        # layer1 conv3 of se_resnet50 at 224^2
    (784, 3, 512, 128, True, 0),        # layer2
    (196, 3, 1024, 256, True, 8),       # layer3, output pitch wider than N
    (49, 5, 2048, 512, True, 0),        # layer4: 245 rows, ragged last tile
    (49, 3, 2048, 1024, False, 0),
    (36, 7, 256, 64, True, 16),
    (1, 300, 512, 128, True, 0),
    (128, 3, 256, 64, False, 0),
    (200, 3, 768, 192, True, 8),
    (3136, 1, 64, 64, True, 8),         # the 64-wide N tile
]


def _gemm_call(a, w, scale, shift, M, N, Kd, R, residual, ldd):
    out = torch.full((M, ldd), float("nan"), dtype=torch.float16, device=dev)
    g = _lib.GemmArgs()
    g.a, g.b, g.scale, g.shift = ops._ptr(a), ops._ptr(w), ops._ptr(scale), ops._ptr(shift)
    g.residual, g.d = ops._ptr(residual), ops._ptr(out)
    g.M, g.N, g.Kd = M, N, Kd
    g.lda, g.ldb, g.ldd = a.stride(0), w.stride(0), ldd
    g.ldr = residual.stride(0) if residual is not None else 0
    g.relu, g.aff_ld, g.aff_rows = 1, scale.stride(0), R
    _lib.check(_lib.load().b2_gemm_sample_affine_f16(ctypes.byref(g), ops._stream()), "b2_gemm_sample_affine_f16")
    return out


@pytest.mark.parametrize("R,ns,N,Kd,with_res,extra", GEMM_CASES)
def test_gemm_sample_affine_matches_fp64(R, ns, N, Kd, with_res, extra):
    g = torch.Generator(device="cpu").manual_seed(R * 7 + N)
    M, ldd = R * ns, N + extra
    a = torch.rand((M, Kd), generator=g).to(torch.float16).to(dev)
    w = (torch.randn((N, Kd), generator=g) / Kd ** 0.5).to(torch.float16).to(dev)
    lda = ops._round_up(N, 4) + 4
    aff = torch.randn((2, ns, lda), generator=g).float().to(dev)
    scale, shift = aff[0], aff[1] * 0.5
    res = None
    if with_res:
        res = torch.randn((M, ldd), generator=g).to(torch.float16).to(dev)
        res[:, N:] = float("nan")                             # columns >= N must never be read
    out = _gemm_call(a, w, scale, shift, M, N, Kd, R, res, ldd)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    assert _lib.load().b2_debug_last_gemm_path() == 2 and kid == PGEMM and info[1] == 2 and info[0] == (64 if ldd <= 64 else 128)
    acc, mag = KR.gemm_acc(a, w)
    rows = torch.arange(M) // R
    sc, sh = scale.double().cpu()[rows, :N], shift.double().cpu()[rows, :N]
    ref, A = acc * sc + sh, mag * sc.abs() + sh.abs()
    if res is not None:
        r = res[:, :N].double().cpu()
        ref, A = ref + r, A + r.abs()
    ref = ref.clamp_min(0.0)
    assert torch.all(out[:, N:] == 0), "pitch columns [N, ldd) must be written as zero"
    worst = KR.worst_ratio(out[:, :N], ref, A, True)
    assert worst <= 1.0, "R=%d N=%d: %s" % (R, N, KR.where_worst(out[:, :N], ref, A, True))
    again = _gemm_call(a, w, scale, shift, M, N, Kd, R, res, ldd)
    assert torch.equal(out, again), "not bitwise repeatable"


def test_gemm_sample_affine_refuses_bad_contract():
    a = torch.zeros((98, 64), dtype=torch.float16, device=dev)
    w = torch.zeros((256, 64), dtype=torch.float16, device=dev)
    aff = torch.zeros((2, 2, 256), dtype=torch.float32, device=dev)
    with pytest.raises(RuntimeError, match="whole number of samples"):
        _gemm_call(a, w, aff[0], aff[1], 98, 256, 64, 50, None, 256)
    with pytest.raises(RuntimeError, match="aligned"):
        _gemm_call(a, w, aff[0][:, 1:], aff[1][:, 1:], 98, 248, 64, 49, None, 248)


# ---------------------------------------------------------------------------------------------
# 2. squeeze-excite
# ---------------------------------------------------------------------------------------------
EXCITE_CASES = [
    # N, S, C2, ldh, C (R = C / 16)
    (4, 3136, 64, 64, 256),        # se_resnet50 layer1
    (3, 3136, 128, 128, 256),      # se_resnext50 layer1
    (3, 784, 256, 256, 512),
    (5, 196, 512, 512, 1024),
    (3, 49, 1024, 1024, 2048),
    (17, 49, 512, 520, 2048),      # more samples than one CTA row, channel pitch > C2
    (2, 1, 128, 128, 512),
]


def excite_ref(h, w3, s3, t3, f1, b1, f2, b2, N, S, C2):
    """fp64 SEModule on bn3(conv3(h)) pooled first (unfolded), plus the magnitudes ``KR.excite_bound`` needs: the fc1 of
    ``KR.excite_ref`` applied to the unfolded affine map bn3(W3 m)."""
    m, habs = KR.excite_mean(h, N, S, C2)
    w3d, s3d, t3d = w3.double().cpu(), s3.double().cpu(), t3.double().cpu()
    f1d = f1.double().cpu()
    return KR.excite_ref(m, habs, (f1d * s3d[None, :]) @ w3d, f1d @ t3d + b1.double().cpu(), f2, b2, s3, t3)


@pytest.mark.parametrize("N,S,C2,ldh,C", EXCITE_CASES)
def test_se_excite_matches_fp64(N, S, C2, ldh, C):
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + C2)
    R = C // 16
    h = torch.zeros((N * S, ldh), dtype=torch.float16)
    h[:, :C2] = (torch.rand((N * S, C2), generator=g) * 3).to(torch.float16)
    w3 = torch.randn((C, C2), generator=g) / C2 ** 0.5
    s3, t3 = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    f1, b1 = torch.randn((R, C), generator=g) / C ** 0.5, torch.randn(R, generator=g) * 0.1
    f2, b2 = torch.randn((C, R), generator=g) / R ** 0.5, torch.randn(C, generator=g) * 0.1
    w1f = ((f1.double() * s3.double()[None, :]) @ w3.double()).float()
    b1f = (f1.double() @ t3.double() + b1.double()).float()
    hd = h.to(dev)
    act = Act(hd, N, 1, 1, S, C2)
    args = [t.to(dev).contiguous() for t in (w1f, b1f, f2, b2, s3, t3)]
    scale, shift = ops.se_excite(act, *args)
    scale2, shift2 = ops.se_excite(act, *args)
    torch.cuda.synchronize()
    assert torch.equal(scale, scale2) and torch.equal(shift, shift2), "not bitwise repeatable"
    r = excite_ref(h, w3, s3, t3, f1, b1, f2, b2, N, S, C2)
    bs, bh = KR.excite_bound(r, w1f, b1f, f2, b2, s3, t3, S, fold_rounding=True)
    for got, want, bnd, what in ((scale, r["scale"], bs, "scale"), (shift, r["shift"], bh, "shift")):
        worst = KR.worst_ratio_of(got[:, :C], want, bnd)
        assert worst <= 1.0, "%s: %s" % (what, KR.where_worst_of(got[:, :C], want, bnd))


# ---------------------------------------------------------------------------------------------
# 3. ceil-mode stem pool
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(112, 112), (111, 111), (57, 113), (7, 7)])
def test_ceil_mode_pool_bit_exact(H, W):
    g = torch.Generator(device="cpu").manual_seed(H * W)
    N, C = 2, 64
    x = torch.randn((N, C, H, W), generator=g).to(torch.float16)
    a = ops.from_ncdhw(x.to(dev), pitch=C)
    y = ops.maxpool2d_ceil(a, 3, 2, 0)
    want = F.max_pool2d(x.float(), 3, 2, ceil_mode=True)
    assert (y.H, y.W) == tuple(want.shape[2:])
    got = y.data.view(N, y.H, y.W, C).permute(0, 3, 1, 2).float().cpu()
    assert torch.equal(got, want)


# ---------------------------------------------------------------------------------------------
# 4. blocks against the fp64 oracle block
# ---------------------------------------------------------------------------------------------
BLOCK_CASES = [
    # id, block class, inplanes, planes, groups, stride, H (input)
    ("se_resnet_identity", PS.SEResNetBottleneck, 256, 64, 1, 1, 56),
    ("se_resnet_projection_strided_conv1", PS.SEResNetBottleneck, 256, 128, 1, 2, 56),
    ("se_resnet_projection_stride1", PS.SEResNetBottleneck, 64, 64, 1, 1, 56),
    ("se_resnext_cg4_stride2", PS.SEResNeXtBottleneck, 256, 64, 32, 2, 56),     # width 128: 4 per group
    ("se_resnext_cg4_layer1", PS.SEResNeXtBottleneck, 64, 64, 32, 1, 56),       # width 128: 4 per group
    ("se_resnext_cg32_stride2", PS.SEResNeXtBottleneck, 1024, 512, 32, 2, 14),  # width 1024: 32 per group
]


@pytest.mark.parametrize("name,cls,inplanes,planes,groups,stride,H", BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_block_matches_oracle(name, cls, inplanes, planes, groups, stride, H):
    torch.manual_seed(5)
    ds = None
    if stride != 1 or inplanes != planes * 4:
        ds = torch.nn.Sequential(torch.nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False), torch.nn.BatchNorm2d(planes * 4))
    blk = cls(inplanes, planes, groups, 16, stride, ds)
    OF.randomize_bn_(blk, 3)
    blk.eval().to(dev)
    x = torch.rand((2, inplanes, H, H), generator=torch.Generator().manual_seed(9)).to(torch.float16)
    a = ops.from_ncdhw(x.to(dev))
    with torch.no_grad():
        y = engine.run_se_bottleneck(blk, a)
    got = ops.to_ncdhw(y).squeeze(2).double().cpu()
    sd = {k: v.detach().double().cpu() for k, v in blk.state_dict().items()}
    want = OS.block(x.double(), {"b." + k: v for k, v in sd.items()}, "b", groups > 1, groups, stride, ds is not None)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s: rel err %.3e" % (name, err)


# ---------------------------------------------------------------------------------------------
# 5. models against the reference fixtures
# ---------------------------------------------------------------------------------------------
def _stages(model, x):
    a = Fn.frozen(lambda t, o: engine._se_stem_body(model.layer0, t, o), ops.from_ncdhw(x))
    out = {"layer0": a}
    for name in ("layer1", "layer2", "layer3", "layer4"):
        for blk in getattr(model, name):
            a = engine.run_se_bottleneck(blk, a)
        out[name] = a
    return out, model.logits(a)


@pytest.mark.parametrize("fname", ["se_resnet50_b2_224.pt", "se_resnext50_32x4d_b2_224.pt"])
def test_model_stages_match_reference_fixture(fname):
    fx = _load(fname)
    model = OS.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        stages, logits = _stages(model, x)
        whole = model(x)
    torch.cuda.synchronize()
    for name, summ in fx["stages"].items():
        t = ops.to_ncdhw(stages[name]).squeeze(2).cpu()
        assert tuple(t.shape) == tuple(summ["shape"]), name
        s, step = sample_of(t)
        assert step == summ["step"]
        err = (s.double() - summ["sample"].double()).abs().max().item() / summ["absmax"]
        assert err <= 1e-2, "%s %s: rel err %.3e" % (fname, name, err)
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s logits: rel err %.3e" % (fname, err)
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(model, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_se_resnext50_32x4d_MSTRN.pt")
    model = OS.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        np.random.seed(fx["seeds"]["tuples"])
        feats = model.features(x)
        logits = model.logits(feats)
    for got, want, tol in ((feats, fx["features"], 1e-2), (logits, fx["logits"], 5e-3)):
        want = want.double()
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= tol, "rel err %.3e" % err
    assert int(logits.argmax()) == int(fx["logits"].argmax())


def test_final_map_other_than_7x7_is_refused():
    torch.manual_seed(0)
    model = P.se_resnet50(pretrained=None).eval().to(dev)
    x = torch.rand((1, 3, 160, 160), device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match="7x7"):
        model(x)
