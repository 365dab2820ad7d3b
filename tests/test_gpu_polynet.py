"""GPU (-m gpu): PolyNet, TRN on it, and the dual GEMM.

1. b2_gemm_dual_f16 against fp64 at the stage B / C close shapes at 256 images and at ragged M and N: the kernel that ran pinned,
   both outputs within the per-element bound of tests/kernel_ref.py (tests/dual_audit.check_gemm_dual), d bit for bit what
   b2_gemm_f16 writes for the same arguments, a second call bitwise equal, and the refusals of its contract.
2. Each module kind (stem, A-2way, B-poly3, B-2way, C-poly3, C-2way, both reductions) against the fp64 oracle module on the
   engine's fp16 input, with its launch count.
3. The model and TRN-MSTRN against the reference's fixtures (oracle/make_golden_polynet.py), and CUDA-graph replays bit-identical
   to the eager forward.
4. tests/dual_audit.audit (tests/model_audit.py's audit, extended to ops_dual) over the forward at 256 images, 331^2, and over TRN-MSTRN at 16 videos x 8 segments.
"""
import functools
import os
import time

import numpy as np
import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops, ops_dual
from pretorched_x_b200.graph import GraphedForward
from oracle import functional as OF
from oracle import polynet as OP
from oracle.make_golden import sample_of
from tests.conftest import has_h100
from tests.dual_audit import audit, check_gemm_dual
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CLOSE = 0.15
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)
# launches per module, once its filters are packed (engine._polynet_*_body)
LAUNCHES = {"Stem": 12, "InceptionResNetA2Way": 9, "InceptionResNetB2Way": 6, "InceptionResNetC2Way": 6,
            "InceptionResNetBPoly3": 12, "InceptionResNetCPoly3": 12, "ReductionA": 5, "ReductionB": 6}


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    import ctypes
    info = (ctypes.c_int * 8)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


# ---------------------------------------------------------------------------------------------
# 1. the dual GEMM
# ---------------------------------------------------------------------------------------------
def _dual_case(M, N, K, seed, residual=True, relu=False):
    g = torch.Generator().manual_seed(seed)
    a = (torch.rand((M, K), generator=g) * 2).half().to(dev)
    b = (torch.randn((N, K), generator=g) / K ** 0.5).half().to(dev)
    sb = (torch.rand(N, generator=g) + 0.5).to(dev)
    tb = (torch.randn(N, generator=g) * 0.1).to(dev)
    s = 0.9
    res = (torch.randn((M, ops._round_up(N, 8)), generator=g)).half().to(dev) if residual else None
    return a, b, (s * sb).contiguous(), (s * tb).contiguous(), sb, tb, res


# (M, N, K): the stage B and C closes at 256 images (19^2 and 9^2 maps), and ragged M / N on both N tiles
DUAL = [(256 * 19 * 19, 1152, 384), (256 * 9 * 9, 2048, 448), (1000, 200, 104), (77, 40, 64), (130, 1160, 192)]


@pytest.mark.parametrize("M,N,K", DUAL, ids=["%dx%dx%d" % c for c in DUAL])
def test_dual_gemm_against_fp64(M, N, K):
    a, b, sc, sh, s2, t2, res = _dual_case(M, N, K, seed=M + N)
    d, d2 = ops_dual.gemm_dual(a, b, sc, sh, s2, t2, M, N, K, residual=res)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    bn = 64 if ops._round_up(N, 8) <= 64 else 128
    assert kid == 6 and info[:3] == [bn, 4, 0] and _lib.load().b2_debug_last_gemm_path() == 2
    ratio, where = check_gemm_dual(a, b, sc, sh, s2, t2, M, N, K, d, d2, residual=res)
    assert ratio <= 1.0, where
    again = ops_dual.gemm_dual(a, b, sc, sh, s2, t2, M, N, K, residual=res)
    assert torch.equal(again[0].view(torch.int16), d.view(torch.int16)) and torch.equal(again[1].view(torch.int16), d2.view(torch.int16))
    plain = ops.gemm(a, b, sc, sh, M, N, K, residual=res)
    assert torch.equal(plain.view(torch.int16), d.view(torch.int16)), "d differs from b2_gemm_f16's output"


def test_dual_gemm_refuses_calls_outside_its_contract():
    import ctypes
    M, N, K = 256, 128, 64
    a, b, sc, sh, s2, t2, res = _dual_case(M, N, K, seed=3)
    d = torch.empty((M, N), dtype=torch.float16, device=dev)
    d2 = torch.empty((M, N), dtype=torch.float16, device=dev)
    lib = _lib.load()

    def call(d2p=d2, ldd2=N, **kw):
        g = ops.GemmArgs()
        g.a, g.b, g.scale, g.shift, g.d = ops._ptr(a), ops._ptr(b), ops._ptr(sc), ops._ptr(sh), ops._ptr(d)
        g.M, g.N, g.Kd, g.lda, g.ldb, g.ldd = M, N, K, K, K, N
        for k, v in kw.items():
            setattr(g, k, v)
        return lib.b2_gemm_dual_f16(ctypes.byref(g), ops._ptr(s2), ops._ptr(t2), ops._ptr(d2p), ldd2, ops._stream())

    assert call() == 0
    torch.cuda.synchronize()
    assert call(per_row=1) == -3 and call(out_f32=1) == -3 and call(aff_ld=N, aff_rows=128) == -3
    assert call(mask=ops._ptr(d), ldm=N) == -3 and call(d2=ops._ptr(d2)) == -3
    assert call(d2p=d) == -1 and call(d2p=a) == -1 and call(ldd2=N + 8) == -1


# ---------------------------------------------------------------------------------------------
# 2. modules against the fp64 oracle
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    m = OP.rescale_(P.polynet(pretrained=None), CLOSE)
    OF.randomize_bn_(m, 3)
    return m.eval().to(dev)


MODULES = [("stem", 3, 331), ("stage_a.0", 384, 39), ("reduction_a", 384, 39), ("stage_b.0", 1152, 19), ("stage_b.1", 1152, 19),
           ("reduction_b", 1152, 19), ("stage_c.0", 2048, 9), ("stage_c.1", 2048, 9)]


@pytest.mark.parametrize("name,C,H", MODULES, ids=[m[0] for m in MODULES])
def test_frozen_module_matches_oracle(model, name, C, H):
    mod = model.get_submodule(name)
    x = (torch.rand((2, C, H, H), generator=torch.Generator().manual_seed(9)) * 4).to(torch.float16)
    a = ops.from_ncdhw(x.to(dev), pitch=8 if C == 3 else None)
    with torch.no_grad():
        engine.Fn.frozen(lambda t, o: engine._polynet_block_body(mod, t), a)     # the first call also packs the filters
        c0 = _lib.launch_count()
        y = engine.Fn.frozen(lambda t, o: engine._polynet_block_body(mod, t), a)
    torch.cuda.synchronize()
    assert _lib.launch_count() - c0 == LAUNCHES[type(mod).__name__]
    got = ops.to_ncdhw(y).squeeze(2).double().cpu()
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    want = OP.module(x.double(), sd, mod, name + ".")
    assert got.shape == want.shape
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s: rel err %.3e" % (name, err)


# ---------------------------------------------------------------------------------------------
# 3. the model and TRN against the reference fixtures
# ---------------------------------------------------------------------------------------------
def test_model_matches_reference_fixture():
    fx = _load("polynet_b2_331.pt")
    m = OP.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
        whole = m(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == (2, 2048, 9, 9) and feats.dtype == torch.float32
    s, step = sample_of(feats.cpu())
    assert step == fx["features"]["step"]
    err = (s.double() - fx["features"]["sample"].double()).abs().max().item() / fx["features"]["absmax"]
    assert err <= 1e-2, "features: rel err %.3e" % err
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "logits: rel err %.3e" % err
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(m, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_polynet_MSTRN.pt")
    m = OP.build_package_model(P, fx).to(dev)
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 2048 and list(m.input_size) == fx["input_size"] == [331, 331]
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


# ---------------------------------------------------------------------------------------------
# 4. every launch of the measured forwards against fp64
# ---------------------------------------------------------------------------------------------
def _audit_build(make, shape):
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    m = OP.rescale_(make(), CLOSE)
    OF.randomize_bn_(m, 1)
    m = m.eval().to(dev)
    for mod in m.modules():
        if hasattr(mod, "sample_tuples"):
            np.random.seed(0)
            picks = mod.sample_tuples()
            mod.sample_tuples = functools.partial(lambda p: p, picks)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1000)).to(dev)
    return m, x


def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


AUDITS = [("polynet", lambda: P.polynet(pretrained=None), (256, 3, 331, 331)),
          ("trn_polynet_MSTRN", lambda: P.TRN(10, num_segments=8, arch="polynet", consensus="MSTRN", pretrained=None, **TRN_KW),
           (16, 8, 3, 331, 331))]


@pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV), reason="a dispatch override is set in the environment")
@pytest.mark.timeout(2400, method="thread")
@pytest.mark.parametrize("name,make,shape", AUDITS, ids=[a[0] for a in AUDITS])
def test_forward_every_launch_against_fp64(name, make, shape):
    m, x = _audit_build(make, shape)
    t0 = time.time()
    rep = audit(lambda: m(x))
    seconds = time.time() - t0
    _report("%s_B%d" % (name, shape[0]), rep, seconds)
    _assert_clean(name, rep)
    entries = {r["entry"] for r in rep.rows}
    assert "gemm_dual" in entries and not any("concat" in e or "copy" in e for e in entries), entries
    want = rep.output.clone()
    rep = None
    real, per_module = engine._polynet_block_body, []

    @functools.wraps(real)
    def counted(module, a):
        c0 = _lib.launch_count()
        y = real(module, a)
        per_module.append((type(module).__name__, _lib.launch_count() - c0))
        return y
    engine._polynet_block_body = counted
    try:
        with torch.no_grad():
            again = m(x)
        torch.cuda.synchronize()
    finally:
        engine._polynet_block_body = real
    assert torch.equal(_bits(again), _bits(want)), "a second eager forward differs from the audited one"
    kinds = [k for k, _ in per_module]
    assert kinds == (["Stem"] + ["InceptionResNetA2Way"] * 10 + ["ReductionA"] + ["InceptionResNetBPoly3", "InceptionResNetB2Way"] * 10
                     + ["ReductionB"] + ["InceptionResNetCPoly3", "InceptionResNetC2Way"] * 5)
    assert all(n == LAUNCHES[k] for k, n in per_module), per_module
    graphed = GraphedForward(m, x, warmup=1)
    got = graphed()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"
