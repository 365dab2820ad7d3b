"""GPU (-m gpu): Xception on the engine.

1. The forward against the reference's fixtures at 299^2 and 224^2 (tests/golden/xception_b2_*.pt): the stem's and every block's
   output within 1e-2 and the logits within 5e-3 of max |ref|, equal arg-max, ``features`` equal to the staged trunk, the whole
   forward equal to the staged one and a CUDA-graph replay bit-identical to it.  A non-square odd input against the oracle in fp64.
2. TRN-MSTRN on Xception against its fixture.
3. The ReLU-on-input depthwise kernel (b2_dwconv3x3_relu_in_ndhwc) against fp64 within the per-element bound of tests/kernel_ref.py,
   with the kernel that ran pinned (KID 19): every channel count of the network's depthwise passes, every map size it produces at
   299^2 and 224^2, signed inputs.
4. Every library launch of the forward at 256 images (299^2) and of TRN-MSTRN at 16 videos x 8 segments held element by element to
   its fp64 bound (tests/xception_audit.py), the launches per forward pinned, and a CUDA-graph replay bit-identical to the audited
   eager output.
5. A Block called on its own on a signed input, start_with_relu True and False, against the oracle in fp64.
"""
import ctypes
import functools
import os
import time

import numpy as np
import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, functions as Fn, ops, ops_xception
from pretorched_x_b200.graph import GraphedForward
from oracle import functional as OF
from oracle import xception as OXc
from oracle.make_golden import sample_of
from tests.conftest import has_h100
from tests.kernel_ref import where_worst, worst_ratio
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report
from tests.xception_audit import KID_DWCONV_RELU_IN, audit, dw_relu_in_ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _stages(model, x):
    """The trunk unit by unit: {stem, block1 .. block12}, bn4's output and the logits."""
    a = Fn.frozen(lambda t, o: engine._xception_stem_body(model, t), ops.from_ncdhw(x, pitch=8))
    stages = {"stem": a}
    for b in OXc.BLOCKS:
        a = getattr(model, b)(a)
        stages[b] = a
    f = Fn.frozen(lambda t, o: engine._xception_exit_body(model, t), a)
    return stages, f, model.logits(f)


# ---------------------------------------------------------------------------------------------
# 1-2. the reference fixtures
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [299, 224])
def test_forward_stages_match_reference_fixture(hw):
    fx = _load("xception_b2_%d.pt" % hw)
    model = OXc.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        stages, f, logits = _stages(model, x)
        whole = model(x)
        feats = model.features(x)
    torch.cuda.synchronize()
    for name, summ in fx["stages"].items():
        t = ops.to_ncdhw(stages[name]).squeeze(2).cpu()
        assert tuple(t.shape) == tuple(summ["shape"]), name
        s, step = sample_of(t)
        assert step == summ["step"]
        err = (s.double() - summ["sample"].double()).abs().max().item() / summ["absmax"]
        assert err <= 1e-2, "%d %s: rel err %.3e" % (hw, name, err)
    assert tuple(feats.shape) == tuple(fx["features"]["shape"])
    assert torch.equal(feats, ops.to_ncdhw(f).squeeze(2))
    s, _ = sample_of(feats.cpu())
    err = (s.double() - fx["features"]["sample"].double()).abs().max().item() / fx["features"]["absmax"]
    assert err <= 1e-2, "features: rel err %.3e" % err
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "logits: rel err %.3e" % err
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(model, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_odd_non_square_input_against_fp64_oracle():
    torch.manual_seed(0)
    model = P.xception(pretrained=None)
    OF.randomize_bn_(model, 1)
    model = model.eval().to(dev)
    x = OF.seeded_input((3, 3, 97, 131), 4).to(dev)
    sd = {k: v.detach().double() if v.is_floating_point() else v for k, v in model.state_dict().items()}
    with torch.no_grad():
        got = model(x)
        want = OXc.forward(x.double(), sd)
        feats = model.features(x)
        wf = OXc.features(x.double(), sd)
    assert tuple(feats.shape) == tuple(wf.shape) == (3, 2048, 3, 4)
    err = (feats.double() - wf).abs().max().item() / wf.abs().max().item()
    assert err <= 1e-2, "features: rel err %.3e" % err
    err = (got.double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "logits: rel err %.3e" % err


@pytest.mark.parametrize("cin,cout,reps,strides,start_with_relu,grow_first", [
    (64, 128, 2, 2, False, True),          # block1's layout: no ReLU opens the first separable convolution
    (128, 128, 3, 1, False, True),         # the same with the identity skip
    (128, 256, 2, 2, True, True),          # block2's layout
    (256, 256, 3, 1, True, True),          # a middle-flow block
    (256, 384, 2, 2, True, False),         # block12's layout (the widening in the last repetition)
])
def test_standalone_block_on_signed_input_against_fp64_oracle(cin, cout, reps, strides, start_with_relu, grow_first):
    """A Block called on its own, on a signed input: the first depthwise pass reads max(x, 0) only when a ReLU opens it."""
    torch.manual_seed(3)
    blk = P.models.xception.Block(cin, cout, reps, strides, start_with_relu=start_with_relu, grow_first=grow_first)
    OF.randomize_bn_(blk, 2)
    blk = blk.eval().to(dev)
    x = OF.seeded_input((2, cin, 23, 17), 5).to(dev)
    sd = {k: v.detach().double() for k, v in blk.state_dict().items() if v.is_floating_point()}
    with torch.no_grad():
        got = blk(x)
        want = OXc.block(x.half().double(), sd, "")
    assert tuple(got.shape) == tuple(want.shape)
    err = (got.double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 1e-2, "rel err %.3e" % err
    if not start_with_relu:                # the same block with a ReLU in front differs: the test sees the first ReLU
        assert (got.double() - OXc.block(x.half().double().relu(), sd, "")).abs().max().item() > 0.1 * want.abs().max().item()


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_xception_MSTRN.pt")
    model = OXc.build_package_model(P, fx).to(dev)
    assert model.frame_feature_dim == 2048
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


# ---------------------------------------------------------------------------------------------
# 3. the ReLU-on-input depthwise kernel against fp64
# ---------------------------------------------------------------------------------------------
CHANNELS = (64, 128, 256, 728, 1024, 1536)
MAPS = (147, 74, 37, 19, 10, 109, 55, 28, 14, 7)       # the depthwise maps at 299^2, then at 224^2


@pytest.mark.parametrize("C", CHANNELS)
def test_depthwise_relu_in_against_fp64(C):
    for hw in MAPS:
        B, ld = 2, C + (8 if hw % 2 else 0)               # odd maps also with a channel pitch past C
        g = torch.Generator().manual_seed(C * 1000 + hw)
        x = (torch.randn(B, hw, hw, C, generator=g) * 3).half()
        w9 = torch.randn(9, C, generator=g) * 0.3
        data = torch.zeros(B * hw * hw, ld, dtype=torch.float16)
        data[:, :C] = x.reshape(-1, C)
        a = ops.Act(data.to(dev), B, 1, hw, hw, C)
        M, pad = B * hw * hw, 2
        buf = torch.full((M + 2 * pad, ld), float("nan"), dtype=torch.float16, device=dev)
        out = buf[pad:pad + M]
        wd = w9.to(dev)
        y = ops_xception.dwconv3x3_relu_in(a, wd, out=out)
        torch.cuda.synchronize()
        assert _last_kernel() == (KID_DWCONV_RELU_IN, [1, 4, 0, 0, 0])
        again = ops_xception.dwconv3x3_relu_in(a, wd)
        torch.cuda.synchronize()
        assert (y.N, y.T, y.H, y.W, y.C, y.ld) == (B, 1, hw, hw, C, ld)
        assert torch.isnan(buf[:pad].float()).all() and torch.isnan(buf[pad + M:].float()).all(), "rows outside out= were written"
        assert torch.all(out[:, C:] == 0), "padding channels [C, ld) not zero"
        assert torch.equal(again.data.view(torch.int16), out.view(torch.int16)), "two identical calls differ"
        ref, A = dw_relu_in_ref(x, w9, device=dev)
        r = worst_ratio(out[:, :C].cpu(), ref.cpu(), A.cpu(), True)
        print("[xception-dw] C%-5d %3dx%-3d ld %d worst err/bound %.4f" % (C, hw, hw, ld, r))
        assert r <= 1.0, "C %d %dx%d: err/bound %.3f at %s" % (C, hw, hw, r, where_worst(out[:, :C].cpu(), ref.cpu(), A.cpu(), True))


# ---------------------------------------------------------------------------------------------
# 4. every launch at the measured batch against fp64
# ---------------------------------------------------------------------------------------------
def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


# once the filters are packed: the input layout pass and the stem's two convolutions; two launches per separable convolution
# (the depthwise pass, the pointwise GEMM), and in blocks 1-3 and 12 the max-pool, the skip's pixel gather and its GEMM; the head's
# ReLU + mean and last_linear
EXPECTED_LAUNCHES = 3 + 2 * (4 * 2 + 8 * 3 + 2) + 4 * 3 + 2
# 34 depthwise passes: all but block1's first (no ReLU opens it) and conv3's (its input is block12's signed sum) read max(x, 0)
RELU_IN_LAUNCHES = 32


def _expected_launches(m):
    """One forward once the filters are packed.  TRN: the backbone without last_linear (a Dropout there), the cast of the frame
    features to fp16, per relation scale the tuple gather and two GEMMs, and the cast + GEMM of the TRN head."""
    if isinstance(m, P.TRN):
        return EXPECTED_LAUNCHES - 1 + 1 + 3 * len(m.temporal_relation.scales) + 2
    return EXPECTED_LAUNCHES


AUDITS = [("xception", functools.partial(P.xception, pretrained=None), (256, 3, 299, 299)),
          ("trn_xception_MSTRN", functools.partial(P.TRN, 10, num_segments=8, arch="xception", consensus="MSTRN", pretrained=None,
                                                   **TRN_KW), (16, 8, 3, 299, 299))]


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
    assert sum(r["launches"] for r in rep.rows if r["entry"] == "dwconv3x3_relu_in") == RELU_IN_LAUNCHES
    assert sum(r["launches"] for r in rep.rows if r["entry"] == "dwconv3x3") == 34 - RELU_IN_LAUNCHES
    want = rep.output.clone()
    rep = None
    c0 = _lib.launch_count()
    with torch.no_grad():
        again = m(x)
    torch.cuda.synchronize()
    assert _lib.launch_count() - c0 == _expected_launches(m)
    assert torch.equal(_bits(again), _bits(want)), "a second eager forward differs from the audited one"
    got = GraphedForward(m, x, warmup=1)()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"
