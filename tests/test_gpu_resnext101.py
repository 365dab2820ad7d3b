"""GPU (-m gpu): ResNeXt-101 32x4d / 64x4d on the engine.

1. Both forwards against the reference's fixtures (tests/golden/resnext101_*_b2_224.pt): per-stage samples within 1e-2 and logits
   within 5e-3 of max |ref|, equal arg-max, the whole forward equal to the staged one and a CUDA-graph replay bit-identical to it.
2. TRN-MSTRN on resnext101_32x4d against its fixture, and a final map other than 7x7 refused.
3. Every library launch of both forwards at 256 images and of TRN-MSTRN at 16 videos x 8 segments (224^2) held element by element
   to the fp64 bound of tests/kernel_ref.py (tests/model_audit.py), the launches per forward pinned, and a CUDA-graph replay
   bit-identical to the audited eager output.
4. The head-only fine-tuning step (fine_tune(5)): last_linear's gradients against fp64 on the engine's features.
"""
import functools
import os
import time

import numpy as np
import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200.graph import GraphedForward
from oracle import functional as OF
from oracle import resnext as OX
from oracle.make_golden import sample_of
from tests.conftest import has_h100
from tests.model_audit import audit
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _stages(model, x):
    """The trunk unit by unit through the public engine entries: {layer0 (after the max-pool) .. layer4}, logits."""
    a = engine.run_stem(model, x)
    stages = {"layer0": a}
    for i in range(1, 5):
        for blk in getattr(model, "layer%d" % i):
            a = engine.run_block(blk, a)
        stages["layer%d" % i] = a
    return stages, model.logits(a)


# ---------------------------------------------------------------------------------------------
# 1-2. the reference fixtures
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fname", ["resnext101_32x4d_b2_224.pt", "resnext101_64x4d_b2_224.pt"])
def test_model_stages_match_reference_fixture(fname):
    fx = _load(fname)
    model = OX.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        stages, logits = _stages(model, x)
        whole = model(x)
        feats = model.features(x)
    torch.cuda.synchronize()
    for name, summ in fx["stages"].items():
        t = ops.to_ncdhw(stages[name]).squeeze(2).cpu()
        assert tuple(t.shape) == tuple(summ["shape"]), name
        s, step = sample_of(t)
        assert step == summ["step"]
        err = (s.double() - summ["sample"].double()).abs().max().item() / summ["absmax"]
        assert err <= 1e-2, "%s %s: rel err %.3e" % (fname, name, err)
    assert torch.equal(feats, ops.to_ncdhw(stages["layer4"]).squeeze(2))
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s logits: rel err %.3e" % (fname, err)
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(model, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_resnext101_32x4d_MSTRN.pt")
    model = OX.build_package_model(P, fx).to(dev)
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


def test_final_map_other_than_7x7_is_refused():
    torch.manual_seed(0)
    model = P.resnext101_32x4d(pretrained=None).eval().to(dev)
    x = torch.rand((1, 3, 256, 256), device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match="7x7"):
        model(x)


# ---------------------------------------------------------------------------------------------
# 3. every launch at the measured batch against fp64
# ---------------------------------------------------------------------------------------------
def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _expected_launches(m):
    """One forward once the filters are packed: the input layout pass, the stem convolution and the max-pool; per block conv1,
    conv2, conv3 with the residual in its epilogue and, in a stage's first block, the projection; the global pool and the head."""
    blocks = [b for i in range(1, 5) for b in getattr(m, "layer%d" % i)]
    return 3 + sum(3 + (b.downsample is not None) for b in blocks) + 2


AUDITS = [(a, functools.partial(getattr(P, a), pretrained=None), (256, 3, 224, 224)) for a in ("resnext101_32x4d", "resnext101_64x4d")]
AUDITS += [("trn_resnext101_32x4d_MSTRN", functools.partial(P.TRN, 10, num_segments=8, arch="resnext101_32x4d", consensus="MSTRN",
                                                            pretrained=None, **TRN_KW), (16, 8, 3, 224, 224))]


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
    if not name.startswith("trn"):
        assert _lib.launch_count() - c0 == _expected_launches(m)
    assert torch.equal(_bits(again), _bits(want)), "a second eager forward differs from the audited one"
    got = GraphedForward(m, x, warmup=1)()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"


# ---------------------------------------------------------------------------------------------
# 4. head-only fine-tuning
# ---------------------------------------------------------------------------------------------
def test_fine_tune_head_gradients_against_fp64():
    torch.manual_seed(0)
    m = P.resnext101_32x4d(pretrained=None).eval().to(dev).fine_tune(5)
    x = torch.randn((4, 3, 224, 224), generator=torch.Generator().manual_seed(7)).to(dev)
    out = m(x)
    gy = torch.randn(out.shape, generator=torch.Generator().manual_seed(8)).to(dev) / 4
    out.backward(gy)
    assert all(p.grad is None for n, p in m.named_parameters() if not n.startswith("last_linear."))
    with torch.no_grad():
        pooled = ops.to_ncdhw(m.features_act(x)).squeeze(2).float().mean((2, 3)).half().double()
    gw = gy.double().t() @ pooled
    gb = gy.double().sum(0)
    A = gy.double().abs().t() @ pooled.abs()
    assert float(((m.last_linear.weight.grad.double() - gw).abs() / (2 ** -8 * A + 2 ** -24)).max()) <= 1.0
    assert float(((m.last_linear.bias.grad.double() - gb).abs() / (2 ** -20 * gy.double().abs().sum(0) + 2 ** -24)).max()) <= 1.0
