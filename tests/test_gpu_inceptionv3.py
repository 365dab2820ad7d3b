"""GPU (-m gpu): Inception-v3 and TRN on it.

1. Each of the eleven blocks (Mixed_5b .. Mixed_7c) against the fp64 oracle block on the engine's fp16 input: 5e-3 of max |ref|.
2. The model and TRN-MSTRN on it against the reference's fixtures (oracle/make_golden_inceptionv3.py), as Inception-v4's are held:
   features within 1e-2 of their abs-max, logits within 5e-3 of max |logit| with the same argmax, a CUDA-graph replay
   bit-identical to the eager forward.
3. tests/model_audit.audit over the forward at 256 images, 299^2, and over TRN-MSTRN at 16 videos x 8 segments: every library
   launch within its fp64 bound, the launches of each block as the block table gives them (no concatenation or copy: every
   branch writes its columns in place), and the audited output equal bit for bit to a GraphedForward replay.
4. A trainable last_linear on the frozen trunk, and the refusal of inputs other than 299x299.
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
from oracle import inceptionv3 as OV3
from oracle.make_golden import sample_of
from tests.conftest import has_h100
from tests.model_audit import audit
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
# launches per block kind: split GEMM + slice convolutions + pool (+ its projection), see engine._inception_block_body
LAUNCHES = {"InceptionA": 6, "InceptionB": 5, "InceptionC": 9, "InceptionD": 6, "InceptionE": 8}
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    m = OV3.fan_in_scale_(P.inceptionv3(pretrained=None))
    OF.randomize_bn_(m, 3)
    return m.eval().to(dev)


# ---------------------------------------------------------------------------------------------
# 1. blocks against the fp64 oracle block
# ---------------------------------------------------------------------------------------------
BLOCKS = [("Mixed_5b", 35), ("Mixed_5c", 35), ("Mixed_5d", 35), ("Mixed_6a", 35), ("Mixed_6b", 17), ("Mixed_6c", 17),
          ("Mixed_6d", 17), ("Mixed_6e", 17), ("Mixed_7a", 17), ("Mixed_7b", 8), ("Mixed_7c", 8)]


@pytest.mark.parametrize("name,H", BLOCKS, ids=[b[0] for b in BLOCKS])
def test_frozen_block_matches_oracle(model, name, H):
    blk = model.get_submodule(name)
    cin = [mod for mod in blk.modules() if isinstance(mod, torch.nn.Conv2d)][0].in_channels
    x = (torch.rand((2, cin, H, H), generator=torch.Generator().manual_seed(9)) * 4).to(torch.float16)
    a = ops.from_ncdhw(x.to(dev))
    with torch.no_grad():
        engine.Fn.frozen(lambda t, o: engine._inception_block_body(blk, t, o), a)     # the first call also packs the filters
        c0 = _lib.launch_count()
        y = engine.Fn.frozen(lambda t, o: engine._inception_block_body(blk, t, o), a)
    torch.cuda.synchronize()
    assert _lib.launch_count() - c0 == LAUNCHES[type(blk).kind]
    got = ops.to_ncdhw(y).squeeze(2).double().cpu()
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    want = OV3.block(x.double(), sd, blk, name + ".")
    assert got.shape == want.shape
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s: rel err %.3e" % (name, err)


# ---------------------------------------------------------------------------------------------
# 2. the model and TRN against the reference fixtures
# ---------------------------------------------------------------------------------------------
def test_model_matches_reference_fixture():
    fx = _load("inceptionv3_b2_299.pt")
    m = OV3.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
        whole = m(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == (2, 2048, 8, 8) and feats.dtype == torch.float32
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
    fx = _load("trn_inceptionv3_MSTRN.pt")
    m = OV3.build_package_model(P, fx).to(dev)
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 2048 and list(m.input_size) == fx["input_size"] == [299, 299]
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
# 3. every launch of the measured forwards against fp64
# ---------------------------------------------------------------------------------------------
def _audit_build(make, shape):
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    m = OV3.fan_in_scale_(make())
    OF.randomize_bn_(m, 1)
    m = m.eval().to(dev)
    # TRN's relation draws its frame tuples per forward: pin one draw so the audited and the captured forward match
    for mod in m.modules():
        if hasattr(mod, "sample_tuples"):
            np.random.seed(0)
            picks = mod.sample_tuples()
            mod.sample_tuples = functools.partial(lambda p: p, picks)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1000)).to(dev)
    return m, x


def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


AUDITS = [("inceptionv3", lambda: P.inceptionv3(pretrained=None), (256, 3, 299, 299)),
          ("trn_inceptionv3_MSTRN", lambda: P.TRN(10, num_segments=8, arch="inceptionv3", consensus="MSTRN", pretrained=None,
                                                  **TRN_KW), (16, 8, 3, 299, 299))]


@pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV), reason="a dispatch override is set in the environment")
@pytest.mark.timeout(1800, method="thread")
@pytest.mark.parametrize("name,make,shape", AUDITS, ids=[a[0] for a in AUDITS])
def test_forward_every_launch_against_fp64(name, make, shape):
    m, x = _audit_build(make, shape)
    t0 = time.time()
    rep = audit(lambda: m(x))
    seconds = time.time() - t0
    _report("%s_B%d" % (name, shape[0]), rep, seconds)
    _assert_clean(name, rep)
    entries = {r["entry"] for r in rep.rows}
    assert not any("concat" in e or "copy" in e for e in entries), entries
    want = rep.output.clone()
    rep = None
    # launches per block, on a second forward (the audited one also packed the filters)
    real, per_block = engine._inception_block_body, []

    @functools.wraps(real)
    def counted(block, a, out=None):
        c0 = _lib.launch_count()
        y = real(block, a, out)
        per_block.append((type(block).kind, _lib.launch_count() - c0))
        return y
    engine._inception_block_body = counted
    try:
        with torch.no_grad():
            again = m(x)
        torch.cuda.synchronize()
    finally:
        engine._inception_block_body = real
    assert torch.equal(_bits(again), _bits(want)), "a second eager forward differs from the audited one"
    assert [k for k, _ in per_block] == ["InceptionA"] * 3 + ["InceptionB"] + ["InceptionC"] * 4 + ["InceptionD"] + ["InceptionE"] * 2
    assert all(n == LAUNCHES[k] for k, n in per_block), per_block
    graphed = GraphedForward(m, x, warmup=1)
    got = graphed()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "the CUDA-graph replay differs from the audited eager forward"


# ---------------------------------------------------------------------------------------------
# 4. head and input size
# ---------------------------------------------------------------------------------------------
def test_trainable_last_linear_on_frozen_trunk(model):
    head = torch.nn.Linear(2048, 7).to(dev)
    old = model.last_linear
    model.last_linear = head
    try:
        x = torch.rand((2, 3, 299, 299), generator=torch.Generator().manual_seed(4)).to(dev)
        model(x).square().sum().backward()
        assert head.weight.grad is not None and float(head.weight.grad.abs().sum()) > 0
        assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith("last_linear"))
        # the gradient the other 2-D families give: that of the head on the fp32 pooled features
        with torch.no_grad():
            pooled = model.features(x).mean((2, 3))
        ref = torch.nn.Linear(2048, 7).to(dev)
        ref.load_state_dict(head.state_dict())
        ref(pooled).square().sum().backward()
        err = (head.weight.grad - ref.weight.grad).abs().max().item() / ref.weight.grad.abs().max().item()
        assert err <= 1e-2, "head gradient rel err %.3e" % err
    finally:
        model.last_linear = old


def test_user_swapped_head_gets_fp32_pooled_features(model):
    old = model.last_linear
    model.last_linear = P.Identity()
    try:
        x = torch.rand((2, 3, 299, 299), generator=torch.Generator().manual_seed(5)).to(dev)
        with torch.no_grad():
            pooled = model(x)
            feats = model.features(x)
        assert pooled.dtype == torch.float32 and tuple(pooled.shape) == (2, 2048)
        err = (pooled - feats.mean((2, 3))).abs().max().item() / feats.abs().max().item()
        assert err <= 1e-3, err
    finally:
        model.last_linear = old


@pytest.mark.parametrize("hw", [224, 320])
def test_input_other_than_299_is_refused(model, hw):
    x = torch.rand((1, 3, hw, hw), device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match="299x299"):
        model(x)
