"""GPU (-m gpu): PNASNet-5-Large on the engine.

1. The forward against the reference's fixture at 331^2 (tests/golden/pnasnet5large_b2_331.pt): conv_0's and every cell's output
   within 1e-2 and the logits within 5e-3 of max |ref|, equal arg-max, ``features`` equal to the staged trunk, and a CUDA-graph
   replay bit-identical to the eager forward.
2. TRN-MSTRN on PNASNet-5-Large against its fixture (4320-d frame features).
3. Every library launch of the forward at 256 images (331^2) and of TRN-MSTRN at 16 videos x 8 segments held element by element to
   its fp64 bound (tests/pnasnet_audit.py), the launches per forward pinned, and a CUDA-graph replay bit-identical to the audited
   eager output.
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
from pretorched_x_b200.models.pnasnet import CELLS
from oracle import functional as OF
from oracle import pnasnet as OPn
from oracle.make_golden import sample_of
from tests.conftest import has_h100
from tests.pnasnet_audit import audit
from tests.test_gpu_model_audit import KNOB_ENV, _assert_clean, _report

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _logical(act, layout):
    """An Act stored in ``layout`` (engine.py's PNASNet channel layouts) as fp32 NCHW of its logical channels."""
    seg, pitch, n = layout
    t = ops.to_ncdhw(act).squeeze(2)
    return torch.cat([t[:, j * pitch:j * pitch + seg] for j in range(n)], 1)


def test_forward_stages_match_reference_fixture():
    fx = _load("pnasnet5large_b2_331.pt")
    model = OPn.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        stages = engine.pnasnet_stages(model, ops.from_ncdhw(x, pitch=8))
        logits = model.logits(stages[-1][1])
        whole = model(x)
        feats = model.features(x)
    torch.cuda.synchronize()
    assert [s[0] for s in stages] == list(fx["stages"]) == OPn.STAGES
    for name, act, layout in stages:
        summ = fx["stages"][name]
        t = _logical(act, layout).cpu()
        assert tuple(t.shape) == tuple(summ["shape"]), name
        if layout[1] != layout[0]:
            assert torch.all(ops.to_ncdhw(act).squeeze(2)[:, layout[0]:layout[1]] == 0), "%s: pad columns not zero" % name
        s, step = sample_of(t)
        assert step == summ["step"]
        err = (s.double() - summ["sample"].double()).abs().max().item() / summ["absmax"]
        print("[pnasnet] %-12s rel err %.3e" % (name, err))
        assert err <= 1e-2, "%s: rel err %.3e" % (name, err)
    assert torch.equal(feats, ops.to_ncdhw(stages[-1][1]).squeeze(2))
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    print("[pnasnet] logits rel err %.3e" % err)
    assert err <= 5e-3, "logits: rel err %.3e" % err
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(model, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_input_size_is_enforced_on_the_gpu():
    model = P.pnasnet5large(pretrained=None).eval().to(dev)
    with pytest.raises(ValueError, match="331x331"):
        model(torch.zeros(1, 3, 299, 299, device=dev))


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_pnasnet5large_MSTRN.pt")
    model = OPn.build_package_model(P, fx).to(dev)
    assert model.frame_feature_dim == 4320
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
# every launch at the measured batch against fp64
# ---------------------------------------------------------------------------------------------
def _bits(t):
    return t.reshape(-1).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _cell_launches(reduction, factorized, stem0=False):
    """A cell once its filters are packed: x_left (ReluConvBn 1, FactorizedReduction 3: two gathers and one GEMM) and x_right (1);
    six separable branches of 4 launches (two depthwise passes, two GEMMs); the max-pools of combinations 0, 1 and 3; five copies
    into the cell output; comb_iter_4_right's gather and GEMM in a reduction cell.  CellStem0: x_right, and comb_iter_0_right's
    GEMM after its pool."""
    if stem0:
        return 1 + 6 * 4 + 3 + 1 + 5 + 2
    return (3 if factorized else 1) + 1 + 6 * 4 + 3 + 5 + (2 if reduction else 0)


# the input layout pass, conv_0, the cells, the head's ReLU + mean and last_linear
EXPECTED_LAUNCHES = 2 + _cell_launches(True, False, stem0=True) + sum(_cell_launches(c[5], c[7]) for c in CELLS) + 2
DEPTHWISE_LAUNCHES = 2 * 6 * 14


def _expected_launches(m):
    """TRN: the backbone without last_linear (a Dropout there), the cast of the frame features to fp16, per relation scale the tuple
    gather and two GEMMs, and the cast + GEMM of the TRN head."""
    if isinstance(m, P.TRN):
        return EXPECTED_LAUNCHES - 1 + 1 + 3 * len(m.temporal_relation.scales) + 2
    return EXPECTED_LAUNCHES


AUDITS = [("pnasnet5large", functools.partial(P.pnasnet5large, pretrained=None), (256, 3, 331, 331)),
          ("trn_pnasnet5large_MSTRN", functools.partial(P.TRN, 10, num_segments=8, arch="pnasnet5large", consensus="MSTRN",
                                                        pretrained=None, **TRN_KW), (16, 8, 3, 331, 331))]


@pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV), reason="a dispatch override is set in the environment")
@pytest.mark.timeout(3000, method="thread")
@pytest.mark.parametrize("name,make,shape", AUDITS, ids=[a[0] for a in AUDITS])
def test_forward_every_launch_against_fp64(name, make, shape):
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    m = make()
    OPn.rescale_(m)
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
    assert sum(r["launches"] for r in rep.rows if r["entry"] == "dwconv_kxk_relu_in") == DEPTHWISE_LAUNCHES
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
