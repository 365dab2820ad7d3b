"""GPU (-m gpu): ResNeXt-3D (resnext3D.py; exported by pretorched/__init__.py:66-72) against the outputs of the unmodified
reference (tests/golden/resnext3d*.pt).  The grouped 3x3x3 convolution runs as its block-diagonal dense filter on the same
slab kernel as the ResNet-3D layers.  Tolerances as for the other networks: per-stage samples <= 1e-2 of the tensor's
max, logits <= 5e-3, arg-max must agree."""
import glob
import os

import pytest
import torch

from oracle import functional as OF
import pretorched_x_b200 as P
from pretorched_x_b200 import engine, ops

pytestmark = pytest.mark.gpu
FIX = [g for g in sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "resnext3d*.pt")))]


@pytest.mark.timeout(240, method="thread")        # first hardware run of this family: a stuck kernel must fail, not hang the tier
@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-3] for p in FIX])
def test_resnext3d_forward_matches_reference_golden(path):
    assert torch.cuda.is_available(), "GPU tests need an H100"
    dev = torch.device("cuda:0")
    fx = torch.load(path, weights_only=False)
    torch.manual_seed(fx["seeds"]["init"])
    m = getattr(P, fx["arch"])(**fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    m = m.eval().to(dev)
    assert OF.digests_match(OF.state_digest({k: v.cpu() for k, v in m.state_dict().items()}), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        a = engine.run_stem(m, x)
        outs = {"maxpool": a}
        for ln in ("layer1", "layer2", "layer3", "layer4"):
            for blk in getattr(m, ln):
                a = engine.run_block(blk, a)
            outs[ln] = a
        logits = m.logits(a)
        assert torch.equal(m(x), logits)                       # public API path == staged walk
    for name, ref in fx["stages"].items():
        if name == "logits":
            continue
        t = ops.to_ncdhw(outs[name]).reshape(-1)[::ref["step"]][:ref["sample"].numel()].cpu().double()
        err = ((t - ref["sample"].double()).abs() / max(ref["absmax"], 1e-12)).max().item()
        assert err <= 1e-2, (name, err)
    err = ((logits.cpu().double() - fx["logits"].double()).abs() / fx["logits"].abs().max().item()).max().item()
    assert err <= 5e-3, err
    assert torch.equal(logits.argmax(1).cpu(), fx["logits"].argmax(1))
    assert m.last_linear is m.fc and tuple(m.features(x).shape) == fx["stages"]["layer4"]["shape"]
