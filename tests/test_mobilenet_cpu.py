"""CPU: MobileNetV2 (pretorched/models/mobilenet.py) -- the parameter container against the reference's fixtures, the oracle
restatement against the reference's outputs, the registry rows, and the argument checks of the depthwise entry points.
No compute call reaches a GPU."""
import ctypes
import glob
import os

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib
from oracle import functional as OF
from oracle import mobilenet as OM

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIX = sorted(glob.glob(os.path.join(GOLDEN, "mobilenetv2_*.pt")))
TRN_FIX = os.path.join(GOLDEN, "trn_mobilenetv2_TRN.pt")


def _load(path):
    return torch.load(path, weights_only=False)


def test_fixtures_present():
    assert len(FIX) == 2 and os.path.exists(TRN_FIX)
    assert {_load(p)["kind"] for p in FIX} == {"mobilenetv2"} and _load(TRN_FIX)["kind"] == "trn_mobilenetv2"


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-3] for p in FIX])
def test_state_dict_layout_and_seeded_init_match_reference(path):
    fx = _load(path)
    torch.manual_seed(fx["seeds"]["init"])
    m = P.mobilenetv2(pretrained=None, **fx["kwargs"])
    sd = m.state_dict()
    assert list(sd) == fx["keys"] and len(sd) == fx["n_state"]
    assert list(sd)[:2] == ["features.0.0.weight", "features.0.1.weight"] and list(sd)[-1] == "last_linear.bias"
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert isinstance(m.features, torch.nn.Sequential) and len(m.features) == 19
    cond = OM.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(cond.state_dict()), fx["weight_digest"])


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-3] for p in FIX])
def test_oracle_reproduces_reference_outputs(path):
    fx = _load(path)
    sd = OM.build_package_model(P, fx).state_dict()
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        logits = OM.forward(x, sd, stages)
    scale = fx["logits"].abs().max().item()
    assert (logits - fx["logits"]).abs().max().item() <= 1e-5 * scale
    for name, ref in fx["stages"].items():
        if name == "logits":
            continue
        got = stages[name].reshape(-1)[::ref["step"]][:ref["sample"].numel()]
        assert tuple(stages[name].shape) == tuple(ref["shape"])
        assert (got - ref["sample"]).abs().max().item() <= 1e-5 * max(ref["absmax"], 1e-12), name


def test_trn_oracle_reproduces_reference_outputs():
    fx = _load(TRN_FIX)
    m = OM.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    st = {}
    with torch.no_grad():
        logits = OM.trn_forward(x, m.state_dict(), fx["segments"], st)
    assert (logits - fx["logits"]).abs().max().item() <= 1e-5 * fx["logits"].abs().max().item()
    assert (st["features"] - fx["features"]).abs().max().item() <= 1e-5 * fx["features"].abs().max().item()


def test_registry_and_trn_backbone():
    assert "mobilenetv2" in P.pretrained_settings and "mobilenetv2" in P.model_names
    row = P.pretrained_settings["mobilenetv2"]["imagenet"]
    assert row["input_size"] == [3, 224, 224] and row["num_classes"] == 1000
    assert P.__dict__["mobilenetv2"] is P.models.mobilenet.mobilenetv2
    t = P.trn(arch="mobilenetv2", pretrained=None)
    assert isinstance(t.base_model, P.models.mobilenet.MobileNetV2)
    assert t.frame_feature_dim == 1280 and t.input_size == [224, 224] and t.mean == row["mean"]


@pytest.mark.parametrize("width_mult", [0.5, 0.75, 1.4])
def test_width_mult_needs_multiples_of_8(width_mult):
    with pytest.raises(NotImplementedError, match="multiple of 8"):
        P.models.mobilenet.MobileNetV2(width_mult=width_mult)


def test_width_mult_with_multiples_of_8_constructs():
    m = P.models.mobilenet.MobileNetV2(num_classes=10, width_mult=2.0)
    assert m.last_linear.in_features == 2560


def test_forward_in_train_mode_raises():
    m = P.mobilenetv2(num_classes=10, pretrained=None)
    m.train()
    with pytest.raises(RuntimeError, match="inference-only"):
        m(torch.zeros(1, 3, 32, 32))
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 32, 32))


def test_depthwise_entry_points_validate_arguments():
    lib = _lib.load()
    buf = ctypes.c_void_p(4096)          # never dereferenced: every call below fails its argument checks first

    def dw(C=32, ld=32, stride=1, N=1, H=8, W=8, null=False):
        x = ctypes.c_void_p(0) if null else buf
        return lib.b2_dwconv3x3_ndhwc(x, buf, buf, buf, buf, N, H, W, C, ld, stride, 1, 1, None)

    for kwargs, msg in ((dict(null=True), b"null"), (dict(C=12, ld=16), b"multiple of 8"), (dict(ld=24), b">= C"),
                        (dict(ld=36), b"multiple of 8"), (dict(stride=3), b"stride"), (dict(N=0), b"empty"),
                        (dict(H=0), b"empty")):
        assert dw(**kwargs) == -1 and msg in lib.b2_last_error(), kwargs
    assert lib.b2_relu6_inplace_ndhwc(None, 4, 8, None) == -1
    assert lib.b2_relu6_inplace_ndhwc(buf, 4, 12, None) == -1
