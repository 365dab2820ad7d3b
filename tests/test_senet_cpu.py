"""CPU: the SENet parameter containers against the reference, as recorded in the fixtures (tests/golden/se_*_b2_224.pt, written
by oracle/make_golden_senet.py from the unmodified reference): state_dict keys, shapes and order, a seeded init bit-identical to
the reference's, the registry rows; and the scope (no senet154, TRN fine-tuning on an SENet backbone refused)."""
import os

import pytest
import torch

import pretorched_x_b200 as P
from oracle import functional as OF

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ["se_resnet50_b2_224.pt", "se_resnext50_32x4d_b2_224.pt"]


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("fname", FIXTURES)
def test_state_dict_layout_and_seeded_init_match_reference(fname):
    fx = _load(fname)
    torch.manual_seed(fx["seeds"]["init"])
    model = P.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])


def test_pretrained_settings_rows_match_reference():
    fx = _load(FIXTURES[0])
    for name, rows in fx["settings"].items():
        if name == "senet154":
            assert name not in P.pretrained_settings
            continue
        assert P.pretrained_settings[name] == rows
        assert name in P.model_names


def test_senet154_not_offered():
    assert "senet154" not in P.__dict__
    from pretorched_x_b200.models import senet as PS
    with pytest.raises(NotImplementedError, match="senet154"):
        PS.SENet(PS.SEResNeXtBottleneck, [3, 8, 36, 3], groups=64, reduction=16)


@pytest.mark.parametrize("arch", ["se_resnext50_32x4d", "se_resnet50"])
def test_trn_on_senet_builds_and_refuses_fine_tune(arch):
    m = P.TRN(10, num_segments=4, arch=arch, consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128, video_feature_dim=64)
    assert m.frame_feature_dim == 2048
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)
