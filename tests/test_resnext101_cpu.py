"""CPU: the ResNeXt-101 parameter containers against the reference, as recorded in the fixtures (tests/golden/resnext101_*_b2_224.pt
and trn_resnext101_32x4d_MSTRN.pt, written by oracle/make_golden_resnext.py from the unmodified reference): state_dict keys, shapes
and order, a seeded init bit-identical to the reference's, the registry rows, checkpoint loading, per-instance weights, the
grouped-kernel route of every conv2, the fine-tuning split and TRN's optimizer-policy groups."""
import os

import pytest
import torch

import pretorched_x_b200 as P
from oracle import functional as OF
from oracle import reference_loader as RL
from oracle import resnext as OX
from pretorched_x_b200 import engine
from pretorched_x_b200.models import resnext as PX

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = ["resnext101_32x4d_b2_224.pt", "resnext101_64x4d_b2_224.pt"]
PARAMS = {"resnext101_32x4d": 44_177_704, "resnext101_64x4d": 83_455_272}


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("fname", FIXTURES)
def test_state_dict_layout_and_seeded_init_match_reference(fname):
    fx = _load(fname)
    torch.manual_seed(fx["seeds"]["init"])
    model = P.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == 626
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert sum(p.numel() for p in model.parameters()) == PARAMS[fx["arch"]]


@pytest.mark.parametrize("fname", FIXTURES)
def test_restatement_of_seeded_model_gives_reference_logits(fname):
    """The package's seeded, BN-randomised weights through the CPU restatement give the reference's logits."""
    fx = _load(fname)
    model = OX.build_package_model(P, fx)
    with torch.no_grad():
        out = OX.forward(OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]), model.state_dict(), fx["arch"])
    torch.testing.assert_close(out, fx["logits"], rtol=1e-4, atol=1e-5)


def test_pretrained_settings_rows_match_reference():
    fx = _load(FIXTURES[0])
    assert set(fx["settings"]) == {"resnext101_32x4d", "resnext101_64x4d"}
    for name, rows in fx["settings"].items():
        assert P.pretrained_settings[name] == rows
        assert name in P.model_names
        assert P.__dict__[name].__name__ == name


@pytest.mark.parametrize("fname", FIXTURES)
def test_checkpoint_shaped_state_dict_loads(fname):
    """A state_dict with the reference's keys, order and shapes (what Cadene's checkpoints hold) loads strictly."""
    fx = _load(fname)
    g = torch.Generator().manual_seed(5)
    ckpt = {k: (torch.randn(shape, generator=g) if not k.endswith("num_batches_tracked") else torch.tensor(7)) for k, shape in fx["keys"]}
    model = P.__dict__[fx["arch"]](pretrained=None)
    model.load_state_dict(ckpt)
    for k, v in model.state_dict().items():
        assert torch.equal(v, ckpt[k]), k
    assert torch.equal(model.layer3[22].conv2.weight, ckpt["features.6.22.0.0.0.3.weight"])
    assert torch.equal(model.layer2[0].downsample[1].running_var, ckpt["features.5.0.0.1.1.running_var"])


@pytest.mark.skipif(not RL.available(), reason="reference tree not available")
def test_reference_state_dict_loads():
    pt = RL.load()
    ref = pt.models.resnext.resnext101_64x4d(num_classes=1000, pretrained=None)
    model = P.resnext101_64x4d(pretrained=None)
    model.load_state_dict(ref.state_dict())
    for (k, v), (k2, v2) in zip(model.state_dict().items(), ref.state_dict().items()):
        assert k == k2 and torch.equal(v, v2)


def test_instances_do_not_share_weights():
    a, b = P.resnext101_32x4d(pretrained=None), P.resnext101_32x4d(pretrained=None)
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert all(pa[k].data_ptr() != pb[k].data_ptr() for k in pa)
    assert not torch.equal(pa["features.4.0.0.0.0.0.weight"], pb["features.4.0.0.0.0.0.weight"])
    with torch.no_grad():
        pa["features.0.weight"].zero_()
    assert pb["features.0.weight"].abs().sum() > 0


@pytest.mark.parametrize("arch,groups", [("resnext101_32x4d", 32), ("resnext101_64x4d", 64)])
def test_block_views_and_grouped_route(arch, groups):
    """Every conv2 is inside the group-aware kernel's contract (4 / 8 / 16 / 32 channels per group, stride 1 or 2); the views
    are the children the reference's keys name."""
    model = P.__dict__[arch](pretrained=None)
    assert model.conv1 is model.features[0] and model.maxpool is model.features[3]
    n = 0
    for i in range(1, 5):
        for b, blk in enumerate(getattr(model, "layer%d" % i)):
            assert isinstance(blk, PX.ResNeXt101Bottleneck)
            assert blk.conv2 is blk[0][0][0][3] and blk.bn3 is blk[0][0][2]
            assert blk.conv2.groups == groups and blk.conv2.weight.shape[1] == 4 << (i - 1)
            assert blk.conv2.stride == ((2, 2) if b == 0 and i > 1 else (1, 1))
            assert engine.grouped_route(blk.conv2)
            assert not engine.grouped_route(blk.conv1) and not engine.grouped_route(blk.conv3)
            assert (blk.downsample is not None) == (b == 0)
            n += 1
    assert n == 33


def test_fine_tune_sets_requires_grad_per_stage():
    """Stage k is features.{3 + k}; k = 5 trains last_linear only; every block of the trained stages passes the engine's check."""
    model = P.resnext101_32x4d(pretrained=None).eval()
    for k in (1, 2, 3, 4, 5):
        model.fine_tune(k)
        trained = tuple("features.%d." % (3 + i) for i in range(k, 5)) + ("last_linear.",)
        for n, p in model.named_parameters():
            assert p.requires_grad == n.startswith(trained), (k, n)
        assert model.ft_begin_index == k
    with pytest.raises(NotImplementedError, match="7x7 convolution"):
        model.fine_tune(0)
    with pytest.raises(ValueError):
        model.fine_tune(6)


def test_resnext3d_blocks_are_still_refused():
    """The new grouped kernels cover in-plane (1x3x3) filters only: ResNeXt-3D's 3x3x3 grouped blocks stay refused."""
    from pretorched_x_b200.models import resnext3d
    blk = next(m for m in P.resnext3d50(num_classes=10).modules() if isinstance(m, resnext3d.ResNeXtBottleneck))
    with pytest.raises(NotImplementedError, match="fine-tuning backward covers"):
        engine.check_trainable_block(blk)


def test_trn_builds_and_policies_match_reference():
    fx = _load("trn_resnext101_32x4d_MSTRN.pt")
    torch.manual_seed(fx["seeds"]["init"])
    m = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    assert m.frame_feature_dim == 2048
    assert m.input_size == [224, 224]
    names = {id(p): n for n, p in m.named_parameters()}
    got = [dict(name=g["name"], lr_mult=g["lr_mult"], decay_mult=g["decay_mult"], params=[names[id(p)] for p in g["params"]])
           for g in m.get_optim_policies()]
    assert got == fx["policies"]
    assert len(m.state_dict()) == fx["n_state"]
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    m.fine_tune(4)
    assert {n.split(".")[0] for n, p in m.named_parameters() if p.requires_grad} == {"base_model", "temporal_relation", "last_linear"}
    assert not any(p.requires_grad for n, p in m.named_parameters() if n.startswith("base_model.features.6."))
