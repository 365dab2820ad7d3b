"""CPU: Inception-v3 against the reference, as recorded in the fixtures (tests/golden/inceptionv3_b2_299.pt and
trn_inceptionv3_MSTRN.pt, written by oracle/make_golden_inceptionv3.py from the unmodified reference): state_dict keys, shapes and
order, a seeded init bit-identical to the reference's, the registry row, the ignored ``num_classes`` under ``pretrained=None``,
checkpoints in torchvision's and in the reference's layout through the factory, the oracle restatement against the reference's
features, stages and logits, TRN on Inception-v3 (its dims, policies, the fine_tune refusal), and the block table: every unit
of each torchvision block mapped exactly once and in torchvision's concatenation order, and the Inception-v4 /
Inception-ResNet-v2 rows unchanged (no GPU needed)."""
import os

import pytest
import torch
import torchvision.models.inception as tvinception

import pretorched_x_b200 as P
from pretorched_x_b200.models import inception as MI
from oracle import functional as OF
from oracle import inceptionv3 as OV3
from oracle.make_golden import sample_of

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
N_STATE, N_PARAMS = 580, 27161264


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_state_dict_layout_and_seeded_init_match_reference():
    fx = _load("inceptionv3_b2_299.pt")
    torch.manual_seed(fx["seeds"]["init"])
    model = P.inceptionv3(pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == N_STATE == fx["n_state"] and sum(p.numel() for p in model.parameters()) == N_PARAMS
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert list(sd)[-2:] == ["last_linear.weight", "last_linear.bias"] and not hasattr(model, "fc")
    assert "AuxLogits.fc.weight" in sd and model.transform_input is False


def test_pretrained_none_ignores_num_classes():
    """torchvision_models.py:383 builds ``inception_v3(pretrained=False)`` without passing num_classes on."""
    fx = _load("inceptionv3_b2_299.pt")
    model = P.inceptionv3(num_classes=10, pretrained=None)
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == [tuple(kv) for kv in fx["keys_num_classes_10"]]
    assert model.last_linear.out_features == 1000


def test_pretrained_settings_row_matches_reference():
    fx = _load("inceptionv3_b2_299.pt")
    assert P.pretrained_settings["inceptionv3"] == fx["settings"]["inceptionv3"]
    assert "inceptionv3" in P.model_names and P.__dict__["inceptionv3"] is P.inceptionv3


def _source():
    torch.manual_seed(5)
    src = P.inceptionv3(pretrained=None)
    OF.randomize_bn_(src, 6)
    return src


def _through_factory(monkeypatch, ckpt, **kw):
    import torch.utils.model_zoo as model_zoo
    seen = []
    monkeypatch.setattr(model_zoo, "load_url", lambda url: seen.append(url) or dict(ckpt))
    torch.manual_seed(7)
    m = P.inceptionv3(**kw)
    return m, seen


@pytest.mark.parametrize("layout", ["torchvision", "reference"])
def test_checkpoint_loads_through_the_factory(monkeypatch, layout):
    """torchvision's zoo checkpoint names the head ``fc`` (and has ``AuxLogits.fc``); the reference's own state_dict names it
    ``last_linear``.  Both load; only the top-level ``fc.`` prefix is renamed."""
    src = _source()
    want = src.state_dict()
    if layout == "torchvision":
        ckpt = {("fc." + k[len("last_linear."):] if k.startswith("last_linear.") else k): v.clone() for k, v in want.items()}
        assert "fc.weight" in ckpt and "AuxLogits.fc.weight" in ckpt and "last_linear.weight" not in ckpt
    else:
        ckpt = {k: v.clone() for k, v in want.items()}
    m, seen = _through_factory(monkeypatch, ckpt)
    assert seen == ["https://download.pytorch.org/models/inception_v3_google-1a9a5a14.pth"]
    got = m.state_dict()
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
        ("RGB", [0, 1], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5], [3, 299, 299])


def test_imagenet_asserts_1000_classes(monkeypatch):
    with pytest.raises(AssertionError, match="num_classes should be 1000"):
        _through_factory(monkeypatch, {}, num_classes=10, pretrained="imagenet")


def test_oracle_reproduces_reference_features_and_logits():
    fx = _load("inceptionv3_b2_299.pt")
    model = OV3.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OV3.features(x, sd, model, stages)
        logits = OV3.logits(feats, sd)
    assert tuple(feats.shape) == tuple(fx["features"]["shape"]) == (2, 2048, 8, 8)
    s, step = sample_of(feats)
    assert step == fx["features"]["step"] and torch.equal(s, fx["features"]["sample"])
    assert list(fx["stages"]) == OV3.STEM + OV3.BLOCKS
    for name, summ in fx["stages"].items():
        s, step = sample_of(stages[name])
        assert tuple(stages[name].shape) == tuple(summ["shape"]) and step == summ["step"] and torch.equal(s, summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


def test_trn_builds_and_refuses_fine_tune():
    fx = _load("trn_inceptionv3_MSTRN.pt")
    m = OV3.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 2048
    assert list(m.input_size) == fx["input_size"] == [299, 299] and m.crop_size == [299, 299]
    assert isinstance(m.base_model.last_linear, torch.nn.Dropout)
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)
    assert P.trn(num_classes=10, arch="inceptionv3", pretrained=None).frame_feature_dim == 2048


def _named(model, groups):
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in groups]


@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(pbn):
    fx = _load("trn_inceptionv3_MSTRN.pt")
    model = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    got = _named(model, model.get_optim_policies())
    assert got == fx["policies"][pbn]
    if pbn:
        assert got[4]["params"] == ["base_model.Conv2d_1a_3x3.bn.weight", "base_model.Conv2d_1a_3x3.bn.bias"]


def test_training_mode_is_refused():
    m = P.inceptionv3(pretrained=None)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 299, 299))


# ---------------------------------------------------------------------------------------------
# the block table
# ---------------------------------------------------------------------------------------------
# block -> input map at 299^2
V3_BLOCKS = {"Mixed_5b": 35, "Mixed_5c": 35, "Mixed_5d": 35, "Mixed_6a": 35, "Mixed_6b": 17, "Mixed_6c": 17, "Mixed_6d": 17,
             "Mixed_6e": 17, "Mixed_7a": 17, "Mixed_7b": 8, "Mixed_7c": 8}


def _row_units(row):
    units = []
    for br in row:
        if br[0] == "fork":
            units += br[1] + list(br[2])
        elif br[0] != "max":
            units += br[1]
    return units


@pytest.mark.parametrize("name", list(V3_BLOCKS))
def test_v3_rows_map_every_unit_once_in_torchvision_order(name):
    """Every BasicConv2d of the block appears exactly once in its row, and the row, walked by the oracle, is torchvision's own
    block forward bit for bit in fp64 (branch order, fork order, the counted padding of the average pool)."""
    torch.manual_seed(0)
    model = OV3.fan_in_scale_(P.inceptionv3(pretrained=None))
    OF.randomize_bn_(model, 2)
    model = model.eval().double()
    blk = model.get_submodule(name)
    assert isinstance(blk, getattr(tvinception, type(blk).kind)) and type(blk).kind in MI.V3_KINDS
    row = MI.BRANCHES[type(blk).kind]
    units = _row_units(row)
    assert sorted(units) == sorted(n for n, _ in blk.named_children()) and len(units) == len(set(units))
    assert all(br[2] is True for br in row if br[0] == "avg")
    cin = [mod for mod in blk.modules() if isinstance(mod, torch.nn.Conv2d)][0].in_channels
    H = V3_BLOCKS[name]
    x = torch.rand((1, cin, H, H), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    sd = {k: v.detach() for k, v in model.state_dict().items()}
    with torch.no_grad():
        want = getattr(tvinception, type(blk).kind).forward(blk, x)       # torchvision's own block forward
        got = OV3.block(x, sd, blk, name + ".")
    assert torch.equal(got, want)


# The Inception-v4 / Inception-ResNet-v2 rows as they were before the Inception-v3 rows were added, with the average pools'
# count_include_pad (False: AvgPool2d(3, 1, 1, count_include_pad=False)) now stated in the row.
V4_ROWS = {
    'Mixed_3a': [('max', 'maxpool'), ('chain', ['conv'])],
    'Mixed_4a': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2', 'branch1.3'])],
    'Mixed_5a': [('chain', ['conv']), ('max', 'maxpool')],
    'Inception_A': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2']),
                    ('avg', ['branch3.1'], False)],
    'Reduction_A': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']), ('max', 'branch2')],
    'Inception_B': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']),
                    ('chain', ['branch2.0', 'branch2.1', 'branch2.2', 'branch2.3', 'branch2.4']), ('avg', ['branch3.1'], False)],
    'Reduction_B': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2', 'branch1.3']),
                    ('max', 'branch2')],
    'Inception_C': [('chain', ['branch0']), ('fork', ['branch1_0'], ('branch1_1a', 'branch1_1b')),
                    ('fork', ['branch2_0', 'branch2_1', 'branch2_2'], ('branch2_3a', 'branch2_3b')), ('avg', ['branch3.1'], False)],
    'Mixed_5b': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2']),
                 ('avg', ['branch3.1'], False)],
    'Block35': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2'])],
    'Mixed_6a': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']), ('max', 'branch2')],
    'Block17': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2'])],
    'Mixed_7a': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1']),
                 ('chain', ['branch2.0', 'branch2.1', 'branch2.2']), ('max', 'branch3')],
    'Block8': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2'])],
}


def test_v4_and_inception_resnet_v2_rows_are_unchanged():
    assert {k: v for k, v in MI.BRANCHES.items() if k not in MI.V3_KINDS} == V4_ROWS
    assert set(MI.BRANCHES) == set(V4_ROWS) | set(MI.V3_KINDS) and MI.RESIDUAL == ('Block35', 'Block17', 'Block8')
    for kind in V4_ROWS:
        assert getattr(MI, kind).kind == kind
