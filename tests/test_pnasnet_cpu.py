"""CPU: PNASNet-5-Large against the reference, as recorded in the fixtures (tests/golden/pnasnet5large_b2_331.pt and
trn_pnasnet5large_MSTRN.pt, written by oracle/make_golden_pnasnet.py from the unmodified reference): state_dict keys, shapes and
order, a seeded init bit-identical to the reference's, both registry rows, both checkpoint layouts through the factory, the oracle
against the reference's stages and logits, TRN on PNASNet (4320-d frame features, policies, the fine_tune refusal), the refusals,
the engine's channel layouts (the padded stem slices and their scattered filter rows, in fp64), the launch count the GPU test pins,
and the ``ops_pnasnet`` audit registration (no GPU needed)."""
import ast
import inspect
import os

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import engine, ops, ops_pnasnet
from pretorched_x_b200.models import pnasnet as MP
from oracle import functional as OF
from oracle import pnasnet as OPn
from oracle.make_golden import sample_of
from tests import model_audit as MA
from tests import pnasnet_audit as PA

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
N_STATE, N_PARAMS = 1380, 86057668
URL = 'http://data.lip6.fr/cadene/pretrainedmodels/pnasnet5large-bf079911.pth'


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_state_dict_layout_and_seeded_init_match_reference():
    fx = _load("pnasnet5large_b2_331.pt")
    torch.manual_seed(fx["seeds"]["init"])
    model = P.pnasnet5large(pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == N_STATE == fx["n_state"] and sum(p.numel() for p in model.parameters()) == N_PARAMS
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert all(m.eps == 0.001 for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d))


def test_pretrained_settings_rows_and_registry():
    fx = _load("pnasnet5large_b2_331.pt")
    assert P.pretrained_settings["pnasnet5large"] == fx["settings"]["pnasnet5large"]
    assert set(P.pretrained_settings["pnasnet5large"]) == {"imagenet", "imagenet+background"}
    assert P.__dict__["pnasnet5large"] is P.pnasnet5large and P.models.settings.model_names.count("pnasnet5large") == 1
    assert inspect.signature(P.pnasnet5large).parameters["pretrained"].default == "imagenet"
    assert P.pnasnet5large(num_classes=10, pretrained=None).last_linear.out_features == 10


@pytest.mark.parametrize("row", ["imagenet", "imagenet+background"])
def test_checkpoint_loads_through_the_factory(monkeypatch, row):
    """Both rows load the same 1001-class checkpoint; 'imagenet' drops the background row of last_linear."""
    import torch.utils.model_zoo as model_zoo
    torch.manual_seed(5)
    src = P.pnasnet5large(num_classes=1001, pretrained=None)
    OF.randomize_bn_(src, 6)
    want = src.state_dict()
    seen = []
    monkeypatch.setattr(model_zoo, "load_url", lambda url: seen.append(url) or {k: v.clone() for k, v in want.items()})
    m = P.pnasnet5large(num_classes=1000 if row == "imagenet" else 1001, pretrained=row)
    assert seen == [URL]
    got = m.state_dict()
    assert list(got) == list(want)
    for k in want:
        w = want[k][1:] if row == "imagenet" and k.startswith("last_linear.") else want[k]
        assert torch.equal(got[k], w), k
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
        ("RGB", [0, 1], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5], [3, 331, 331])
    with pytest.raises(AssertionError, match="num_classes should be"):
        P.pnasnet5large(num_classes=10, pretrained=row)


def test_oracle_reproduces_reference_stages_and_logits():
    fx = _load("pnasnet5large_b2_331.pt")
    model = OPn.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OPn.features(x, sd, stages)
        logits = OPn.logits(feats, sd)
    assert list(fx["stages"]) == OPn.STAGES
    assert [fx["stages"][n]["shape"][2] for n in OPn.STAGES] == [165, 83, 42] + [42] * 4 + [21] * 4 + [11] * 4
    for name, summ in fx["stages"].items():
        s, step = sample_of(stages[name])
        assert tuple(stages[name].shape) == tuple(summ["shape"]) and step == summ["step"] and torch.equal(s, summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


def test_trn_builds_with_4320d_frame_features_and_refuses_fine_tune():
    fx = _load("trn_pnasnet5large_MSTRN.pt")
    m = OPn.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 4320
    assert list(m.input_size) == fx["input_size"] == [331, 331]
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)


@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(pbn):
    fx = _load("trn_pnasnet5large_MSTRN.pt")
    model = P.TRN(10, num_segments=fx["segments"], arch="pnasnet5large", consensus="MSTRN", pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    names = {id(p): n for n, p in model.named_parameters()}
    got = [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
           for g in model.get_optim_policies()]
    assert got == fx["policies"][pbn]


def test_training_mode_input_size_and_parts_are_refused():
    m = P.pnasnet5large(pretrained=None)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 331, 331))
    m.eval()
    a = ops.Act(torch.zeros((299 * 299, 8), dtype=torch.float16), 1, 1, 299, 299, 3)
    with pytest.raises(ValueError, match="331x331"):
        m.features_act(a)
    with pytest.raises(ValueError, match="11x11"):
        engine.run_pnasnet_head(m, ops.Act(torch.zeros((9 * 9, 4320), dtype=torch.float16), 1, 1, 9, 9, 4320))
    with pytest.raises(NotImplementedError, match="inside its PNASNet cell"):
        m.cell_0(torch.zeros(1, 270, 42, 42), torch.zeros(1, 540, 42, 42))


def test_padded_layout_scatter_matches_the_dense_product_in_fp64():
    """A stem cell's output stores five 54-wide combinations at pitch 56; a filter packed for it by engine._scatter has zero columns
    at the pad positions, so its product with the padded tensor equals the reference's product with the dense one."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(7, 270, generator=g, dtype=torch.float64)
    w = torch.randn(216, 270, generator=g, dtype=torch.float64)
    layout = (54, 56, 5)
    xp = torch.zeros(7, 280, dtype=torch.float64)
    for j in range(5):
        xp[:, 56 * j:56 * j + 54] = x[:, 54 * j:54 * (j + 1)]
    wp = engine._scatter(w, layout, 280)
    assert torch.equal(wp[:, 54:56], torch.zeros(216, 2, dtype=torch.float64))
    assert torch.allclose(xp @ wp.t(), x @ w.t(), rtol=1e-13, atol=1e-12)
    with pytest.raises(ValueError, match="does not read the layout"):
        engine._scatter(w, (54, 56, 5), 272)


def test_every_launching_entry_of_ops_pnasnet_is_audited():
    """Every function of pretorched_x_b200/ops_pnasnet.py whose body calls ``_lib.check(`` is in tests/pnasnet_audit.py's table, with
    a check and exactly the parameters of its signature; nothing of it is also an entry of ``ops``."""
    with open(ops_pnasnet.__file__) as f:
        tree = ast.parse(f.read())
    launching = {node.name for node in ast.walk(tree) if isinstance(node, ast.FunctionDef)
                 and any(isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "check"
                         and isinstance(c.func.value, ast.Name) and c.func.value.id == "_lib" for c in ast.walk(node))}
    assert launching == set(PA.ENTRIES) == set(PA.CHECKS) == {"dwconv_kxk_relu_in", "gather_offset"}
    for name, params in PA.ENTRIES.items():
        assert tuple(inspect.signature(getattr(ops_pnasnet, name)).parameters) == params
        assert not hasattr(ops, name) and name not in MA.KNOWN


def test_cell_table_follows_the_reference():
    m = P.pnasnet5large(pretrained=None)
    assert [n for n, _ in m.named_children()] == ["conv_0", "cell_stem_0"] + [c[0] for c in MP.CELLS] + \
        ["relu", "avg_pool", "dropout", "last_linear"]
    for name, il, ol, ir, orr, red, zp, match in MP.CELLS:
        cell = getattr(m, name)
        assert isinstance(cell.conv_prev_1x1, MP.FactorizedReduction) == match
        assert (cell.comb_iter_4_right is not None) == red
        assert (cell.comb_iter_0_left.zero_pad is not None) == zp
